"""What stage A of the encoder works on, restated with numpy for the autocorrelation tests: the signals and their wasted bits
(stream_encoder.c:3777-3867, 5077-5099), the section list of apply_apodization_ (:4318-4392), and blocks that reach the
edges of both."""
import numpy as np

import oraclelib
import signals as sigs

SUBDIVIDE_TUKEY = 1
MAX_LPC_ORDER = 32


def apod(cls, t, p=0.0, start=0.0, end=0.0, parts=0):
    a = cls()
    a.type, a.p, a.start, a.end, a.parts = t, p, start, end, parts
    return a


# one window of every apodization type (oracle numbering, flac_oracle.h)
WINDOW_TYPES = [apod(oraclelib.Apod, 0, 0.5), apod(oraclelib.Apod, 0, 0.0), apod(oraclelib.Apod, 0, 1.0)] + \
    [apod(oraclelib.Apod, t) for t in (2, 3, 4, 5, 6, 7, 9, 10, 11, 12, 13, 14, 17)] + \
    [apod(oraclelib.Apod, 8, 0.2), apod(oraclelib.Apod, 15, 0.2, 0.1, 0.6), apod(oraclelib.Apod, 16, 0.2, 0.3, 0.7)]


def sections(cfg, bs):
    """(apodization, partial, data_len, part_size, data_shift) of every autocorrelation apply_apodization_ computes for a
    block of bs samples, in its order: each apodization's whole window, then subdivide_tukey's partial windows by depth."""
    out = []
    for a in range(cfg.num_apodizations):
        ap = cfg.apodizations[a]
        out.append((a, 0, bs, 0, 0))
        if ap.type == SUBDIVIDE_TUKEY:
            for b in range(2, ap.parts + 1):
                if bs // b <= MAX_LPC_ORDER:  # :4349-4357
                    continue
                for part in range(2 if b == 2 else b):
                    out.append((a, 1, bs // b, bs // b // 2, (part * bs) // b))
    return out


def wasted_bits(sig):
    """get_wasted_bits_ of each row: trailing zero bits of the OR of its samples, 0 for a silent row."""
    o = np.bitwise_or.reduce(sig.astype(np.int64), axis=1)
    w = np.zeros(sig.shape[0], dtype=np.int64)
    for i, v in enumerate(o):
        while v and not (v >> w[i]) & 1:
            w[i] += 1
    return w


def signals(x, nb, bs, channels, bps, mid_side, loose):
    """(signals int64 [items, bs] before their wasted bits are shifted out, meta int32 [items, 2] (wasted bits, subframe bps;
    0, 0 for the pair a loose mid-side block does not code), active bool [items]), item = block * nsig + signal."""
    blk = np.asarray(x, dtype=np.int64).reshape(nb, bs, channels)
    rows = [blk[:, :, c] for c in range(channels)]
    active = [np.ones(nb, dtype=bool)] * channels
    if channels == 2 and mid_side:
        L, R = rows
        rows += [(L + R) >> 1, L - R]
        if loose:
            dl, dr = np.diff(L, axis=1), np.diff(R, axis=1)
            lr = (np.abs(dl) + np.abs(dr)).sum(axis=1)
            ms = (np.abs((dl + dr) >> 1) + np.abs(dl - dr)).sum(axis=1)
            indep = lr < ms
            active = [indep, indep, ~indep, ~indep]
        else:
            active = [np.ones(nb, dtype=bool)] * 4
    nsig = len(rows)
    sig = np.stack(rows, axis=1).reshape(nb * nsig, bs)
    act = np.stack(active, axis=1).reshape(nb * nsig)
    w = np.minimum(wasted_bits(sig), bps)
    side = np.zeros(nsig, dtype=np.int64)
    if nsig == 4:
        side[3] = 1
    meta = np.stack([w, bps - w + np.tile(side, nb)], axis=1)
    meta[~act] = 0
    return sig, meta.astype(np.int32), act


KINDS = ("music", "noise", "wasted", "silent", "mid_wasted", "dc", "negative_odd_sum")


def mixed_blocks(nb, bs, channels, bps, seed, kinds=KINDS):
    """int32 [nb * bs, channels]: block b is of kind kinds[b % len(kinds)] --
    music: music-like; noise: full-scale noise (24-bit: the side signal needs 25 bits, and (float)x rounds);
    wasted: channel c shifted left by 1 + (b + c) % 8 bits (at most bps - 2); silent: zeros; dc: a constant per channel;
    mid_wasted: odd multiples of 2^w on L (4k + 1) and R (4k + 3), so mid and side waste more bits than L and R;
    negative_odd_sum: L + R odd and negative, where mid = (L + R) >> 1 rounds toward minus infinity."""
    rng = np.random.default_rng(seed)
    lo, hi = -(1 << (bps - 1)), (1 << (bps - 1)) - 1
    music = sigs.music_like(nb * bs, channels, bps, 44100, seed=seed).astype(np.int64).reshape(nb, bs, channels)
    out = np.empty((nb, bs, channels), dtype=np.int64)
    wmax = max(1, min(8, bps - 3))
    for b in range(nb):
        kind = kinds[b % len(kinds)]
        if kind == "music":
            blk = music[b]
        elif kind == "noise":
            blk = rng.integers(lo, hi + 1, (bs, channels))
        elif kind == "wasted":
            blk = np.stack([rng.integers(lo >> w, (hi >> w) + 1, bs) << w for w in (1 + (b + c) % wmax for c in range(channels))], axis=1)
        elif kind == "silent":
            blk = np.zeros((bs, channels), dtype=np.int64)
        elif kind == "dc":
            blk = np.broadcast_to(rng.integers(lo, hi + 1, channels), (bs, channels))
        elif kind == "mid_wasted":
            w = 1 + b % wmax
            m = (1 << (bps - 1)) >> w
            k = rng.integers(-(m // 4), (m - 4) // 4 + 1, (bs, channels))
            blk = (4 * k + np.where(np.arange(channels) % 2 == 0, 1, 3)) << w
        else:
            left = rng.integers(lo, lo // 4, bs)
            right = rng.integers(0, hi // 4, bs)
            right = np.where((left + right) % 2 == 0, right + 1, right)
            blk = np.stack([left, right] + [rng.integers(lo, hi + 1, bs) for _ in range(channels - 2)], axis=1)[:, :channels]
        out[b] = blk
    assert out.min() >= lo and out.max() <= hi
    return out.reshape(nb * bs, channels).astype(np.int32)
