"""Pins the oracle (oracle/flac_oracle.c) against the compiled reference at every input format the encoder takes: every bit depth
4-24 x every channel count 1-8, the frame header's sample-rate code classes and their edges, and -p / limit_min_bitrate at low
depths and odd channel counts. Every stream ends in a short last block, where the reference's own dispatch paths disagree.

The reference is run with its C / SSE dispatch (disable_isa=16): its AVX2 routine for the fixed-order guess drops the last
(n - 4) % 4 samples of a block (DESIGN.md, G4), which only a short last block shows. The oracle -- and the CUDA engine -- follow
the C routine. A second test shows that the oracle's `x86_avx2_fixed_guess` mode equals the reference as an AVX2 host
dispatches it, on the same streams. The GPU tests (test_gpu_formats.py) compare the engine with the oracle on these formats;
the signal generators here are shared with them."""
import numpy as np
import pytest

import oraclelib
import reflib
import signals
from conftest import require_ref

SIGNAL_KINDS = ("music", "noise", "alternate", "wasted", "const")


def alternation(n, ch, bps, seed):
    """Full-scale opposite-phase alternation: odd channels are the even ones' mirror image, so left - right sits at its
    bound 2^bps - 1 (the side channel needs bps + 1 bits). The run length changes every few samples."""
    rng = np.random.default_rng(seed)
    hi, lo = (1 << (bps - 1)) - 1, -(1 << (bps - 1))
    runs = rng.integers(1, 9, size=n)
    phase = (np.repeat(np.arange(runs.size), runs)[:n] % 2).astype(bool)
    x = np.empty((n, ch), dtype=np.int32)
    for c in range(ch):
        up = phase if c % 2 == 0 else ~phase
        x[:, c] = np.where(up, hi, lo)
    return np.ascontiguousarray(x)


def wasted(n, ch, bps, seed):
    """Each channel with its own number of wasted bits; the first channel keeps a single significant bit (bps - wasted == 1)."""
    x = np.empty((n, ch), dtype=np.int32)
    rng = np.random.default_rng(seed)
    for c in range(ch):
        w = bps - 1 if c == 0 else 1 + (seed + c) % (bps - 1)
        keep = bps - w
        if keep == 1:
            v = rng.integers(-1, 1, size=n).astype(np.int32)
        else:
            v = signals.music_like(n, 1, keep, 44100, seed=seed + c)[:, 0]
        x[:, c] = v.astype(np.int64) << w
    return np.ascontiguousarray(x)


def make_signal(kind, n, ch, bps, rate=44100, seed=1, bs=4096):
    if kind == "music":
        return signals.music_like(n, ch, bps, rate, seed=seed)
    if kind == "noise":
        return signals.white_noise(n, ch, bps, seed=seed)
    if kind == "alternate":
        return alternation(n, ch, bps, seed)
    if kind == "wasted":
        return wasted(n, ch, bps, seed)
    assert kind == "const"
    # one channel constant (not zero) through the second block while the others stay live
    x = signals.music_like(n, ch, bps, rate, seed=seed)
    c = seed % ch
    x[bs:2 * bs, c] = -(1 << (bps - 1)) + 1 + seed % 3
    return x


def short_tail(rng, bs):
    """A last block shorter than bs whose length is not a multiple of 4, small or large."""
    cands = [t for t in (1, 2, 3, 5, 7, 15, 17, 31, 33, 35) if t < bs]
    if bs > 40:
        cands.append(int(rng.integers(36, bs)))
    t = int(rng.choice(cands))
    return t if t % 4 else t - 1


def format_streams(level, seed=0):
    """(ch, bps, kind, x, blocksize) over every channel count 1-8 x every bit depth 4-24: one full block and a short last block
    (two full blocks at -0, so the fixed predictor sees a regular block before the tail). The signal kind rotates over the cells."""
    rng = np.random.default_rng(1000 + level + seed)
    bs = 1152 if level < 3 else 4096
    out = []
    for ch in range(1, 9):
        for bps in range(4, 25):
            kind = SIGNAL_KINDS[(ch + bps + level) % len(SIGNAL_KINDS)]
            n = bs * (2 if level == 0 else 1) + short_tail(rng, bs)
            if kind == "const":
                n = 2 * bs + short_tail(rng, bs)
            out.append((ch, bps, kind, make_signal(kind, n, ch, bps, seed=ch * 31 + bps, bs=bs), bs))
    return out


def c_dispatch_reference(x, bps, rate, level, bs=0, **ref_kw):
    """The strict reference through its C / SSE routines (the fixed-order guess the oracle and the engine follow)."""
    _, _, frames = reflib.encode(x, bps, rate=rate, level=level, blocksize=bs, variant="strict",
                                 opts=reflib.RefEncOpts(streamable_subset=0, disable_isa=16, **ref_kw))
    return frames


def oracle_frames(x, bps, rate, level, bs=0, **cfg):
    return oraclelib.Encoder(oraclelib.preset(x.shape[1], bps, rate, level, bs, **cfg)).encode_stream(x)


def differing(got, want):
    assert len(got) == len(want), f"frame count {len(got)} != {len(want)}"
    return [i for i, (a, b) in enumerate(zip(got, want)) if a != b]


@pytest.mark.parametrize("level", [0, 1, 2, 5, 8])
def test_every_depth_and_channel_count(level):
    require_ref()
    bad = []
    for ch, bps, kind, x, bs in format_streams(level):
        d = differing(oracle_frames(x, bps, 44100, level), c_dispatch_reference(x, bps, 44100, level))
        if d:
            bad.append((ch, bps, kind, x.shape[0] % bs, d))
    assert not bad, f"(channels, bps, signal, tail, frames) that differ: {bad}"


def test_avx2_fixed_guess_mode_equals_host_dispatch():
    """G4 pinned: the oracle with x86_avx2_fixed_guess=1 equals the reference as this host dispatches it, frame for frame, on
    the same streams. Skipped where the host does not take the AVX2 routine (both dispatches then agree on every stream)."""
    require_ref()
    avx2_seen = False
    bad = []
    for level in (0, 2, 5, 8):
        for ch, bps, kind, x, bs in format_streams(level):
            _, _, host = reflib.encode(x, bps, rate=44100, level=level, variant="strict", opts=reflib.RefEncOpts(streamable_subset=0))
            if not avx2_seen and host != c_dispatch_reference(x, bps, 44100, level):
                avx2_seen = True
            d = differing(oracle_frames(x, bps, 44100, level, x86_avx2_fixed_guess=1), host)
            if d:
                bad.append((level, ch, bps, kind, d))
    if not avx2_seen:
        pytest.skip("this host does not dispatch to the AVX2 routine")
    assert not bad, f"(level, channels, bps, signal, frames) that differ: {bad}"


# Sample rates by frame-header code (stream_encoder_framing.c): table codes 1-11; 12 = kHz in 8 bits (multiple of 1000, at most
# 255000); 14 = tens of Hz in 16 bits (multiple of 10, at most 655350); 13 = Hz in 16 bits (at most 65535); 0 = STREAMINFO's.
RATES = {
    "table": [8000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000],
    "khz": [1000, 12000, 255000],
    "ten_hz": [10, 37800, 50010, 256000, 655350],
    "hz": [1, 11025, 12345, 65535],
    "streaminfo": [65537, 655360, 705600, 1048575],
}
ALL_RATES = [(cls, r) for cls in RATES for r in RATES[cls]]


def rate_cases():
    """(class, rate, channels, bps, level, blocksize): odd depths, 1-5 channels, and blocksizes whose header code is from the
    table, 8 bits (up to 256) or 16 bits."""
    bss = [0, 16, 17, 255, 257, 1000, 4608]
    for k, (cls, rate) in enumerate(ALL_RATES):
        yield cls, rate, 1 + k % 5, (5, 13, 17, 21, 23, 7)[k % 6], (0, 2, 5, 8)[k % 4], bss[k % len(bss)]


@pytest.mark.parametrize("cls,rate,ch,bps,level,bs", list(rate_cases()), ids=[f"{c[0]}-{c[1]}" for c in rate_cases()])
def test_sample_rate_codes(cls, rate, ch, bps, level, bs):
    require_ref()
    bsz = bs or (1152 if level < 3 else 4096)
    x = signals.music_like(2 * bsz + bsz // 3 + 3, ch, bps, 44100, seed=rate % 97)
    frames = oracle_frames(x, bps, rate, level, bs)
    assert differing(frames, c_dispatch_reference(x, bps, rate, level, bs)) == []


@pytest.mark.parametrize("ch", [1, 2, 5, 7])
@pytest.mark.parametrize("bps", [4, 5, 6, 7, 8])
def test_precision_search_and_limit_min_bitrate_at_low_depths(ch, bps):
    """flac -p and limit_min_bitrate, alone and together, at 4-8 bits on blocks of silence, a DC level, the last channel
    constant and the first channel constant."""
    require_ref()
    bs = 4096
    x = signals.music_like(bs * 5 + 3 + 4 * bps, ch, bps, 44100, seed=bps * 10 + ch)
    x[bs:2 * bs] = 0
    x[2 * bs:3 * bs] = 3 - (1 << (bps - 1))
    x[3 * bs:4 * bs, ch - 1] = 1
    x[4 * bs:5 * bs, 0] = -1
    for cfg, ref in ((dict(do_qlp_coeff_prec_search=1), dict(prec_search=1)), (dict(limit_min_bitrate=1), dict(limit_min_bitrate=1)),
                     (dict(do_qlp_coeff_prec_search=1, limit_min_bitrate=1), dict(prec_search=1, limit_min_bitrate=1))):
        for level in (2, 5, 8):
            d = differing(oracle_frames(x, bps, 44100, level, **cfg), c_dispatch_reference(x, bps, 44100, level, **ref))
            assert d == [], (cfg, level, d)
