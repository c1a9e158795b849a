"""The encoder's LPC stage at its rarely taken branches, against the oracle (oracle/flac_oracle.c), which
test_oracle_lpc_edges.py pins against the reference at these inputs.

  * k_lpc (through flac_b200.debug_lpc, in its k_lpc<8>, <12> and <32> instantiations) equals fo_lpc_candidates slot for slot on
    constructed autocorrelations: the shift clamped at 15, negative shifts, shifts below -16, cmax == 0, clipped coefficients,
    the 17-bit precision cap, skipped orders, Levinson's early stop, autoc[0] == 0, punch-out windows with a stale last entry and
    a root smaller than the partial, limit without a wide prediction, and wasted bits undone by the 2^-2w rescale. Its wide / limit flags equal the reference's
    rules: limit = max residual bps > 32, wide = prediction before the shift wider than 32 bits, or limit.
  * Whole encodes of the PCM inputs of lpcedges.py (negative shifts, 64-bit and checked residuals, a checked residual that
    leaves int32, 32-bit partition sums that wrap, a 25-bit side channel) equal the oracle frame for frame on every stage-B
    path: k_search5 + k_emit3 (1-2 channels), k_search5 + k_emit3<PAIR> + k_join (5 and 7 channels), the general kernels
    (natural blocksizes and FB200_DEBUG_PATH=7) and the tiled kernels (FB200_DEBUG_PATH=22, and 16384 / 40000).
    The encoder's chosen plans are compared too: on the 5-channel input each of the join, general and tiled paths chooses LPC
    subframes with a 64-bit residual, so the emit's wide residual runs there."""
import math

import numpy as np
import pytest

import lpcedges
import oraclelib
from test_gpu_formats import check, fast_blocksize

pytestmark = pytest.mark.gpu

MIN_PREC, NPREC = 5, 11


_expected = {}


def expected_slots(row, root, kind, mo, sbps, wasted, unshifted, cfg, bs, per_win):
    """The slots k_lpc should write for one (item, window): {slot: oracle candidate, wide, limit}, from fo_lpc_candidates (one
    oracle call per distinct input)."""
    key = (kind, row.tobytes(), None if root is None else root.tobytes(), mo, sbps, wasted, unshifted, cfg.do_qlp_coeff_prec_search,
           cfg.do_exhaustive_model_search, cfg.qlp_coeff_precision, bs)
    if key not in _expected:
        _expected[key] = _expected_slots(row, root, kind, mo, sbps, wasted, unshifted, cfg, bs, per_win)
    return _expected[key]


def _expected_slots(row, root, kind, mo, sbps, wasted, unshifted, cfg, bs, per_win):
    if sbps == 0:
        return {}
    ac = lpcedges.effective_autoc(kind, row, root, mo, wasted, unshifted)
    cands = oraclelib.lpc_candidates(ac, mo, sbps, bs, cfg)
    if not cands:
        return {}
    lo = 1 if cfg.do_exhaustive_model_search else cands[0].order
    minp = MIN_PREC if cfg.do_qlp_coeff_prec_search else cfg.qlp_coeff_precision
    nprec = NPREC if cfg.do_qlp_coeff_prec_search else 1
    out = {}
    for c in cands:
        if c.status == 0:
            slot = (c.order - lo) * nprec + (c.precision_tried - minp)
            assert 0 <= slot < per_win
            out[slot] = (c,) + oraclelib.lpc_flags(sbps, c.qlp, c.order, c.shift)
    return out


def run_hook(rows, pairs, mo, ps, ex, prec, sbps_of, wasted_of=lambda k: 0, unshifted=False, bs=4096):
    """One debug_lpc launch: item k analyses rows[k] (window 0) and punch-out pair k % len(pairs) (window 1). Returns the
    number of slots compared and the mismatches."""
    import flac_b200
    n = len(rows)
    ac = np.zeros((3, n, lpcedges.LAGS))
    for k, row in enumerate(rows):
        ac[0, k] = row
        _, root, part = pairs[k % len(pairs)]
        ac[1, k], ac[2, k] = part, root
    meta = np.array([[wasted_of(k), sbps_of(k)] for k in range(n)], dtype=np.int32)
    wins = np.array([[0, 0, 0], [1, 1, 2]], dtype=np.int32)
    got = flac_b200.debug_lpc(ac, meta, wins, mo, prec, ps, ex, bs, autoc_unshifted=unshifted)
    cfg = oraclelib.preset(1, 16, 44100, 8, bs, do_qlp_coeff_prec_search=ps, do_exhaustive_model_search=ex, qlp_coeff_precision=prec)
    per_win = got.shape[1] // 2
    bad, compared = [], 0
    for k in range(n):
        for w, (kind, row, root) in enumerate(((0, ac[0, k], None), (1, ac[1, k], ac[2, k]))):
            want = expected_slots(row, root, kind, mo, int(meta[k, 1]), int(meta[k, 0]), unshifted, cfg, bs, per_win)
            g = got[k, w * per_win:(w + 1) * per_win]
            compared += per_win
            where = (mo, ps, ex, prec, k, w)
            valid = set(np.flatnonzero(g[:, 0]).tolist())
            if valid != set(want) or not np.all((g[:, 0] == 0) | (g[:, 0] == 1)):
                bad.append((where, "valid slots", sorted(valid ^ set(want))[:5]))
                continue
            for s, (c, wide, limit) in want.items():
                have = (int(g[s, 1]), int(g[s, 2]), int(g[s, 3]), int(g[s, 4]), int(g[s, 5]), g[s, 8:].tolist())
                need = (c.order, c.precision, c.shift, wide, limit, list(c.qlp))
                if have != need:
                    bad.append((where, s, have, need))
    return compared, bad


def hook_rows():
    return [r for _, r in lpcedges.constructed_rows()], lpcedges.punchout_pairs()


def test_k_lpc_equals_oracle_candidates():
    """max_order 1-32 (all three k_lpc instantiations), precision 5-15, precision search and exhaustive search on and off,
    subframe bps 4-25 (17 and 18 in every launch)."""
    rows, pairs = hook_rows()
    oraclelib.lpc_counters(reset=True)
    total, bad = 0, []
    for mo in range(1, 33):
        for combo in range(4):
            ps, ex = combo & 1, combo >> 1
            prec = MIN_PREC + (mo + combo) % NPREC
            sb = [17, 18] + [4 + (mo * 5 + combo * 11 + j * 7) % 22 for j in range(2)]
            n, b = run_hook(rows * len(sb), pairs, mo, ps, ex, prec, lambda k: sb[k // len(rows)])
            total += n
            bad += b
    assert not bad, f"{len(bad)} of {total} slots differ, first {bad[:3]}"
    c = oraclelib.lpc_counters()
    assert all(c[k] for k in ("shift_clamped", "negative_shift", "shift_too_small", "cmax_zero", "coef_clipped", "precision_capped",
                              "order_skipped", "levinson_early")), c


@pytest.mark.parametrize("mo", [8, 12, 32])
def test_k_lpc_undoes_wasted_bits(mo):
    """autoc_unshifted: rows of the signal before 1-8 wasted bits were shifted out, scaled by 2^-2w in k_lpc."""
    rows, pairs = hook_rows()
    for ps, ex in ((0, 0), (1, 1)):
        n, bad = run_hook(rows * 8, pairs, mo, ps, ex, 12, lambda k: 6 + k % 20, wasted_of=lambda k: 1 + k // len(rows),
                          unshifted=True)
        assert not bad, f"{len(bad)} of {n} slots differ, first {bad[:3]}"


def chosen_wide_lpc(x, bps, level, bs, **cfg):
    """Encode x's full blocks in one launch: the number of chosen subframes that are LPC with a 64-bit residual, from the
    encoder's plans and from the oracle's."""
    import flac_b200
    nb, ch = x.shape[0] // bs, x.shape[1]
    enc = flac_b200.Encoder(flac_b200.preset(ch, bps, 44100, level, bs, **cfg), max_blocks_per_launch=nb)
    try:
        enc.encode_frames(x[:nb * bs])
        plans, ca = enc.debug_plans(nb)
        nsig = enc.nsig
    finally:
        enc.close()
    o = oraclelib.Encoder(oraclelib.preset(ch, bps, 44100, level, bs, **cfg))
    got = want = 0
    for b in range(nb):
        sigs = range(ch) if nsig == ch else {0: (0, 1), 1: (0, 3), 2: (3, 1), 3: (2, 3)}[int(ca[b])]
        got += sum(1 for s in sigs if plans[b * nsig + s].type == 3 and plans[b * nsig + s].wide)
        _, plan = o.encode_frame(x[b * bs:(b + 1) * bs], b, want_plan=True)
        for c in range(ch):
            sub = plan.sub[c]
            if sub.type == 3:
                want += oraclelib.lpc_flags(sub.subframe_bps, sub.qlp_coeff, sub.order, sub.qlp_shift)[0]
    return got, want


PATHS = [("natural", None), ("debug_path_7", ("FB200_DEBUG_PATH", "7")), ("tiled", ("FB200_DEBUG_PATH", "22"))]


@pytest.mark.parametrize("env", PATHS, ids=[p[0] for p in PATHS])
@pytest.mark.parametrize("case", lpcedges.pcm_cases(), ids=[c[0] for c in lpcedges.pcm_cases()])
def test_encodes_on_every_path(monkeypatch, case, env):
    name, ch, bps, level, bs, cfg, x = case
    path = "fast" if env[1] is None and fast_blocksize(bs, level, ch) else "general"
    if env[1]:
        monkeypatch.setenv(*env[1])
    check(x, bps, 44100, level, bs, path, what=name, **cfg)
    got, want = chosen_wide_lpc(x, bps, level, bs, **cfg)
    assert got == want, f"{name} ({env[0]}): {got} chosen LPC subframes with a 64-bit residual, the oracle {want}"
    if name == "5ch 24-bit":
        assert got > 0, f"{name} ({env[0]}): the emit's 64-bit residual did not run"


@pytest.mark.parametrize("bs", [16384, 40000])
def test_tiled_natural_blocksizes(bs):
    x = lpcedges.with_bursts(lpcedges.integrated(bs + 777, 1, 24, 8, seed=bs, bs=bs), 24, bs, "end", width=48)
    check(x, 24, 44100, 8, bs, "general", what="tiled", max_lpc_order=32, do_qlp_coeff_prec_search=1)
    got, want = chosen_wide_lpc(x, 24, 8, bs, max_lpc_order=32, do_qlp_coeff_prec_search=1)
    assert got == want
    y = lpcedges.integrated(bs + 5, 2, 24, 6, seed=bs + 1, bs=bs, opposed=True)
    check(y, 24, 44100, 8, bs, "general", what="tiled stereo")


def search_cases():
    """(blocks [n, bs], CandDesc words [n, 40], oracle estimates [n], bs) for the general search kernel's evaluation: quantised
    candidates of a few steep constructed rows (sbps 24, -p -e, order up to 32) on every full block of two burst inputs. Their checked residuals leave int32 and their 32-bit partition sums wrap; the counters show that both happen."""
    rows = [lpcedges.ar_autoc(a, k) for a, k in ((0.99, 7), (0.99, 8), (0.9, 8), (0.95, 8), (0.9, 9), (0.999, 12), (0.999, 24))]
    cfg = oraclelib.preset(1, 24, 44100, 8, 4096, **lpcedges.EXHAUSTIVE_32)
    quantised = [c for r in rows for c in oraclelib.lpc_candidates(r, 32, 24, 4096, cfg) if c.status == 0]
    # the predictors (1 - z^-1)^k at shift 0, k = 5..7: on a full-scale alternating burst each residual is about 2^(23 + k),
    # so 8 of them pass 2^32 without leaving int32
    for k in (5, 6, 7):
        for shift in (0, 1):
            c = oraclelib.LpcCand(status=0, order=k, precision_tried=15, precision=15, shift=shift)
            for j in range(k):
                c.qlp[j] = (-1) ** j * math.comb(k, j + 1) << shift
            quantised.append(c)
    out = []
    # at 512 samples and -8 the partitions are 8 samples (32-bit sums at 24 bits) only for orders below 8
    for name, bs, cands in (("wrap 24-bit bs 512", 512, [c for c in quantised if c.order < 8]), ("overflow 24-bit", 4096, quantised[::7])):
        x = next(c[6] for c in lpcedges.pcm_cases() if c[0] == name)[:, 0]
        blocks = [x[b * bs:(b + 1) * bs] for b in range(x.size // bs)]
        o = oraclelib.Encoder(oraclelib.preset(1, 24, 44100, 8, bs))
        sig, words, want = [], [], []
        for blk in blocks:
            blk = np.ascontiguousarray(blk, dtype=np.int32)
            for c in cands:
                wide, limit = oraclelib.lpc_flags(24, c.qlp, c.order, c.shift)
                sig.append(blk)
                words.append([1, c.order, c.precision, c.shift, wide, limit, 0, 0] + list(c.qlp))
                e = oraclelib.lib().fo_lpc_estimate(o.h, blk.ctypes.data, bs, 24, 0, oraclelib.C.byref(c), 0, 6)
                want.append(0xffffffff if e == 0 else e)
        out.append((np.array(sig), np.array(words, dtype=np.int32), np.array(want, dtype=np.uint32), bs))
    return out


def test_search_rejects_and_wraps_like_the_reference():
    """The general search kernel's per-candidate estimate (fb200_debug_evaluate_lpc) equals the oracle's on candidates whose
    checked residual leaves int32 (rejected: no estimate) and whose 32-bit partition sums wrap (the estimate the reference's
    wrapped sums give). On the encodes these branches are taken but never change which candidate wins, so only the estimates
    show whether a kernel takes them as the reference does."""
    import flac_b200
    oraclelib.lpc_counters(reset=True)
    cases = search_cases()
    c = oraclelib.lpc_counters()
    assert c["limit_rejected"] > 0 and c["narrow_wrapped"] > 0, c
    for sig, words, want, bs in cases:
        got = flac_b200.debug_evaluate_lpc(sig, np.tile([0, 24], (sig.shape[0], 1)), words, 0, 6, 31)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"bs {bs}: {bad.size} of {want.size} estimates differ, first {[(int(i), int(got[i]), int(want[i])) for i in bad[:5]]}"
