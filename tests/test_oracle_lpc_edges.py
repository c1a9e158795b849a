"""Pins the oracle's LPC stage at its rarely taken branches against the compiled reference, and shows that the inputs of
lpcedges.py reach every one of them.

The music-like, noise, sine and alternation inputs of the other tests almost never leave the quantiser's common path. The PCM
inputs here (integrated noise at 16-24 bits, a 25-bit side channel, full-scale bursts where the window gives them no weight)
reach negative shifts, the shift clamp, clipped coefficients, the 17-bit precision cap, skipped orders, residuals wider than
32 bits, checked residuals that leave int32, and 32-bit partition sums that wrap. Each stream ends in a short last block. The
reference runs with its C dispatch (disable_isa=16), as in test_oracle_formats.py.

Two edges are reached only through constructed autocorrelations (fo_lpc_candidates, and k_lpc in test_gpu_lpc_edges.py):
  * a shift below -16 needs a coefficient of at least 2^(precision + 15) >= 2^20. A predictor that large amplifies the
    rounding of the integer samples by more than 2^20, so its expected bits exceed any subframe's bps and the order guess
    never picks it; even the exhaustive search on the steepest inputs here stays below 2^14;
  * Levinson's error is exactly 0.0 only when a reflection coefficient is exactly +-1, i.e. the windowed block is exactly
    predictable; a block that is, is constant or verbatim before LPC runs, and a window's float rounding breaks the rest."""
import numpy as np
import pytest

import lpcedges
import oraclelib
from conftest import require_ref
from test_oracle_formats import c_dispatch_reference, differing

PCM_ONLY_MISSES = {"shift_too_small", "levinson_early"}


def oracle_frames(name, ch, bps, level, bs, cfg, x):
    return oraclelib.Encoder(oraclelib.preset(ch, bps, 44100, level, bs, **cfg)).encode_stream(x)


@pytest.mark.parametrize("case", lpcedges.pcm_cases(), ids=[c[0] for c in lpcedges.pcm_cases()])
def test_pcm_edges_equal_reference(case):
    require_ref()
    name, ch, bps, level, bs, cfg, x = case
    assert x.shape[0] % bs, "every stream ends in a short last block"
    want = c_dispatch_reference(x, bps, 44100, level, bs, **lpcedges.ref_opts(cfg))
    assert differing(oracle_frames(*case), want) == []


def constructed_sweep():
    """fo_lpc_candidates over every constructed row and punch-out pair at max_order 1-32, precision 5-15, subframe bps 4-25,
    precision search and exhaustive search on and off."""
    rows = [r for _, r in lpcedges.constructed_rows()]
    rows += [lpcedges.effective_autoc(1, p, r, 32, 0, False) for _, r, p in lpcedges.punchout_pairs()]
    n = 0
    for mo in range(1, 33):
        for combo in range(4):
            ps, ex = combo & 1, combo >> 1
            cfg = oraclelib.preset(1, 16, 44100, 8, 4096, do_qlp_coeff_prec_search=ps, do_exhaustive_model_search=ex,
                                   qlp_coeff_precision=5 + (mo + combo) % 11)
            for k, row in enumerate(rows):
                sbps = 4 + (mo + k + combo) % 22
                n += len(oraclelib.lpc_candidates(row[:mo + 1], mo, sbps, 4096, cfg))
    return n


def test_every_edge_is_reached():
    """Every counter of the oracle's LPC stage is non-zero over the inputs of lpcedges.py, and the PCM inputs alone reach all
    but the two edges the module docstring rules out."""
    oraclelib.lpc_counters(reset=True)
    for case in lpcedges.pcm_cases():
        oracle_frames(*case)
    pcm = oraclelib.lpc_counters(reset=True)
    assert constructed_sweep() > 0
    rows = oraclelib.lpc_counters(reset=True)
    assert [k for k, v in pcm.items() if v == 0 and k not in PCM_ONLY_MISSES] == [], pcm
    assert [k for k in pcm if pcm[k] + rows[k] == 0] == [], (pcm, rows)


def test_candidates_follow_the_reference_rules():
    """fo_lpc_candidates' list on the constructed rows: each order that is tried is tried at every precision of the search,
    capped at 32 - bps - ilog2(order) for subframes of 17 bits or fewer; dropped candidates carry quantize's codes."""
    for _, row in lpcedges.constructed_rows():
        for sbps in (4, 16, 17, 18, 25):
            cfg = oraclelib.preset(1, 16, 44100, 8, 4096, do_qlp_coeff_prec_search=1, do_exhaustive_model_search=1)
            cands = oraclelib.lpc_candidates(row, 32, sbps, 4096, cfg)
            if row[0] == 0:
                assert cands == []
                continue
            for c in cands:
                assert 1 <= c.order <= 32
                if c.status == 3:
                    continue
                cap = 32 - sbps - int(np.log2(c.order))
                assert c.precision == (min(c.precision_tried, cap) if sbps <= 17 else c.precision_tried)
                assert c.status in (0, 1, 2)
                if c.status == 0:
                    assert 0 <= c.shift <= 15
                    assert all(-(1 << (c.precision - 1)) <= q < (1 << (c.precision - 1)) for q in c.qlp[:c.order])
