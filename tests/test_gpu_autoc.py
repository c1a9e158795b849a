"""Stage A on the GPU, record for record: the autocorrelation rows k_autoc4 (fused and meta routes, modes 0/1/2) and k_autoc3
(planar route) leave in the workspace, compared with the oracle's rows (fo_stage_a, pinned to the reference by
tests/test_oracle_autoc.py) as uint64 bit patterns, together with each signal's wasted bits, subframe bps and OR word.

Frames rarely show an autocorrelation error: a summation-order slip or a stale sample changes the LPC candidates of tonal
24-bit material but hardly ever of music or noise, so these sums are checked directly. The matrix reaches every route and
kernel mode, all five LAGS instantiations across their edges, 1-8 channels, fast, general, tiny and tiled blocksizes, every
window type, partial windows at unaligned shifts, and signals at the edges of wasted-bit and mid-side handling."""
from collections import namedtuple

import numpy as np
import pytest

import flac_b200
import oraclelib
import stagea

pytestmark = pytest.mark.gpu

SPEC32 = ("tukey(0.5);partial_tukey(2);punchout_tukey(3);subdivide_tukey(4);bartlett;bartlett_hann;blackman;"
          "blackman_harris_4term_92db;connes;flattop;gauss(0.2);hamming;hann;kaiser_bessel;nuttall;rectangle;triangle;welch;"
          "tukey(0.1);tukey(0.9);gauss(0.4);subdivide_tukey(3/0.2);partial_tukey(3/0.3/0.5);punchout_tukey(2/0.25/0.1);hann;welch")

# route: what the inputs select -- planar when FB200_DEBUG_PATH bit 1 is set or the blocksize leaves the fast stage-B kernels
# (general and tiled sizes; 1024 and 1152 at level 8, whose partitions of order 6 are shorter than k_search5's runs), meta for
# loose mid-side (level 4), fused otherwise
Case = namedtuple("Case", "name channels bps bs level lpc spec nb tail debug route")
CASES = [
    Case("s16_4096_l5", 2, 16, 4096, 5, 8, None, 48, 0, 0, "fused"),
    Case("s24_4096_sub5", 2, 24, 4096, 8, 12, "subdivide_tukey(5)", 24, 0, 0, "fused"),
    Case("s16_4608_spec32", 2, 16, 4608, 8, 16, SPEC32, 8, 0, 0, "fused"),
    Case("s16_1024_chunks", 2, 16, 1024, 5, 8, None, 600, 300, 0, "fused"),
    Case("s16_1152_lpc1", 2, 16, 1152, 5, 1, "hann", 40, 0, 0, "fused"),
    Case("s12_4096_lpc7", 2, 12, 4096, 5, 7, "tukey(0.5);partial_tukey(2);punchout_tukey(3)", 16, 0, 0, "fused"),
    Case("m16_4096_lpc6", 1, 16, 4096, 8, 6, "tukey(0.5);partial_tukey(2);punchout_tukey(3)", 64, 0, 0, "fused"),
    Case("m24_8192_lpc32", 1, 24, 8192, 8, 32, "subdivide_tukey(3)", 8, 0, 0, "fused"),
    Case("m16_1024_lpc11", 1, 16, 1024, 5, 11, "hann;welch;gauss(0.3)", 70, 0, 0, "fused"),
    Case("c3_4096_lpc8", 3, 16, 4096, 5, 8, "subdivide_tukey(3)", 40, 0, 0, "fused"),
    Case("c5_4608_lpc15", 5, 20, 4608, 8, 15, "subdivide_tukey(5)", 13, 0, 0, "fused"),
    Case("c6_1152_lpc12", 6, 16, 1152, 5, 12, "subdivide_tukey(2);blackman", 22, 0, 0, "fused"),
    Case("c8_4096_lpc31", 8, 24, 4096, 8, 31, None, 9, 0, 0, "fused"),
    Case("c8_1024_lpc16", 8, 16, 1024, 5, 16, "nuttall;connes", 12, 0, 0, "fused"),
    Case("s16_4096_loose", 2, 16, 4096, 4, 8, None, 40, 0, 0, "meta"),
    Case("s24_4608_loose_lpc32", 2, 24, 4608, 4, 32, "subdivide_tukey(3)", 14, 0, 0, "meta"),
    Case("s16_1000", 2, 16, 1000, 5, 8, None, 40, 0, 0, "planar"),
    Case("s24_4095_sub5", 2, 24, 4095, 8, 12, "subdivide_tukey(5)", 20, 0, 0, "planar"),
    Case("c3_4097_lpc16", 3, 16, 4097, 8, 16, "flattop;kaiser_bessel", 20, 0, 0, "planar"),
    Case("m16_192_sub8", 1, 16, 192, 8, 12, "subdivide_tukey(8)", 64, 0, 0, "planar"),
    Case("c5_576_lpc31", 5, 16, 576, 8, 31, "triangle;bartlett_hann", 16, 0, 0, "planar"),
    Case("s16_16", 2, 16, 16, 8, 16, None, 100, 0, 0, "planar"),
    Case("m24_17", 1, 24, 17, 8, 16, "welch", 100, 0, 0, "planar"),
    Case("c6_33", 6, 16, 33, 8, 32, "subdivide_tukey(2)", 40, 0, 0, "planar"),
    Case("s24_16384", 2, 24, 16384, 8, 12, "subdivide_tukey(3)", 3, 0, 0, "planar"),
    Case("m16_40000_lpc7", 1, 16, 40000, 5, 7, None, 2, 0, 0, "planar"),
    Case("s16_65535", 2, 16, 65535, 5, 8, None, 2, 0, 0, "planar"),
    Case("s16_4096_forced", 2, 16, 4096, 5, 8, None, 48, 0, 1, "planar"),
    Case("m24_8192_forced_lpc32", 1, 24, 8192, 8, 32, "subdivide_tukey(3)", 8, 0, 1, "planar"),
    Case("c6_4096_forced_lpc6", 6, 16, 4096, 8, 6, "gauss(0.2);rectangle", 12, 0, 1, "planar"),
]


def kernel_lags(lags):
    """The LAGS instantiation the launchers pick (autoc_kernel_lags)."""
    return next(k for k in (7, 9, 13, 17, 33) if lags <= k)


def case_lags(c):
    return min(c.lpc, c.bs - 1) + 1


def case_mode(c):
    return None if c.route == "planar" else 0 if c.channels == 1 else 1 if c.channels == 2 else 2


def _configs(c):
    over = dict(max_lpc_order=c.lpc)
    if c.spec:
        over["apodization"] = c.spec
    return (flac_b200.preset(c.channels, c.bps, 44100, c.level, blocksize=c.bs, **over),
            oraclelib.preset(c.channels, c.bps, 44100, c.level, c.bs, **over))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _mismatches(c, got_k, got, want, items, nsig, limit=6):
    """got / want: [nsec, len(items), LAGS] records of the listed items."""
    bad = np.argwhere(_bits(got) != _bits(want))
    lines = [f"{c.name}: route {got_k['route']} mode {case_mode(c)} LAGS {got_k['kernel_lags']}: {len(bad)} values differ"]
    for sec, i, lag in bad[:limit]:
        item = items[i]
        lines.append(f"  block {item // nsig} signal {item % nsig} section {sec} lag {lag}: got {got[sec, i, lag]!r} "
                     f"({_bits(got)[sec, i, lag]:#018x}) want {want[sec, i, lag]!r} ({_bits(want)[sec, i, lag]:#018x})")
    return "\n".join(lines)


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_stage_a_records_match_the_oracle(c, monkeypatch):
    if c.debug:
        monkeypatch.setenv("FB200_DEBUG_PATH", str(c.debug))
    else:
        monkeypatch.delenv("FB200_DEBUG_PATH", raising=False)
    fcfg, ocfg = _configs(c)
    if c.spec == SPEC32:
        assert fcfg.num_apodizations == ocfg.num_apodizations == 32
    x = stagea.mixed_blocks(c.nb, c.bs, c.channels, c.bps, seed=c.bs + c.channels)
    pcm = x
    if c.tail:  # a short last block of its own geometry and chunk, behind the full blocks compared here
        pcm = np.concatenate([x, stagea.mixed_blocks(1, c.tail, c.channels, c.bps, seed=7)])
    enc = flac_b200.Encoder(fcfg, device=0)
    try:
        enc.encode(pcm)
        got = enc.debug_autoc(c.nb)
    finally:
        enc.close()
    oenc = oraclelib.Encoder(ocfg)
    nsig = enc.nsig
    K = got["kernel_lags"]
    assert got["route"] == c.route, f"{c.name}: stage A took the {got['route']} route"
    assert got["lags"] == case_lags(c) and K == kernel_lags(case_lags(c))
    secs = stagea.sections(oenc.cfg, c.bs)
    assert got["sections"].tolist() == [[a * c.bs, p, n, ps, sh] for a, p, n, ps, sh in secs]

    fused = c.route == "fused"
    want, want_meta, want_or = oenc.stage_a(x, K, K, unshifted=fused)
    sig, meta_np, active = stagea.signals(x, c.nb, c.bs, c.channels, c.bps, oenc.cfg.do_mid_side, oenc.cfg.loose_mid_side)
    assert np.array_equal(want_meta, meta_np) and np.array_equal(want_or, np.where(
        active, np.bitwise_or.reduce(sig.astype(np.uint32), axis=1), 0).astype(np.uint32))
    if fused:
        assert active.all()
        # the sums of x scale exactly: rows(x >> w) == rows(x) * 2^-2w, the rescale k_lpc applies to the fused route's records
        shifted, _, _ = oenc.stage_a(x, K, K, unshifted=False)
        scale = np.ldexp(1.0, -2 * want_meta[:, 0].astype(np.int64))[None, :, None]
        assert np.array_equal(_bits(want * scale), _bits(shifted)), f"{c.name}: 2^-2w identity"
        assert np.array_equal(got["sigor"], want_or), f"{c.name}: sigor items {np.flatnonzero(got['sigor'] != want_or)[:8]}"
    # items of the pair a loose mid-side block does not code (subframe bps 0) are skipped by the kernels
    live = np.flatnonzero(active)
    assert np.array_equal(got["meta"][live], want_meta[live]), \
        f"{c.name}: meta of items {live[(got['meta'][live] != want_meta[live]).any(1)][:8]}"
    g, w = got["rows"][:, live, :K], want[:, live, :K]
    same = np.array_equal(_bits(g), _bits(w))
    assert same, _mismatches(c, got, g, w, live, nsig)


def test_hook_refuses_a_call_that_did_not_fit_one_workspace_set():
    """Past max_blocks_per_launch the chunks share two workspace sets in turn, and no record of the early blocks survives."""
    enc = flac_b200.Encoder(flac_b200.preset(2, 16, 44100, 5, blocksize=1024), device=0, max_blocks_per_launch=4)
    try:
        enc.encode(stagea.mixed_blocks(4, 1024, 2, 16, seed=3))
        assert enc.debug_autoc(4)["route"] == "fused"
        with pytest.raises(flac_b200.FlacB200Error) as ei:
            enc.debug_autoc(5)  # more blocks than the call encoded
        assert ei.value.code == -3  # FB200_ERR_INVALID
        enc.encode(stagea.mixed_blocks(10, 1024, 2, 16, seed=3))
        with pytest.raises(flac_b200.FlacB200Error) as ei:
            enc.debug_autoc(4)
        assert ei.value.code == -3 and "workspace" in str(ei.value)
    finally:
        enc.close()


def test_matrix_reaches_every_route_mode_lag_count_and_shape():
    """Asserted from the cases' inputs: each case above also asserts that the route it names is the one that ran."""
    kl = {r: {kernel_lags(case_lags(c)) for c in CASES if c.route == r} for r in ("fused", "meta", "planar")}
    assert kl["fused"] | kl["meta"] == kl["planar"] == {7, 9, 13, 17, 33}
    assert {case_mode(c) for c in CASES if c.route == "fused"} == {0, 1, 2}
    assert any(c.debug & 1 for c in CASES) and any(c.route == "planar" and not c.debug for c in CASES)
    assert {c.lpc for c in CASES} >= {1, 6, 7, 8, 11, 12, 15, 16, 31, 32}
    assert {c.channels for c in CASES} >= {1, 2, 3, 5, 6, 8}
    assert {c.bs for c in CASES} >= {1024, 1152, 4096, 4608, 8192, 192, 576, 1000, 4095, 4097, 16, 17, 33, 16384, 40000, 65535}
    # warps of 32 items that start mid-block: 3, 5 and 6 signals per block with more than one warp per section
    assert all(any(c.channels == n and c.nb * n > 64 for c in CASES) for n in (3, 5, 6))
    # several stage-A chunks (host chunks of at least 256 blocks) read back from their slices
    assert any(c.nb > 512 for c in CASES)
    specs = ";".join(c.spec or "tukey(0.5)" for c in CASES)
    for name in ("tukey", "partial_tukey", "punchout_tukey", "subdivide_tukey", "bartlett", "bartlett_hann", "blackman",
                 "blackman_harris_4term_92db", "connes", "flattop", "gauss", "hamming", "hann", "kaiser_bessel", "nuttall",
                 "rectangle", "triangle", "welch"):
        assert any(item.split("(")[0] == name for item in specs.split(";")), name
    # partial sections at shifts that are not multiples of 4 with odd part sizes, and sections skipped at bs / b <= 32
    cfgs = [(c, oraclelib.preset(c.channels, c.bps, 44100, c.level, c.bs, max_lpc_order=c.lpc, **({"apodization": c.spec} if c.spec else {})))
            for c in CASES]
    parts = [s for c, cfg in cfgs for s in stagea.sections(cfg, c.bs) if s[1]]
    assert any(sh % 4 and ps % 2 for _, _, _, ps, sh in parts)
    assert any(any(a.type == stagea.SUBDIVIDE_TUKEY and c.bs // a.parts <= 32 for a in cfg.apodizations[:cfg.num_apodizations])
               for c, cfg in cfgs)
