"""The oracle's stage-A arithmetic pinned to the compiled reference, bit for bit (CPU only).

fo_autocorrelation is the sum every autocorrelation kernel is compared with (tests/test_gpu_autoc.py): each lag's products
added in ascending sample order, every partial sum rounded. Here it is held to every routine the strict build's dispatch can
call on an x86-64 host (stream_encoder.c:1055-1066, :2978-2982): FLAC__lpc_compute_autocorrelation on both of its branches
(data_len < 32 or lag > 16; the deduplicated MAX_LAG body) and, where the CPU has FMA, the _intrin_fma_lag_{8,12,16}
routines within their lag ranges. The SSE2 routines (descending order) and the shipped-flags build (reassociated) are not
asserted on: DESIGN.md G2/G3. fo_window_data / fo_window_data_partial are held to FLAC__lpc_window_data / _partial, and
fo_stage_a's rows, meta and OR words to the reference's routines on the signals stream_encoder.c forms."""
import ctypes as C
import os

import numpy as np
import pytest

import oraclelib
import reflib
import signals
import stagea
from conftest import require_ref

FMA_ROUTINES = ((8, "FLAC__lpc_compute_autocorrelation_intrin_fma_lag_8"), (12, "FLAC__lpc_compute_autocorrelation_intrin_fma_lag_12"),
                (16, "FLAC__lpc_compute_autocorrelation_intrin_fma_lag_16"))
LENGTHS = [33, 34, 63, 64, 100, 577, 1152, 1365, 4095, 4096, 16384]
TINY = [1, 2, 3, 16, 17, 31]


def _strict():
    require_ref()
    L = C.CDLL(reflib._path("strict"))
    for name in ["FLAC__lpc_compute_autocorrelation"] + [n for _, n in FMA_ROUTINES]:
        f = getattr(L, name)
        f.restype = None
        f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
    L.FLAC__lpc_window_data.restype = None
    L.FLAC__lpc_window_data.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    L.FLAC__lpc_window_data_partial.restype = None
    L.FLAC__lpc_window_data_partial.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    return L


def _host_has_fma():
    try:
        with open("/proc/cpuinfo") as f:
            return any(line.startswith("flags") and " fma " in line + " " for line in f)
    except OSError:
        return False


def _ref_autoc(fn, data, lags):
    d = np.ascontiguousarray(data, dtype=np.float32)
    out = np.full(40, np.nan)  # the MAX_LAG bodies write MAX_LAG entries whatever `lag` is
    fn(d.ctypes.data, d.size, lags, out.ctypes.data)
    return out[:lags]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64 if a.dtype == np.float64 else np.uint32)


def _inputs(rng, n):
    """(label, float32 data) of length n: samples of 8 to 25 bits times real windows of every apodization type, and times
    random weights."""
    out = []
    for bits in (8, 16, 24, 25):
        x = rng.integers(-(1 << (bits - 1)), 1 << (bits - 1), n, dtype=np.int64).astype(np.int32)
        for apod in stagea.WINDOW_TYPES if n >= 2 else ():
            w = oraclelib.window(apod, n)
            out.append((f"{bits}-bit x window type {apod.type}", oraclelib.window_data(x, w)))
        out.append((f"{bits}-bit x random weights", oraclelib.window_data(x, rng.random(n, dtype=np.float32))))
    return out


def _check_routine(fn, name, data, lags, label):
    want = oraclelib.autocorrelation(data, lags)
    got = _ref_autoc(fn, data, lags)
    bad = np.flatnonzero(_bits(got) != _bits(want))
    assert bad.size == 0, f"{name}, {label}, data_len {data.size}, lags {lags}: lag {bad[0]} ref {got[bad[0]]!r} oracle {want[bad[0]]!r}"


def test_autocorrelation_equals_the_plain_routine_on_both_branches():
    L = _strict()
    rng = np.random.default_rng(11)
    fn = L.FLAC__lpc_compute_autocorrelation
    n_checked = 0
    for n in TINY + LENGTHS:
        for label, data in _inputs(rng, n):
            # data_len < 32 or lag > 16: the per-sample loop (lag <= data_len, lpc.c:142-143); else the MAX_LAG body
            lag_set = range(1, n + 1) if n < 32 else [1, 2, 7, 8, 9, 12, 13, 16, 17, 24, 32, 33]
            for lags in lag_set:
                if lags <= 33:
                    _check_routine(fn, "FLAC__lpc_compute_autocorrelation", data, lags, label)
                    n_checked += 1
    assert n_checked > 1000


def test_autocorrelation_equals_the_fma_routines():
    L = _strict()
    if not _host_has_fma():
        pytest.skip("the host CPU does not report fma: the _intrin_fma_lag_* routines are not called here")
    rng = np.random.default_rng(12)
    for n in LENGTHS:
        for label, data in _inputs(rng, n):
            for max_lag, name in FMA_ROUTINES:
                for lags in sorted({1, max_lag // 2, max_lag - 1, max_lag}):
                    _check_routine(getattr(L, name), name, data, lags, label)


def _ref_window_partial(L, x, w, part_size, data_shift, init):
    out = np.full(x.size, init, dtype=np.float32)
    L.FLAC__lpc_window_data_partial(x.ctypes.data, w.ctypes.data, out.ctypes.data, x.size, part_size, data_shift)
    return out


def test_window_data_equals_the_reference():
    L = _strict()
    rng = np.random.default_rng(13)
    for n in (2, 17, 1000, 4096, 4097):
        for bits in (8, 16, 24, 25):
            # 25 bits: (float)x rounds, the case where the float product is not exact
            x = rng.integers(-(1 << (bits - 1)), 1 << (bits - 1), n, dtype=np.int64).astype(np.int32)
            for apod in stagea.WINDOW_TYPES:
                w = oraclelib.window(apod, n)
                want = np.zeros(n, dtype=np.float32)
                L.FLAC__lpc_window_data(x.ctypes.data, w.ctypes.data, want.ctypes.data, n)
                got = oraclelib.window_data(x, w)
                assert np.array_equal(_bits(got), _bits(want)), f"window_data n {n} bits {bits} type {apod.type}"


def test_window_data_partial_equals_the_reference():
    L = _strict()
    rng = np.random.default_rng(14)
    init = np.float32(-7.25)  # entries neither routine writes must stay as they were
    for n in (64, 577, 4095, 4096):
        x = rng.integers(-(1 << 24), 1 << 24, n, dtype=np.int64).astype(np.int32)
        w = oraclelib.window(stagea.apod(oraclelib.Apod, 0, 0.5), n)
        cases = set()
        for b in range(2, 9):   # the sections subdivide_tukey(b) makes: odd part sizes, shifts with data_shift % 4 != 0
            for part in range(b):
                cases.add(((n // b) // 2, (part * n) // b))
        for ps in (1, 2, 3, n // 4, n // 2 - 1, n // 2):
            for shift in (0, 1, n - 2 * ps - 1, n - 2 * ps, n - 2 * ps + 1, n - ps - 1, n - ps, n - ps + 1):
                if 0 <= shift < n:  # part_size + data_shift near and past data_len, overlapping halves
                    cases.add((ps, shift))
        for ps, shift in sorted(cases):
            want = _ref_window_partial(L, x, w, ps, shift, init)
            got = oraclelib.window_data_partial(x, w, ps, shift, init=init)
            assert np.array_equal(_bits(got), _bits(want)), f"window_data_partial n {n} part_size {ps} data_shift {shift}"


@pytest.mark.parametrize("channels,bps,bs,spec,mid_side,loose", [
    (2, 16, 4096, "tukey(0.5);subdivide_tukey(5)", 1, 0),
    (2, 24, 1000, "partial_tukey(2);welch;subdivide_tukey(3)", 1, 1),
    (3, 20, 577, "gauss(0.2);punchout_tukey(3)", 0, 0),
    (1, 8, 40, "subdivide_tukey(2);hann", 0, 0),
])
def test_stage_a_rows_follow_the_reference(channels, bps, bs, spec, mid_side, loose):
    """fo_stage_a against the reference's window routines and its dispatched autocorrelation on the signals, wasted bits and
    OR words computed here with numpy, section by section in the order apply_apodization_ walks them."""
    L = _strict()
    nb = 6
    x = stagea.mixed_blocks(nb, bs, channels, bps, seed=bs)
    cfg = oraclelib.preset(channels, bps, 44100, 8, bs, apodization=spec, do_mid_side=mid_side, loose_mid_side=loose,
                           max_lpc_order=min(12, bs - 1))
    enc = oraclelib.Encoder(cfg)
    max_order = min(cfg.max_lpc_order, bs - 1)
    lags = max_order + 1
    autoc = L.FLAC__lpc_compute_autocorrelation
    if _host_has_fma() and bs > 32 and max_order < 16:  # stream_encoder.c:1055-1066, :2978-2982
        autoc = getattr(L, FMA_ROUTINES[0 if max_order < 8 else 1 if max_order < 12 else 2][1])
    for unshifted in (False, True):
        rows, meta, sigor = enc.stage_a(x, lags, lags + 2, unshifted=unshifted)
        sig, want_meta, active = stagea.signals(x, nb, bs, channels, bps, mid_side, loose)
        secs = stagea.sections(cfg, bs)
        assert rows.shape[0] == len(secs)
        assert np.array_equal(meta, want_meta)
        assert np.array_equal(sigor, np.where(active, np.bitwise_or.reduce(sig.astype(np.uint32), axis=1), 0).astype(np.uint32))
        wins = [oraclelib.window(cfg.apodizations[a], bs) for a in range(cfg.num_apodizations)]
        for item in np.flatnonzero(active):
            s = sig[item] if unshifted else sig[item] >> want_meta[item, 0]
            s = np.ascontiguousarray(s, dtype=np.int32)
            for k, (a, partial, dlen, ps, shift) in enumerate(secs):
                d = np.zeros(bs, dtype=np.float32)
                if partial:
                    L.FLAC__lpc_window_data_partial(s.ctypes.data, wins[a].ctypes.data, d.ctypes.data, bs, ps, shift)
                else:
                    L.FLAC__lpc_window_data(s.ctypes.data, wins[a].ctypes.data, d.ctypes.data, bs)
                want = _ref_autoc(autoc, d[:dlen], lags)
                assert np.array_equal(_bits(rows[k, item, :lags]), _bits(want)), f"item {item} section {k} unshifted {unshifted}"
                assert np.all(rows[k, item, lags:] == 0.0)
        assert np.all(rows[:, ~active] == 0.0)
