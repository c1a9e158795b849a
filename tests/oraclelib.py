"""ctypes bindings for oracle/liboracle.so (the CPU restatement) -- test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_DIR = os.path.abspath(os.path.join(_HERE, "..", "oracle"))
FO_MAX_LPC_ORDER = 32
FO_MAX_PARTITIONS = 256


class Apod(C.Structure):
    _fields_ = [("type", C.c_int32), ("p", C.c_float), ("parts", C.c_int32), ("start", C.c_float), ("end", C.c_float)]


class Config(C.Structure):
    _fields_ = [
        ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("sample_rate", C.c_uint32), ("blocksize", C.c_uint32),
        ("do_mid_side", C.c_int32), ("loose_mid_side", C.c_int32),
        ("max_lpc_order", C.c_uint32), ("qlp_coeff_precision", C.c_uint32),
        ("do_qlp_coeff_prec_search", C.c_int32), ("do_exhaustive_model_search", C.c_int32),
        ("min_residual_partition_order", C.c_uint32), ("max_residual_partition_order", C.c_uint32),
        ("num_apodizations", C.c_uint32), ("apodizations", Apod * 32),
        ("disable_constant_subframes", C.c_int32), ("disable_fixed_subframes", C.c_int32),
        ("disable_verbatim_subframes", C.c_int32), ("limit_min_bitrate", C.c_int32), ("x86_avx2_fixed_guess", C.c_int32),
    ]


class SubframePlan(C.Structure):
    _fields_ = [
        ("type", C.c_int32), ("order", C.c_int32), ("wasted_bits", C.c_int32), ("subframe_bps", C.c_int32),
        ("qlp_precision", C.c_int32), ("qlp_shift", C.c_int32), ("qlp_negative_shift", C.c_int32),
        ("qlp_coeff", C.c_int32 * FO_MAX_LPC_ORDER),
        ("rice_method", C.c_int32), ("partition_order", C.c_int32), ("rice_params", C.c_int32 * FO_MAX_PARTITIONS),
        ("estimate_bits", C.c_uint32),
    ]


class FramePlan(C.Structure):
    _fields_ = [("channel_assignment", C.c_int32), ("sub", SubframePlan * 8), ("cand", SubframePlan * 4),
                ("cand_valid", C.c_uint32 * 4)]


class LpcCand(C.Structure):
    _fields_ = [("status", C.c_int32), ("order", C.c_int32), ("precision_tried", C.c_int32), ("precision", C.c_int32),
                ("shift", C.c_int32), ("negative_shift", C.c_int32), ("qlp", C.c_int32 * FO_MAX_LPC_ORDER)]


FO_MAX_LPC_CANDIDATES = FO_MAX_LPC_ORDER * 11
LPC_COUNTERS = ("shift_clamped", "negative_shift", "shift_too_small", "cmax_zero", "coef_clipped", "round_half", "precision_capped",
                "order_skipped", "levinson_early", "wide", "limit", "limit_rejected", "narrow_wrapped")


class LpcCounters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in LPC_COUNTERS]


class StreamInfo(C.Structure):
    _fields_ = [("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("sample_rate", C.c_uint32)]


_lib = None


def build():
    subprocess.run(["make", "-s", "oracle"], cwd=ORACLE_DIR, check=True)


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(path):
            build()
        L = C.CDLL(path)
        L.fo_config_preset.argtypes = [C.POINTER(Config), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
        L.fo_encoder_new.restype = C.c_void_p
        L.fo_encoder_new.argtypes = [C.POINTER(Config)]
        L.fo_encoder_delete.argtypes = [C.c_void_p]
        L.fo_encoder_config.restype = C.POINTER(Config)
        L.fo_encoder_config.argtypes = [C.c_void_p]
        L.fo_encode_frame.restype = C.c_size_t
        L.fo_encode_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(FramePlan)]
        L.fo_encode_stream.restype = C.c_int
        L.fo_encode_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                       C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.fo_decode_frame.restype = C.c_size_t
        L.fo_decode_frame.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(StreamInfo), C.c_void_p, C.c_size_t,
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
        L.fo_crc8.restype = C.c_uint8
        L.fo_crc8.argtypes = [C.c_void_p, C.c_size_t]
        L.fo_crc16.restype = C.c_uint16
        L.fo_crc16.argtypes = [C.c_void_p, C.c_size_t]
        L.fo_window_tukey.argtypes = [C.c_void_p, C.c_int32, C.c_float]
        L.fo_config_set_apodization.argtypes = [C.POINTER(Config), C.c_char_p]
        L.fo_window.restype = C.c_int
        L.fo_window.argtypes = [C.POINTER(Apod), C.c_void_p, C.c_int32]
        L.fo_autocorrelation.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.fo_window_data.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
        L.fo_window_data_partial.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
        L.fo_stage_a.restype = C.c_int
        L.fo_stage_a.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                 C.c_void_p]
        L.fo_lpc_candidates.restype = C.c_size_t
        L.fo_lpc_candidates.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(Config), C.POINTER(LpcCand)]
        L.fo_lpc_estimate.restype = C.c_uint32
        L.fo_lpc_estimate.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(LpcCand), C.c_uint32, C.c_uint32]
        L.fo_lpc_counters_get.argtypes = [C.POINTER(LpcCounters), C.c_int]
        L.fo_max_prediction_value_before_shift.restype = C.c_uint64
        L.fo_max_prediction_value_before_shift.argtypes = [C.c_uint32, C.c_void_p, C.c_uint32]
        L.fo_max_residual_bps.restype = C.c_uint32
        L.fo_max_residual_bps.argtypes = [C.c_uint32, C.c_void_p, C.c_uint32, C.c_int]
        L.fo_silog2.restype = C.c_uint32
        L.fo_silog2.argtypes = [C.c_int64]
        _lib = L
    return _lib


def preset(channels, bps, rate, level, blocksize=0, **over):
    cfg = Config()
    lib().fo_config_preset(C.byref(cfg), channels, bps, rate, level, blocksize)
    for k, v in over.items():
        if k == "apodization":
            lib().fo_config_set_apodization(C.byref(cfg), v.encode() if isinstance(v, str) else v)
        else:
            setattr(cfg, k, v)
    return cfg


def window(apod, length):
    out = np.empty(length, dtype=np.float32)
    if not lib().fo_window(C.byref(apod), out.ctypes.data, length):
        raise ValueError("unknown apodization type")
    return out


def autocorrelation(data, lags):
    """fo_autocorrelation: lags sums of the float32 data, each in ascending sample order."""
    d = np.ascontiguousarray(data, dtype=np.float32)
    out = np.zeros(lags, dtype=np.float64)
    lib().fo_autocorrelation(d.ctypes.data, d.size, lags, out.ctypes.data)
    return out


def window_data(x, win):
    """fo_window_data: x[i] * win[i] in float (lpc.c:68-74)."""
    x = np.ascontiguousarray(x, dtype=np.int32)
    w = np.ascontiguousarray(win, dtype=np.float32)
    out = np.zeros(x.size, dtype=np.float32)
    lib().fo_window_data(x.ctypes.data, w.ctypes.data, out.ctypes.data, x.size)
    return out


def window_data_partial(x, win, part_size, data_shift, init=0.0):
    """fo_window_data_partial over data_len = len(x) (lpc.c:82-94); entries it does not write keep `init`."""
    x = np.ascontiguousarray(x, dtype=np.int32)
    w = np.ascontiguousarray(win, dtype=np.float32)
    out = np.full(x.size, init, dtype=np.float32)
    lib().fo_window_data_partial(x.ctypes.data, w.ctypes.data, out.ctypes.data, x.size, part_size, data_shift)
    return out


def lpc_candidates(autoc, max_order, subframe_bps, blocksize, cfg):
    """fo_lpc_candidates: the candidates of one autocorrelation row (autoc[0 .. max_order]) in evaluation order."""
    a = np.ascontiguousarray(autoc, dtype=np.float64)
    assert a.size >= max_order + 1
    out = (LpcCand * FO_MAX_LPC_CANDIDATES)()
    n = lib().fo_lpc_candidates(a.ctypes.data, max_order, subframe_bps, blocksize, C.byref(cfg), out)
    return list(out[:n])


def lpc_counters(reset=False):
    c = LpcCounters()
    lib().fo_lpc_counters_get(C.byref(c), int(reset))
    return {n: getattr(c, n) for n in LPC_COUNTERS}


def lpc_flags(subframe_bps, qlp, order, shift):
    """(wide, limit) as the reference decides them (stream_encoder.c:4601-4617): limit = max residual bps > 32, wide = the
    prediction before the shift needs more than 32 bits, or limit."""
    q = np.ascontiguousarray(np.asarray(qlp[:order], dtype=np.int32))
    limit = lib().fo_max_residual_bps(subframe_bps, q.ctypes.data, order, shift) > 32
    pred = lib().fo_max_prediction_value_before_shift(subframe_bps, q.ctypes.data, order)
    return int(limit or lib().fo_silog2(pred) > 32), int(limit)


class Encoder:
    def __init__(self, cfg):
        self.h = lib().fo_encoder_new(C.byref(cfg))
        if not self.h:
            raise ValueError("configuration outside oracle scope")
        self.cfg = lib().fo_encoder_config(self.h).contents

    def close(self):
        if self.h:
            lib().fo_encoder_delete(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def encode_frame(self, pcm, frame_number=0, want_plan=False):
        pcm = np.ascontiguousarray(pcm, dtype=np.int32)
        n, ch = pcm.shape
        cap = 64 + n * ch * 5
        out = np.zeros(cap, dtype=np.uint8)
        plan = FramePlan() if want_plan else None
        ln = lib().fo_encode_frame(self.h, pcm.ctypes.data, n, frame_number, out.ctypes.data, cap,
                                   C.byref(plan) if want_plan else None)
        if ln == 0:
            raise RuntimeError("fo_encode_frame failed")
        return (out[:ln].tobytes(), plan) if want_plan else out[:ln].tobytes()

    def stage_a(self, pcm, lags, lag_stride=None, unshifted=False):
        """fo_stage_a on whole blocks of cfg.blocksize: (rows float64 [nsec, items, lag_stride], meta int32 [items, 2], sigor
        uint32 [items]), item = block * nsig + signal."""
        pcm = np.ascontiguousarray(pcm, dtype=np.int32)
        n, ch = pcm.shape
        bs = self.cfg.blocksize
        assert n % bs == 0 and ch == self.cfg.channels
        nb = n // bs
        nsig = ch + (2 if self.cfg.do_mid_side else 0)
        lag_stride = lag_stride or lags
        nsec_max = sum(1 + (sum(b if b > 2 else 2 for b in range(2, a.parts + 1)) if a.type == 1 else 0)
                       for a in self.cfg.apodizations[:self.cfg.num_apodizations])
        rows = np.zeros(nsec_max * nb * nsig * lag_stride, dtype=np.float64)
        meta = np.zeros((nb * nsig, 2), dtype=np.int32)
        sigor = np.zeros(nb * nsig, dtype=np.uint32)
        nsec = lib().fo_stage_a(self.h, pcm.ctypes.data, nb, lags, lag_stride, int(unshifted), rows.ctypes.data, rows.size,
                                meta.ctypes.data, sigor.ctypes.data)
        if nsec < 0:
            raise ValueError("fo_stage_a: bad arguments")
        return rows[:nsec * nb * nsig * lag_stride].reshape(nsec, nb * nsig, lag_stride), meta, sigor

    def encode_stream(self, pcm):
        pcm = np.ascontiguousarray(pcm, dtype=np.int32)
        n, ch = pcm.shape
        bs = self.cfg.blocksize
        cap = 1024 + n * ch * 5 + 64 * (n // bs + 2)
        out = np.zeros(cap, dtype=np.uint8)
        maxf = n // bs + 2
        fs = np.zeros(maxf, dtype=np.uint32)
        out_len, nf = C.c_size_t(0), C.c_size_t(0)
        rc = lib().fo_encode_stream(self.h, pcm.ctypes.data, n, out.ctypes.data, cap, C.byref(out_len), fs.ctypes.data, maxf, C.byref(nf))
        if rc != 0:
            raise RuntimeError("fo_encode_stream failed")
        frames, pos = [], 0
        for s in fs[:nf.value]:
            frames.append(out[pos:pos + int(s)].tobytes())
            pos += int(s)
        return frames


def decode_frames(stream_bytes, channels, bps, rate, max_samples):
    """Decode consecutive frames (no metadata header). Returns int32 [samples, channels]."""
    buf = np.frombuffer(stream_bytes, dtype=np.uint8)
    si = StreamInfo(channels, bps, rate)
    out = np.zeros((max_samples, channels), dtype=np.int32)
    pos, done = 0, 0
    bs, ch, b, num = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
    L = lib()
    while pos < buf.size:
        used = L.fo_decode_frame(buf.ctypes.data + pos, buf.size - pos, C.byref(si), out.ctypes.data + done * channels * 4,
                                 max_samples - done, C.byref(bs), C.byref(ch), C.byref(b), C.byref(num))
        if used == 0:
            raise RuntimeError(f"fo_decode_frame failed at byte {pos}")
        pos += used
        done += bs.value
    return out[:done]
