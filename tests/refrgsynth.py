"""ctypes binding of oracle/_ref/libFLAC_ref_rgsynth.so (built by oracle/ref_rgsynth.mk from the unmodified
replaygain_synthesis.c) -- test infrastructure only. The reference's dither generator is process-global, so each call loads a
fresh copy of the library and the generator starts at draw 0 (then `burn` draws are spent on a scratch buffer)."""
import ctypes as C
import os
import shutil
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "..", "oracle", "_ref", "libFLAC_ref_rgsynth.so")


def available():
    return os.path.exists(PATH)


def _fresh():
    d = tempfile.mkdtemp()
    p = os.path.join(d, "rgs.so")
    shutil.copy(PATH, p)
    L = C.CDLL(p)
    shutil.rmtree(d)
    L.ref_rgsynth.restype = C.c_int
    L.ref_rgsynth.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_double, C.c_int, C.c_int, C.c_uint64,
                              C.c_void_p]
    L.ref_tanh_array.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    return L


def synth(x, blocks, bps, scale, hard_limit, shaping, first_draw=0):
    """apply_gain over x (int32 [samples, channels]) delivered in `blocks`; returns val32 [samples, channels]."""
    x = np.ascontiguousarray(x, dtype=np.int32)
    b = np.ascontiguousarray(blocks, dtype=np.uint32)
    out = np.empty_like(x)
    assert _fresh().ref_rgsynth(x.ctypes.data, x.shape[1], x.shape[0], b.ctypes.data, b.size, bps, scale, 1 if hard_limit else 0, shaping,
                                first_draw, out.ctypes.data) == 0
    return out


def tanh(x):
    """The host libm's tanh() over x (float64), called from C."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.empty_like(x)
    _fresh().ref_tanh_array(x.ctypes.data, y.ctypes.data, x.size)
    return y
