"""flac_b200 -- H100-native FLAC block encode/decode engine.

This package is only the host-side Python mirror of the C ABI in include/flac_b200.h
(libflac_b200.so: hand-written sm_90a CUDA kernels + host C++). There is no CPU fallback:
if the shared library is missing or no CUDA device is present every compute call raises.

Names mirror the reference's encoder/decoder interface (FLAC__stream_encoder_set_* knobs
-> EncoderConfig fields; reference: include/FLAC/stream_encoder.h:738-1289).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libflac_b200.so")

FB200_OK = 0
ERRORS = {-1: "CUDA", -2: "UNSUPPORTED", -3: "INVALID", -4: "OUTPUT_TOO_SMALL", -5: "BAD_STREAM", -6: "ALLOC"}
APOD_TUKEY, APOD_SUBDIVIDE_TUKEY = 0, 1
MAX_LPC_ORDER = 32
MAX_PARTITIONS = 256


class FlacB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"flac_b200 error {code} ({ERRORS.get(code, '?')}): {msg}")
        self.code = code


class Apodization(C.Structure):
    _fields_ = [("type", C.c_int32), ("p", C.c_float), ("parts", C.c_int32), ("start", C.c_float), ("end", C.c_float)]


class EncoderConfig(C.Structure):
    _fields_ = [
        ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("sample_rate", C.c_uint32), ("blocksize", C.c_uint32),
        ("do_mid_side_stereo", C.c_int32), ("loose_mid_side_stereo", C.c_int32),
        ("max_lpc_order", C.c_uint32), ("qlp_coeff_precision", C.c_uint32),
        ("do_qlp_coeff_prec_search", C.c_int32), ("do_exhaustive_model_search", C.c_int32),
        ("min_residual_partition_order", C.c_uint32), ("max_residual_partition_order", C.c_uint32),
        ("num_apodizations", C.c_uint32), ("apodizations", Apodization * 32),
        ("disable_constant_subframes", C.c_int32), ("disable_fixed_subframes", C.c_int32),
        ("disable_verbatim_subframes", C.c_int32), ("limit_min_bitrate", C.c_int32),
    ]


class DecoderConfig(C.Structure):
    _fields_ = [("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("sample_rate", C.c_uint32), ("blocksize", C.c_uint32)]


class SubframePlan(C.Structure):
    """Mirror of fb200::SubframePlan (debug/stage-level parity checks)."""
    _fields_ = [
        ("type", C.c_int32), ("order", C.c_int32), ("wasted", C.c_int32), ("bps", C.c_int32),
        ("precision", C.c_int32), ("shift", C.c_int32), ("method", C.c_int32), ("porder", C.c_int32),
        ("est_bits", C.c_uint32), ("wide", C.c_int32), ("pad0", C.c_int32), ("pad1", C.c_int32),
        ("qlp", C.c_int32 * MAX_LPC_ORDER), ("params", C.c_uint8 * MAX_PARTITIONS),
    ]


class SubframeInfo(C.Structure):
    """Mirror of fb200_subframe_info (what FLAC__Frame.subframes[] carries)."""
    _fields_ = [("type", C.c_uint8), ("order", C.c_uint8), ("wasted_bits", C.c_uint8), ("qlp_coeff_precision", C.c_uint8),
                ("quantization_level", C.c_int8), ("entropy_method", C.c_uint8), ("partition_order", C.c_uint8), ("reserved", C.c_uint8),
                ("qlp_coeff", C.c_int32 * MAX_LPC_ORDER), ("warmup", C.c_int32 * MAX_LPC_ORDER)]


_lib = None


def lib():
    """Loads libflac_b200.so; raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FlacB200Error(-1, f"{LIB_PATH} not built (python -m flac_b200.build); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.fb200_version.restype = C.c_char_p
    L.fb200_last_error.restype = C.c_char_p
    L.fb200_device_count.restype = C.c_int
    L.fb200_encoder_config_preset.restype = C.c_int
    L.fb200_encoder_config_preset.argtypes = [C.POINTER(EncoderConfig), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    L.fb200_encoder_config_set_apodization.restype = C.c_int
    L.fb200_encoder_config_set_apodization.argtypes = [C.POINTER(EncoderConfig), C.c_char_p]
    L.fb200_window.restype = C.c_int
    L.fb200_window.argtypes = [C.POINTER(Apodization), C.c_int32, C.c_void_p]
    L.fb200_encoder_create.restype = C.c_int
    L.fb200_encoder_create.argtypes = [C.POINTER(EncoderConfig), C.c_int, C.c_uint32, C.POINTER(C.c_void_p)]
    L.fb200_encoder_destroy.argtypes = [C.c_void_p]
    L.fb200_encoder_get_config.restype = C.c_int
    L.fb200_encoder_get_config.argtypes = [C.c_void_p, C.POINTER(EncoderConfig)]
    L.fb200_encoder_max_frame_bytes.restype = C.c_size_t
    L.fb200_encoder_max_frame_bytes.argtypes = [C.c_void_p]
    L.fb200_encoder_launch_count.restype = C.c_uint64
    L.fb200_encoder_launch_count.argtypes = [C.c_void_p]
    L.fb200_encode_host.restype = C.c_int
    L.fb200_encode_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint32)]
    L.fb200_encode_host_packed.restype = C.c_int
    L.fb200_encode_host_packed.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p,
                                           C.POINTER(C.c_uint32)]
    L.fb200_encoder_set_file_blocks.restype = C.c_int
    L.fb200_encoder_set_file_blocks.argtypes = [C.c_void_p, C.c_uint32]
    L.fb200_encode_device.restype = C.c_int
    L.fb200_encode_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p,
                                      C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_void_p, C.c_int]
    L.fb200_encoder_set_profiling.restype = C.c_int
    L.fb200_encoder_set_profiling.argtypes = [C.c_void_p, C.c_int]
    L.fb200_encoder_get_profile.restype = C.c_int
    L.fb200_encoder_get_profile.argtypes = [C.c_void_p, C.POINTER(C.c_double * 7), C.POINTER(C.c_uint64 * 7), C.c_int]
    L.fb200_debug_copy_plans.restype = C.c_int
    L.fb200_debug_copy_plans.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p]
    if hasattr(L, "fb200_decoder_create"):
        L.fb200_decoder_create.restype = C.c_int
        L.fb200_decoder_create.argtypes = [C.POINTER(DecoderConfig), C.c_int, C.c_uint32, C.POINTER(C.c_void_p)]
        L.fb200_decoder_destroy.argtypes = [C.c_void_p]
        L.fb200_decode_host.restype = C.c_int
        L.fb200_decode_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.fb200_decode_host_packed.restype = C.c_int
        L.fb200_decode_host_packed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint64,
                                               C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
        L.fb200_decode_device.restype = C.c_int
        L.fb200_decode_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                          C.c_void_p, C.c_int]
        L.fb200_decoder_get_frame_status.restype = C.c_int
        L.fb200_decoder_get_frame_status.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.fb200_decoder_enable_subframe_info.restype = C.c_int
        L.fb200_decoder_enable_subframe_info.argtypes = [C.c_void_p, C.c_int]
        L.fb200_decoder_get_subframe_info.restype = C.c_int
        L.fb200_decoder_get_subframe_info.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.fb200_decoder_index_host.restype = C.c_int
        L.fb200_decoder_index_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.fb200_decode_indexed_host.restype = C.c_int
        L.fb200_decode_indexed_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        L.fb200_decoder_launch_count.restype = C.c_uint64
        L.fb200_decoder_launch_count.argtypes = [C.c_void_p]
        L.fb200_decoder_set_profiling.restype = C.c_int
        L.fb200_decoder_set_profiling.argtypes = [C.c_void_p, C.c_int]
        L.fb200_decoder_get_profile.restype = C.c_int
        L.fb200_decoder_get_profile.argtypes = [C.c_void_p, C.POINTER(C.c_double * 3), C.POINTER(C.c_uint64 * 3), C.c_int]
    _lib = L
    return L


def _check(rc):
    if rc != FB200_OK:
        raise FlacB200Error(rc, lib().fb200_last_error().decode(errors="replace"))


def pack_pcm(pcm, bytes_per_sample):
    """int32 [samples, channels] -> packed little-endian bytes (what a WAV data chunk holds)."""
    pcm = np.ascontiguousarray(pcm, dtype=np.int32)
    if bytes_per_sample == 2:
        return pcm.astype("<i2").view(np.uint8).reshape(-1)
    if bytes_per_sample == 3:
        return np.ascontiguousarray(pcm.astype("<i4").view(np.uint8).reshape(-1, 4)[:, :3]).reshape(-1)
    return pcm.astype("<i4").view(np.uint8).reshape(-1)


def preset(channels, bits_per_sample, sample_rate, compression_level, blocksize=0, **overrides):
    """== FLAC__stream_encoder_set_compression_level + channels/bps/rate/blocksize."""
    cfg = EncoderConfig()
    _check(lib().fb200_encoder_config_preset(C.byref(cfg), channels, bits_per_sample, sample_rate, compression_level, blocksize))
    for k, v in overrides.items():
        if k == "apodization":  # == FLAC__stream_encoder_set_apodization(specification string)
            _check(lib().fb200_encoder_config_set_apodization(C.byref(cfg), v.encode() if isinstance(v, str) else v))
        else:
            setattr(cfg, k, v)
    return cfg


def window(apodization, length):
    """The float window table the encoder uploads for one Apodization at this block length."""
    out = np.empty(length, dtype=np.float32)
    _check(lib().fb200_window(C.byref(apodization), length, out.ctypes.data))
    return out


class Encoder:
    """Batch block encoder bound to one GPU."""

    def __init__(self, cfg, device=0, max_blocks_per_launch=0):
        self._h = C.c_void_p()
        _check(lib().fb200_encoder_create(C.byref(cfg), device, max_blocks_per_launch, C.byref(self._h)))
        self.cfg = EncoderConfig()
        _check(lib().fb200_encoder_get_config(self._h, C.byref(self.cfg)))
        self.max_frame_bytes = lib().fb200_encoder_max_frame_bytes(self._h)
        self.nsig = self.cfg.channels + (2 if (self.cfg.channels == 2 and self.cfg.do_mid_side_stereo) else 0)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().fb200_encoder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self):
        return int(lib().fb200_encoder_launch_count(self._h))

    def num_frames(self, samples):
        bs = self.cfg.blocksize
        return (samples + bs - 1) // bs

    def encode(self, pcm, first_frame_number=0, out=None, offsets=None):
        """pcm: int32 ndarray [samples, channels] in host memory. Returns (stream uint8 ndarray, offsets uint64[nframes+1])."""
        pcm = np.ascontiguousarray(pcm, dtype=np.int32)
        n, ch = pcm.shape
        assert ch == self.cfg.channels
        nfr = self.num_frames(n)
        if out is None:
            out = np.empty(nfr * self.max_frame_bytes + 64, dtype=np.uint8)
        if offsets is None:
            offsets = np.zeros(nfr + 1, dtype=np.uint64)
        nf = C.c_uint32(0)
        _check(lib().fb200_encode_host(self._h, pcm.ctypes.data, n, first_frame_number, out.ctypes.data, out.size,
                                       offsets.ctypes.data, C.byref(nf)))
        assert nf.value == nfr
        return out[:int(offsets[nfr])], offsets

    def encode_packed(self, packed, bytes_per_sample, samples, first_frame_number=0, out=None, offsets=None):
        """packed: uint8 ndarray of little-endian signed samples (2 or 3 bytes each, interleaved), `samples` per channel."""
        packed = np.ascontiguousarray(packed, dtype=np.uint8)
        assert packed.size == samples * self.cfg.channels * bytes_per_sample
        nfr = self.num_frames(samples)
        if out is None:
            out = np.empty(nfr * self.max_frame_bytes + 64, dtype=np.uint8)
        if offsets is None:
            offsets = np.zeros(nfr + 1, dtype=np.uint64)
        nf = C.c_uint32(0)
        _check(lib().fb200_encode_host_packed(self._h, packed.ctypes.data, bytes_per_sample, samples, first_frame_number, out.ctypes.data,
                                              out.size, offsets.ctypes.data, C.byref(nf)))
        assert nf.value == nfr
        return out[:int(offsets[nfr])], offsets

    def set_file_blocks(self, blocks_per_file):
        _check(lib().fb200_encoder_set_file_blocks(self._h, blocks_per_file))

    def encode_frames(self, pcm, first_frame_number=0):
        stream, offs = self.encode(pcm, first_frame_number)
        return [stream[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(len(offs) - 1)]

    def encode_device(self, d_pcm_ptr, samples, d_out_ptr, out_capacity, d_offsets_ptr, first_frame_number=0, stream=0, sync=False):
        """Device-resident path: raw device pointers (e.g. torch tensor .data_ptr()). Returns (nframes, total_bytes|None)."""
        nf = C.c_uint32(0)
        total = C.c_uint64(0)
        _check(lib().fb200_encode_device(self._h, d_pcm_ptr, samples, first_frame_number, d_out_ptr, out_capacity, d_offsets_ptr,
                                         C.byref(nf), C.byref(total), C.c_void_p(stream), 1 if sync else 0))
        return nf.value, (total.value if sync else None)

    PROF_NAMES = ("k_prep", "k_autoc", "k_lpc", "k_search", "k_emit", "k_scan", "k_gather")

    def set_profiling(self, on=True):
        _check(lib().fb200_encoder_set_profiling(self._h, 1 if on else 0))

    def profile(self, reset=True):
        """{kernel: (total_ms, launches)} from CUDA events recorded between the kernels."""
        ms = (C.c_double * 7)()
        n = (C.c_uint64 * 7)()
        _check(lib().fb200_encoder_get_profile(self._h, C.byref(ms), C.byref(n), 1 if reset else 0))
        return {name: (ms[i], int(n[i])) for i, name in enumerate(self.PROF_NAMES)}

    def debug_plans(self, nblocks):
        plans = (SubframePlan * (nblocks * self.nsig))()
        ca = np.zeros(nblocks, dtype=np.uint32)
        _check(lib().fb200_debug_copy_plans(self._h, nblocks, plans, C.sizeof(SubframePlan), ca.ctypes.data))
        return plans, ca


class Decoder:
    """Batch frame decoder bound to one GPU."""

    def __init__(self, channels, bits_per_sample, sample_rate, blocksize, device=0, max_frames_per_launch=0):
        self.cfg = DecoderConfig(channels, bits_per_sample, sample_rate, blocksize)
        self._h = C.c_void_p()
        _check(lib().fb200_decoder_create(C.byref(self.cfg), device, max_frames_per_launch, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().fb200_decoder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self):
        return int(lib().fb200_decoder_launch_count(self._h))

    PROF_NAMES = ("k_dec_walk", "k_dec_crc", "k_dec_frames")

    def set_profiling(self, on=True):
        _check(lib().fb200_decoder_set_profiling(self._h, 1 if on else 0))

    def profile(self, reset=True):
        ms = (C.c_double * 3)()
        n = (C.c_uint64 * 3)()
        _check(lib().fb200_decoder_get_profile(self._h, C.byref(ms), C.byref(n), 1 if reset else 0))
        return {name: (ms[i], int(n[i])) for i, name in enumerate(self.PROF_NAMES)}

    def decode(self, stream, offsets, total_samples=None):
        """stream: uint8 ndarray of back-to-back frames; offsets: uint64[nframes+1]. Returns int32 [samples, channels]."""
        stream = np.ascontiguousarray(stream, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        nfr = offsets.size - 1
        cap = nfr * self.cfg.blocksize
        out = np.empty((cap, self.cfg.channels), dtype=np.int32)
        ns = C.c_uint64(0)
        bad = C.c_uint32(0)
        _check(lib().fb200_decode_host(self._h, stream.ctypes.data, offsets.ctypes.data, nfr, out.ctypes.data, cap, C.byref(ns), C.byref(bad)))
        if bad.value:
            raise FlacB200Error(-5, f"{bad.value} frames failed to decode")
        n = ns.value if total_samples is None else total_samples
        return out[:n]

    def decode_packed(self, stream, offsets, bytes_per_sample, out=None):
        """As decode(), the samples narrowed on the device to packed little-endian PCM. Returns (uint8 bytes, samples per channel)."""
        stream = np.ascontiguousarray(stream, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        nfr = offsets.size - 1
        cap = nfr * self.cfg.blocksize
        if out is None:
            out = np.empty(cap * self.cfg.channels * bytes_per_sample, dtype=np.uint8)
        ns = C.c_uint64(0)
        bad = C.c_uint32(0)
        _check(lib().fb200_decode_host_packed(self._h, stream.ctypes.data, offsets.ctypes.data, nfr, out.ctypes.data, bytes_per_sample, cap,
                                              C.byref(ns), C.byref(bad)))
        if bad.value:
            raise FlacB200Error(-5, f"{bad.value} frames failed to decode")
        return out[:ns.value * self.cfg.channels * bytes_per_sample], ns.value

    def frame_status(self, nframes):
        """Per-frame status words of the last host decode: low byte 0 = ok, upper 24 bits = blocksize."""
        st = np.zeros(nframes, dtype=np.uint32)
        _check(lib().fb200_decoder_get_frame_status(self._h, st.ctypes.data, nframes))
        return st

    def enable_subframe_info(self, on=True):
        _check(lib().fb200_decoder_enable_subframe_info(self._h, 1 if on else 0))

    def subframe_info(self, nframes):
        """[(frame, channel)] SubframeInfo records of the last decode call (after enable_subframe_info)."""
        info = (SubframeInfo * (nframes * self.cfg.channels))()
        _check(lib().fb200_decoder_get_subframe_info(self._h, info, nframes))
        return info

    def index(self, stream, capacity=1 << 20):
        """GPU front end: ascending byte offsets of every sync code + self-consistent frame header in `stream`
        (which stays resident on the device for decode_indexed)."""
        stream = np.ascontiguousarray(stream, dtype=np.uint8)
        cand = np.zeros(capacity, dtype=np.uint64)
        n = C.c_uint32(0)
        _check(lib().fb200_decoder_index_host(self._h, stream.ctypes.data, stream.size, cand.ctypes.data, capacity, C.byref(n)))
        self._indexed_bytes = stream.size
        return cand[:n.value].copy()

    def decode_indexed(self, begins, max_frame_bytes):
        """Decode the frames starting at `begins` of the indexed stream. Returns (pcm [n*blocksize, ch], status, frame_bytes)."""
        begins = np.ascontiguousarray(begins, dtype=np.uint64)
        n = begins.size
        out = np.zeros((n * self.cfg.blocksize, self.cfg.channels), dtype=np.int32)
        st = np.zeros(n, dtype=np.uint32)
        fb = np.zeros(n, dtype=np.uint32)
        _check(lib().fb200_decode_indexed_host(self._h, begins.ctypes.data, n, max_frame_bytes, self._indexed_bytes, out.ctypes.data,
                                               n * self.cfg.blocksize, st.ctypes.data, fb.ctypes.data))
        return out, st, fb

    def decode_device(self, d_frames_ptr, d_offsets_ptr, nframes, d_pcm_ptr, pcm_capacity_samples, d_status_ptr, stream=0, sync=False):
        _check(lib().fb200_decode_device(self._h, d_frames_ptr, d_offsets_ptr, nframes, d_pcm_ptr, pcm_capacity_samples, d_status_ptr,
                                         C.c_void_p(stream), 1 if sync else 0))
