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
ERRORS = {-1: "CUDA", -2: "UNSUPPORTED", -3: "INVALID", -4: "OUTPUT_TOO_SMALL", -5: "BAD_STREAM", -6: "ALLOC", -7: "VERIFY"}
ERR_VERIFY = -7
APOD_TUKEY, APOD_SUBDIVIDE_TUKEY = 0, 1
MAX_LPC_ORDER = 32
MAX_PARTITIONS = 256


class FlacB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"flac_b200 error {code} ({ERRORS.get(code, '?')}): {msg}")
        self.code = code


class Apodization(C.Structure):
    _fields_ = [("type", C.c_int32), ("p", C.c_float), ("parts", C.c_int32), ("start", C.c_float), ("end", C.c_float)]


class DebugAutocInfo(C.Structure):
    _fields_ = [("nsec", C.c_uint32), ("lags", C.c_uint32), ("kernel_lags", C.c_uint32), ("lag_stride", C.c_uint32), ("route", C.c_int32)]


class EncoderConfig(C.Structure):
    _fields_ = [
        ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("sample_rate", C.c_uint32), ("blocksize", C.c_uint32),
        ("do_mid_side_stereo", C.c_int32), ("loose_mid_side_stereo", C.c_int32),
        ("max_lpc_order", C.c_uint32), ("qlp_coeff_precision", C.c_uint32),
        ("do_qlp_coeff_prec_search", C.c_int32), ("do_exhaustive_model_search", C.c_int32),
        ("min_residual_partition_order", C.c_uint32), ("max_residual_partition_order", C.c_uint32),
        ("num_apodizations", C.c_uint32), ("apodizations", Apodization * 32),
        ("disable_constant_subframes", C.c_int32), ("disable_fixed_subframes", C.c_int32),
        ("disable_verbatim_subframes", C.c_int32), ("limit_min_bitrate", C.c_int32), ("x86_avx2_fixed_guess", C.c_int32),
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


class CandDesc(C.Structure):
    """Mirror of fb200::CandDesc: one LPC candidate slot of k_lpc (debug_lpc)."""
    _fields_ = [
        ("valid", C.c_int32), ("order", C.c_int32), ("precision", C.c_int32), ("shift", C.c_int32),
        ("wide", C.c_int32), ("limit", C.c_int32), ("pad0", C.c_int32), ("pad1", C.c_int32),
        ("qlp", C.c_int32 * MAX_LPC_ORDER),
    ]


class SubframeInfo(C.Structure):
    """Mirror of fb200_subframe_info (what FLAC__Frame.subframes[] carries)."""
    _fields_ = [("type", C.c_uint8), ("order", C.c_uint8), ("wasted_bits", C.c_uint8), ("qlp_coeff_precision", C.c_uint8),
                ("quantization_level", C.c_int8), ("entropy_method", C.c_uint8), ("partition_order", C.c_uint8), ("reserved", C.c_uint8),
                ("qlp_coeff", C.c_int32 * MAX_LPC_ORDER), ("warmup", C.c_int32 * MAX_LPC_ORDER)]


class FileInfo(C.Structure):
    """Mirror of fb200_file_info: one file of an encode_files batch."""
    _fields_ = [("first_frame", C.c_uint64), ("nframes", C.c_uint32), ("streaminfo", C.c_uint8 * 34)]


class FlacFileInfo(C.Structure):
    """Mirror of fb200_flac_file_info: one complete .flac file of an encode_flac_files batch."""
    _fields_ = [("offset", C.c_uint64), ("bytes", C.c_uint64), ("audio_offset", C.c_uint64), ("first_frame", C.c_uint64),
                ("nframes", C.c_uint32), ("seek_points", C.c_uint32), ("streaminfo", C.c_uint8 * 34), ("reserved", C.c_uint8 * 6)]


class PcmFileInfo(C.Structure):
    """Mirror of fb200_pcm_file_info: what fb200_pcm_files_probe found in one WAV / RF64 / Wave64 / AIFF / AIFF-C file."""
    _fields_ = [("status", C.c_uint32), ("kind", C.c_uint32), ("channels", C.c_uint32), ("container_bits", C.c_uint32), ("shift", C.c_uint32),
                ("bits_per_sample", C.c_uint32), ("sample_rate", C.c_uint32), ("is_unsigned", C.c_uint32), ("is_big_endian", C.c_uint32),
                ("channel_mask", C.c_uint32), ("data_offset", C.c_uint64), ("declared", C.c_uint64), ("samples", C.c_uint64),
                ("error_", C.c_char * 96)]

    @property
    def error(self):
        return self.error_.decode(errors="replace")


class PcmEncodeOptions(C.Structure):
    _fields_ = [("seek_spacing_s", C.c_int32), ("padding", C.c_int32), ("md5", C.c_uint32), ("replay_gain", C.c_uint32)]


class ReplayGainFile(C.Structure):
    """fb200_replaygain_file: one file of device PCM for fb200_replaygain_device."""
    _fields_ = [("first_value", C.c_uint64), ("samples", C.c_uint64), ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32),
                ("sample_rate", C.c_uint32), ("album", C.c_uint32)]


class ReplayGainInfo(C.Structure):
    """fb200_replaygain_info: the values the REPLAYGAIN_* tags print, and the file's 50 ms windows."""
    _fields_ = [("track_gain", C.c_float), ("track_peak", C.c_float), ("album_gain", C.c_float), ("album_peak", C.c_float), ("windows", C.c_uint64)]


class FlacReencodeOptions(C.Structure):
    _fields_ = [("seek_spacing_s", C.c_int32), ("padding", C.c_int32), ("replay_gain", C.c_uint32), ("reserved", C.c_uint32)]


class FlacReencodeInfo(C.Structure):
    """Mirror of fb200_flac_reencode_info: one listed file of a reencode_flac_files call."""
    _fields_ = [("status", C.c_uint32), ("error_", C.c_char * 92), ("file", FlacFileInfo)]

    @property
    def error(self):
        return self.error_.decode(errors="replace")


REENCODE_OK, REENCODE_INPUT, REENCODE_NO_TOTAL, REENCODE_DAMAGED, REENCODE_MD5_MISMATCH, REENCODE_METADATA = range(6)


class AddReplayGainOptions(C.Structure):
    _fields_ = [("scan_only", C.c_uint32), ("whole_files", C.c_uint32), ("reserved", C.c_uint32)]


class AddReplayGainInfo(C.Structure):
    """Mirror of fb200_add_replaygain_info: one listed file of an add_replay_gain call."""
    _fields_ = [("status", C.c_uint32), ("album", C.c_uint32), ("error_", C.c_char * 88), ("rg", ReplayGainInfo), ("offset", C.c_uint64),
                ("bytes", C.c_uint64), ("head_bytes", C.c_uint64), ("audio_offset_in", C.c_uint64), ("in_place", C.c_uint32), ("pad", C.c_uint32)]

    @property
    def error(self):
        return self.error_.decode(errors="replace")


ADD_RG_OK, ADD_RG_INPUT, ADD_RG_FORMAT, ADD_RG_DECODE, ADD_RG_ALBUM, ADD_RG_METADATA, ADD_RG_NOT_WRITTEN = range(7)
ADD_REPLAYGAIN_GROWTH = 256  # FB200_ADD_REPLAYGAIN_GROWTH

PCM_OK, PCM_NOT_CONTAINER, PCM_MALFORMED, PCM_UNSUPPORTED = range(4)
PCM_WAVE, PCM_RF64, PCM_WAVE64, PCM_AIFF, PCM_AIFF_C = range(1, 6)


class FileDecodeInfo(C.Structure):
    """Mirror of fb200_file_decode_info: one file of a decode_files batch."""
    _fields_ = [("status", C.c_uint32), ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("sample_rate", C.c_uint32),
                ("min_blocksize", C.c_uint32), ("max_blocksize", C.c_uint32), ("total_samples", C.c_uint64), ("samples", C.c_uint64),
                ("first_value", C.c_uint64), ("nframes", C.c_uint32), ("errors", C.c_uint32), ("samples_missing", C.c_uint64),
                ("md5_state", C.c_int32), ("md5", C.c_uint8 * 16)]


class SampleRange(C.Structure):
    """Mirror of fb200_sample_range: samples [first_sample, first_sample + samples) per channel of one indexed file."""
    _fields_ = [("file", C.c_uint32), ("reserved", C.c_uint32), ("first_sample", C.c_uint64), ("samples", C.c_uint64)]


class RangeDecodeInfo(C.Structure):
    """Mirror of fb200_range_decode_info: one range of a decode_ranges call."""
    _fields_ = [("status", C.c_uint32), ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32), ("nframes", C.c_uint32),
                ("first_value", C.c_uint64), ("values", C.c_uint64), ("samples_missing", C.c_uint64), ("candidates", C.c_uint64)]


class FileVerifyInfo(C.Structure):
    """Mirror of fb200_file_verify_info: the verify record of one file of an encode_files call (its first failing frame)."""
    _fields_ = [("status", C.c_uint32), ("frame_number", C.c_uint32), ("frame_status", C.c_uint32), ("channel", C.c_uint32),
                ("sample", C.c_uint32), ("reserved", C.c_uint32), ("absolute_sample", C.c_uint64), ("expected", C.c_int32), ("got", C.c_int32)]


VERIFY_OK, VERIFY_DECODER_ERROR, VERIFY_MISMATCH = range(3)
VERIFY_WRONG_FRAME = 10  # frame_status: the coded frame number or blocksize is not this frame's
PERTURB_FRAME_BYTE, PERTURB_INPUT = 0, 1

FILE_OK, FILE_NOT_FLAC, FILE_NO_STREAMINFO, FILE_BAD_STREAMINFO, FILE_UNSUPPORTED, FILE_WIDTH, FILE_TOO_BIG, FILE_NO_TOTAL = range(8)


class PcmDecodeOptions(C.Structure):
    """Mirror of fb200_pcm_decode_options: the container kind and subformat flac -d writes, MD5 checking, --channel-map=none."""
    _fields_ = [("kind", C.c_uint32), ("subformat", C.c_uint32), ("md5", C.c_uint32), ("channel_map_none", C.c_uint32)]


class PcmDecodeInfo(C.Structure):
    """Mirror of fb200_pcm_decode_info: one container of a decode_pcm_files call."""
    _fields_ = [("status", C.c_uint32), ("tool_ok", C.c_uint32), ("channels", C.c_uint32), ("bits_per_sample", C.c_uint32),
                ("container_bits", C.c_uint32), ("sample_rate", C.c_uint32), ("channel_mask", C.c_uint32), ("extensible", C.c_uint32),
                ("header_bytes", C.c_uint32), ("reserved", C.c_uint32), ("offset", C.c_uint64), ("bytes", C.c_uint64), ("samples", C.c_uint64),
                ("samples_missing", C.c_uint64), ("nframes", C.c_uint32), ("errors", C.c_uint32), ("md5_state", C.c_int32), ("md5", C.c_uint8 * 16)]


PCM_SUB_AUTO, PCM_SUB_WAVE_PCM, PCM_SUB_WAVE_EXTENSIBLE, PCM_SUB_AIFF_C_NONE, PCM_SUB_AIFF_C_SOWT = range(5)
PCM_KINDS = {"wave": PCM_WAVE, "rf64": PCM_RF64, "wave64": PCM_WAVE64, "aiff": PCM_AIFF, "aiff-c": PCM_AIFF_C}
PCM_SUBFORMATS = {None: PCM_SUB_AUTO, "pcm": PCM_SUB_WAVE_PCM, "extensible": PCM_SUB_WAVE_EXTENSIBLE, "none": PCM_SUB_AIFF_C_NONE,
                  "sowt": PCM_SUB_AIFF_C_SOWT}


def pcm_decode_options(kind="wave", subformat=None, md5=True, channel_map_none=False):
    """PcmDecodeOptions from names: kind "wave", "rf64", "wave64", "aiff" or "aiff-c"; subformat None, "pcm" (legacy WAVE),
    "extensible", "none" or "sowt" (AIFF-C), as flac -d's --force-*-format options select them."""
    return PcmDecodeOptions(PCM_KINDS[kind] if isinstance(kind, str) else kind,
                            PCM_SUBFORMATS[subformat] if subformat is None or isinstance(subformat, str) else subformat,
                            1 if md5 else 0, 1 if channel_map_none else 0)


RGS_LIMIT_NONE, RGS_LIMIT_PEAK, RGS_LIMIT_HARD = range(3)
RGS_APPLIED, RGS_NO_TAGS, RGS_BPS, RGS_GAIN, RGS_NOT_DECODED = range(5)


class ReplayGainSynthesis(C.Structure):
    """Mirror of fb200_replaygain_synthesis: what flac -d --apply-replaygain-which-is-not-lossless[=SPEC] applies, and whether a
    list of whole files is one invocation (per_file 0: the dither generator runs on from file to file) or one per file."""
    _fields_ = [("preamp", C.c_double), ("album", C.c_uint32), ("limiter", C.c_uint32), ("noise_shaping", C.c_uint32), ("per_file", C.c_uint32)]


class ReplayGainSynthesisInfo(C.Structure):
    """Mirror of fb200_replaygain_synthesis_info: the tool's decision for one container and where its dither draws lie."""
    _fields_ = [("status", C.c_uint32), ("album_used", C.c_uint32), ("reference", C.c_double), ("gain", C.c_double), ("peak", C.c_double),
                ("scale", C.c_double), ("first_draw", C.c_uint64), ("draws", C.c_uint64)]


def replaygain_synthesis(spec=None, per_file=False):
    """fb200_replaygain_synthesis_parse: the option's SPEC (None: the option without '='). Raises on a spec the tool rejects."""
    rg = ReplayGainSynthesis()
    _check(lib().fb200_replaygain_synthesis_parse(None if spec is None else spec.encode(), C.byref(rg)))
    rg.per_file = 1 if per_file else 0
    return rg


def replaygain_synthesis_file(blob, spec=None):
    """fb200_replaygain_synthesis_file: the tool's decision and scale for one .flac (its metadata only)."""
    rg = spec if isinstance(spec, ReplayGainSynthesis) else replaygain_synthesis(spec)
    b = np.frombuffer(bytes(blob), dtype=np.uint8)
    info = ReplayGainSynthesisInfo()
    _check(lib().fb200_replaygain_synthesis_file(b.ctypes.data, b.size, C.byref(rg), C.byref(info)))
    return info


def pcm_header(channels, bits_per_sample, sample_rate, samples, channel_mask=0, **opts):
    """fb200_pcm_header: the header flac -d writes for these facts (channel_mask: the file's tag, 0 for none). Raises where the
    tool refuses the kind for this length (code -2)."""
    opt = pcm_decode_options(**opts)
    buf = (C.c_uint8 * 128)()
    n = C.c_uint32(0)
    _check(lib().fb200_pcm_header(C.byref(opt), channels, bits_per_sample, sample_rate, channel_mask, samples, buf, 128, C.byref(n)))
    return bytes(buf[:n.value])

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
    L.fb200_host_x86_avx2_fixed_guess.restype = C.c_int
    L.fb200_host_x86_avx2_fixed_guess.argtypes = []
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
    L.fb200_encode_files_host.restype = C.c_int
    L.fb200_encode_files_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                          C.POINTER(C.c_uint64), C.c_void_p]
    L.fb200_encode_files_device.restype = C.c_int
    L.fb200_encode_files_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                            C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
    L.fb200_encode_flac_files_host.restype = C.c_int
    L.fb200_encode_flac_files_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p]
    L.fb200_encode_flac_files_device.restype = C.c_int
    L.fb200_encode_flac_files_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
    L.fb200_encoder_set_verify.restype = C.c_int
    L.fb200_pcm_files_probe.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p]
    L.fb200_encode_pcm_files_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(PcmEncodeOptions), C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p]
    L.fb200_encode_pcm_files_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(PcmEncodeOptions), C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
    L.fb200_reencode_flac_files_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(FlacReencodeOptions), C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p]
    L.fb200_reencode_flac_files_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(FlacReencodeOptions), C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
    L.fb200_encode_pcm_files_ranges_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(PcmEncodeOptions),
                                                     C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                     C.POINTER(C.c_uint64), C.c_void_p]
    L.fb200_encode_pcm_files_ranges_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(PcmEncodeOptions),
                                                       C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                       C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
    L.fb200_reencode_flac_files_ranges_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(FlacReencodeOptions),
                                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p]
    L.fb200_reencode_flac_files_ranges_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(FlacReencodeOptions),
                                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_uint64),
                                                          C.c_void_p, C.c_void_p]
    L.fb200_skip_until.restype = C.c_int
    L.fb200_skip_until.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.fb200_encoder_set_verify.argtypes = [C.c_void_p, C.c_int]
    L.fb200_replaygain_device.restype = C.c_int
    L.fb200_replaygain_device.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.fb200_debug_replaygain_windows.restype = C.c_int
    L.fb200_debug_replaygain_windows.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                                 C.POINTER(C.c_uint64), C.c_void_p]
    L.fb200_replaygain_rewrite_head.restype = C.c_int
    L.fb200_replaygain_rewrite_head.argtypes = [C.c_void_p, C.c_uint64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_uint64,
                                                C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    L.fb200_pcm_header.restype = C.c_int
    L.fb200_replaygain_synthesis_parse.restype = C.c_int
    L.fb200_replaygain_synthesis_parse.argtypes = [C.c_char_p, C.POINTER(ReplayGainSynthesis)]
    L.fb200_replaygain_synthesis_file.restype = C.c_int
    L.fb200_replaygain_synthesis_file.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(ReplayGainSynthesis), C.POINTER(ReplayGainSynthesisInfo)]
    L.fb200_debug_tanh.restype = C.c_int
    L.fb200_debug_tanh.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int]
    L.fb200_debug_replaygain_synthesis.restype = C.c_int
    L.fb200_debug_replaygain_synthesis.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_double,
                                                   C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p]
    L.fb200_pcm_header.argtypes = [C.POINTER(PcmDecodeOptions), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint32,
                                   C.POINTER(C.c_uint32)]
    L.fb200_encoder_get_verify.restype = C.c_int
    L.fb200_encoder_get_verify.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.fb200_debug_perturb_verify.restype = C.c_int
    L.fb200_debug_perturb_verify.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    L.fb200_encoder_set_profiling.restype = C.c_int
    L.fb200_encoder_set_profiling.argtypes = [C.c_void_p, C.c_int]
    L.fb200_encoder_get_profile.restype = C.c_int
    L.fb200_encoder_get_profile.argtypes = [C.c_void_p, C.POINTER(C.c_double * 7), C.POINTER(C.c_uint64 * 7), C.c_int]
    L.fb200_debug_copy_plans.restype = C.c_int
    L.fb200_debug_evaluate_lpc.restype = C.c_int
    L.fb200_debug_evaluate_lpc.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                           C.c_uint32, C.c_uint32, C.c_void_p]
    L.fb200_debug_lpc.restype = C.c_int
    L.fb200_debug_lpc.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                  C.c_uint32, C.c_int, C.c_int, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32)]
    L.fb200_debug_copy_plans.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p]
    L.fb200_debug_copy_autoc.restype = C.c_int
    L.fb200_debug_copy_autoc.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                         C.POINTER(DebugAutocInfo)]
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
        L.fb200_decode_files_index.restype = C.c_int
        L.fb200_decode_files_index.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]
        L.fb200_decode_files_host.restype = C.c_int
        L.fb200_decode_files_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_void_p]
        L.fb200_decode_files_device.restype = C.c_int
        L.fb200_decode_files_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
        L.fb200_decode_files_ranges_host.restype = C.c_int
        L.fb200_decode_files_ranges_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64),
                                                     C.c_void_p]
        L.fb200_decode_files_ranges_device.restype = C.c_int
        L.fb200_decode_files_ranges_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                                       C.c_void_p, C.c_void_p]
        L.fb200_decode_pcm_files_host.restype = C.c_int
        L.fb200_decode_pcm_files_host.argtypes = [C.c_void_p, C.POINTER(PcmDecodeOptions), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                                  C.POINTER(C.c_uint64), C.c_void_p]
        L.fb200_decode_pcm_files_device.restype = C.c_int
        L.fb200_decode_pcm_files_device.argtypes = [C.c_void_p, C.POINTER(PcmDecodeOptions), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                                    C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
        L.fb200_decode_pcm_files_replaygain_host.restype = C.c_int
        L.fb200_decode_pcm_files_replaygain_host.argtypes = [C.c_void_p, C.POINTER(PcmDecodeOptions), C.POINTER(ReplayGainSynthesis), C.c_void_p,
                                                             C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p]
        L.fb200_decode_pcm_files_replaygain_device.restype = C.c_int
        L.fb200_decode_pcm_files_replaygain_device.argtypes = [C.c_void_p, C.POINTER(PcmDecodeOptions), C.POINTER(ReplayGainSynthesis), C.c_void_p,
                                                               C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p,
                                                               C.c_void_p]
        L.fb200_add_replaygain_flac_files_host.restype = C.c_int
        L.fb200_add_replaygain_flac_files_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(AddReplayGainOptions),
                                                           C.c_void_p, C.c_size_t, C.c_void_p]
        L.fb200_add_replaygain_flac_files_device.restype = C.c_int
        L.fb200_add_replaygain_flac_files_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(AddReplayGainOptions),
                                                             C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.fb200_debug_add_replaygain_windows.restype = C.c_int
        L.fb200_debug_add_replaygain_windows.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                                         C.POINTER(C.c_uint64)]
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


def flac_file(streaminfo, frames):
    """A minimal .flac file: the "fLaC" marker, STREAMINFO as the last metadata block, then the frames."""
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + bytes(streaminfo) + b"".join(frames)


METADATA_PADDING, METADATA_APPLICATION, METADATA_SEEKTABLE, METADATA_VORBIS_COMMENT, METADATA_CUESHEET, METADATA_PICTURE = range(1, 7)


def metadata_block(type, body, last=False):
    """One metadata block in stream syntax: the 4-byte header (last flag, type, 24-bit length), then the body."""
    body = bytes(body)
    assert 0 <= type < 128 and len(body) < 1 << 24
    return bytes([(0x80 if last else 0) | type]) + len(body).to_bytes(3, "big") + body


def padding_block(n):
    return metadata_block(METADATA_PADDING, bytes(n))


def vorbis_comment_block(comments, vendor=b""):
    """A VORBIS_COMMENT of "NAME=value" entries (str or bytes); the encoder replaces the vendor string with its own."""
    ent = [c.encode() if isinstance(c, str) else bytes(c) for c in comments]
    body = len(vendor).to_bytes(4, "little") + vendor + len(ent).to_bytes(4, "little")
    return metadata_block(METADATA_VORBIS_COMMENT, body + b"".join(len(e).to_bytes(4, "little") + e for e in ent))


SEEKPOINT_PLACEHOLDER = (1 << 64) - 1


def seektable_block(points):
    """A SEEKTABLE of (sample_number, stream_offset, frame_samples) points, 18 big-endian bytes each."""
    return metadata_block(METADATA_SEEKTABLE, b"".join(s.to_bytes(8, "big") + o.to_bytes(8, "big") + n.to_bytes(2, "big") for s, o, n in points))


def seektable_template(spacing, total):
    """The template points FLAC__metadata_object_seektable_template_append_spaced_points_by_samples(spacing, total) makes
    (what flac -S <spacing>s uses): one at every multiple of spacing below total, at most 32768 of them."""
    if spacing <= 0 or total <= 0:
        return []
    num = 1 + total // spacing - (1 if total % spacing == 0 else 0)
    if num > 32768:
        num, spacing = 32768, total // 32768
    return [(j * spacing, 0, 0) for j in range(num)]


def _batch(blobs):
    """A list of files (bytes-like) -> (one uint8 array of them back to back, offsets[n + 1])."""
    parts = [bytes(b) for b in blobs]
    offs = np.cumsum([0] + [len(p) for p in parts], dtype=np.uint64)
    return np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8), offs


def probe_pcm_files(blobs, data=None, offsets=None):
    """fb200_pcm_files_probe: one PcmFileInfo per WAV / RF64 / Wave64 / AIFF / AIFF-C file (status PCM_OK or why not). Give
    `data` / `offsets` (a batch already laid out back to back) instead of blobs to probe it in place."""
    if data is None:
        data, offsets = _batch(blobs)
    n = len(offsets) - 1
    arr = (PcmFileInfo * max(n, 1))()
    _check(lib().fb200_pcm_files_probe(data.ctypes.data, int(offsets[-1]), offsets.ctypes.data, n, arr))
    return list(arr[:n])


def skip_until(skip, until, rate, total):
    """flac --skip=skip --until=until (str each, None = not given) for a stream of `total` samples per channel at `rate` Hz:
    (first_sample, samples) as the tool computes them. Raises FlacB200Error (code -3, the tool's message) where the tool
    refuses the pair, and for a range of 0 samples."""
    first, n = C.c_uint64(0), C.c_uint64(0)
    enc = lambda v: None if v is None else str(v).encode()
    _check(lib().fb200_skip_until(enc(skip), enc(until), rate, total, C.byref(first), C.byref(n)))
    return first.value, n.value


def _tags(tags, nfiles):
    """None, one list of "NAME=value" for every file, or one list per file -> (blob, offsets[nfiles + 1]) or (None, None)."""
    if tags is None:
        return None, None
    per = [tags] * nfiles if (len(tags) == 0 or isinstance(tags[0], (str, bytes))) else list(tags)
    assert len(per) == nfiles
    parts = [b"".join((t.encode() if isinstance(t, str) else bytes(t)) + b"\0" for t in ts) for ts in per]
    return np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8), np.cumsum([0] + [len(p) for p in parts], dtype=np.uint64)


def encode_pcm_files(blobs, level=5, device=0, **config):
    """flac *.wav: every WAV / RF64 / Wave64 / AIFF / AIFF-C file in `blobs` to the .flac file the flac tool writes for it.
    Files are grouped by (channels, bits per sample, rate), one Encoder(preset(..., level, **config)) per group and one call
    each; the Encoder.encode_pcm_files options (tags, seek_spacing_s, padding, md5, replay_gain) may be given too. With
    replay_gain the files are one album, as one invocation of the tool makes them: they must share one encoder configuration
    (ValueError otherwise). Returns, in input order, (flac bytes, None) per file encoded, or (None, reason) for a file the probe
    did not pass."""
    opts = {k: config.pop(k) for k in ("tags", "seek_spacing_s", "padding", "md5", "replay_gain") if k in config}
    blobs = [bytes(b) for b in blobs]
    infos = probe_pcm_files(blobs)
    res = [(None, f"{i.error}") for i in infos]
    groups = {}
    for f, i in enumerate(infos):
        if i.status == PCM_OK:
            groups.setdefault((i.channels, i.bits_per_sample, i.sample_rate), []).append(f)
    if opts.get("replay_gain") and len(groups) > 1:
        raise ValueError(f"replay_gain makes one album of one call, and these files need {len(groups)} encoder configurations: {sorted(groups)}")
    for (ch, bps, rate), idx in groups.items():
        enc = Encoder(preset(ch, bps, rate, level, **config), device=device)
        try:
            kw = dict(opts)
            if isinstance(kw.get("tags"), list) and kw["tags"] and not isinstance(kw["tags"][0], (str, bytes)):
                kw["tags"] = [kw["tags"][f] for f in idx]
            out = enc.encode_pcm_files([blobs[f] for f in idx], **kw)
        finally:
            enc.close()
        for f, o in zip(idx, out):
            res[f] = (o, None)
    return res


def reencode_flac_files(blobs, level=5, device=0, **config):
    """flac -f *.flac: every .flac file in `blobs` re-encoded to the .flac file the flac tool writes from it. The files are
    indexed once by one Decoder, grouped by (channels, bits per sample, rate), and re-encoded by one Encoder(preset(..., level,
    **config)) per group, one call each; the Encoder.reencode_flac_files options (tags, seek_spacing_s, padding, replay_gain) may
    be given too. With replay_gain the files are one album: they must share one encoder configuration (ValueError otherwise).
    Returns, in input order, (flac bytes, None) per file re-encoded, or (None, reason) for a file that failed."""
    opts = {k: config.pop(k) for k in ("tags", "seek_spacing_s", "padding", "replay_gain") if k in config}
    blobs = [bytes(b) for b in blobs]
    dec = Decoder(2, 16, 44100, 4096, device=device)
    try:
        infos, _ = dec.index_files(blobs)
        res = [(None, f"index status {i.status}") for i in infos]
        groups = {}
        for f, i in enumerate(infos):
            if i.status == FILE_OK:
                groups.setdefault((i.channels, i.bits_per_sample, i.sample_rate), []).append(f)
        if opts.get("replay_gain") and len(groups) > 1:
            raise ValueError(f"replay_gain makes one album of one call, and these files need {len(groups)} encoder configurations: {sorted(groups)}")
        for (ch, bps, rate), idx in groups.items():
            enc = Encoder(preset(ch, bps, rate, level, **config), device=device)
            try:
                kw = dict(opts)
                if isinstance(kw.get("tags"), list) and kw["tags"] and not isinstance(kw["tags"][0], (str, bytes)):
                    kw["tags"] = [kw["tags"][f] for f in idx]
                out, rinfo = enc.reencode_flac_files(dec, idx, infos=True, **kw)
            finally:
                enc.close()
            for f, o, r in zip(idx, out, rinfo):
                res[f] = (o, None) if r.status == REENCODE_OK else (None, r.error)
        return res
    finally:
        dec.close()


def _replaygain_files(files):
    arr = (ReplayGainFile * max(len(files), 1))()
    for k, f in enumerate(files):
        arr[k] = f if isinstance(f, ReplayGainFile) else ReplayGainFile(*f)
    return arr


def replaygain_device(d_pcm_ptr, pcm_values, files, device=0, stream=0):
    """fb200_replaygain_device: ReplayGain of int32 device PCM in decode_files_device's layout. files: ReplayGainFile or
    (first_value, samples, channels, bits_per_sample, sample_rate, album) per file; files with the same album id form an album.
    Returns [ReplayGainInfo per file]."""
    arr = _replaygain_files(files)
    info = (ReplayGainInfo * max(len(files), 1))()
    _check(lib().fb200_replaygain_device(device, d_pcm_ptr, pcm_values, arr, len(files), info, C.c_void_p(stream)))
    return list(info[:len(files)])


def debug_evaluate_lpc(signals, meta, cands, min_po, max_po, rice_limit, device=0):
    """Test hook fb200_debug_evaluate_lpc: the general search kernel's estimate of cands[i] (int32 [n, 40] CandDesc words, as
    debug_lpc returns them) on signals[i] (int32 [n, blocksize]) with meta[i] = (wasted bits, subframe bps); 0xffffffff when
    the candidate is rejected."""
    s = np.ascontiguousarray(signals, dtype=np.int32)
    m = np.ascontiguousarray(meta, dtype=np.int32).reshape(-1, 2)
    c = np.ascontiguousarray(cands, dtype=np.int32).reshape(-1, C.sizeof(CandDesc) // 4)
    n, bs = s.shape
    assert m.shape[0] == n and c.shape[0] == n
    est = np.zeros(n, dtype=np.uint32)
    _check(lib().fb200_debug_evaluate_lpc(device, s.ctypes.data, m.ctypes.data, c.ctypes.data, C.sizeof(CandDesc), n, bs, min_po, max_po,
                                          rice_limit, est.ctypes.data))
    return est


def debug_lpc(autoc, meta, cands, max_order, qlp_precision, prec_search, exhaustive, blocksize, autoc_unshifted=False, device=0):
    """Test hook fb200_debug_lpc: the encoder's LPC analysis kernel on given autocorrelations.
    autoc: float64 [nsec, nitems, lag_stride]; meta: int [nitems, 2] (wasted bits, subframe bps); cands: int [nwin, 3] (kind, sec,
    root). Returns int32 [nitems, nwin * slots per window, 40]: each slot's CandDesc fields in order (valid, order, precision,
    shift, wide, limit, two pad words, qlp[32])."""
    a = np.ascontiguousarray(autoc, dtype=np.float64)
    m = np.ascontiguousarray(meta, dtype=np.int32).reshape(-1, 2)
    c = np.ascontiguousarray(cands, dtype=np.int32).reshape(-1, 3)
    nsec, nitems, lag_stride = a.shape
    assert m.shape[0] == nitems
    per_item = c.shape[0] * (max_order if exhaustive else 1) * (15 - 5 + 1 if prec_search else 1)
    out = (CandDesc * (nitems * per_item))()
    nslots = C.c_uint32(0)
    _check(lib().fb200_debug_lpc(device, a.ctypes.data, nsec, lag_stride, m.ctypes.data, c.ctypes.data, c.shape[0], nitems, max_order,
                                 qlp_precision, int(prec_search), int(exhaustive), blocksize, int(autoc_unshifted), out,
                                 C.sizeof(CandDesc), C.byref(nslots)))
    assert nslots.value == per_item
    return np.frombuffer(out, dtype=np.int32).reshape(nitems, per_item, C.sizeof(CandDesc) // 4).copy()


def debug_replaygain_windows(d_pcm_ptr, pcm_values, files, capacity, device=0, stream=0):
    """fb200_debug_replaygain_windows: every window's mean square, file after file (float64 array)."""
    arr = _replaygain_files(files)
    out = np.empty(max(int(capacity), 1), dtype=np.float64)
    n = C.c_uint64(0)
    _check(lib().fb200_debug_replaygain_windows(device, d_pcm_ptr, pcm_values, arr, len(files), out.ctypes.data, int(capacity), C.byref(n),
                                                C.c_void_p(stream)))
    return out[:n.value]


def replaygain_rewrite_head(flac, track_gain, track_peak, album_gain, album_peak):
    """fb200_replaygain_rewrite_head: the head metaflac --add-replay-gain writes for one .flac file (bytes) with these values.
    Returns (head bytes, audio_offset_in, in_place); raises FlacB200Error when metaflac's chain would refuse the file."""
    flac = bytes(flac)
    cap = len(flac) + ADD_REPLAYGAIN_GROWTH
    head = np.empty(cap, dtype=np.uint8)
    n, audio, in_place = C.c_uint64(), C.c_uint64(), C.c_uint32()
    _check(lib().fb200_replaygain_rewrite_head(flac, len(flac), track_gain, track_peak, album_gain, album_peak, head.ctypes.data, cap, C.byref(n),
                                               C.byref(audio), C.byref(in_place)))
    return head[:n.value].tobytes(), audio.value, bool(in_place.value)


def add_replay_gain(blobs, albums=None, device=0):
    """metaflac --add-replay-gain, one invocation per album: every .flac file in `blobs` indexed once and tagged in one call.
    albums: an album id per file (None: one album). Returns, in input order, (new file bytes or None, AddReplayGainInfo)."""
    blobs = [bytes(b) for b in blobs]
    dec = Decoder(2, 16, 44100, 4096, device=device)
    try:
        dec.index_files(blobs)
        out, infos = dec.add_replay_gain(list(range(len(blobs))), albums=albums, whole_files=True)
        return [(o if i.status == ADD_RG_OK else None, i) for o, i in zip(out, infos)]
    finally:
        dec.close()


def decode_pcm_files(blobs, kind="wave", device=0, **opts):
    """flac -d *.flac: every .flac file in `blobs` to the container file the flac tool writes for it, in one call (the mirror of
    encode_pcm_files). opts: subformat, md5, ranges, channel_map_none as Decoder.decode_pcm_files takes them. Returns, in input
    order (or range order), (container bytes, PcmDecodeInfo); the bytes are empty when info.status is not FILE_OK."""
    dec = Decoder(2, 16, 44100, 4096, device=device)
    try:
        dec.index_files([bytes(b) for b in blobs])
        return dec.decode_pcm_files(kind=kind, **opts)
    finally:
        dec.close()


def decode_pcm_files_replaygain(blobs, spec=None, per_file=False, kind="wave", device=0, **opts):
    """flac -d --apply-replaygain-which-is-not-lossless[=SPEC] *.flac in one call: as decode_pcm_files, with ReplayGain applied
    where the tool applies it. per_file False: the list is one invocation of the tool (its dither generator runs on from file to
    file, in list order); True: one invocation per file. Returns, in input (or range) order, (container bytes, PcmDecodeInfo,
    ReplayGainSynthesisInfo)."""
    dec = Decoder(2, 16, 44100, 4096, device=device)
    try:
        dec.index_files([bytes(b) for b in blobs])
        return dec.decode_pcm_files_replaygain(spec=spec, per_file=per_file, kind=kind, **opts)
    finally:
        dec.close()


def debug_tanh(x, device=0):
    """fb200_debug_tanh: the device restatement of the host libm's tanh over x (float64)."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.empty_like(x)
    _check(lib().fb200_debug_tanh(x.ctypes.data, y.ctypes.data, x.size, device))
    return y


def debug_replaygain_synthesis(x, blocks, bps, scale, hard_limit, noise_shaping, first_draw=0, device=0):
    """fb200_debug_replaygain_synthesis: apply_gain's val32 for int32 x [samples, channels] delivered in `blocks`."""
    x = np.ascontiguousarray(x, dtype=np.int32)
    b = np.ascontiguousarray(blocks, dtype=np.uint32)
    out = np.empty_like(x)
    _check(lib().fb200_debug_replaygain_synthesis(device, x.ctypes.data, x.shape[1], x.shape[0], b.ctypes.data, b.size, bps, scale,
                                                  1 if hard_limit else 0, noise_shaping, first_draw, out.ctypes.data))
    return out


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


def host_x86_avx2_fixed_guess():
    """1 when libFLAC on this host guesses fixed orders with its x86 AVX2 routine (EncoderConfig.x86_avx2_fixed_guess for the
    frames the flac tool writes here), else 0. Needs no GPU."""
    return int(lib().fb200_host_x86_avx2_fixed_guess())


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

    def files_capacity(self, lengths):
        """(frames, output bytes) that always suffice for encode_files* of files with these lengths."""
        nfr = sum(self.num_frames(int(n)) for n in lengths)
        return nfr, nfr * self.max_frame_bytes + 64

    def encode_files(self, pcm, lengths, bytes_per_sample=4, md5=True):
        """Whole files in one call. pcm: int32 [sum(lengths), channels], the files back to back; crosses to the device as
        bytes_per_sample-byte little-endian samples. Returns one (streaminfo: 34 bytes, [frame bytes, ...]) per file, each
        file numbered and terminated as its own stream (flac_file() makes a .flac of it)."""
        pcm = np.ascontiguousarray(pcm, dtype=np.int32)
        lengths = np.ascontiguousarray(lengths, dtype=np.uint64)
        assert pcm.shape == (int(lengths.sum()), self.cfg.channels)
        data = pack_pcm(pcm, bytes_per_sample)
        nfr, cap = self.files_capacity(lengths)
        out = np.empty(cap, dtype=np.uint8)
        offsets = np.zeros(nfr + 1, dtype=np.uint64)
        infos = (FileInfo * max(lengths.size, 1))()
        nf = C.c_uint64(0)
        _check(lib().fb200_encode_files_host(self._h, data.ctypes.data, bytes_per_sample, lengths.ctypes.data, lengths.size, 1 if md5 else 0,
                                             out.ctypes.data, out.size, offsets.ctypes.data, C.byref(nf), infos))
        res = []
        for f in range(lengths.size):
            i0, n = int(infos[f].first_frame), int(infos[f].nframes)
            res.append((bytes(infos[f].streaminfo), [out[int(offsets[i]):int(offsets[i + 1])].tobytes() for i in range(i0, i0 + n)]))
        return res

    def encode_files_device(self, d_pcm_ptr, lengths, d_out_ptr, out_capacity, d_offsets_ptr, md5=True, stream=0):
        """Device-resident encode_files: int32 PCM, output and offsets[nframes + 1] (uint64) are device pointers. Returns after
        completion with (nframes, [(first_frame, nframes, streaminfo)] per file)."""
        lengths = np.ascontiguousarray(lengths, dtype=np.uint64)
        infos = (FileInfo * max(lengths.size, 1))()
        nf = C.c_uint64(0)
        _check(lib().fb200_encode_files_device(self._h, d_pcm_ptr, lengths.ctypes.data, lengths.size, 1 if md5 else 0, d_out_ptr, out_capacity,
                                               d_offsets_ptr, C.byref(nf), infos, C.c_void_p(stream)))
        return nf.value, [(int(i.first_frame), int(i.nframes), bytes(i.streaminfo)) for i in infos[:lengths.size]]

    @staticmethod
    def _metadata(metadata, nfiles):
        """None, one list of blocks for every file, or one list per file -> (blob, offsets[nfiles + 1]) or (None, None)."""
        if metadata is None:
            return None, None
        per = [metadata] * nfiles if (len(metadata) == 0 or isinstance(metadata[0], (bytes, bytearray))) else list(metadata)
        assert len(per) == nfiles
        parts = [b"".join(bytes(b) for b in blocks) for blocks in per]
        blob = np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8)
        return blob, np.cumsum([0] + [len(p) for p in parts], dtype=np.uint64)

    def flac_files_capacity(self, lengths, metadata=None):
        """Output bytes that always suffice for encode_flac_files* of these files with this metadata."""
        _, cap = self.files_capacity(lengths)
        blob, _ = self._metadata(metadata, len(lengths))
        per_file = 42 + 8 + 64 + 256  # fLaC + STREAMINFO, the default VORBIS_COMMENT with the vendor string
        return cap + len(lengths) * per_file + (0 if blob is None else 2 * blob.size)

    def encode_flac_files(self, pcm, lengths, metadata=None, bytes_per_sample=4, md5=True, infos=False):
        """Whole .flac files in one call: as encode_files, each file written complete -- fLaC, STREAMINFO, the default
        VORBIS_COMMENT unless one is given, the metadata blocks in order (seek table marked), the frames. metadata: None, a list of
        blocks (metadata_block() etc.) for every file, or one such list per file. Returns one bytes per file (with infos=True,
        ([bytes], [FlacFileInfo]))."""
        pcm = np.ascontiguousarray(pcm, dtype=np.int32)
        lengths = np.ascontiguousarray(lengths, dtype=np.uint64)
        assert pcm.shape == (int(lengths.sum()), self.cfg.channels)
        data = pack_pcm(pcm, bytes_per_sample)
        blob, moffs = self._metadata(metadata, lengths.size)
        out = np.empty(self.flac_files_capacity(lengths, metadata), dtype=np.uint8)
        arr = (FlacFileInfo * max(lengths.size, 1))()
        nf = C.c_uint64(0)
        _check(lib().fb200_encode_flac_files_host(self._h, data.ctypes.data, bytes_per_sample, lengths.ctypes.data, lengths.size, 1 if md5 else 0,
                                                  None if blob is None else blob.ctypes.data, None if moffs is None else moffs.ctypes.data,
                                                  out.ctypes.data, out.size, None, C.byref(nf), arr))
        files = [out[int(i.offset):int(i.offset + i.bytes)].tobytes() for i in arr[:lengths.size]]
        return (files, list(arr[:lengths.size])) if infos else files

    def encode_flac_files_device(self, d_pcm_ptr, lengths, d_out_ptr, out_capacity, d_offsets_ptr=None, metadata=None, md5=True, stream=0):
        """Device-resident encode_flac_files: int32 PCM, output and (optional) offsets[nframes + 1] (uint64) are device pointers.
        Returns after completion with (nframes, [FlacFileInfo per file]); file f is out[info.offset, info.offset + info.bytes)."""
        lengths = np.ascontiguousarray(lengths, dtype=np.uint64)
        blob, moffs = self._metadata(metadata, lengths.size)
        arr = (FlacFileInfo * max(lengths.size, 1))()
        nf = C.c_uint64(0)
        _check(lib().fb200_encode_flac_files_device(self._h, d_pcm_ptr, lengths.ctypes.data, lengths.size, 1 if md5 else 0,
                                                    None if blob is None else blob.ctypes.data, None if moffs is None else moffs.ctypes.data,
                                                    d_out_ptr, out_capacity, d_offsets_ptr, C.byref(nf), arr, C.c_void_p(stream)))
        return nf.value, list(arr[:lengths.size])

    def pcm_files_capacity(self, infos, tags=None, padding=-1, replay_gain=False, ranges=None):
        """Output bytes that always suffice for encode_pcm_files* of these probed files (or of these (file, first_sample,
        samples) ranges of them)."""
        if ranges is not None:  # a range naming no file makes the call fail: it needs no room
            q = [(int(f), int(n)) for f, _, n in np.asarray(ranges, dtype=np.uint64).reshape(-1, 3) if f < len(infos)]
            infos = [infos[f] for f, _ in q]
            lengths = declared = [n for _, n in q]
        else:
            lengths, declared = [int(i.samples) for i in infos], [int(i.declared) for i in infos]
        _, cap = self.files_capacity(lengths)
        tb, _ = _tags(tags, len(infos))
        extra = 0
        for i, d in zip(infos, declared):
            points = min(32768, d // max(i.sample_rate // 2, 1) + 1)
            extra += 18 * points + (0 if not padding else padding if padding > 0 else 65536) + 42 + 8 + 64 + 256 + 64 + (190 if replay_gain else 0)
        return cap + extra + (0 if tb is None else tb.size + 4 * tb.size)

    def _pcm_call(self, host, data, offsets, infos, tags, seek_spacing_s, padding, md5, out, out_capacity, frame_offsets, stream=0, replay_gain=False,
                  ranges=None):
        n = len(infos)
        arr = (PcmFileInfo * max(n, 1))(*infos)
        if ranges is not None:
            rarr, nout = Decoder.sample_ranges(ranges)
        else:
            nout = n
        files = (FlacFileInfo * max(nout, 1))()
        tb, toffs = _tags(tags, nout)
        opt = PcmEncodeOptions(seek_spacing_s, padding, 1 if md5 else 0, 1 if replay_gain else 0)
        nf = C.c_uint64(0)
        head = [self._h, data, offsets.ctypes.data, n, arr, C.byref(opt)]
        tail = [None if tb is None else tb.ctypes.data, None if toffs is None else toffs.ctypes.data, out, out_capacity, frame_offsets, C.byref(nf), files]
        if ranges is not None:
            if host:
                _check(lib().fb200_encode_pcm_files_ranges_host(*head, rarr, nout, *tail))
            else:
                _check(lib().fb200_encode_pcm_files_ranges_device(*head, rarr, nout, *tail, C.c_void_p(stream)))
        elif host:
            _check(lib().fb200_encode_pcm_files_host(*head, *tail))
        else:
            _check(lib().fb200_encode_pcm_files_device(*head, *tail, C.c_void_p(stream)))
        return nf.value, list(files[:nout])

    def encode_pcm_files(self, blobs, tags=None, seek_spacing_s=10, padding=-1, md5=True, infos=False, replay_gain=False, ranges=None):
        """flac [-T ...] [-S <n>s] [-P n] [--replay-gain] *.wav in one call: every file (bytes of a WAV / RF64 / Wave64 / AIFF /
        AIFF-C file) must probe OK with this encoder's channels, bits per sample and rate. tags: None, one list of "NAME=value"
        for every file, or one list per file. seek_spacing_s 0 = -S-, padding -1 = the tool's default, 0 = --no-padding.
        replay_gain: the REPLAYGAIN_* tags, the call's files being one album. ranges: None, or (file, first_sample, samples) per
        output ((n, 3) array or list): one .flac per range, as flac --skip=first_sample --until=first_sample+samples writes it
        (tags then per range; only the files a range names must probe OK). Returns one bytes per file or range (with infos=True,
        ([bytes], [FlacFileInfo]))."""
        data, offsets = _batch(blobs)
        pinfo = probe_pcm_files(None, data, offsets)
        out = np.empty(self.pcm_files_capacity(pinfo, tags, padding, replay_gain, ranges), dtype=np.uint8)
        _, files = self._pcm_call(True, data.ctypes.data, offsets, pinfo, tags, seek_spacing_s, padding, md5, out.ctypes.data, out.size, None,
                                  replay_gain=replay_gain, ranges=ranges)
        res = [out[int(i.offset):int(i.offset + i.bytes)].tobytes() for i in files]
        return (res, files) if infos else res

    def encode_pcm_files_device(self, d_data_ptr, offsets, pinfo, d_out_ptr, out_capacity, d_offsets_ptr=None, tags=None, seek_spacing_s=10,
                                padding=-1, md5=True, stream=0, replay_gain=False, ranges=None):
        """Device-resident encode_pcm_files: the files back to back at d_data_ptr (offsets[n + 1] into it, host), probed as
        probe_pcm_files(None, host copy, offsets) found them; out and (optional) frame offsets are device pointers. Returns
        (nframes, [FlacFileInfo per file, or per range with ranges])."""
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        return self._pcm_call(False, d_data_ptr, offsets, pinfo, tags, seek_spacing_s, padding, md5, d_out_ptr, out_capacity, d_offsets_ptr, stream,
                              replay_gain, ranges)

    def reencode_capacity(self, decoder, files, tags=None, seek_spacing_s=-1, padding=-1, replay_gain=False, lengths=None):
        """Output bytes that always suffice for reencode_flac_files* of these files of the decoder's indexed batch (lengths:
        samples encoded per entry when not the files' totals, as for ranges)."""
        infos, sizes = decoder._files_infos, decoder._files_sizes
        if lengths is None:
            lengths = [max(int(infos[f].total_samples), 1) for f in files]
        _, cap = self.files_capacity(lengths)
        tb, _ = _tags(tags, len(files))
        extra = 0
        for f, n in zip(files, lengths):
            i = infos[f]
            points = min(32768, int(n) // max(i.sample_rate // 2, 1) + 1)
            # the input's metadata (at most its file), a new seek table, VORBIS_COMMENT and PADDING
            extra += sizes[f] + 18 * points + max(padding, 65536) + 42 + 8 + 64 + 256 + 64 + (190 if replay_gain else 0)
        return cap + extra + (0 if tb is None else tb.size + 4 * tb.size)

    def _reencode_call(self, host, decoder, files, tags, seek_spacing_s, padding, replay_gain, out, out_capacity, frame_offsets, stream=0, ranges=None):
        if ranges is not None:
            arg, n = Decoder.sample_ranges(ranges)
        else:
            files = np.ascontiguousarray(files, dtype=np.uint32)
            arg, n = files.ctypes.data, files.size
        info = (FlacReencodeInfo * max(n, 1))()
        tb, toffs = _tags(tags, n)
        opt = FlacReencodeOptions(seek_spacing_s, padding, 1 if replay_gain else 0, 0)
        nf = C.c_uint64(0)
        args = [self._h, decoder._h, arg, n, C.byref(opt), None if tb is None else tb.ctypes.data, None if toffs is None else toffs.ctypes.data,
                out, out_capacity, frame_offsets, C.byref(nf), info]
        if ranges is not None:
            fn = lib().fb200_reencode_flac_files_ranges_host if host else lib().fb200_reencode_flac_files_ranges_device
        else:
            fn = lib().fb200_reencode_flac_files_host if host else lib().fb200_reencode_flac_files_device
        _check(fn(*args) if host else fn(*args, C.c_void_p(stream)))
        return nf.value, list(info[:n])

    def reencode_flac_files(self, decoder, files, tags=None, seek_spacing_s=-1, padding=-1, replay_gain=False, infos=False):
        """flac -f [-T ...] [-S ..] [-P n] [--replay-gain] *.flac in one call: files (indices into the batch decoder.index_files
        left resident) re-encoded with this encoder's settings; every one that indexed OK must have its channels, bits per sample
        and rate. seek_spacing_s -1 = no -S (the input's SEEKTABLE kept), 0 = -S-; padding -1 = no -P (the input's PADDING
        merged), 0 = --no-padding. Returns one bytes per file, empty for a file that failed (with infos=True, ([bytes],
        [FlacReencodeInfo]): status REENCODE_* and the reason)."""
        files = [int(f) for f in files]
        out = np.empty(self.reencode_capacity(decoder, files, tags, seek_spacing_s, padding, replay_gain), dtype=np.uint8)
        _, info = self._reencode_call(True, decoder, files, tags, seek_spacing_s, padding, replay_gain, out.ctypes.data, out.size, None)
        res = [out[int(i.file.offset):int(i.file.offset + i.file.bytes)].tobytes() for i in info]
        return (res, info) if infos else res

    def reencode_flac_files_device(self, decoder, files, d_out_ptr, out_capacity, d_offsets_ptr=None, tags=None, seek_spacing_s=-1, padding=-1,
                                   replay_gain=False, stream=0):
        """Device-resident reencode_flac_files: out and (optional) frame offsets are device pointers. Returns (nframes,
        [FlacReencodeInfo per file]); file f is out[info.file.offset, + info.file.bytes) when its status is REENCODE_OK."""
        return self._reencode_call(False, decoder, files, tags, seek_spacing_s, padding, replay_gain, d_out_ptr, out_capacity, d_offsets_ptr, stream)

    def reencode_ranges_capacity(self, decoder, ranges, tags=None, seek_spacing_s=-1, padding=-1, replay_gain=False):
        """Output bytes that always suffice for reencode_flac_ranges* of these (file, first_sample, samples) ranges."""
        q = [(int(f), int(n)) for f, _, n in np.asarray(ranges, dtype=np.uint64).reshape(-1, 3) if f < len(decoder._files_infos)]
        return self.reencode_capacity(decoder, [f for f, _ in q], tags, seek_spacing_s, padding, replay_gain, [n for _, n in q])

    def reencode_flac_ranges(self, decoder, ranges, tags=None, seek_spacing_s=-1, padding=-1, replay_gain=False, infos=False):
        """flac -f --skip --until [-T ...] [-S ..] [-P n] [--replay-gain] *.flac in one call: one .flac per (file, first_sample,
        samples) range ((n, 3) array or list) of the batch decoder.index_files left resident, as the tool writes it for
        --skip=first_sample --until=first_sample+samples; options and results as reencode_flac_files, tags per range."""
        out = np.empty(self.reencode_ranges_capacity(decoder, ranges, tags, seek_spacing_s, padding, replay_gain), dtype=np.uint8)
        _, info = self._reencode_call(True, decoder, None, tags, seek_spacing_s, padding, replay_gain, out.ctypes.data, out.size, None, ranges=ranges)
        res = [out[int(i.file.offset):int(i.file.offset + i.file.bytes)].tobytes() for i in info]
        return (res, info) if infos else res

    def reencode_flac_ranges_device(self, decoder, ranges, d_out_ptr, out_capacity, d_offsets_ptr=None, tags=None, seek_spacing_s=-1, padding=-1,
                                    replay_gain=False, stream=0):
        """Device-resident reencode_flac_ranges. Returns (nframes, [FlacReencodeInfo per range])."""
        return self._reencode_call(False, decoder, None, tags, seek_spacing_s, padding, replay_gain, d_out_ptr, out_capacity, d_offsets_ptr, stream,
                                   ranges=ranges)

    def set_verify(self, on=True):
        """flac -V for encode_files / encode_files_device: every frame is decoded on the device and compared with the input; a
        file that fails makes the call raise FlacB200Error with code ERR_VERIFY (verify_info() then says which and where).
        While on, the block entry points (encode, encode_packed, encode_device) raise with code -2 (UNSUPPORTED)."""
        _check(lib().fb200_encoder_set_verify(self._h, 1 if on else 0))

    def verify_info(self, nfiles):
        """The FileVerifyInfo records of the last encode_files* call (which must have verified nfiles files)."""
        infos = (FileVerifyInfo * max(nfiles, 1))()
        _check(lib().fb200_encoder_get_verify(self._h, infos, nfiles))
        return list(infos[:nfiles])

    def debug_perturb_verify(self, file, what, a, b, xor_mask):
        """Test hook: for the next encode_files* call, flip bits after encoding and before verifying. what=PERTURB_FRAME_BYTE:
        byte b of frame a of the file; what=PERTURB_INPUT: the input value (sample a, channel b) of the file."""
        _check(lib().fb200_debug_perturb_verify(self._h, file, what, a, b, xor_mask))

    PROF_NAMES = ("k_prep", "k_autoc", "k_lpc", "k_search", "k_emit", "k_scan", "k_gather")

    def set_profiling(self, on=True):
        _check(lib().fb200_encoder_set_profiling(self._h, 1 if on else 0))

    def profile(self, reset=True):
        """{kernel: (total_ms, launches)} from CUDA events recorded between the kernels."""
        ms = (C.c_double * 7)()
        n = (C.c_uint64 * 7)()
        _check(lib().fb200_encoder_get_profile(self._h, C.byref(ms), C.byref(n), 1 if reset else 0))
        return {name: (ms[i], int(n[i])) for i, name in enumerate(self.PROF_NAMES)}

    STAGE_A_ROUTES = ("fused", "meta", "planar")

    def debug_autoc(self, nblocks):
        """Test hook fb200_debug_copy_autoc: what stage A left for the first nblocks full blocks of the last encode call. Returns
        a dict: route ("fused" / "meta" / "planar"), lags (LPC lags), kernel_lags (lags each record holds), rows float64
        [nsec, nblocks * nsig, lag_stride] (only [..., :kernel_lags] written), meta int32 [items, 2] (wasted bits, subframe bps),
        sigor uint32 [items] (None off the fused route) and sections int32 [nsec, 5] (win_off, partial, data_len, part_size,
        data_shift)."""
        info = DebugAutocInfo()
        _check(lib().fb200_debug_copy_autoc(self._h, nblocks, None, 0, None, None, None, 0, C.byref(info)))
        nitems = nblocks * self.nsig
        rows = np.full((info.nsec, nitems, info.lag_stride), np.nan)
        meta = np.zeros((nitems, 2), dtype=np.int32)
        sigor = np.zeros(nitems, dtype=np.uint32)
        secs = np.zeros((info.nsec, 5), dtype=np.int32)
        _check(lib().fb200_debug_copy_autoc(self._h, nblocks, rows.ctypes.data, rows.size, meta.ctypes.data, sigor.ctypes.data,
                                            secs.ctypes.data, info.nsec, C.byref(info)))
        route = self.STAGE_A_ROUTES[info.route]
        return dict(route=route, lags=info.lags, kernel_lags=info.kernel_lags, rows=rows, meta=meta,
                    sigor=sigor if route == "fused" else None, sections=secs)

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

    def index_files(self, blobs):
        """Whole .flac files (bytes each): parsed, copied to the device and indexed, resident for decode_files /
        decode_files_device. Returns ([FileDecodeInfo per file], total values of the output)."""
        data = np.frombuffer(b"".join(blobs), dtype=np.uint8)
        offsets = np.cumsum([0] + [len(b) for b in blobs], dtype=np.uint64)
        infos = (FileDecodeInfo * max(len(blobs), 1))()
        total = C.c_uint64(0)
        _check(lib().fb200_decode_files_index(self._h, data.ctypes.data if data.size else None, data.size, offsets.ctypes.data, len(blobs), infos,
                                              C.byref(total)))
        self._files_index = (len(blobs), total.value)
        self._files_infos, self._files_sizes = list(infos[:len(blobs)]), [len(b) for b in blobs]
        return list(infos[:len(blobs)]), total.value

    def decode_files(self, blobs, bytes_per_sample=4, md5=True):
        """Index and decode whole .flac files. Returns per file (pcm, info): int32 [samples, channels] for bytes_per_sample 4,
        else packed little-endian uint8 [samples, channels * bytes_per_sample]."""
        _, total = self.index_files(blobs)
        out = np.empty(total * bytes_per_sample, dtype=np.uint8)
        infos = (FileDecodeInfo * max(len(blobs), 1))()
        _check(lib().fb200_decode_files_host(self._h, out.ctypes.data, bytes_per_sample, total, 1 if md5 else 0, infos))
        res = []
        for i in infos[:len(blobs)]:
            a, n, ch = int(i.first_value) * bytes_per_sample, int(i.samples), max(int(i.channels), 1)
            part = out[a:a + n * ch * bytes_per_sample]
            res.append((part.view(np.int32).reshape(n, ch) if bytes_per_sample == 4 else part.reshape(n, ch * bytes_per_sample), i))
        return res

    def decode_files_device(self, d_pcm_ptr, capacity_values, md5=True, stream=0):
        """Decode the files of the last index_files into int32 device memory (file f at infos[f].first_value). Returns after
        completion with [FileDecodeInfo per file]."""
        n = self._files_index[0] if getattr(self, "_files_index", None) else 0
        infos = (FileDecodeInfo * max(n, 1))()
        _check(lib().fb200_decode_files_device(self._h, d_pcm_ptr, capacity_values, 1 if md5 else 0, infos, C.c_void_p(stream)))
        return list(infos[:n])

    @staticmethod
    def sample_ranges(ranges):
        """(n, 3) array or list of (file, first_sample, samples) -> a SampleRange array."""
        q = np.asarray(ranges, dtype=np.uint64).reshape(-1, 3)
        arr = (SampleRange * max(len(q), 1))()
        for k, (f, s, n) in enumerate(q):
            arr[k].file, arr[k].first_sample, arr[k].samples = int(f), int(s), int(n)
        return arr, len(q)

    def decode_ranges(self, ranges, bytes_per_sample=4):
        """Samples [first_sample, first_sample + samples) of files of the last index_files, each range (file, first_sample, samples)
        of `ranges` ((n, 3) array or list). Returns per range (pcm, info) as decode_files does: int32 [samples, channels] for
        bytes_per_sample 4, else packed little-endian uint8 [samples, channels * bytes_per_sample]; empty for a range whose status
        is not FILE_OK."""
        arr, n = self.sample_ranges(ranges)
        infos = (RangeDecodeInfo * max(n, 1))()
        total = C.c_uint64(0)
        rc = lib().fb200_decode_files_ranges_host(self._h, arr, n, None, bytes_per_sample, 0, C.byref(total), infos)
        if rc not in (FB200_OK, -4):
            _check(rc)
        out = np.empty(max(total.value, 1) * bytes_per_sample, dtype=np.uint8)
        _check(lib().fb200_decode_files_ranges_host(self._h, arr, n, out.ctypes.data, bytes_per_sample, total.value, C.byref(total), infos))
        res = []
        for i in infos[:n]:
            a, ch = int(i.first_value) * bytes_per_sample, max(int(i.channels), 1)
            m = int(i.values) // ch
            part = out[a:a + m * ch * bytes_per_sample]
            res.append((part.view(np.int32).reshape(m, ch) if bytes_per_sample == 4 else part.reshape(m, ch * bytes_per_sample), i))
        return res

    def decode_ranges_device(self, ranges, d_pcm_ptr, capacity_values, stream=0):
        """decode_ranges into int32 device memory (range r at infos[r].first_value). Returns after completion with
        ([RangeDecodeInfo per range], total values)."""
        arr, n = self.sample_ranges(ranges)
        infos = (RangeDecodeInfo * max(n, 1))()
        total = C.c_uint64(0)
        _check(lib().fb200_decode_files_ranges_device(self._h, arr, n, d_pcm_ptr, capacity_values, C.byref(total), infos, C.c_void_p(stream)))
        return list(infos[:n]), total.value

    def _pcm_args(self, kind, subformat, md5, ranges, channel_map_none):
        opt = pcm_decode_options(kind, subformat, md5, channel_map_none)
        if ranges is None:
            n = self._files_index[0] if getattr(self, "_files_index", None) else 0
            return opt, None, 0, n
        arr, n = self.sample_ranges(ranges)
        return opt, arr, n, n

    def decode_pcm_files(self, kind="wave", subformat=None, md5=True, ranges=None, channel_map_none=False):
        """flac -d over the files of the last index_files: one container file per file (ranges None) or per (file, first_sample,
        samples) range (flac -d --skip / --until), as the flac tool writes it for `kind` ("wave", "rf64", "wave64", "aiff",
        "aiff-c") and `subformat` (None, "pcm", "extensible"; "none" or "sowt" for AIFF-C). Returns [(bytes, PcmDecodeInfo)]; the
        bytes are empty when info.status is not FILE_OK. info.tool_ok says whether the tool would keep the file."""
        opt, arr, nr, n = self._pcm_args(kind, subformat, md5, ranges, channel_map_none)
        infos = (PcmDecodeInfo * max(n, 1))()
        total = C.c_uint64(0)
        rc = lib().fb200_decode_pcm_files_host(self._h, C.byref(opt), arr, nr, None, 0, C.byref(total), infos)
        if rc not in (FB200_OK, -4):
            _check(rc)
        out = np.empty(max(total.value, 1), dtype=np.uint8)
        if rc != FB200_OK:
            _check(lib().fb200_decode_pcm_files_host(self._h, C.byref(opt), arr, nr, out.ctypes.data, total.value, C.byref(total), infos))
        return [(out[int(i.offset):int(i.offset) + int(i.bytes)].tobytes(), i) for i in infos[:n]]

    def decode_pcm_files_device(self, d_out_ptr, out_capacity, kind="wave", subformat=None, md5=True, ranges=None, channel_map_none=False,
                                stream=0):
        """decode_pcm_files into device memory (any alignment; container i at infos[i].offset). out_capacity 0 sizes the call.
        Returns after completion with ([PcmDecodeInfo per container], total bytes)."""
        opt, arr, nr, n = self._pcm_args(kind, subformat, md5, ranges, channel_map_none)
        infos = (PcmDecodeInfo * max(n, 1))()
        total = C.c_uint64(0)
        rc = lib().fb200_decode_pcm_files_device(self._h, C.byref(opt), arr, nr, d_out_ptr, out_capacity, C.byref(total), infos, C.c_void_p(stream))
        if not (rc == -4 and out_capacity == 0):
            _check(rc)
        return list(infos[:n]), total.value

    def decode_pcm_files_replaygain(self, spec=None, per_file=False, kind="wave", subformat=None, md5=True, ranges=None, channel_map_none=False):
        """flac -d --apply-replaygain-which-is-not-lossless[=SPEC] over the files of the last index_files: decode_pcm_files with
        ReplayGain applied where the tool applies it (spec None: the option without '='). per_file as decode_pcm_files_replaygain.
        Returns [(bytes, PcmDecodeInfo, ReplayGainSynthesisInfo)]."""
        opt, arr, nr, n = self._pcm_args(kind, subformat, md5, ranges, channel_map_none)
        rg = spec if isinstance(spec, ReplayGainSynthesis) else replaygain_synthesis(spec, per_file)
        infos = (PcmDecodeInfo * max(n, 1))()
        rginfos = (ReplayGainSynthesisInfo * max(n, 1))()
        total = C.c_uint64(0)
        rc = lib().fb200_decode_pcm_files_replaygain_host(self._h, C.byref(opt), C.byref(rg), arr, nr, None, 0, C.byref(total), infos, rginfos)
        if rc not in (FB200_OK, -4):
            _check(rc)
        out = np.empty(max(total.value, 1), dtype=np.uint8)
        if rc != FB200_OK:
            _check(lib().fb200_decode_pcm_files_replaygain_host(self._h, C.byref(opt), C.byref(rg), arr, nr, out.ctypes.data, total.value, C.byref(total),
                                                                infos, rginfos))
        return [(out[int(i.offset):int(i.offset) + int(i.bytes)].tobytes(), i, r) for i, r in zip(infos[:n], rginfos[:n])]

    def decode_pcm_files_replaygain_device(self, d_out_ptr, out_capacity, spec=None, per_file=False, kind="wave", subformat=None, md5=True,
                                           ranges=None, channel_map_none=False, stream=0):
        """decode_pcm_files_replaygain into device memory (container i at infos[i].offset). out_capacity 0 sizes the call. Returns
        after completion with ([PcmDecodeInfo], [ReplayGainSynthesisInfo], total bytes)."""
        opt, arr, nr, n = self._pcm_args(kind, subformat, md5, ranges, channel_map_none)
        rg = spec if isinstance(spec, ReplayGainSynthesis) else replaygain_synthesis(spec, per_file)
        infos = (PcmDecodeInfo * max(n, 1))()
        rginfos = (ReplayGainSynthesisInfo * max(n, 1))()
        total = C.c_uint64(0)
        rc = lib().fb200_decode_pcm_files_replaygain_device(self._h, C.byref(opt), C.byref(rg), arr, nr, d_out_ptr, out_capacity, C.byref(total), infos,
                                                            rginfos, C.c_void_p(stream))
        if not (rc == -4 and out_capacity == 0):
            _check(rc)
        return list(infos[:n]), list(rginfos[:n]), total.value

    def _add_rg_args(self, files, albums, scan, whole_files):
        files = np.ascontiguousarray(files, dtype=np.uint32)
        alb = None if albums is None else np.ascontiguousarray(albums, dtype=np.uint32)
        if alb is not None and alb.size != files.size:
            raise ValueError("albums needs one id per listed file")
        opt = AddReplayGainOptions(1 if scan else 0, 1 if whole_files else 0, 0)
        return files, alb, opt, (AddReplayGainInfo * max(files.size, 1))()

    def add_replay_gain_capacity(self, files):
        """Bytes an add_replay_gain call over `files` may need (FB200_ADD_REPLAYGAIN_GROWTH per file over the input's size)."""
        return sum(self._files_sizes[int(f)] + ADD_REPLAYGAIN_GROWTH for f in files if int(f) < len(self._files_sizes))

    def add_replay_gain(self, files, albums=None, scan=False, whole_files=True):
        """metaflac --add-replay-gain (scan: --scan-replay-gain) over files of the last index_files, one invocation per album id.
        Returns ([bytes per listed file: the complete new file (whole_files) or its new head; empty when not written],
        [AddReplayGainInfo per listed file])."""
        files, alb, opt, infos = self._add_rg_args(files, albums, scan, whole_files)
        cap = 0 if scan else self.add_replay_gain_capacity(files)
        out = np.empty(max(cap, 1), dtype=np.uint8)
        _check(lib().fb200_add_replaygain_flac_files_host(self._h, files.ctypes.data, None if alb is None else alb.ctypes.data, files.size, C.byref(opt),
                                                          out.ctypes.data, cap, infos))
        res = list(infos[:files.size])
        return [out[int(i.offset):int(i.offset) + int(i.bytes)].tobytes() for i in res], res

    def add_replay_gain_device(self, files, d_out_ptr, out_capacity, albums=None, scan=False, whole_files=True, stream=0):
        """add_replay_gain into device memory (file i at infos[i].offset, any alignment). Returns after completion with
        [AddReplayGainInfo per listed file]."""
        files, alb, opt, infos = self._add_rg_args(files, albums, scan, whole_files)
        _check(lib().fb200_add_replaygain_flac_files_device(self._h, files.ctypes.data, None if alb is None else alb.ctypes.data, files.size,
                                                            C.byref(opt), d_out_ptr, out_capacity, infos, C.c_void_p(stream)))
        return list(infos[:files.size])

    def debug_add_replay_gain_windows(self, files, albums=None):
        """fb200_debug_add_replaygain_windows: every window's mean square of the listed files' analysis (float64 array)."""
        files = np.ascontiguousarray(files, dtype=np.uint32)
        alb = None if albums is None else np.ascontiguousarray(albums, dtype=np.uint32)
        cap = sum(int(self._files_infos[int(f)].samples) for f in files) // 400 + 1
        out = np.empty(cap, dtype=np.float64)
        n = C.c_uint64(0)
        _check(lib().fb200_debug_add_replaygain_windows(self._h, files.ctypes.data, None if alb is None else alb.ctypes.data, files.size,
                                                        out.ctypes.data, cap, C.byref(n)))
        return out[:n.value]

    def decode_device(self, d_frames_ptr, d_offsets_ptr, nframes, d_pcm_ptr, pcm_capacity_samples, d_status_ptr, stream=0, sync=False):
        _check(lib().fb200_decode_device(self._h, d_frames_ptr, d_offsets_ptr, nframes, d_pcm_ptr, pcm_capacity_samples, d_status_ptr,
                                         C.c_void_p(stream), 1 if sync else 0))
