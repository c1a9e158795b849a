"""EncoderConfig.x86_avx2_fixed_guess: with 1, subframes libFLAC guesses with its _wide routine take the sums of
FLAC__fixed_compute_best_predictor_wide_intrin_avx2, the routine an x86-64 host with AVX2 runs (DESIGN.md, G4), so the frames are
the oracle's in that mode on every stage-B path and through every entry point, and the files are the flac tool's byte for byte
on either kind of host when the field is set from host_x86_avx2_fixed_guess()."""
import numpy as np
import pytest

import flac_b200 as fb
import oraclelib
import refcli
import reffile
import signals
from test_gpu_encode_ranges import tool as tool_range
from test_gpu_flac_files import vendor
from test_gpu_formats import assert_same, check, fast_blocksize
from test_gpu_lpc_edges import PATHS
from test_gpu_reencode_files import identity_inputs, tool, tool_args, wav_of

pytestmark = pytest.mark.gpu

# (blocksize, samples): short last blocks whose n = bs - 4 has n % 4 of 1, 2 and 3 at 1152 and 4096; the non-standard -b 4095 and
# 1001, whose full blocks have n % 4 == 3 and 1; blocksizes up to 65535 (tiled on the natural path at 65535)
INPUTS = [(1152, 1152 + 900 + r) for r in (1, 2, 3)] + [(4096, 4096 + 3000 + r) for r in (1, 2, 3)] + \
         [(4095, 4095 + 2001), (1001, 2 * 1001 + 502), (16387, 16387 + 4002), (65535, 65535 + 1003)]

_oracle = {}


def oracle_frames(x, bits, rate, level, bs, mode, key):
    k = key + (level, bs, mode)
    if k not in _oracle:
        _oracle[k] = oraclelib.Encoder(oraclelib.preset(x.shape[1], bits, rate, level, bs, x86_avx2_fixed_guess=mode)).encode_stream(x)
    return _oracle[k]


@pytest.mark.parametrize("bits", [16, 20, 24])
@pytest.mark.parametrize("env", PATHS, ids=[p[0] for p in PATHS])
def test_frames_equal_the_oracle_in_both_modes(monkeypatch, env, bits):
    if env[1]:
        monkeypatch.setenv(*env[1])
    differ = 0
    for ch in (1, 2, 6):
        for level in (0, 2, 5, 8):
            for k, (bs, n) in enumerate(INPUTS):
                x = signals.music_like(n, ch, bits, 44100, seed=100 * ch + bits + k)
                want = [oracle_frames(x, bits, 44100, level, bs, m, (ch, bits, k)) for m in (0, 1)]
                differ += sum(a != b for a, b in zip(*want))
                for m in (0, 1):
                    enc = fb.Encoder(fb.preset(ch, bits, 44100, level, bs, x86_avx2_fixed_guess=m), max_blocks_per_launch=4)
                    try:
                        got = enc.encode_frames(x)
                    finally:
                        enc.close()
                    assert_same(got, want[m], f"{env[0]} mode {m} {ch}ch {bits}-bit -{level} bs {bs} n {n}")
    if bits > 16:
        assert differ > 0, f"{env[0]} {bits}-bit: no frame of the matrix differs between the two modes"


STANDARD = [192, 576, 1152, 2304, 4608, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768]


@pytest.mark.parametrize("bs", STANDARD)
def test_full_standard_blocks_are_the_same_in_both_modes(bs):
    """k_search5 takes only blocksizes with bs - 4 a multiple of 4, where the two routines' sums are equal: it has no mode"""
    for ch, bits in ((1, 20), (2, 24)):
        x = signals.music_like(2 * bs, ch, bits, 44100, seed=bs + ch)
        for level in (5, 8):
            c = oracle_frames(x, bits, 44100, level, bs, 0, ("std", ch, bits))
            assert c == oracle_frames(x, bits, 44100, level, bs, 1, ("std", ch, bits)), f"{ch}ch {bits}-bit -{level} bs {bs}"
            path = "fast" if fast_blocksize(bs, level, ch) else "general"
            for m in (0, 1):
                check(x, bits, 44100, level, bs, path, what=f"mode {m}", x86_avx2_fixed_guess=m)


# files whose short last blocks (bs 1152 at -2) the two modes guess differently: the first is the one DESIGN.md's G4 names
ENTRY_LENGTHS = [1152 * 3 + 19, 1152 * 2 + 1001, 1152 + 518]


def entry_files():
    return [signals.music_like(n, 2, 24, 44100, seed=1 + i) for i, n in enumerate(ENTRY_LENGTHS)]


def mode1(x):
    return oraclelib.Encoder(oraclelib.preset(2, 24, 44100, 2, x86_avx2_fixed_guess=1)).encode_stream(x)


def frame_sizes(streaminfo):
    return int.from_bytes(streaminfo[4:7], "big"), int.from_bytes(streaminfo[7:10], "big")


def check_flac(blob, x, what):
    """a .flac's frames are the oracle's mode-1 frames of x, and STREAMINFO's min / max frame size are theirs"""
    want = mode1(x)
    _, ao = reffile.blocks(blob)
    assert blob[ao:] == b"".join(want), f"{what}: frames"
    sizes = [len(f) for f in want]
    assert frame_sizes(blob[8:42]) == (min(sizes), max(sizes)), f"{what}: min / max frame size"


def test_every_entry_point_honours_the_field():
    xs = entry_files()
    assert any(mode1(x) != oraclelib.Encoder(oraclelib.preset(2, 24, 44100, 2)).encode_stream(x) for x in xs), "no file differs"
    pcm, lengths = np.concatenate(xs), [x.shape[0] for x in xs]
    wavs = [wav_of(x, 24, 44100) for x in xs]
    ranges = [(0, 5, 1152 * 2 + 7), (1, 1000, 1001 + 1152), (2, 1, 1152 + 517), (0, 0, lengths[0])]
    enc = fb.Encoder(fb.preset(2, 24, 44100, 2, x86_avx2_fixed_guess=1))
    try:
        for verify in (False, True):
            enc.set_verify(verify)
            what = f"verify {verify}"
            for k, (si, frames) in enumerate(enc.encode_files(pcm, lengths)):
                want = mode1(xs[k])
                assert frames == want, f"encode_files {what} file {k}"
                sizes = [len(f) for f in want]
                assert frame_sizes(si) == (min(sizes), max(sizes)), f"encode_files {what} file {k}: min / max frame size"
            flacs = enc.encode_flac_files(pcm, lengths)
            for k, b in enumerate(flacs):
                check_flac(b, xs[k], f"encode_flac_files {what} file {k}")
            for k, b in enumerate(enc.encode_pcm_files(wavs)):
                check_flac(b, xs[k], f"encode_pcm_files {what} file {k}")
            for (f, a, n), b in zip(ranges, enc.encode_pcm_files(wavs, ranges=ranges)):
                check_flac(b, xs[f][a:a + n], f"encode_pcm_files ranges {what} {(f, a, n)}")
            dec = fb.Decoder(2, 16, 44100, 4096)
            try:
                dec.index_files(flacs)
                for k, b in enumerate(enc.reencode_flac_files(dec, range(len(xs)))):
                    check_flac(b, xs[k], f"reencode_flac_files {what} file {k}")
                for (f, a, n), b in zip(ranges, enc.reencode_flac_ranges(dec, ranges)):
                    check_flac(b, xs[f][a:a + n], f"reencode_flac_ranges {what} {(f, a, n)}")
            finally:
                dec.close()
    finally:
        enc.close()
    # the module-level helpers pass the field through their **config
    for k, (b, err) in enumerate(fb.encode_pcm_files(wavs, 2, x86_avx2_fixed_guess=1)):
        assert err is None, err
        check_flac(b, xs[k], f"flac_b200.encode_pcm_files file {k}")
    for k, (b, err) in enumerate(fb.reencode_flac_files(flacs, 2, x86_avx2_fixed_guess=1)):
        assert err is None, err
        check_flac(b, xs[k], f"flac_b200.reencode_flac_files file {k}")


def need_tool():
    if not refcli.available():
        pytest.skip("oracle/_ref/flac_ref not built")


@pytest.mark.parametrize("level", [0, 5, 8])
def test_six_channel_24_bit_reencode_is_the_tools(level):
    need_tool()
    blobs = identity_inputs(6, 24, 48000)
    out = fb.reencode_flac_files(blobs, level, x86_avx2_fixed_guess=fb.host_x86_avx2_fixed_guess())
    for k, (b, (o, err)) in enumerate(zip(blobs, out)):
        assert err is None, err
        rc, want = tool(b, tool_args(level))
        assert rc == 0 and o == want, f"file {k}"


@pytest.mark.parametrize("level", [0, 5, 8])
@pytest.mark.parametrize("bits,rate", [(20, 48000), (24, 96000)])
def test_wav_encodes_are_the_tools(level, bits, rate):
    need_tool()
    bs = 1152 if level == 0 else 4096
    lengths = [2 * bs + 1001, bs + 2002, 3 * bs + 3003, bs - 2]
    xs = [signals.music_like(n, 2, bits, rate, seed=bits + level + i) for i, n in enumerate(lengths)]
    wavs = [wav_of(x, bits, rate) for x in xs]
    host = fb.host_x86_avx2_fixed_guess()
    for k, (o, err) in enumerate(fb.encode_pcm_files(wavs, level, x86_avx2_fixed_guess=host)):
        assert err is None, err
        rc, want, stderr = refcli.encode(wavs[k], [f"-{level}"])
        assert rc == 0, stderr
        assert o == reffile.with_vendor(want, vendor()), f"file {k}"
    ranges = [(0, 3, bs + 5), (1, bs - 1, 2001), (2, 17, 2 * bs + 1), (3, 0, bs - 3)]
    enc = fb.Encoder(fb.preset(2, bits, rate, level, x86_avx2_fixed_guess=host))
    try:
        got = enc.encode_pcm_files(wavs, ranges=ranges)
    finally:
        enc.close()
    for (f, a, n), o in zip(ranges, got):
        assert o == tool_range(wavs[f], [f"-{level}"], a, n), (f, a, n)


@pytest.mark.parametrize("value", [2, -1])
def test_other_values_are_refused(value):
    with pytest.raises(fb.FlacB200Error) as ei:
        fb.Encoder(fb.preset(2, 16, 44100, 5, x86_avx2_fixed_guess=value))
    assert ei.value.code == -3
