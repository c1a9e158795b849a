"""fb200_decode_pcm_files_replaygain_* against the reference: fb_tanh against the host libm's tanh bit for bit, k_rg_synth
against the unmodified replaygain_synthesis.c (oracle/_ref/libFLAC_ref_rgsynth.so) on constructed blocks, and every container
against the flac tool's `flac -d --apply-replaygain-which-is-not-lossless[=SPEC]` output, one tool process over a list of files
(per_file 0) or one per file (per_file 1), with damaged files and sample ranges."""
import numpy as np
import pytest

import flac_b200 as fb
import refcli
import refrgsynth
import signals
from rgsfiles import add_vorbis_comment, album_tags, tagged_flac, tool_decode_many
from test_gpu_decode_files import variable_stream
from test_pcm_header import FORMATS, with_total_zero

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (refcli.available() and refrgsynth.available()), reason="reference binaries not built")]

FLAGS = {(k, s): f for k, s, f in FORMATS}


def test_tanh_bit_exact_against_host_libm():
    rng = np.random.default_rng(3)
    parts = [rng.uniform(0, 22, 6_000_000)]
    for c in (0.0, 0.5, 1.0, 22.0, 0.5 * np.log(2) / 2, 1.5 * np.log(2) / 2, 28 * np.log(2) / 2):
        parts.append(c + rng.uniform(-1e-3, 1e-3, 500_000))
        parts.append(c + rng.uniform(-1e-9, 1e-9, 100_000))
    parts.append(np.ldexp(rng.uniform(0.5, 1, 200_000), -rng.integers(1, 1070, 200_000)))  # tiny and subnormal
    parts.append(-rng.uniform(0, 30, 200_000))
    parts.append(np.array([0.0, -0.0, 5e-324, 2.0 ** -55, 2.0 ** -54, 22.0, np.inf, -np.inf]))
    x = np.concatenate(parts)
    assert x.size >= 10_000_000
    got, want = fb.debug_tanh(x), refrgsynth.tanh(x)
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert bad.size == 0, f"{bad.size} of {x.size} differ, e.g. x={x[bad[0]]!r}: device {got[bad[0]].hex()} host {want[bad[0]].hex()}"


def constructed(n, ch, bps, rng):
    lim = 1 << (bps - 1)
    x = rng.integers(-lim, lim, (n, ch), dtype=np.int64)
    edges = np.array([lim - 1, -lim, 0, 1, -1, lim - 2, -lim + 1])
    k = min(n, 64)
    x[:k] = edges[rng.integers(0, edges.size, (k, ch))]
    return x.astype(np.int32)


def mixed_blocks(n, rng):
    pool = [1, 31, 32, 33, 4096, 65535]
    out, left = [], n
    while left:
        b = min(left, int(pool[rng.integers(0, len(pool))]))
        out.append(b)
        left -= b
    return out


SCALES = [10 ** (-90 / 20), 10 ** (-6 / 20), 1.0, 10 ** (6 / 20), 10 ** (18 / 20), 10 ** (90 / 20)]


@pytest.mark.parametrize("shaping", [0, 1, 2, 3])
@pytest.mark.parametrize("hard", [False, True])
def test_synthesis_equals_the_reference(shaping, hard):
    rng = np.random.default_rng(shaping * 2 + hard)
    for bps in range(4, 25):
        ch = int(rng.integers(1, 9))
        n = int(rng.integers(1, 70000)) if bps % 4 == 0 else int(rng.integers(1, 3000))
        x = constructed(n, ch, bps, rng)
        blocks = mixed_blocks(n, rng)
        scale = float(np.float32(SCALES[bps % len(SCALES)]))
        draw = [0, 2, 1 << 20][bps % 3]
        got = fb.debug_replaygain_synthesis(x, blocks, bps, scale, hard, shaping, draw)
        want = refrgsynth.synth(x, blocks, bps, scale, hard, shaping, draw)
        assert np.array_equal(got, want), (bps, ch, n, scale, draw, np.argwhere(got != want)[:3])


def test_synthesis_long_chain_and_far_start():
    rng = np.random.default_rng(11)
    x = (np.sin(np.arange(10_000_000) / 50.0) * 30000).astype(np.int32).reshape(-1, 1)
    blocks = [4096] * (x.shape[0] // 4096) + [x.shape[0] % 4096]
    got = fb.debug_replaygain_synthesis(x, blocks, 16, 1.5, True, 3, 0)
    assert np.array_equal(got, refrgsynth.synth(x, blocks, 16, 1.5, True, 3, 0))
    y = constructed(5000, 2, 16, rng)
    got = fb.debug_replaygain_synthesis(y, [5000], 16, 0.8, False, 1, 1 << 31)
    assert np.array_equal(got, refrgsynth.synth(y, [5000], 16, 0.8, False, 1, 1 << 31))


# The two registers' periods (3 x 5 x 17 x 257 x 65537 and 7 x 47 x 73 x 178481, replaygain_synthesis.c:78): after both, the generator
# is back where it started, so a start there must give draw 2's output. The jump to it uses every one of the 64 matrix powers.
PERIOD = (3 * 5 * 17 * 257 * 65537) * (7 * 47 * 73 * 178481)


@pytest.mark.parametrize("shaping", [1, 3])
def test_synthesis_far_start_draws(shaping):
    rng = np.random.default_rng(40 + shaping)
    y = constructed(3000, 3, 16, rng)
    blocks = [1000, 33, 1967]
    want = refrgsynth.synth(y, blocks, 16, 1.25, True, shaping, 2)
    assert np.array_equal(fb.debug_replaygain_synthesis(y, blocks, 16, 1.25, True, shaping, 2 + PERIOD), want)
    # a start past 2^40 equals the same start one full period later
    far = (1 << 40) + 2
    a = fb.debug_replaygain_synthesis(y, blocks, 16, 1.25, True, shaping, far)
    assert np.array_equal(a, fb.debug_replaygain_synthesis(y, blocks, 16, 1.25, True, shaping, far + PERIOD))
    assert not np.array_equal(a, want)


def loud_batch():
    """Files of several widths and channel counts, some untagged, with gains that drive values past 0.5 (the tanh branch)."""
    files = []
    cases = [(2, 16, 9001, album_tags(8.5, 11.0)), (1, 8, 5000, album_tags(-3.0, 2.0)), (3, 24, 4001, album_tags(4.0, 6.0)),
             (2, 16, 3000, ["TITLE=untagged"]), (6, 20, 2500, album_tags(12.0, 9.0, 0.3, 0.2)), (8, 12, 2000, album_tags(-1.0, 3.0)),
             (2, 4, 1500, album_tags(6.0, 6.0))]
    for i, (ch, bps, n, tags) in enumerate(cases):
        files.append(tagged_flac(tags, ch=ch, bps=bps, n=n, seed=i))
    files.append(tagged_flac(album_tags(2.0, 5.0), ch=2, bps=16, n=40001, seed=20, args=["--lax", "--blocksize=16384"]))
    files.append(with_total_zero(tagged_flac(album_tags(7.0, 9.5), ch=2, bps=16, n=7001, seed=21)))
    x = signals.music_like(1000 * 3 + 4096 * 2 + 500 * 4 + 700, 2, 16, 44100, seed=22)
    var = variable_stream(x, 16, [(1000, 3000), (4096, 8192), (500, 2000), (256, 700)])
    files.append(add_vorbis_comment(var, [t.encode() for t in album_tags(9.0, 10.5, 0.9, 0.95)]))
    return files


@pytest.fixture(scope="module")
def batch():
    return loud_batch()


@pytest.mark.parametrize("spec", [None, "0aL", "12tLn1", "-6an2", "20aLn3", "6tl"])
def test_one_invocation_over_the_list(batch, spec):
    rc, want, err = tool_decode_many(batch, spec)
    assert rc == 0, err
    res = fb.decode_pcm_files_replaygain(batch, spec=spec)
    for f, (got, info, rg) in enumerate(res):
        assert info.tool_ok == 1
        assert got == want[f], (spec, f, rg.status, len(got), len(want[f]))
    assert any(r.status == fb.RGS_NO_TAGS for _, _, r in res) and any(r.status == fb.RGS_APPLIED for _, _, r in res)
    # per_file 1: one process per file
    for f, (got, info, rg) in enumerate(fb.decode_pcm_files_replaygain(batch, spec=spec, per_file=True)):
        assert got == tool_decode_many([batch[f]], spec)[1][0], (spec, f)


def test_tanh_branch_is_reached(batch):
    x = fb.Decoder(2, 16, 44100, 4096)
    x.index_files(batch[:1])
    (got, info, rg), = x.decode_pcm_files_replaygain(spec="20aLn3")
    plain, = x.decode_pcm_files()
    x.close()
    pcm = np.frombuffer(plain[0][info.header_bytes:info.header_bytes + info.samples * 4], dtype="<i2").astype(np.float64)
    assert np.any(np.abs(pcm * rg.scale / 32768) > 0.5)


@pytest.mark.parametrize("kind,sub", [(k, s) for k, s, _ in FORMATS])
def test_every_kind(batch, kind, sub):
    rc, want, err = tool_decode_many(batch, None, FLAGS[(kind, sub)])
    assert rc == 0, err
    for f, (got, info, rg) in enumerate(fb.decode_pcm_files_replaygain(batch, kind=kind, subformat=sub)):
        assert got == want[f], (kind, sub, f)


def test_damaged_file_keeps_later_files_draws():
    files = [tagged_flac(album_tags(3.0, 4.0), ch=2, bps=16, n=20000, seed=30 + i) for i in range(5)]
    b = bytearray(files[1])
    b[len(b) // 2] ^= 0x55  # a CRC-damaged frame in the middle of file 2
    files[1] = bytes(b)
    rc, want, err = tool_decode_many(files, None)
    res = fb.decode_pcm_files_replaygain(files)
    assert res[1][1].tool_ok == 0 and rc != 0
    assert res[0][0] == want[0]
    for f in (2, 3, 4):
        assert res[f][1].tool_ok == 1 and res[f][0] == want[f], f


def test_ranges_each_equal_their_own_tool_run(batch):
    ranges = [(0, 1000, 5000), (2, 17, 3001), (7, 16383, 20000), (0, 4095, 2)]
    dec = fb.Decoder(2, 16, 44100, 4096)
    dec.index_files(batch)
    res = dec.decode_pcm_files_replaygain(ranges=ranges)
    dec.close()
    for (f, s, n), (got, info, rg) in zip(ranges, res):
        rc, want, err = tool_decode_many([batch[f]], None, [f"--skip={s}", f"--until={s + n}"])
        assert rc == 0, err
        assert got == want[0], (f, s, n)
