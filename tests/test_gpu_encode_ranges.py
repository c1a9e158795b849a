"""flac --skip / --until in one call: sample ranges of WAV / RF64 / Wave64 / AIFF / AIFF-C files (fb200_encode_pcm_files_ranges_*,
Encoder.encode_pcm_files(ranges=...)) and of an indexed batch of .flac files (fb200_reencode_flac_files_ranges_*,
Encoder.reencode_flac_ranges) encoded to the .flac files the reference flac tool (oracle/_ref/flac_ref) writes for
--skip=first_sample --until=first_sample+samples, byte for byte with the vendor string the one allowed difference. Also: the
tool's range rules for FLAC input's SEEKTABLE, CUESHEET, PADDING and MD5, ReplayGain over ranges of several files, verify, both
entry points, per-range failures, caller errors before any launch, and launches that do not grow with the number of ranges."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import flac_b200 as fb
import flacsynth
import refcli
import reffile
from test_gpu_flac_files import vendor
from test_gpu_pcm_files import mixed_files
from test_gpu_reencode_files import cuesheet, make_flac, tool_args, with_blocks
from test_pcm_probe import aiff, fmt_chunk, pack, samples, wav

pytestmark = pytest.mark.gpu


def need_tool():
    if not refcli.available():
        pytest.skip("oracle/_ref/flac_ref not built")


def tool(blob, args, first, n, name="in.wav"):
    rc, out, err = refcli.encode(blob, list(args) + [f"--skip={first}", f"--until={first + n}"], name=name)
    assert rc == 0, err
    return reffile.with_vendor(out, vendor())


def positions(n, bs):
    """(first_sample, samples) inside a file of n samples: on and off frame boundaries, from 0, to the end, one sample, shorter
    than a block, across the short last block, the whole file"""
    tail = n % bs or bs
    cand = [(0, n), (0, 1), (n - 1, 1), (bs, bs), (bs - 1, bs + 2), (17, bs // 2), (n - tail - 3, tail + 3), (n // 3, n // 2),
            (0, bs), (1, n - 1)]
    return [(a, k) for a, k in cand if a >= 0 and k >= 1 and a + k <= n]


def ranges_of(lengths, bs, seed):
    """every position of every file, shuffled, with one range repeated and one overlapping another"""
    r = [(f, a, k) for f, n in enumerate(lengths) for a, k in positions(n, bs)]
    r += [r[3], (r[5][0], r[5][1] + 1, r[5][2])]
    np.random.default_rng(seed).shuffle(r)
    return r


def pcm_blobs(ch, bits, rate, seed, lengths):
    blobs = mixed_files(len(lengths), ch, bits, rate, seed, lengths=lengths)
    if ch <= 2:  # AIFF-C NONE as well
        x = samples(lengths[0], ch, bits, seed + 99)
        cont = (bits + 7) // 8 * 8
        blobs.append(aiff(pack(x, cont, cont - bits, big=True), ch, rate, bits, lengths[0], aifc=b"NONE"))
    return blobs


@pytest.mark.parametrize("level,ch,bits,rate", [(0, 2, 16, 44100), (5, 1, 16, 44100), (8, 2, 24, 96000), (5, 6, 16, 48000), (5, 2, 20, 48000),
                                                (5, 1, 8, 22050)])
def test_containers_as_the_tool(level, ch, bits, rate):
    need_tool()
    enc = fb.Encoder(fb.preset(ch, bits, rate, level))
    bs = enc.cfg.blocksize
    lengths = [3 * bs + 1234, 2 * bs, 777, bs + 1]
    blobs = pcm_blobs(ch, bits, rate, seed=level + ch * 10 + bits, lengths=lengths)
    lengths = [i.samples for i in fb.probe_pcm_files(blobs)]
    ranges = ranges_of(lengths, bs, seed=level)
    try:
        got = enc.encode_pcm_files(blobs, ranges=ranges)
    finally:
        enc.close()
    assert len(got) == len(ranges)
    for (f, a, k), o in zip(ranges, got):
        assert o == tool(blobs[f], [f"-{level}"], a, k), (f, a, k)


@pytest.mark.parametrize("opts,args", [
    (dict(seek_spacing_s=0), ["-S-"]), (dict(seek_spacing_s=2), ["-S", "2s"]), (dict(padding=0), ["-P", "0"]),
    (dict(padding=4096), ["-P", "4096"]), (dict(md5=False), ["--no-md5-sum"]),
])
def test_container_options_as_the_tool(opts, args):
    need_tool()
    blobs = mixed_files(3, 2, 16, 44100, seed=4, lengths=[44100 * 5 + 11, 50000, 9000])
    ranges = [(0, 1000, 44100 * 4), (1, 0, 50000), (2, 4095, 3), (0, 44100 * 5, 11)]
    enc = fb.Encoder(fb.preset(2, 16, 44100, 5))
    try:
        got = enc.encode_pcm_files(blobs, ranges=ranges, **opts)
    finally:
        enc.close()
    for (f, a, k), o in zip(ranges, got):
        assert o == tool(blobs[f], ["-5"] + args, a, k), (f, a, k)


def test_tags_and_channel_mask_per_range():
    need_tool()
    x = samples(20000, 4, 16, 8)
    quad = wav(pack(x, 16, 0), fmt_chunk(4, 44100, 16, 16, 0x33, True))
    ranges = [(0, 0, 5000), (0, 5000, 15000), (0, 100, 100)]
    tags = [["TITLE=one"], ["TITLE=two", "ARTIST=a"], []]
    enc = fb.Encoder(fb.preset(4, 16, 44100, 5))
    try:
        got = enc.encode_pcm_files([quad], ranges=ranges, tags=tags)
    finally:
        enc.close()
    for (f, a, k), t, o in zip(ranges, tags, got):
        assert o == tool(quad, ["-5"] + [v for tag in t for v in ("-T", tag)], a, k)


def run_tool_album(blobs, args, ext):
    """one flac invocation over every blob -> [output with our vendor string]"""
    with tempfile.TemporaryDirectory() as d:
        names = [f"f{k:03d}.{ext}" for k in range(len(blobs))]
        for nm, b in zip(names, blobs):
            with open(os.path.join(d, nm), "wb") as f:
                f.write(b)
        os.mkdir(os.path.join(d, "out"))
        r = subprocess.run([refcli.PATH, "-f", "-s", *args, "--output-prefix=out/", *names], cwd=d, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        return [reffile.with_vendor(open(os.path.join(d, "out", nm.rsplit(".", 1)[0] + ".flac"), "rb").read(), vendor()) for nm in names]


def test_replay_gain_over_ranges_of_several_files():
    """--replay-gain with one --skip / --until over three files is one album: one tool invocation against one call"""
    need_tool()
    a, b = 3000, 3000 + 44100 * 2
    blobs = mixed_files(3, 2, 16, 44100, seed=21, lengths=[44100 * 3, 44100 * 3 + 500, 44100 * 2 + 3000])
    want = run_tool_album(blobs, ["-8", "--replay-gain", f"--skip={a}", f"--until={b}"], "wav")
    enc = fb.Encoder(fb.preset(2, 16, 44100, 8))
    try:
        got = enc.encode_pcm_files(blobs, ranges=[(f, a, b - a) for f in range(3)], replay_gain=True)
    finally:
        enc.close()
    assert got == want
    flacs = [make_flac(44100 * 3 + 77 * k, 2, 16, 44100, seed=30 + k) for k in range(3)]
    want = run_tool_album(flacs, ["-8", "--replay-gain", f"--skip={a}", f"--until={b}"], "flac")
    out, info = reencode(flacs, 8, [(f, a, b - a) for f in range(3)], replay_gain=True)
    assert [i.status for i in info] == [fb.REENCODE_OK] * 3
    assert out == want


def reencode(blobs, level, ranges, **kw):
    dec = fb.Decoder(2, 16, 44100, 4096)
    try:
        infos, _ = dec.index_files([bytes(b) for b in blobs])
        i = infos[ranges[0][0]]
        enc = fb.Encoder(fb.preset(i.channels, i.bits_per_sample, i.sample_rate, level))
        try:
            return enc.reencode_flac_ranges(dec, ranges, infos=True, **kw)
        finally:
            enc.close()
    finally:
        dec.close()


def check_flac_same(blobs, level, ranges, **kw):
    out, info = reencode(blobs, level, ranges, **kw)
    for (f, a, k), o, i in zip(ranges, out, info):
        assert i.status == fb.REENCODE_OK, i.error
        assert o == tool(blobs[f], tool_args(level, **kw), a, k, name="in.flac"), (f, a, k)


@pytest.mark.parametrize("level,ch,bits,rate", [(0, 2, 16, 44100), (5, 1, 16, 44100), (8, 2, 24, 96000), (5, 6, 16, 48000), (5, 2, 20, 48000)])
def test_flac_input_as_the_tool(level, ch, bits, rate):
    """inputs of other blocksizes than the encoder's, and variable-blocksize streams"""
    need_tool()
    blobs = [make_flac(5000 + 3011 * k, ch, bits, rate, seed=ch * 100 + bits + k, args=a)
             for k, a in enumerate([("-0",), ("-8", "-b", "1152"), ("-5", "-b", "576", "-P", "0")])]
    if (ch, bits, rate) == (2, 16, 44100):
        rng = np.random.default_rng(7)
        blobs.append(flacsynth.flac_file(flacsynth.make_stream(rng, flacsynth.Format(2, 16, 44100), 30, variable=True)))
    dec = fb.Decoder(2, 16, 44100, 4096)
    try:
        lengths = [int(i.total_samples) for i in dec.index_files(blobs)[0]]
    finally:
        dec.close()
    bs = 4096 if level else 1152
    ranges = ranges_of(lengths, bs, seed=level + 1)
    if bits > 16:
        # the tool's AVX2 fixed-order guess skips the last (n - 4) % 4 samples of a 20- or 24-bit block (DESIGN.md, G4), so a short
        # last block of another length can differ from the C routine this engine follows
        ranges = [r for r in ranges if r[2] % bs % 4 == 0]
    check_flac_same(blobs, level, ranges)


@pytest.mark.parametrize("opts", [{}, {"seek_spacing_s": 0}, {"seek_spacing_s": 2}, {"padding": 0}, {"padding": 4096},
                                  {"tags": ["ARTIST=someone"]}], ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()) or "default")
def test_flac_input_metadata_rules(opts):
    """SEEKTABLE kept for the whole-file range only, CUESHEET kept when its lead-out is the range's length, PADDING merged, and a
    wrong STREAMINFO MD5 not checked"""
    need_tool()
    n = 44100 * 3 + 77
    base = make_flac(n, 2, 16, 44100, seed=11, args=("-5", "-S-", "--no-padding"))
    seek = fb.seektable_block([(0, 0, 0), (44100, 0, 0), (100000, 0, 0), (fb.SEEKPOINT_PLACEHOLDER, 0, 0)])
    vc = fb.vorbis_comment_block(["ALBUM=a"], vendor=b"other")
    with_seek = with_blocks(base, [seek, vc, fb.padding_block(300), fb.padding_block(40)])
    cue_len = with_blocks(base, [cuesheet(50000), vc])
    bad_md5 = bytearray(make_flac(n, 2, 16, 44100, seed=12, args=("-5", "-b", "1152", "-S", "1s")))
    bad_md5[8 + 18] ^= 1
    blobs = [with_seek, cue_len, bytes(bad_md5)]
    ranges = [(0, 0, n), (0, 1, n - 1), (0, 0, n - 1), (1, 1000, 50000), (1, 0, n), (1, 7, 49999), (2, 0, n), (2, 4000, 60000)]
    check_flac_same(blobs, 5, ranges, **opts)


def test_flac_damage_and_totals():
    """a damaged frame inside a range is DAMAGED and the call goes on; a range away from it is OK and equals the same range of
    an undamaged copy; a file whose STREAMINFO total is 0 gives NO_TOTAL for each of its ranges"""
    need_tool()
    base = make_flac(40000, 2, 16, 44100, seed=80)
    _, audio = reffile.blocks(base)
    flipped = bytearray(base)
    flipped[audio + 5000] ^= 0x10  # inside the first or second 4096-sample frame
    no_total = bytearray(base)
    no_total[8 + 13] &= 0xF0
    no_total[8 + 14:8 + 18] = bytes(4)
    ranges = [(0, 0, 12000), (0, 20000, 15000), (1, 20000, 15000), (2, 100, 1000), (0, 30000, 10000)]
    out, info = reencode([bytes(flipped), base, bytes(no_total)], 5, ranges)
    assert [i.status for i in info] == [fb.REENCODE_DAMAGED, fb.REENCODE_OK, fb.REENCODE_OK, fb.REENCODE_NO_TOTAL, fb.REENCODE_OK]
    assert out[0] == b"" and out[3] == b"" and info[0].file.bytes == 0
    assert out[1] == out[2] == tool(base, tool_args(5), 20000, 15000, name="in.flac")
    assert out[4] == tool(base, tool_args(5), 30000, 10000, name="in.flac")


def test_verify_and_both_entry_points():
    need_tool()
    import torch
    blobs = mixed_files(3, 2, 16, 44100, seed=5, lengths=[30000, 9000, 4097])
    ranges = [(0, 100, 20000), (2, 0, 4097), (1, 4096, 10), (0, 0, 30000)]
    data, offsets = fb._batch(blobs)
    pinfo = fb.probe_pcm_files(None, data, offsets)
    enc = fb.Encoder(fb.preset(2, 16, 44100, 5))
    enc.set_verify(True)
    try:
        host = enc.encode_pcm_files(blobs, ranges=ranges)
        assert all(v.status == fb.VERIFY_OK for v in enc.verify_info(len(ranges)))
        cap = enc.pcm_files_capacity(pinfo, ranges=ranges)
        d_data = torch.from_numpy(data.copy()).cuda()
        d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        _, files = enc.encode_pcm_files_device(d_data.data_ptr(), offsets, pinfo, d_out.data_ptr(), cap, ranges=ranges)
        torch.cuda.synchronize()
        outb = d_out.cpu().numpy().tobytes()
        assert [outb[i.offset:i.offset + i.bytes] for i in files] == host
        assert all(v.status == fb.VERIFY_OK for v in enc.verify_info(len(ranges)))
    finally:
        enc.close()
    flacs = [make_flac(30000, 2, 16, 44100, seed=40), make_flac(9000, 2, 16, 44100, seed=41, args=("-5", "-b", "1152"))]
    franges = [(0, 100, 20000), (1, 0, 9000), (1, 1151, 2), (0, 0, 30000)]
    dec = fb.Decoder(2, 16, 44100, 4096)
    enc = fb.Encoder(fb.preset(2, 16, 44100, 5))
    enc.set_verify(True)
    try:
        dec.index_files(flacs)
        host, hinfo = enc.reencode_flac_ranges(dec, franges, infos=True)
        assert all(v.status == fb.VERIFY_OK for v in enc.verify_info(len(franges)))
        cap = enc.reencode_ranges_capacity(dec, franges)
        d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        _, dinfo = enc.reencode_flac_ranges_device(dec, franges, d_out.data_ptr(), cap)
        torch.cuda.synchronize()
        outb = d_out.cpu().numpy().tobytes()
        assert [outb[i.file.offset:i.file.offset + i.file.bytes] for i in dinfo] == host
        for (f, a, k), h in zip(franges, host):
            assert h == tool(flacs[f], tool_args(5), a, k, name="in.flac")
    finally:
        enc.close()
        dec.close()


def test_caller_errors_before_any_launch():
    need_tool()
    blobs = mixed_files(2, 2, 16, 44100, seed=6, lengths=[10000, 5000])
    flacs = [make_flac(10000, 2, 16, 44100, seed=7)]
    enc = fb.Encoder(fb.preset(2, 16, 44100, 5))
    dec = fb.Decoder(2, 16, 44100, 4096)
    try:
        dec.index_files(flacs)
        n0 = enc.launches + dec.launches
        for ranges, msg in [([(0, 9000, 1001)], "--until value is after end of input"), ([(0, 10001, 1)], "value of --skip exceeds input size"),
                            ([(1, 0, 0)], "range 0 is empty"), ([(2, 0, 10)], "file 2 of a batch of 2")]:
            with pytest.raises(fb.FlacB200Error, match="-3.*" + msg):
                enc.encode_pcm_files(blobs, ranges=ranges)
        for ranges, msg in [([(0, 9000, 1001)], r"samples \[9000, 10001\) of file 0"), ([(0, 5, 0)], "range 0 is empty"),
                            ([(1, 0, 10)], "file 1 of a batch of 1")]:
            with pytest.raises(fb.FlacB200Error, match="-3.*" + msg):
                enc.reencode_flac_ranges(dec, ranges)
        assert enc.launches + dec.launches == n0
        # a data chunk cut short: what is present is encoded; a range starting past it is refused
        short = blobs[0][:-4 * 2000]
        assert fb.probe_pcm_files([short])[0].samples == 8000
        with pytest.raises(fb.FlacB200Error, match="past the 8000 samples present"):
            enc.encode_pcm_files([short], ranges=[(0, 8000, 100)])
        got = enc.encode_pcm_files([short], ranges=[(0, 7000, 2000)])
        rc, want, _ = refcli.encode(short, ["-5", "--skip=7000", "--until=9000"])
        assert got[0] == reffile.with_vendor(want, vendor())
        # capacity 0 fails with OUTPUT_TOO_SMALL
        data, offsets = fb._batch(blobs)
        pinfo = fb.probe_pcm_files(None, data, offsets)
        out = np.empty(16, np.uint8)
        with pytest.raises(fb.FlacB200Error) as e:
            enc._pcm_call(True, data.ctypes.data, offsets, pinfo, None, 10, -1, True, out.ctypes.data, 0, None, ranges=[(0, 0, 100)])
        assert e.value.code == -4
    finally:
        enc.close()
        dec.close()


def test_launches_do_not_grow_with_ranges():
    need_tool()
    blobs = mixed_files(2, 2, 16, 44100, seed=9, lengths=[44100 * 4, 44100 * 3])
    flacs = [make_flac(44100 * 4, 2, 16, 44100, seed=10), make_flac(44100 * 3, 2, 16, 44100, seed=11)]
    counts = []
    for n in (4, 64):
        rng = np.random.default_rng(n)
        ranges = []
        for i in range(n):  # the encoder groups short last blocks by length: the same three lengths in both calls
            ranges.append((i % 2, int(rng.integers(0, 44100 * 2)), (30000, 5000, 44100)[i % 3]))
        enc = fb.Encoder(fb.preset(2, 16, 44100, 5))
        dec = fb.Decoder(2, 16, 44100, 4096)
        try:
            dec.index_files(flacs)
            n0 = enc.launches + dec.launches
            enc.encode_pcm_files(blobs, ranges=ranges)
            n1 = enc.launches + dec.launches
            out, info = enc.reencode_flac_ranges(dec, ranges, infos=True)
            assert all(i.status == fb.REENCODE_OK for i in info)
            counts.append((n1 - n0, enc.launches + dec.launches - n1))
        finally:
            enc.close()
            dec.close()
    assert counts[0] == counts[1]
