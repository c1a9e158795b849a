"""flac -f *.flac in one call (fb200_reencode_flac_files_host / _device, flac_b200.reencode_flac_files): every output file byte
for byte what the reference flac tool (oracle/_ref/flac_ref) writes when it re-encodes the same .flac file with the same options,
the vendor string being the one allowed difference; the tool's metadata policy for FLAC input rule by rule; ReplayGain over an
album; per-file failures; mixed batches through both entry points with verify; and launches that do not grow with the number of
files."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import flac_b200 as fb
import flacsynth
import oraclelib
import refcli
import reffile
import reflib
import signals
from test_gpu_flac_files import vendor
from test_pcm_probe import fmt_chunk, pack, samples, wav

pytestmark = pytest.mark.gpu


def need_tool():
    if not refcli.available():
        pytest.skip("oracle/_ref/flac_ref not built")


def wav_of(x, bits, rate, mask=None):
    ch = x.shape[1]
    cont = (bits + 7) // 8 * 8
    if ch > 2 or bits % 8:
        fmt = fmt_chunk(ch, rate, cont, bits, mask if mask is not None else (1 << ch) - 1, True)
    else:
        fmt = fmt_chunk(ch, rate, cont)
    return wav(pack(x, cont, cont - bits, unsigned=cont == 8), fmt)


def make_flac(n, ch, bits, rate, seed, args=("-5",)):
    """A .flac the tool writes from a WAV of n seeded samples."""
    rc, out, err = refcli.encode(wav_of(samples(n, ch, bits, seed), bits, rate), args)
    assert rc == 0, err
    return out


def tool_args(level, seek_spacing_s=-1, padding=-1, tags=None, replay_gain=False):
    a = [f"-{level}"]
    if seek_spacing_s == 0:
        a.append("-S-")
    elif seek_spacing_s > 0:
        a += ["-S", f"{seek_spacing_s}s"]
    if padding == 0:
        a.append("--no-padding")
    elif padding > 0:
        a += ["-P", str(padding)]
    for t in tags or ():
        a += ["-T", t]
    if replay_gain:
        a.append("--replay-gain")
    return a


def tool(blob, args):
    """(exit code, the tool's output with our vendor string or None) of flac -f args in.flac"""
    rc, out, err = refcli.encode(blob, args, name="in.flac")
    return rc, (reffile.with_vendor(out, vendor()) if out is not None else None)


def ours(blobs, level, files=None, **kw):
    """Index blobs once and re-encode `files` (default all) with one encoder of the first listed file's format."""
    dec = fb.Decoder(2, 16, 44100, 4096)
    try:
        infos, _ = dec.index_files([bytes(b) for b in blobs])
        files = list(range(len(blobs))) if files is None else files
        i = infos[files[0]]
        enc = fb.Encoder(fb.preset(i.channels, i.bits_per_sample, i.sample_rate, level))
        try:
            return enc.reencode_flac_files(dec, files, infos=True, **kw)
        finally:
            enc.close()
    finally:
        dec.close()


def check_same(blobs, level, **kw):
    out, info = ours(blobs, level, **kw)
    for b, o, i in zip(blobs, out, info):
        rc, want = tool(b, tool_args(level, **kw))
        assert rc == 0 and i.status == fb.REENCODE_OK, (rc, i.status, i.error)
        assert o == want


def identity_inputs(ch, bits, rate):
    """three files the tool wrote at other levels and blocksizes"""
    return [make_flac(5000 + 3011 * k, ch, bits, rate, seed=ch * 100 + bits + k, args=a)
            for k, a in enumerate([("-0",), ("-8", "-b", "1152"), ("-5", "-b", "576", "-P", "0")])]


@pytest.mark.parametrize("level", [0, 5, 8])
@pytest.mark.parametrize("ch,bits,rate", [(1, 16, 44100), (2, 16, 44100), (2, 24, 96000), (6, 16, 48000), (2, 20, 48000)])
def test_byte_identity(level, ch, bits, rate):
    need_tool()
    check_same(identity_inputs(ch, bits, rate), level)


def host_dispatches_avx2_fixed_guess():
    """Whether the reference on this host takes its AVX2 fixed-order guess, which drops the last (n - 4) % 4 samples of a block
    (DESIGN.md, G4): a 24-bit stream whose short last block the two routines guess differently."""
    x = signals.music_like(1152 * 3 + 19, 2, 24, 44100, seed=1)
    _, _, host = reflib.encode(x, 24, rate=44100, level=2, variant="strict", opts=reflib.RefEncOpts(streamable_subset=0))
    _, _, c_path = reflib.encode(x, 24, rate=44100, level=2, variant="strict", opts=reflib.RefEncOpts(streamable_subset=0, disable_isa=16))
    return host != c_path


@pytest.mark.parametrize("level", [0, 5, 8])
def test_byte_identity_six_channel_24_bit(level):
    """6ch/24/48, where the tool's short last frame can differ from ours on an AVX2 host (G4): our frames are the oracle's (C
    fixed-order guess) for the decoded samples, the tool's are the oracle's in the mode the host dispatches, and the files are
    byte-identical wherever those two agree. Otherwise only the last frame and STREAMINFO's min / max frame size differ, and
    ours are the min / max of our own frames."""
    need_tool()
    if not reflib.available("strict"):
        pytest.skip("oracle/_ref not built")
    avx2 = host_dispatches_avx2_fixed_guess()
    blobs = identity_inputs(6, 24, 48000)
    out, info = ours(blobs, level)
    dec = fb.Decoder(2, 16, 44100, 4096)
    try:
        decoded = dec.decode_files(blobs)
    finally:
        dec.close()
    for k, (b, o, i, (x, _)) in enumerate(zip(blobs, out, info, decoded)):
        assert i.status == fb.REENCODE_OK, i.error
        rc, want = tool(b, tool_args(level))
        assert rc == 0
        c_frames = oraclelib.Encoder(oraclelib.preset(6, 24, 48000, level)).encode_stream(x)
        host_frames = oraclelib.Encoder(oraclelib.preset(6, 24, 48000, level, x86_avx2_fixed_guess=int(avx2))).encode_stream(x)
        ao, (_, want_ao) = int(i.file.audio_offset), reffile.blocks(want)
        assert o[ao:] == b"".join(c_frames), f"file {k}: our frames are not the oracle's"
        assert want[want_ao:] == b"".join(host_frames), f"file {k}: the tool's frames are not the oracle's (avx2 {avx2})"
        if c_frames == host_frames:
            assert o == want, f"file {k}"
            continue
        assert c_frames[:-1] == host_frames[:-1], f"file {k}: a full block differs"
        sizes = [len(f) for f in c_frames]
        si = 8 + 4  # STREAMINFO's min_framesize (24 bits) and max_framesize (24 bits)
        assert o[si:si + 6] == min(sizes).to_bytes(3, "big") + max(sizes).to_bytes(3, "big"), f"file {k}: min / max frame size"
        assert ao == want_ao and o[:si] + o[si + 6:ao] == want[:si] + want[si + 6:ao], f"file {k}: metadata"


@pytest.mark.parametrize("level", [0, 5, 8])
def test_six_channel_24_bit_frames_are_the_encoders(level):
    """6ch/24/48: every re-encoded file's frames and STREAMINFO are what fb200_encode_flac_files_* writes for the decoded samples"""
    need_tool()
    blobs = identity_inputs(6, 24, 48000)
    out, info = ours(blobs, level)
    dec = fb.Decoder(2, 16, 44100, 4096)
    enc = fb.Encoder(fb.preset(6, 24, 48000, level))
    try:
        dec_out = dec.decode_files(blobs)
        pcm = np.concatenate([x for x, _ in dec_out])
        want, winfo = enc.encode_flac_files(pcm, [x.shape[0] for x, _ in dec_out], infos=True)
    finally:
        enc.close()
        dec.close()
    for o, i, w, wi in zip(out, info, want, winfo):
        assert i.status == fb.REENCODE_OK, i.error
        assert o[int(i.file.audio_offset):] == w[int(wi.audio_offset):]
        assert bytes(i.file.streaminfo) == bytes(wi.streaminfo)


def test_inputs_of_every_shape():
    """variable-blocksize streams and junk after the last frame; an ID3v2-prefixed file, which the tool refuses (main.c:1524)"""
    need_tool()
    rng = np.random.default_rng(7)
    blobs = []
    for k in range(3):
        st = flacsynth.make_stream(rng, flacsynth.Format(2, 16, 44100), 30, variable=True)
        blobs.append(flacsynth.flac_file(st))
    base = make_flac(20000, 2, 16, 44100, seed=3)
    blobs.append(base + b"TAG" + bytes(125))
    check_same(blobs, 5)
    id3 = b"ID3\x04\x00\x00\x00\x00\x00\x20" + bytes(32) + base
    assert tool(id3, tool_args(5))[0] != 0
    out, info = ours([base, id3], 5)
    assert [i.status for i in info] == [fb.REENCODE_OK, fb.REENCODE_INPUT] and out[1] == b""
    assert out[0] == tool(base, tool_args(5))[1]


OPTIONS = [{}, {"seek_spacing_s": 0}, {"seek_spacing_s": 5}, {"padding": 0}, {"padding": 1000}, {"tags": ["ARTIST=someone", "TITLE=x"]}]


def with_blocks(flac, blocks):
    """flac's STREAMINFO, then `blocks` (stream syntax, last flags fixed), then its audio"""
    bl, audio = reffile.blocks(flac)
    assert bl[0][0] == 0
    allb = [fb.metadata_block(0, bl[0][2])] + list(blocks)
    out = b"fLaC" + b"".join((bytes([b[0] | (0x80 if k == len(allb) - 1 else 0)]) + b[1:]) for k, b in enumerate(allb))
    return out + flac[audio:]


def cuesheet(lead_out):
    body = bytearray(128) + (0).to_bytes(8, "big") + bytes(259) + bytes([2])
    for num, off in ((1, 0), (170, lead_out)):
        body += off.to_bytes(8, "big") + bytes([num]) + bytes(12) + bytes(14) + bytes([1 if num != 170 else 0])
        if num != 170:
            body += (0).to_bytes(8, "big") + bytes([1]) + bytes(3)
    return fb.metadata_block(fb.METADATA_CUESHEET, body)


def picture():
    mime, desc, data = b"image/jpeg", b"front", b"\xff\xd8" + bytes(50)
    body = (3).to_bytes(4, "big") + len(mime).to_bytes(4, "big") + mime + len(desc).to_bytes(4, "big") + desc + (16).to_bytes(4, "big") * 2
    body += (24).to_bytes(4, "big") + (0).to_bytes(4, "big") + len(data).to_bytes(4, "big") + data
    return fb.metadata_block(fb.METADATA_PICTURE, body)


def policy_inputs():
    n = 44100 * 3 + 77
    base = make_flac(n, 2, 16, 44100, seed=11, args=("-5", "-S-", "--no-padding"))
    vc = fb.vorbis_comment_block(["ALBUM=a", "WAVEFORMATEXTENSIBLE_CHANNEL_MASK=0x0003"], vendor=b"other")
    seek = fb.seektable_block([(0, 0, 0), (44100, 0, 0), (100000, 0, 0), (fb.SEEKPOINT_PLACEHOLDER, 0, 0)])
    return {
        "no_vc": with_blocks(base, [fb.padding_block(10)]),
        "vc_mask": with_blocks(base, [vc, fb.padding_block(100)]),
        "two_paddings": with_blocks(base, [vc, fb.padding_block(300), fb.metadata_block(fb.METADATA_APPLICATION, b"abcd" + bytes(9)),
                                           fb.padding_block(40), cuesheet(n)]),
        "picture_app": with_blocks(base, [picture(), fb.metadata_block(fb.METADATA_APPLICATION, b"test" + b"xyz"), vc]),
        "unknown": with_blocks(base, [fb.metadata_block(9, b"\x01\x02\x03"), vc]),
        "cue_right": with_blocks(base, [cuesheet(n), vc]),
        "cue_wrong": with_blocks(base, [cuesheet(n - 1), vc]),
        "kept_seektable": with_blocks(base, [seek, vc]),
        # the tool's own table over 1152-sample frames (a point every second), kept and moved to the new 4096-sample frames
        "kept_seektable_1152": make_flac(n, 2, 16, 44100, seed=12, args=("-5", "-b", "1152", "-S", "1s")),
    }


@pytest.mark.parametrize("opts", OPTIONS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()) or "default")
def test_metadata_policy(opts):
    need_tool()
    cases = policy_inputs()
    for level in (5,):
        out, info = ours(list(cases.values()), level, **opts)
        for (name, blob), o, i in zip(cases.items(), out, info):
            rc, want = tool(blob, tool_args(level, **opts))
            assert rc == 0, name
            assert i.status == fb.REENCODE_OK, (name, i.error)
            assert o == want, name


def run_tool_album(blobs, args):
    """one flac -f invocation over every blob (files in one directory) -> [output with our vendor string]"""
    with tempfile.TemporaryDirectory() as d:
        names = [f"f{k:03d}.flac" for k in range(len(blobs))]
        for nm, b in zip(names, blobs):
            with open(os.path.join(d, nm), "wb") as f:
                f.write(b)
        os.mkdir(os.path.join(d, "out"))
        r = subprocess.run([refcli.PATH, "-f", "-s", *args, "--output-prefix=out/", *names], cwd=d, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        res = []
        for nm in names:
            with open(os.path.join(d, "out", nm), "rb") as f:
                res.append(reffile.with_vendor(f.read(), vendor()))
        return res


@pytest.mark.parametrize("rate", [44100, 96000])
def test_replay_gain_album(rate):
    need_tool()
    blobs = [make_flac(rate + 4567 * k, 2, 16, rate, seed=50 + k) for k in range(3)]
    want = run_tool_album(blobs, tool_args(8, replay_gain=True))
    out, info = ours(blobs, 8, replay_gain=True)
    for o, i, w in zip(out, info, want):
        assert i.status == fb.REENCODE_OK, i.error
        assert o == w


def vorbis_comment_block(entries, count=None, tail=b""):
    """a VORBIS_COMMENT whose entry count (default: the entries') and trailing bytes may disagree with its entries"""
    le = lambda v: v.to_bytes(4, "little")
    body = le(5) + b"other" + le(len(entries) if count is None else count)
    for e in entries:
        body += le(len(e)) + e
    return fb.metadata_block(fb.METADATA_VORBIS_COMMENT, body + tail)


def damaged_inputs():
    good = [make_flac(30000 + 1000 * k, 2, 16, 44100, seed=70 + k) for k in range(2)]
    base = make_flac(30000, 2, 16, 44100, seed=80)
    bl, audio = reffile.blocks(base)
    si = bytearray(bl[0][2])
    no_total = bytearray(base)
    no_total[8 + 13] &= 0xF0
    no_total[8 + 14:8 + 18] = bytes(4)
    flipped = bytearray(base)
    flipped[audio + 5000] ^= 0x10
    truncated = base[:audio + (len(base) - audio) // 2]
    bad_md5 = bytearray(base)
    bad_md5[8 + 18] ^= 1
    seek = fb.seektable_block([(44100, 0, 0), (0, 0, 0)])
    bad_seek = with_blocks(base, [seek])
    # the tool's decoder fails a VORBIS_COMMENT with bytes after its last entry; the encoder takes one VORBIS_COMMENT at most
    vc_bytes_left = with_blocks(base, [vorbis_comment_block([b"A=1"], tail=b"\0\0"), fb.padding_block(10)])
    two_vcs = with_blocks(base, [vorbis_comment_block([b"A=1"]), fb.padding_block(10), vorbis_comment_block([b"B=2"])])
    assert bytes(si) == bytes(base[8:42])
    return good, [(bytes(no_total), fb.REENCODE_NO_TOTAL), (bytes(flipped), fb.REENCODE_DAMAGED), (bytes(truncated), fb.REENCODE_DAMAGED),
                  (bytes(bad_md5), fb.REENCODE_MD5_MISMATCH), (bad_seek, fb.REENCODE_METADATA), (vc_bytes_left, fb.REENCODE_METADATA),
                  (two_vcs, fb.REENCODE_METADATA)]


def test_failures():
    need_tool()
    good, bad = damaged_inputs()
    for blob, status in bad:
        rc, _ = tool(blob, tool_args(5))
        assert rc != 0, status
        blobs = [good[0], blob, good[1]]
        out, info = ours(blobs, 5)
        assert [i.status for i in info] == [fb.REENCODE_OK, status, fb.REENCODE_OK], [i.error for i in info]
        assert out[1] == b"" and info[1].file.bytes == 0
        for k in (0, 2):
            assert out[k] == tool(blobs[k], tool_args(5))[1]


@pytest.mark.parametrize("tags", [
    pytest.param(None, id="input_tags", marks=pytest.mark.xfail(strict=True, reason=(
        "the tool's decoder keeps the entries that fit (read_metadata_vorbiscomment_) and re-encodes the file; the input list "
        "reads the block with the encoder's rule that its fields fill it exactly, and fails the file"))),
    pytest.param(["TITLE=x"], id="new_tags"),
])
def test_vorbis_comment_count_past_block(tags):
    """A VORBIS_COMMENT whose count claims more entries than the block holds: the tool re-encodes the file; with -T, the
    input's VORBIS_COMMENT goes unread."""
    need_tool()
    base = make_flac(30000, 2, 16, 44100, seed=81)
    blob = with_blocks(base, [vorbis_comment_block([b"A=1", b"B=2"], count=3), fb.padding_block(10)])
    rc, want = tool(blob, tool_args(5, tags=tags))
    assert rc == 0
    out, info = ours([blob], 5, tags=tags)
    assert info[0].status == fb.REENCODE_OK, info[0].error
    assert out[0] == want


def reencode_raw(enc, dec, files, replay_gain=False, reserved=0, tags=None, tag_offsets=None):
    """fb200_reencode_flac_files_host with a real 1 MB output: an error can only come from the call's own checks"""
    files = np.ascontiguousarray(files, dtype=np.uint32)
    out = np.empty(1 << 20, dtype=np.uint8)
    info = (fb.FlacReencodeInfo * max(files.size, 1))()
    opt = fb.FlacReencodeOptions(-1, -1, 1 if replay_gain else 0, reserved)
    nf = C.c_uint64(0)
    fb._check(fb.lib().fb200_reencode_flac_files_host(enc._h, dec._h, files.ctypes.data, files.size, C.byref(opt),
                                                      None if tags is None else tags.ctypes.data,
                                                      None if tag_offsets is None else tag_offsets.ctypes.data, out.ctypes.data, out.size,
                                                      None, C.byref(nf), info))


def test_caller_errors():
    """Each caller error fails the whole call with FB200_ERR_INVALID and its own message, before anything is launched."""
    need_tool()
    rng = np.random.default_rng(3)
    var96 = flacsynth.flac_file(flacsynth.make_stream(rng, flacsynth.Format(2, 16, 96000), 20, variable=True))
    blobs = [make_flac(5000, 2, 16, 44100, seed=1),                               # 0: the 2 / 16 / 44.1 encoder's format
             make_flac(5000, 1, 16, 44100, seed=2),                               # 1: another format
             make_flac(5000, 6, 16, 48000, seed=3),                               # 2: 6 channels
             make_flac(5000, 2, 16, 7000, seed=4),                                # 3: a rate ReplayGain does not take
             make_flac(20000, 2, 16, 96000, seed=5, args=("-5", "-b", "1153")),   # 4: 96 kHz, fixed blocksize not a multiple of 2
             var96]                                                               # 5: 96 kHz, variable blocksizes
    dec = fb.Decoder(2, 16, 44100, 4096)
    encs = {f: fb.Encoder(fb.preset(*f, 5)) for f in ((2, 16, 44100), (6, 16, 48000), (2, 16, 7000), (2, 16, 96000))}
    e = encs[(2, 16, 44100)]
    try:
        with pytest.raises(fb.FlacB200Error, match="-3.*no batch of files is indexed"):
            reencode_raw(e, dec, [0])
        dec.index_files(blobs)
        n0 = sum(x.launches for x in encs.values()) + dec.launches
        cases = [
            (e, [1], {}, r"file 1 is 1 ch / 16 bits / 44100 Hz, the encoder 2 / 16 / 44100"),
            (e, [0, 0], {}, r"file 0 is listed twice"),
            (e, [0, 6], {}, r"files\[1\] = 6, the batch has 6 files"),
            (e, [0], {"reserved": 1}, r"reserved must be 0"),
            (e, [0], {"tags": np.frombuffer(b"A=b\0", np.uint8), "tag_offsets": np.array([0, 3], np.uint64)}, r"tags of file 0 do not end in a NUL"),
            (encs[(6, 16, 48000)], [2], {"replay_gain": True}, r"6 channels; --replay-gain takes 1 or 2"),
            (encs[(2, 16, 7000)], [3], {"replay_gain": True}, r"invalid sample rate 7000 for --replay-gain"),
            (encs[(2, 16, 96000)], [4], {"replay_gain": True}, r"file 4: blocksizes 1153-1153 at 96000 Hz"),
            (encs[(2, 16, 96000)], [5], {"replay_gain": True}, r"file 5: blocksizes \d+-\d+ at 96000 Hz"),
        ]
        for enc, files, kw, msg in cases:
            with pytest.raises(fb.FlacB200Error, match=r"-3.*" + msg):
                reencode_raw(enc, dec, files, **kw)
        assert sum(x.launches for x in encs.values()) + dec.launches == n0
    finally:
        for x in encs.values():
            x.close()
        dec.close()


def test_mixed_batch_host_device_verify():
    need_tool()
    import torch
    fmts = [(2, 16, 44100), (1, 24, 48000), (6, 16, 48000)]
    blobs = [make_flac(9000 + 2500 * k, *fmts[k % 3], seed=90 + k) for k in range(9)]
    res = fb.reencode_flac_files(blobs, level=5)
    for b, (o, why) in zip(blobs, res):
        assert why is None
        assert o == tool(b, tool_args(5))[1]
    dec = fb.Decoder(2, 16, 44100, 4096)
    try:
        infos, _ = dec.index_files(blobs)
        idx = [k for k in range(9) if k % 3 == 0]
        enc = fb.Encoder(fb.preset(*fmts[0], 5))
        enc.set_verify(True)
        try:
            host, hinfo = enc.reencode_flac_files(dec, idx, infos=True)
            assert all(v.status == fb.VERIFY_OK for v in enc.verify_info(len(idx)))
            cap = enc.reencode_capacity(dec, idx)
            d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
            d_off = torch.zeros(10000, dtype=torch.int64, device="cuda")
            nf, dinfo = enc.reencode_flac_files_device(dec, idx, d_out.data_ptr(), cap, d_off.data_ptr())
            torch.cuda.synchronize()
            outb = d_out.cpu().numpy().tobytes()
            offs = d_off[:nf + 1].cpu().numpy()
            for h, hi, di in zip(host, hinfo, dinfo):
                assert outb[di.file.offset:di.file.offset + di.file.bytes] == h
                assert hi.file.offset == di.file.offset and hi.file.nframes == di.file.nframes
                first = int(di.file.first_frame)
                assert offs[first] == di.file.offset + di.file.audio_offset
            assert offs[nf] == dinfo[-1].file.offset + dinfo[-1].file.bytes
        finally:
            enc.close()
        # decoding each output gives the input's samples and MD5
        got = fb.Decoder(2, 16, 44100, 4096)
        try:
            want = dec.decode_files([blobs[k] for k in idx])
            again = got.decode_files(host)
            for (a, ia), (b, ib) in zip(want, again):
                assert np.array_equal(a, b) and ib.md5_state == 1 and bytes(ia.md5) == bytes(ib.md5)
        finally:
            got.close()
    finally:
        dec.close()


def test_launches_do_not_grow_with_files():
    need_tool()
    one = make_flac(4096 * 3 + 100, 2, 16, 44100, seed=5)
    counts = []
    for n in (1, 50):
        dec = fb.Decoder(2, 16, 44100, 4096)
        enc = fb.Encoder(fb.preset(2, 16, 44100, 5))
        try:
            dec.index_files([one] * n)
            n0 = enc.launches + dec.launches
            enc.reencode_flac_files(dec, list(range(n)))
            counts.append(enc.launches + dec.launches - n0)
        finally:
            enc.close()
            dec.close()
    assert counts[0] == counts[1]
