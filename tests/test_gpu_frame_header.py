"""The FLAC frame-header reader on every decode path: the block path's status (k_dec_walk), the stream index (k_dec_scan)
and the whole-file index (the host reader). Single synthesised frames (tests/flacsynth.py) get their header rewritten code
point by code point, reserved bit by reserved bit, UTF-8 length by UTF-8 length, with broken CRC-8s and syncs, and cut by
the end of the bytes given. The three readers must agree: the block path reports the first rule a header breaks, in the
order sync, early header rules, CRC-8, late header rules; the index lists a frame iff its header holds; the files path
decodes it iff its header holds and agrees with STREAMINFO."""
import numpy as np
import pytest

import flacsynth as fs
from test_gpu_decode_grammar import _raw_block_decode

pytestmark = pytest.mark.gpu

OK, BAD_SYNC, BAD_HEADER, CRC8, UNSUPPORTED, LENGTH, MISMATCH = 0, 1, 2, 3, 4, 6, 8
HEADER_FAILURES = (BAD_SYNC, BAD_HEADER, CRC8, LENGTH)
CH, BPS, RATE, MAX_BS = 2, 16, 44100, 4608


def header(bs_code, sr_code, ca_code, bps_code, number_bytes, bs=0, sr_hint=b"", variable=False, res1=0, res2=0, sync=0x3FFE):
    """Header bytes with a correct CRC-8; hints: the blocksize from `bs`, the rate from `sr_hint`."""
    h = fs.BitWriter()
    h.put(sync, 14)
    h.put(res1, 1)
    h.put(1 if variable else 0, 1)
    h.put(bs_code, 4)
    h.put(sr_code, 4)
    h.put(ca_code, 4)
    h.put(bps_code, 3)
    h.put(res2, 1)
    head = h.getbytes() + number_bytes
    if bs_code == 6:
        head += bytes([bs - 1])
    elif bs_code == 7:
        head += (bs - 1).to_bytes(2, "big")
    head += sr_hint
    return head + bytes([fs.crc8(head)])


def header_bytes(data):
    """Length of the (valid) header at the start of a synthesised frame, CRC-8 included."""
    ones = 8 - (data[4] ^ 0xFF).bit_length()  # leading 1 bits of the number's first byte
    n = 5 + max(ones - 1, 0)
    bs_code, sr_code = data[2] >> 4, data[2] & 15
    n += {6: 1, 7: 2}.get(bs_code, 0) + {12: 1, 13: 2, 14: 2}.get(sr_code, 0)
    assert fs.crc8(data[:n]) == data[n]
    return n + 1


def rehead(f, head):
    """The frame f with its header replaced by `head` and the CRC-16 recomputed."""
    body = f.data[header_bytes(f.data):-2]
    frame = head + body
    return frame + fs.crc16(frame).to_bytes(2, "big")


def zero_number(nbytes):
    """Frame / sample number 0 in `nbytes` bytes of FLAC's UTF-8 coding (overlong for nbytes > 1; 7 bytes: lead 0xFE)."""
    if nbytes == 1:
        return b"\x00"
    lead = 0xFE if nbytes == 7 else (0xFF << (8 - nbytes)) & 0xFF
    return bytes([lead]) + b"\x80" * (nbytes - 1)


def flip_crc8(head):
    return head[:-1] + bytes([head[-1] ^ 0x01])


class Frames:
    """Base frames of the stream format, number 0, by (blocksize, channel assignment)."""

    def __init__(self):
        self.rng = np.random.default_rng(20261019)
        self.fmt = fs.Format(CH, BPS, RATE)
        self.cache = {}

    def get(self, bs=1152, ca=0, variable=False):
        key = (bs, ca, variable)
        if key not in self.cache:
            self.cache[key] = fs.make_frame(self.rng, self.fmt, bs, 0, variable, ca=ca)
        return self.cache[key]


def cases():
    """(name, base frame, frame bytes, block-path status). The base frame gives the PCM a valid frame decodes to."""
    F = Frames()
    z1 = zero_number(1)
    out = []

    def add(name, base, data, status):
        out.append((name, base, data, status))

    # blocksize codes: each valid code over a frame of that many samples; 13-15 exceed the decoder's blocksize
    bs_of = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, 6: 100, 7: 1000, **{c: 256 << (c - 8) for c in range(8, 13)}}
    for c in range(16):
        base = F.get(bs_of.get(c, 256))
        st = BAD_HEADER if c == 0 else MISMATCH if c >= 13 else OK
        add(f"bs_code{c}", base, rehead(base, header(c, 9, 1, 4, z1, bs=base.blocksize)), st)
    # sample-rate codes: the rate does not bind the block path; 12-14 carry a hint
    base = F.get()
    hints = {12: bytes([44]), 13: (44100).to_bytes(2, "big"), 14: (4410).to_bytes(2, "big")}
    for c in range(16):
        add(f"sr_code{c}", base, rehead(base, header(3, c, 1, 4, z1, sr_hint=hints.get(c, b""))), BAD_HEADER if c == 15 else OK)
    # channel codes: 1 and 8-10 are the stream's two channels (independent, left/side, right/side, mid/side)
    for c in range(16):
        b = F.get(ca=c - 7 if 8 <= c <= 10 else 0)
        st = OK if c in (1, 8, 9, 10) else MISMATCH if c < 8 else BAD_HEADER
        add(f"ca_code{c}", b, rehead(b, header(3, 9, c, 4, z1)), st)
    # bits-per-sample codes: 0 (STREAMINFO) and 4 (16) are the stream's; 7 (32 bits) is past what the decoder takes
    for c in range(8):
        st = {0: OK, 4: OK, 3: BAD_HEADER, 7: UNSUPPORTED}.get(c, MISMATCH)
        add(f"bps_code{c}", base, rehead(base, header(3, 9, 1, c, z1)), st)
    # reserved bits
    add("reserved_after_sync", base, rehead(base, header(3, 9, 1, 4, z1, res1=1)), BAD_HEADER)
    add("reserved_after_bps", base, rehead(base, header(3, 9, 1, 4, z1, res2=1)), BAD_HEADER)
    # UTF-8 numbers of 1-7 bytes, fixed and variable blocking; a bad continuation byte; bad lead bytes
    for variable in (False, True):
        b = F.get(variable=variable)
        for n in range(1, 8):
            num = zero_number(n)
            st = BAD_HEADER if n == 7 and not variable else OK
            add(f"utf8_{n}_var{int(variable)}", b, rehead(b, header(3, 9, 1, 4, num, variable=variable)), st)
            if n > 1:
                bad = num[:-1] + b"\x40"
                add(f"utf8_{n}_var{int(variable)}_bad_cont", b, rehead(b, header(3, 9, 1, 4, bad, variable=variable)), BAD_HEADER)
        for lead in (0x80, 0xBF, 0xFF):
            add(f"utf8_lead{lead:02x}_var{int(variable)}", b, rehead(b, header(3, 9, 1, 4, bytes([lead]), variable=variable)), BAD_HEADER)
    # CRC-8 and sync
    add("crc8", base, rehead(base, flip_crc8(header(3, 9, 1, 4, z1))), CRC8)
    add("sync_byte0", base, rehead(base, header(3, 9, 1, 4, z1, sync=0x3F7E)), BAD_SYNC)
    add("sync_byte1", base, rehead(base, header(3, 9, 1, 4, z1, sync=0x3FFC)), BAD_SYNC)
    add("sync_and_crc8", base, rehead(base, flip_crc8(header(3, 9, 1, 4, z1, sync=0x3FEE))), BAD_SYNC)
    # precedence: the early rules come before the CRC-8, the late ones (channel code, bps code 3) after it
    add("crc8_bs_code0", base, rehead(base, flip_crc8(header(0, 9, 1, 4, z1))), BAD_HEADER)
    add("crc8_sr_code15", base, rehead(base, flip_crc8(header(3, 15, 1, 4, z1))), BAD_HEADER)
    add("crc8_reserved", base, rehead(base, flip_crc8(header(3, 9, 1, 4, z1, res2=1))), BAD_HEADER)
    add("crc8_bad_utf8", base, rehead(base, flip_crc8(header(3, 9, 1, 4, b"\xC0\x40"))), BAD_HEADER)
    for c in (11, 12, 15):
        add(f"crc8_ca_code{c}", base, rehead(base, flip_crc8(header(3, 9, c, 4, z1))), CRC8)
    add("crc8_bps_code3", base, rehead(base, flip_crc8(header(3, 9, 1, 3, z1))), CRC8)
    # fewer than 6 bytes
    for n in range(1, 6):
        add(f"len{n}", base, base.data[:n], LENGTH)
    return out


def long_header_frame():
    """A frame whose header holds every optional field: a 3-byte number (0), 16-bit blocksize and 16-bit rate (12 bytes)."""
    F = Frames()
    base = F.get(bs=1000)
    head = header(7, 13, 1, 4, zero_number(3), bs=1000, sr_hint=(44100).to_bytes(2, "big"))
    assert len(head) == 12
    return base, rehead(base, head), len(head)


def _files(items):
    """One .flac file per (base frame, frame bytes): STREAMINFO of the base frame's format and blocksize."""
    fmt = fs.Format(CH, BPS, RATE)
    out = []
    for base, data in items:
        st = fs.Stream(fmt, data[1] & 1 == 1 if len(data) > 1 else False, [base], base.blocksize)
        out.append(fs.streaminfo_block(st, md5=False) + data)
    return out


def test_header_rules_on_every_path():
    import flac_b200
    cs = cases()
    frames = [fs.Frame(data=d, pcm=b.pcm, blocksize=b.blocksize, number=0, ca=b.ca, subs=[], facts=set()) for _, b, d, _ in cs]

    # (a) the block path, exact offsets
    dec = flac_b200.Decoder(CH, BPS, RATE, MAX_BS)
    try:
        pcm, status = _raw_block_decode(dec, frames)
        for i, (name, base, _, want) in enumerate(cs):
            assert (status[i] & 0xFF) == want, f"{name}: block path status {status[i] & 0xFF}, want {want}"
            if want == OK:
                assert np.array_equal(pcm[i * MAX_BS:i * MAX_BS + base.blocksize], base.pcm), name

        # (b) the stream index lists the frame iff its header holds
        for name, _, data, want in cs:
            listed = 0 in [int(c) for c in dec.index(np.frombuffer(data, dtype=np.uint8))]
            assert listed == (want not in HEADER_FAILURES), f"{name}: index lists it: {listed}"
    finally:
        dec.close()

    # (c) the whole-file index (host reader) takes the frame iff the block path decodes it
    dec = flac_b200.Decoder(CH, BPS, RATE, MAX_BS)
    try:
        res = dec.decode_files(_files([(b, d) for _, b, d, _ in cs]), md5=False)
        for (name, base, _, want), (y, info) in zip(cs, res):
            assert info.nframes == (1 if want == OK else 0), f"{name}: files path decoded {info.nframes} frames"
            if want == OK:
                assert np.array_equal(y, base.pcm), name
    finally:
        dec.close()


def test_header_cut_by_end_of_buffer():
    """The index and the files path never take a header that the end of the buffer cuts."""
    import flac_b200
    base, data, hl = long_header_frame()
    dec = flac_b200.Decoder(CH, BPS, RATE, MAX_BS)
    try:
        assert 0 in [int(c) for c in dec.index(np.frombuffer(data, dtype=np.uint8))]
        for n in range(1, hl):
            assert 0 not in [int(c) for c in dec.index(np.frombuffer(data[:n], dtype=np.uint8))], f"cut to {n} bytes"
        res = dec.decode_files(_files([(base, data)] + [(base, data[:n]) for n in range(1, hl)]), md5=False)
        assert res[0][1].nframes == 1 and np.array_equal(res[0][0], base.pcm)
        for n, (_, info) in zip(range(1, hl), res[1:]):
            assert info.nframes == 0, f"cut to {n} bytes"
    finally:
        dec.close()


def test_frame_shorter_than_its_header():
    """Block path: a frame whose given length ends inside its header is DEC_LENGTH, whatever bytes follow it."""
    import flac_b200
    base, data, hl = long_header_frame()
    cut = [fs.Frame(data=data[:n], pcm=base.pcm, blocksize=base.blocksize, number=0, ca=0, subs=[], facts=set()) for n in range(1, hl)]
    whole = fs.Frame(data=data, pcm=base.pcm, blocksize=base.blocksize, number=0, ca=0, subs=[], facts=set())
    frames = [f for c in cut for f in (c, whole)]  # each cut frame followed by the whole one: its header's bytes come next
    dec = flac_b200.Decoder(CH, BPS, RATE, MAX_BS)
    try:
        _, status = _raw_block_decode(dec, frames)
    finally:
        dec.close()
    for i in range(len(cut)):
        assert (status[2 * i] & 0xFF) == LENGTH, f"cut to {i + 1} bytes: status {status[2 * i] & 0xFF}"
        assert (status[2 * i + 1] & 0xFF) == OK
