"""A seeded corpus of damaged .flac files, and the reference decoder's account of each -- test infrastructure only.

Each entry starts from a clean base file and applies one mutation class at a seeded place. A class is named for the decoder
rule it reaches: a bit flip in one region of a frame, a byte inserted or deleted, a truncation, lost frames (one, and runs
around the reference's 50-frame and 5-second caps on silence), frames repeated or reordered, header look-alikes with a valid
CRC-8 (inside a verbatim frame's samples, in junk, and a damaged frame holding a complete frame), frames whose header
disagrees with STREAMINFO or whose samples do not fit bits per sample, junk and tags, two damaged stretches, and damage
across the chunk boundary of a decode with max_frames_per_launch = 8.

trace() drives the reference libFLAC's FLAC__stream_decoder_* API (oracle/_ref/libFLAC_ref.so, or any library with the same
API, such as libflac_b200.so) over a file held in memory, with the read, seek, tell, length and eof callbacks init_FILE would
give it, and records every write and every error in order. tool_decode() runs the reference flac tool's `flac -d` over the
corpus in one process.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from dataclasses import dataclass, field

import numpy as np

import flacsynth as fs
import refcli
import reflib
import signals

# ---------------------------------------------------------------- frames


def header_len(frame):
    """Bytes of a frame header before its CRC-8."""
    n = 0
    while n < 7 and frame[4] & (0x80 >> n):
        n += 1
    pos = 5 + (n - 1 if n > 1 else 0)
    bs_code, sr_code = frame[2] >> 4, frame[2] & 15
    pos += 1 if bs_code == 6 else 2 if bs_code == 7 else 0
    pos += 1 if sr_code == 12 else 2 if sr_code in (13, 14) else 0
    return pos


def const_frame(number, bs, rate, ch, bps, value=0, variable=False, rate_in_header=False):
    """A valid frame of CONSTANT subframes: blocksize, rate, channels and bits per sample in its header."""
    h = fs.BitWriter()
    h.put(0x3FFE, 14)
    h.put(0, 1)
    h.put(1 if variable else 0, 1)
    h.put(7, 4)
    h.put(13 if rate_in_header else 0, 4)
    h.put(ch - 1, 4)
    h.put(fs.BPS_CODE[bps], 3)
    h.put(0, 1)
    head = h.getbytes() + fs.utf8_number(number) + (bs - 1).to_bytes(2, "big")
    if rate_in_header:
        head += rate.to_bytes(2, "big")
    head += bytes([fs.crc8(head)])
    b = fs.BitWriter()
    for _ in range(ch):
        b.put(0, 8)
        b.put(value & ((1 << bps) - 1), bps)
    b.pad(0)
    body = head + b.getbytes()
    return body + fs.crc16(body).to_bytes(2, "big")


def verbatim_frame(number, pcm, bps, plant=()):
    """A valid frame of VERBATIM subframes (fixed blocking, rate and bits per sample from STREAMINFO) whose first channel's
    samples spell each (sample index, bytes) of `plant` in their big-endian bytes."""
    pcm = pcm.copy()
    step = bps // 8
    for at, blob in plant:
        blob = bytes(blob) + bytes(-len(blob) % step)
        for j in range(len(blob) // step):
            v = int.from_bytes(blob[j * step:(j + 1) * step], "big", signed=True)
            pcm[at + j, 0] = v
    bs, ch = pcm.shape
    h = fs.BitWriter()
    h.put(0x3FFE, 14)
    h.put(0, 2)
    h.put(7, 4)
    h.put(0, 4)
    h.put(ch - 1, 4)
    h.put(0, 4)
    head = h.getbytes() + fs.utf8_number(number) + (bs - 1).to_bytes(2, "big")
    head += bytes([fs.crc8(head)])
    b = fs.BitWriter()
    for c in range(ch):
        b.put(2, 8)
        b.put_array(pcm[:, c].astype(np.int64) & ((1 << bps) - 1), bps)
    body = head + b.getbytes()
    return body + fs.crc16(body).to_bytes(2, "big"), pcm


def streaminfo(min_bs, max_bs, rate, ch, bps, total, md5):
    packed = (rate << 44) | ((ch - 1) << 41) | ((bps - 1) << 36) | total
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + min_bs.to_bytes(2, "big") + max_bs.to_bytes(2, "big") + bytes(6) + packed.to_bytes(8, "big") + md5


def md5_of(x, bps):
    return hashlib.md5(x.astype("<i4").view(np.uint8).reshape(-1, 4)[:, :(bps + 7) // 8].tobytes()).digest()


# ---------------------------------------------------------------- bases


@dataclass
class Base:
    name: str
    head: bytes               # "fLaC" + metadata
    frames: list              # frame bytes
    pcm: np.ndarray           # int32 [samples, channels]
    ch: int
    bps: int
    rate: int
    bs: int                   # fixed blocksize (0: variable blocking)
    starts: list = field(default_factory=list)   # first sample of each frame

    def file(self, frames=None, tail=b""):
        return self.head + b"".join(self.frames if frames is None else frames) + tail


def ref_base(name, n, ch, bps, rate, bs, seed):
    """Frames by the reference encoder, STREAMINFO with total_samples and MD5 written in (its harness has no seek callback)."""
    x = signals.music_like(n, ch, bps, rate, seed=seed)
    stream, hdr, frames = reflib.encode(x, bps, rate=rate, level=5, blocksize=bs, md5=True, opts=reflib.RefEncOpts(streamable_subset=0))
    head = streaminfo(bs, bs, rate, ch, bps, n, md5_of(x, bps))  # the encoder's other metadata blocks are left out
    return Base(name, head, list(frames), x, ch, bps, rate, bs, [i * bs for i in range(len(frames))])


def synth_variable_base(seed):
    """Variable blocking (sample-numbered frames) from flacsynth: stereo 16-bit, blocksizes 32-600."""
    rng = np.random.default_rng(seed)
    fmt = fs.Format(2, 16, 44100)
    frames, pcm, starts, sample = [], [], [], 0
    for _ in range(40):
        f = fs.make_frame(rng, fmt, int(rng.integers(32, 600)), sample, True)
        frames.append(f.data)
        pcm.append(f.pcm)
        starts.append(sample)
        sample += f.blocksize
    x = np.concatenate(pcm)
    bss = [p.shape[0] for p in pcm]
    head = streaminfo(min(bss), max(bss), fmt.rate, 2, 16, len(x), md5_of(x, 16))
    return Base("var16", head, frames, x, 2, 16, fmt.rate, 0, starts)


def verbatim_base(seed, nframes=24, bs=1152):
    """Mono 16-bit 8 kHz verbatim frames: byte-aligned samples where header look-alikes can be planted."""
    rng = np.random.default_rng(seed)
    frames, pcm = [], []
    for i in range(nframes):
        f, p = verbatim_frame(i, rng.integers(-30000, 30000, size=(bs, 1)).astype(np.int32), 16)
        frames.append(f)
        pcm.append(p)
    x = np.concatenate(pcm)
    return Base("verb16", streaminfo(bs, bs, 8000, 1, 16, len(x), md5_of(x, 16)), frames, x, 1, 16, 8000, bs,
                [i * bs for i in range(nframes)])


# ---------------------------------------------------------------- the corpus


@dataclass
class Entry:
    name: str
    cls: str
    base: Base
    data: bytes
    where: tuple = ()         # the frame indices the mutation touched


# the regions of a frame a bit flip may hit: (class, function (frame, rng) -> (byte offset, bit mask))
def _flip_regions():
    return {
        "flip_sync": lambda f, r: (lambda at: (at, 1 << int(r.integers(2 if at else 0, 8))))(int(r.integers(0, 2))),
        "flip_reserved": lambda f, r: (1, 0x02),
        "flip_bs_code": lambda f, r: (2, 0x10 << int(r.integers(0, 4))),
        "flip_rate_code": lambda f, r: (2, 1 << int(r.integers(0, 4))),
        "flip_ch_code": lambda f, r: (3, 0x10 << int(r.integers(0, 4))),
        "flip_bps_code": lambda f, r: (3, 0x02 << int(r.integers(0, 3))),
        "flip_number": lambda f, r: (4, 1 << int(r.integers(0, 7))),
        "flip_crc8": lambda f, r: (header_len(f), 1 << int(r.integers(0, 8))),
        "flip_subframe_header": lambda f, r: (header_len(f) + 1, 1 << int(r.integers(1, 8))),
        "flip_residual": lambda f, r: (int(r.integers(header_len(f) + 4, len(f) - 2)), 1 << int(r.integers(0, 8))),
        "flip_crc16": lambda f, r: (len(f) - 2 + int(r.integers(0, 2)), 1 << int(r.integers(0, 8))),
    }


FLIP_CLASSES = tuple(_flip_regions())
LOST_RUNS = (1, 49, 50, 51, 60)


def _flip(frame, at, mask):
    b = bytearray(frame)
    b[at] ^= mask
    return bytes(b)


def _with_crcs(frame):
    """The frame with its CRC-8 and CRC-16 recomputed over its (edited) bytes."""
    hl = header_len(frame)
    b = bytearray(frame)
    b[hl] = fs.crc8(b[:hl])
    b[-2:] = fs.crc16(b[:-2]).to_bytes(2, "big")
    return bytes(b)


def _junk(rng, n):
    return bytes(rng.integers(0, 0xFF, size=n, dtype=np.uint8))  # no 0xFF: no sync code


def mutations(base, rng):
    """Every class that fits this base: [(class, frames, tail, where)]."""
    F, n = base.frames, len(base.frames)
    out = []

    def k_mid():
        return int(rng.integers(2, n - 3))

    regions = _flip_regions()
    for cls in FLIP_CLASSES:
        k = k_mid()
        at, mask = regions[cls](F[k], rng)
        out.append((cls, F[:k] + [_flip(F[k], at, mask)] + F[k + 1:], b"", (k,)))
    # a reserved bit set in a header whose CRCs are valid: the sync's (libFLAC never syncs on it) and the one after the
    # bits-per-sample code (libFLAC reads the header and reports it unparseable)
    k = k_mid()
    out.append(("reserved_sync_valid_crc", F[:k] + [_with_crcs(_flip(F[k], 1, 0x02))] + F[k + 1:], b"", (k,)))
    k = k_mid()
    out.append(("reserved_bps_valid_crc", F[:k] + [_with_crcs(_flip(F[k], 3, 0x01))] + F[k + 1:], b"", (k,)))
    k = k_mid()
    at = int(rng.integers(header_len(F[k]) + 2, len(F[k]) - 2))
    out.append(("insert_byte", F[:k] + [F[k][:at] + bytes([int(rng.integers(0, 255))]) + F[k][at:]] + F[k + 1:], b"", (k,)))
    k = k_mid()
    at = int(rng.integers(header_len(F[k]) + 2, len(F[k]) - 2))
    out.append(("delete_byte", F[:k] + [F[k][:at] + F[k][at + 1:]] + F[k + 1:], b"", (k,)))
    # truncations: the file ends inside the last kept frame's header, subframes or footer, or between two frames
    k = k_mid()
    out.append(("trunc_header", F[:k] + [F[k][:3]], b"", (k,)))
    out.append(("trunc_subframe", F[:k] + [F[k][:header_len(F[k]) + 1 + (len(F[k]) - header_len(F[k])) // 2]], b"", (k,)))
    out.append(("trunc_footer", F[:k] + [F[k][:-1]], b"", (k,)))
    out.append(("trunc_between", F[:k], b"", (k,)))
    out.append(("lost_first", F[1:], b"", (0,)))
    out.append(("lost_last", F[:-1], b"", (n - 1,)))
    for run in LOST_RUNS:
        if n >= run + 4:
            k = int(rng.integers(1, n - run - 1))
            out.append((f"lost_run{run}", F[:k] + F[k + run:], b"", tuple(range(k, k + run))))
    if base.bs and base.rate * 5 < 50 * base.bs and n * base.bs > base.rate * 5 + 3 * base.bs:
        run = (base.rate * 5) // base.bs + 2
        out.append(("lost_run_5s", F[:1] + F[1 + run:], b"", tuple(range(1, 1 + run))))
    k = k_mid()
    out.append(("repeat", F[:k + 1] + [F[k]] + F[k + 1:], b"", (k,)))
    k = k_mid()
    out.append(("swap", F[:k] + [F[k + 1], F[k]] + F[k + 2:], b"", (k, k + 1)))
    k = k_mid()
    out.append(("move_to_end", F[:k] + F[k + 1:] + [F[k]], b"", (k,)))
    # header look-alikes with a valid CRC-8: in junk between frames, and a damaged frame that holds a complete frame
    k = k_mid()
    nxt = F[k + 1]
    out.append(("lookalike_junk", F[:k + 1] + [nxt[:header_len(nxt) + 1] + _junk(rng, 40)] + F[k + 1:], b"", (k + 1,)))
    k = k_mid()
    cut = header_len(F[k]) + 1 + (len(F[k]) - header_len(F[k])) // 2
    out.append(("embedded_frame", F[:k] + [F[k][:cut] + F[k] + F[k][cut:]] + F[k + 1:], b"", (k,)))
    # junk with no header between frames; tags after the last frame
    k = k_mid()
    out.append(("junk_between", F[:k] + [_junk(rng, int(rng.integers(1, 200)))] + F[k:], b"", (k,)))
    out.append(("id3v1_tail", F, b"TAG" + bytes(125), ()))
    out.append(("ape_tail", F, b"APETAGEX" + (2000).to_bytes(4, "little") + (32).to_bytes(4, "little") + bytes(16), ()))
    # two damaged stretches; damage across the chunk boundary of max_frames_per_launch = 8
    k = int(rng.integers(2, max(3, n // 2 - 2)))
    k2 = int(rng.integers(k + 3, n - 1))
    out.append(("two_stretches", F[:k] + [_flip(F[k], len(F[k]) // 2, 0x10)] + F[k + 1:k2] + [_flip(F[k2], len(F[k2]) // 2, 0x10)] + F[k2 + 1:],
                b"", (k, k2)))
    if n > 10:
        out.append(("chunk_boundary", F[:7] + [_flip(F[7], len(F[7]) // 2, 0x04), _flip(F[8], len(F[8]) // 2, 0x04)] + F[9:], b"", (7, 8)))
    # frames with valid CRCs that break a rule of the stream (fixed blocking only: the frame replaces frame k by number)
    if base.bs:
        k = k_mid()
        others = [c for c in (1, 2, 6) if c != base.ch]
        out.append(("mismatch_channels", F[:k] + [const_frame(k, base.bs, base.rate, others[0], base.bps)] + F[k + 1:], b"", (k,)))
        obps = 16 if base.bps != 16 else 24
        out.append(("mismatch_bps", F[:k] + [const_frame(k, base.bs, base.rate, base.ch, obps)] + F[k + 1:], b"", (k,)))
        orate = 16000 if base.rate != 16000 else 8000
        out.append(("mismatch_rate", F[:k] + [const_frame(k, base.bs, orate, base.ch, base.bps, rate_in_header=True)] + F[k + 1:], b"", (k,)))
        out.append(("blocksize_over_max", F[:k] + [const_frame(k, base.bs + 1, base.rate, base.ch, base.bps)] + F[k + 1:], b"", (k,)))
        if base.bps in (8, 16, 24):
            oob = fs.make_frame(rng, fs.Format(base.ch, base.bps, base.rate), base.bs, k, False, invalid="sample_range")
            out.append(("out_of_bounds", F[:k] + [oob.data] + F[k + 1:], b"", (k,)))
    return out


def lookalike_mutations(base, rng):
    """Header look-alikes planted in a good verbatim frame's samples (base: verbatim_base): the reference never looks inside
    a frame it decoded, so the file decodes clean."""
    F, n, bs = base.frames, len(base.frames), base.bs
    out = []
    for cls, count in (("lookalike_verbatim", 1), ("lookalike_verbatim32", 32)):
        k = int(rng.integers(2, n - 3))
        nxt = F[k + 1][:header_len(F[k + 1]) + 1]
        plant = [(8 + 8 * j, nxt) for j in range(count)]
        f, pcm = verbatim_frame(k, base.pcm[k * bs:(k + 1) * bs], 16, plant)
        out.append((cls, F[:k] + [f] + F[k + 1:], b"", (k,), (k, pcm)))
    # a complete valid frame (numbered like the next one) inside a verbatim frame
    k = int(rng.integers(2, n - 3))
    f, pcm = verbatim_frame(k, base.pcm[k * bs:(k + 1) * bs], 16, [(100, const_frame(k + 1, bs, base.rate, 1, 16, value=0x1234))])
    out.append(("frame_in_verbatim", F[:k] + [f] + F[k + 1:], b"", (k,), (k, pcm)))
    return out


_BASES = None


def bases():
    global _BASES
    if _BASES is None:
        _BASES = [
            ref_base("s16_bs192", 192 * 80, 2, 16, 8000, 192, seed=11),
            ref_base("m8_bs16", 16 * 120, 1, 8, 8000, 16, seed=12),
            ref_base("x6_24_bs1152", 1152 * 14 + 500, 6, 24, 48000, 1152, seed=13),
            ref_base("s16_8k_bs4096", 4096 * 16, 2, 16, 8000, 4096, seed=14),
            ref_base("m24_bs4096", 4096 * 12 + 77, 1, 24, 44100, 4096, seed=15),
            synth_variable_base(seed=16),
            verbatim_base(seed=17),
        ]
    return _BASES


_CORPUS = None


def corpus(seed=20261018):
    """[Entry]: every base clean, then every class that fits each base, at seeded places."""
    global _CORPUS
    if _CORPUS is not None:
        return _CORPUS
    rng = np.random.default_rng(seed)
    out = []
    for b in bases():
        out.append(Entry(f"{b.name}/clean", "clean", b, b.file()))
        muts = mutations(b, rng)
        if b.name == "verb16":
            for cls, frames, tail, where, (k, pcm) in lookalike_mutations(b, rng):
                b2 = Base(b.name, b.head, b.frames, b.pcm.copy(), b.ch, b.bps, b.rate, b.bs, b.starts)
                b2.pcm[k * b.bs:(k + 1) * b.bs] = pcm
                b2.head = streaminfo(b.bs, b.bs, b.rate, 1, 16, len(b2.pcm), md5_of(b2.pcm, 16))
                out.append(Entry(f"{b.name}/{cls}", cls, b2, b2.head + b"".join(frames) + tail, where))
        for cls, frames, tail, where in muts:
            out.append(Entry(f"{b.name}/{cls}", cls, b, b.head + b"".join(frames) + tail, where))
    _CORPUS = out
    return out


# ---------------------------------------------------------------- the decoder API trace

DREAD = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_ubyte), C.POINTER(C.c_size_t), C.c_void_p)
DSEEK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_void_p)
DTELL = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p)
DLEN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p)
DEOF = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p)
DWRITE = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.POINTER(C.c_int32)), C.c_void_p)
DMETA = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p)
DERR = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_void_p)

LOST_SYNC, BAD_HEADER, FRAME_CRC_MISMATCH, UNPARSEABLE_STREAM, BAD_METADATA, OUT_OF_BOUNDS, MISSING_FRAME = range(7)


def api(lib):
    """Argument types of the FLAC__stream_decoder_* calls used here, set on a loaded library."""
    lib.FLAC__stream_decoder_new.restype = C.c_void_p
    lib.FLAC__stream_decoder_init_stream.argtypes = [C.c_void_p, DREAD, DSEEK, DTELL, DLEN, DEOF, DWRITE, DMETA, DERR, C.c_void_p]
    lib.FLAC__stream_decoder_set_md5_checking.argtypes = [C.c_void_p, C.c_int]
    for n in ("finish", "delete", "get_state", "process_until_end_of_stream"):
        getattr(lib, "FLAC__stream_decoder_" + n).argtypes = [C.c_void_p]
    return lib


def ref_lib():
    return api(C.CDLL(os.path.join(reflib.REF_DIR, "libFLAC_ref.so")))


@dataclass
class Write:
    sample: int
    blocksize: int
    rate: int
    bps: int
    pcm: np.ndarray           # int32 [blocksize, channels]


@dataclass
class Trace:
    events: list              # Write, or an int error status, in the order the callbacks came
    state: int                # decoder state after process_until_end_of_stream
    ok: bool                  # process_until_end_of_stream's result
    md5_ok: bool              # finish()'s result (MD5 checking on)

    @property
    def writes(self):
        return [e for e in self.events if isinstance(e, Write)]

    @property
    def errors(self):
        return [e for e in self.events if not isinstance(e, Write)]

    def error_marks(self):
        """For each error, how many writes came before it; as a sorted set (where errors fall between writes)."""
        marks, w = set(), 0
        for e in self.events:
            if isinstance(e, Write):
                w += 1
            else:
                marks.add(w)
        return sorted(marks)


def trace(lib, data):
    """Decode `data` through the library's stream decoder with callbacks over the bytes, as init_FILE sets them up."""
    st = {"pos": 0}
    events = []

    def read(dec, buf, nbytes, client):
        n = min(nbytes[0], len(data) - st["pos"])
        if n <= 0:
            nbytes[0] = 0
            return 1  # END_OF_STREAM
        C.memmove(buf, data[st["pos"]:st["pos"] + n], n)
        st["pos"] += n
        nbytes[0] = n
        return 0

    def seek(dec, off, client):
        if off > len(data):
            return 1
        st["pos"] = off
        return 0

    def tell(dec, out, client):
        out[0] = st["pos"]
        return 0

    def length(dec, out, client):
        out[0] = len(data)
        return 0

    def eof(dec, client):
        return int(st["pos"] >= len(data))

    def write(dec, frame, buffers, client):
        h = C.cast(frame, C.POINTER(C.c_uint32))
        bs, ch = h[0], h[2]
        sample = C.cast(frame + 24, C.POINTER(C.c_uint64))[0]
        blk = np.stack([np.ctypeslib.as_array(buffers[c], shape=(bs,)).copy() for c in range(ch)], axis=1) if bs else np.zeros((0, ch), np.int32)
        events.append(Write(int(sample), int(bs), int(h[1]), int(h[4]), blk))
        return 0

    def meta(dec, m, client):
        pass

    def error(dec, status, client):
        events.append(int(status))

    cbs = (DREAD(read), DSEEK(seek), DTELL(tell), DLEN(length), DEOF(eof), DWRITE(write), DMETA(meta), DERR(error))
    d = C.c_void_p(lib.FLAC__stream_decoder_new())
    lib.FLAC__stream_decoder_set_md5_checking(d, 1)
    assert lib.FLAC__stream_decoder_init_stream(d, *cbs, None) == 0
    ok = bool(lib.FLAC__stream_decoder_process_until_end_of_stream(d))
    state = int(lib.FLAC__stream_decoder_get_state(d))
    md5_ok = bool(lib.FLAC__stream_decoder_finish(d))
    lib.FLAC__stream_decoder_delete(d)
    return Trace(events, state, ok, md5_ok)


def is_silence(prev, w):
    """A frame the decoder made up for a gap: all zero, right after the previous write and in its format (the reference copies
    that frame's header), no longer than it. No frame of the corpus is all zero in the stream's own format."""
    return prev is not None and w.sample == prev.sample + prev.blocksize and w.blocksize <= prev.blocksize and not w.pcm.any() \
        and (w.rate, w.bps, w.pcm.shape[1]) == (prev.rate, prev.bps, prev.pcm.shape[1])


def placed(tr, samples, ch):
    """The output the engine promises from a trace: every frame at its sample number, zeros elsewhere, cut at `samples`.
    Returns (pcm, covered) where covered marks the samples some decoded frame (not a silence frame) wrote."""
    out = np.zeros((samples, ch), np.int32)
    covered = np.zeros(samples, bool)
    prev = None
    for w in tr.writes:
        silent = is_silence(prev, w)
        prev = w
        if w.sample >= samples or w.pcm.shape[1] != ch:
            continue
        m = min(w.blocksize, samples - w.sample)
        out[w.sample:w.sample + m] = w.pcm[:m]
        if not silent:
            covered[w.sample:w.sample + m] = True
    return out, covered


def sequential(tr):
    """The reference's output as its client sees it: every write in order."""
    ws = tr.writes
    return np.concatenate([w.pcm for w in ws]) if ws else None


def ascending(tr):
    """True when every write starts where the previous one ended (no overlap, no gap left after silence)."""
    end = None
    for w in tr.writes:
        if end is not None and w.sample != end:
            return False
        end = w.sample + w.blocksize
    return True


# ---------------------------------------------------------------- the flac tool


def tool_decode(blobs):
    """`flac -d -f -s` on each file, one process per file. Returns [(exit status, output bytes or None where the tool deleted
    its output)]."""
    res = []
    with tempfile.TemporaryDirectory() as d:
        for i, b in enumerate(blobs):
            p = os.path.join(d, f"f{i}.flac")
            with open(p, "wb") as fh:
                fh.write(bytes(b))
            r = subprocess.run([refcli.PATH, "-d", "-f", "-s", p], capture_output=True, timeout=120)
            o = p[:-5] + ".wav"
            res.append((r.returncode, open(o, "rb").read() if os.path.exists(o) else None))
        return res


# ---------------------------------------------------------------- the frame-header scan


_UTF8_LEAD = ((0x80, 0x00), (0xE0, 0xC0), (0xF0, 0xE0), (0xF8, 0xF0), (0xFC, 0xF8), (0xFE, 0xFC), (0xFF, 0xFE))


def scan(buf):
    """Every byte offset that carries a sync code and a self-consistent frame header, restated from libFLAC's frame_sync_ and
    read_frame_header_ (stream_decoder.c:2321-2371, 2624-2947): sync 0xFFF8 / 0xFFF9 (reserved bit 0), blocksize code not 0,
    rate code not 15, channel code at most 10, bits-per-sample code not 3, the reserved bit after it 0, a well-formed UTF-8
    number (7 bytes only with variable blocking), the whole header and its CRC-8 inside the buffer, and the CRC-8 right."""
    b = np.frombuffer(bytes(buf), dtype=np.uint8)
    n = b.size
    out = []
    if n < 6:
        return out
    q = np.nonzero((b[:n - 5] == 0xFF) & ((b[1:n - 4] & 0xFE) == 0xF8))[0]
    for p in q.tolist():
        h = b[p:]
        bs_code, sr_code, ca_code, bps_code = h[2] >> 4, h[2] & 15, h[3] >> 4, (h[3] >> 1) & 7
        if (h[3] & 1) or bs_code == 0 or sr_code == 15 or ca_code > 10 or bps_code == 3:
            continue
        first = int(h[4])
        # continuation bytes after the lead byte: 0xxxxxxx 0, 110xxxxx 1, 1110xxxx 2, ... 1111110x 5, 11111110 6
        nb = next((k for k, (mask, val) in enumerate(_UTF8_LEAD) if first & mask == val), None)
        if nb is None or (nb == 6 and not h[1] & 1):
            continue
        hl = 5 + nb + (1 if bs_code == 6 else 2 if bs_code == 7 else 0) + (1 if sr_code == 12 else 2 if sr_code >= 13 else 0)
        if hl + 1 > n - p:
            continue
        if any((int(h[5 + k]) & 0xC0) != 0x80 for k in range(nb)):
            continue
        if fs.crc8(bytes(h[:hl])) != h[hl]:
            continue
        out.append(p)
    return out
