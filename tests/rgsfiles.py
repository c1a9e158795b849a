"""Small .flac files with ReplayGain tags, made by the reference flac tool (oracle/_ref/flac_ref), and the tool's
--apply-replaygain-which-is-not-lossless decode over one or many of them -- test infrastructure only."""
import os
import subprocess
import tempfile

import refcli
from test_pcm_probe import fmt_chunk, pack, samples, wav


def tagged_flac(tags, ch=2, bps=16, n=3000, seed=0, args=()):
    """A .flac the tool encodes from an EXTENSIBLE WAV of n samples, with each of `tags` ("NAME=value") as a -T tag."""
    container = (bps + 7) // 8 * 8
    x = samples(n, ch, bps, seed)
    data = pack(x, container, container - bps, unsigned=container == 8)
    extra = ["--lax"] if bps < 8 else []
    for t in tags:
        extra += ["-T", t]
    rc, flac, err = refcli.encode(wav(data, fmt_chunk(ch, 44100, container, valid=bps, mask=0, extensible=True)), extra + list(args))
    assert rc == 0, err
    return flac


def add_vorbis_comment(flac, entries):
    """The .flac with one more VORBIS_COMMENT block (raw entries, bytes each) after its last metadata block."""
    b = bytearray(flac)
    body = (0).to_bytes(4, "little") + len(entries).to_bytes(4, "little") + b"".join(len(e).to_bytes(4, "little") + e for e in entries)
    pos = 4
    while True:
        last, length = b[pos] & 0x80, int.from_bytes(b[pos + 1:pos + 4], "big")
        if last:
            b[pos] &= 0x7F
            end = pos + 4 + length
            break
        pos += 4 + length
    b[end:end] = bytes([0x84]) + len(body).to_bytes(3, "big") + body
    return bytes(b)


def album_tags(track_gain, album_gain, track_peak=0.5, album_peak=0.7):
    return [f"REPLAYGAIN_TRACK_GAIN={track_gain:+.2f} dB", f"REPLAYGAIN_TRACK_PEAK={track_peak:.8f}",
            f"REPLAYGAIN_ALBUM_GAIN={album_gain:+.2f} dB", f"REPLAYGAIN_ALBUM_PEAK={album_peak:.8f}"]


def option(spec):
    return "--apply-replaygain-which-is-not-lossless" + ("" if spec is None else "=" + spec)


def tool_decode_many(flacs, spec, args=(), silent=True):
    """One `flac -d -f [-s] --apply-replaygain-which-is-not-lossless[=SPEC] [args] f0.flac f1.flac ...` process. Returns (exit code,
    [output bytes or None per file], stderr)."""
    with tempfile.TemporaryDirectory() as d:
        names = []
        for i, f in enumerate(flacs):
            p = os.path.join(d, f"f{i}.flac")
            with open(p, "wb") as fh:
                fh.write(bytes(f))
            names.append(p)
        ext = (".aifc" if any("aiff-c" in a for a in args) else ".aiff" if any("aiff" in a for a in args) else ".w64" if any("wave64" in a for a in args)
               else ".rf64" if any("rf64" in a for a in args) else ".wav")
        r = subprocess.run([refcli.PATH, "-d", "-f", *(["-s"] if silent else []), option(spec), *args, *names], capture_output=True, text=True,
                           timeout=600)
        outs = []
        for p in names:
            o = p[:-5] + ext
            outs.append(open(o, "rb").read() if os.path.exists(o) else None)
        return r.returncode, outs, r.stderr
