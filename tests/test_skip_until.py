"""fb200_skip_until (flac_b200.skip_until): the flac tool's --skip / --until arithmetic, checked against the tool itself. A ramp
(each sample's value is its index) is encoded by oracle/_ref/flac_ref with the same strings and the tool's output decoded by the
tool: the first decoded value is the range's first sample, STREAMINFO's total its length, and every pair the tool refuses is
FB200_ERR_INVALID here. Needs no GPU."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import flac_b200 as fb
import refcli
from test_pcm_probe import fmt_chunk, pack, wav


def need_tool():
    if not refcli.available():
        pytest.skip("oracle/_ref/flac_ref not built")


def ramp_wav(n, rate):
    """24-bit mono WAV whose sample i holds i - 2^23"""
    x = (np.arange(n, dtype=np.int64) - (1 << 23)).astype(np.int32).reshape(-1, 1)
    return wav(pack(x, 24, 0), fmt_chunk(1, rate, 24))


def tool_range(blob, skip, until, name="in.wav"):
    """(exit code, first decoded index or None, STREAMINFO total or None) of flac [--skip] [--until] on blob"""
    args = ([f"--skip={skip}"] if skip is not None else []) + ([f"--until={until}"] if until is not None else [])
    rc, out, _ = refcli.encode(blob, args, name=name)
    if rc != 0:
        return rc, None, None
    total = refcli.streaminfo(out)[3]
    if total == 0:
        return rc, None, 0
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "a.flac"), os.path.join(d, "a.raw")
        with open(src, "wb") as f:
            f.write(out)
        r = subprocess.run([refcli.PATH, "-d", "-f", "-s", "--force-raw-format", "--endian=little", "--sign=signed", src, "-o", dst],
                           capture_output=True, timeout=300)
        assert r.returncode == 0, r.stderr
        raw = open(dst, "rb").read(3)
    first = int.from_bytes(raw, "little", signed=True) + (1 << 23)
    return rc, first, total


def ours(skip, until, rate, total):
    try:
        return fb.skip_until(skip, until, rate, total)
    except fb.FlacB200Error as e:
        assert e.code == -3, e
        return None


RATE = 44100
N = 2 * RATE + 123
CASES = [
    (None, None), ("0", None), ("1000", "5000"), ("1000", None), (None, "5000"),
    ("0:00.1", "0:01.5"), ("0:00,1", "0:01,5"), ("0:01.000", None), ("00:00.5", "1:0"),
    ("0:00.7", "0:01.3"), ("0:00.29", "0:00.57"), ("0:01.9", None),  # seconds * rate just below an integer
    ("1000", "+500"), ("1000", "-500"), ("1000", "-0"), ("1000", "+0"), (None, "-0"), (None, "+0"), ("0:00.5", "+0:00.25"),
    (None, "-0:00.5"), ("0", str(N)), (str(N - 1), None), ("0", "1"),
    (str(N), None),                                     # skip at the length: the tool writes no frames
    ("1000", "500"), ("1000", "1000"), (None, str(N + 1)), (str(N + 1), None), (None, "-999999"), ("0:03", None), (None, "0:03"),
    ("+10", None), ("-10", None), ("+0", None),        # a relative skip
    ("abc", None), (None, "1:xx"), ("1.5", None), ("", None), (None, ""), ("1:2:3", None), ("9223372036854775808", None),
    ("99999999999999999999", None), ("0:99999999999999999", None), (None, "+-5"), ("0x10", None), (" 5", None),
]


@pytest.mark.parametrize("skip,until", CASES)
def test_against_the_tool(skip, until):
    need_tool()
    rc, first, total = tool_range(ramp_wav(N, RATE), skip, until)
    got = ours(skip, until, RATE, N)
    if rc != 0:
        assert got is None, (rc, got)
    elif total == 0:
        assert got is None, "a range of 0 samples is refused (the tool writes a stream without frames)"
    else:
        assert got == (first, total)


def test_low_rate_relative_zero():
    """At 8 kHz -0:00.00001 is -0.08 samples: truncated to 0, so the end of the stream, as the tool has it"""
    need_tool()
    n = 8000 + 17
    for skip, until in [(None, "-0:00.00001"), ("100", "+0:00.0001"), ("100", "-0:00.0002")]:
        rc, first, total = tool_range(ramp_wav(n, 8000), skip, until)
        assert rc == 0
        assert ours(skip, until, 8000, n) == (first, total)


def test_unknown_length():
    """STREAMINFO total_samples 0: any --until but the end is refused, and so is a --skip past 0"""
    need_tool()
    n = 30000
    rc, flac, _ = refcli.encode(ramp_wav(n, RATE), ["-S-"])
    assert rc == 0
    blob = bytearray(flac)
    blob[8 + 13] &= 0xF0
    blob[8 + 14:8 + 18] = bytes(4)
    for skip, until in [(None, "1000"), (None, "-5"), (None, "+5"), ("10", None), ("10", "-0"), (None, None)]:
        rc, first, total = tool_range(bytes(blob), skip, until, name="in.flac")
        got = ours(skip, until, RATE, 0)
        assert got is None  # either the tool refuses it, or it encodes an unknown length this engine does not take
        if until not in (None, "-0") or skip not in (None, "0"):
            assert rc != 0, (skip, until)


def test_messages():
    with pytest.raises(fb.FlacB200Error, match="invalid value for --skip"):
        fb.skip_until("+1", None, RATE, N)
    with pytest.raises(fb.FlacB200Error, match="invalid value for --until"):
        fb.skip_until(None, "x", RATE, N)
    with pytest.raises(fb.FlacB200Error, match="--until value is before --skip point"):
        fb.skip_until("10", "5", RATE, N)
    with pytest.raises(fb.FlacB200Error, match="--until value is after end of input"):
        fb.skip_until(None, str(N + 1), RATE, N)
    with pytest.raises(fb.FlacB200Error, match="value of --skip exceeds input size"):
        fb.skip_until(str(N + 1), None, RATE, N)
    with pytest.raises(fb.FlacB200Error, match="cannot use --until when input length is unknown"):
        fb.skip_until(None, "5", RATE, 0)
    with pytest.raises(fb.FlacB200Error, match="value of --skip is too large"):
        fb.skip_until("0:99999999999999999", None, RATE, N)
    assert fb.skip_until("0:00.1", "+0:00.1", RATE, N) == (4410, 4410)
