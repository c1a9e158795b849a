"""fb200_replaygain_synthesis_parse and fb200_replaygain_synthesis_file against the reference flac tool's own messages (flac -d
--apply-replaygain-which-is-not-lossless[=SPEC]): the option's parse, and the decision and gain it takes from each file's tags.
Device-free."""
import re

import pytest

import flac_b200 as fb
import refcli
from rgsfiles import add_vorbis_comment, album_tags, tagged_flac, tool_decode_many

pytestmark = pytest.mark.skipif(not refcli.available(), reason="oracle/_ref/flac_ref not built")

INFO = re.compile(r"INFO: applying (album|track) ReplayGain \(gain=(-?[0-9.]+)dB\+preamp=(-?[0-9.]+)dB, (no|low|medium|high) noise shaping, "
                  r"(no|peak|hard) limiting\)")


@pytest.fixture(scope="module")
def tagged():
    return tagged_flac(album_tags(-3.25, -5.5))


@pytest.mark.parametrize("spec", [None, "", "0", "6tln2", "-3aLn3", "1e1", "12an0", "n4", "x", "a b", "5n"])
def test_parse_matches_the_tool(tagged, spec):
    rc, _, err = tool_decode_many([tagged], spec, silent=False)
    try:
        rg = fb.replaygain_synthesis(spec)
    except fb.FlacB200Error:
        assert rc == 1 and "bad specification string" in err, err
        return
    assert rc == 0, err
    m = INFO.search(err)
    assert m, err
    assert m.group(1) == ("album" if rg.album else "track")
    assert m.group(3) == f"{rg.preamp:0.1f}"
    assert m.group(4) == ["no", "low", "medium", "high"][rg.noise_shaping]
    assert m.group(5) == ["no", "peak", "hard"][rg.limiter]


TAG_CASES = {
    "both": album_tags(-3.25, -5.5),
    "track_only": ["REPLAYGAIN_TRACK_GAIN=-2.50 dB", "REPLAYGAIN_TRACK_PEAK=0.5"],
    "album_only": ["REPLAYGAIN_ALBUM_GAIN=+4.75 dB", "REPLAYGAIN_ALBUM_PEAK=0.25"],
    "neither": ["TITLE=x"],
    "mixed_case": ["ReplayGain_Track_Gain=-1.50 dB", "replaygain_track_peak=0.4", "REPLAYGAIN_album_GAIN=+2.25 dB", "Replaygain_Album_Peak=0.3"],
    "plus_and_spaces": ["REPLAYGAIN_TRACK_GAIN=  +3.5 dB", "REPLAYGAIN_TRACK_PEAK=0.5", "REPLAYGAIN_ALBUM_GAIN=+3.5junk", "REPLAYGAIN_ALBUM_PEAK= 0.9x"],
    "long_values": ["REPLAYGAIN_TRACK_GAIN=-1.25000000000000000000000000000000000007 dB", "REPLAYGAIN_TRACK_PEAK=0.5",
                    "REPLAYGAIN_ALBUM_GAIN=-0.000000000000000000000000000012345", "REPLAYGAIN_ALBUM_PEAK=0.5"],
    "short_values": ["REPLAYGAIN_TRACK_GAIN=7", "REPLAYGAIN_TRACK_PEAK=0.5", "REPLAYGAIN_ALBUM_GAIN=12", "REPLAYGAIN_ALBUM_PEAK=1"],
    "negative_peak": ["REPLAYGAIN_TRACK_GAIN=-2.00 dB", "REPLAYGAIN_TRACK_PEAK=-0.5", "REPLAYGAIN_ALBUM_GAIN=-4.00 dB", "REPLAYGAIN_ALBUM_PEAK=0.5"],
    "gain_91": ["REPLAYGAIN_TRACK_GAIN=91 dB", "REPLAYGAIN_TRACK_PEAK=0.5", "REPLAYGAIN_ALBUM_GAIN=91 dB", "REPLAYGAIN_ALBUM_PEAK=0.5"],
    "no_peak": ["REPLAYGAIN_TRACK_GAIN=-2.00 dB", "REPLAYGAIN_ALBUM_GAIN=-4.00 dB", "REPLAYGAIN_ALBUM_PEAK=0.5"],
}


@pytest.mark.parametrize("case", sorted(TAG_CASES))
@pytest.mark.parametrize("spec", [None, "0tn1", "3l"])
def test_file_decision_matches_the_tool(case, spec):
    flac = tagged_flac(TAG_CASES[case])
    rc, _, err = tool_decode_many([flac], spec, silent=False)
    assert rc == 0, err
    info = fb.replaygain_synthesis_file(flac, spec)
    m = INFO.search(err)
    if info.status == fb.RGS_APPLIED:
        assert m, err
        assert m.group(2) == f"{info.gain:0.2f}", (err, info.gain, info.album_used)
    else:
        assert not m, err
        want = {fb.RGS_NO_TAGS: "can't get", fb.RGS_GAIN: "found gain value doesn't make sense", fb.RGS_BPS: "between 4 and 24"}[info.status]
        assert want in err, (info.status, err)


def test_32_bit_stream_is_decoded_plainly():
    flac = tagged_flac(album_tags(-1.0, -2.0), bps=32)
    rc, _, err = tool_decode_many([flac], None, silent=False)
    info = fb.replaygain_synthesis_file(flac, None)
    assert info.status == fb.RGS_BPS
    assert "bit-per-sample value must be between 4 and 24" in err, err


def test_the_last_vorbis_comment_block_decides():
    flac = add_vorbis_comment(tagged_flac(album_tags(-3.0, -6.0)), [b"REPLAYGAIN_TRACK_GAIN=-9.00 dB", b"REPLAYGAIN_TRACK_PEAK=0.5"])
    rc, _, err = tool_decode_many([flac], None, silent=False)
    info = fb.replaygain_synthesis_file(flac, None)
    assert rc == 0, err
    assert info.status == fb.RGS_APPLIED and info.album_used == 0 and info.gain == -9.0
    assert INFO.findall(err)[-1][1] == "-9.00", err


@pytest.mark.parametrize("entries", [
    [b"REPLAYGAIN_ALBUM_GAIN=-6.5\0", b"REPLAYGAIN_ALBUM_PEAK=0.5\0"],       # values with a trailing NUL: the raw length counts
    [b"REPLAYGAIN_ALBUM_GAIN=-6.5\0\0\0", b"REPLAYGAIN_ALBUM_PEAK=0.25"],
    [b"REPLAYGAIN_ALBUM_GAIN=-4.75", b"REPLAYGAIN_ALBUM_PEAK=0.5\0zz"],
])
def test_entries_are_read_at_their_raw_length(entries):
    flac = add_vorbis_comment(tagged_flac(["TITLE=x"]), entries)
    rc, _, err = tool_decode_many([flac], None, silent=False)
    info = fb.replaygain_synthesis_file(flac, None)
    assert rc == 0, err
    m = INFO.search(err)
    assert m and info.status == fb.RGS_APPLIED, err
    assert m.group(2) == f"{info.gain:0.2f}", (err, info.gain)
