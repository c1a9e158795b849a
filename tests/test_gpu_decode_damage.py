"""Every decode path on damaged .flac files (tests/damage.py) against the reference libFLAC's decoder and the reference
flac tool: fb200_decode_files_* (whole call, and max_frames_per_launch = 8; 2-, 3- and 4-byte output; device output),
fb200_decode_files_ranges_*, fb200_decode_pcm_files_* (tool_ok and bytes) and the drop-in FLAC__stream_decoder_* shell.

What the engine promises from libFLAC's trace of a file (damage.placed): every frame libFLAC wrote at its sample number,
zeros elsewhere, cut at STREAMINFO's total_samples. A mismatch is allowed only where a row of DIVERGENCES names it; each row
is one predicate over the corpus entry and the trace, with the reason and the stream_decoder.c lines it departs from, and
the same sentence is in include/flac_b200.h and DESIGN.md."""
import numpy as np
import pytest

import damage
import reflib
import refcli
import refmetaflac

pytestmark = pytest.mark.gpu


def _format_differs(e, tr):
    return any(w.pcm.shape[1] != e.base.ch or w.bps != e.base.bps for w in tr.writes)


def _over_max_blocksize(e, tr):
    return bool(e.base.bs) and any(w.blocksize > e.base.bs for w in tr.writes)


def _overlapping(e, tr):
    ends = [(w.sample, w.sample + w.blocksize) for w in tr.writes]
    return any(b[0] < a[1] for a, b in zip(ends, ends[1:]))


def _backwards(e, tr):
    return any(b.sample < a.sample for a, b in zip(tr.writes, tr.writes[1:]))


def _hole(e, tr):
    _, covered = damage.placed(tr, len(e.base.pcm), e.base.ch)
    return not covered.all()


# classes whose damage removes frame headers (so the index has no candidate there) without leaving one that fails
HEADER_LOST = {"flip_sync", "flip_reserved", "flip_bs_code", "flip_rate_code", "flip_ch_code", "flip_bps_code", "flip_number",
               "flip_crc8", "reserved_sync_valid_crc", "reserved_bps_valid_crc"} | {f"lost_run{r}" for r in damage.LOST_RUNS} | {"lost_run_5s"}
JUNK = {"junk_between", "id3v1_tail", "ape_tail"}

# The checks a row may waive: "files" (decode_files output, samples_missing, md5_state), "files_errors" (decode_files `errors`),
# "ranges", "tool" (tool_ok and the bytes against flac -d), "dropin" (the drop-in decoder's writes), "dropin_errors" (where its
# errors fall between writes), "replaygain" (add-ReplayGain DECODE against metaflac).
# name: (predicate over the corpus entry and libFLAC's trace, the checks it waives, reason, stream_decoder.c lines departed from)
DIVERGENCES = {
    "header_disagrees": (lambda e, tr: e.cls in ("mismatch_channels", "mismatch_bps", "blocksize_over_max")
                         and (_format_differs(e, tr) or _over_max_blocksize(e, tr)), {"files", "dropin", "dropin_errors", "replaygain"},
                         "a frame whose channels, bits per sample or blocksize disagree with STREAMINFO is not indexed, so its "
                         "samples are lost; libFLAC decodes and writes it", "2624-2947"),
    "overlap": (lambda e, tr: e.cls in ("repeat", "swap", "move_to_end") and _overlapping(e, tr), {"files", "replaygain"},
                "a frame that starts before the end of the frame placed before it (a repeated or reordered frame) is not "
                "placed, its samples are zeros unless another frame covers them, and it counts as an error; libFLAC writes "
                "every frame in stream order", "2483-2554"),
    "range_sees_its_frames": (lambda e, tr: e.cls in ("swap", "move_to_end") and _backwards(e, tr), {"ranges"},
                              "a range walks only the frames that meet it: a frame the whole-file decode drops because an "
                              "earlier frame in the file ends past its first sample is placed by a range that does not "
                              "meet that earlier frame", "2483-2554"),
    "lost_without_candidate": (lambda e, tr: e.cls in HEADER_LOST and _hole(e, tr), {"files_errors"},
                               "`errors` counts damaged stretches the index found a candidate in; a frame lost with its header "
                               "(a damaged header, or frames cut out) shows only in samples_missing, where libFLAC reports "
                               "lost sync, a bad header or a missing frame", "2483-2498"),
    "trailing_junk": (lambda e, tr: e.cls in ("id3v1_tail", "ape_tail"), {"dropin_errors"},
                      "the drop-in decoder reports nothing for bytes after the last frame (an ID3v1 or APE tag); libFLAC "
                      "reports them as lost sync", "2321-2371"),
    "junk": (lambda e, tr: e.cls in JUNK, {"files_errors", "tool"},
             "junk that carries no frame header (and ID3v1 / APE tags) is never seen by the index; libFLAC reports it as "
             "lost sync", "2321-2371"),
}


def waived(e, tr, check):
    return [n for n, (pred, checks, _, _) in DIVERGENCES.items() if check in checks and pred(e, tr)]


@pytest.fixture(scope="module")
def world():
    if not reflib.available("default"):
        pytest.skip("oracle/_ref not present")
    entries = damage.corpus()
    L = damage.ref_lib()
    return entries, [damage.trace(L, e.data) for e in entries]


def decoder(max_frames=0):
    import flac_b200
    return flac_b200.Decoder(2, 16, 44100, 4096, max_frames_per_launch=max_frames)


def _pack(x, nbytes):
    return x.astype("<i4").view(np.uint8).reshape(x.shape[0], x.shape[1], 4)[:, :, :nbytes].reshape(x.shape[0], -1)


def _check_files(entries, traces, res, nbytes, failures, tag):
    for e, tr, (y, info) in zip(entries, traces, res):
        assert info.status == 0, f"{e.name}: status {info.status}"
        want, covered = damage.placed(tr, int(info.samples), e.base.ch)
        if not waived(e, tr, "files"):
            if not np.array_equal(y, want if nbytes == 4 else _pack(want, nbytes)):
                failures.append(f"{tag} {e.name}: output differs from libFLAC's frames placed by sample number")
            if int(info.samples_missing) != int((~covered).sum()):
                failures.append(f"{tag} {e.name}: samples_missing {info.samples_missing}, libFLAC left {(~covered).sum()} uncovered")
            md5_want = 1 if np.array_equal(want, e.base.pcm[:int(info.samples)]) else 2
            if info.md5_state != md5_want:
                failures.append(f"{tag} {e.name}: md5_state {info.md5_state}, want {md5_want}")
        if (info.errors > 0) != bool(tr.errors) and not waived(e, tr, "files_errors") and not waived(e, tr, "files"):
            failures.append(f"{tag} {e.name}: errors {info.errors}, libFLAC reported {tr.errors}")


@pytest.mark.parametrize("max_frames,nbytes", [(0, 4), (8, 4), (0, 2), (0, 3)])
def test_decode_files_follow_libflac(world, max_frames, nbytes):
    entries, traces = world
    wide = [(e, t) for e, t in zip(entries, traces) if nbytes == 4 or e.base.bps <= 8 * nbytes]
    es, ts = [e for e, _ in wide], [t for _, t in wide]
    dec = decoder(max_frames)
    res = dec.decode_files([e.data for e in es], bytes_per_sample=nbytes)
    dec.close()
    failures = []
    _check_files(es, ts, res, nbytes, failures, f"[{max_frames},{nbytes}]")
    assert not failures, "\n".join(failures)


def test_decode_files_device_matches_host(world):
    import torch
    entries, _ = world
    blobs = [e.data for e in entries]
    dec = decoder()
    host = dec.decode_files(blobs)
    infos, total = dec.index_files(blobs)
    out = torch.zeros(total, dtype=torch.int32, device="cuda:0")
    dinfos = dec.decode_files_device(out.data_ptr(), total)
    dec.close()
    got = out.cpu().numpy()
    for e, (y, hi), di in zip(entries, host, dinfos):
        a, n = int(di.first_value), int(di.samples) * max(int(di.channels), 1)
        assert np.array_equal(got[a:a + n], y.reshape(-1)), e.name
        assert (di.errors, di.samples_missing, di.md5_state) == (hi.errors, hi.samples_missing, hi.md5_state), e.name


def test_ranges_are_slices_of_the_whole_decode(world):
    entries, traces = world
    blobs = [e.data for e in entries]
    dec = decoder()
    whole = dec.decode_files(blobs)
    rng = np.random.default_rng(7)
    ranges = []
    for f, (y, info) in enumerate(whole):
        n = int(info.samples)
        for _ in range(3):
            a = int(rng.integers(0, n))
            ranges.append((f, a, int(rng.integers(1, n - a + 1))))
    res = dec.decode_ranges(ranges)
    dec.close()
    for (f, a, m), (y, info) in zip(ranges, res):
        if waived(entries[f], traces[f], "ranges"):
            continue
        assert np.array_equal(y, whole[f][0][a:a + m]), f"{entries[f].name} [{a}, {a + m})"


def test_tool_ok_follows_flac_d(world):
    if not refcli.available():
        pytest.skip("oracle/_ref/flac_ref not present")
    entries, traces = world
    tool = damage.tool_decode([e.data for e in entries])
    dec = decoder()
    dec.index_files([e.data for e in entries])
    res = dec.decode_pcm_files("wave")
    dec.close()
    failures = []
    for e, tr, (rc, t), (blob, info) in zip(entries, traces, tool, res):
        if waived(e, tr, "tool"):
            continue
        if info.tool_ok != (rc == 0):
            failures.append(f"{e.name}: tool_ok {info.tool_ok}, flac -d exited {rc}")
        elif rc == 0 and blob != t:
            failures.append(f"{e.name}: bytes differ from flac -d")
    assert not failures, "\n".join(failures)


def test_scan_candidates_equal_the_header_rules(world):
    """fb200_decoder_index_host's candidates are exactly damage.scan's: every corpus file, and each cut so that its last
    candidate's header (with CRC-8) ends at the last byte of the buffer, one byte short of it, and after 5 bytes."""
    entries, _ = world
    dec = decoder()
    failures = []
    for e in entries:
        bufs = [e.data]
        last = damage.scan(e.data)[-1]
        hl = damage.header_len(e.data[last:])
        bufs += [e.data[:last + hl + 1], e.data[:last + hl], e.data[:last + 5]]
        for j, b in enumerate(bufs):
            got = dec.index(np.frombuffer(b, dtype=np.uint8)).tolist()
            want = damage.scan(b)
            if got != want:
                failures.append(f"{e.name} buffer {j}: {len(got)} candidates, want {len(want)}: "
                                f"extra {sorted(set(got) - set(want))[:4]} missing {sorted(set(want) - set(got))[:4]}")
    dec.close()
    assert not failures, "\n".join(failures)


def _metaflac_fails(blobs):
    """metaflac --add-replay-gain on each file alone: whether it fails during analysis (decoding the file)."""
    import os
    import subprocess
    import tempfile
    res = []
    with tempfile.TemporaryDirectory() as d:
        for i, b in enumerate(blobs):
            p = os.path.join(d, f"f{i}.flac")
            with open(p, "wb") as fh:
                fh.write(bytes(b))
            r = subprocess.run([refmetaflac.PATH, "--add-replay-gain", p], capture_output=True, text=True, timeout=120)
            res.append(r.returncode != 0 and "during analysis" in r.stderr)
    return res


def test_verdicts_follow_decode_files(world):
    """The re-encode's DAMAGED status is set for exactly the files decode_files marks damaged (an error or a sample missing);
    the add-ReplayGain DECODE status for exactly the files metaflac --add-replay-gain fails while decoding."""
    import flac_b200
    if not refmetaflac.available():
        pytest.skip("oracle/_ref/metaflac_ref not present")
    entries, traces = world
    failures = []
    by_fmt = {}
    for i, e in enumerate(entries):
        by_fmt.setdefault((e.base.ch, e.base.bps, e.base.rate), []).append(i)
    for (ch, bps, rate), idx in by_fmt.items():
        blobs = [entries[i].data for i in idx]
        dec = decoder()
        files = dec.decode_files(blobs)
        damaged = [info.errors > 0 or info.samples_missing > 0 for _, info in files]
        enc = flac_b200.Encoder(flac_b200.preset(ch, bps, rate, 5))
        _, rinfo = enc.reencode_flac_files(dec, list(range(len(idx))), infos=True)
        enc.close()
        _, ainfo = dec.add_replay_gain(list(range(len(idx))), albums=list(range(len(idx))), scan=True)
        dec.close()
        tool = _metaflac_fails(blobs)
        for i, d, r, a, t in zip(idx, damaged, rinfo, ainfo, tool):
            e = entries[i]
            if (r.status == flac_b200.REENCODE_DAMAGED) != d:
                failures.append(f"{e.name}: re-encode status {r.status}, decode_files damaged {d}")
            if a.status in (flac_b200.ADD_RG_OK, flac_b200.ADD_RG_DECODE) and (a.status == flac_b200.ADD_RG_DECODE) != t \
                    and not waived(e, traces[i], "replaygain"):
                failures.append(f"{e.name}: add-ReplayGain status {a.status}, metaflac {'fails' if t else 'passes'} the decode")
    assert not failures, "\n".join(failures)


def test_dropin_decoder_writes_what_libflac_writes(world):
    import flac_b200
    entries, traces = world
    ours = damage.api(flac_b200.lib())
    failures = []
    for e, tr in zip(entries, traces):
        if waived(e, tr, "dropin"):
            continue
        got = damage.trace(ours, e.data)
        a = [(w.sample, w.blocksize) for w in got.writes]
        b = [(w.sample, w.blocksize) for w in tr.writes]
        if a != b:
            failures.append(f"{e.name}: writes (sample, blocksize) {a[:3]}..{len(a)} vs libFLAC {b[:3]}..{len(b)}")
            continue
        if not all(np.array_equal(x.pcm, y.pcm) for x, y in zip(got.writes, tr.writes)):
            failures.append(f"{e.name}: written samples differ")
        if got.error_marks() != tr.error_marks() and not waived(e, tr, "dropin_errors"):
            failures.append(f"{e.name}: errors after writes {got.error_marks()} ({got.errors}), libFLAC {tr.error_marks()} ({tr.errors})")
    assert not failures, "\n".join(failures)
