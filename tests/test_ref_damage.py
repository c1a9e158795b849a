"""The damaged-file corpus (tests/damage.py) reaches the reference decoder behaviour each mutation class is named for, so the
GPU comparisons in test_gpu_decode_damage.py cannot quietly stop testing anything. CPU only: libFLAC through ctypes."""
import numpy as np
import pytest

import damage
import reflib


@pytest.fixture(scope="module")
def traced():
    if not reflib.available("default"):
        pytest.skip("oracle/_ref not present")
    L = damage.ref_lib()
    return [(e, damage.trace(L, e.data)) for e in damage.corpus()]


def _silence(tr):
    ws = tr.writes
    return sum(w.blocksize for p, w in zip([None] + ws, ws) if damage.is_silence(p, w))


def test_corpus_size_and_classes():
    if not reflib.available("default"):
        pytest.skip("oracle/_ref not present")
    c = damage.corpus()
    assert 200 <= len(c) <= 400
    classes = {e.cls for e in c}
    for cls in damage.FLIP_CLASSES + ("insert_byte", "delete_byte", "trunc_header", "trunc_subframe", "trunc_footer", "trunc_between",
                                      "lost_first", "lost_last", "lost_run_5s", "repeat", "swap", "move_to_end", "lookalike_junk",
                                      "embedded_frame", "lookalike_verbatim", "lookalike_verbatim32", "frame_in_verbatim",
                                      "mismatch_channels", "mismatch_bps", "mismatch_rate", "blocksize_over_max", "out_of_bounds",
                                      "junk_between", "id3v1_tail", "ape_tail", "two_stretches", "chunk_boundary",
                                      "reserved_sync_valid_crc", "reserved_bps_valid_crc"):
        assert cls in classes, cls
    for run in damage.LOST_RUNS:
        assert f"lost_run{run}" in classes
    assert {e.base.ch for e in c} >= {1, 2, 6} and {e.base.bps for e in c} >= {8, 16, 24}
    assert {e.base.bs for e in c} >= {16, 192, 1152, 4096, 0}


def test_each_class_reaches_its_libflac_behaviour(traced):
    for e, tr in traced:
        n, bs, ch = len(e.base.pcm), e.base.bs, e.base.ch
        got = sum(w.blocksize for w in tr.writes)
        if e.cls in ("clean", "lookalike_verbatim", "lookalike_verbatim32", "frame_in_verbatim"):
            # libFLAC never looks inside a frame it decoded: the look-alikes cost nothing
            assert tr.errors == [] and tr.md5_ok and np.array_equal(damage.sequential(tr), e.base.pcm), e.name
        elif e.cls.startswith("flip_") or e.cls in ("insert_byte", "delete_byte", "two_stretches", "chunk_boundary"):
            # a damaged frame: an error, then silence for it, so the output keeps its length
            assert tr.errors and got == n and _silence(tr) >= (bs or 1) * (2 if e.cls in ("two_stretches", "chunk_boundary") else 1), e.name
        elif e.cls == "reserved_sync_valid_crc":
            # libFLAC never syncs on 0xFFFA / 0xFFFB: the frame is lost sync, then silence
            assert tr.errors[0] == damage.LOST_SYNC and damage.UNPARSEABLE_STREAM not in tr.errors and got == n \
                and _silence(tr) == (e.base.starts[e.where[0] + 1] - e.base.starts[e.where[0]]), e.name
        elif e.cls == "reserved_bps_valid_crc":
            # the header is read and refused as unparseable, then silence
            assert tr.errors[0] == damage.UNPARSEABLE_STREAM and got == n and _silence(tr) > 0, e.name
        elif e.cls in ("lost_run1", "lost_run49", "lost_run50"):
            assert tr.errors == [damage.MISSING_FRAME] and got == n and damage.ascending(tr), e.name
        elif e.cls in ("lost_run51", "lost_run60"):
            # silence stops at 50 of the previous frame's blocks: the output is short and later frames move earlier
            run = int(e.cls[8:])
            assert _silence(tr) == 50 * bs and got == n - (run - 50) * bs and not damage.ascending(tr), e.name
        elif e.cls == "lost_run_5s":
            # ... or at 5 seconds, whichever binds first
            assert 5 * e.base.rate < 50 * bs and _silence(tr) == 5 * e.base.rate and got < n, e.name
        elif e.cls in ("lost_first", "lost_last", "trunc_header", "trunc_between"):
            # no silence before the first frame or after the last: a shorter stream, and no error
            assert tr.errors == [] and got < n and _silence(tr) == 0, e.name
        elif e.cls in ("trunc_subframe", "trunc_footer"):
            assert tr.errors and got < n, e.name
        elif e.cls == "repeat":
            # the repeated frame is written twice, without an error
            s = [w.sample for w in tr.writes]
            assert tr.errors == [] and len(s) != len(set(s)), e.name
        elif e.cls in ("swap", "move_to_end"):
            assert damage.MISSING_FRAME in tr.errors and got > n, e.name
        elif e.cls in ("lookalike_junk", "embedded_frame"):
            # the look-alike fails; the rewind to just after it finds the real frame: nothing is lost
            assert tr.errors and tr.md5_ok and np.array_equal(damage.sequential(tr), e.base.pcm), e.name
        elif e.cls in ("junk_between", "id3v1_tail", "ape_tail"):
            assert tr.errors == [damage.LOST_SYNC] and tr.md5_ok, e.name
        elif e.cls == "mismatch_channels":
            assert tr.errors == [] and any(w.pcm.shape[1] != ch for w in tr.writes), e.name
        elif e.cls == "mismatch_bps":
            assert tr.errors == [] and any(w.bps != e.base.bps for w in tr.writes), e.name
        elif e.cls == "mismatch_rate":
            assert tr.errors == [] and any(w.rate != e.base.rate for w in tr.writes), e.name
        elif e.cls == "blocksize_over_max":
            assert tr.errors == [] and any(w.blocksize > bs for w in tr.writes), e.name
        elif e.cls == "out_of_bounds":
            assert damage.OUT_OF_BOUNDS in tr.errors and _silence(tr) == bs, e.name
        else:
            raise AssertionError(f"{e.name}: no expectation for class {e.cls}")
