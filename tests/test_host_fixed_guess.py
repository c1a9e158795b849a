"""flac_b200.host_x86_avx2_fixed_guess() says which fixed-order guess libFLAC takes on this host: the reference, dispatched as
this host dispatches it, writes other frames than with its AVX2 routine disabled exactly when the function returns 1. Needs
libflac_b200.so to load, not a GPU."""
import pytest

import flac_b200 as fb
import reflib
import signals


def test_host_detection_agrees_with_the_reference_dispatch():
    if not reflib.available("strict"):
        pytest.skip("oracle/_ref not built")
    # a stream whose short last block the two routines guess differently (DESIGN.md, G4)
    x = signals.music_like(1152 * 3 + 19, 2, 24, 44100, seed=1)
    _, _, host = reflib.encode(x, 24, rate=44100, level=2, variant="strict", opts=reflib.RefEncOpts(streamable_subset=0))
    _, _, c_path = reflib.encode(x, 24, rate=44100, level=2, variant="strict", opts=reflib.RefEncOpts(streamable_subset=0, disable_isa=16))
    assert fb.host_x86_avx2_fixed_guess() == int(host != c_path)
