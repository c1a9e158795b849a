"""The CUDA encoder against the oracle (oracle/flac_oracle.c, C fixed-order routine), frame for frame, at every input format
and on every stage-B kernel path:

  * every bit depth 4-24 x 1-8 channels at -0 / -5 / -8 (and -1 for stereo), signals rotating over music, full-scale noise,
    full-scale opposite-phase alternation, wasted bits (down to one significant bit) and one constant channel;
  * per kernel path -- k_search5 + k_emit3 (1-2 channels) / k_emit3<PAIR> + k_join (3-8 channels, k_search5 in CTAs of four
    signals above four), the general kernels, the tiled kernels -- bit depths on both sides of every 16-bit switch at 1-8
    channels, and -p / limit_min_bitrate at 5 and 7 channels;
  * every frame-header code class through each header writer: sample rates (table, kHz, Hz, tens of Hz, STREAMINFO's), coded
    and uncoded bits per sample, table / 8-bit / 16-bit blocksize codes and the UTF-8 frame-number widths;
  * whole files at 5 and 7 channels with tails of 1-31 samples.

Each cell meant for the fast kernels also checks, with the encoder's CUDA-event profile, that no k_scan / k_gather ran for its
full blocks (only the general and tiled emits use them), so a cell cannot silently test another path. The oracle itself is
pinned against the reference at these formats by test_oracle_formats.py."""
import numpy as np
import pytest

import oraclelib
from test_gpu_files import want_streaminfo
from test_oracle_formats import ALL_RATES, SIGNAL_KINDS, make_signal, short_tail

pytestmark = pytest.mark.gpu

# levels by their largest residual partition order (stream_encoder.c compression_levels_)
MAX_PO = {0: 3, 1: 3, 2: 3, 3: 4, 4: 4, 5: 5, 6: 6, 7: 6, 8: 6}
PATH_BPS = [4, 5, 8, 15, 16, 17, 23, 24]
PATH_CH = [1, 2, 3, 5, 6, 7, 8]


def fast_blocksize(bs, level, ch=2):
    """Whether build_geometry puts full blocks of bs on k_search5 + k_emit3: a power-of-two number of 32 x 32 or 32 x 36 tiles
    whose finest partitions are whole runs, and one emit thread per run of each channel (of each pair above two channels)."""
    for rt in (32, 36):
        if bs % (32 * rt) == 0:
            tiles = bs // (32 * rt)
            return tiles & (tiles - 1) == 0 and (bs >> MAX_PO[level]) % rt == 0 and bs // rt * min(ch, 2) <= 256
    return False


def oracle_frames(x, bps, rate, level, bs, first=0, **cfg):
    o = oraclelib.Encoder(oraclelib.preset(x.shape[1], bps, rate, level, bs, **cfg))
    if first == 0:
        return o.encode_stream(x)
    return [o.encode_frame(x[j:j + bs], first + j // bs) for j in range(0, x.shape[0], bs)]


def assert_same(got, want, what):
    assert len(got) == len(want), f"{what}: frame count {len(got)} != {len(want)}"
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    assert not bad, f"{what}: {len(bad)}/{len(want)} frames differ, first {bad[:5]}"


def check(x, bps, rate, level, bs, path, first=0, what="", **cfg):
    """Encode x (full blocks of bs and maybe a short last block) on a small encoder, compare with the oracle, then encode it
    again with the profile on: path "fast" means no k_scan / k_gather for the full blocks (the short last block always takes
    the general kernels, one launch set), "general" means the full blocks ran them too."""
    import flac_b200
    gcfg = {{"loose_mid_side": "loose_mid_side_stereo", "do_mid_side": "do_mid_side_stereo"}.get(k, k): v for k, v in cfg.items()}
    enc = flac_b200.Encoder(flac_b200.preset(x.shape[1], bps, rate, level, bs, **gcfg), max_blocks_per_launch=4)
    try:
        got = enc.encode_frames(x, first_frame_number=first)
        what = f"{what} {x.shape[1]}ch {bps}-bit {rate} Hz -{level} bs {bs} n {x.shape[0]} {cfg}"
        assert_same(got, oracle_frames(x, bps, rate, level, bs, first, **cfg), what)
        nfull, tail = divmod(x.shape[0], bs)
        if nfull:
            enc.set_profiling(True)
            again = enc.encode_frames(x, first_frame_number=first)
            prof = enc.profile()
            enc.set_profiling(False)
            assert again == got, f"{what}: frames change with the profile on"
            scans, gathers = prof["k_scan"][1], prof["k_gather"][1]
            assert prof["k_search"][1] > 0 and prof["k_emit"][1] > 0, f"{what}: no profile recorded {prof}"
            if path == "fast":
                assert scans == gathers == (1 if tail else 0), f"{what}: meant for the fast kernels, ran k_scan {scans} x"
            else:
                assert scans > (1 if tail else 0), f"{what}: meant for the general kernels, k_scan ran {scans} x"
    finally:
        enc.close()


# ---- every bit depth x every channel count

@pytest.mark.parametrize("bps", range(4, 25))
@pytest.mark.parametrize("level", [0, 5, 8])
def test_format_matrix(level, bps):
    rng = np.random.default_rng(level * 100 + bps)
    for ch in range(1, 9):
        kind = SIGNAL_KINDS[(ch + bps + level) % len(SIGNAL_KINDS)]
        x = make_signal(kind, 2 * 4096 + short_tail(rng, 4096), ch, bps, seed=ch * 7 + bps, bs=4096)
        check(x, bps, 44100, level, 4096, "fast", what=kind)


@pytest.mark.parametrize("bps", range(4, 25))
def test_format_matrix_loose_mid_side(bps):
    rng = np.random.default_rng(7000 + bps)
    kind = SIGNAL_KINDS[bps % len(SIGNAL_KINDS)]
    x = make_signal(kind, 2 * 4096 + short_tail(rng, 4096), 2, bps, seed=bps, bs=4096)
    check(x, bps, 44100, 1, 4096, "fast", what=kind)


# ---- kernel paths

def path_cells(seed):
    rng = np.random.default_rng(seed)
    for k, (bps, ch) in enumerate((b, c) for b in PATH_BPS for c in PATH_CH):
        yield k, bps, ch, SIGNAL_KINDS[k % len(SIGNAL_KINDS)], rng


@pytest.mark.parametrize("bs", [1024, 1152, 2304, 4096, 4608])
def test_fast_kernels(bs):
    """k_search5 + k_emit3 (1-2 channels) and k_search5 (sig_group above four signals) + k_emit3<PAIR> + k_join (3-8)."""
    levels = [lv for lv in range(9) if fast_blocksize(bs, lv)]
    assert levels
    for k, bps, ch, kind, rng in path_cells(bs):
        level = levels[k % len(levels)]
        x = make_signal(kind, 2 * bs + short_tail(rng, bs), ch, bps, seed=k + bs, bs=bs)
        check(x, bps, 44100, level, bs, "fast", what=kind)


@pytest.mark.parametrize("bs", [16, 17, 576, 1000])
def test_general_kernels(bs):
    for k, bps, ch, kind, rng in path_cells(bs):
        level = k % 9
        x = make_signal(kind, 2 * bs + short_tail(rng, bs), ch, bps, seed=k + bs, bs=bs)
        check(x, bps, 44100, level, bs, "general", what=kind)


@pytest.mark.parametrize("env,value", [("FB200_DEBUG_PATH", "7"), ("FB200_DEBUG_PATH", "22")], ids=["debug_path_7", "tiled"])
def test_forced_paths_on_regular_blocksizes(monkeypatch, env, value):
    """The general kernels (FB200_DEBUG_PATH=7) and the tiled kernels (FB200_DEBUG_PATH=22) on blocksizes the fast
    kernels would take."""
    monkeypatch.setenv(env, value)
    for k, bps, ch, kind, rng in path_cells(len(value)):
        bs = (4096, 1152, 4608, 2304)[k % 4]
        x = make_signal(kind, 2 * bs + short_tail(rng, bs), ch, bps, seed=k, bs=bs)
        check(x, bps, 44100, (0, 2, 5, 8, 1, 3, 4, 6, 7)[k % 9], bs, "general", what=kind)


def constant_blocks(bs, ch, bps, seed):
    x = make_signal("music", bs * 5 + 13, ch, bps, seed=seed, bs=bs)
    x[bs:2 * bs] = 0                                  # every channel constant
    x[2 * bs:3 * bs] = 5 - (1 << (bps - 1))           # DC
    x[3 * bs:4 * bs, ch - 1] = 1                      # the last channel constant (limit_min_bitrate's second pass)
    x[4 * bs:5 * bs, 0] = -1                          # the first channel constant
    return x


PATHS = [("fast", 4096, None), ("fast", 1152, None), ("general", 1000, None), ("general", 4096, ("FB200_DEBUG_PATH", "7")),
         ("general", 4608, ("FB200_DEBUG_PATH", "22"))]


@pytest.mark.parametrize("path,bs,env", PATHS, ids=[f"{p}-{b}-{e[0] if e else 'default'}" for p, b, e in PATHS])
@pytest.mark.parametrize("ch", [5, 7])
def test_min_bitrate_and_precision_search_at_odd_channel_counts(monkeypatch, path, bs, env, ch):
    """limit_min_bitrate re-searches the last channel, which above four signals sits in k_search5's partial last CTA."""
    if env:
        monkeypatch.setenv(*env)
    for bps in (4, 8, 17, 24):
        x = constant_blocks(bs, ch, bps, seed=bps + ch)
        for cfg in (dict(limit_min_bitrate=1), dict(do_qlp_coeff_prec_search=1), dict(limit_min_bitrate=1, do_qlp_coeff_prec_search=1)):
            for level in ((2, 5) if bs == 1152 else (5, 8)):
                check(x, bps, 44100, level, bs, path, **cfg)


# ---- frame-header codes through each writer

# (writer, channels, full-block blocksizes, expected path, environment): emit3_frame_header serves k_emit3 (1-2 channels) and
# k_join (3-8); put_frame_header serves the general and the tiled emit. Every fast-path blocksize has a table code (8192 takes
# k_emit3 for mono only), so the 8- and 16-bit blocksize codes reach the frame header through put_frame_header alone.
WRITERS = {
    "emit3": ([1, 2], [4096, 1152, 2304, 4608, 1024, 2048], "fast", None),
    "emit3_mono_8192": ([1], [8192], "fast", None),
    "join": ([3, 5, 6, 7, 8], [4096, 1152, 2304, 4608], "fast", None),
    "general": ([1, 2, 5, 8], [1000, 16, 255, 257, 192, 576, 512], "general", None),
    "tiled": ([1, 2, 6, 7], [4096, 1000, 256, 17], "general", ("FB200_DEBUG_PATH", "22")),
}
CODED_OR_NOT = [8, 12, 16, 20, 24, 4, 7, 13, 17, 23]


def writer_level(k, bs, ch, path):
    level = (5, 0, 8, 2)[k % 4]
    return level if path != "fast" or fast_blocksize(bs, level, ch) else 0


@pytest.mark.parametrize("writer", sorted(WRITERS))
def test_header_codes(monkeypatch, writer):
    chs, bss, path, env = WRITERS[writer]
    if env:
        monkeypatch.setenv(*env)
    rng = np.random.default_rng(len(writer))
    for k, (cls, rate) in enumerate(ALL_RATES):
        ch, bs, bps = chs[k % len(chs)], bss[k % len(bss)], CODED_OR_NOT[k % len(CODED_OR_NOT)]
        level = writer_level(k, bs, ch, path)
        x = make_signal("music", 2 * bs + short_tail(rng, bs), ch, bps, seed=k, bs=bs)
        check(x, bps, rate, level, bs, path, what=f"{writer} {cls}")


# UTF-8 coded frame numbers: 1 to 6 bytes, each width's last value and the next
FIRST_FRAMES = [126, 2046, 65534, 0x1FFFFE, 0x3FFFFFE, 0x7FFFFFFD]


@pytest.mark.parametrize("writer", sorted(WRITERS))
def test_frame_number_widths(monkeypatch, writer):
    chs, bss, path, env = WRITERS[writer]
    if env:
        monkeypatch.setenv(*env)
    rng = np.random.default_rng(99)
    for k, first in enumerate(FIRST_FRAMES):
        ch, bs, bps = chs[k % len(chs)], bss[k % len(bss)], CODED_OR_NOT[k % len(CODED_OR_NOT)]
        level = writer_level(k, bs, ch, path)
        x = make_signal("music", 2 * bs + short_tail(rng, bs), ch, bps, seed=k, bs=bs)
        check(x, bps, 48000, level, bs, path, first=first, what=f"{writer} first frame {first}")


# ---- whole files: tails of every small length at odd channel counts

@pytest.mark.parametrize("bps,level", [(4, 5), (13, 8), (23, 0)])
@pytest.mark.parametrize("ch", [5, 7])
def test_files_with_short_tails(ch, bps, level):
    import flac_b200
    bs, rate = 4096, 48000
    tails = [1, 2, 3, 4, 5, 15, 16, 17, 31]
    lengths = [bs * (1 + k % 3) + t for k, t in enumerate(tails)] + tails[:4]
    parts = [make_signal(SIGNAL_KINDS[k % len(SIGNAL_KINDS)], n, ch, bps, rate, seed=k, bs=bs) for k, n in enumerate(lengths)]
    x = np.concatenate(parts)
    enc = flac_b200.Encoder(flac_b200.preset(ch, bps, rate, level, bs), max_blocks_per_launch=4)
    try:
        res = enc.encode_files(x, lengths, bytes_per_sample=2 if bps <= 16 else 3)
    finally:
        enc.close()
    for f, (xf, (si, frames)) in enumerate(zip(parts, res)):
        assert_same(frames, oracle_frames(xf, bps, rate, level, bs), f"file {f} ({xf.shape[0]} samples)")
        assert si == want_streaminfo(xf, frames, bs, bps, rate), f"file {f}: STREAMINFO"
