"""flac -5 --skip --until on one GPU: 200 stereo 16-bit 44.1 kHz files of 60 s (seeded signals), each cut into 10 clips of 5 s
(2 000 .flac outputs, MD5 on), in one call per arm:

  pcm_ranges   Encoder.encode_pcm_files(ranges=...)'s C call (fb200_encode_pcm_files_ranges_host) over the WAV files
  flac_ranges  Encoder.reencode_flac_ranges's C call (fb200_reencode_flac_files_ranges_host) over the same files as .flac (written
               at -5 beforehand), indexed once outside the timed calls
  flac_ref     the reference flac tool, one process per clip, 16 at a time, on WAV input (when oracle/_ref/flac_ref is present;
               timed on --ref-clips clips and scaled to the batch)

Rates are clip samples (per channel x channels) over the call's wall time, host copies included. The card's name and power limit
are read in the same run. Prints one JSON line.

    python tools/bench_encode_ranges.py [--files 200] [--seconds 60] [--clips 10] [--clip-seconds 5] [--level 5] [--reps 5]
                                        [--procs 16] [--ref-clips 160]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import flac_b200 as fb  # noqa: E402
import refcli  # noqa: E402
from bench_pcm_files import make_files  # noqa: E402

RATE = 44100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=200)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--clips", type=int, default=10)
    ap.add_argument("--clip-seconds", type=int, default=5)
    ap.add_argument("--level", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--procs", type=int, default=16)
    ap.add_argument("--ref-clips", type=int, default=160)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    wavs = make_files(a.files, a.seconds, RATE)
    clip = a.clip_seconds * RATE
    step = (a.seconds * RATE - clip - 7) // max(a.clips - 1, 1)
    ranges = [(f, c * step + (f % 7), clip) for f in range(a.files) for c in range(a.clips)]  # off frame boundaries
    enc = fb.Encoder(fb.preset(2, 16, RATE, a.level))
    flacs = enc.encode_pcm_files(wavs)
    dec = fb.Decoder(2, 16, RATE, 4096)
    dec.index_files(flacs)
    data, offsets = fb._batch(wavs)
    pinfo = fb.probe_pcm_files(None, data, offsets)
    pout = np.empty(enc.pcm_files_capacity(pinfo, ranges=ranges), dtype=np.uint8)
    fout = np.empty(enc.reencode_ranges_capacity(dec, ranges), dtype=np.uint8)

    def pcm_ranges():
        return enc._pcm_call(True, data.ctypes.data, offsets, pinfo, None, 10, -1, True, pout.ctypes.data, pout.size, None, ranges=ranges)

    def flac_ranges():
        return enc._reencode_call(True, dec, None, None, -1, -1, False, fout.ctypes.data, fout.size, None, ranges=ranges)

    _, pfiles = pcm_ranges()
    _, finfo = flac_ranges()
    assert all(i.status == fb.REENCODE_OK for i in finfo)
    # the two arms encode the same samples: the same frames after each file's metadata
    for k in (0, len(ranges) // 2, len(ranges) - 1):
        p, r = pfiles[k], finfo[k].file
        assert pout[p.offset + p.audio_offset:p.offset + p.bytes].tobytes() == fout[r.offset + r.audio_offset:r.offset + r.bytes].tobytes()
    clip_samples = len(ranges) * clip * 2
    res = {"gpu": gpu, "files": a.files, "seconds": a.seconds, "clips": len(ranges), "clip_seconds": a.clip_seconds, "level": a.level,
           "clip_samples": clip_samples}
    for name, fn in (("pcm_ranges", pcm_ranges), ("flac_ranges", flac_ranges)):
        fn()
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        med = float(np.median(ts))
        res[name + "_ms"] = round(1e3 * med, 2)
        res[name + "_ms_min"] = round(1e3 * min(ts), 2)
        res[name + "_gsamples_s"] = round(clip_samples / med / 1e9, 3)
    enc.close()
    dec.close()
    if refcli.available():
        with tempfile.TemporaryDirectory() as d:
            paths = []
            for f in range(a.files):
                p = os.path.join(d, f"f{f}.wav")
                with open(p, "wb") as fh:
                    fh.write(wavs[f])
                paths.append(p)
            jobs = ranges[::max(len(ranges) // a.ref_clips, 1)][:a.ref_clips]

            def one(k):
                f, s, n = jobs[k]
                return subprocess.run([refcli.PATH, "-f", "-s", f"-{a.level}", f"--skip={s}", f"--until={s + n}", paths[f], "-o",
                                       os.path.join(d, f"c{k}.flac")], stderr=subprocess.DEVNULL).returncode

            t0 = time.perf_counter()
            with ThreadPoolExecutor(a.procs) as pool:
                rcs = list(pool.map(one, range(len(jobs))))
            assert not any(rcs)
            ms = 1e3 * (time.perf_counter() - t0) * len(ranges) / len(jobs)
            res["flac_ref_%dproc_ms" % a.procs] = round(ms, 1)
            res["flac_ref_%dproc_gsamples_s" % a.procs] = round(clip_samples / (ms / 1e3) / 1e9, 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
