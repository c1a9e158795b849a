"""flac -d --apply-replaygain-which-is-not-lossless on one GPU: 200 stereo 16-bit 44.1 kHz files of 60 s, made at -5 from seeded
signals (fb200_encode_pcm_files_host) and tagged as one album by fb200_add_replaygain_flac_files_host, decoded to WAVE by one call of

  rg_default  fb200_decode_pcm_files_replaygain_host, the option without '=' (album gain, hard limiter, low shaping), per_file 0,
              MD5 on
  rg_0aL      the same with =0aL (no dither: every value on its own)
  rg_12aLn1   the same with =12aLn1 (+12 dB preamp: the hard limiter, and so fb_tanh, runs on every value past half scale)
  plain       fb200_decode_pcm_files_host (flac -d)

The three arms alternate, --reps rounds after a warm-up; each is a host clock around the synchronous call (median and min).
k_rg_synth's device time comes from separate torch.profiler runs of one rg_default and one rg_12aLn1 call, with the share of
values each sends through the limiter (|x| x scale > half scale, over the decoded samples). The reference arms run the flac tool
(oracle/_ref/flac_ref) on copies: one process over all files (the only run that gives the per_file 0 bytes; compared), and --procs
processes of one file each over --ref-files files (compared with per_file 1; the time of those files, multiplied by
files / ref-files: scaled, not a run over the batch). The card's name and power
limit are read in the same run. Prints one JSON line.

    python tools/bench_decode_replaygain.py [--files 200] [--seconds 60] [--reps 5] [--procs 16] [--ref-files 16]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=200)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--procs", type=int, default=16)
    ap.add_argument("--ref-files", type=int, default=16)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    e5 = fb.Encoder(fb.preset(2, 16, 44100, 5))
    flacs = e5.encode_pcm_files(make_files(a.files, a.seconds))
    e5.close()
    dec = fb.Decoder(2, 16, 44100, 4096)
    dec.index_files(flacs)
    tagged, info = dec.add_replay_gain(list(range(a.files)), albums=[0] * a.files)
    assert all(i.status == fb.ADD_RG_OK for i in info)
    dec.index_files(tagged)
    res = {"gpu": gpu, "files": a.files, "seconds": a.seconds, "samples": a.files * a.seconds * 44100 * 2}
    arms = {"rg_default": lambda: dec.decode_pcm_files_replaygain(), "rg_0aL": lambda: dec.decode_pcm_files_replaygain(spec="0aL"),
            "rg_12aLn1": lambda: dec.decode_pcm_files_replaygain(spec="12aLn1"), "plain": lambda: dec.decode_pcm_files()}
    outs = {k: f() for k, f in arms.items()}
    assert all(r.status == fb.RGS_APPLIED for _, _, r in outs["rg_default"])
    times = {k: [] for k in arms}
    for _ in range(a.reps):
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)
    for k, ts in times.items():
        res[k + "_ms"], res[k + "_ms_min"] = round(1e3 * float(np.median(ts)), 2), round(1e3 * min(ts), 2)
    from torch.profiler import ProfilerActivity, profile
    def limited_share(rg):  # values the hard limiter takes: |x| / 2^15 x scale > 0.5
        over = total = 0
        for (b, i), (_, _, r) in zip(outs["plain"], rg):
            x = np.abs(np.frombuffer(b, dtype="<i2", count=2 * int(i.samples), offset=int(i.header_bytes)).astype(np.int32))
            over += int(np.count_nonzero(x * r.scale > 16384.0))
            total += x.size
        return round(over / total, 4)

    steps = a.seconds * 44100
    for name, spec in (("rg_default", None), ("rg_12aLn1", "12aLn1")):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rg = dec.decode_pcm_files_replaygain(spec=spec)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.count:
                kern[ev.key[:60]] = round(ev.device_time_total / 1e3, 3)
        res[name + "_profile_kernels_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:6])
        synth = sum(v for k, v in kern.items() if "k_rg_synth<" in k)
        res[name + "_k_rg_synth_ns_per_step"] = round(1e6 * synth / steps, 1)  # one chain per warp, all chains at once: a chain's steps
        res[name + "_limited_share"] = limited_share(rg)
    per_file = dec.decode_pcm_files_replaygain(per_file=True)
    dec.close()
    if refcli.available():
        with tempfile.TemporaryDirectory() as d:
            paths = []
            for k, b in enumerate(tagged):
                p = os.path.join(d, f"f{k}.flac")
                with open(p, "wb") as f:
                    f.write(b)
                paths.append(p)
            t0 = time.perf_counter()
            rc = subprocess.run([refcli.PATH, "-d", "-f", "-s", "--apply-replaygain-which-is-not-lossless", *paths]).returncode
            res["flac_ref_1proc_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
            assert rc == 0
            res["flac_ref_1proc_identical"] = all(open(p[:-5] + ".wav", "rb").read() == outs["rg_default"][k][0] for k, p in enumerate(paths))
            sub = paths[:a.ref_files]
            t0 = time.perf_counter()
            with ThreadPoolExecutor(a.procs) as pool:
                rcs = list(pool.map(lambda p: subprocess.run([refcli.PATH, "-d", "-f", "-s", "--apply-replaygain-which-is-not-lossless", p]).returncode, sub))
            assert not any(rcs)
            res["flac_ref_%dproc_ms" % a.procs] = round(1e3 * (time.perf_counter() - t0) * a.files / len(sub), 1)
            res["flac_ref_per_file_identical"] = all(open(p[:-5] + ".wav", "rb").read() == per_file[k][0] for k, p in enumerate(sub))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
