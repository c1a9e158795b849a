"""Batch-of-files encode benchmark (fb200_encode_files_host / _device).

    python tools/bench_files.py [--steps 3] [--scale 1.0] [--only NAME] [--no-ref] [--fixed-guess c|host]

Per workload (ragged file lengths, seeded):
  device_*      fb200_encode_files_device, int32 PCM already on the device, host clock around the (synchronous) call
  host_*        fb200_encode_files_host end to end: packed PCM from pinned host memory to file-major frames in pinned host memory
  *_md5_off / *_md5_on   files/s and Gsamples/s (all channels)
  md5_chain_mb_s  largest file's MD5 input bytes / device call time with MD5 on: the chain rate if the MD5 stream is the call's critical path
  tails_ms      device call over the files' tails alone (the general-path launches, one set per distinct tail length)
  ref_*         the reference with MD5 on, one encoder per file over every host thread
  frames_equal / streaminfo_equal  every frame and every STREAMINFO (MD5 on) against the strict reference encoding each file alone,
                dispatched as this host dispatches it
  --fixed-guess host  encode with x86_avx2_fixed_guess = host_x86_avx2_fixed_guess() (the flac tool's frames on this host; default
                c: the C routine), and time the device call and the tails with the field at 0 and at the host's value, alternating
  equal-length whole-block files, MD5 off: fb200_encode_files_device vs fb200_encode_device + set_file_blocks on the same input,
  alternating in one process (compaction + gather over the single-stream path)
Prints one JSON line with the GPU's name and power limit (read-only nvidia-smi query)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import flac_b200  # noqa: E402
import reflib  # noqa: E402
import signals  # noqa: E402

WORKLOADS = [  # name, channels, bps, rate, level, blocksize, files, lengths(rng, scale)
    ("8ch_24_192_l8_125files", 8, 24, 192000, 8, 4096, 125,
     lambda rng, s, n: ((rng.integers(80, 121, size=n) * 4096 + rng.integers(1, 4096, size=n)) * s).astype(np.int64)),
    ("stereo_16_44_l5_200files", 2, 16, 44100, 5, 4096, 200,
     lambda rng, s, n: ((60 * 44100 + rng.integers(-2 * 44100, 2 * 44100, size=n)) * s).astype(np.int64)),
]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if q.returncode == 0 and q.stdout.strip() else ("?", "?")
    return name, power


def make_pcm(total, ch, bps, rate):
    """music_like audio: a seeded 64-block base tiled to length, one LSB flipped every 7 samples so blocks differ."""
    base = signals.music_like(4096 * 64, ch, bps, rate, seed=1)
    x = np.ascontiguousarray(np.tile(base, ((total + base.shape[0] - 1) // base.shape[0], 1))[:total])
    x[::7, 0] ^= 1
    return x


def timed(fn, steps):
    fn()
    t = time.perf_counter()
    for _ in range(steps):
        fn()
    return (time.perf_counter() - t) / steps


def run(name, ch, bps, rate, level, bs, nfiles, lengths_fn, steps, scale, with_ref, fixed_guess):
    import torch
    lengths = np.maximum(lengths_fn(np.random.default_rng(7), scale, nfiles), 1).astype(np.uint64)
    total = int(lengths.sum())
    x = make_pcm(total, ch, bps, rate)
    guess = flac_b200.host_x86_avx2_fixed_guess() if fixed_guess == "host" else 0
    enc = flac_b200.Encoder(flac_b200.preset(ch, bps, rate, level, bs, x86_avx2_fixed_guess=guess))
    nfr, cap = enc.files_capacity(lengths)
    d_pcm = torch.from_numpy(x).cuda()
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_off = torch.zeros(nfr + 1, dtype=torch.int64, device="cuda")
    nsamp = total * ch
    r = {"workload": name, "files": nfiles, "samples_per_channel": total, "frames": nfr, "scale": scale, "x86_avx2_fixed_guess": guess}

    def dev(md5, lens=lengths):
        return enc.encode_files_device(d_pcm.data_ptr(), lens, d_out.data_ptr(), cap, d_off.data_ptr(), md5=md5)

    nbytes = 2 if bps <= 16 else 3
    h_in = torch.from_numpy(flac_b200.pack_pcm(x, nbytes)).pin_memory()
    h_out = torch.empty(cap, dtype=torch.uint8).pin_memory()
    h_off = torch.zeros(nfr + 1, dtype=torch.int64).pin_memory()
    infos = (flac_b200.FileInfo * nfiles)()
    nf = C.c_uint64(0)

    def host(md5):
        flac_b200._check(flac_b200.lib().fb200_encode_files_host(enc._h, h_in.data_ptr(), nbytes, lengths.ctypes.data, nfiles, 1 if md5 else 0,
                                                                  h_out.data_ptr(), cap, h_off.data_ptr(), C.byref(nf), infos))

    for md5 in (False, True):
        tag = "md5_on" if md5 else "md5_off"
        td = timed(lambda: dev(md5), steps)
        th = timed(lambda: host(md5), steps)
        r["device_files_s_" + tag] = round(nfiles / td, 1)
        r["device_gsps_" + tag] = round(nsamp / td / 1e9, 2)
        r["host_files_s_" + tag] = round(nfiles / th, 1)
        r["host_gsps_" + tag] = round(nsamp / th / 1e9, 2)
        if md5:
            r["md5_chain_mb_s"] = round(int(lengths.max()) * ch * ((bps + 7) // 8) / td / 1e6, 1)
            r["device_ms_md5_on"] = round(td * 1e3, 2)
        else:
            r["device_ms_md5_off"] = round(td * 1e3, 2)
    tails = lengths % np.uint64(bs)
    tails = tails[tails > 0]
    r["distinct_tail_lengths"] = int(np.unique(tails).size)
    r["tails_ms"] = round(timed(lambda: dev(False, tails), steps) * 1e3, 2)
    if fixed_guess == "host":
        # the field at 0 and at the host's value, alternating: device call (MD5 off) and tails alone
        enc_c = flac_b200.Encoder(flac_b200.preset(ch, bps, rate, level, bs))
        ms = {"c": ([], []), "host": ([], [])}
        for _ in range(5):
            for e, m in ((enc_c, "c"), (enc, "host")):
                for lens, acc in zip((lengths, tails), ms[m]):
                    acc.append(round(timed(lambda: e.encode_files_device(d_pcm.data_ptr(), lens, d_out.data_ptr(), cap, d_off.data_ptr(), md5=False),
                                           steps) * 1e3, 2))
        enc_c.close()
        r["fixed_guess_ms"] = {m: {"device_ms_md5_off": v[0], "tails_ms": v[1]} for m, v in ms.items()}

    # outputs of the last host call (MD5 on) against the reference, file by file
    out, off = h_out.numpy(), h_off.numpy()
    got = [(bytes(infos[f].streaminfo), [out[off[i]:off[i + 1]].tobytes() for i in range(infos[f].first_frame, infos[f].first_frame + infos[f].nframes)])
           for f in range(nfiles)]
    starts = np.concatenate([[0], np.cumsum(lengths.astype(np.int64))])
    if with_ref and reflib.available("strict"):
        from test_gpu_files import want_streaminfo

        def ref_one(f, variant):
            # the harness writes without a seek callback, so its own STREAMINFO is never patched: the expectation is computed
            # from its frames and the input, as update_metadata_ would write it
            xf = x[starts[f]:starts[f + 1]]
            _, _, frames = reflib.encode(xf, bps, rate=rate, level=level, blocksize=bs, md5=True, variant=variant)
            return want_streaminfo(xf, frames, bs, bps, rate), frames
        workers = os.cpu_count() or 1
        with ThreadPoolExecutor(workers) as pool:
            ref = list(pool.map(lambda f: ref_one(f, "strict"), range(nfiles)))
        r["frames_equal"] = sum(a[1] == b[1] for a, b in zip(got, ref))
        r["streaminfo_equal"] = sum(a[0] == b[0] for a, b in zip(got, ref))
        bad = [f for f in range(nfiles) if got[f][1] != ref[f][1]]
        if bad:  # which frames, and what the single-stream entry point gives for the same file
            r["frames_differ"] = []
            for f in bad[:8]:
                xf = x[starts[f]:starts[f + 1]]
                single = enc.encode_frames(xf)
                r["frames_differ"].append({"file": f, "samples": int(lengths[f]), "nframes": len(got[f][1]), "ref_nframes": len(ref[f][1]),
                                           "differing": [i for i, (a, b) in enumerate(zip(got[f][1], ref[f][1])) if a != b][:10],
                                           "single_stream_equals_ref": single == ref[f][1], "single_stream_equals_files": single == got[f][1]})
        t = time.perf_counter()
        with ThreadPoolExecutor(workers) as pool:
            list(pool.map(lambda f: ref_one(f, "default"), range(nfiles)))
        tr = time.perf_counter() - t
        r["ref_files_s_md5_on"] = round(nfiles / tr, 1)
        r["ref_gsps_md5_on"] = round(nsamp / tr / 1e9, 3)
        r["host_threads"] = workers
    del h_in, h_out
    enc.close()
    return r


def equal_length(steps, pairs=5):
    """125 files of 100 whole blocks, stereo 16-bit -5, MD5 off: files entry point vs encode_device + set_file_blocks."""
    import torch
    ch, bps, rate, bs, nfiles, blocks = 2, 16, 44100, 4096, 125, 100
    lengths = np.full(nfiles, blocks * bs, dtype=np.uint64)
    x = make_pcm(int(lengths.sum()), ch, bps, rate)
    enc = flac_b200.Encoder(flac_b200.preset(ch, bps, rate, 5, bs))
    nfr, cap = enc.files_capacity(lengths)
    d_pcm = torch.from_numpy(x).cuda()
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    d_off = torch.zeros(nfr + 1, dtype=torch.int64, device="cuda")

    def files():
        enc.encode_files_device(d_pcm.data_ptr(), lengths, d_out.data_ptr(), cap, d_off.data_ptr(), md5=False)

    def single():
        enc.set_file_blocks(blocks)
        enc.encode_device(d_pcm.data_ptr(), x.shape[0], d_out.data_ptr(), cap, d_off.data_ptr(), sync=True)
        enc.set_file_blocks(0)

    tf, ts = [], []
    for _ in range(pairs):
        tf.append(timed(files, steps))
        ts.append(timed(single, steps))
    enc.close()
    return {"workload": "equal_length_stereo_16_l5_125x100blocks", "files_ms": [round(v * 1e3, 3) for v in tf],
            "file_blocks_ms": [round(v * 1e3, 3) for v in ts], "overhead_pct_median": round((np.median(tf) / np.median(ts) - 1) * 100, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every file length")
    ap.add_argument("--only", default=None)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--fixed-guess", choices=("c", "host"), default="c", help="x86_avx2_fixed_guess: 0, or host_x86_avx2_fixed_guess()")
    a = ap.parse_args()
    name, power = gpu_info()
    res = []
    for w in WORKLOADS:
        if a.only and a.only != w[0]:
            continue
        res.append(run(*w, a.steps, a.scale, not a.no_ref, a.fixed_guess))
    if not a.only:
        res.append(equal_length(a.steps))
    print(json.dumps({"gpu": name, "power_limit": power, "steps": a.steps, "results": res}))


if __name__ == "__main__":
    main()
