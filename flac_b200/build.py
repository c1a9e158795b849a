"""Builds flac_b200/libflac_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m flac_b200.build [--force]

Flags that matter for bit-exactness: -fmad=false (no FMA contraction of the LPC analysis),
host side -ffp-contract=off (window tables use the host libm exactly like the reference).
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = [os.path.join(HERE, "csrc", f) for f in ("encoder.cu", "general_kernels.cu", "autoc_kernel.cu", "search_kernel.cu", "emit_kernel.cu",
                                              "tiled_kernels.cu", "files_kernels.cu", "md5_kernel.cu", "files_decode_kernels.cu", "flac_parse.cu", "decoder.cu",
                                              "stream_api.cu", "flac_metadata.cu", "pcm_container.cu", "replaygain_kernel.cu",
                                              "reencode.cu", "add_replaygain.cu", "replaygain_synthesis.cu")]
OBJ_DIR = os.path.join(HERE, "csrc", "_obj")
HDR = sorted(glob.glob(os.path.join(HERE, "csrc", "*.h")) + glob.glob(os.path.join(HERE, "csrc", "*.cuh"))) + [
    os.path.join(HERE, "..", "include", "flac_b200.h"), os.path.join(HERE, "..", "include", "flac_b200_stream.h")]
OUT = os.path.join(HERE, "libflac_b200.so")

NVCC_FLAGS = [
    "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-fmad=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=default",
]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.exists(p) and os.path.getmtime(p) > t for p in SRC + HDR + [__file__])


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.exists(p) and os.path.getmtime(p) > t for p in [src, __file__] + HDR)


def build(force=False, verbose=False):
    """One object per translation unit, compiled in parallel (each .cu is a kernel family), then linked."""
    from concurrent.futures import ThreadPoolExecutor
    srcs = [s for s in SRC if os.path.exists(s)]
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ_DIR, exist_ok=True)
    objs = [os.path.join(OBJ_DIR, os.path.basename(s)[:-3] + ".o") for s in srcs]

    def compile_one(pair):
        src, obj = pair
        if not force and not _stale(obj, src):
            return ""
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("nvcc failed compiling " + src)
        return r.stderr

    with ThreadPoolExecutor(len(srcs)) as pool:
        logs = list(pool.map(compile_one, zip(srcs, objs)))
    r = subprocess.run([nvcc, "-shared", "-o", OUT] + objs + ["-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed linking libflac_b200.so")
    if verbose:
        print("".join(logs))
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
