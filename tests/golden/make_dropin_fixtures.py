"""Generates tests/golden/dropin_v1.json from the reference's headers and example clients -- run where the reference's
sources are and `make -C oracle ref` has built oracle/_ref/obj_default:

    python tests/golden/make_dropin_fixtures.py <reference source dir>

The fixture stores
  * struct_layout: what tests/test_dropin_examples.py's LAYOUT_PROBE prints when compiled against the reference's
    FLAC/all.h (sizes and field offsets of the structs a client reads through the callbacks);
  * decode_client_symbols / encode_client_symbols: the FLAC__ symbols the unmodified examples/c/{decode,encode}/file/main.c
    leave for the library to define when they are linked the way oracle/Makefile `examples` links them (the encode
    client together with the reference's metadata object helpers, whose own FLAC__ needs count too).
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, ".."))

from test_dropin_examples import LAYOUT_PROBE, METADATA_OBJECTS  # noqa: E402


def _syms(obj, flag):
    out = subprocess.run(["nm", flag, obj], capture_output=True, text=True, check=True).stdout
    return {line.split()[-1] for line in out.splitlines() if line.split() and line.split()[-1].startswith("FLAC__")}


def _client_needs(ref, tmp, client, helpers):
    obj = os.path.join(tmp, client + ".o")
    subprocess.run(["gcc", "-O1", "-include", "inttypes.h", f"-I{ref}/include", "-c", f"{ref}/examples/c/{client}/file/main.c", "-o", obj],
                   check=True)
    undefined, defined = set(), set()
    for o in [obj] + helpers:
        undefined |= _syms(o, "-u")
        defined |= _syms(o, "--defined-only")
    return sorted(undefined - defined)


def main():
    ref = sys.argv[1]
    helpers = [os.path.join(ROOT, "oracle", "_ref", "obj_default", o + ".o") for o in METADATA_OBJECTS]
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "layout.c")
        with open(src, "w") as fh:
            fh.write(LAYOUT_PROBE % '#include "FLAC/all.h"')
        exe = os.path.join(tmp, "layout")
        subprocess.run(["gcc", src, "-o", exe, f"-I{ref}/include"], check=True)
        layout = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
        out = {"struct_layout": layout.splitlines(),
               "decode_client_symbols": _client_needs(ref, tmp, "decode", []),
               "encode_client_symbols": _client_needs(ref, tmp, "encode", helpers)}
    with open(os.path.join(HERE, "dropin_v1.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    print("wrote", len(out["struct_layout"]), "layout lines,", len(out["decode_client_symbols"]), "+", len(out["encode_client_symbols"]), "symbols")


if __name__ == "__main__":
    main()
