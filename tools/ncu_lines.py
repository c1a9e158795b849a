"""Attribute an ncu source-page (SASS) export to CUDA source lines using nvdisasm line info.

    ncu -i rep.ncu-rep --page source --csv --kernel-name regex:k_search3 > sass.csv
    cuobjdump -xelf all libflac_b200.so ; nvdisasm -g -c encoder.sm_90a.cubin > dis.txt
    python tools/ncu_lines.py sass.csv[.gz] dis.txt <mangled-function-name> [top] [kernel-name-substring]

With several kernels in one export, the last argument picks the launch whose demangled name contains it (default: first).

Joins by instruction order (the ncu export lists the function's SASS in program order).
Inlined code is attributed to the innermost line nvdisasm reports."""
import csv
import re
import sys
from collections import defaultdict


def main():
    sass_csv, dis, func = sys.argv[1], sys.argv[2], sys.argv[3]
    top = int(sys.argv[4]) if len(sys.argv) > 4 else 40
    pick = sys.argv[5] if len(sys.argv) > 5 else None
    import gzip
    import io
    fh = io.TextIOWrapper(gzip.open(sass_csv)) if sass_csv.endswith(".gz") else open(sass_csv)
    rows = list(csv.reader(fh))
    his = [i for i, r in enumerate(rows) if "Instructions Executed" in r]
    hi = his[0]
    if pick:
        hi = next(i for i in his if i > 0 and pick in ",".join(rows[i - 1]))
    h = rows[hi]
    ie, ss, so = h.index("Instructions Executed"), h.index("# Samples"), h.index("Source")
    inst = []
    for r in rows[hi + 1:]:
        if r and r[0] == "Kernel Name":
            break  # a second captured launch follows: the first is enough
        if len(r) > ie and r[ie].isdigit():
            inst.append((r[so].strip(), int(r[ie] or 0), int(r[ss] or 0)))
    lines = open(dis).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.startswith(".text." + func))
    cur = ("?", 0)
    seq = []
    for l in lines[start + 1:]:
        if l.startswith(".text.") or l.startswith("//--------------------- .text"):
            if seq:
                break
        m = re.search(r'//## File "([^"]+)", line (\d+)', l)
        if m:
            cur = (m.group(1).split("/")[-1], int(m.group(2)))
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
        if m:
            seq.append((cur, m.group(2).strip()))
    print(f"ncu rows {len(inst)}  nvdisasm instructions {len(seq)}")
    n = min(len(inst), len(seq))
    by = defaultdict(lambda: [0, 0, defaultdict(int)])
    for k in range(n):
        (f, ln), txt = seq[k]
        op = re.sub(r"^@!?U?P\d+\s+", "", inst[k][0]).split(" ")[0].split(".")[0]
        b = by[(f, ln)]
        b[0] += inst[k][1]
        b[1] += inst[k][2]
        b[2][op] += inst[k][1]
    tot = sum(b[0] for b in by.values()) or 1
    tots = sum(b[1] for b in by.values()) or 1
    print(f"total warp-instructions {tot}  samples {tots}")
    src = {}
    for (f, ln), b in sorted(by.items(), key=lambda kv: -kv[1][0])[:top]:
        if f not in src:
            try:
                src[f] = open("flac_b200/csrc/" + f).read().split("\n")
            except OSError:
                src[f] = []
        text = src[f][ln - 1].strip()[:90] if 0 < ln <= len(src[f]) else ""
        ops = " ".join(f"{o}:{c * 100 // max(b[0], 1)}" for o, c in sorted(b[2].items(), key=lambda kv: -kv[1])[:4])
        print(f"{b[0] / tot * 100:5.1f}% inst {b[1] / tots * 100:5.1f}% smp  {f}:{ln:<4d} {text}   [{ops}]")


if __name__ == "__main__":
    main()
