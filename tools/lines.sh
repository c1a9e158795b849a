#!/bin/bash
# usage: tools/lines.sh <tu: emit_kernel|search_kernel|decoder|autoc_kernel|general_kernels> <source.csv.gz> <mangled-prefix> <kernel-substring> [top]
# Disassembles the translation unit's cubin out of the built library into .scratch/ and prints the per-source-line table.
set -e
cd "$(dirname "$0")/.."
mkdir -p .scratch/cub3
( cd .scratch/cub3 && rm -f *.cubin && cuobjdump -xelf "$1" ../../flac_b200/libflac_b200.so > /dev/null && nvdisasm -g -c "$1".sm_90a.cubin > "dis_$1.txt" && rm -f *.cubin )
python tools/ncu_lines.py "$2" ".scratch/cub3/dis_$1.txt" "$3" "${5:-45}" "$4"
rm -f ".scratch/cub3/dis_$1.txt"
