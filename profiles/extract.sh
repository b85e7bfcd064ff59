#!/bin/sh
# usage: [CUBIN=serve_slots_kernel] extract.sh <report.ncu-rep> <outdir>  — raw metrics, SASS page and nvdisasm of the
# translation unit the profiled kernel lives in (serve_slots_kernel, serve_slots_wide_kernel, serve_kernel ...), current library
set -e
mkdir -p "$2/cub"; (cd "$2/cub" && rm -f *.cubin *.sass && cuobjdump -xelf all "$(cd "$(dirname "$0")/.." && pwd)/gofr_b200/libgofr_b200.so" >/dev/null 2>&1 && nvdisasm --print-line-info ${CUBIN:-serve_slots_kernel}.sm_90a.cubin > serve_kernel.sass)
ncu -i "$1" --page raw --csv > "$2/raw.csv" 2>/dev/null
ncu -i "$1" --page source --csv > "$2/src.csv" 2>/dev/null
