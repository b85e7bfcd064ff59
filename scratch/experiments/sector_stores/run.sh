#!/bin/bash
# run.sh [steps] — builds sector_stores.cu in a temporary directory and runs it on GPU 0 (one JSON line per pattern)
set -e
here="$(cd "$(dirname "$0")" && pwd)"
tmp=$(mktemp -d)
trap 'rm -rf "$tmp"' EXIT
"${NVCC:-/usr/local/cuda/bin/nvcc}" -gencode arch=compute_90a,code=sm_90a -O3 -o "$tmp/sector_stores" "$here/sector_stores.cu"
"$tmp/sector_stores" "${1:-50}"
