#!/bin/bash
# closed-loop gRPC front-end load (decode → SayHello → encode per RPC) on one GPU; run from the repo root.
# Results (the card's name and power limit, then one JSON line per configuration) go to $OUT_DIR, by default a new
# temporary directory.
set -e
D=${OUT_DIR:-$(mktemp -d -t proto_frontend.XXXXXX)}; mkdir -p "$D"; echo "results in $D"
LIB=$(python -c "from gofr_b200 import _build; print(_build.build())")
g++ -O2 -std=c++17 -pthread scratch/frontend_bench/proto_bench.cpp -o "$D"/proto_bench "$LIB" -Wl,-rpath,$(dirname "$LIB")
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee "$D"/gpu.txt
CFGS=${CFGS:-"16,64,200 64,64,200 256,256,200"}
for cfg in $CFGS; do
  IFS=, read -r T B W <<< "$cfg"
  timeout 120 "$D"/proto_bench $T $B $W ${SECS:-3} | tee -a "$D"/results.jsonl
done
