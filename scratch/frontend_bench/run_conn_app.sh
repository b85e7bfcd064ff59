#!/bin/bash
# closed-loop load on the closure-path front-end (read → route → trivial closures → respond, 1–8 pipelined config-2
# requests per read), beside gofr_conn_frontend_serve and the route + respond_ex floor, on one GPU; run from the repo root.  Results (the card's name and power limit, then one JSON line per configuration) go to $OUT_DIR, by default a new
# temporary directory.
set -e
D=${OUT_DIR:-$(mktemp -d -t conn_app_frontend.XXXXXX)}; mkdir -p "$D"; echo "results in $D"
python - <<PY
from gofr_b200 import synth
from gofr_b200.table import Table
buf, off = synth.http_streams(65536, reqs=(1, 8))
open("$D/table.img", "wb").write(Table(synth.config2_spec()).serialize())
buf.tofile("$D/buf.bin"); off.tofile("$D/off.bin")
PY
LIB=$(python -c "from gofr_b200 import _build; print(_build.build())")
g++ -O2 -std=c++17 -pthread scratch/frontend_bench/conn_app_bench.cpp -o "$D"/conn_app_bench "$LIB" -Wl,-rpath,$(dirname "$LIB")
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee "$D"/gpu.txt
CFGS=${CFGS:-"16,64,200 64,64,200 256,256,200 1024,1024,200"}
for cfg in $CFGS; do
  IFS=, read -r T B W <<< "$cfg"
  timeout 120 "$D"/conn_app_bench "$D"/table.img "$D"/buf.bin "$D"/off.bin $T $B $W ${SECS:-3} | tee -a "$D"/results.jsonl
done
