#!/usr/bin/env python
"""kbench.py — kernel-only timing of the slot-layout serve kernel (config 2 by default), for same-box A/B runs:
   GOFR_LIB_PATH=scratch/variants/libgofr_X.so python scratch/kbench.py [--check] [--workload config2|config4|config3]
Prints one line: mean CUDA-event time per launch, requests/s, roofline fraction (config 2)."""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from gofr_b200 import spec as S, synth
from gofr_b200.engine import Engine
from gofr_b200.table import Table

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=1 << 20)
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--check", action="store_true")
ap.add_argument("--workload", default="config2")
ap.add_argument("--layout", default="slots")
ap.add_argument("--slot", type=int, default=0)
ap.add_argument("--tag", default="")
a = ap.parse_args()
date = S.http_date(1789974595)
if a.workload == "config2":
    spec, batch = synth.config2_spec(S.FRAME_WIRE), synth.config2_batch(a.n)
    slot = a.slot or 528
elif a.workload == "config4":
    spec, batch = synth.config4_spec(), synth.config4_batch(a.n)
    slot = a.slot or 1024
else:
    spec, batch = synth.config3_spec(), synth.config3_batch(a.n)
    slot = a.slot or 1024
n = batch.n
eng = Engine(Table(spec), 0)
eng.set_timing(True)
db = eng.upload(batch)
if a.layout == "slots":
    s_out = torch.zeros(n * slot, dtype=torch.uint8, device="cuda")
    s_len = torch.zeros(n, dtype=torch.int32, device="cuda")
    s_meta = torch.zeros(n, dtype=torch.int32, device="cuda")
    step = lambda: eng.serve_device_slots(db, date, slot, out=s_out, out_len=s_len, meta=s_meta)
else:
    resp = eng.alloc_responses(n, n * 1024)
    step = lambda: eng.serve_device(db, date, resp)
for _ in range(5):
    step()
torch.cuda.synchronize()
eng.kernel_time_ms(reset=True)
for _ in range(a.steps):
    step()
torch.cuda.synchronize()
ms, k = eng.kernel_time_ms(reset=True)
per = ms / k
line = {"tag": a.tag or os.environ.get("GOFR_LIB_PATH", "in-tree"), "workload": a.workload, "layout": a.layout, "n": n, "kernel_ms": round(per, 5), "Greq_s": round(n / per / 1e6, 3)}
if a.workload == "config2":
    algo = batch.input_bytes() + n * synth.C2_WIRE_BYTES + 8 * n + 4
    line["frac"] = round(algo / (per / 1e3) / 1e9 / 3350.0, 4)  # H100 SXM data-sheet HBM3 bandwidth
if a.check:
    from tests import oracle as O
    m = min(n, 1 << 16)
    o1, f1, m1 = O.OracleTable(spec).serve(batch.slice(0, m), date)
    if a.layout == "slots":
        out = s_out[:m * slot].cpu().numpy().reshape(m, slot)
        ln = s_len[:m].cpu().numpy().view(np.uint32)
        ok = np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32)) and np.array_equal(s_meta[:m].cpu().numpy().view(np.uint32), m1)
        bad = 0
        for i in range(m):
            L = int(ln[i])
            if L <= slot and out[i, :L].tobytes() != o1[int(f1[i]):int(f1[i]) + L].tobytes():
                bad += 1
            if L <= slot and out[i, L:(L + 15) & ~15].any():
                bad += 1
        line["check"] = "ok" if ok and not bad else f"MISMATCH ({bad} responses, columns {'ok' if ok else 'differ'})"
    else:
        out, off, meta = resp.to_host()
        ok = np.array_equal(off[:m + 1], f1) and np.array_equal(meta[:m], m1) and np.array_equal(out[:int(f1[m])], o1[:int(f1[m])])
        line["check"] = "ok" if ok else "MISMATCH"
print(json.dumps(line))
