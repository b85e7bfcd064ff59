#!/usr/bin/env python
"""http_frame_bench.py — kernel time of gofr_http_frame_device beside gofr_http_parse_device on the same bytes.

    python scratch/http_frame_bench.py [--steps 30] [--warmup 5] [--scale 1.0]

Three connection mixes: 1 Mi connections x 1 request, 256 Ki x 4 pipelined requests, 1 Mi x 1 request with a partial tail on
5 % of them.  Per mix one JSON line: mean CUDA-event time per launch of each kernel (events on the launch stream, after
warm-ups), the framer's algorithmic bytes (buffer + buf_off in; record column + first / consumed / status out) and the rate
they give, and the card's name and power limit read in the same run.  The framer's output is compared with the oracle's
before it is timed.  Not part of bench.py."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from gofr_b200 import _abi, synth
from gofr_b200.engine import Engine
from gofr_b200.table import Table
from tests import http_frame_oracle as FO

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--warmup", type=int, default=5)
ap.add_argument("--scale", type=float, default=1.0, help="connection counts are multiplied by this (rehearsals)")
a = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
eng = Engine(Table(synth.config1_spec()), 0)
eng.set_timing(True)
L = _abi.lib()


def timed(call):
    for _ in range(a.warmup):
        call()
    torch.cuda.synchronize()
    eng.kernel_time_ms(reset=True)
    for _ in range(a.steps):
        call()
    torch.cuda.synchronize()
    ms, k = eng.kernel_time_ms(reset=True)
    assert k == a.steps
    return ms / k


mixes = [("1Mi x 1 request", int((1 << 20) * a.scale), dict(reqs=(1, 1))),
         ("256Ki x 4 pipelined", int((1 << 18) * a.scale), dict(reqs=(4, 4))),
         ("1Mi x 1 request, 5% partial tails", int((1 << 20) * a.scale), dict(reqs=(1, 1), tail_every=20))]
for name, n, kw in mixes:
    buf, off = synth.http_streams(n, **kw)
    d_buf, rec, first, consumed, status = eng.http_frame_device(buf, off)
    want = FO.http_frame(buf, off)
    total = int(want[1][-1])
    got = (rec[:total + 1], first, consumed, status)
    assert all(np.array_equal(w, g.cpu().numpy().view(np.uint32)) for w, g in zip(want, got)), name
    d_off = torch.from_numpy(off.view(np.int32)).cuda()
    st = torch.cuda.current_stream().cuda_stream
    frame_ms = timed(lambda: _abi.check(L.gofr_http_frame_device(
        eng._e, d_buf.data_ptr(), d_off.data_ptr(), n, rec.data_ptr(), rec.numel() - 1, first.data_ptr(), consumed.data_ptr(),
        status.data_ptr(), st), "gofr_http_frame_device"))
    desc, arena, pstatus, spans = eng.http_parse_resident(d_buf, rec, total)
    parse_ms = timed(lambda: _abi.check(L.gofr_http_parse_device(
        eng._e, d_buf.data_ptr(), rec.data_ptr(), total, desc.data_ptr(), arena.data_ptr(), pstatus.data_ptr(), spans.data_ptr(), st),
        "gofr_http_parse_device"))
    algo = int(buf.size) + 4 * (n + 1) + 4 * (total + 1) + 4 * (n + 1) + 8 * n
    print(json.dumps({"mix": name, "connections": n, "records": total, "buffer_bytes": int(buf.size),
                      "frame_kernel_ms": round(frame_ms, 4), "parse_kernel_ms": round(parse_ms, 4),
                      "frame_algorithmic_bytes": algo, "frame_GB_s": round(algo / frame_ms / 1e6, 1),
                      "steps": a.steps, "warmup": a.warmup, "card": card}), flush=True)
eng.close()
