#!/usr/bin/env python
"""conn_bench.py — gofr_conn_batch_submit from pinned host buffers beside gofr_batch_submit_slots on the same requests.

    python scratch/conn_bench.py [--steps 10] [--warmup 3] [--scale 1.0]

Config 2, 1 Mi connections, two mixes: one request per connection and four pipelined requests per connection.  Per mix one
JSON line, all measured in the same run:
  conn_ms    host clock around submit + wait of the connection batch (frame, parse, compact, serve, egress);
  slots_ms   the same around gofr_batch_submit_slots on the same requests, parsed on the host beforehand (not timed);
  floor_ms   the PCIe floor of each call: its bytes in and out over the pinned copy bandwidths measured in this run (the
             two directions overlap, so the larger of the two);
and the card's name and power limit.  The two calls' response bytes are compared before anything is timed.  Not part of
bench.py."""
import argparse, ctypes as C, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from gofr_b200 import _abi, synth, spec as S
from gofr_b200.engine import Engine, conn_batch_bound, pin_batch, pinned_array
from gofr_b200.table import Table
from tests import oracle as O
from tests import http_frame_oracle as FO

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--scale", type=float, default=1.0, help="connection counts are multiplied by this (rehearsals)")
a = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
table = Table(synth.config2_spec())
eng = Engine(table, 0)
L = _abi.lib()
DATE = S.http_date(1_700_000_000)
SLOT = 512


def pinned_copy(x: np.ndarray) -> np.ndarray:
    p = pinned_array(x.nbytes).view(x.dtype)
    p[:] = x
    return p


def copy_gbps():
    """pinned H2D and D2H bandwidth, GB/s, with 256 MiB copies"""
    h = torch.empty(256 << 20, dtype=torch.uint8).pin_memory()
    d = torch.empty_like(h, device="cuda")
    out = []
    for f in (lambda: d.copy_(h, non_blocking=True), lambda: h.copy_(d, non_blocking=True)):
        f(); torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(5):
            f()
        torch.cuda.synchronize()
        out.append(5 * h.numel() / (time.perf_counter() - t) / 1e9)
    return out


def timed(call):
    for _ in range(a.warmup):
        call()
    t = time.perf_counter()
    for _ in range(a.steps):
        call()
    return (time.perf_counter() - t) * 1e3 / a.steps


h2d_gbps, d2h_gbps = copy_gbps()
n = int((1 << 20) * a.scale)
for reqs in (1, 4):
    buf, off = synth.http_streams(n, reqs=(reqs, reqs))
    req_cap, out_cap = conn_batch_bound(table, off)
    pbuf, poff = pinned_copy(buf), pinned_copy(off)
    cols = {k: pinned_array(4 * (req_cap + 1)).view(np.uint32) for k in ("out_off", "meta", "req_at")}
    ids = pinned_array(16 * req_cap)
    per_conn = {k: pinned_array(4 * (n + 1)).view(np.uint32) for k in ("req_first", "consumed", "conn_status")}
    out = pinned_array(out_cap)
    cb = _abi.ConnBatch(buf=pbuf.ctypes.data, buf_off=poff.ctypes.data, buf_bytes=pbuf.size, n_conns=n, date=DATE, trace_seed=7)
    cr = _abi.ConnResp(out=out.ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=cols["out_off"].ctypes.data,
                       meta=cols["meta"].ctypes.data, req_at=cols["req_at"].ctypes.data, trace_ids=ids.ctypes.data,
                       req_first=per_conn["req_first"].ctypes.data, consumed=per_conn["consumed"].ctypes.data,
                       conn_status=per_conn["conn_status"].ctypes.data)

    def conn():
        t = C.c_uint64()
        _abi.check(L.gofr_conn_batch_submit(eng._e, C.byref(cb), C.byref(cr), C.byref(t)), "gofr_conn_batch_submit")
        _abi.check(L.gofr_batch_wait(eng._e, t.value), "gofr_batch_wait")

    # the same requests, parsed on the host, with the ids the connection batch gave them
    conn()
    k = int(per_conn["req_first"][n])
    rec, _, _, _ = FO.http_frame(buf, off)
    d, arena, st, _ = O.http_parse(buf, rec)
    assert k == len(rec) - 1 and (st == 0).all()
    batch = pin_batch(S.RequestBatch(d, ids[:16 * k].reshape(k, 16).copy(), arena))
    sout, slen, smeta = pinned_array(k * SLOT), pinned_array(4 * k).view(np.uint32), pinned_array(4 * k).view(np.uint32)
    slots = lambda: eng.serve_host_slots(batch, DATE, SLOT, sout, slen, smeta)
    slots()
    assert (slen <= SLOT).all() and int(slen.sum()) == int(cr.out_bytes)
    o = sout.reshape(k, SLOT)
    for i in np.linspace(0, k - 1, 2000).astype(np.int64):
        assert o[i, :slen[i]].tobytes() == out[cols["out_off"][i]:cols["out_off"][i + 1]].tobytes(), i
    conn_ms, slots_ms = timed(conn), timed(slots)
    conn_in = buf.nbytes + off.nbytes
    conn_out = int(cr.out_bytes) + k * (4 * 3 + 16) + n * 12
    slots_in, slots_out = k * 32 + arena.nbytes, k * (SLOT + 8)
    floor = lambda bi, bo: max(bi / h2d_gbps, bo / d2h_gbps) / 1e6
    print(json.dumps({"mix": f"config2 {n} connections x {reqs} requests", "requests": k, "conn_ms": round(conn_ms, 3),
                      "conn_floor_ms": round(floor(conn_in, conn_out), 3), "slots_ms": round(slots_ms, 3),
                      "slots_floor_ms": round(floor(slots_in, slots_out), 3), "h2d_GBps": round(h2d_gbps, 1),
                      "d2h_GBps": round(d2h_gbps, 1), "card": card}), flush=True)
