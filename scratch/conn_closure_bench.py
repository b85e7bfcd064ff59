#!/usr/bin/env python
"""Connection buffers served with handler closures (gofr_conn_batch_route, then gofr_conn_batch_respond with records built
ahead of time) against gofr_conn_batch_submit on the fused config-2 table, on the same bytes.

    python scratch/conn_closure_bench.py [--conns N] [--iters K] [--out results.json]

The closure table is config 2 with every route a GOFR_H_RESULT closure whose record is the config-2 Profile row; the fused
table is config 2 itself.  Outputs go to pinned buffers allocated once.  Batch times are host clocks around each call (both
end in a synchronise); the H2D / D2H byte counts are computed from the columns each call moves.  The card's name and power
limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gofr_b200 import _abi, synth  # noqa: E402
from gofr_b200 import spec as S  # noqa: E402
from gofr_b200.engine import Engine, conn_batch_bound, pinned_array  # noqa: E402
from gofr_b200.table import Table  # noqa: E402


def closure_spec():
    routes = [S.Route(S.M_GET, "/api/v1/r%02d" % k, S.H_RESULT, schema_id=1) for k in range(16)]
    return S.TableSpec(schemas=[synth.C2_SCHEMA], routes=routes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conns", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    buf, off = synth.http_streams(a.conns, reqs=(1, 8))
    n = a.conns
    date = S.http_date(1_700_000_000)
    L = _abi.lib()
    res = {"card": card, "conns": n, "buf_bytes": int(buf.size)}
    spec_c, spec_f = closure_spec(), synth.config2_spec()
    eng_c, eng_f = Engine(Table(spec_c), 0), Engine(Table(spec_f), 0)
    req_cap, out_cap = conn_batch_bound(eng_f.table, off)
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=date, trace_seed=1)

    def pin(count, dt):
        return pinned_array(max(count, 1) * np.dtype(dt).itemsize).view(dt)

    # stage 1 outputs
    r = dict(desc=pin(req_cap, S.DESC_DTYPE), arena=pin(buf.size + 64, np.uint8), meta=pin(req_cap, np.uint32),
             vars=pin(req_cap * 8, np.uint32), req_at=pin(req_cap, np.uint32), ids=pin(req_cap * 16, np.uint8),
             first=pin(n + 1, np.uint32), cons=pin(n, np.uint32), st=pin(n, np.uint32))
    cr = _abi.ConnRoute(req_cap=req_cap, desc=r["desc"].ctypes.data, arena=r["arena"].ctypes.data, meta=r["meta"].ctypes.data,
                        vars=r["vars"].ctypes.data, req_at=r["req_at"].ctypes.data, trace_ids=r["ids"].ctypes.data,
                        req_first=r["first"].ctypes.data, consumed=r["cons"].ctypes.data, conn_status=r["st"].ctypes.data)
    _abi.check(L.gofr_conn_batch_route(eng_c._e, C.byref(cb), C.byref(cr)), "route")
    k = int(r["first"][n])
    # the closures' records, built ahead of time: each request's Profile row
    rows = synth.config2_batch(k)
    ar = rows.arena.tobytes()
    recs = [S.result_record(S.RESULT_DATA, ar[int(d["arena_off"]) + 12:int(d["arena_off"]) + 12 + int(d["data_len"])])
            for d in rows.desc]
    rec_off_np = np.cumsum([0] + [len(x) for x in recs]).astype(np.uint32)
    rec = pin(int(rec_off_np[-1]), np.uint8)
    rec[:] = np.frombuffer(b"".join(recs), np.uint8)
    rec_off = pin(k + 1, np.uint32)
    rec_off[:] = rec_off_np
    rr = _abi.ConnResults(rec=rec.ctypes.data, rec_off=rec_off.ctypes.data, rec_bytes=rec.size, n_req=k)
    oc = out_cap + 8 * rec.size
    o = dict(out=pin(oc, np.uint8), off=pin(req_cap + 1, np.uint32), meta=pin(req_cap, np.uint32), at=pin(req_cap, np.uint32),
             ids=pin(req_cap * 16, np.uint8), first=pin(n + 1, np.uint32), cons=pin(n, np.uint32), st=pin(n, np.uint32))
    co = _abi.ConnResp(out=o["out"].ctypes.data, out_cap=oc, req_cap=req_cap, out_off=o["off"].ctypes.data, meta=o["meta"].ctypes.data,
                       req_at=o["at"].ctypes.data, trace_ids=o["ids"].ctypes.data, req_first=o["first"].ctypes.data,
                       consumed=o["cons"].ctypes.data, conn_status=o["st"].ctypes.data)
    t = C.c_uint64()

    def route():
        _abi.check(L.gofr_conn_batch_route(eng_c._e, C.byref(cb), C.byref(cr)), "route")

    def respond():
        _abi.check(L.gofr_conn_batch_respond(eng_c._e, C.byref(cb), C.byref(rr), C.byref(co), None, C.byref(t)), "respond")
        _abi.check(L.gofr_batch_wait(eng_c._e, t.value), "wait")

    def submit():
        _abi.check(L.gofr_conn_batch_submit(eng_f._e, C.byref(cb), C.byref(co), C.byref(t)), "submit")
        _abi.check(L.gofr_batch_wait(eng_f._e, t.value), "wait")

    times = {"route": [], "respond": [], "fused_submit": []}
    for it in range(a.iters + 3):   # three warm-up rounds, then the timed ones, the three calls alternating
        for name, fn in (("route", route), ("respond", respond), ("fused_submit", submit)):
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            if it >= 3:
                times[name].append(dt * 1e3)
    res["requests"] = k
    res["closure_records"] = k
    res["record_bytes"] = int(rec.size)
    res["response_bytes_closures"] = int(co.out_bytes)
    for name, v in times.items():
        res[name + "_ms_median"] = float(np.median(v))
        res[name + "_ms_min"] = float(np.min(v))
    res["route_plus_respond_ms_median"] = res["route_ms_median"] + res["respond_ms_median"]
    conn_cols = 4 * (n + 1) + 8 * n
    res["h2d_bytes"] = {"route": int(buf.size) + 4 * (n + 1),
                        "respond": int(buf.size) + 4 * (n + 1) + int(rec.size) + 4 * (k + 1),
                        "fused_submit": int(buf.size) + 4 * (n + 1)}
    res["d2h_bytes"] = {"route": k * (16 + 4 + 32 + 4 + 16) + int(off[-1] - off[0]) + conn_cols,
                        "respond": int(co.out_bytes) + k * (4 + 4 + 4 + 16) + conn_cols}
    submit()
    res["d2h_bytes"]["fused_submit"] = int(co.out_bytes) + k * (4 + 4 + 4 + 16) + conn_cols
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    eng_c.close()
    eng_f.close()


if __name__ == "__main__":
    main()
