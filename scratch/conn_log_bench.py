#!/usr/bin/env python
"""conn_log_bench.py — what middleware.Logging's lines add to gofr_conn_batch_submit, from pinned host buffers.

    python scratch/conn_log_bench.py [--steps 10] [--warmup 3] [--scale 1.0]

Config 2 connection streams, two mixes: 1 Mi connections of one request, and 256 Ki connections of four pipelined requests.
Per mix one JSON line, measured in the same run:
  plain_ms / log_ms    host clock around submit + wait, without and with the log (alternating runs, median of each);
  gather_ms, reqlog_ms, pack_ms
                       kernel ms of the log's three kernels per batch and per chunk (torch.profiler, in a run of its
                       own); chunks are counted as conn_plan cuts them (65 536 connections or 8 MiB, whichever is less);
  reqlog_unstaged      share of the log lines' reqlog tiles whose strings span more than the kernel's 24 KiB staging
                       buffer (computed on the host from the gather's placement rule), so that they are read from HBM;
and the card's name and power limit.  The lines are compared with the request-log oracle on a sample before anything is
timed.  Not part of bench.py."""
import argparse, ctypes as C, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from gofr_b200 import _abi, synth, spec as S
from gofr_b200.engine import Engine, conn_batch_bound, conn_log_bound, pinned_array
from gofr_b200.table import Table

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--scale", type=float, default=1.0, help="connection counts are multiplied by this (rehearsals)")
a = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
table = Table(synth.config2_spec())
eng = Engine(table, 0)
L = _abi.lib()
DATE = S.http_date(1_700_000_000)
LOG_NS = 1_700_000_000_500_000_000


def conn_chunks(off: np.ndarray, chunk: int = 65536, budget: int = 8 << 20):
    """the connection ranges [lo, hi) conn_plan (engine.cu) cuts: at most `chunk` connections whose bytes fit `budget`, at
    least one"""
    out, lo, n = [], 0, len(off) - 1
    while lo < n:
        hi = lo
        while hi < n and hi - lo < chunk:
            if hi > lo and int(off[hi + 1]) - int(off[lo]) > budget:
                break
            hi += 1
        out.append((lo, hi))
        lo = hi
    return out


def pinned_copy(x: np.ndarray) -> np.ndarray:
    p = pinned_array(x.nbytes).view(x.dtype)
    p[:] = x
    return p


for n, reqs in ((int((1 << 20) * a.scale), 1), (int((1 << 18) * a.scale), 4)):
    buf, off = synth.http_streams(n, reqs=(reqs, reqs))
    remote, roff, start = synth.conn_clients(n)
    req_cap, out_cap = conn_batch_bound(table, off)
    line_cap, lout_cap = conn_log_bound(off, roff)
    pbuf, poff, premote, proff, pstart = map(pinned_copy, (buf, off, remote, roff, start))
    cols = {k: pinned_array(4 * (req_cap + 1)).view(np.uint32) for k in ("out_off", "meta", "req_at")}
    ids = pinned_array(16 * req_cap)
    per_conn = {k: pinned_array(4 * (n + 1)).view(np.uint32) for k in ("req_first", "consumed", "conn_status")}
    out = pinned_array(out_cap)
    lout, log_off, log_req = pinned_array(lout_cap), pinned_array(4 * (line_cap + 1)).view(np.uint32), pinned_array(4 * line_cap).view(np.uint32)
    cb = _abi.ConnBatch(buf=pbuf.ctypes.data, buf_off=poff.ctypes.data, buf_bytes=pbuf.size, n_conns=n, date=DATE, trace_seed=7)
    cr = _abi.ConnResp(out=out.ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=cols["out_off"].ctypes.data,
                       meta=cols["meta"].ctypes.data, req_at=cols["req_at"].ctypes.data, trace_ids=ids.ctypes.data,
                       req_first=per_conn["req_first"].ctypes.data, consumed=per_conn["consumed"].ctypes.data,
                       conn_status=per_conn["conn_status"].ctypes.data)
    cl = _abi.ConnLog(remote=premote.ctypes.data, remote_off=proff.ctypes.data, start_unix_ns=pstart.ctypes.data, log_unix_ns=LOG_NS,
                      tz_offset_s=0, line_cap=line_cap, out=lout.ctypes.data, out_cap=lout_cap, log_off=log_off.ctypes.data,
                      log_req=log_req.ctypes.data)

    def run(log):
        t = C.c_uint64()
        if log:
            _abi.check(L.gofr_conn_batch_submit_log(eng._e, C.byref(cb), C.byref(cr), C.byref(cl), C.byref(t)), "submit_log")
        else:
            _abi.check(L.gofr_conn_batch_submit(eng._e, C.byref(cb), C.byref(cr), C.byref(t)), "submit")
        _abi.check(L.gofr_batch_wait(eng._e, t.value), "gofr_batch_wait")

    # check a sample of lines against the request-log oracle (what the model of tests/test_conn_log.py composes)
    run(True)
    k, m = int(per_conn["req_first"][n]), int(cl.lines)
    assert m == k and np.array_equal(log_req[:m], np.arange(m, dtype=np.uint32))
    from tests import oracle as O
    from tests import http_frame_oracle as FO
    sample = np.arange(0, n, max(1, n // 500))
    sb = [buf[off[c]:off[c + 1]] for c in sample]
    soff = np.cumsum([0] + [len(x) for x in sb]).astype(np.uint32)
    sbuf = np.concatenate(sb)
    rec, _, _, _ = FO.http_frame(sbuf, soff)
    _, _, _, spans = O.http_parse(sbuf, rec)
    b = sbuf.tobytes()
    recs = []
    for q, c in enumerate(sample.tolist()):
        for j in range(reqs):
            sp = spans[q * reqs + j]
            get = lambda f: b[int(sp[f] & 0xFFFFFFFF):int(sp[f] & 0xFFFFFFFF) + int(sp[f] >> 32)]
            kk = int(per_conn["req_first"][c]) + j
            recs.append(S.LogRec(int(start[c]), LOG_NS - int(start[c]), LOG_NS, get(0), get(2), get(3), remote[roff[c]:roff[c + 1]].tobytes(),
                                 get(1), int(cols["meta"][kk] & 0xFFFF), 0, ids[16 * kk:16 * kk + 16].tobytes()))
    wo, wf = O.request_log(S.LogBatch.pack(recs))
    got = b"".join(lout[log_off[int(per_conn["req_first"][c]) + j]:log_off[int(per_conn["req_first"][c]) + j + 1]].tobytes()
                   for c in sample.tolist() for j in range(reqs))
    assert got == wo[:int(wf[-1])].tobytes()

    # reqlog tiles past the staging buffer: a tile's strings span from its first line's to past its last line's
    # (rec_off - alo) + k * R within each chunk conn_plan cuts
    ranges = conn_chunks(off)
    R = int(np.diff(roff.astype(np.int64)).max())
    unstaged = tiles = 0
    for c0, c1 in ranges:
        k0 = int(per_conn["req_first"][c0])
        at = cols["req_at"][k0:int(per_conn["req_first"][c1])].astype(np.int64)
        pos = at - (int(off[c0]) & ~15) + np.arange(len(at)) * R
        end = np.append(pos[1:], pos[-1] + 400)
        for t0 in range(0, len(pos), 128):
            tiles += 1
            unstaged += int(end[min(t0 + 127, len(pos) - 1)] - pos[t0] > 24 * 1024)

    times = {False: [], True: []}
    for _ in range(a.warmup):
        run(False); run(True)
    for _ in range(a.steps):
        for log in (False, True):
            torch.cuda.synchronize()
            t = time.perf_counter()
            run(log)
            times[log].append((time.perf_counter() - t) * 1e3)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(True)
        torch.cuda.synchronize()
    chunks = len(ranges)
    kt = {"gather": 0.0, "reqlog": 0.0, "pack": 0.0}
    for ev in prof.key_averages():
        for key, name in (("gather", "conn_log_kernel"), ("reqlog", "reqlog_kernel"), ("pack", "chunk_pack_kernel")):
            if name in ev.key:
                kt[key] += ev.device_time_total / 1e3
    print(json.dumps({"mix": f"config2 {n} connections x {reqs} requests", "requests": k, "lines": m, "log_bytes": int(cl.out_bytes),
                      "chunks": chunks, "conns_per_chunk": round(n / chunks), "gather_ms": round(kt["gather"], 3),
                      "reqlog_ms": round(kt["reqlog"], 3), "pack_ms": round(kt["pack"], 3), "plain_ms": round(float(np.median(times[False])), 3), "log_ms": round(float(np.median(times[True])), 3),
                      "gather_ms_per_chunk": round(kt["gather"] / chunks, 4), "reqlog_ms_per_chunk": round(kt["reqlog"] / chunks, 4),
                      "pack_ms_per_chunk": round(kt["pack"] / chunks, 4), "reqlog_unstaged_tiles": f"{unstaged}/{tiles}",
                      "remote_max": R, "card": card}), flush=True)
