#!/usr/bin/env python
"""proto_log_bench.py — what the gRPC LoggingInterceptor's lines add to gofr_proto_batch_encode, from pinned host buffers.

    python scratch/proto_log_bench.py [--steps 10] [--warmup 3] [--n 1048576] [--out results/proto_log_bench.json]

One batch of n HelloResponse rows ("Hello caller-<i>!") with one RPCLog record each (method /Hello/SayHello, every call
logging), pinned buffers, measured in the same run:
  plain_ms / log_ms   host clock around gofr_proto_batch_encode + wait, and around gofr_proto_batch_encode_log + wait (the
                      two alternate; median and range of each);
  cpu_ms              the C restatement of the same lines (oracle/orc_reqlog.c) on the host's CPUs, one slice of the batch
                      per thread: the work the call takes off the host;
and the card's name, power limit and SM clocks, read in the same run.  The frames are compared with the call without a
log and the lines with the oracle's before anything is timed.  Not part of bench.py."""
import argparse, ctypes as C, json, os, subprocess, sys, threading, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from gofr_b200 import _abi, spec as S
from gofr_b200.engine import Engine, batch_log_bound, nested_bound, pinned_array
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--n", type=int, default=1 << 20)
ap.add_argument("--out", default="")
a = ap.parse_args()


def smi(q):
    return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()


def pinned_copy(x):
    p = pinned_array(x.nbytes).view(x.dtype).reshape(x.shape)
    p[:] = x
    return p


eng = Engine(Table(synth.config1_spec()), 0)
L = _abi.lib()
HELLO = [[S.ProtoNField(1, S.PB_STRING)]]
LOG_NS = 1_700_000_000_500_000_000
METHOD = b"/Hello/SayHello"
n = a.n

# ---- rows: HelloResponse{message: "Hello caller-<i>!"}, each its length word and its bytes padded to 4 ----
msgs = [b"Hello caller-%d!" % i for i in range(n)]
lens = np.array([len(m) for m in msgs], np.uint32)
padded = (lens + 3) & ~np.uint32(3)
row_off = np.zeros(n + 1, np.uint32)
row_off[1:] = np.cumsum(4 + padded)
rows = bytearray(int(row_off[-1]) + 16)
for i, m in enumerate(msgs):
    o = int(row_off[i])
    rows[o:o + 4] = len(m).to_bytes(4, "little")
    rows[o + 4:o + 4 + len(m)] = m
rows = pinned_copy(np.frombuffer(bytes(rows), np.uint8))
row_off = pinned_copy(row_off)

# ---- log records: the handler's clock and the span's trace id per call, the method once per record ----
desc = np.zeros(n, S.LOG_DESC_DTYPE)
desc["start_unix_ns"] = LOG_NS - 2_000_000 - (np.arange(n, dtype=np.int64) % 1_000_003) * 997
desc["elapsed_ns"] = 12_345 + np.arange(n, dtype=np.int64) % 50_000
desc["arena_off"] = 0
desc["method_len"] = len(METHOD)
desc["tz_offset_s"] = 19800
desc["kind"] = S.LOG_RPC
log = S.LogBatch(pinned_copy(desc), pinned_copy(synth.trace_ids(7, np.arange(n))), pinned_copy(np.frombuffer(METHOD, np.uint8)))

per_byte, per_record = nested_bound(HELLO, 0, False)
out_cap = per_byte * int(row_off[-1]) + per_record * n
log_cap = batch_log_bound(log)
out, off, meta = pinned_array(out_cap + 64), pinned_array((n + 1) * 4).view(np.uint32), pinned_array(n * 4).view(np.uint32)
lout, loff = pinned_array(log_cap + 64), pinned_array((n + 1) * 4).view(np.uint32)
nm, nf, k = S.proto_nested_tables(HELLO)
pb = _abi.ProtoBatch(data=rows.ctypes.data, data_bytes=rows.size, off=row_off.ctypes.data, n=n)
ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out_cap, out_off=off.ctypes.data, meta=meta.ctypes.data)
lb = _abi.BatchLog(desc=log.desc.ctypes.data, arena=log.arena.ctypes.data, arena_bytes=log.arena.size, log_unix_ns=LOG_NS,
                   out=lout.ctypes.data, out_cap=log_cap, log_off=loff.ctypes.data)
t = C.c_uint64()


def run(with_log):
    t0 = time.perf_counter()
    if with_log:
        _abi.check(L.gofr_proto_batch_encode_log(eng._e, nm.ctypes.data, 1, nf.ctypes.data, k, 0, None, C.byref(pb),
                                                 log.trace_ids.ctypes.data, C.byref(ob), C.byref(lb), C.byref(t)),
                   "gofr_proto_batch_encode_log")
    else:
        _abi.check(L.gofr_proto_batch_encode(eng._e, nm.ctypes.data, 1, nf.ctypes.data, k, 0, None, C.byref(pb), C.byref(ob),
                                             C.byref(t)), "gofr_proto_batch_encode")
    _abi.check(L.gofr_batch_wait(eng._e, t.value), "gofr_batch_wait")
    return (time.perf_counter() - t0) * 1e3


# ---- check before timing: frames as without the log, a sample of lines against the oracle ----
run(False)
plain_out, plain_off, plain_meta = bytes(out[:int(off[n])]), off.copy(), meta.copy()
assert (plain_meta == S.GRPC_OK).all()
run(True)
assert bytes(out[:int(off[n])]) == plain_out and (off == plain_off).all() and (meta == plain_meta).all()
fill = log.desc.copy()
fill["log_unix_ns"] = LOG_NS
ks = 4096
wo, wf = O.request_log(S.LogBatch(fill[:ks].copy(), log.trace_ids[:ks].copy(), log.arena))
got = [bytes(lout[int(loff[i]):int(loff[i + 1])]) for i in range(ks)]
assert got == [wo[int(wf[j]):int(wf[j + 1])].tobytes() for j in range(ks)], "lines differ from the oracle"
lines, log_bytes = int(lb.lines), int(lb.out_bytes)
assert lines == n

# ---- the C restatement of the same lines on the host's CPUs ----
nthreads = os.cpu_count() or 1
bounds = np.linspace(0, n, nthreads + 1).astype(np.int64)
cpu_out = [np.zeros(int(b1 - b0) * (320 + 7 * len(METHOD)) + 64, np.uint8) for b0, b1 in zip(bounds, bounds[1:])]
cpu_off = [np.zeros(int(b1 - b0) + 1, np.uint32) for b0, b1 in zip(bounds, bounds[1:])]
ids = np.ascontiguousarray(log.trace_ids)
arena = np.ascontiguousarray(log.arena)
OL = O.lib()


def cpu_slice(j):
    b0, b1 = int(bounds[j]), int(bounds[j + 1])
    OL.orc_request_log(fill[b0:].ctypes.data, ids[b0:].ctypes.data, arena.ctypes.data, b1 - b0, cpu_out[j].ctypes.data,
                       cpu_out[j].size, cpu_off[j].ctypes.data)


def cpu_run():
    t0 = time.perf_counter()
    th = [threading.Thread(target=cpu_slice, args=(j,)) for j in range(nthreads)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    return (time.perf_counter() - t0) * 1e3


cpu_run()
assert sum(int(o[-1]) for o in cpu_off) == log_bytes

for _ in range(a.warmup):
    run(False), run(True)
clocks_before = smi("clocks.sm")
plain, logged = [], []
for _ in range(a.steps):
    plain.append(run(False))
    logged.append(run(True))
clocks_after = smi("clocks.sm")
cpu = [cpu_run() for _ in range(3)]
res = {
    "metric": "proto_log_ms", "n": n, "steps": a.steps,
    "plain_ms": float(np.median(plain)), "plain_ms_range": [round(min(plain), 3), round(max(plain), 3)],
    "log_ms": float(np.median(logged)), "log_ms_range": [round(min(logged), 3), round(max(logged), 3)],
    "cpu_ms": float(np.median(cpu)), "cpu_threads": nthreads, "lines": lines, "log_bytes": log_bytes,
    "frame_bytes": len(plain_out),
    "card": smi("name"), "power_limit": smi("power.limit"), "sm_clock_max": smi("clocks.max.sm"),
    "sm_clock_before": clocks_before, "sm_clock_after": clocks_after,
}
res["log_over_plain"] = res["log_ms"] / res["plain_ms"]
print(json.dumps(res))
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(json.dumps(res) + "\n")
