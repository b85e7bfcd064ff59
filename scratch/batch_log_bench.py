#!/usr/bin/env python
"""batch_log_bench.py — what middleware.Logging's lines add to gofr_batch_submit, from pinned host buffers.

    python scratch/batch_log_bench.py [--steps 10] [--warmup 3] [--n 1048576] [--out results/batch_log_bench.json]

One batch of n config-2 requests (synth.config2_batch) with one log record each (the config-2 log strings of
synth.reqlog_batch), pinned buffers, measured in the same run:
  plain_ms / log_ms   host clock around gofr_batch_submit + wait, and around gofr_batch_submit_log + wait (the two
                      alternate, median of each);
  cpu_ms              the C restatement of the same lines (oracle/orc_reqlog.c) on the host's CPUs, one slice of the batch
                      per thread: the work the call takes off the host;
and the card's name, power limit and SM clocks, read in the same run.  The lines are compared with the expectation of
tests/test_batch_log.py on a sample before anything is timed.  Not part of bench.py."""
import argparse, ctypes as C, json, os, subprocess, sys, threading, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from gofr_b200 import _abi, synth, spec as S
from gofr_b200.engine import Engine, batch_log_bound, pin_batch, pinned_array
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


spec = synth.config2_spec()
table = Table(spec)
eng = Engine(table, 0)
L = _abi.lib()
DATE = S.http_date(1_700_000_000)
LOG_NS = 1_700_000_000_500_000_000


def log_records(n):
    """n config-2 log records: synth.reqlog_batch's first 64 Ki repeated (the strings of one period, offsets rebased)"""
    p = min(n, 65536)
    base = synth.reqlog_batch(p)
    reps = (n + p - 1) // p
    desc = np.tile(base.desc, reps)[:n].copy()
    desc["arena_off"] += (np.arange(n) // p).astype(np.uint32) * np.uint32(base.arena.size)
    return S.LogBatch(desc, np.tile(base.trace_ids, (reps, 1))[:n].copy(), np.tile(base.arena, reps))


def pinned_copy(x):
    p = pinned_array(x.nbytes).view(x.dtype)
    p[:] = x
    return p


n = a.n
batch = pin_batch(synth.config2_batch(n))
log = log_records(n)
log = S.LogBatch(pinned_copy(log.desc), log.trace_ids, pinned_copy(log.arena))
keys = np.stack([batch.desc["path_len"], batch.desc["query_len"], batch.desc["data_len"]], 1).astype(np.int64)
uk, cnt = np.unique(keys, axis=0, return_counts=True)
out_cap = int(sum(int(L.gofr_table_response_bound(table.handle, int(k[0]), int(k[1]), int(k[2]))) * int(c) for k, c in zip(uk, cnt)))
log_cap = batch_log_bound(log)
out, off, meta = pinned_array(out_cap + 64), pinned_array((n + 1) * 4).view(np.uint32), pinned_array(n * 4).view(np.uint32)
lout, loff = pinned_array(log_cap + 64), pinned_array((n + 1) * 4).view(np.uint32)
rb = _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data, arena=batch.arena.ctypes.data,
                   arena_bytes=batch.arena.size, n=n, date=DATE)
ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out_cap, out_off=off.ctypes.data, meta=meta.ctypes.data)
lb = _abi.BatchLog(desc=log.desc.ctypes.data, arena=log.arena.ctypes.data, arena_bytes=log.arena.size, log_unix_ns=LOG_NS,
                   out=lout.ctypes.data, out_cap=log_cap, log_off=loff.ctypes.data)
t = C.c_uint64()


def run(with_log):
    t0 = time.perf_counter()
    if with_log:
        _abi.check(L.gofr_batch_submit_log(eng._e, C.byref(rb), C.byref(ob), C.byref(lb), C.byref(t)), "gofr_batch_submit_log")
    else:
        _abi.check(L.gofr_batch_submit(eng._e, C.byref(rb), C.byref(ob), C.byref(t)), "gofr_batch_submit")
    _abi.check(L.gofr_batch_wait(eng._e, t.value), "gofr_batch_wait")
    return (time.perf_counter() - t0) * 1e3


# ---- check before timing: responses as without the log, a sample of lines against the expectation ----
run(False)
plain_out = bytes(out[:int(off[n])])
plain_meta = meta.copy()
run(True)
assert bytes(out[:int(off[n])]) == plain_out and (meta == plain_meta).all()
k = 4096
sel = np.nonzero(((meta[:k] >> 16) != 0xFFFF) & ((meta[:k] & 0xFFFF) != 0))[0]
d = log.desc[sel].copy()
d["status"], d["log_unix_ns"], d["elapsed_ns"] = meta[sel] & 0xFFFF, LOG_NS, LOG_NS - d["start_unix_ns"]
wo, wf = O.request_log(S.LogBatch(d, batch.trace_ids[sel].copy(), log.arena))
got = [bytes(lout[int(loff[i]):int(loff[i + 1])]) for i in sel.tolist()]
assert got == [wo[int(wf[j]):int(wf[j + 1])].tobytes() for j in range(len(sel))], "lines differ from the expectation"
lines, log_bytes = int(lb.lines), int(lb.out_bytes)

# ---- the C restatement of the same lines on the host's CPUs ----
fill = log.desc.copy()
fill["status"], fill["log_unix_ns"], fill["elapsed_ns"] = meta & 0xFFFF, LOG_NS, LOG_NS - fill["start_unix_ns"]
nthreads = os.cpu_count() or 1
bounds = np.linspace(0, n, nthreads + 1).astype(np.int64)
per = 320 + 6 * sum(log.desc[f].astype(np.int64) for f in ("method_len", "ua_len", "xff_len", "remote_len", "uri_len"))
cpu_out = [np.zeros(int(per[b0:b1].sum()) + 64, np.uint8) for b0, b1 in zip(bounds, bounds[1:])]
cpu_off = [np.zeros(int(b1 - b0) + 1, np.uint32) for b0, b1 in zip(bounds, bounds[1:])]
ids = np.ascontiguousarray(batch.trace_ids)
OL = O.lib()


def cpu_slice(j):
    b0, b1 = int(bounds[j]), int(bounds[j + 1])
    OL.orc_request_log(fill[b0:].ctypes.data, ids[b0:].ctypes.data, log.arena.ctypes.data, b1 - b0, cpu_out[j].ctypes.data,
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
    "metric": "batch_log_ms", "n": n, "steps": a.steps, "plain_ms": float(np.median(plain)), "log_ms": float(np.median(logged)),
    "plain_ms_all": [round(x, 3) for x in plain], "log_ms_all": [round(x, 3) for x in logged],
    "cpu_ms": float(np.median(cpu)), "cpu_threads": nthreads, "lines": lines, "log_bytes": log_bytes,
    "card": smi("name"), "power_limit": smi("power.limit"), "sm_clock_max": smi("clocks.max.sm"),
    "sm_clock_before": clocks_before, "sm_clock_after": clocks_after,
}
res["log_over_plain"] = res["log_ms"] / res["plain_ms"]
print(json.dumps(res))
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(json.dumps(res) + "\n")
