"""middleware.Logging's RequestLog line for every request of a host batch (gofr_batch_submit_log / _slots_log), CPU side.

The expectation composes oracles the project already checks: the serving oracle gives every request's meta; the requests
the middleware wraps (route matched, status known) and the caller asked a line for (kind GOFR_LOG_REQUEST) get a LogBatch
record with that status, the batch's log time and the elapsed time; the request-log oracle writes their lines; every
other request has an empty line.  Here: the line decision's device code (batch_log_device.cuh through tests/emu) against
that rule on mixed traffic, the capacity bound on hostile strings, and the argument checks that need no GPU."""
import ctypes as C

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from tests import oracle as O
from tests.emu import emu_batch_log

DATE = S.http_date(1_700_000_000)
LOG_NS = 1_700_000_000_123_456_789
ITEM = S.Schema(7, "main.Item", [S.Field("SKU", S.F_STRING, "sku"), S.Field("Qty", S.F_INT32, "qty")])


def mixed_spec(defaults: bool = True, stage2: bool = False) -> S.TableSpec:
    """config 1's routes plus a panicking handler, Bind and a closure result route.  stage2: the GOFR_H_HOST routes are
    GOFR_H_RESULT routes (the closures have run: stage 2 of the split API), so their former holes get statuses."""
    host = S.H_RESULT if stage2 else S.H_HOST
    return S.TableSpec(schemas=[ITEM], default_routes=defaults, routes=[
        S.Route(S.M_GET, "/hello", S.H_PARAM_FORMAT, s0=b"name", s1=b"World", s2=b"Hello ", s3=b"!"),
        S.Route(S.M_GET, "/error", S.H_STATIC_ERROR, s0=b"some error occurred"),
        S.Route(S.M_GET, "/redis", host, schema_id=7 if stage2 else 0),
        S.Route(S.M_GET, "/trace", host, schema_id=7 if stage2 else 0),
        S.Route(S.M_GET, "/panic", S.H_PANIC),
        S.Route(S.M_POST, "/items", S.H_BIND_ECHO, schema_id=7),
    ])


def mixed_requests(n: int, seed: int = 1, stage2: bool = False, long_every: int = 0):
    """n requests drawn from every kind of answer: handlers, OPTIONS (CORS), HEAD, catch-all / mux 404, 405, cleanPath
    301, health, panics, Bind successes and errors, and the GOFR_H_HOST routes (stage2: their closures' results)"""
    rng = np.random.default_rng(seed)
    row = ITEM.encode_row(["A-1", 3])
    hole = S.result_record(S.RESULT_DATA, row) if stage2 else b""
    kinds = [S.Req(S.M_GET, b"/hello"), S.Req(S.M_GET, b"/hello", b"name=gofr"), S.Req(S.M_OPTIONS, b"/hello"),
             S.Req(S.M_HEAD, b"/hello"), S.Req(S.M_GET, b"/nowhere"), S.Req(S.M_POST, b"/hello"),
             S.Req(S.M_GET, b"/hello/../hello"), S.Req(S.M_GET, b"//hello"), S.Req(S.M_GET, b"/.well-known/health"),
             S.Req(S.M_GET, b"/error"), S.Req(S.M_GET, b"/panic"), S.Req(S.M_POST, b"/items", data=b'{"sku":"x","qty":2}'),
             S.Req(S.M_POST, b"/items", data=b'{"sku":1}'), S.Req(S.M_POST, b"/items", data=b'{"qty":'),
             S.Req(S.M_GET, b"/redis", data=hole), S.Req(S.M_GET, b"/trace", data=hole)]
    reqs = []
    for i in range(n):
        r = kinds[int(rng.integers(len(kinds)))]
        if long_every and i % long_every == 0:
            r = S.Req(S.M_GET, b"/hello", b"name=" + b"n" * 1500)
        reqs.append(S.Req(r.method, r.path, r.query, r.data))
    b = S.RequestBatch.pack(reqs)
    b.trace_ids[:] = synth.trace_ids(seed, np.arange(n))
    return b


def log_records(n: int, seed: int = 1, none_every: int = 5, hostile_every: int = 7) -> S.LogBatch:
    """config-2 log strings (synth.reqlog_batch) with some hostile ones; every none_every-th record asks for no line.
    The clock and status fields are garbage: the call fills them."""
    lb = synth.reqlog_batch(n, seed=seed, hostile_every=hostile_every)
    if none_every:
        lb.desc["kind"][::none_every] = S.LOG_NONE
    lb.desc["status"] = 999
    lb.desc["log_unix_ns"] = -5
    lb.desc["elapsed_ns"] = 77
    return lb


def admitted(meta: np.ndarray, kind: np.ndarray) -> np.ndarray:
    """include/gofr_b200.h: a line exactly when a matched route answered, the status is known and a line was asked for"""
    return ((meta >> 16) != 0xFFFF) & ((meta & 0xFFFF) != 0) & (kind == S.LOG_REQUEST)


def expectation(spec: S.TableSpec, batch: S.RequestBatch, log: S.LogBatch, log_ns: int = LOG_NS, date: bytes = DATE):
    """(responses, meta, lines): the serving oracle's answers and every request's line (b"" when it has none)"""
    out, off, meta = O.OracleTable(spec).serve(batch, date)
    sel = np.nonzero(admitted(meta, log.desc["kind"]))[0]
    d = log.desc[sel].copy()
    d["status"] = meta[sel] & 0xFFFF
    d["log_unix_ns"] = log_ns
    d["elapsed_ns"] = log_ns - d["start_unix_ns"]
    lines = [b""] * batch.n
    if len(sel):
        lo, lf = O.request_log(S.LogBatch(d, batch.trace_ids[sel].copy(), log.arena))
        for j, i in enumerate(sel.tolist()):
            lines[i] = lo[int(lf[j]):int(lf[j + 1])].tobytes()
    return O.responses(out, off), meta, lines


@pytest.mark.parametrize("defaults,stage2", [(True, False), (False, False), (True, True)])
def test_emu_line_decision_matches_rule(defaults, stage2):
    n = 3000
    spec, batch, log = mixed_spec(defaults, stage2), mixed_requests(n, seed=3, stage2=stage2), log_records(n, seed=3)
    _, meta, want = expectation(spec, batch, log)
    d, has = emu_batch_log.fill(log.desc, meta, LOG_NS)
    assert (has == admitted(meta, log.desc["kind"])).all()
    assert has.any() and (~has).any()
    assert (d["status"][has] == meta[has] & 0xFFFF).all() and (d["log_unix_ns"][has] == LOG_NS).all()
    assert (d["elapsed_ns"][has] == LOG_NS - d["start_unix_ns"][has]).all()
    assert (d[~has] == log.desc[~has]).all()    # a request without a line keeps its record untouched
    sel = np.nonzero(has)[0]
    lo, lf = O.request_log(S.LogBatch(d[sel].copy(), batch.trace_ids[sel].copy(), log.arena))
    got = [lo[int(lf[j]):int(lf[j + 1])].tobytes() for j in range(len(sel))]
    assert got == [want[i] for i in sel.tolist()]
    assert all(want[i] == b"" for i in np.nonzero(~has)[0].tolist())
    # the traffic covers the cases the rule tells apart
    st, rt = meta & 0xFFFF, meta >> 16
    assert (rt == 0xFFFF).any() and (st == 0).any() != stage2 and ((log.desc["kind"] == S.LOG_NONE) & (rt != 0xFFFF)).any()


def _bound(desc) -> int:
    cap = C.c_uint64()
    _abi.check(_abi.lib().gofr_batch_log_bound(desc.ctypes.data, len(desc), C.byref(cap)), "gofr_batch_log_bound")
    return int(cap.value)


def test_bound_covers_hostile_lines():
    worst = [b"\x01" * 65535, b"<" * 65535, b"\xff" * 65535, b"\xe2\x80\xa8" * 21845, b'"\\' * 32767]
    recs = []
    for k, s in enumerate(worst):
        recs.append(S.LogRec(-1, -999_999_999_999, 4_102_444_799_999_999_999, s, s, s, s, s, 65535,
                             -(12 * 3600 + 59 * 60 + 59)))
        recs.append(S.LogRec(1, 2, 3, b"GET", b"", b" , ".join([b"10.0.0.%d" % j for j in range(5000)])[:65535], b"", s, 404))
    recs.append(S.LogRec(0, 0, 0, b"", b"", b"", b"", b"", 0))
    lb = S.LogBatch.pack(recs)
    lo, lf = O.request_log(lb)
    lens = np.diff(lf.astype(np.int64))
    strings = lb.desc[["method_len", "ua_len", "xff_len", "remote_len", "uri_len"]]
    per = np.array([320 + 6 * sum(int(x) for x in r) for r in strings.tolist()])
    assert (lens <= per).all()
    assert _bound(lb.desc) == per.sum() >= lens.sum()
    # records that ask for no line take no room
    lb.desc["kind"][1::2] = S.LOG_NONE
    assert _bound(lb.desc) == per[0::2].sum()


def test_argument_errors_without_gpu():
    L = _abi.lib()
    cap = C.c_uint64()
    assert L.gofr_batch_log_bound(None, 1, C.byref(cap)) == 1
    assert L.gofr_batch_log_bound(None, 0, None) == 1
    assert L.gofr_batch_log_bound(None, 0, C.byref(cap)) == 0 and cap.value == 0
    rb, ob, sb, lb = _abi.ReqBatch(), _abi.RespBatch(), _abi.SlotBatch(), _abi.BatchLog()
    t = C.c_uint64()
    assert L.gofr_batch_submit_log(None, C.byref(rb), C.byref(ob), C.byref(lb), C.byref(t)) == 1
    assert L.gofr_batch_submit_slots_log(None, C.byref(rb), C.byref(sb), C.byref(lb), C.byref(t)) == 1
    assert L.gofr_frontend_set_log_clock(None, 5) == 1
    n = C.c_uint32()
    assert L.gofr_frontend_serve_log(None, 0, b"/", 1, b"", 0, 0, b"", 0, b"\0" * 16, None, None, None, 0, C.byref(n), None,
                                     None, 0, C.byref(n)) == 1
    assert L.gofr_frontend_create_log(None, None, 1, 1, 16, 16, 16) == 1


def test_abi_layout():
    assert C.sizeof(_abi.BatchLog) == 72
    assert _abi.BatchLog.lines.offset == 56 and _abi.BatchLog.out_bytes.offset == 64


@pytest.mark.parametrize("args", ["16 200 8 100", "32 100 64 50", "8 100 1 0"])
def test_frontend_log_fan_in_fan_out_tsan(args):
    """no GPU: the log front-end's batching (frontend.cpp) against a stub engine under ThreadSanitizer — callers mixing
    serve and serve_log each get their own response and line, a batch without a logging caller takes the plain call, a
    line longer than line_cap is reported with its length, nothing races."""
    import json
    import os
    import subprocess
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
    exe = os.path.join(here, "frontend_log_stress")
    srcs = [os.path.join(here, "frontend_log_stress.cpp"), os.path.join(here, "..", "..", "gofr_b200", "csrc", "frontend.cpp")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-Wall", srcs[0], "-o", exe],
                              cwd=here)
    r = subprocess.run([exe] + args.split(), capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ThreadSanitizer" not in r.stderr, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    t, n, _ = (int(v) for v in args.split()[:3])
    assert res["bad"] == 0 and res["requests"] == t * n and res["log_batches"] > 0
