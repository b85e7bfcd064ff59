"""The gRPC LoggingInterceptor's RPCLog line for every call of a proto encode batch (gofr_proto_batch_encode_log) and through
the per-message front-end (gofr_proto_frontend_call_log), CPU side.

The expectation composes oracles the project already checks: a call whose record says GOFR_LOG_RPC gets the request-log
oracle's line for that record with the batch's log time (its start, elapsed time, zone and method are the caller's, its id
the span's trace id); a GOFR_LOG_NONE record gets an empty line; the response row and its encoding do not matter.  Here:
the line decision's device code (batch_log_device.cuh through tests/emu) against that rule, gofr_batch_log_bound against
the oracle's line lengths at their worst, the argument checks that need no GPU, and the front-end's log staging against
stub batch calls under ThreadSanitizer."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from tests import oracle as O
from tests.emu import emu_proto_log

LOG_NS = 1_700_000_000_123_456_789
METHOD = b"/Hello/SayHello"
HOSTILE = [b'/pkg.Svc/"quoted"\\', b"/a\x01\x1f\x7f/b", b"/\xff\xfe\xc0\xaf", b"/\xe2\x80\xa8\xe2\x80\xa9",
           b"/<html>&amp;", b"/\t\r\n", "/ünïcödé/日本".encode(), b""]
MAX_RESPONSE_TIME = -(2 ** 63)                 # time.Since(start) at its most negative: 17 characters of microseconds
# The clock fields are int64 nanoseconds, which reach the years 1677 and 2262 and no further: years 0 and 9999 are not on
# this clock, and a year always takes four digits.  These are its extremes.
CLOCK_MIN, CLOCK_MAX = -(2 ** 63), 2 ** 63 - 1


def rpc_records(n: int, seed: int = 1, none_every: int = 5, hostile_every: int = 7) -> S.LogBatch:
    """n RPC log records: /Hello/SayHello, and every hostile_every-th one a hostile method; every none_every-th record asks
    for no line.  status and log_unix_ns are garbage: the call ignores the first and fills the second."""
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(n):
        m = HOSTILE[i // hostile_every % len(HOSTILE)] if hostile_every and i % hostile_every == 0 else METHOD
        start = LOG_NS - int(rng.integers(0, 5_000_000_000))
        recs.append(S.LogRec(start, int(rng.integers(-10, 10 ** 12)), -5, m, b"ua", b"xff", b"remote", b"/uri", 999,
                             int(rng.integers(-14 * 3600, 14 * 3600)),
                             kind=S.LOG_NONE if none_every and i % none_every == 0 else S.LOG_RPC))
    return S.LogBatch.pack(recs, seed=seed)


def oracle_lines(lb: S.LogBatch):
    """the request-log oracle's line for every record of lb, as it is (orc_reqlog.c), with room for twice-escaped methods"""
    n = lb.n
    if n == 0:
        return []
    cap = 400 * n + 7 * int(lb.arena.size) + 64
    out, off = np.zeros(cap, np.uint8), np.zeros(n + 1, np.uint32)
    arena = lb.arena if lb.arena.size else np.zeros(1, np.uint8)
    assert O.lib().orc_request_log(lb.desc.ctypes.data, lb.trace_ids.ctypes.data, arena.ctypes.data, n, out.ctypes.data, cap,
                                   off.ctypes.data) == 0
    return [out[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)]


def expectation(log: S.LogBatch, log_ns: int = LOG_NS):
    """every record's line under gofr_proto_batch_encode_log's rule (b"" when it has none)"""
    sel = np.nonzero(log.desc["kind"] == S.LOG_RPC)[0]
    lines = [b""] * log.n
    if len(sel):
        d = log.desc[sel].copy()
        d["log_unix_ns"] = log_ns
        for j, line in zip(sel.tolist(), oracle_lines(S.LogBatch(d, log.trace_ids[sel].copy(), log.arena))):
            lines[j] = line
    return lines


def test_emu_line_decision_matches_rule():
    log = rpc_records(3000, seed=3)
    d, has = emu_proto_log.fill(log.desc, LOG_NS)
    rpc = log.desc["kind"] == S.LOG_RPC
    assert (has == rpc).all() and has.any() and (~has).any()
    assert (d["log_unix_ns"][has] == LOG_NS).all()
    # elapsed_ns is the caller's, the status is nobody's business: both stay as they came
    assert (d["elapsed_ns"] == log.desc["elapsed_ns"]).all() and (d["status"] == log.desc["status"]).all()
    assert (d[~has] == log.desc[~has]).all()
    # whatever the status field holds, the same calls get lines
    other = log.desc.copy()
    other["status"] = np.arange(log.n) % 600
    assert (emu_proto_log.fill(other, LOG_NS)[1] == has).all()
    # the filled records are exactly what the oracle's lines are made from
    sel = np.nonzero(has)[0]
    want = expectation(log)
    assert oracle_lines(S.LogBatch(d[sel].copy(), log.trace_ids[sel].copy(), log.arena)) == [want[i] for i in sel.tolist()]
    assert all(want[i] == b"" for i in np.nonzero(~has)[0].tolist())


def test_emu_other_kinds_get_no_line():
    log = rpc_records(8, seed=4, none_every=0)
    log.desc["kind"] = [S.LOG_REQUEST, S.LOG_NONE, 3, 0xFFFFFFFF, S.LOG_RPC, S.LOG_REQUEST, S.LOG_RPC, S.LOG_NONE]
    _, has = emu_proto_log.fill(log.desc, LOG_NS)
    assert has.tolist() == [False, False, False, False, True, False, True, False]


def _bound(desc) -> int:
    cap = C.c_uint64()
    _abi.check(_abi.lib().gofr_batch_log_bound(desc.ctypes.data, len(desc), C.byref(cap)), "gofr_batch_log_bound")
    return int(cap.value)


def _extreme_records(method: bytes):
    """RPC records of one method at the clock's extremes: the largest responseTime, zone offsets across the whole range,
    and log and start times at both ends of the clock (with nine fraction digits, the longest time text)"""
    recs = []
    zones = [-(23 * 3600 + 59 * 60 + 59), -(12 * 3600 + 59 * 60 + 59), -3600 - 1, -1, 0, 1, 5 * 3600 + 45 * 60, 14 * 3600,
             23 * 3600 + 59 * 60 + 59]
    for tz in zones:
        for start, log_ns in [(CLOCK_MIN + 86400 * 10 ** 9 + 1, CLOCK_MIN + 86400 * 10 ** 9 + 3),
                              (CLOCK_MAX - 86400 * 10 ** 9, CLOCK_MAX - 86400 * 10 ** 9 + 1), (1, -1)]:
            recs.append(S.LogRec(start, MAX_RESPONSE_TIME, log_ns, method, tz_offset_s=tz, kind=S.LOG_RPC))
    recs.append(S.LogRec(CLOCK_MAX - 86400 * 10 ** 9, CLOCK_MAX, 123_456_789, method, kind=S.LOG_RPC))
    return recs


@pytest.mark.parametrize("method", [b"", b"\x01" * 65535, b"<" * 65535, b"\xff" * 65535, b"\xe2\x80\xa8" * 21845,
                                    b'"\\' * 32767, b"\n" * 65535, b"/Hello/SayHello"],
                         ids=["empty", "ctrl", "lt", "invalid_utf8", "u2028", "quote_backslash", "newline", "plain"])
def test_bound_covers_rpc_lines(method):
    """every line no longer than its record's share of gofr_batch_log_bound, and the fixed part within 320 bytes, at the
    worst method bytes and the clock's extremes (a method of 0x01 bytes needs 7 per byte: 6 would not do)"""
    lb = S.LogBatch.pack(_extreme_records(method))
    lens = np.array([len(x) for x in oracle_lines(lb)])
    per = np.array([_bound(lb.desc[i:i + 1]) for i in range(lb.n)])
    assert (per == 320 + 7 * len(method) + 6 * len(b"/")).all()   # LogRec's default uri: checked, counted, not logged
    assert (lens <= per).all(), (lens.max(), per.max())
    assert _bound(lb.desc) == per.sum()
    if method == b"":
        assert lens.max() <= 320
    # the RPCLog fixed part alone: the same records with the method gone
    d = lb.desc.copy()
    d["method_len"] = 0
    assert max(len(x) for x in oracle_lines(S.LogBatch(d, lb.trace_ids, lb.arena))) <= 320


def test_bound_unchanged_for_request_and_none_records():
    recs = [S.LogRec(1, 2, 3, b"\x01" * 1000, b"u" * 10, b"x" * 20, b"r" * 30, b"/" * 40, 200),
            S.LogRec(1, 2, 3, b"GET", kind=S.LOG_NONE), S.LogRec(1, 2, 3, b"POST", b"", b"", b"", b"/a", 404)]
    lb = S.LogBatch.pack(recs)
    assert _bound(lb.desc) == (320 + 6 * 1100) + 0 + (320 + 6 * 6)
    lb.desc["kind"][0] = S.LOG_RPC
    assert _bound(lb.desc) == (320 + 6 * 1100 + 1000) + (320 + 6 * 6)


def test_argument_errors_without_gpu():
    L = _abi.lib()
    pb, ob, lb = _abi.ProtoBatch(), _abi.RespBatch(), _abi.BatchLog()
    t = C.c_uint64()
    nm, nf, k = S.proto_nested_tables([[S.ProtoNField(1, S.PB_STRING)]])
    ids = (C.c_uint8 * 16)()
    assert L.gofr_proto_batch_encode_log(None, nm.ctypes.data, 1, nf.ctypes.data, k, 0, None, C.byref(pb), ids, C.byref(ob),
                                         C.byref(lb), C.byref(t)) == 1
    assert L.gofr_proto_batch_encode_log(None, nm.ctypes.data, 1, nf.ctypes.data, k, 0, None, C.byref(pb), ids, C.byref(ob),
                                         None, C.byref(t)) == 1
    f = C.c_void_p()
    assert L.gofr_proto_frontend_create_log(C.byref(f), None, nm.ctypes.data, 1, nf.ctypes.data, k, 0, None, 0, 1, 1, 16, 16) == 1
    assert L.gofr_proto_frontend_set_log_clock(None, 5) == 1
    n, st, ln = C.c_uint32(), C.c_uint32(), C.c_uint32()
    d = np.zeros(1, S.LOG_DESC_DTYPE)
    assert L.gofr_proto_frontend_call_log(None, b"", 0, b"\0" * 16, d.ctypes.data, b"", None, 0, C.byref(n), C.byref(st), None,
                                          0, C.byref(ln)) == 1


@pytest.mark.parametrize("args", ["16 200 8 100", "32 100 64 50", "8 100 1 0"])
def test_proto_frontend_log_fan_in_fan_out_tsan(args):
    """no GPU: the encode front-end's log staging (proto_frontend.cpp) against stub batch calls under ThreadSanitizer —
    callers mixing call, call_log and log-only calls (an empty row: the handler failed) each get their own message and
    line, a batch without a logging caller takes the plain call, a line longer than line_cap is reported with its length,
    a decode front-end takes no log staging, nothing races."""
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
    exe = os.path.join(here, "proto_frontend_log_stress")
    srcs = [os.path.join(here, "proto_frontend_log_stress.cpp"),
            os.path.join(here, "..", "..", "gofr_b200", "csrc", "proto_frontend.cpp"),
            os.path.join(here, "..", "..", "gofr_b200", "csrc", "frontend_ring.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-Wall", srcs[0], "-o", exe],
                              cwd=here)
    r = subprocess.run([exe] + args.split(), capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ThreadSanitizer" not in r.stderr, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    t, n = (int(v) for v in args.split()[:2])
    assert res["bad"] == 0 and res["violations"] == 0 and res["calls"] == t * n
    assert res["log_batches"] > 0 and res["failed"] > 0 and res["short"] > 0
