"""middleware.Logging's RequestLog line for every request served from connection buffers (gofr_conn_batch_submit_log).

The model composes oracles the project already checks, none of them device code: the framer's oracle → drop the tails →
the request-head oracle (its spans) → the serving oracle (meta) → keep the requests Logging runs for and whose status is
known (route matched, status != 0) → a LogBatch of their spans, remote strings and clocks → the request-log oracle.
CPU: the gather's device code (conn_log_device.cuh through tests/emu) against the model, the line set against the
X-Correlation-Id headers of the oracle's responses, the capacity bound, the ABI layout and the argument checks.  GPU: every
log column and the responses against the model across tables, chunk sizes, caller memory kinds, hostile strings and
capacities, the launches without a log, and the device-resident chain."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.engine import ConnLog, conn_log_bound
from tests import oracle as O
from tests import test_conn_batch as CB
from tests.emu import emu_conn_log

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATE = CB.DATE
LOG_NS = 1_700_000_000_123_456_789
TZ = 3600 + 30 * 60
SEED = 0xC0FFEE


# ---- the model ----
def logged(meta: np.ndarray, spans: np.ndarray) -> np.ndarray:
    """include/gofr_b200.h: a device line for route matched, status known, and method, User-Agent, X-Forwarded-For and
    target each at most 65535 bytes (spans: the request heads' spans, one row per request)"""
    lens = spans[:, [S_METHOD, S_UA, S_XFF, S_TARGET]] >> np.uint64(32)
    return ((meta >> 16) != 0xFFFF) & ((meta & 0xFFFF) != 0) & (lens <= 0xFFFF).all(axis=1)


def model(spec, buf, off, seed, remote, remote_off, start, log_ns=LOG_NS, tz=TZ):
    """the response columns of test_conn_batch's model, plus the log: (dict, LogBatch of the logged requests)"""
    rec, first, consumed, status, idx, req_first, ids = CB.model_requests(buf, off, seed)
    d, a, s, spans = O.http_parse(buf, rec)
    o, f, m = O.OracleTable(spec).serve(S.RequestBatch(d[idx].copy(), ids, a), DATE)
    n = len(off) - 1
    conn = np.repeat(np.arange(n), np.diff(req_first.astype(np.int64)))
    sel = np.nonzero(logged(m, spans[idx]))[0]
    b, rb = buf.tobytes(), remote.tobytes()
    recs = []
    for k in sel.tolist():
        sp = spans[idx[k]]
        get = lambda j: b[int(sp[j] & 0xFFFFFFFF):int(sp[j] & 0xFFFFFFFF) + int(sp[j] >> 32)]
        c = int(conn[k])
        recs.append(S.LogRec(int(start[c]), log_ns - int(start[c]), log_ns, get(S_METHOD), get(S_UA), get(S_XFF),
                             rb[int(remote_off[c]):int(remote_off[c + 1])], get(S_TARGET), int(m[k] & 0xFFFF), tz, ids[k].tobytes()))
    lb = S.LogBatch.pack(recs)
    lo, lf = O.request_log(lb)
    want = dict(out=o[:int(f[-1])], out_off=f, meta=m, req_at=rec[idx].astype(np.uint32), trace_ids=ids, req_first=req_first,
                consumed=consumed, conn_status=status, log=lo[:int(lf[-1])], log_off=lf, log_req=sel.astype(np.uint32))
    return want, lb


S_METHOD, S_TARGET, S_UA, S_XFF = 0, 1, 2, 3


def _clients(n, seed=synth.SEED, edge=True):
    """seeded remote addresses and clocks; with edge, some remote strings of 0 and of 255 bytes"""
    remote, roff, start = synth.conn_clients(n, seed)
    if not edge:
        return remote, roff, start
    strs = [remote[roff[c]:roff[c + 1]].tobytes() for c in range(n)]
    for c in range(0, n, 9):
        strs[c] = b""
    for c in range(4, n, 13):
        strs[c] = (b"[fe80::%x%%eth0]:" % c + b"9" * 255)[:255]
    remote = np.frombuffer(b"".join(strs) or b"\0", np.uint8)[:sum(map(len, strs))].copy()
    return remote, np.cumsum([0] + [len(x) for x in strs]).astype(np.uint32), start


# requests mux answers itself, without middleware: a cleanPath 301 and a 405
UNROUTED = [b"GET /x/../hello HTTP/1.1\r\nHost: h\r\n\r\n", b"PUT /hello HTTP/1.1\r\nHost: h\r\nContent-Length: 0\r\n\r\n"]


def _streams(n, seed=synth.SEED, **kw):
    """test_conn_batch's streams with holes (config 1's /redis) and requests mux answers without middleware among the
    directed messages"""
    msgs = UNROUTED * 3 + [CB.HOLE] * 3 + [m for m, _ in CB.GOOD] + CB.DEFERRED + CB.BIG
    return synth.http_streams(n, seed=seed, tail_every=kw.pop("tail_every", 5), defer_every=kw.pop("defer_every", 11),
                              seed_msgs=msgs, **kw)


# served requests whose User-Agent or X-Forwarded-For value is longer than gofr_log_desc's 16-bit lengths: no device line
LONG = [b"GET /hello HTTP/1.1\r\nHost: h\r\nUser-Agent: " + b"u" * 70000 + b"\r\n\r\n",
        b"GET /hello HTTP/1.1\r\nHost: h\r\nX-Forwarded-For: " + b"1" * 70000 + b", 10.0.0.1\r\n\r\n",
        b"GET /hello HTTP/1.1\r\nHost: h\r\nUser-Agent: " + b"v" * 65535 + b"\r\n\r\n"]


def _long_streams():
    return synth.http_streams(600, seed=5, tail_every=5, defer_every=11, seed_msgs=LONG)


def _log(remote, roff, start, **kw):
    return ConnLog(remote, roff, start, LOG_NS, TZ, **kw)


# ---- CPU ----
def _emu_chunk(spec, buf, off, seed, remote, roff, start, lo, hi):
    """the gather's device code over connections [lo, hi) as the engine stages them: (desc, ids, log_req, arena)"""
    rec, first, _, status, idx, req_first, ids = CB.model_requests(buf, off, seed)
    d, a, _, spans = O.http_parse(buf, rec)
    _, _, meta = O.OracleTable(spec).serve(S.RequestBatch(d[idx].copy(), ids, a), DATE)
    alo = int(off[lo]) & ~15
    k0, k1, r0 = int(req_first[lo]), int(req_first[hi]), int(first[lo])
    g = emu_conn_log.gather(first[lo:hi + 1] - first[lo], status[lo:hi], req_first[lo:hi + 1], rec[r0:], spans[r0:], meta[k0:k1],
                            ids[k0:k1], buf[alo:int(off[hi]) + 16], alo, remote, roff[lo:hi + 1], start[lo:hi], LOG_NS, TZ, k0)
    return g


def _check_gathered(g, lb, sel):
    """the gather's lines against the model's LogBatch: every field but arena_off, the five strings, ids, request indices
    and the formatted lines"""
    desc, ids, req, _, arena = g
    assert np.array_equal(req, sel)
    assert np.array_equal(ids, lb.trace_ids)
    fields = [f for f in S.LOG_DESC_DTYPE.names if f != "arena_off"]
    for f in fields:
        assert np.array_equal(desc[f], lb.desc[f]), f
    lens = ("method_len", "ua_len", "xff_len", "remote_len", "uri_len")
    total = sum(desc[f].astype(np.int64) for f in lens)
    ab, mb = arena.tobytes(), lb.arena.tobytes()
    for m in range(len(desc)):
        a0, b0 = int(desc["arena_off"][m]), int(lb.desc["arena_off"][m])
        assert ab[a0:a0 + int(total[m])] == mb[b0:b0 + int(total[m])], m
    got = O.request_log(S.LogBatch(desc.copy(), ids.copy(), arena))
    want = O.request_log(lb)
    assert got[0][:int(got[1][-1])].tobytes() == want[0][:int(want[1][-1])].tobytes() and np.array_equal(got[1], want[1])


def test_gather_device_code_equals_model():
    """config 1 (holes: /redis is GOFR_H_HOST) and config 2; empty connections, MORE / DEFER tails, remote strings of 0 and
    255 bytes; the whole batch as one chunk and a chunk that starts at a later connection"""
    for spec, holes in ((synth.config1_spec(), True), (synth.config2_spec(), False)):
        for kw in ({}, {"tail_every": 3, "defer_every": 7}, {"reqs": (1, 1)}):
            buf, off = _streams(3000, **kw)
            off = np.concatenate([off[:1400], np.full(130, off[1399], np.uint32), off[1400:], np.full(5, off[-1], np.uint32)])
            n = len(off) - 1
            remote, roff, start = _clients(n)
            want, lb = model(spec, buf, off, SEED, remote, roff, start)
            if holes:
                assert ((want["meta"] & 0xFFFF) == 0).sum() > 0 and ((want["meta"] >> 16) == 0xFFFF).sum() > 0
            g = _emu_chunk(spec, buf, off, SEED, remote, roff, start, 0, n)
            _check_gathered(g, lb, want["log_req"])
            # a later chunk: connections 517.. of the same batch give the same lines as the batch gives them
            lo = 1517
            k0 = int(want["req_first"][lo])
            g = _emu_chunk(spec, buf, off, SEED, remote, roff, start, lo, n)
            m0 = int(np.searchsorted(want["log_req"], k0))
            sub = S.LogBatch(lb.desc[m0:].copy(), lb.trace_ids[m0:].copy(), lb.arena)
            _check_gathered(g, sub, want["log_req"][m0:])


def test_long_strings_have_no_device_line():
    """a User-Agent or X-Forwarded-For value longer than 65535 bytes: the request is served, and it has no device line
    (the host logs it); one of exactly 65535 bytes is logged in full.  The gather's device code agrees"""
    spec = synth.config1_spec()
    buf, off = _long_streams()
    remote, roff, start = _clients(len(off) - 1)
    want, lb = model(spec, buf, off, SEED, remote, roff, start)
    rec, _, _, _, idx, _, _ = CB.model_requests(buf, off, SEED)
    _, _, _, spans = O.http_parse(buf, rec)
    ln = spans[idx] >> np.uint64(32)
    long_ = (ln[:, S_UA] > 0xFFFF) | (ln[:, S_XFF] > 0xFFFF)
    assert long_.sum() >= 4 and (want["meta"][long_] & 0xFFFF == 200).all()
    assert not np.isin(np.nonzero(long_)[0], want["log_req"]).any()
    assert (lb.desc["ua_len"] == 65535).sum() >= 2
    _check_gathered(_emu_chunk(spec, buf, off, SEED, remote, roff, start, 0, len(off) - 1), lb, want["log_req"])


def test_line_set_is_the_correlation_header_set():
    """independently of meta: a request has a line exactly when the oracle's response carries an X-Correlation-Id header,
    and the line's id is that header's value"""
    for spec, holes in ((synth.config1_spec(), True), (synth.config2_spec(), False)):
        buf, off = _streams(1200, seed=3)
        remote, roff, start = _clients(len(off) - 1)
        want, lb = model(spec, buf, off, SEED, remote, roff, start)
        resp = O.responses(want["out"], want["out_off"])
        has = []
        for k, r in enumerate(resp):
            head = r.split(b"\r\n\r\n", 1)[0]
            vals = [ln[len(b"X-Correlation-Id: "):] for ln in head.split(b"\r\n") if ln.startswith(b"X-Correlation-Id: ")]
            if vals:
                has.append(k)
                m = int(np.searchsorted(want["log_req"], k))
                assert m < len(want["log_req"]) and want["log_req"][m] == k
                line = want["log"][int(want["log_off"][m]):int(want["log_off"][m + 1])].tobytes()
                assert b'"id":"' + vals[0] + b'"' in line, k
        assert np.array_equal(np.array(has, np.uint32), want["log_req"])


def test_bound_covers_what_the_model_needs():
    """gofr_conn_log_bound against the lines and bytes the model needs, on the seeds of the response bound's test"""
    for spec in (synth.config1_spec(), synth.config2_spec()):
        for seed in range(12):
            buf, off = _streams(250, seed=seed, reqs=(0, 4))
            remote, roff, start = _clients(len(off) - 1, seed=seed)
            want, _ = model(spec, buf, off, seed, remote, roff, start)
            line_cap, out_cap = conn_log_bound(off, roff)
            assert line_cap >= len(want["log_req"]) and out_cap >= int(want["log_off"][-1]), seed
    lc, oc = conn_log_bound(np.array([0, 100, 100, 116], np.uint32), np.array([0, 255, 255, 256], np.uint32))
    assert lc == (100 // 16 + 1) + 1 + 2 and oc == lc * 320 + 6 * (116 + 7 * 255 + 2 * 1)


def _c_layout():
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "gofr_b200.h"
#define F(T, f) printf(#T " " #f " %zu\n", offsetof(T, f));
int main(void) {
    printf("gofr_conn_log size %zu\n", sizeof(gofr_conn_log));
    F(gofr_conn_log, remote) F(gofr_conn_log, remote_off) F(gofr_conn_log, start_unix_ns) F(gofr_conn_log, log_unix_ns)
    F(gofr_conn_log, tz_offset_s) F(gofr_conn_log, line_cap) F(gofr_conn_log, out) F(gofr_conn_log, out_cap)
    F(gofr_conn_log, log_off) F(gofr_conn_log, log_req) F(gofr_conn_log, lines) F(gofr_conn_log, reserved)
    F(gofr_conn_log, out_bytes)
    return 0;
}
"""
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "l.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "l"), os.path.join(d, "l.c")])
        return subprocess.run([os.path.join(d, "l")], capture_output=True, text=True, check=True).stdout.split("\n")


def test_abi_layout_matches_ctypes():
    lines = [ln.split() for ln in _c_layout() if ln]
    for name, field, value in lines:
        if field == "size":
            assert C.sizeof(_abi.ConnLog) == int(value)
        else:
            assert getattr(_abi.ConnLog, field).offset == int(value), field
    assert sum(1 for ln in lines if ln[1] != "size") == len(_abi.ConnLog._fields_)


def test_invalid_arguments_without_a_gpu():
    L = _abi.lib()
    off = np.array([0, 40], np.uint32)
    buf = np.zeros(40, np.uint8)
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=40, n_conns=1, date=DATE, trace_seed=1)
    cr, cl, t = _abi.ConnResp(), _abi.ConnLog(), C.c_uint64()
    for n in (0, 1):
        cb.n_conns = n
        assert L.gofr_conn_batch_submit_log(None, C.byref(cb), C.byref(cr), C.byref(cl), C.byref(t)) == 1
        assert L.gofr_conn_batch_submit_log(None, C.byref(cb), C.byref(cr), None, C.byref(t)) == 1
    assert L.gofr_conn_batch_submit_log(None, None, None, None, None) == 1
    # the bound: null arguments, decreasing offsets, a remote string of 256 bytes
    roff = np.array([0, 7], np.uint32)
    lc, oc = C.c_uint32(), C.c_uint64()
    assert L.gofr_conn_log_bound(None, roff.ctypes.data, 1, C.byref(lc), C.byref(oc)) == 1
    assert L.gofr_conn_log_bound(off.ctypes.data, None, 1, C.byref(lc), C.byref(oc)) == 1
    assert L.gofr_conn_log_bound(off.ctypes.data, roff.ctypes.data, 1, None, C.byref(oc)) == 1
    bad = np.array([0, 40, 39], np.uint32)
    assert L.gofr_conn_log_bound(bad.ctypes.data, np.array([0, 1, 2], np.uint32).ctypes.data, 2, C.byref(lc), C.byref(oc)) == 1
    for r in ([0, 5, 4], [0, 0, 256]):
        ra = np.array(r, np.uint32)
        assert L.gofr_conn_log_bound(np.array([0, 20, 40], np.uint32).ctypes.data, ra.ctypes.data, 2, C.byref(lc), C.byref(oc)) == 1
    assert L.gofr_conn_log_bound(np.array([0, 20, 40], np.uint32).ctypes.data, np.array([0, 0, 255], np.uint32).ctypes.data, 2,
                                 C.byref(lc), C.byref(oc)) == 0
    assert L.gofr_conn_log_bound(None, None, 0, C.byref(lc), C.byref(oc)) == 0 and lc.value == 0 and oc.value == 0


# ---- GPU ----
LOG_COLS = ("log_off", "log_req")


def _check(got, want, what=""):
    CB._check(got, want, what)
    lg = got.log
    assert lg.out.tobytes() == want["log"].tobytes(), what
    assert lg.lines == len(want["log_req"]) and lg.out_bytes == int(want["log_off"][-1]), what
    assert np.array_equal(lg.log_off, want["log_off"]) and np.array_equal(lg.log_req, want["log_req"]), what


@pytest.mark.gpu
def test_gpu_log_columns_equal_model():
    """config 1 and 2, batches around a tile, 40 000 connections with tiles of empty connections; pinned and pageable"""
    from gofr_b200.engine import Engine
    for spec, holes in ((synth.config1_spec(), True), (synth.config2_spec(), False)):
        eng = Engine(synth_table(spec), 0)
        cases = [(_streams(n, seed=n + 1), f"n={n}") for n in (1, 127, 128, 129)]
        buf, off = _streams(40000)
        off = np.concatenate([off[:20001], np.full(300, off[20000], np.uint32), off[20001:], np.full(200, off[-1], np.uint32)])
        cases.append(((buf, off), "40000"))
        for (b, o), what in cases:
            remote, roff, start = _clients(len(o) - 1)
            want, _ = model(spec, b, o, SEED, remote, roff, start)
            for pinned in (True, False):
                _check(eng.serve_connections(b, o, DATE, SEED, pinned=pinned, log=_log(remote, roff, start)), want, (what, pinned))
        got = eng.serve_connections(np.zeros(0, np.uint8), np.zeros(1, np.uint32), DATE, 1,
                                    log=_log(np.zeros(0, np.uint8), np.zeros(1, np.uint32), np.zeros(0, np.int64)))
        assert got.log.lines == 0 and got.log.out.size == 0
        eng.close()


def synth_table(spec):
    from gofr_b200.table import Table
    return Table(spec)


@pytest.mark.gpu
def test_gpu_chunk_sizes_and_a_large_connection():
    """identical outputs for every chunk size; a 9 MiB connection of pipelined requests is a chunk of its own"""
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(synth_table(spec), 0)
    buf, off = _streams(2500)
    remote, roff, start = _clients(len(off) - 1)
    want, _ = model(spec, buf, off, 42, remote, roff, start)
    for chunk in (1, 7, 1000, 65536):
        eng.set_chunk(chunk)
        for pinned in (True, False):
            _check(eng.serve_connections(buf, off, DATE, 42, pinned=pinned, log=_log(remote, roff, start)), want, (chunk, pinned))
    eng.close()
    spec = synth.config1_spec()
    eng = Engine(synth_table(spec), 0)
    buf, off = _streams(3000)
    get = b"GET /hello?name=x HTTP/1.1\r\nHost: localhost:8000\r\nUser-Agent: curl/8.4.0\r\nX-Forwarded-For: ,9.9.9.9\r\n\r\n"
    huge = np.frombuffer(get * (9 * 2**20 // len(get) + 1), np.uint8)
    cut = int(off[1500])
    buf2 = np.concatenate([buf[:cut], huge, buf[cut:]])
    off2 = np.concatenate([off[:1501], off[1500:] + np.uint32(huge.size)]).astype(np.uint32)
    remote, roff, start = _clients(len(off2) - 1)
    want, _ = model(spec, buf2, off2, 5, remote, roff, start)
    for pinned in (True, False):
        _check(eng.serve_connections(buf2, off2, DATE, 5, pinned=pinned, log=_log(remote, roff, start)), want, pinned)
    eng.close()


HOSTILE = [
    b"GET /hello?name=<b>&x=1 HTTP/1.1\r\nHost: h\r\nUser-Agent: caf\xc3\xa9 \xff\xfe\xc3 bot\r\n\r\n",
    b"GET /hello?q=a<>&b HTTP/1.1\r\nHost: h\r\nX-Forwarded-For: \xc2\xa0203.0.113.9\xe2\x80\xa8 , 10.0.0.1\r\n\r\n",
    b"GET /hello HTTP/1.1\r\nHost: h\r\nX-Forwarded-For: ,10.0.0.1\r\nUser-Agent: \xe2\x80\xa8\x80\r\n\r\n",
    b"GET /hello HTTP/1.1\r\nHost: h\r\nX-Forwarded-For:    \xe2\x80\xa8  \t\r\n\r\n",
    b"OPTIONS /hello HTTP/1.1\r\nHost: h\r\nUser-Agent: " + b"\xf0\x9f\x98\x80<&>" * 700 + b"\r\n\r\n",
    b"GET /hello?" + b"a=%3C&b=<>&" * 300 + b" HTTP/1.1\r\nHost: h\r\nUser-Agent: " + b"u" * 3000 + b"\r\n\r\n",
]


def _hostile_streams():
    return synth.http_streams(3000, seed=9, tail_every=5, defer_every=11, seed_msgs=HOSTILE + UNROUTED)


def test_hostile_streams_are_logged():
    """the hostile corpus is served and logged by the model (so the GPU test below checks what it claims to)"""
    buf, off = _hostile_streams()
    remote, roff, start = _clients(len(off) - 1, seed=9)
    want, lb = model(synth.config1_spec(), buf, off, SEED, remote, roff, start)
    log = want["log"].tobytes()
    assert (lb.desc["ua_len"] > 2000).sum() > 20 and b"\\ufffd" in log and b"\\u003c" in log and b"\\u2028" in log
    assert (lb.desc["status"] == 200).sum() > 100 and (lb.desc["remote_len"] == 0).sum() > 0 and (lb.desc["remote_len"] == 255).sum() > 0
    assert b'"ip":"203.0.113.9"' in log and b'"method":"OPTIONS"' in log


@pytest.mark.gpu
def test_gpu_hostile_strings():
    """User-Agent bytes >= 0x80 and invalid UTF-8, <>& in targets, forwarded addresses wrapped in U+00A0 / U+2028 and spaces,
    a leading comma (the remote string is used), and heads long enough that the reqlog tiles run unstaged"""
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(synth_table(spec), 0)
    buf, off = _hostile_streams()
    remote, roff, start = _clients(len(off) - 1, seed=9)
    want, _ = model(spec, buf, off, SEED, remote, roff, start)
    for pinned in (True, False):
        _check(eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, log=_log(remote, roff, start)), want, pinned)
    eng.close()


@pytest.mark.gpu
def test_gpu_long_strings_have_no_device_line():
    """User-Agent and X-Forwarded-For values past 65535 bytes: no device line, nothing wrapped; 65535 bytes: logged in full"""
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(synth_table(spec), 0)
    buf, off = _long_streams()
    remote, roff, start = _clients(len(off) - 1)
    want, _ = model(spec, buf, off, SEED, remote, roff, start)
    for chunk in (65536, 50):
        eng.set_chunk(chunk)
        for pinned in (True, False):
            _check(eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, log=_log(remote, roff, start)), want, (chunk, pinned))
    eng.close()


def _submit_log(eng, buf, off, seed, remote, roff, start, line_cap, out_cap, pinned, canary=64, log=True):
    """gofr_conn_batch_submit_log (or gofr_conn_batch_submit when not log) with the responses' bound and `canary` guard bytes
    behind each log capacity → (rc, response arrays, log arrays, ConnLog)"""
    from gofr_b200.engine import conn_batch_bound, pinned_array
    n = len(off) - 1
    alloc = (lambda c, dt: pinned_array(c * np.dtype(dt).itemsize).view(dt)) if pinned else (lambda c, dt: np.empty(c, dt))
    req_cap, rout_cap = conn_batch_bound(eng.table, off)
    a = dict(out=alloc(rout_cap + 1, np.uint8), out_off=alloc(req_cap + 1, np.uint32), meta=alloc(req_cap, np.uint32),
             req_at=alloc(req_cap, np.uint32), trace_ids=alloc(req_cap * 16, np.uint8), req_first=alloc(n + 1, np.uint32),
             consumed=alloc(n, np.uint32), conn_status=alloc(n, np.uint32))
    lg = dict(out=alloc(out_cap + canary, np.uint8), log_off=alloc(line_cap + 1 + canary, np.uint32), log_req=alloc(line_cap + canary, np.uint32))
    for v in list(a.values()) + list(lg.values()):
        v.view(np.uint8)[:] = 0xA5
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=DATE, trace_seed=seed)
    cr = _abi.ConnResp(out=a["out"].ctypes.data, out_cap=rout_cap, req_cap=req_cap, out_off=a["out_off"].ctypes.data,
                       meta=a["meta"].ctypes.data, req_at=a["req_at"].ctypes.data, trace_ids=a["trace_ids"].ctypes.data,
                       req_first=a["req_first"].ctypes.data, consumed=a["consumed"].ctypes.data, conn_status=a["conn_status"].ctypes.data)
    cl = _abi.ConnLog(remote=remote.ctypes.data, remote_off=roff.ctypes.data, start_unix_ns=start.ctypes.data, log_unix_ns=LOG_NS,
                      tz_offset_s=TZ, line_cap=line_cap, out=lg["out"].ctypes.data, out_cap=out_cap, log_off=lg["log_off"].ctypes.data,
                      log_req=lg["log_req"].ctypes.data)
    L = _abi.lib()
    t = C.c_uint64()
    if log:
        rc = L.gofr_conn_batch_submit_log(eng._e, C.byref(cb), C.byref(cr), C.byref(cl), C.byref(t))
    else:
        rc = L.gofr_conn_batch_submit(eng._e, C.byref(cb), C.byref(cr), C.byref(t))
    if rc == 0:
        rc = L.gofr_batch_wait(eng._e, t.value)
    return rc, a, lg, cl


def _responses_equal(a, want):
    k = len(want["meta"])
    assert a["out"][:len(want["out"])].tobytes() == want["out"].tobytes()
    for key in CB.COLS:
        got = a[key][:len(want[key]) * (16 if key == "trace_ids" else 1)]
        assert np.array_equal(got, want[key].reshape(-1)), key
    assert k == int(want["req_first"][-1])


@pytest.mark.gpu
def test_gpu_capacity():
    """line_cap or out_cap one short: GOFR_ERR_CAPACITY, nothing written at or past either capacity, the needed counts
    reported, and the response columns complete"""
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(synth_table(spec), 0)
    buf, off = _streams(3000)
    remote, roff, start = _clients(len(off) - 1)
    want, _ = model(spec, buf, off, 3, remote, roff, start)
    lines, nbytes = len(want["log_req"]), int(want["log_off"][-1])

    def untouched(lg, lc, oc):
        return all((v.view(np.uint8)[k:] == 0xA5).all() for v, k in ((lg["out"], oc), (lg["log_off"], 4 * (lc + 1)), (lg["log_req"], 4 * lc)))

    for chunk in (65536, 700):
        eng.set_chunk(chunk)
        for pinned in (True, False):
            rc, a, lg, cl = _submit_log(eng, buf, off, 3, remote, roff, start, lines, nbytes, pinned)   # exactly enough
            assert rc == 0 and cl.lines == lines and cl.out_bytes == nbytes and untouched(lg, lines, nbytes)
            assert lg["out"][:nbytes].tobytes() == want["log"].tobytes()
            assert np.array_equal(lg["log_off"][:lines + 1], want["log_off"]) and np.array_equal(lg["log_req"][:lines], want["log_req"])
            _responses_equal(a, want)
            for lc, oc in ((lines - 1, nbytes), (lines, nbytes - 1)):
                rc, a, lg, cl = _submit_log(eng, buf, off, 3, remote, roff, start, lc, oc, pinned)
                assert rc == 7, (lc, oc, pinned)                                      # GOFR_ERR_CAPACITY
                assert untouched(lg, lc, oc), (lc, oc, pinned)
                assert cl.lines == lines and cl.out_bytes == nbytes
                _responses_equal(a, want)
    eng.close()


@pytest.mark.gpu
def test_gpu_responses_and_launches_unchanged():
    """the responses of the logged call are those of gofr_conn_batch_submit byte for byte; without a log the call launches
    what it launched before (frame, parse, compact, serve per chunk, plus advance and egress when pinned), and a log adds
    gather, reqlog and pack (plus advance and egress when pinned) per chunk with lines"""
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(synth_table(spec), 0)
    buf, off = _streams(2000)
    remote, roff, start = _clients(len(off) - 1)
    want, _ = model(spec, buf, off, 11, remote, roff, start)
    lc, oc = conn_log_bound(off, roff)
    for pinned in (True, False):
        n0 = eng.launch_count()
        rc, a0, _, _ = _submit_log(eng, buf, off, 11, remote, roff, start, lc, oc, pinned, log=False)
        n1 = eng.launch_count()
        rc1, a1, _, _ = _submit_log(eng, buf, off, 11, remote, roff, start, lc, oc, pinned)
        n2 = eng.launch_count()
        assert rc == 0 and rc1 == 0
        assert n1 - n0 == (6 if pinned else 4)                                          # one chunk
        assert n2 - n1 == (n1 - n0) + (5 if pinned else 3)
        for k in a0:
            assert a0[k].tobytes() == a1[k].tobytes(), k
        _responses_equal(a1, want)
    eng.close()


@pytest.mark.gpu
def test_gpu_refuses_a_chunk_past_4_gib():
    """one connection so large that its log strings could pass 32-bit offsets: refused before anything is enqueued, and the
    engine serves the next batch"""
    from gofr_b200.engine import Engine
    spec = synth.config2_spec()
    eng = Engine(synth_table(spec), 0)
    big = np.zeros(260 << 20, np.uint8)
    off = np.array([0, big.size], np.uint32)
    remote = np.full(255, ord("9"), np.uint8)
    roff, start = np.array([0, 255], np.uint32), np.zeros(1, np.int64)
    rc, _, _, _ = _submit_log(eng, big, off, 1, remote, roff, start, 16, 4096, False)
    assert rc == 2                                                                       # GOFR_ERR_UNSUPPORTED
    buf, off = _streams(300)
    remote, roff, start = _clients(len(off) - 1)
    want, _ = model(spec, buf, off, 1, remote, roff, start)
    _check(eng.serve_connections(buf, off, DATE, 1, log=_log(remote, roff, start)), want)
    eng.close()


@pytest.mark.gpu
def test_gpu_equals_device_resident_chain():
    """frame → parse → serve in HBM, then gofr_requestlog_device on descriptors built on the host from those spans and
    meta words, gives the same lines"""
    import torch
    from gofr_b200.engine import DeviceBatch, Engine
    spec = synth.config1_spec()
    eng = Engine(synth_table(spec), 0)
    buf, off = _streams(5000)
    remote, roff, start = _clients(len(off) - 1)
    got = eng.serve_connections(buf, off, DATE, SEED, log=_log(remote, roff, start))
    d_buf, d_rec, first, _, _ = eng.http_frame_device(buf, off)
    total = int(first[-1].item())
    desc, arena, _, spans = eng.http_parse_resident(d_buf, d_rec, total)
    _, _, _, _, idx, req_first, ids = CB.model_requests(buf, off, SEED)
    k = len(idx)
    cdesc = desc.view(-1, 16)[torch.from_numpy(idx).cuda()].reshape(-1).contiguous()
    resp = eng.alloc_responses(k, int(got.out_off[-1]) + 4096)
    eng.serve_device(DeviceBatch(cdesc, torch.from_numpy(ids.reshape(-1).copy()).cuda(), arena, k, 0), DATE, resp)
    _, _, meta = resp.to_host()
    sp = spans.cpu().numpy().view(np.uint64)[idx]
    conn = np.repeat(np.arange(len(off) - 1), np.diff(req_first.astype(np.int64)))
    b, rb = buf.tobytes(), remote.tobytes()
    recs = []
    for j in np.nonzero(logged(meta, sp))[0].tolist():
        get = lambda q: b[int(sp[j, q] & 0xFFFFFFFF):int(sp[j, q] & 0xFFFFFFFF) + int(sp[j, q] >> 32)]
        c = int(conn[j])
        recs.append(S.LogRec(int(start[c]), LOG_NS - int(start[c]), LOG_NS, get(S_METHOD), get(S_UA), get(S_XFF),
                             rb[int(roff[c]):int(roff[c + 1])], get(S_TARGET), int(meta[j] & 0xFFFF), TZ, ids[j].tobytes()))
    d_out, d_off = eng.request_log_device(S.LogBatch.pack(recs))
    lo = d_off.cpu().numpy().view(np.uint32)
    assert np.array_equal(lo, got.log.log_off) and d_out[:int(lo[-1])].cpu().numpy().tobytes() == got.log.out.tobytes()
    assert np.array_equal(np.nonzero(logged(meta, sp))[0].astype(np.uint32), got.log.log_req)
    eng.close()
