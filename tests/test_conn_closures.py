"""Connection buffers served with handler closures in two calls: gofr_conn_batch_route (frame, parse, route; export what a
closure needs) and gofr_conn_batch_respond (splice the closures' GOFR_H_RESULT records in, answer every request).

The model composes what the project already checks on its own: the framer's oracle with the tails dropped → the
request-head oracle → the router oracle (stage 1), then Python closures that build result records, the splice restated in
numpy, and the serving oracle (stage 2), with test_conn_log's composition for the log lines.  CPU: the splice's device code
through tests/emu against the numpy splice, the parsed-form invariant the arena export relies on, the bound, the ABI layout
and the argument checks.  GPU: every column of both stages against the model across tables, chunk sizes and caller memory."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.engine import ConnLog, conn_respond_bound
from gofr_b200.table import Table
from tests import oracle as O
from tests import test_conn_batch as CB
from tests import test_conn_log as CL
from tests.emu import emu_conn_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATE = CB.DATE
SEED = 0x5EED_C10
ITEM = S.Schema(7, "main.Item", [S.Field("SKU", S.F_STRING, "sku"), S.Field("Qty", S.F_INT32, "qty"),
                                 S.Field("Note", S.F_STRING, "note", omitempty=True)])


def r4(x: int) -> int:
    return (x + 3) & ~3


# ---- tables whose user routes are closures (GOFR_H_RESULT) next to fused kinds and GOFR_H_HOST holes ----
def c1_spec() -> S.TableSpec:
    """config 1 with its datasource handlers as closures that return strings, errors or nil, and an item API"""
    return S.TableSpec(schemas=[ITEM], routes=[
        S.Route(S.M_GET, "/hello", S.H_PARAM_FORMAT, s0=b"name", s1=b"World", s2=b"Hello ", s3=b"!"),
        S.Route(S.M_GET, "/error", S.H_STATIC_ERROR, s0=b"some error occurred"),
        S.Route(S.M_GET, "/redis", S.H_RESULT),
        S.Route(S.M_GET, "/trace", S.H_HOST),
        S.Route(S.M_GET, "/mysql", S.H_RESULT),
        S.Route(S.M_POST, "/echo", S.H_RESULT, schema_id=7),
        S.Route(S.M_DELETE, "/users/{id}", S.H_RESULT, schema_id=7),
        S.Route(S.M_GET, "/api/v1/r{n}", S.H_RESULT, schema_id=7),
    ])


def c2_spec() -> S.TableSpec:
    """config 2 with every other route a closure returning the Profile row (or an error, nil, ...)"""
    routes = [S.Route(S.M_GET, "/api/v1/r%02d" % k, S.H_RESULT if k % 2 == 0 else S.H_ROW, schema_id=1) for k in range(16)]
    routes.append(S.Route(S.M_POST, "/echo", S.H_RESULT, schema_id=1))
    return S.TableSpec(schemas=[synth.C2_SCHEMA], routes=routes)


BIG_RECORD = 64 * 1024


def closure(spec: S.TableSpec, route: int, k: int, path: bytes, body: bytes) -> bytes:
    """The closure of `route` for request k: a GOFR_H_RESULT record built from what stage 1 exported (path, body).  Every
    outcome, a record far longer than its request, an empty record (the request's own body stays) and a malformed one."""
    if route >= len(spec.routes) or spec.routes[route].kind != S.H_RESULT:   # the table's default routes, fused kinds
        return b""
    R = spec.routes[route]
    rec = S.result_record
    sel = k % 13
    if sel == 0:
        return rec(S.RESULT_STRING, b"Hello " + path + b" <" + body[:20] + b">")
    if sel == 1:
        return rec(S.RESULT_ERROR, b"db: connection refused at " + path)
    if sel == 2:
        return rec(S.RESULT_NIL)
    if sel == 3:
        return rec(S.RESULT_MISSING, b"http: no such file")
    if sel == 4:
        return rec(S.RESULT_RAW_STRING, b"raw \"" + path + b"\"", S.RAW_ERR if k % 2 else S.RAW_OK)
    if sel == 5:
        return rec(S.RESULT_RAW_NIL)
    if sel == 6:
        return b"\x09\x00\x00\x00"                                    # unknown outcome: answered like a panic
    if sel == 7:
        return b""                                                    # no record: the request's own body stays
    if sel == 8:
        return rec(S.RESULT_STRING, bytes(range(256)) * (BIG_RECORD // 256))
    if not R.schema_id:
        return rec(S.RESULT_STRING, b"%d" % k)
    if R.schema_id == 7:
        vals = ["SKU-%d" % k, k % 1000, "" if k % 3 else "n&b"]
        sch = ITEM
    else:
        vals = [k, "name%d" % k, "e%d@x" % k, k % 2 == 0, k % 1000]
        sch = synth.C2_SCHEMA
    if sel in (9, 10):
        return rec(S.RESULT_DATA, sch.encode_row(vals))
    if sel == 11:
        return S.result_both(sch, vals, b"partial: %d" % k)
    return rec(S.RESULT_RAW_DATA, sch.encode_row(vals))


# ---- the model ----
def model_stage1(spec, buf, off, seed):
    """every column gofr_conn_batch_route returns, with the oracle's parsed requests (desc into the oracle's arena)"""
    rec, first, consumed, status, idx, req_first, ids = CB.model_requests(buf, off, seed)
    d, a, s, spans = O.http_parse(buf, rec)
    assert (s[idx] == 0).all()
    desc = d[idx].copy()
    meta, vars_ = O.route(O.OracleTable(spec), S.RequestBatch(desc, ids, a))
    return dict(desc=desc, arena=a, meta=meta, vars=vars_, req_at=rec[idx].astype(np.uint32), trace_ids=ids,
                req_first=req_first, consumed=consumed, conn_status=status, spans=spans[idx], req_conn=np.repeat(
                    np.arange(len(off) - 1), np.diff(req_first.astype(np.int64))))


def parsed(desc, arena, k):
    """(path, query, body) of request k"""
    x = desc[k]
    a, pl, ql, dl = int(x["arena_off"]), int(x["path_len"]), int(x["query_len"]), int(x["data_len"])
    b = arena.tobytes() if isinstance(arena, np.ndarray) else arena
    return b[a:a + pl], b[a + pl:a + pl + ql], b[a + r4(pl + ql):a + r4(pl + ql) + dl]


def run_closures(spec, m1):
    """the closures of the requests stage 1 left to them (status 0 on a GOFR_H_RESULT route) → (rec, rec_off)"""
    recs = []
    for k in range(len(m1["meta"])):
        st, route = int(m1["meta"][k]) & 0xFFFF, int(m1["meta"][k]) >> 16
        if st == 0 and route != S.ROUTE_NONE:
            path, _, body = parsed(m1["desc"], m1["arena"], k)
            recs.append(closure(spec, route, k, path, body))
        else:
            recs.append(b"")
    rec_off = np.cumsum([0] + [len(r) for r in recs]).astype(np.uint32)
    return np.frombuffer(b"".join(recs) or b"\0", np.uint8)[:int(rec_off[-1])].copy(), rec_off


def splice_np(desc, arena, rec, rec_off):
    """the splice restated: every request's path | query | pad4 | data | pad4 in request order, data its record when that is
    not empty, else its body → (descriptors into the new arena, new arena with 16 bytes of slack)"""
    ab, rb = arena.tobytes(), bytes(rec)
    out = bytearray()
    nd = desc.copy()
    for i in range(len(desc)):
        x = desc[i]
        a, pq = int(x["arena_off"]), int(x["path_len"]) + int(x["query_len"])
        r0, r1 = int(rec_off[i]), int(rec_off[i + 1])
        data = rb[r0:r1] if r1 > r0 else ab[a + r4(pq):a + r4(pq) + int(x["data_len"])]
        nd[i]["arena_off"] = len(out)
        nd[i]["data_len"] = len(data)
        out += ab[a:a + pq] + b"\0" * (r4(pq) - pq) + data + b"\0" * (r4(len(data)) - len(data))
    return nd, np.frombuffer(bytes(out) + b"\0" * 16, np.uint8).copy()


def model_stage2(spec, m1, rec, rec_off, remote=None, roff=None, start=None):
    """every column gofr_conn_batch_respond returns (and its log lines when remote is given)"""
    sd, sa = splice_np(m1["desc"], m1["arena"], rec, rec_off)
    o, f, m = O.OracleTable(spec).serve(S.RequestBatch(sd, m1["trace_ids"], sa), DATE)
    want = dict(out=o[:int(f[-1])], out_off=f, meta=m, req_at=m1["req_at"], trace_ids=m1["trace_ids"], req_first=m1["req_first"],
                consumed=m1["consumed"], conn_status=m1["conn_status"])
    if remote is None:
        return want
    sel = np.nonzero(CL.logged(m, m1["spans"]))[0]
    recs = []
    for k in sel.tolist():
        sp = m1["spans"][k]
        get = lambda j: m1["buf"][int(sp[j] & 0xFFFFFFFF):int(sp[j] & 0xFFFFFFFF) + int(sp[j] >> 32)]
        c = int(m1["req_conn"][k])
        recs.append(S.LogRec(int(start[c]), CL.LOG_NS - int(start[c]), CL.LOG_NS, get(CL.S_METHOD), get(CL.S_UA), get(CL.S_XFF),
                             remote.tobytes()[int(roff[c]):int(roff[c + 1])], get(CL.S_TARGET), int(m[k] & 0xFFFF), CL.TZ,
                             m1["trace_ids"][k].tobytes()))
    lo, lf = O.request_log(S.LogBatch.pack(recs))
    want.update(log=lo[:int(lf[-1])], log_off=lf, log_req=sel.astype(np.uint32))
    return want


def _streams(n, seed=synth.SEED, **kw):
    """pipelined connections with tails and defers, 30 KB bodies and 9 KB headers, holes and closure routes"""
    msgs = [m for m, _ in CB.GOOD] + CB.DEFERRED + CB.BIG + [CB.HOLE, b"GET /trace HTTP/1.1\r\nHost: h\r\n\r\n"] + CL.UNROUTED
    return synth.http_streams(n, seed=seed, tail_every=kw.pop("tail_every", 5), defer_every=kw.pop("defer_every", 11),
                              seed_msgs=msgs, **kw)


def _model(spec, buf, off, seed):
    m1 = model_stage1(spec, buf, off, seed)
    m1["buf"] = buf.tobytes()
    return m1


# ---- CPU ----
@pytest.mark.parametrize("mis", [0, 1, 2, 3])
def test_splice_device_code_equals_numpy(mis):
    """every source alignment of paths, bodies and records, empty records, empty paths and queries, a 0-request chunk and a
    later chunk (req0 != 0), with the Writer flushing as one lane decides, at every decision point and at random"""
    rng = np.random.default_rng(100 + mis)
    n = 400
    desc = np.zeros(n, S.DESC_DTYPE)
    arena = bytearray()
    recs = []
    for i in range(n):
        while len(arena) % 4:
            arena.append(0)
        pl = [0, 1, 2, 3, 4, 5, 11, 200][i % 8]
        ql = [0, 1, 3, 0, 7][i % 5]
        dl = [0, 1, 2, 3, 4, 33, 1000][i % 7]
        desc[i] = (len(arena), pl, ql, dl, S.M_GET, 0, 0)
        arena += rng.integers(1, 256, pl + ql, dtype=np.uint8).tobytes()
        while len(arena) % 4:
            arena.append(0)
        arena += rng.integers(0, 256, dl, dtype=np.uint8).tobytes()
        recs.append(b"" if i % 3 == 0 else rng.integers(0, 256, [1, 2, 3, 4, 5, 70, 300][i % 7], dtype=np.uint8).tobytes())
    arena = np.frombuffer(bytes(arena), np.uint8).copy()
    # record i is rec[starts[i]:starts[i + 1]]: a non-empty one is followed by 0..3 filler bytes of its own, so the records
    # after it start at every alignment; an empty one takes no bytes
    rec = bytearray()
    starts = np.zeros(n + 1, np.uint32)
    for i, r in enumerate(recs):
        starts[i] = len(rec)
        if r:
            rec += r + b"\xAB" * (i % 4)
    starts[n] = len(rec)
    assert {int(starts[i]) % 4 for i in range(n) if recs[i]} == {0, 1, 2, 3}
    for req0, cnt in ((0, n), (37, 200), (n, 0), (5, 1)):
        d = desc[req0:req0 + cnt]
        want_d, want_a = splice_np(d, arena, rec, starts[req0:req0 + cnt + 1])
        size = int(want_a.size) - 16
        for any_mode in (0, 1, 2):
            out, off, got_d = emu_conn_result.splice(d, arena, rec, starts, req0=req0, start=0, mis=mis, any_mode=any_mode)
            assert out[:size].tobytes() == want_a[:size].tobytes(), (req0, any_mode)
            assert (out[size:] == 0xEE).all()                       # nothing past the last request is written
            assert np.array_equal(off[:-1], want_d["arena_off"]) and int(off[-1]) == size
            assert got_d.tobytes() == want_d.tobytes()


def test_splice_of_parsed_connections_equals_numpy():
    """the splice of real parsed requests (the request-head oracle's arena) with closure records"""
    spec = c1_spec()
    buf, off = _streams(300)
    m1 = _model(spec, buf, off, SEED)
    rec, rec_off = run_closures(spec, m1)
    want_d, want_a = splice_np(m1["desc"], m1["arena"], rec, rec_off)
    out, got_off, got_d = emu_conn_result.splice(m1["desc"], m1["arena"], rec, rec_off)
    size = int(want_a.size) - 16
    assert out[:size].tobytes() == want_a[:size].tobytes() and got_d.tobytes() == want_d.tobytes()


def test_parsed_form_lies_inside_its_message():
    """the invariant the arena export relies on (include/gofr_b200.h): a request's parsed form starts at its raw offset
    rounded up to 4 and ends inside its own message — 1-byte targets, bodies of every length mod 4, chunked bodies, long
    queries, percent-decoded paths, at every raw alignment"""
    msgs = [b"GET / HTTP/1.1\r\nHost: h\r\n\r\n", b"GET /?a HTTP/1.1\r\nHost: h\r\n\r\n", b"HEAD / HTTP/1.1\r\nHost: h\r\n\r\n"]
    for dl in range(0, 12):
        msgs.append(b"POST / HTTP/1.1\r\nHost: h\r\nContent-Length: %d\r\n\r\n" % dl + b"x" * dl)
        msgs.append(b"PUT /%s HTTP/1.1\r\nHost: a\r\nContent-Length: %d\r\n\r\n" % (b"p" * dl, dl) + b"y" * dl)
        msgs.append(b"POST / HTTP/1.1\r\nHost: h\r\nTransfer-Encoding: chunked\r\n\r\n" +
                    (b"%x\r\n" % dl + b"z" * dl + b"\r\n" if dl else b"") + b"0\r\n\r\n")
    msgs.append(b"GET /%41%42?" + b"q" * 300 + b" HTTP/1.1\r\nHost: h\r\n\r\n")
    msgs += [m for m, _ in CB.GOOD] + CB.BIG
    checked = 0
    for lead in range(4):
        raw = b"\0" * lead + b"".join(msgs)
        off = np.cumsum([lead] + [len(m) for m in msgs]).astype(np.uint32)
        off = np.concatenate([[0], off]).astype(np.uint32)
        d, _, s, _ = O.http_parse(np.frombuffer(raw, np.uint8).copy(), off)
        for i in range(1, len(off) - 1):
            if s[i] != 0:
                continue
            x = d[i]
            pq = int(x["path_len"]) + int(x["query_len"])
            assert int(x["arena_off"]) == r4(int(off[i])), i
            assert int(x["arena_off"]) + r4(pq) + int(x["data_len"]) <= int(off[i + 1]), (lead, i)
            assert int(off[i + 1]) - int(off[i]) > pq + int(x["data_len"]) + 6
            checked += 1
    assert checked >= 4 * (len(msgs) - 1)
    # and over framed streams
    buf, boff = _streams(2000)
    rec, first, _, status, idx, _, _ = CB.model_requests(buf, boff, 1)
    d, _, s, _ = O.http_parse(buf, rec)
    for k in idx.tolist():
        x = d[k]
        assert int(x["arena_off"]) + r4(int(x["path_len"]) + int(x["query_len"])) + int(x["data_len"]) <= int(rec[k + 1])


def test_respond_bound_covers_what_the_model_needs():
    for spec in (c1_spec(), c2_spec()):
        t = Table(spec)
        for seed in range(4):
            buf, off = _streams(200, seed=seed)
            m1 = _model(spec, buf, off, seed)
            rec, rec_off = run_closures(spec, m1)
            want = model_stage2(spec, m1, rec, rec_off)
            assert conn_respond_bound(t, m1["desc"], rec_off) >= int(want["out_off"][-1])
    L = _abi.lib()
    oc = C.c_uint64()
    d = np.zeros(2, S.DESC_DTYPE)
    bad = np.array([0, 5, 4], np.uint32)
    assert L.gofr_conn_respond_bound(t.handle, d.ctypes.data, 2, bad.ctypes.data, C.byref(oc)) == 1   # decreasing
    assert L.gofr_conn_respond_bound(t.handle, None, 2, bad.ctypes.data, C.byref(oc)) == 1
    assert L.gofr_conn_respond_bound(t.handle, d.ctypes.data, 2, None, C.byref(oc)) == 1
    assert L.gofr_conn_respond_bound(None, d.ctypes.data, 0, None, C.byref(oc)) == 1
    assert L.gofr_conn_respond_bound(t.handle, None, 0, None, C.byref(oc)) == 0 and oc.value == 0
    # an empty record counts the request's own body
    one = np.zeros(1, S.DESC_DTYPE)
    one["data_len"] = 100
    z = np.zeros(2, np.uint32)
    assert L.gofr_conn_respond_bound(t.handle, one.ctypes.data, 1, z.ctypes.data, C.byref(oc)) == 0
    assert oc.value == L.gofr_table_response_bound(t.handle, 0, 0, 100)


def _c_layout():
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "gofr_b200.h"
#define F(T, f) printf(#T " " #f " %zu\n", offsetof(T, f));
int main(void) {
    printf("gofr_conn_route size %zu\n", sizeof(gofr_conn_route));
    printf("gofr_conn_results size %zu\n", sizeof(gofr_conn_results));
    F(gofr_conn_route, req_cap) F(gofr_conn_route, reserved) F(gofr_conn_route, desc) F(gofr_conn_route, arena)
    F(gofr_conn_route, meta) F(gofr_conn_route, vars) F(gofr_conn_route, req_at) F(gofr_conn_route, trace_ids)
    F(gofr_conn_route, req_first) F(gofr_conn_route, consumed) F(gofr_conn_route, conn_status)
    F(gofr_conn_results, rec) F(gofr_conn_results, rec_off) F(gofr_conn_results, rec_bytes) F(gofr_conn_results, n_req)
    F(gofr_conn_results, reserved)
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
    structs = {"gofr_conn_route": _abi.ConnRoute, "gofr_conn_results": _abi.ConnResults}
    for name, field, value in lines:
        T = structs[name]
        if field == "size":
            assert C.sizeof(T) == int(value), name
        else:
            assert getattr(T, field).offset == int(value), (name, field)
    assert sum(1 for ln in lines if ln[1] != "size") == len(_abi.ConnRoute._fields_) + len(_abi.ConnResults._fields_)


def test_invalid_arguments_without_a_gpu():
    L = _abi.lib()
    off = np.array([0, 40], np.uint32)
    buf = np.zeros(40, np.uint8)
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=40, n_conns=1, date=DATE, trace_seed=1)
    t = C.c_uint64()
    for n in (0, 1):
        cb.n_conns = n
        assert L.gofr_conn_batch_route(None, C.byref(cb), C.byref(_abi.ConnRoute())) == 1
        assert L.gofr_conn_batch_respond(None, C.byref(cb), C.byref(_abi.ConnResults()), C.byref(_abi.ConnResp()), None, C.byref(t)) == 1
    assert L.gofr_conn_batch_route(None, None, None) == 1
    assert L.gofr_conn_batch_respond(None, None, None, None, None, None) == 1


# ---- GPU ----
ROUTE_COLS = ("meta", "vars", "req_at", "trace_ids", "req_first", "consumed", "conn_status")


def _check_stage1(got, m1, what=""):
    for k in ROUTE_COLS:
        assert np.array_equal(np.asarray(getattr(got, k)), m1[k]), (what, k)
    n = len(m1["meta"])
    assert len(got.desc) == n
    keep = ["path_len", "query_len", "data_len", "method", "flags", "aux"]
    for f in keep:
        assert np.array_equal(got.desc[f], m1["desc"][f]), (what, f)
    assert np.array_equal(got.desc["arena_off"], m1["desc"]["arena_off"]), what      # the raw offset rounded up to 4
    ga, wa = got.arena.tobytes(), m1["arena"].tobytes()
    for k in range(n):
        assert parsed(got.desc, ga, k) == parsed(m1["desc"], wa, k), (what, k)


def _check_stage2(got, want, what=""):
    CB._check(got, want, what)
    if "log" in want:
        CL._check(got, want, what)


def _engine(spec):
    from gofr_b200.engine import Engine
    return Engine(Table(spec), 0)


@pytest.mark.gpu
def test_gpu_both_stages_equal_model():
    """config-1 and config-2 tables with closure routes, streams with tails, defers, 30 KB bodies, 9 KB headers and 64 KiB
    records; chunk sizes 1, 7 and the default; pinned and pageable caller memory; with and without the log lines"""
    for spec in (c1_spec(), c2_spec()):
        eng = _engine(spec)
        for n, chunks in ((150, (1, 7, 65536)), (6000, (7, 65536))):
            buf, off = _streams(n, seed=n)
            m1 = _model(spec, buf, off, SEED)
            rec, rec_off = run_closures(spec, m1)
            remote, roff, start = CL._clients(n)
            want = model_stage2(spec, m1, rec, rec_off, remote, roff, start)
            assert (want["meta"] & 0xFFFF != 0).sum() > (want["meta"] & 0xFFFF == 0).sum()
            for chunk in chunks:
                eng.set_chunk(chunk)
                for pinned in (True, False):
                    what = (spec.routes[-1].kind, n, chunk, pinned)
                    g1 = eng.route_connections(buf, off, SEED, pinned=pinned)
                    _check_stage1(g1, m1, what)
                    # closures run on what stage 1 exported
                    grec, groff = run_closures(spec, dict(m1, meta=g1.meta, desc=g1.desc, arena=g1.arena))
                    assert grec.tobytes() == rec.tobytes() and np.array_equal(groff, rec_off)
                    log = ConnLog(remote, roff, start, CL.LOG_NS, CL.TZ)
                    got = eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, results=(rec, rec_off), log=log)
                    _check_stage2(got, want, what)
                    got = eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, results=(rec, rec_off))
                    CB._check(got, want, what)
        eng.close()


@pytest.mark.gpu
def test_gpu_spliced_arena_larger_than_the_chunk():
    """every closure answers with a 64 KiB record: one chunk's spliced arena is many times its buffer bytes"""
    spec = c2_spec()
    eng = _engine(spec)
    buf, off = synth.http_streams(400, reqs=(1, 5))
    m1 = _model(spec, buf, off, 1)
    recs = [S.result_record(S.RESULT_STRING, b"%06d" % k * (BIG_RECORD // 6)) if (int(m) & 0xFFFF) == 0 else b""
            for k, m in enumerate(m1["meta"])]
    rec_off = np.cumsum([0] + [len(r) for r in recs]).astype(np.uint32)
    rec = np.frombuffer(b"".join(recs), np.uint8).copy()
    assert rec.size > 20 * buf.size
    want = model_stage2(spec, m1, rec, rec_off)
    for chunk in (65536, 50):
        eng.set_chunk(chunk)
        for pinned in (True, False):
            CB._check(eng.serve_connections(buf, off, DATE, 1, pinned=pinned, results=(rec, rec_off)), want, (chunk, pinned))
    eng.close()


@pytest.mark.gpu
def test_gpu_no_results_equal_submit_log():
    """res = NULL and results that are all empty answer byte for byte as gofr_conn_batch_submit_log, and res = NULL launches
    exactly its kernels"""
    spec = c1_spec()
    eng = _engine(spec)
    buf, off = _streams(3000)
    n = len(off) - 1
    remote, roff, start = CL._clients(n)
    log = ConnLog(remote, roff, start, CL.LOG_NS, CL.TZ)
    for pinned in (True, False):
        base = eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, log=log)
        k = len(base.meta)
        empty = (np.zeros(0, np.uint8), np.zeros(k + 1, np.uint32))
        got = eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, log=log, results=empty)
        for f in ("out", "out_off", "meta", "req_at", "trace_ids", "req_first", "consumed", "conn_status"):
            assert np.array_equal(np.asarray(getattr(got, f)), np.asarray(getattr(base, f))), f
        assert got.log.out.tobytes() == base.log.out.tobytes() and np.array_equal(got.log.log_req, base.log.log_req)
        # res = NULL through the new entry point: the same bytes and the same launches
        from gofr_b200.engine import conn_batch_bound, conn_log_bound
        rc_, oc_ = conn_batch_bound(eng.table, off)
        lc_, loc_ = conn_log_bound(off, roff)
        L = _abi.lib()
        for fn in ("respond", "submit_log"):
            a = dict(out=np.zeros(oc_, np.uint8), off=np.zeros(rc_ + 1, np.uint32), meta=np.zeros(rc_, np.uint32),
                     at=np.zeros(rc_, np.uint32), ids=np.zeros(rc_ * 16, np.uint8), first=np.zeros(n + 1, np.uint32),
                     cons=np.zeros(n, np.uint32), st=np.zeros(n, np.uint32), lout=np.zeros(loc_, np.uint8),
                     loff=np.zeros(lc_ + 1, np.uint32), lreq=np.zeros(lc_, np.uint32))
            cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=DATE, trace_seed=SEED)
            cr = _abi.ConnResp(out=a["out"].ctypes.data, out_cap=oc_, req_cap=rc_, out_off=a["off"].ctypes.data, meta=a["meta"].ctypes.data,
                               req_at=a["at"].ctypes.data, trace_ids=a["ids"].ctypes.data, req_first=a["first"].ctypes.data,
                               consumed=a["cons"].ctypes.data, conn_status=a["st"].ctypes.data)
            cl = _abi.ConnLog(remote=remote.ctypes.data, remote_off=roff.ctypes.data, start_unix_ns=start.ctypes.data,
                              log_unix_ns=CL.LOG_NS, tz_offset_s=CL.TZ, line_cap=lc_, out=a["lout"].ctypes.data, out_cap=loc_,
                              log_off=a["loff"].ctypes.data, log_req=a["lreq"].ctypes.data)
            t = C.c_uint64()
            l0 = eng.launch_count()
            if fn == "respond":
                assert L.gofr_conn_batch_respond(eng._e, C.byref(cb), None, C.byref(cr), C.byref(cl), C.byref(t)) == 0
            else:
                assert L.gofr_conn_batch_submit_log(eng._e, C.byref(cb), C.byref(cr), C.byref(cl), C.byref(t)) == 0
            assert L.gofr_batch_wait(eng._e, t.value) == 0
            launches = eng.launch_count() - l0
            if fn == "respond":
                first = (a, launches)
            else:
                assert launches == first[1]
                for key in a:
                    assert np.array_equal(a[key], first[0][key]), key
        assert first[0]["out"][:int(base.out_off[-1])].tobytes() == base.out.tobytes()
    eng.close()


@pytest.mark.gpu
def test_gpu_capacity_mismatch_and_bad_records():
    """a short req_cap in stage 1 reports what the batch needs; an n_req mismatch, decreasing record offsets and offsets
    past rec_bytes are refused with GOFR_ERR_INVALID, and the next call on the same engine is correct"""
    spec = c2_spec()
    eng = _engine(spec)
    buf, off = _streams(3000)
    m1 = _model(spec, buf, off, SEED)
    rec, rec_off = run_closures(spec, m1)
    want = model_stage2(spec, m1, rec, rec_off)
    k = len(m1["meta"])
    for chunk in (65536, 400):
        eng.set_chunk(chunk)
        for pinned in (True, False):
            with pytest.raises(_abi.GofrError) as ei:
                eng.route_connections(buf, off, SEED, pinned=pinned, req_cap=k - 1)
            assert ei.value.code == 7
            # the per-connection columns and req_first[n] through the C call directly
            r = eng.route_connections(buf, off, SEED, pinned=pinned, req_cap=k)
            _check_stage1(r, m1, (chunk, pinned))
            bad_cases = [(rec, rec_off[:-1]), (rec, np.concatenate([rec_off, [rec_off[-1]]]))]
            dec = rec_off.copy()
            j = int(np.nonzero(rec_off[:-1] > 0)[0][-1])
            dec[j + 1] = dec[j] - 1
            bad_cases.append((rec, dec))
            past = rec_off.copy()
            past[-1] = rec.size + 1
            bad_cases.append((rec, past))
            for brec, boff in bad_cases:
                with pytest.raises(_abi.GofrError) as ei:
                    eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, results=(brec, boff))
                assert ei.value.code == 1
                CB._check(eng.serve_connections(buf, off, DATE, SEED, pinned=pinned, results=(rec, rec_off)), want, (chunk, pinned))
    # stage 1's short capacity: per-connection columns complete, req_first[n] what the batch needed
    L = _abi.lib()
    n = len(off) - 1
    cols = dict(desc=np.zeros(k, S.DESC_DTYPE), arena=np.zeros(buf.size + 64, np.uint8), meta=np.zeros(k, np.uint32),
                vars=np.zeros(k * 8, np.uint32), at=np.zeros(k, np.uint32), ids=np.zeros(k * 16, np.uint8),
                first=np.zeros(n + 1, np.uint32), cons=np.zeros(n, np.uint32), st=np.zeros(n, np.uint32))
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=DATE, trace_seed=SEED)
    cr = _abi.ConnRoute(req_cap=k // 2, desc=cols["desc"].ctypes.data, arena=cols["arena"].ctypes.data, meta=cols["meta"].ctypes.data,
                        vars=cols["vars"].ctypes.data, req_at=cols["at"].ctypes.data, trace_ids=cols["ids"].ctypes.data,
                        req_first=cols["first"].ctypes.data, consumed=cols["cons"].ctypes.data, conn_status=cols["st"].ctypes.data)
    assert L.gofr_conn_batch_route(eng._e, C.byref(cb), C.byref(cr)) == 7
    assert np.array_equal(cols["first"], m1["req_first"]) and np.array_equal(cols["cons"], m1["consumed"])
    assert np.array_equal(cols["st"], m1["conn_status"]) and (cols["meta"][k // 2:] == 0).all()
    eng.close()


@pytest.mark.gpu
def test_gpu_bind_on_the_exported_batch():
    """gofr_batch_bind on stage 1's (desc, trace_ids, arena) gives what it gives on the model's batch"""
    spec = S.TableSpec(schemas=[ITEM], routes=[S.Route(S.M_POST, "/echo", S.H_RESULT, schema_id=7)])
    eng = _engine(spec)
    bodies = [b'{"sku":"A","qty":3}', b'{"sku":1}', b'{"qty":"x"}', b'', b'{"note":"n\\u0041"}']
    msgs = [b"POST /echo HTTP/1.1\r\nHost: h\r\nContent-Length: %d\r\n\r\n" % len(x) + x for x in bodies]
    buf, off = synth.http_streams(500, tail_every=4, seed_msgs=msgs * 20)
    m1 = _model(spec, buf, off, 3)
    got = eng.route_connections(buf, off, 3)
    _check_stage1(got, m1)
    b_got = got.batch
    b_want = S.RequestBatch(m1["desc"], m1["trace_ids"], m1["arena"])
    L = _abi.lib()
    res = []
    for b in (b_got, b_want):
        rb = _abi.ReqBatch(desc=b.desc.ctypes.data, trace_ids=b.trace_ids.ctypes.data, arena=b.arena.ctypes.data,
                           arena_bytes=b.arena.size, n=b.n, date=b"")
        rows, ln, st = np.zeros(b.n * 256, np.uint8), np.zeros(b.n, np.uint32), np.zeros(b.n, np.uint32)
        _abi.check(L.gofr_batch_bind(eng._e, 7, C.byref(rb), rows.ctypes.data, 256, ln.ctypes.data, st.ctypes.data), "bind")
        res.append((rows.reshape(b.n, 256), ln, st))
    (r1, l1, s1), (r2, l2, s2) = res
    assert np.array_equal(l1, l2) and np.array_equal(s1, s2)
    for i in range(b_got.n):
        if l1[i] <= 256:
            assert r1[i, :l1[i]].tobytes() == r2[i, :l2[i]].tobytes()
    assert (s1 == 0).sum() > 0
    eng.close()


def _compile_example(tmp_path):
    from gofr_b200 import _build
    _abi.lib()  # builds the library if needed
    exe = str(tmp_path / "conn_routes")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "cpp", "conn_routes.cpp"), "-o", exe, _build.LIB,
                           "-Wl,-rpath," + os.path.dirname(_build.LIB)])
    return exe


def test_cpp_connection_example_compiles(tmp_path):
    """no GPU: examples/cpp/conn_routes.cpp (App::ServeConnections) builds against the library with -Werror"""
    assert os.path.exists(_compile_example(tmp_path))


@pytest.mark.gpu
def test_gpu_cpp_connection_example(tmp_path):
    """App::ServeConnections on pipelined connections with a partial tail: the bodies the reference's route test expects,
    and per connection the concatenation of what App::Serve returns for the same requests, trace ids and date"""
    r = subprocess.run([_compile_example(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    assert r.stdout.strip().endswith("ok")
