"""Connection receive buffers in host memory served in one call (gofr_conn_batch_submit): frame, parse, drop the tails, serve.

The model composes what the project already checks on its own: the framer's oracle (tests/http_frame_oracle.c) → drop the
last record of every MORE / DEFER connection → the request-head oracle → the serving oracle, with the trace ids restated in
numpy.  CPU: the compact step's device code (conn_device.cuh through tests/emu) against the model, the trace-id function,
the capacity bound, the ABI layout and the argument checks.  GPU: every output column against the model across batch
shapes, chunk sizes, caller memory kinds and capacities, and against the device-resident chain."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.engine import conn_batch_bound
from gofr_b200.table import Table
from tests import oracle as O
from tests import http_frame_oracle as FO
from tests.emu import emu_conn
from tests.test_http_parse import DEFERRED, GOOD

DONE = 0
DATE = S.http_date(1_700_000_000)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOLE = b"GET /redis HTTP/1.1\r\nHost: h\r\n\r\n"       # config 1: a GOFR_H_HOST route, answered on the host
BIG = [b"GET /big HTTP/1.1\r\nHost: h\r\nX-Pad: " + b"p" * 9000 + b"\r\n\r\n",
       b"POST /echo HTTP/1.1\r\nHost: h\r\nContent-Length: 30000\r\n\r\n" + b"b" * 30000]


# ---- the model ----
def trace_ids(seed: int, conn: np.ndarray, j: np.ndarray) -> np.ndarray:
    """include/gofr_b200.h: x = splitmix64(seed ^ splitmix64(c)); bytes 0-7 = splitmix64(x + 2j), 8-15 = splitmix64(x + 2j + 1)"""
    with np.errstate(over="ignore"):
        x = synth.splitmix64(np.uint64(seed) ^ synth.splitmix64(conn.astype(np.uint64)))
        j2 = j.astype(np.uint64) * np.uint64(2)
        lo, hi = synth.splitmix64(x + j2), synth.splitmix64(x + j2 + np.uint64(1))
    return np.stack([lo, hi], axis=1).astype("<u8").view(np.uint8).reshape(-1, 16)


def model_requests(buf, off, seed):
    """framing with the tails dropped → (rec, first, consumed, status, idx (the records that are requests), req_first, ids)"""
    rec, first, consumed, status = FO.http_frame(buf, off)
    n = len(off) - 1
    counts = (np.diff(first.astype(np.int64)) - (status != DONE)).astype(np.int64)
    conn = np.repeat(np.arange(n, dtype=np.int64), counts)
    req_first = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    j = np.arange(len(conn), dtype=np.int64) - req_first[conn].astype(np.int64) if len(conn) else np.zeros(0, np.int64)
    idx = first[conn].astype(np.int64) + j if len(conn) else np.zeros(0, np.int64)
    return rec, first, consumed, status, idx, req_first, trace_ids(seed, conn, j)


def model(spec, buf, off, seed, date=DATE):
    """every column gofr_conn_batch_submit returns, as a dict"""
    rec, first, consumed, status, idx, req_first, ids = model_requests(buf, off, seed)
    d, a, s, _ = O.http_parse(buf, rec)
    assert (s[idx] == 0).all()                       # every whole request is in the subset
    desc = d[idx].copy()
    o, f, m = O.OracleTable(spec).serve(S.RequestBatch(desc, ids, a), date)
    return dict(out=o[:int(f[-1])], out_off=f, meta=m, req_at=rec[idx].astype(np.uint32), trace_ids=ids, req_first=req_first,
                consumed=consumed, conn_status=status)


def _streams(n, seed=synth.SEED, holes=False, **kw):
    msgs = [m for m, _ in GOOD] + DEFERRED + BIG + ([HOLE] * 8 if holes else [])
    return synth.http_streams(n, seed=seed, tail_every=kw.pop("tail_every", 5), defer_every=kw.pop("defer_every", 11),
                              seed_msgs=msgs, **kw)


# ---- CPU ----
def test_compact_device_code_equals_model():
    for kw in ({}, {"tail_every": 3, "defer_every": 7}, {"reqs": (1, 1)}, {"reqs": (0, 1), "tail_every": 2}):
        buf, off = synth.http_streams(1500, **kw)
        # empty connections in the middle and at the end
        off = np.concatenate([off[:700], np.full(130, off[699], np.uint32), off[700:], np.full(5, off[-1], np.uint32)])
        seed = 0x1234_5678_9ABC_DEF0
        rec, first, consumed, status, idx, req_first, ids = model_requests(buf, off, seed)
        d, _, _, _ = O.http_parse(buf, rec)
        for conn0, req0 in ((0, 0), (0, 77)):
            g_desc, g_at, g_ids, g_first = emu_conn.compact(first, status, rec, d, seed, conn0, req0)
            assert np.array_equal(g_first, req_first + np.uint32(req0))
            assert np.array_equal(g_at, rec[idx]) and np.array_equal(g_ids, ids)
            assert g_desc.tobytes() == d[idx].tobytes()
        if kw.get("reqs") == (1, 1):
            assert np.array_equal(np.diff(req_first.astype(np.int64)), (np.diff(off.astype(np.int64)) > 0).astype(np.int64))


def test_compact_of_a_later_chunk_keys_ids_by_batch_index():
    """a chunk that starts at connection conn0 gives the ids the whole batch gives those connections"""
    buf, off = synth.http_streams(300, tail_every=4)
    seed = 99
    rec, first, _, status, idx, req_first, ids = model_requests(buf, off, seed)
    d, _, _, _ = O.http_parse(buf, rec)
    lo = 120
    sub_first = first[lo:] - first[lo]
    _, at, g_ids, g_first = emu_conn.compact(sub_first, status[lo:], rec[int(first[lo]):], d[int(first[lo]):], seed, lo, int(req_first[lo]))
    k = int(req_first[lo])
    assert np.array_equal(g_first, req_first[lo:]) and np.array_equal(g_ids, ids[k:]) and np.array_equal(at, rec[idx[k:]])


def test_trace_id_function_equals_numpy_statement():
    rng = np.random.default_rng(7)
    for seed in (0, 1, 0xFFFFFFFFFFFFFFFF, int(rng.integers(0, 2**63))):
        for c, j in ((0, 0), (1, 0), (0, 1), (0xFFFFFFFF, 0xFFFFFFFF), (40000, 3), (int(rng.integers(0, 2**32)), 17)):
            want = trace_ids(seed, np.array([c]), np.array([j]))[0].tobytes()
            assert emu_conn.trace_id(seed, c, j) == want, (seed, c, j)


def test_bound_covers_what_the_model_needs():
    """gofr_conn_batch_bound against the requests and response bytes the model needs, on thousands of seeded connections
    with 30 KB bodies and 9 KB headers among them"""
    for spec in (synth.config1_spec(), synth.config2_spec()):
        t = Table(spec)
        for seed in range(12):
            buf, off = _streams(250, seed=seed, holes=True, reqs=(0, 4))
            m = model(spec, buf, off, seed)
            req_cap, out_cap = conn_batch_bound(t, off)
            assert req_cap >= int(m["req_first"][-1]) and out_cap >= int(m["out_off"][-1]), seed
    # the bound is also what the framer states: one request per 16 bytes plus one per connection
    t = Table(synth.config2_spec())
    off = np.array([0, 100, 100, 116], np.uint32)
    rc, _ = conn_batch_bound(t, off)
    assert rc == 116 // 16 + 3


def _c_layout():
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "gofr_b200.h"
#define F(T, f) printf(#T " " #f " %zu\n", offsetof(T, f));
int main(void) {
    printf("gofr_conn_batch size %zu\n", sizeof(gofr_conn_batch));
    printf("gofr_conn_resp size %zu\n", sizeof(gofr_conn_resp));
    F(gofr_conn_batch, buf) F(gofr_conn_batch, buf_off) F(gofr_conn_batch, buf_bytes) F(gofr_conn_batch, n_conns)
    F(gofr_conn_batch, date) F(gofr_conn_batch, pad) F(gofr_conn_batch, trace_seed)
    F(gofr_conn_resp, out) F(gofr_conn_resp, out_cap) F(gofr_conn_resp, req_cap) F(gofr_conn_resp, reserved)
    F(gofr_conn_resp, out_off) F(gofr_conn_resp, meta) F(gofr_conn_resp, req_at) F(gofr_conn_resp, trace_ids)
    F(gofr_conn_resp, req_first) F(gofr_conn_resp, consumed) F(gofr_conn_resp, conn_status) F(gofr_conn_resp, out_bytes)
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
    structs = {"gofr_conn_batch": _abi.ConnBatch, "gofr_conn_resp": _abi.ConnResp}
    for name, field, value in lines:
        T = structs[name]
        if field == "size":
            assert C.sizeof(T) == int(value), name
        else:
            assert getattr(T, field).offset == int(value), (name, field)
    assert sum(1 for ln in lines if ln[1] != "size") == len(_abi.ConnBatch._fields_) + len(_abi.ConnResp._fields_)


def test_invalid_arguments_without_a_gpu():
    L = _abi.lib()
    off = np.array([0, 40], np.uint32)
    buf = np.zeros(40, np.uint8)
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=40, n_conns=1, date=DATE, trace_seed=1)
    cr = _abi.ConnResp()
    t = C.c_uint64()
    for n in (0, 1):
        cb.n_conns = n
        assert L.gofr_conn_batch_submit(None, C.byref(cb), C.byref(cr), C.byref(t)) == 1
    assert L.gofr_conn_batch_submit(None, None, None, None) == 1
    # the bound: null arguments and decreasing offsets
    tab = Table(synth.config2_spec())
    rc, oc = C.c_uint32(), C.c_uint64()
    assert L.gofr_conn_batch_bound(None, off.ctypes.data, 1, C.byref(rc), C.byref(oc)) == 1
    assert L.gofr_conn_batch_bound(tab.handle, None, 1, C.byref(rc), C.byref(oc)) == 1
    assert L.gofr_conn_batch_bound(tab.handle, off.ctypes.data, 1, None, C.byref(oc)) == 1
    bad = np.array([0, 40, 39], np.uint32)
    assert L.gofr_conn_batch_bound(tab.handle, bad.ctypes.data, 2, C.byref(rc), C.byref(oc)) == 1
    assert L.gofr_conn_batch_bound(tab.handle, None, 0, C.byref(rc), C.byref(oc)) == 0 and rc.value == 0 and oc.value == 0


# ---- GPU ----
COLS = ("out_off", "meta", "req_at", "trace_ids", "req_first", "consumed", "conn_status")


def _check(got, want, what=""):
    assert got.out.tobytes() == want["out"].tobytes(), what
    for k in COLS:
        assert np.array_equal(np.asarray(getattr(got, k)), want[k]), (what, k)


def _submit(eng, buf, off, seed, req_cap, out_cap, pinned, canary=64):
    """gofr_conn_batch_submit into buffers with `canary` guard bytes behind each capacity → (rc, arrays)"""
    from gofr_b200.engine import pinned_array
    n = len(off) - 1
    if pinned:
        alloc = lambda count, dt: pinned_array(count * np.dtype(dt).itemsize).view(dt)
    else:
        alloc = lambda count, dt: np.empty(count, dt)
    a = dict(out=alloc(out_cap + canary, np.uint8), out_off=alloc(req_cap + 1 + canary, np.uint32),
             meta=alloc(req_cap + canary, np.uint32), req_at=alloc(req_cap + canary, np.uint32),
             trace_ids=alloc((req_cap + canary) * 16, np.uint8), req_first=alloc(n + 1, np.uint32), consumed=alloc(max(n, 1), np.uint32),
             conn_status=alloc(max(n, 1), np.uint32))
    for v in a.values():
        v.view(np.uint8)[:] = 0xA5
    buf = np.ascontiguousarray(buf)
    off = np.ascontiguousarray(off, dtype=np.uint32)
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=DATE, trace_seed=seed)
    cr = _abi.ConnResp(out=a["out"].ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=a["out_off"].ctypes.data,
                       meta=a["meta"].ctypes.data, req_at=a["req_at"].ctypes.data, trace_ids=a["trace_ids"].ctypes.data,
                       req_first=a["req_first"].ctypes.data, consumed=a["consumed"].ctypes.data, conn_status=a["conn_status"].ctypes.data)
    L = _abi.lib()
    t = C.c_uint64()
    rc = L.gofr_conn_batch_submit(eng._e, C.byref(cb), C.byref(cr), C.byref(t))
    if rc == 0:
        rc = L.gofr_batch_wait(eng._e, t.value)
    return rc, a, int(cr.out_bytes)


def _untouched(a, req_cap, out_cap):
    """no byte at or past either capacity was written"""
    return all((v.view(np.uint8)[k:] == 0xA5).all() for v, k in (
        (a["out"], out_cap), (a["out_off"], 4 * (req_cap + 1)), (a["meta"], 4 * req_cap), (a["req_at"], 4 * req_cap),
        (a["trace_ids"], 16 * req_cap)))


@pytest.mark.gpu
def test_gpu_columns_equal_model():
    from gofr_b200.engine import Engine
    for spec, holes in ((synth.config1_spec(), True), (synth.config2_spec(), False)):
        eng = Engine(Table(spec), 0)
        cases = [(_streams(n, seed=n + 1, holes=holes), f"n={n}") for n in (1, 127, 128, 129)]
        buf, off = _streams(40000, holes=holes)
        # connections beyond the 26 KiB staging budget (BIG), tiles of empty connections in the middle and at the end
        off = np.concatenate([off[:20001], np.full(300, off[20000], np.uint32), off[20001:], np.full(200, off[-1], np.uint32)])
        cases.append(((buf, off), "40000"))
        for (b, o), what in cases:
            want = model(spec, b, o, 0xC0FFEE)
            for pinned in (True, False):
                got = eng.serve_connections(b, o, DATE, 0xC0FFEE, pinned=pinned)
                _check(got, want, (what, pinned))
            if holes and what == "40000":
                assert (want["meta"] & 0xFFFF == 0).sum() > 0       # GOFR_H_HOST holes: no bytes
        # no connections
        got = eng.serve_connections(np.zeros(0, np.uint8), np.zeros(1, np.uint32), DATE, 1)
        assert got.out.size == 0 and got.req_first.tolist() == [0]
        eng.close()


@pytest.mark.gpu
def test_gpu_connection_larger_than_a_chunk():
    """one connection of 9 MiB of pipelined requests (a chunk of its own, past the 8 MiB chunk budget) between ordinary ones"""
    from gofr_b200.engine import Engine
    spec = synth.config2_spec()
    eng = Engine(Table(spec), 0)
    buf, off = _streams(3000)
    get = b"GET /hello?name=x HTTP/1.1\r\nHost: localhost:8000\r\nUser-Agent: curl/8.4.0\r\n\r\n"
    huge = np.frombuffer(get * (9 * 2**20 // len(get) + 1), np.uint8)
    cut = int(off[1500])
    buf2 = np.concatenate([buf[:cut], huge, buf[cut:]])
    off2 = np.concatenate([off[:1501], off[1500:] + np.uint32(huge.size)]).astype(np.uint32)
    want = model(spec, buf2, off2, 5)
    for pinned in (True, False):
        _check(eng.serve_connections(buf2, off2, DATE, 5, pinned=pinned), want, pinned)
    eng.close()


@pytest.mark.gpu
def test_gpu_chunk_sizes_give_identical_outputs():
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(Table(spec), 0)
    buf, off = _streams(2500, holes=True)
    want = model(spec, buf, off, 42)
    for chunk in (1, 7, 1000, 65536):
        eng.set_chunk(chunk)
        for pinned in (True, False):
            _check(eng.serve_connections(buf, off, DATE, 42, pinned=pinned), want, (chunk, pinned))
    eng.close()


@pytest.mark.gpu
def test_gpu_capacity_and_invalid_offsets():
    from gofr_b200.engine import Engine
    spec = synth.config2_spec()
    eng = Engine(Table(spec), 0)
    buf, off = _streams(3000)
    want = model(spec, buf, off, 3)
    n_req, n_bytes = int(want["req_first"][-1]), int(want["out_off"][-1])
    for chunk in (65536, 700):
        eng.set_chunk(chunk)
        for pinned in (True, False):
            rc, a, ob = _submit(eng, buf, off, 3, n_req, n_bytes, pinned)           # exactly enough
            assert rc == 0 and ob == n_bytes and _untouched(a, n_req, n_bytes)
            assert a["out"][:n_bytes].tobytes() == want["out"].tobytes()
            for k in COLS:
                got = a[k][:len(want[k]) * (16 if k == "trace_ids" else 1)]
                assert np.array_equal(got, want[k].reshape(-1)), (k, pinned)
            for rq, oc in ((n_req - 1, n_bytes), (n_req, n_bytes - 1)):            # one request or one byte short
                rc, a, ob = _submit(eng, buf, off, 3, rq, oc, pinned)
                assert rc == 7                                                      # GOFR_ERR_CAPACITY
                assert _untouched(a, rq, oc), (rq, oc, pinned)
                assert ob == n_bytes and int(a["req_first"][len(off) - 1]) == n_req     # what the batch needed
                for k in ("req_first", "consumed", "conn_status"):                  # per-connection columns complete
                    assert np.array_equal(a[k][:len(want[k])], want[k]), k
    # a bad offset in a later chunk: refused, and the engine serves the next batch correctly
    eng.set_chunk(500)
    bad = off.copy()
    bad[2600] = bad[2599] - 1
    for pinned in (True, False):
        rc, _, _ = _submit(eng, buf, bad, 3, n_req + 100, n_bytes + 100, pinned)
        assert rc == 1
        past = off.copy()
        past[-1] = buf.size + 1
        assert _submit(eng, buf, past, 3, n_req + 100, n_bytes + 100, pinned)[0] == 1
        _check(eng.serve_connections(buf, off, DATE, 3, pinned=pinned), want, pinned)
    eng.close()


@pytest.mark.gpu
def test_gpu_equals_device_resident_chain():
    """the per-request responses equal those of frame → parse → gofr_serve_device in HBM with the same ids"""
    import torch
    from gofr_b200.engine import DeviceBatch, Engine
    spec = synth.config1_spec()
    eng = Engine(Table(spec), 0)
    buf, off = _streams(6000, holes=True)
    seed = 0xABCDEF
    got = eng.serve_connections(buf, off, DATE, seed)
    d_buf, d_rec, first, consumed, status = eng.http_frame_device(buf, off)
    total = int(first[-1].item())
    desc, arena, parsed, _ = eng.http_parse_resident(d_buf, d_rec, total)
    _, _, _, _, idx, _, ids = model_requests(buf, off, seed)
    k = len(idx)
    d_idx = torch.from_numpy(idx).cuda()
    cdesc = desc.view(-1, 16)[d_idx].reshape(-1).contiguous()
    d_ids = torch.from_numpy(ids.reshape(-1).copy()).cuda()
    resp = eng.alloc_responses(k, int(got.out_off[-1]) + 4096)
    eng.serve_device(DeviceBatch(cdesc, d_ids, arena, k, 0), DATE, resp)
    o, f, m = resp.to_host()
    assert np.array_equal(f, got.out_off) and np.array_equal(m, got.meta) and o.tobytes() == got.out.tobytes()
    assert np.array_equal(got.trace_ids, ids)
    eng.close()
