"""gofr_conn_app_frontend_* and gofr_conn_batch_respond_ex: handler-closure apps served one connection read per call, in two
independent batching rounds (route, then respond) with the closures on the caller's thread.

Without a GPU: both rounds of conn_app_frontend.cpp against stub route, bind and respond-ex calls under ThreadSanitizer
(timer-closed, full and one-read batches with and without lines, respond batches mixing route batches, seed 0 with full
batches, capacity reruns, 0-byte and oversize reads, a caller parked between its two calls, a caller with a wrong record
count), the trace-key helper of the compact kernel, argument checks and the ctypes prototypes.  On the GPU: respond_ex
against respond with the keys of (trace_seed, c) and with the connections permuted, and every caller against the model of
test_conn_closures.py (framer → heads → route → Bind → closures → splice → serve → log) evaluated with the ids its route
call returned, in three batching regimes with and without lines, the binds against gofr_batch_bind on the caller's exported
batch, and a parked caller beside a gofr_conn_frontend on one engine."""
import ctypes as C
import json
import os
import random
import re
import subprocess
import threading

import numpy as np
import pytest

from gofr_b200 import _abi
from tests import test_conn_closures as CC
from tests import test_conn_frontend as TF
from tests import test_conn_log as TL

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INVALID, CAPACITY = 1, 7
DONE, MORE, DEFER = 0, 1, 2
SEED = 0x5EED_A99
M64 = (1 << 64) - 1


def splitmix64(x: int) -> int:
    z = (x + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def conn_trace_key(seed: int, c: int) -> int:
    return splitmix64(seed ^ splitmix64(c))


# ---------------------------------------------------------------------------------------------------------------
# without a GPU
# ---------------------------------------------------------------------------------------------------------------
def _stress_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("stress") / "conn_app_frontend_stress")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-Wall", "-Wextra", "-Werror",
                           os.path.join(HERE, "emu", "conn_app_frontend_stress.cpp"), "-o", exe])
    return exe


@pytest.fixture(scope="module")
def stress_exe(tmp_path_factory):
    return _stress_exe(tmp_path_factory)


@pytest.mark.parametrize("args", [
    "16 200 64 200 2000 1 7 0 0",       # batches close on the timer (16 callers < 64)
    "32 100 8 100000 1500 1 7 0 0",     # batches close because they are full
    "16 50 1 0 300 1 7 0 0",            # one read per batch
    "16 200 64 200 2000 0 7 0 0",       # without lines
    "64 40 64 100000 200 0 0 0 0",      # seed 0, full batches of 64: every read still gets its own key
    "32 100 8 100000 1500 1 7 1 1",     # a caller parked between its calls; callers with one record too many
    "16 50 1 0 300 0 7 1 1",
])
def test_two_rounds_under_tsan(stress_exe, args):
    """no GPU: every caller gets the route answer and the responses made from ITS read, records, key, remote string and
    clock, rebased to its buffers; each connection comes back with the key its route call handed out; respond batches mix
    route batches; a batch refused for its output capacity is served again; 0-byte reads are answered without a batch and
    oversize reads refused; a parked caller does not hold anybody up; a wrong record count fails only its caller"""
    r = subprocess.run([stress_exe] + args.split(), capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ThreadSanitizer" not in r.stderr, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    t, n, max_batch = (int(v) for v in args.split()[:3])
    park, bad = int(args.split()[7]), int(args.split()[8])
    assert res["bad"] == 0 and res["violations"] == 0 and res["largest"] <= max_batch
    assert res["empty"] > 0 and res["over"] > 0 and res["bound"] > 0 and res["rebound"] > 0 and res["hosts"] > 0
    assert res["keys"] == res["route_reads"]
    if max_batch > 1:
        assert res["reruns"] > 0 and res["reruns"] == res["refused"]
    else:
        assert res["route_batches"] == res["route_reads"] and res["respond_batches"] == res["respond_reads"]
    if 1 < max_batch != t:     # when every thread fits one batch, respond batches may repeat the route batches exactly
        assert res["mixed"] > 0
    if park:
        assert res["parked_ok"] == 1
    if bad:
        assert res["invalid_got"] > 0 and res["isolated"] > 0
    else:
        assert res["isolated"] == 0 and res["invalid_got"] == 0


def test_trace_key_helper_on_the_host(tmp_path):
    """conn_device.cuh's conn_key, compiled for the host: without a key column it is conn_trace_key(seed, conn0 + i), with
    one it is the column's key"""
    src = tmp_path / "key.cpp"
    src.write_text('#include "%s"\n#include <cstdio>\nint main() {\n  const uint64_t keys[3] = {11, 0xFFFFFFFFFFFFFFFFull, 7};\n'
                   '  for (uint32_t i = 0; i < 3; i++) printf("%%llu %%llu %%llu\\n", (unsigned long long)gofr::conn_key(nullptr, 0x5EEDull, 40, i),\n'
                   '    (unsigned long long)gofr::conn_trace_key(0x5EEDull, 40 + i), (unsigned long long)gofr::conn_key(keys, 0x5EEDull, 40, i));\n}\n'
                   % os.path.join(ROOT, "gofr_b200", "csrc", "conn_device.cuh"))
    exe = str(tmp_path / "key")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", str(src), "-o", exe])
    rows = [tuple(int(v) for v in ln.split()) for ln in subprocess.check_output([exe], text=True).splitlines()]
    assert [r[2] for r in rows] == [11, M64, 7]
    for i, (a, b, _) in enumerate(rows):
        assert a == b == conn_trace_key(0x5EED, 40 + i)


def test_argument_checks():
    """no GPU: the entry points refuse bad arguments before they allocate or queue anything"""
    L = _abi.lib()
    f = C.c_void_p()
    fake = C.c_void_p(0x10)
    schema = (C.c_uint32 * 1)(7)
    assert L.gofr_conn_app_frontend_create(C.byref(f), None, 16, 100, 4096, 1, 0, 1, None, 0, None) == INVALID
    assert L.gofr_conn_app_frontend_create(None, fake, 16, 100, 4096, 1, 0, 1, None, 0, None) == INVALID
    assert L.gofr_conn_app_frontend_create(C.byref(f), fake, 0, 100, 4096, 1, 0, 1, None, 0, None) == INVALID
    assert L.gofr_conn_app_frontend_create(C.byref(f), fake, 16, 100, 4096, 1, 0, 1, schema, 1, None) == INVALID
    assert L.gofr_conn_app_frontend_create(C.byref(f), fake, 1 << 16, 100, 1 << 16, 1, 0, 1, None, 0, None) == CAPACITY
    assert L.gofr_conn_app_frontend_route(None, b"GET", 3, None, None, None) == INVALID
    assert L.gofr_conn_app_frontend_respond(None, b"GET", 3, 0, None, b"", 0, 0, None, None) == INVALID
    assert L.gofr_conn_app_frontend_stats(None, None) == INVALID
    assert L.gofr_conn_app_frontend_set_clock(None, 1) == INVALID
    L.gofr_conn_app_frontend_destroy(None)
    assert L.gofr_conn_batch_respond_ex(None, None, None, None, None, None, None) == INVALID


def test_prototypes_match_the_header():
    """the ctypes prototypes take as many arguments as include/gofr_b200.h declares, and the structs match the header's"""
    L = _abi.lib()
    header = open(os.path.join(ROOT, "include", "gofr_b200.h")).read()
    decls = dict((m.group(1), m.group(2)) for m in re.finditer(r"\b(gofr_conn_app_frontend_[a-z_]+|gofr_conn_batch_respond_ex)\s*\(([^)]*)\)", header))
    assert set(decls) == {"gofr_conn_app_frontend_create", "gofr_conn_app_frontend_destroy", "gofr_conn_app_frontend_set_clock",
                          "gofr_conn_app_frontend_stats", "gofr_conn_app_frontend_route", "gofr_conn_app_frontend_respond",
                          "gofr_conn_batch_respond_ex"}
    for name, params in decls.items():
        assert len(getattr(L, name).argtypes) == len(params.split(",")), name
    for struct, cls in (("gofr_conn_app_bind", _abi.ConnAppBind), ("gofr_conn_app_stats", _abi.ConnAppStats)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), header, re.S).group(1)
        names = re.findall(r"(\w+)(?:\s*,|\s*;)", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
        assert names == [n for n, _ in cls._fields_], struct
    assert C.sizeof(_abi.ConnAppBind) == 40 and C.sizeof(_abi.ConnAppStats) == 56


# ---------------------------------------------------------------------------------------------------------------
# the GPU
# ---------------------------------------------------------------------------------------------------------------
def _c1_route_schema():
    spec = CC.c1_spec()
    return spec, {r: (7, len(CC.ITEM.fields)) for r, rt in enumerate(spec.routes) if rt.schema_id == 7}


@pytest.mark.gpu
def test_gpu_respond_ex_equals_respond():
    """with keys conn_trace_key(seed, c) respond_ex is respond, byte for byte (responses, every column, the lines); with the
    connections permuted and their keys with them, every connection's answer is the unpermuted one"""
    from gofr_b200.engine import ConnLog
    spec = CC.c1_spec()
    eng = CC._engine(spec)
    buf, off = CC._streams(300, seed=5)
    n = len(off) - 1
    m1 = CC._model(spec, buf, off, SEED)
    rec, rec_off = CC.run_closures(spec, m1)
    remote, roff, start = TL._clients(n)
    log = ConnLog(remote, roff, start, TL.LOG_NS, TL.TZ)
    want = CC.model_stage2(spec, m1, rec, rec_off, remote, roff, start)
    keys = np.array([conn_trace_key(SEED, c) for c in range(n)], np.uint64)
    base = eng.serve_connections(buf, off, CC.DATE, SEED, results=(rec, rec_off), log=log)
    got = eng.serve_connections(buf, off, CC.DATE, SEED, results=(rec, rec_off), log=log, trace_key=keys)
    CC._check_stage2(got, want)
    for k in ("out", "out_off", "meta", "req_at", "trace_ids", "req_first", "consumed", "conn_status"):
        assert np.array_equal(getattr(got, k), getattr(base, k)), k
    for k in ("out", "log_off", "log_req"):
        assert np.array_equal(getattr(got.log, k), getattr(base.log, k)), k
    # permuted: connection c of the new batch is connection perm[c] of the old one, with its key, records and client
    perm = np.random.default_rng(3).permutation(n)
    rf = base.req_first.astype(np.int64)
    parts, recs, roffs, rems, starts = [], [], [0], [], []
    b, r, rb = buf.tobytes(), rec.tobytes(), remote.tobytes()
    for c in perm.tolist():
        parts.append(b[int(off[c]):int(off[c + 1])])
        for k in range(rf[c], rf[c + 1]):
            recs.append(r[int(rec_off[k]):int(rec_off[k + 1])])
            roffs.append(roffs[-1] + len(recs[-1]))
        rems.append(rb[int(roff[c]):int(roff[c + 1])])
        starts.append(int(start[c]))
    pbuf = np.frombuffer(b"".join(parts), np.uint8).copy()
    poff = np.cumsum([0] + [len(p) for p in parts]).astype(np.uint32)
    prec = np.frombuffer(b"".join(recs) or b"\0", np.uint8)[:roffs[-1]].copy()
    prem = np.frombuffer(b"".join(rems) or b"\0", np.uint8).copy()
    proff = np.cumsum([0] + [len(x) for x in rems]).astype(np.uint32)
    plog = ConnLog(prem, proff, np.array(starts, np.int64), TL.LOG_NS, TL.TZ)
    pg = eng.serve_connections(pbuf, poff, CC.DATE, 12345, results=(prec, np.array(roffs, np.uint32)), log=plog,
                               trace_key=keys[perm])
    prf = pg.req_first.astype(np.int64)
    for i, c in enumerate(perm.tolist()):
        k0, k1, p0, p1 = rf[c], rf[c + 1], prf[i], prf[i + 1]
        assert k1 - k0 == p1 - p0
        assert base.out[base.out_off[k0]:base.out_off[k1]].tobytes() == pg.out[pg.out_off[p0]:pg.out_off[p1]].tobytes(), c
        assert np.array_equal(base.meta[k0:k1], pg.meta[p0:p1]) and np.array_equal(base.trace_ids[k0:k1], pg.trace_ids[p0:p1])
        assert base.consumed[c] == pg.consumed[i] and base.conn_status[c] == pg.conn_status[i]
        m0, m1_ = np.searchsorted(base.log.log_req, [k0, k1])
        q0, q1 = np.searchsorted(pg.log.log_req, [p0, p1])
        assert base.log.out[base.log.log_off[m0]:base.log.log_off[m1_]].tobytes() == pg.log.out[pg.log.log_off[q0]:pg.log.log_off[q1]].tobytes()
    eng.close()


def _closure_records(spec, route, c, fixed=False):
    """what a caller's closures produce for its routed read c (the model's closure with index c * 1000 + j, or 0 for every
    request when fixed)"""
    recs = []
    for j in range(len(route.meta)):
        st, rid = int(route.meta[j]) & 0xFFFF, int(route.meta[j]) >> 16
        if st == 0 and rid != 0xFFFF:
            path, _, body = CC.parsed(route.desc, route.arena, j)
            recs.append(CC.closure(spec, rid, 0 if fixed else c * 1000 + j, path, body))
        else:
            recs.append(b"")
    return b"".join(recs), np.cumsum([0] + [len(x) for x in recs]).astype(np.uint32)


def model_for_reads(spec, buf, off, ids, remote=None, roff=None, start=None):
    """the closure-path model for the reads buf[off[c]:off[c + 1]] as one batch, with the ids their route calls returned and
    the records _closure_records gives each read → (records of the whole batch, test_conn_closures.model_stage2's dict)"""
    m1 = CC._model(spec, buf, off, 0)
    m1["trace_ids"] = ids
    rf = m1["req_first"].astype(np.int64)
    recs = []
    for c in range(len(off) - 1):
        for j in range(rf[c + 1] - rf[c]):
            k = rf[c] + j
            st, rid = int(m1["meta"][k]) & 0xFFFF, int(m1["meta"][k]) >> 16
            recs.append(CC.closure(spec, rid, c * 1000 + j, *CC.parsed(m1["desc"], m1["arena"], k)[::2])
                        if st == 0 and rid != 0xFFFF else b"")
    rec = np.frombuffer(b"".join(recs) or b"\0", np.uint8)[:sum(map(len, recs))].copy()
    rec_off = np.cumsum([0] + [len(x) for x in recs]).astype(np.uint32)
    return b"".join(recs), CC.model_stage2(spec, m1, rec, rec_off, remote, roff, start)


def _app_front_end(eng, log, route_schema, **kw):
    from gofr_b200.frontend import ConnAppFrontend
    fe = ConnAppFrontend(eng, log=log, tz_offset_s=TL.TZ, seed=SEED, route_schema=route_schema, **kw)
    fe.set_clock(TL.LOG_NS)
    return fe


def _bind_rows(eng, route):
    """gofr_batch_bind on the caller's exported (desc, trace_ids, arena) → [(status, row)] per request"""
    b = route.route.batch
    if not b.n:
        return []
    rb = _abi.ReqBatch(desc=b.desc.ctypes.data, trace_ids=b.trace_ids.ctypes.data, arena=b.arena.ctypes.data,
                       arena_bytes=b.arena.size, n=b.n, date=b"")
    slot = 1024
    rows, ln, st = np.zeros(b.n * slot, np.uint8), np.zeros(b.n, np.uint32), np.zeros(b.n, np.uint32)
    _abi.check(_abi.lib().gofr_batch_bind(eng._e, 7, C.byref(rb), rows.ctypes.data, slot, ln.ctypes.data, st.ctypes.data), "bind")
    return [(int(st[i]), rows[i * slot:i * slot + int(ln[i])].tobytes()) for i in range(b.n)]


@pytest.mark.gpu
@pytest.mark.parametrize("log", [True, False])
@pytest.mark.parametrize("max_batch,wait_us,threads", TF.REGIMES)
def test_gpu_reads_equal_model(max_batch, wait_us, threads, log):
    """config 1 with closure routes (three of them binding main.Item), streams with tails, defers and holes: each read routed,
    its closures run and its records handed back from its own thread; every caller against the model evaluated with the ids
    its route call returned, every X-Correlation-Id the route call's id, and the binds equal gofr_batch_bind's on the
    caller's exported batch"""
    spec, rs = _c1_route_schema()
    eng = CC._engine(spec)
    fe = _app_front_end(eng, log, rs, max_batch=max_batch, max_wait_us=wait_us, max_conn_bytes=64 << 10)
    buf, off = CC._streams(900 if max_batch > 1 else 300, seed=max_batch)
    n = len(off) - 1
    reads = [buf[int(off[c]):int(off[c + 1])].tobytes() for c in range(n)]
    remote, roff, start = TL._clients(n, seed=max_batch)
    rems = [remote[int(roff[c]):int(roff[c + 1])].tobytes() for c in range(n)]
    routes, got, recs = [None] * n, [None] * n, [None] * n

    def work(t):
        for c in range(t, n, threads):
            r = fe.route(reads[c])
            rec, rec_off = _closure_records(spec, r.route, c)
            routes[c], recs[c] = r, (rec, rec_off)
            got[c] = fe.respond(reads[c], r.trace_key, rec, rec_off, rems[c], int(start[c]))

    TF.run_threads(threads, work)
    ids = np.concatenate([r.route.trace_ids for r in routes])
    mrec, want = model_for_reads(spec, buf, off, ids, *((remote, roff, start) if log else ()))
    assert mrec == b"".join(r for r, _ in recs)     # the closures saw the model's parsed requests
    g = TF.assemble(got, reads)
    CC._check_stage2(g, want, (max_batch, log))
    assert np.array_equal(g.trace_ids, ids)
    assert TF.check_ids(g) > 0
    for c in range(0, n, 5):   # each route call's parsed forms: the model's, 4-aligned in the caller's arena
        got_r = routes[c].route
        r1 = CC._model(spec, buf[int(off[c]):int(off[c + 1])].copy(), np.array([0, len(reads[c])], np.uint32), 0)
        for k in ("meta", "vars", "req_at", "req_first", "consumed", "conn_status"):
            assert np.array_equal(np.asarray(getattr(got_r, k)), r1[k]), (c, k)
        assert (got_r.desc["arena_off"] % 4 == 0).all()
        for j in range(len(got_r.meta)):
            assert CC.parsed(got_r.desc, got_r.arena, j) == CC.parsed(r1["desc"], r1["arena"], j), (c, j)
    # the binds: what gofr_batch_bind gives on the caller's own exported batch
    n_bound = 0
    for c in range(0, n, 7):
        r = routes[c]
        want_rows = _bind_rows(eng, r)
        for j in range(len(r.route.meta)):
            st, rid = int(r.route.meta[j]) & 0xFFFF, int(r.route.meta[j]) >> 16
            row = r.rows[int(r.row_off[j]):int(r.row_off[j + 1])].tobytes()
            if st == 0 and rid in rs:
                assert (int(r.bind_status[j]), row) == want_rows[j], (c, j)
                n_bound += 1
            else:
                assert int(r.bind_status[j]) == 0xFFFFFFFF and row == b"", (c, j)
    assert n_bound > 0
    st = fe.stats()
    assert st["route_reads"] == st["respond_reads"] == sum(1 for x in reads if x) and st["isolated"] == 0
    if max_batch == 1:
        assert st["route_batches"] == st["respond_batches"] == st["route_reads"]
    fe.close()
    eng.close()


@pytest.mark.gpu
def test_gpu_cut_streams_equal_the_whole_stream():
    """reads cut at seeded places with the tails kept on MORE: the concatenated answers and final state equal the whole
    stream's through gofr_conn_batch_route / _respond as one batch"""
    spec, rs = _c1_route_schema()
    eng = CC._engine(spec)
    fe = _app_front_end(eng, False, rs, max_batch=32, max_wait_us=300, max_conn_bytes=64 << 10)
    buf, off = CC._streams(240, seed=21)
    n = len(off) - 1
    streams = [buf[int(off[c]):int(off[c + 1])].tobytes() for c in range(n)]
    per = [None] * n
    threads = 16

    def work(t):
        rnd = random.Random(2000 + t)
        for c in range(t, n, threads):
            s, held, pos, calls = streams[c], b"", 0, []
            for cut in TF._cuts(rnd, len(s)):
                held += s[pos:cut]
                pos = cut
                r = fe.route(held)
                rec, rec_off = _closure_records(spec, r.route, 0, fixed=True)
                g = fe.respond(held, r.trace_key, rec, rec_off)
                assert np.array_equal(g.trace_ids, r.route.trace_ids)
                calls.append(g)
                held = held[int(g.consumed[0]):]
                if int(g.conn_status[0]) == DEFER:
                    break
            per[c] = (calls, held + s[pos:])

    TF.run_threads(threads, work)
    r1 = eng.route_connections(buf, off, 0)
    rec, rec_off = _closure_records(spec, r1, 0, fixed=True)
    whole = eng.serve_connections(buf, off, CC.DATE, 0, results=(np.frombuffer(rec or b"\0", np.uint8)[:len(rec)].copy(), rec_off))
    strip = lambda b: re.sub(rb"X-Correlation-Id: [0-9a-f]{32}\r\n", b"", b)
    for c in range(n):
        calls, left = per[c]
        g = TF.assemble(calls, [b""] * len(calls))
        k0, k1 = int(whole.req_first[c]), int(whole.req_first[c + 1])
        assert np.array_equal(g.meta, whole.meta[k0:k1]), c
        assert strip(g.out.tobytes()) == strip(whole.out[int(whole.out_off[k0]):int(whole.out_off[k1])].tobytes()), c
        assert int(g.conn_status[-1]) == int(whole.conn_status[c]), c
        assert left == streams[c][int(whole.consumed[c]):], c
    assert sum(len(calls) for calls, _ in per) > 2 * n
    fe.close()
    eng.close()


@pytest.mark.gpu
def test_gpu_parked_caller_and_shared_engine():
    """a caller parked between its two calls while the other threads each finish full route → respond cycles, beside a
    gofr_conn_frontend and a gofr_frontend on the same engine: everybody finishes with the model's answers"""
    from gofr_b200.frontend import ConnFrontend, Frontend
    spec, rs = _c1_route_schema()
    eng = CC._engine(spec)
    fe = _app_front_end(eng, True, rs, max_batch=16, max_wait_us=200, max_conn_bytes=64 << 10)
    cf = ConnFrontend(eng, max_batch=16, max_wait_us=200, max_conn_bytes=64 << 10, log=True, tz_offset_s=TL.TZ, seed=1)
    cf.set_clock(TL.LOG_NS)
    pf = Frontend(eng, max_batch=16, max_wait_us=200, slot_bytes=1024, max_request_bytes=2048)
    buf, off = CC._streams(200, seed=33)
    n = len(off) - 1
    reads = [buf[int(off[c]):int(off[c + 1])].tobytes() for c in range(n)]
    got, routes, others_done = [None] * n, [None] * n, threading.Event()
    done_count = [0]
    lock = threading.Lock()
    threads = 8

    def work(t):
        if t == 0:       # parked: routes, then waits for every other thread to finish its reads
            r = fe.route(reads[0])
            assert others_done.wait(300)
            rec, rec_off = _closure_records(spec, r.route, 0)
            routes[0], got[0] = r, fe.respond(reads[0], r.trace_key, rec, rec_off)
            return
        for c in range(t, n, threads - 1):
            r = fe.route(reads[c])
            rec, rec_off = _closure_records(spec, r.route, c)
            routes[c], got[c] = r, fe.respond(reads[c], r.trace_key, rec, rec_off)
            cf.serve(reads[c])
            pf.serve(0, b"/hello", b"name=x", resp_cap=65536)
        with lock:
            done_count[0] += 1
            if done_count[0] == threads - 1:
                others_done.set()

    TF.run_threads(threads, work)
    _, want = model_for_reads(spec, buf, off, np.concatenate([r.route.trace_ids for r in routes]))
    CC._check_stage2(TF.assemble(got, reads), want, "parked")
    pf.close()
    cf.close()
    fe.close()
    eng.close()


def _compile_example(exe):
    from gofr_b200 import _build
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "cpp", "conn_app_frontend.cpp"), "-o", exe, _build.LIB,
                           "-Wl,-rpath," + os.path.dirname(_build.LIB)])


def test_cpp_example_compiles(tmp_path):
    _abi.lib()
    _compile_example(str(tmp_path / "conn_app_frontend"))


@pytest.mark.gpu
def test_gpu_cpp_example(tmp_path):
    """examples/cpp/conn_app_frontend.cpp: the reference's server-routes app, every route a gofr::App closure, served by one
    thread per connection through App::ServeRead on pipelined reads cut at arbitrary places with the tails kept; it checks
    every body the reference expects, every X-Correlation-Id against the id returned for it, and that no id repeats"""
    _abi.lib()
    exe = str(tmp_path / "conn_app_frontend")
    _compile_example(exe)
    r = subprocess.run([exe, "16", "4"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ": ok" in r.stdout, r.stdout
