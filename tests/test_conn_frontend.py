"""gofr_conn_frontend_*: many threads hand in one read of one connection each, as net/http's connection goroutines read, and
each gets back what gofr_conn_batch_submit_log gives for that connection as a batch of one, with the trace ids of the batch
it joined.

Without a GPU: the fan-in / fan-out of conn_frontend.cpp against stub batch calls under ThreadSanitizer (reads of 0 bytes
and past max_conn_bytes, short caller capacities and the rerun after an output grows included), argument checks and the
ctypes prototypes.  On the GPU, against the model of test_conn_log.py (framer → request heads → serve → log) evaluated with
the ids and the Date each call returned: three batching regimes with and without lines, cut streams whose concatenated
answers equal the whole stream's, output growth, short caller capacities, and a per-request front-end on the same engine."""
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
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.engine import ConnLogLines, ConnResponses
from tests import oracle as O
from tests import test_conn_batch as CB
from tests import test_conn_log as TL

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INVALID, CAPACITY = 1, 7
DONE, MORE, DEFER = 0, 1, 2
CLOCK_NS = TL.LOG_NS                       # Date and log time of every batch
DATE = S.http_date(CLOCK_NS // 10**9)
SEED = 0x5EED

# what closes the batches: the timer (16 callers < 64), a full batch (the timer is far away), every read alone
REGIMES = [(64, 200, 16), (8, 100000, 32), (1, 0, 16)]


# ---------------------------------------------------------------------------------------------------------------
# without a GPU
# ---------------------------------------------------------------------------------------------------------------
def _stress_exe():
    exe = os.path.join(HERE, "emu", "conn_frontend_stress")
    srcs = [os.path.join(HERE, "emu", "conn_frontend_stress.cpp")] + \
           [os.path.join(ROOT, "gofr_b200", "csrc", f) for f in ("conn_frontend.cpp", "frontend_ring.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-Wall", "-Wextra", srcs[0],
                               "-o", exe], cwd=os.path.dirname(exe))
    return exe


@pytest.mark.parametrize("args", [
    "16 200 64 200 2000 1",      # batches close on the timer (16 callers < 64)
    "32 100 8 100000 1500 1",    # batches close because they are full
    "16 50 1 0 300 1",           # one read per batch
    "64 50 16 100 800 1",
    "16 200 64 200 2000 0",      # without lines
    "32 100 8 100000 4000 0",
    "64 40 64 100000 200 0",     # full batches of 64: batch b's slot c and batch c's slot b draw distinct ids
])
def test_conn_frontend_fan_in_fan_out_tsan(args):
    """no GPU: the batching of conn_frontend.cpp against stub batch calls that check every batch as the engine does, under
    ThreadSanitizer — every caller gets the answer made from ITS read, remote string and clock, rebased to its buffers;
    callers one byte short get GOFR_ERR_CAPACITY with the exact need; an empty read is answered without a batch and a read
    past max_conn_bytes is refused; batches never exceed max_batch; a batch refused for its output capacity is served again;
    every trace id is distinct; nothing races."""
    r = subprocess.run([_stress_exe()] + args.split(), capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ThreadSanitizer" not in r.stderr, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    t, n, max_batch = (int(v) for v in args.split()[:3])
    assert res["bad"] == 0 and res["violations"] == 0 and res["largest"] <= max_batch
    assert res["conns"] == res["queued"] and res["queued"] + res["empty"] + res["over"] == t * n
    assert res["short"] > 0 and res["empty"] > 0 and res["at_max"] > 0 and res["over"] > 0 and res["ids"] > 0
    assert res["stub_batches"] == res["batches"] + res["reruns"] and res["reruns"] == res["refused"]
    if max_batch >= 8:
        assert res["reruns"] > 0
    if max_batch == 1:
        assert res["batches"] == res["queued"]


def test_conn_frontend_argument_checks():
    """no GPU: the entry points refuse bad arguments before they allocate or queue anything"""
    L = _abi.lib()
    f = C.c_void_p()
    fake = C.c_void_p(0x10)
    assert L.gofr_conn_frontend_create(C.byref(f), None, 16, 100, 4096, 1, 0, 1) == INVALID
    assert L.gofr_conn_frontend_create(None, fake, 16, 100, 4096, 1, 0, 1) == INVALID
    assert L.gofr_conn_frontend_create(C.byref(f), fake, 0, 100, 4096, 1, 0, 1) == INVALID
    assert L.gofr_conn_frontend_create(C.byref(f), fake, 1 << 31, 100, 1, 1, 0, 1) == INVALID
    # max_batch * max_conn_bytes past the ring's 32-bit arena claim
    assert L.gofr_conn_frontend_create(C.byref(f), fake, 1 << 16, 100, 1 << 16, 1, 0, 1) == CAPACITY
    assert L.gofr_conn_frontend_create(C.byref(f), fake, 2, 100, 0xFFFFFFFF, 0, 0, 1) == CAPACITY
    first, one = (C.c_uint32 * 2)(), (C.c_uint32 * 1)()
    cr = _abi.ConnResp(out_off=C.addressof(one), req_first=C.addressof(first), consumed=C.addressof(one), conn_status=C.addressof(one))
    assert L.gofr_conn_frontend_serve(None, b"GET", 3, b"", 0, 0, C.byref(cr), None) == INVALID
    assert L.gofr_conn_frontend_stats(None, None, None, None) == INVALID
    assert L.gofr_conn_frontend_set_clock(None, 1) == INVALID
    L.gofr_conn_frontend_destroy(None)


def test_prototypes_match_the_header():
    """the ctypes prototypes take as many arguments as include/gofr_b200.h declares, and the outputs reuse the batch call's
    structs (their layouts are checked by test_conn_batch.py and test_conn_log.py)"""
    L = _abi.lib()
    header = open(os.path.join(ROOT, "include", "gofr_b200.h")).read()
    decls = dict((m.group(1), m.group(2)) for m in re.finditer(r"\b(gofr_conn_frontend_[a-z_]+)\s*\(([^)]*)\)", header))
    assert set(decls) == {"gofr_conn_frontend_create", "gofr_conn_frontend_destroy", "gofr_conn_frontend_set_clock",
                          "gofr_conn_frontend_stats", "gofr_conn_frontend_serve"}
    for name, params in decls.items():
        assert len(getattr(L, name).argtypes) == len(params.split(",")), name
    assert L.gofr_conn_frontend_serve.argtypes[6] is C.POINTER(_abi.ConnResp)
    assert L.gofr_conn_frontend_serve.argtypes[7] is C.POINTER(_abi.ConnLog)


# ---------------------------------------------------------------------------------------------------------------
# the model: test_conn_log's composition of oracles, with the trace ids given
# ---------------------------------------------------------------------------------------------------------------
def model(spec, reads, ids, remote, start, log):
    """reads: the bytes of each call; ids: uint8[requests, 16], the ids the calls returned in call order; remote / start: each
    call's remote string and clock → test_conn_log.model's dict for the calls as one batch"""
    buf = np.frombuffer(b"".join(reads) or b"\0", np.uint8)[:sum(map(len, reads))].copy()
    off = np.cumsum([0] + [len(r) for r in reads]).astype(np.uint32)
    rec, first, consumed, status, idx, req_first, _ = CB.model_requests(buf, off, 0)
    assert len(idx) == len(ids)
    d, a, _, spans = O.http_parse(buf, rec)
    o, f, m = O.OracleTable(spec).serve(S.RequestBatch(d[idx].copy(), ids, a), DATE)
    want = dict(out=o[:int(f[-1])], out_off=f, meta=m, req_at=rec[idx].astype(np.uint32), trace_ids=ids, req_first=req_first,
                consumed=consumed, conn_status=status)
    if log:
        conn = np.repeat(np.arange(len(reads)), np.diff(req_first.astype(np.int64)))
        sel = np.nonzero(TL.logged(m, spans[idx]))[0]
        b = buf.tobytes()
        recs = []
        for k in sel.tolist():
            sp = spans[idx[k]]
            get = lambda j: b[int(sp[j] & 0xFFFFFFFF):int(sp[j] & 0xFFFFFFFF) + int(sp[j] >> 32)]
            c = int(conn[k])
            recs.append(S.LogRec(int(start[c]), CLOCK_NS - int(start[c]), CLOCK_NS, get(TL.S_METHOD), get(TL.S_UA), get(TL.S_XFF),
                                 remote[c], get(TL.S_TARGET), int(m[k] & 0xFFFF), TL.TZ, ids[k].tobytes()))
        lo, lf = O.request_log(S.LogBatch.pack(recs))
        want.update(log=lo[:int(lf[-1])], log_off=lf, log_req=sel.astype(np.uint32))
    return want


def assemble(got, reads):
    """the per-call results as one batch's ConnResponses, in call order"""
    out, out_off, meta, req_at, ids, req_first, consumed, status = [], [0], [], [], [], [0], [], []
    lout, log_off, log_req = [], [0], []
    at = 0
    for r, g in zip(reads, got):
        k0 = req_first[-1]
        out.append(g.out.tobytes())
        out_off += (g.out_off[1:].astype(np.int64) + out_off[-1]).tolist()
        meta += g.meta.tolist()
        req_at += (g.req_at.astype(np.int64) + at).tolist()
        ids.append(g.trace_ids)
        req_first.append(k0 + int(g.req_first[1]))
        consumed.append(int(g.consumed[0]))
        status.append(int(g.conn_status[0]))
        if g.log is not None:
            lout.append(g.log.out.tobytes())
            log_off += (g.log.log_off[1:].astype(np.int64) + log_off[-1]).tolist()
            log_req += (g.log.log_req.astype(np.int64) + k0).tolist()
        at += len(r)
    u32 = lambda v: np.array(v, np.uint32)
    log = None
    if got and got[0].log is not None:
        lb = b"".join(lout)
        log = ConnLogLines(np.frombuffer(lb, np.uint8), u32(log_off), u32(log_req), len(log_req), len(lb))
    return ConnResponses(np.frombuffer(b"".join(out), np.uint8), u32(out_off), u32(meta), u32(req_at),
                         np.concatenate(ids) if ids else np.zeros((0, 16), np.uint8), u32(req_first), u32(consumed), u32(status), log)


def check(spec, got, reads, remote, start, log, what=""):
    g = assemble(got, reads)
    want = model(spec, reads, g.trace_ids, remote, start, log)
    (TL._check if log else CB._check)(g, want, what)
    check_ids(g)
    return g


def check_ids(g):
    """every id is distinct, and a response with an X-Correlation-Id header carries its own id there"""
    ids = g.trace_ids
    assert len({i.tobytes() for i in ids}) == len(ids)
    resp = O.responses(g.out, g.out_off)
    headers = 0
    for k, r in enumerate(resp):
        for ln in r.split(b"\r\n\r\n", 1)[0].split(b"\r\n"):
            if ln.startswith(b"X-Correlation-Id: "):
                assert ln[len(b"X-Correlation-Id: "):] == ids[k].tobytes().hex().encode(), k
                headers += 1
    return headers


def run_threads(n_threads, work):
    errs = []

    def body(t):
        try:
            work(t)
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=body, args=(t,)) for t in range(n_threads)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in th), "front-end hung"
    assert not errs, errs


def _front_end(spec, log, **kw):
    from gofr_b200.engine import Engine
    from gofr_b200.frontend import ConnFrontend
    from gofr_b200.table import Table
    eng = Engine(Table(spec), 0)
    fe = ConnFrontend(eng, log=log, tz_offset_s=TL.TZ, seed=SEED, **kw)
    fe.set_clock(CLOCK_NS)
    return eng, fe


# ---------------------------------------------------------------------------------------------------------------
# the GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("log", [True, False])
@pytest.mark.parametrize("max_batch,wait_us,threads", REGIMES)
def test_gpu_reads_equal_model(max_batch, wait_us, threads, log):
    """config 1 (holes), requests mux answers alone, DEFER connections and MORE tails, 30 KB bodies and 9 KB headers: each
    read from its own thread, every result against the model with the ids it returned"""
    spec = synth.config1_spec()
    buf, off = TL._streams(1200 if max_batch > 1 else 400, seed=max_batch)
    n = len(off) - 1
    remote, roff, start = TL._clients(n, seed=max_batch)
    reads = [buf[int(off[c]):int(off[c + 1])].tobytes() for c in range(n)]
    rems = [remote[int(roff[c]):int(roff[c + 1])].tobytes() for c in range(n)]
    eng, fe = _front_end(spec, log, max_batch=max_batch, max_wait_us=wait_us, max_conn_bytes=64 << 10)
    got = [None] * n

    def work(t):
        for c in range(t, n, threads):
            got[c] = fe.serve(reads[c], rems[c], int(start[c]))

    run_threads(threads, work)
    g = check(spec, got, reads, rems, start, log, (max_batch, log))
    assert ((g.meta & 0xFFFF) == 0).sum() > 0 and (g.conn_status == DEFER).sum() > 0 and (g.conn_status == MORE).sum() > 0
    batches, conns, _ = fe.stats()
    assert conns == sum(1 for r in reads if r) and batches <= conns
    if max_batch == 1:
        assert batches == conns
    fe.close()
    eng.close()


def _cuts(rnd, n):
    """seeded places to cut a stream of n bytes into reads: none, a few, or every few bytes"""
    if n < 2:
        return [n]
    k = rnd.choice([0, 1, 3, 6, n // 7])
    return sorted(rnd.sample(range(1, n), min(k, n - 1))) + [n]


@pytest.mark.gpu
@pytest.mark.parametrize("log", [True, False])
def test_gpu_cut_streams_equal_the_whole_stream(log):
    """each thread feeds its connections' streams as reads cut at seeded places, keeping the tail on MORE: everything written
    equals the model's responses for the whole stream, request by request, and the final state is the whole stream's"""
    spec = synth.config1_spec()
    buf, off = TL._streams(480, seed=21)
    n = len(off) - 1
    streams = [buf[int(off[c]):int(off[c + 1])].tobytes() for c in range(n)]
    remote, roff, start = TL._clients(n, seed=21)
    rems = [remote[int(roff[c]):int(roff[c + 1])].tobytes() for c in range(n)]
    eng, fe = _front_end(spec, log, max_batch=32, max_wait_us=300, max_conn_bytes=64 << 10)
    threads = 24
    per_stream = [None] * n

    def work(t):
        rnd = random.Random(1000 + t)
        for c in range(t, n, threads):
            s, held, pos, calls = streams[c], b"", 0, []
            for cut in _cuts(rnd, len(s)):
                held += s[pos:cut]
                pos = cut
                r = fe.serve(held, rems[c], int(start[c]))
                calls.append(r)
                held = held[int(r.consumed[0]):]     # MORE: the tail the next read extends; DEFER: what net/http gets
                if int(r.conn_status[0]) == DEFER:
                    break
            per_stream[c] = (calls, held + s[pos:])

    run_threads(threads, work)
    # the whole streams, with the ids the cut reads were given, in stream order
    whole = []
    for calls, left in per_stream:
        g = assemble(calls, [b""] * len(calls))     # req_at is not compared: it is relative to each read
        whole.append((g, int(g.conn_status[-1]), left))
    ids = np.concatenate([g.trace_ids for g, _, _ in whole])
    want = model(spec, streams, ids, rems, start, log)
    for c in range(n):
        g, status, left = whole[c]
        k0, k1 = int(want["req_first"][c]), int(want["req_first"][c + 1])
        assert g.out.tobytes() == want["out"][int(want["out_off"][k0]):int(want["out_off"][k1])].tobytes(), c
        assert np.array_equal(g.meta, want["meta"][k0:k1]), c
        assert status == int(want["conn_status"][c]), c
        assert left == streams[c][int(want["consumed"][c]):], c
        if log:
            m0, m1 = np.searchsorted(want["log_req"], [k0, k1])
            assert g.log.out.tobytes() == want["log"][int(want["log_off"][m0]):int(want["log_off"][m1])].tobytes(), c
            assert np.array_equal(g.log.log_req, want["log_req"][m0:m1] - k0), c
    assert sum(len(calls) for calls, _ in per_stream) > 2 * n and (want["conn_status"] == MORE).sum() > 0
    check_ids(assemble([g for g, _, _ in whole], [b""] * n))
    fe.close()
    eng.close()


@pytest.mark.gpu
def test_gpu_outputs_grow_and_the_batch_is_served_again():
    """full batches of reads of one to three requests with 8 KB responses each pass the first 64 KiB of output: the batch is
    served again into larger outputs, and every caller still gets the model's bytes"""
    spec = synth.config1_spec()
    big = b"GET /hello?name=" + b"x" * 8000 + b" HTTP/1.1\r\nHost: h\r\n\r\n"
    reads = [big * (1 + c % 3) for c in range(64)]
    rems = [b"10.0.0.%d:80" % c for c in range(64)]
    start = np.arange(64, dtype=np.int64) + 1_700_000_000_000_000_000
    eng, fe = _front_end(spec, True, max_batch=8, max_wait_us=100000, max_conn_bytes=64 << 10)
    got = [None] * 64

    def work(t):
        for c in range(t, 64, 8):
            got[c] = fe.serve(reads[c], rems[c], int(start[c]))

    run_threads(8, work)
    g = check(spec, got, reads, rems, start, True)
    assert len(g.meta) == sum(1 + c % 3 for c in range(64)) and int(g.out_off[-1]) > len(g.meta) * 8000
    _, conns, reruns = fe.stats()
    assert conns == 64 and reruns > 0
    fe.close()
    eng.close()


def _serve_raw(fe, read, out_cap, req_cap, line_cap, log_cap):
    """gofr_conn_frontend_serve with the caller's capacities → (rc, out_bytes, requests, lines, log bytes, out)"""
    out = np.zeros(max(out_cap, 1), np.uint8)
    out_off, meta, at = np.zeros(req_cap + 1, np.uint32), np.zeros(max(req_cap, 1), np.uint32), np.zeros(max(req_cap, 1), np.uint32)
    first, one, two = np.zeros(2, np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint32)
    lout, loff, lreq = np.zeros(max(log_cap, 1), np.uint8), np.zeros(line_cap + 1, np.uint32), np.zeros(max(line_cap, 1), np.uint32)
    cr = _abi.ConnResp(out=out.ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data,
                       req_at=at.ctypes.data, req_first=first.ctypes.data, consumed=one.ctypes.data, conn_status=two.ctypes.data)
    cl = _abi.ConnLog(line_cap=line_cap, out=lout.ctypes.data, out_cap=log_cap, log_off=loff.ctypes.data, log_req=lreq.ctypes.data)
    rc = _abi.lib().gofr_conn_frontend_serve(fe._f, read, len(read), b"", 0, 0, C.byref(cr), C.byref(cl))
    return rc, int(cr.out_bytes), int(first[1]), int(cl.lines), int(cl.out_bytes), out


@pytest.mark.gpu
def test_gpu_short_caller_capacities():
    """a caller one byte, request or line short gets GOFR_ERR_CAPACITY with what it needed; the next calls on the same
    front-end are served correctly"""
    spec = synth.config1_spec()
    eng, fe = _front_end(spec, True, max_batch=4, max_wait_us=50, max_conn_bytes=64 << 10)
    read = b"".join(m for m, _ in CB.GOOD[:4])
    full = fe.serve(read)
    nb, nr, nl, lb = len(full.out), len(full.meta), full.log.lines, full.log.out_bytes
    assert nb > 0 and nr > 1 and nl > 0
    assert _serve_raw(fe, read, nb, nr, nl, lb)[0] == 0
    for caps in ((nb - 1, nr, nl, lb), (nb, nr - 1, nl, lb), (nb, nr, nl - 1, lb), (nb, nr, nl, lb - 1)):
        rc, ob, reqs, lines, lbytes, out = _serve_raw(fe, read, *caps)
        assert rc == CAPACITY and (ob, reqs, lines, lbytes) == (nb, nr, nl, lb), caps
    with pytest.raises(_abi.GofrError):          # a read past max_conn_bytes: refused before it is queued
        fe.serve(b"G" * ((64 << 10) + 1))
    empty = fe.serve(b"")                        # nothing to frame: answered without a batch
    assert int(empty.conn_status[0]) == DONE and len(empty.meta) == 0
    reads = [read] * 6
    got = [fe.serve(r) for r in reads]
    check(spec, got, reads, [b""] * 6, np.zeros(6, np.int64), True)
    fe.close()
    eng.close()


@pytest.mark.gpu
def test_gpu_per_request_and_connection_front_ends_share_an_engine():
    """a gofr_frontend and a gofr_conn_frontend on one engine, both busy at once: both give the oracle's answers"""
    from gofr_b200.frontend import Frontend
    from tests import test_frontend as TF
    spec = synth.config1_spec()
    eng, fe = _front_end(spec, True, max_batch=32, max_wait_us=200, max_conn_bytes=64 << 10)
    pf = Frontend(eng, max_batch=32, max_wait_us=200, slot_bytes=1024, max_request_bytes=2048)
    pf.set_clock(CLOCK_NS // 10**9)
    batch = synth.config1_batch(400)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    reqs = TF._requests(batch)
    buf, off = TL._streams(400, seed=8)
    n = len(off) - 1
    reads = [buf[int(off[c]):int(off[c + 1])].tobytes() for c in range(n)]
    remote, roff, start = TL._clients(n, seed=8)
    rems = [remote[int(roff[c]):int(roff[c + 1])].tobytes() for c in range(n)]
    got, per = [None] * n, [None] * batch.n

    def work(t):
        if t % 2:
            for c in range(t // 2, n, 8):
                got[c] = fe.serve(reads[c], rems[c], int(start[c]))
        else:
            for i in range(t // 2, batch.n, 8):
                m, p, q, d, tid, fl = reqs[i]
                per[i] = pf.serve(m, p, q, d, tid, fl, resp_cap=65536)

    run_threads(16, work)
    check(spec, got, reads, rems, start, True)
    ob = o1.tobytes()
    for i, (resp, meta) in enumerate(per):
        assert resp == ob[int(f1[i]):int(f1[i + 1])] and meta == int(m1[i]), i
    pf.close()
    fe.close()
    eng.close()


def _compile_example(exe):
    from gofr_b200 import _build
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "cpp", "conn_frontend.cpp"), "-o", exe, _build.LIB,
                           "-Wl,-rpath," + os.path.dirname(_build.LIB)])


def test_cpp_example_compiles(tmp_path):
    _abi.lib()
    _compile_example(str(tmp_path / "conn_frontend"))


@pytest.mark.gpu
def test_gpu_cpp_example(tmp_path):
    """examples/cpp/conn_frontend.cpp: threads that own connections send the reference's route-test requests as reads cut
    at arbitrary places through gofr::ConnFrontend, keep the tails, answer the holes with App::ServeHTTP, and check every body
    the reference expects, every X-Correlation-Id against its returned id, and the final state of every connection"""
    _abi.lib()
    exe = str(tmp_path / "conn_frontend")
    _compile_example(exe)
    r = subprocess.run([exe, "16", "6"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ": ok" in r.stdout, r.stdout
