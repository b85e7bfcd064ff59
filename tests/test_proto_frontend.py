"""gofr_proto_frontend_*: many threads hand in one gRPC message (or one response row) each, as grpc-go calls its codec once per
message, and each gets back what gofr_proto_batch_decode / _encode give for that record alone.

Without a GPU: argument checks on the library, the fan-in / fan-out of proto_frontend.cpp against stub batch calls under
ThreadSanitizer, and the build of examples/cpp/grpc_server.cpp.  On the GPU, in child processes (H.run_child): decode and
encode against the batch calls and the model in three batching regimes, a decode and an encode front-end beside the HTTP
front-end on one engine, capacities, and the example against python protobuf."""
import ctypes as C
import json
import os
import random
import subprocess
import threading

import pytest

from gofr_b200 import _abi
from gofr_b200 import _build
from gofr_b200 import spec as S
from tests import proto_nested_harness as H
from tests import proto_nested_model as M
from tests import test_proto_batch as PB

F = S.ProtoNField
OK, BAD_UTF8, BAD_ROW, DEFER = S.GRPC_OK, S.GRPC_BAD_UTF8, S.GRPC_BAD_ROW, S.GRPC_DEFER
INVALID, CAPACITY = 1, 7
ROOT = H.ROOT_DIR
HERE = os.path.dirname(os.path.abspath(__file__))

# what closes the batches: the timer (16 callers < 64), a full batch (the timer is far away), every record alone
REGIMES = [(64, 200, 16), (8, 100000, 32), (1, 0, 4)]


# ---------------------------------------------------------------------------------------------------------------
# without a GPU
# ---------------------------------------------------------------------------------------------------------------
def _create(engine, msgs, decode=1, max_batch=16, max_wait_us=100, max_record_bytes=1024, root=0):
    nm, nf, k = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    f = C.c_void_p()
    rc = _abi.lib().gofr_proto_frontend_create(C.byref(f), engine, nm.ctypes.data, len(msgs), nf.ctypes.data, k, root,
                                               None if pr is None else pr.ctypes.data, decode, max_batch, max_wait_us,
                                               max_record_bytes)
    return rc, f


def _bound_code(msgs, decode, root=0):
    nm, nf, k = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    pb, prec = C.c_uint32(), C.c_uint32()
    return _abi.lib().gofr_proto_nested_bound(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root,
                                              None if pr is None else pr.ctypes.data, decode, C.byref(pb), C.byref(prec))


def test_proto_frontend_argument_checks():
    """no GPU: the entry points refuse bad arguments before they touch anything.  create looks at the engine only after
    its arguments, the description and the capacity have passed, so a dummy engine handle stands in for the refusals."""
    L = _abi.lib()
    msgs = [[F(1, S.PB_STRING)]]
    fake = C.c_void_p(0x10)
    assert _create(None, msgs)[0] == INVALID
    nm, nf, k = S.proto_nested_tables(msgs)
    assert L.gofr_proto_frontend_create(None, fake, nm.ctypes.data, 1, nf.ctypes.data, k, 0, None, 1, 16, 100, 1024) == INVALID
    assert _create(fake, msgs, max_batch=0)[0] == INVALID
    # a bad description: the code gofr_proto_nested_bound gives for it, in both directions
    for bad, root, _ in H.LIMIT_DESCRIPTIONS + [([[F(1, S.PB_STRING)]], 1, None)]:
        for decode in (0, 1):
            want = _bound_code(bad, decode, root)
            if want != 0:
                assert _create(fake, bad, decode=decode, root=root)[0] == want, (bad, root)
    # max_batch * (per_byte * (max_record_bytes + 5) + per_record) beyond the batch call's 32-bit offsets
    for decode in (0, 1):
        pb, prec = PB.nested_bound(msgs, 0, bool(decode))
        big = (1 << 32) // (pb * (1024 + 5) + prec) + 1
        assert _create(fake, msgs, decode=decode, max_batch=big)[0] == CAPACITY
        assert _create(fake, msgs, decode=decode, max_batch=16, max_record_bytes=0xFFFFFFFF)[0] == CAPACITY
    n, st = C.c_uint32(), C.c_uint32()
    buf = C.create_string_buffer(8)
    assert L.gofr_proto_frontend_call(None, b"x", 1, buf, 8, C.byref(n), C.byref(st)) == INVALID
    assert L.gofr_proto_frontend_stats(None, None, None) == INVALID
    L.gofr_proto_frontend_destroy(None)


def _stress_exe():
    exe = os.path.join(HERE, "emu", "proto_frontend_stress")
    srcs = [os.path.join(HERE, "emu", "proto_frontend_stress.cpp")] + \
           [os.path.join(ROOT, "gofr_b200", "csrc", f) for f in ("proto_frontend.cpp", "frontend_ring.h")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-Wall", "-Wextra", srcs[0],
                               "-o", exe], cwd=os.path.dirname(exe))
    return exe


@pytest.mark.parametrize("args", [
    "1 16 200 64 200 256",       # decode, batches close on the timer (16 callers < 64)
    "1 32 100 8 100000 256",     # decode, batches close because they are full
    "1 4 50 1 0 64",             # decode, one record per batch
    "0 16 200 64 200 300",       # encode: rows padded to 4
    "0 32 100 8 100000 1000",
    "0 4 50 1 0 64",
    "1 64 50 16 100 0",          # every record empty: max_record_bytes 0
])
def test_proto_frontend_fan_in_fan_out_tsan(args):
    """no GPU: the batching of proto_frontend.cpp against stub batch calls that check every batch as the engine does, under
    ThreadSanitizer — every caller gets the result made from ITS record (empty ones and ones at max_record_bytes included),
    callers one byte short get GOFR_ERR_CAPACITY with the exact length, batches never exceed max_batch, nothing races."""
    r = subprocess.run([_stress_exe()] + args.split(), capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1"))
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ThreadSanitizer" not in r.stderr, r.stderr
    res = json.loads(r.stdout.strip().splitlines()[-1])
    _, t, n, max_batch, _, max_rec = (int(v) for v in args.split())
    assert res["bad"] == 0 and res["violations"] == 0 and res["records"] == t * n and res["largest"] <= max_batch
    assert res["short"] > 0 and res["empty"] > 0 and res["at_max"] > 0
    if max_batch == 1:
        assert res["batches"] == t * n


def _compile_server(exe):
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-pthread", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "cpp", "grpc_server.cpp"), "-o", exe, _build.LIB,
                           "-Wl,-rpath," + os.path.dirname(_build.LIB)])


def test_grpc_server_compiles(tmp_path):
    _abi.lib()
    _compile_server(str(tmp_path / "grpc_server"))


# ---------------------------------------------------------------------------------------------------------------
# the GPU (child processes)
# ---------------------------------------------------------------------------------------------------------------
def _records(data, off):
    return [bytes(data[int(off[i]):int(off[i + 1])]) for i in range(len(off) - 1)]


def _run_calls(fe, inputs, threads):
    """every input through fe.call from `threads` threads at once → [(bytes, status)]"""
    got = [None] * len(inputs)
    errs = []

    def work(t):
        try:
            for i in range(t, len(inputs), threads):
                got[i] = fe.call(inputs[i])
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in range(threads)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in th), "front-end hung"
    assert not errs, errs
    return got


def _unpadded(row):
    k = 0
    while k < 3 and k < len(row) and row[-1 - k] == 0:
        k += 1
    return row[:len(row) - k]


def _type_sets(rnd):
    """(msgs, values maker): the harness's random map and presence type sets"""
    return [(H.rand_map_types(rnd), H.rand_map_value), (H.rand_presence_types(rnd), H.rand_presence_value),
            (H.rand_map_types(rnd), H.rand_map_value)]


def _decode_sets(rnd, n):
    """(msgs, frames): random type sets, then the large-map type with 65..4097 entries and singular messages sent twice
    (DEFER); every seventh frame damaged"""
    sets = []
    for msgs, make in _type_sets(rnd):
        rows, off = S.pack_proto_nested_rows(msgs, 0, [make(rnd, msgs, 0) for _ in range(n)])
        frames, meta = M.encode(msgs, 0, rows, off)
        sets.append((msgs, [f for f, m in zip(frames, meta) if m == OK]))
    sets.append((PB.LM_MSGS, PB._lm_frames(rnd, n)))
    return [(msgs, PB._damage(rnd, frames)) for msgs, frames in sets]


def _gpu_decode(seed):
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.frontend import ProtoFrontend
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    eng = Engine(Table(synth.config1_spec()), 0)
    checked, statuses = 0, set()
    for msgs, frames in _decode_sets(rnd, 400):
        want_rows, want_meta = PB.model_decode(msgs, frames)
        want_rows = [bytes(r) for r in want_rows]
        raw, in_off = H.pack_frames(frames)
        b_out, b_off, b_meta = eng.proto_decode_batch(msgs, 0, raw, in_off)       # the frames as one batch
        b_rows = _records(b_out, b_off)
        assert list(b_meta) == list(want_meta) and b_rows == want_rows
        max_rec = max(len(f) for f in frames)
        for max_batch, wait_us, threads in REGIMES:
            fe = ProtoFrontend(eng, msgs, 0, True, max_batch=max_batch, max_wait_us=wait_us, max_record_bytes=max_rec)
            n = len(frames) if max_batch > 1 else 120
            got = _run_calls(fe, [f[5:] for f in frames[:n]], threads)
            for i, (row, status) in enumerate(got):
                assert (row, status) == (b_rows[i], int(b_meta[i])), (i, status, int(b_meta[i]))
            batches, records = fe.stats()
            assert records == n and (batches == n if max_batch == 1 else batches <= n)
            fe.close()
            checked += n
            statuses |= {s for _, s in got}
    assert {OK, DEFER, S.GRPC_BAD_PROTO} <= statuses, statuses
    eng.close()
    print("%d messages decoded one call at a time, equal to the batch call and the model" % checked)


def _gpu_encode(seed):
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.frontend import ProtoFrontend
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    eng = Engine(Table(synth.config1_spec()), 0)
    checked, statuses = 0, set()
    utf = [[F(1, S.PB_STRING), F(2, S.PB_MESSAGE, True, 1)], [F(1, S.PB_STRING, True)]]
    utf_make = lambda rnd, msgs, m: ["ok" if rnd.random() < 0.8 else "\udcff", [["a", "\udcfe" if rnd.random() < 0.1 else "b"]]]
    for msgs, make in _type_sets(rnd) + [(utf, utf_make)]:
        rows, off = PB._spoil(rnd, msgs, [make(rnd, msgs, 0) for _ in range(400)])
        frames, meta = M.encode(msgs, 0, rows, off)
        want = [f[5:] for f in frames]
        b_out, b_off, b_meta = eng.proto_encode_batch(msgs, 0, rows, off)
        assert list(b_meta) == list(meta) and [f[5:] for f in _records(b_out, b_off)] == want
        # every third row handed in without the zero bytes that end its last word: the front-end pads it again
        inputs = [_unpadded(r) if i % 3 == 0 else r for i, r in enumerate(_records(rows, off))]
        max_rec = max(len(r) for r in inputs)
        for max_batch, wait_us, threads in REGIMES:
            fe = ProtoFrontend(eng, msgs, 0, False, max_batch=max_batch, max_wait_us=wait_us, max_record_bytes=max_rec)
            n = len(inputs) if max_batch > 1 else 120
            got = _run_calls(fe, inputs[:n], threads)
            for i, (msg, status) in enumerate(got):
                assert (msg, status) == (want[i], int(meta[i])), (i, status, int(meta[i]))
            fe.close()
            checked += n
            statuses |= {s for _, s in got}
    assert {OK, BAD_ROW, BAD_UTF8} <= statuses, statuses
    eng.close()
    print("%d rows encoded one call at a time, equal to the batch call and the model" % checked)


def _gpu_both_servers(seed):
    """a decode and an encode front-end and the HTTP front-end on one engine: unary RPCs (decode → closure → encode)
    interleaved with config-2 HTTP requests"""
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.frontend import Frontend, ProtoFrontend
    from gofr_b200.table import Table
    from tests import oracle as O
    from tests.test_frontend import CLOCK, DATE, _requests
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    spec, batch = synth.config2_spec(), synth.config2_batch(600, escape_every=5)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    ob = o1.tobytes()
    reqs = _requests(batch)
    msgs = H.rand_map_types(rnd)
    values = [H.rand_map_value(rnd, msgs, 0) for _ in range(600)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, meta = M.encode(msgs, 0, rows, off)
    frames = [f for f, m in zip(frames, meta) if m == OK]
    want_rows, want_meta = PB.model_decode(msgs, frames)
    want_rows = [bytes(r) for r in want_rows]
    eng = Engine(Table(spec), 0)
    http = Frontend(eng, max_batch=32, max_wait_us=200, slot_bytes=1024, max_request_bytes=2048)
    http.set_clock(CLOCK)
    max_rec = max(len(f) for f in frames) + max(len(r) for r in want_rows)
    dec = ProtoFrontend(eng, msgs, 0, True, max_batch=32, max_wait_us=200, max_record_bytes=max_rec)
    enc = ProtoFrontend(eng, msgs, 0, False, max_batch=32, max_wait_us=200, max_record_bytes=max_rec)
    threads, bad, errs = 24, [], []

    def work(t):
        try:
            for i in range(t, max(len(frames), len(reqs)), threads):
                if i < len(frames):
                    row, st = dec.call(frames[i][5:])
                    if (row, st) != (want_rows[i], want_meta[i]):
                        bad.append(("decode", i))
                    elif st == OK:
                        msg, st2 = enc.call(row)                       # the closure returns the request as its response
                        if (msg, st2) != (frames[i][5:], OK):
                            bad.append(("encode", i))
                if i < len(reqs):
                    m, p, q, d, tid, fl = reqs[i]
                    resp, mt = http.serve(m, p, q, d, tid, fl)
                    if resp != ob[int(f1[i]):int(f1[i + 1])] or mt != int(m1[i]):
                        bad.append(("http", i))
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in range(threads)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in th) and not errs, errs
    assert not bad, bad[:10]
    assert dec.stats()[1] == len(frames) and http.stats()[1] == len(reqs)
    for x in (dec, enc, http):
        x.close()
    eng.close()
    print("%d RPCs and %d HTTP requests on one engine, equal to the model and the oracle" % (len(frames), len(reqs)))


def _gpu_capacity(seed):
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.frontend import ProtoFrontend
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    eng = Engine(Table(synth.config1_spec()), 0)
    L = _abi.lib()
    msgs = [[F(1, S.PB_STRING), F(2, S.PB_INT64, True)]]
    vals = [["n%d" % k * rnd.randint(0, 5), [rnd.randrange(-9, 9) for _ in range(rnd.randint(0, 6))]] for k in range(40)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, vals)
    frames, _ = M.encode(msgs, 0, rows, off)
    want_rows = [bytes(r) for r in PB.model_decode(msgs, frames)[0]]
    row_in = _records(rows, off)
    for decode, inputs, want in ((True, [f[5:] for f in frames], want_rows), (False, row_in, [f[5:] for f in frames])):
        fe = ProtoFrontend(eng, msgs, 0, decode, max_batch=8, max_wait_us=50, max_record_bytes=256)
        assert max(len(x) for x in inputs) <= 256
        # a record over max_record_bytes: refused before it is queued
        with pytest.raises(_abi.GofrError) as e:
            fe.call(b"\x0a\xff\x01" + b"a" * 255 if decode else b"\xff\0\0\0\0\0\0\0" + b"a" * 256)
        assert e.value.code == CAPACITY and fe.stats() == (0, 0)
        for i, x in enumerate(inputs):
            w = want[i]
            for cap in ([len(w) - 1, len(w)] if w else [0]):
                buf = C.create_string_buffer(max(cap, 1))
                n, st = C.c_uint32(0xFFFFFFFF), C.c_uint32()
                rc = L.gofr_proto_frontend_call(fe._f, x, len(x), buf, cap, C.byref(n), C.byref(st))
                assert n.value == len(w) and st.value == OK, (i, cap)
                if cap < len(w):
                    assert rc == CAPACITY
                else:
                    assert rc == 0 and buf.raw[:cap] == w
            assert fe.call(x) == (w, OK)                   # the same front-end keeps answering
        fe.close()
    eng.close()
    print("capacities: refused, one byte short and exact, as documented")


@pytest.mark.gpu
def test_gpu_decode_one_call_at_a_time():
    out = H.run_child("import tests.test_proto_frontend as t; t._gpu_decode(7070)", timeout=1800)
    assert "equal to the batch call and the model" in out


@pytest.mark.gpu
def test_gpu_encode_one_call_at_a_time():
    out = H.run_child("import tests.test_proto_frontend as t; t._gpu_encode(7171)", timeout=1800)
    assert "equal to the batch call and the model" in out


@pytest.mark.gpu
def test_gpu_grpc_and_http_front_ends_share_an_engine():
    out = H.run_child("import tests.test_proto_frontend as t; t._gpu_both_servers(7272)")
    assert "equal to the model and the oracle" in out


@pytest.mark.gpu
def test_gpu_capacity():
    out = H.run_child("import tests.test_proto_frontend as t; t._gpu_capacity(7373)")
    assert "as documented" in out


@pytest.mark.gpu
def test_gpu_grpc_server(tmp_path):
    """examples/cpp/grpc_server.cpp serves SayHello per RPC from 16 threads; every response is python protobuf's bytes"""
    _abi.lib()
    exe = str(tmp_path / "grpc_server")
    _compile_server(exe)
    r = subprocess.run([exe, "16", "20"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln.split("\t") for ln in r.stdout.splitlines()]
    assert len(lines) == 320
    assert [m for m, _ in lines[:3]] == ["Hello world!", "Hello 123!", "Hello World!"]
    cls = H.py_classes([[F(1, S.PB_STRING)]])[0]
    for m, hx in lines:
        obj = cls()
        setattr(obj, obj.DESCRIPTOR.fields[0].name, m)
        assert bytes.fromhex(hx) == obj.SerializeToString()
