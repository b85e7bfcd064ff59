"""gofr_proto_batch_encode_log and the encode front-end's call_log on the GPU: frames, offsets, meta and out_bytes identical to
gofr_proto_batch_encode on the same batches, every line equal to the request-log oracle's RPCLog line for its record (the
expectation of tests/test_proto_log.py) and empty for GOFR_LOG_NONE, across message types, chunk sizes and pinned,
pageable and mixed buffers; the capacity rule; empty batches; the argument checks that need an engine; many front-end
callers against a pinned log clock; and examples/cpp/grpc_server.cpp's log file."""
import calendar
import ctypes as C
import json
import random
import re
import subprocess
import threading

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from tests import proto_nested_harness as H
from tests import test_proto_frontend as PF
from tests import test_proto_log as P

pytestmark = pytest.mark.gpu

F = S.ProtoNField
HELLO = [[F(1, S.PB_STRING)]]      # HelloResponse { string message = 1; }
LOG_NS = P.LOG_NS


@pytest.fixture(scope="module")
def eng():
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    e = Engine(Table(synth.config1_spec()), 0)
    yield e
    e.set_chunk(65536)
    e.close()


def pack_rows(rows):
    """rows (bytes, each a multiple of 4 long; b"": a call whose handler failed) back to back → (data, off)"""
    off = np.zeros(len(rows) + 1, np.uint32)
    for i, r in enumerate(rows):
        assert len(r) % 4 == 0
        off[i + 1] = off[i] + len(r)
    data = np.frombuffer(b"".join(rows) + b"\0" * 16, np.uint8).copy()
    return data, off


def hello_row(msg: bytes) -> bytes:
    return len(msg).to_bytes(4, "little") + msg + b"\0" * (-len(msg) % 4)


def hello_batch(n: int, seed: int, empty_every: int = 11):
    rnd = random.Random(seed)
    rows = [b"" if empty_every and i % empty_every == 3 else hello_row(b"Hello caller-%d%s!" % (i, b"x" * rnd.randrange(40)))
            for i in range(n)]
    return pack_rows(rows)


def type_batches(seed: int):
    """(msgs, data, off) for HelloResponse rows and random nested types with maps and with presence, some rows empty"""
    rnd = random.Random(seed)
    out = [(HELLO,) + hello_batch(900, seed)]
    for msgs, make in ((H.rand_map_types(rnd), H.rand_map_value), (H.rand_presence_types(rnd), H.rand_presence_value)):
        rows, off = S.pack_proto_nested_rows(msgs, 0, [make(rnd, msgs, 0) for _ in range(700)])
        recs = [rows[int(off[i]):int(off[i + 1])].tobytes() if i % 13 != 5 else b"" for i in range(len(off) - 1)]
        out.append((msgs,) + pack_rows(recs))
    return out


def log_for(n: int, seed: int) -> S.LogBatch:
    """P.rpc_records with a 65535-byte method of every hostile kind on a few records"""
    log = P.rpc_records(n, seed=seed)
    recs = []
    for i in range(n):
        d = log.desc[i]
        m = log.arena[int(d["arena_off"]):int(d["arena_off"]) + int(d["method_len"])].tobytes()
        if i % 97 == 1:
            m = (b'"\\\x01<\xff\xe2\x80\xa8' * 8192)[:65535]
        recs.append(S.LogRec(int(d["start_unix_ns"]), int(d["elapsed_ns"]), -5, m, b"", b"", b"", b"", 999,
                             int(d["tz_offset_s"]), log.trace_ids[i].tobytes(), int(d["kind"])))
    return S.LogBatch.pack(recs)


def plain(eng, msgs, data, off):
    out, out_off, meta = eng.proto_encode_batch(msgs, 0, data, off, pinned=True)
    return out.tobytes(), out_off.copy(), meta.copy()


def check(eng, msgs, data, off, log, want_lines, pinned=True, log_pinned=None):
    frames, out_off, meta = plain(eng, msgs, data, off)
    r = eng.proto_encode_batch_log(msgs, 0, data, off, log, LOG_NS, pinned=pinned, log_pinned=log_pinned)
    n = len(off) - 1
    assert r.rc == 0
    assert r.out_bytes == len(frames) and r.out[:r.out_bytes].tobytes() == frames
    assert (r.out_off[:n + 1] == out_off[:n + 1]).all() and (r.meta == meta).all()
    assert (r.out[-16:] == 0xAB).all() and (r.lines_out[-16:] == 0xAB).all()
    got = r.line_list()
    assert got == want_lines
    assert r.lines == sum(1 for x in want_lines if x) and r.log_bytes == sum(map(len, want_lines)) == int(r.log_off[n])


@pytest.mark.parametrize("chunk", [1, 7, 128, 0])
def test_encode_log_sweep(eng, chunk):
    eng.set_chunk(chunk or 65536)
    try:
        for k, (msgs, data, off) in enumerate(type_batches(chunk + 5)):
            n = len(off) - 1 if chunk not in (1, 7) else 200
            off = off[:n + 1]
            log = log_for(n, seed=chunk * 7 + k)
            want = P.expectation(log)
            assert any(want) and not all(want)
            check(eng, msgs, data, off, log, want)
            for bufs in ((False, False), (True, False), (False, True)):
                check(eng, msgs, data, off, log, want, *bufs)
    finally:
        eng.set_chunk(65536)


def test_capacity_one_short_and_empty_batches(eng):
    data, off = hello_batch(3000, seed=9)
    log = log_for(3000, seed=9)
    want = P.expectation(log)
    frames, out_off, meta = plain(eng, HELLO, data, off)
    need = sum(map(len, want))
    for pinned in (True, False):
        # the lines one byte short: GOFR_ERR_CAPACITY with what the batch needed, the responses complete
        r = eng.proto_encode_batch_log(HELLO, 0, data, off, log, LOG_NS, pinned=pinned, log_out_cap=need - 1,
                                       raise_on_capacity=False)
        assert r.rc == 7 and r.lines == sum(1 for x in want if x) and r.log_bytes == need
        assert r.out_bytes == len(frames) and r.out[:r.out_bytes].tobytes() == frames and (r.meta == meta).all()
        assert (r.lines_out[need - 1:need - 1 + 16] == 0xAB).all()
        # the frames one byte short: the same, the other way round
        r = eng.proto_encode_batch_log(HELLO, 0, data, off, log, LOG_NS, pinned=pinned, out_cap=len(frames) - 1,
                                       raise_on_capacity=False)
        assert r.rc == 7 and r.out_bytes == len(frames) and (r.meta == meta).all()
        assert r.line_list() == want and r.log_bytes == need
        assert (r.out[len(frames) - 1:len(frames) - 1 + 16] == 0xAB).all()
    empty = S.LogBatch.pack([])
    for pinned in (True, False):
        r = eng.proto_encode_batch_log(HELLO, 0, np.zeros(16, np.uint8), np.zeros(1, np.uint32), empty, LOG_NS, pinned=pinned)
        assert r.rc == 0 and r.lines == 0 and r.log_bytes == 0 and r.out_bytes == 0 and int(r.log_off[0]) == 0


def _raw(eng, data, off, log, ids):
    L = _abi.lib()
    nm, nf, k = S.proto_nested_tables(HELLO)
    n = len(off) - 1
    cap = 64 * n + 64
    out, out_off, meta = np.zeros(cap, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.uint32)
    lout, log_off = np.zeros(1 << 20, np.uint8), np.zeros(n + 1, np.uint32)
    pb = _abi.ProtoBatch(data=data.ctypes.data, data_bytes=data.size, off=off.ctypes.data, n=n)
    ob = _abi.RespBatch(out=out.ctypes.data, out_cap=cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data, out_bytes=0)
    lb = _abi.BatchLog(desc=log.desc.ctypes.data, arena=log.arena.ctypes.data if log.arena.size else None,
                       arena_bytes=log.arena.size, log_unix_ns=LOG_NS, out=lout.ctypes.data, out_cap=lout.size,
                       log_off=log_off.ctypes.data, lines=0, reserved=0, out_bytes=0)
    t = C.c_uint64()
    rc = L.gofr_proto_batch_encode_log(eng._e, nm.ctypes.data, 1, nf.ctypes.data, k, 0, None, C.byref(pb), ids, C.byref(ob),
                                       C.byref(lb), C.byref(t))
    if rc == 0:
        assert L.gofr_batch_wait(eng._e, t.value) == 0
    return rc


def test_argument_errors(eng):
    data, off = hello_batch(20, seed=2)
    log = log_for(20, seed=2)
    assert _raw(eng, data, off, log, log.trace_ids.ctypes.data) == 0
    assert _raw(eng, data, off, log, None) == 1                      # no trace ids
    bad = S.LogBatch(log.desc.copy(), log.trace_ids, log.arena)
    bad.desc["kind"][4] = S.LOG_REQUEST                              # an HTTP line has no meaning here
    assert _raw(eng, data, off, bad, log.trace_ids.ctypes.data) == 1
    bad.desc["kind"][4] = 7
    assert _raw(eng, data, off, bad, log.trace_ids.ctypes.data) == 1
    bad = S.LogBatch(log.desc.copy(), log.trace_ids, log.arena)
    bad.desc["arena_off"][3] = log.arena.size                        # strings past the arena
    assert _raw(eng, data, off, bad, log.trace_ids.ctypes.data) == 1
    # the engine serves on after refusing
    assert _raw(eng, data, off, log, log.trace_ids.ctypes.data) == 0
    from gofr_b200.frontend import ProtoFrontend
    with pytest.raises(_abi.GofrError):
        ProtoFrontend(eng, HELLO, 0, True, max_log_bytes=64)             # a decode front-end takes no log


def test_frontend_many_threads(eng):
    """16 threads mixing call, call_log, log-only calls (the handler failed: an empty row) and GOFR_LOG_NONE on one encode
    front-end with a pinned log clock: each message is what the plain front-end gives, each line the oracle's"""
    from gofr_b200.frontend import ProtoFrontend
    fe = ProtoFrontend(eng, HELLO, 0, False, max_batch=64, max_wait_us=200, max_record_bytes=512, max_log_bytes=70000)
    fe_plain = ProtoFrontend(eng, HELLO, 0, False, max_batch=64, max_wait_us=200, max_record_bytes=512)
    fe.set_log_clock(LOG_NS)
    n = 1600
    data, off = hello_batch(n, seed=21)
    log = log_for(n, seed=21)
    rows = [data[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)]
    want_lines = P.expectation(log)
    recs = []
    for i in range(n):
        d = log.desc[i]
        m = log.arena[int(d["arena_off"]):int(d["arena_off"]) + int(d["method_len"])].tobytes()
        recs.append(S.LogRec(int(d["start_unix_ns"]), int(d["elapsed_ns"]), 0, m, b"", b"", b"", b"", 0, int(d["tz_offset_s"]),
                             kind=int(d["kind"])))
    got, errs = [None] * n, []

    def work(t):
        try:
            for i in range(t, n, 16):
                if i % 5 == 2:
                    got[i] = fe.call(rows[i]) + (None,)
                else:
                    got[i] = fe.call(rows[i], log=recs[i], trace_id=log.trace_ids[i].tobytes())
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in range(16)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in th), "front-end hung"
    assert not errs, errs
    want_msgs = PF._run_calls(fe_plain, rows, 8)
    for i in range(n):
        msg, status, line = got[i]
        assert (msg, status) == want_msgs[i], i
        if line is not None:
            assert line == want_lines[i], i
    assert sum(1 for i in range(n) if i % 5 != 2 and want_lines[i]) > 800
    b, r = fe.stats()
    assert r == n and b < n
    fe.close()
    fe_plain.close()


_TIME = re.compile(r"^(\d{4})-(\d\d)-(\d\d)T(\d\d):(\d\d):(\d\d)(?:\.(\d{1,9}))?(Z|[+-]\d\d:\d\d)$")


def _unix_ns(text: str):
    """an RFC 3339 time as the logger writes it → (unix ns, zone offset in seconds)"""
    m = _TIME.match(text)
    assert m, text
    y, mo, d, h, mi, s = (int(x) for x in m.groups()[:6])
    frac = int((m.group(7) or "").ljust(9, "0"))
    z = m.group(8)
    off = 0 if z == "Z" else (1 if z[0] == "+" else -1) * (int(z[1:3]) * 3600 + int(z[4:6]) * 60)
    return (calendar.timegm((y, mo, d, h, mi, s)) - off) * 10 ** 9 + frac, off


def test_grpc_server_log(tmp_path):
    """examples/cpp/grpc_server.cpp with a log path: one RPCLog line per call, each the oracle's line for the clock
    readings, zone and trace id it carries, method /Hello/SayHello; its standard output stays the same"""
    exe = str(tmp_path / "grpc_server")
    _abi.lib()
    PF._compile_server(exe)
    path = str(tmp_path / "rpc.log")
    r = subprocess.run([exe, "16", "20", path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    out = [ln.split("\t") for ln in r.stdout.splitlines()]
    assert len(out) == 320 and [m for m, _ in out[:3]] == ["Hello world!", "Hello 123!", "Hello World!"]
    raw = open(path, "rb").read()
    lines = raw.splitlines(keepends=True)
    assert len(lines) == 320
    recs = []
    for i, ln in enumerate(lines):
        entry = json.loads(ln)
        msg = json.loads(entry["message"])
        assert entry["Level"] == "INFO" and msg["method"] == "/Hello/SayHello"
        assert bytes.fromhex(msg["id"]) == (i + 1).to_bytes(16, "big")
        log_ns, zone = _unix_ns(entry["time"])
        start_ns, zone2 = _unix_ns(msg["startTime"])
        assert zone in (0, zone2) and msg["responseTime"] >= 0
        recs.append(S.LogRec(start_ns, msg["responseTime"] * 1000, log_ns, b"/Hello/SayHello", tz_offset_s=zone2,
                             trace_id=bytes.fromhex(msg["id"]), kind=S.LOG_RPC))
    assert P.oracle_lines(S.LogBatch.pack(recs)) == lines
