"""The chunk pipeline of the calls on a request or proto batch, on the GPU: gofr_batch_submit, _slots, _log and
_slots_log, gofr_proto_batch_decode / _encode.  Covers what the per-call tests do not: the log calls with one output
pinned and the other pageable, each output's capacity one short, gofr_batch_submit short of out_cap (it reports what was
written, the log calls what the batch needed), launches per call, and empty batches."""
import ctypes as C

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200.engine import pinned_array
from tests import test_batch_log as M

pytestmark = pytest.mark.gpu

SLOT = 512
FILL = 0xAB            # every output buffer starts filled with it, so that bytes the call leaves alone are seen
CAPACITY = 7           # GOFR_ERR_CAPACITY


@pytest.fixture(scope="module")
def setup():
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    spec = M.mixed_spec(True, True)
    e = Engine(Table(spec), 0)
    yield spec, e
    e.close()


@pytest.fixture
def chunk(setup, request):
    """the engine's chunk size for one test, restored after it"""
    _, e = setup
    e.set_chunk(request.param)
    yield request.param
    e.set_chunk(65536)


def _untouched(*arrs) -> bool:
    return all((a.view(np.uint8) == FILL).all() for a in arrs)


def _buf(pinned: bool, count: int, dtype=np.uint8) -> np.ndarray:
    a = pinned_array(max(count, 1) * np.dtype(dtype).itemsize).view(dtype) if pinned else np.empty(max(count, 1), dtype)
    a.view(np.uint8)[:] = FILL
    return a


def _inputs(n: int, seed: int):
    batch, log = M.mixed_requests(n, seed=seed, stage2=True, long_every=37), M.log_records(n, seed=seed)
    return batch, log


def _req(batch):
    return _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data, arena=batch.arena.ctypes.data,
                         arena_bytes=batch.arena.size, n=batch.n, date=M.DATE)


def _need(e, batch) -> int:
    L = _abi.lib()
    return sum(int(L.gofr_table_response_bound(e.table.handle, int(d["path_len"]), int(d["query_len"]), int(d["data_len"])))
               for d in batch.desc)


def serve(e, batch, log=None, slot_bytes=0, resp_pinned=True, lines_pinned=True, out_cap=None, log_cap=None):
    """one of the four serve calls and its wait: every output buffer (with the bytes past its capacity), the reported
    counts and the wait's code"""
    L = _abi.lib()
    n = batch.n
    r = {}
    r["meta"] = _buf(resp_pinned, n, np.uint32)
    if slot_bytes:
        r["out"], r["out_len"] = _buf(resp_pinned, n * slot_bytes), _buf(resp_pinned, n, np.uint32)
        ob = _abi.SlotBatch(out=r["out"].ctypes.data, slot_bytes=slot_bytes, reserved=0, out_len=r["out_len"].ctypes.data,
                            meta=r["meta"].ctypes.data)
    else:
        out_cap = _need(e, batch) if out_cap is None else out_cap
        r["out"], r["out_off"] = _buf(resp_pinned, out_cap + 16), _buf(resp_pinned, n + 1, np.uint32)
        ob = _abi.RespBatch(out=r["out"].ctypes.data, out_cap=out_cap, out_off=r["out_off"].ctypes.data,
                            meta=r["meta"].ctypes.data, out_bytes=0)
    t = C.c_uint64()
    if log is None:
        fn = L.gofr_batch_submit_slots if slot_bytes else L.gofr_batch_submit
        rc = fn(e._e, C.byref(_req(batch)), C.byref(ob), C.byref(t))
    else:
        from gofr_b200.engine import batch_log_bound
        log_cap = batch_log_bound(log) if log_cap is None else log_cap
        r["lines_out"], r["log_off"] = _buf(lines_pinned, log_cap + 16), _buf(lines_pinned, n + 1, np.uint32)
        lb = _abi.BatchLog(desc=log.desc.ctypes.data, arena=log.arena.ctypes.data if log.arena.size else None,
                           arena_bytes=log.arena.size, log_unix_ns=M.LOG_NS, out=r["lines_out"].ctypes.data, out_cap=log_cap,
                           log_off=r["log_off"].ctypes.data, lines=0, reserved=0, out_bytes=0)
        fn = L.gofr_batch_submit_slots_log if slot_bytes else L.gofr_batch_submit_log
        rc = fn(e._e, C.byref(_req(batch)), C.byref(ob), C.byref(lb), C.byref(t))
    assert rc == 0, L.gofr_last_error()
    r["rc"] = int(L.gofr_batch_wait(e._e, t.value))
    if not slot_bytes:
        r["out_bytes"] = int(ob.out_bytes)
    if log is not None:
        r["lines"], r["log_bytes"] = int(lb.lines), int(lb.out_bytes)
    return r


def _packed(out, off, n):
    b = out.tobytes()
    return [b[int(off[i]):int(off[i + 1])] for i in range(n)]


def _same(a, b):
    """the same outputs; a slot's bytes past its response are the device buffer's, not the call's"""
    assert a.keys() == b.keys()
    for k in a:
        if k == "out" and "out_len" in a:
            assert _slots(a) == _slots(b)
        elif isinstance(a[k], np.ndarray):
            assert a[k].tobytes() == b[k].tobytes(), k
        else:
            assert a[k] == b[k], k


@pytest.mark.parametrize("chunk", [1, 7, 65536], indirect=True)
@pytest.mark.parametrize("slot_bytes", [0, SLOT])
def test_log_calls_mixed_residency(setup, chunk, slot_bytes):
    spec, e = setup
    batch, log = _inputs(300 if chunk < 65536 else 3000, seed=chunk + slot_bytes)
    want_resp, want_meta, want_lines = M.expectation(spec, batch, log)
    pinned = serve(e, batch, log, slot_bytes)
    assert pinned["rc"] == 0 and (pinned["meta"] == want_meta).all()
    assert _packed(pinned["lines_out"], pinned["log_off"], batch.n) == want_lines
    if not slot_bytes:
        assert _packed(pinned["out"], pinned["out_off"], batch.n) == want_resp
    for resp_pinned, lines_pinned in ((True, False), (False, True)):
        _same(serve(e, batch, log, slot_bytes, resp_pinned, lines_pinned), pinned)


@pytest.mark.parametrize("chunk", [7], indirect=True)
@pytest.mark.parametrize("short,slot_bytes", [("responses", 0), ("lines", 0), ("lines", SLOT)])  # slots have no byte capacity
@pytest.mark.parametrize("pinned", [True, False])
def test_log_calls_one_short(setup, chunk, short, slot_bytes, pinned):
    spec, e = setup
    batch, log = _inputs(300, seed=3)
    want_resp, want_meta, want_lines = M.expectation(spec, batch, log)
    resp_need, line_need = sum(map(len, want_resp)), sum(map(len, want_lines))
    out_cap = resp_need - 1 if short == "responses" else None
    log_cap = line_need - 1 if short == "lines" else None
    r = serve(e, batch, log, slot_bytes, pinned, pinned, out_cap=out_cap, log_cap=log_cap)
    assert r["rc"] == CAPACITY
    assert (r["meta"] == want_meta).all()
    assert r["lines"] == sum(1 for x in want_lines if x) and r["log_bytes"] == line_need
    if not slot_bytes:
        assert r["out_bytes"] == resp_need
    if short == "lines":
        assert (r["lines_out"][line_need - 1:] == FILL).all()
        if slot_bytes:
            assert all(x == want_resp[i] for i, x in enumerate(_slots(r)) if x is not None)
        else:
            assert _packed(r["out"], r["out_off"], batch.n) == want_resp
    else:
        assert (r["out"][resp_need - 1:] == FILL).all()
        assert _packed(r["lines_out"], r["log_off"], batch.n) == want_lines


def _slots(r):
    """the responses that fit their slot (None for the others)"""
    return [r["out"][i * SLOT:i * SLOT + int(r["out_len"][i])].tobytes() if r["out_len"][i] <= SLOT else None
            for i in range(len(r["out_len"]))]


@pytest.mark.parametrize("chunk", [7], indirect=True)
@pytest.mark.parametrize("pinned", [True, False])
@pytest.mark.parametrize("short", ["one", "half"])
def test_submit_short_reports_written(setup, chunk, pinned, short):
    """gofr_batch_submit short of out_cap: the chunks that fit in order are written whole, the others dropped whole, and
    out_bytes == out_off[n] are the bytes written"""
    spec, e = setup
    batch, log = _inputs(300, seed=17)
    want_resp, want_meta, _ = M.expectation(spec, batch, log)
    need = sum(map(len, want_resp))
    cap = need - 1 if short == "one" else need // 2
    r = serve(e, batch, resp_pinned=pinned, out_cap=cap)
    assert r["rc"] == CAPACITY
    kept, written = [], 0
    for lo in range(0, batch.n, chunk):
        size = sum(map(len, want_resp[lo:lo + chunk]))
        if written + size <= cap:
            kept.append((lo, written))
            written += size
    assert 0 < written < need
    assert r["out_bytes"] == written and int(r["out_off"][batch.n]) == written
    assert r["out"][:written].tobytes() == b"".join(b"".join(want_resp[lo:lo + chunk]) for lo, _ in kept)
    for lo, at in kept:
        for i in range(lo, min(lo + chunk, batch.n)):
            assert int(r["out_off"][i]) == at
            at += len(want_resp[i])
    assert (r["meta"] == want_meta).all()
    assert (r["out"][cap:] == FILL).all()


@pytest.mark.parametrize("chunk", [128, 65536], indirect=True)
@pytest.mark.parametrize("pinned", [True, False])
@pytest.mark.parametrize("call", ["submit", "slots", "log", "slots_log"])
def test_launches_per_call(setup, chunk, pinned, call):
    """serve, plus advance and egress per pinned packed output, plus the batch-log and pack kernels with a log"""
    _, e = setup
    n = 300
    batch, log = _inputs(n, seed=5)
    slot_bytes = SLOT if call.startswith("slots") else 0
    logged = call.endswith("log")
    before = e.launch_count()
    r = serve(e, batch, log if logged else None, slot_bytes, pinned, pinned)
    assert r["rc"] == 0
    chunks = -(-n // chunk)
    per_chunk = 1 + (2 if pinned and not slot_bytes else 0) + ((2 + (2 if pinned else 0)) if logged else 0)
    assert e.launch_count() - before == chunks * per_chunk


def test_empty_batches(setup):
    """n == 0: out_off[0] and log_off[0] are 0 where given, nothing else is touched, nothing is launched"""
    _, e = setup
    L = _abi.lib()
    empty = S.RequestBatch(np.zeros(0, S.DESC_DTYPE), np.zeros((0, 16), np.uint8), np.zeros(16, np.uint8))
    log = M.log_records(1)
    before = e.launch_count()
    for call in ("submit", "slots", "log", "slots_log"):
        out, off, meta = _buf(False, 64), _buf(False, 4, np.uint32), _buf(False, 4, np.uint32)
        lout, loff = _buf(False, 64), _buf(False, 4, np.uint32)
        rb = _req(empty)
        if call.startswith("slots"):
            ob = _abi.SlotBatch(out=out.ctypes.data, slot_bytes=SLOT, reserved=0, out_len=off.ctypes.data, meta=meta.ctypes.data)
        else:
            ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out.size, out_off=off.ctypes.data, meta=meta.ctypes.data,
                                out_bytes=99)
        lb = _abi.BatchLog(desc=log.desc.ctypes.data, arena=log.arena.ctypes.data, arena_bytes=log.arena.size,
                           log_unix_ns=M.LOG_NS, out=lout.ctypes.data, out_cap=lout.size, log_off=loff.ctypes.data, lines=5,
                           reserved=0, out_bytes=99)
        t = C.c_uint64()
        fn = {"submit": L.gofr_batch_submit, "slots": L.gofr_batch_submit_slots, "log": L.gofr_batch_submit_log,
              "slots_log": L.gofr_batch_submit_slots_log}[call]
        args = (C.byref(rb), C.byref(ob)) + ((C.byref(lb),) if call.endswith("log") else ()) + (C.byref(t),)
        assert fn(e._e, *args) == 0 and L.gofr_batch_wait(e._e, t.value) == 0, call
        assert _untouched(out, meta, loff[1:], lout), call
        if call.startswith("slots"):
            assert _untouched(off), call
        else:
            assert off[0] == 0 and _untouched(off[1:]) and ob.out_bytes == 0, call
        if call.endswith("log"):
            assert loff[0] == 0 and lb.lines == 0 and lb.out_bytes == 0, call
        else:
            assert _untouched(loff), call
        # the same call without any buffers
        none = _abi.RespBatch(out_bytes=99) if not call.startswith("slots") else _abi.SlotBatch(slot_bytes=SLOT)
        nlog = _abi.BatchLog(lines=5, out_bytes=99)
        args = (C.byref(_req(empty)), C.byref(none)) + ((C.byref(nlog),) if call.endswith("log") else ()) + (C.byref(t),)
        assert fn(e._e, *args) == 0 and L.gofr_batch_wait(e._e, t.value) == 0, call
        assert call.startswith("slots") or none.out_bytes == 0, call
        assert not call.endswith("log") or (nlog.lines == 0 and nlog.out_bytes == 0), call
    msgs = [[S.ProtoNField(1, S.PB_STRING)]]
    nm, nf, k = S.proto_nested_tables(msgs)
    for fn in (L.gofr_proto_batch_decode, L.gofr_proto_batch_encode):
        out, off, meta = _buf(False, 64), _buf(False, 4, np.uint32), _buf(False, 4, np.uint32)
        pb = _abi.ProtoBatch(data=None, data_bytes=0, off=None, n=0)
        ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out.size, out_off=off.ctypes.data, meta=meta.ctypes.data, out_bytes=99)
        t = C.c_uint64()
        assert fn(e._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, None, C.byref(pb), C.byref(ob), C.byref(t)) == 0
        assert L.gofr_batch_wait(e._e, t.value) == 0
        assert off[0] == 0 and _untouched(off[1:], out, meta) and ob.out_bytes == 0
    assert e.launch_count() == before
