"""gofr_batch_submit_log / _slots_log and the per-request front-end's serve_log on the GPU: responses and meta byte-identical
to the calls without a log, lines equal to the expectation of tests/test_batch_log.py and to the device-resident chain
(gofr_serve_device, then the filled records through gofr_requestlog_device), across tables, both layouts, pinned and
pageable buffers and chunk sizes; the capacity rule; the argument checks; many front-end callers mixing serve and
serve_log."""
import ctypes as C
import threading

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from tests import test_batch_log as M

pytestmark = pytest.mark.gpu

SLOT = 512
SPECS = {"defaults": (True, False), "mux_only": (False, False), "stage2": (True, True)}


@pytest.fixture(scope="module", params=list(SPECS))
def setup(request):
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    defaults, stage2 = SPECS[request.param]
    spec = M.mixed_spec(defaults, stage2)
    e = Engine(Table(spec), 0)
    yield spec, stage2, e
    e.close()


def _plain(e, batch):
    """gofr_batch_submit and gofr_batch_submit_slots on the same batch: (packed responses, meta, slot responses, meta)"""
    n = batch.n
    cap = 4096 * n + 65536
    out, off, meta = np.zeros(cap, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.uint32)
    e.serve_host(batch, M.DATE, out, off, meta)
    so, sl, sm = np.zeros(n * SLOT, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    e.serve_host_slots(batch, M.DATE, SLOT, so, sl, sm)
    slots = [so[i * SLOT:i * SLOT + int(sl[i])].tobytes() if sl[i] <= SLOT else None for i in range(n)]
    return [out[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)], meta, slots, sl, sm


def _device_chain(e, batch, log):
    """gofr_serve_device, then the records the rule admits, filled from its meta, through gofr_requestlog_device"""
    import torch
    b = e.upload(batch)
    resp = e.alloc_responses(batch.n, 4096 * batch.n + 65536)
    e.serve_device(b, M.DATE, resp)
    torch.cuda.synchronize()
    meta = resp.meta.cpu().numpy().view(np.uint32)[:batch.n]
    sel = np.nonzero(M.admitted(meta, log.desc["kind"]))[0]
    lines = [b""] * batch.n
    if len(sel):
        d = log.desc[sel].copy()
        d["status"], d["log_unix_ns"], d["elapsed_ns"] = meta[sel] & 0xFFFF, M.LOG_NS, M.LOG_NS - d["start_unix_ns"]
        d_out, d_off = e.request_log_device(S.LogBatch(d, batch.trace_ids[sel].copy(), log.arena))
        off = d_off.cpu().numpy().view(np.uint32)
        raw = d_out[:int(off[-1])].cpu().numpy().tobytes()
        for j, i in enumerate(sel.tolist()):
            lines[i] = raw[int(off[j]):int(off[j + 1])]
    return lines


@pytest.mark.parametrize("chunk", [1, 7, 128, 0])
def test_batch_log_sweep(setup, chunk):
    spec, stage2, e = setup
    n = 300 if chunk in (1, 7) else 5000
    batch, log = M.mixed_requests(n, seed=chunk + 11, stage2=stage2, long_every=97), M.log_records(n, seed=chunk + 11)
    want_resp, want_meta, want_lines = M.expectation(spec, batch, log)
    assert sum(map(len, want_lines)) > 0
    e.set_chunk(chunk or 65536)
    try:
        packed, meta, slots, slen, smeta = _plain(e, batch)
        assert packed == want_resp and (meta == want_meta).all()
        for pinned in (True, False):
            r = e.serve_host_log(batch, M.DATE, log, M.LOG_NS, pinned=pinned)
            assert r.rc == 0
            assert r.responses() == packed and (r.meta == meta).all()
            assert r.out_bytes == sum(map(len, packed))
            assert r.line_list() == want_lines
            assert r.lines == sum(1 for x in want_lines if x) and r.log_bytes == sum(map(len, want_lines))
            s = e.serve_host_log(batch, M.DATE, log, M.LOG_NS, slot_bytes=SLOT, pinned=pinned)
            assert s.rc == 0 and (s.out_len == slen).all() and (s.meta == smeta).all()
            assert [x if slen[i] <= SLOT else None for i, x in enumerate(s.responses(SLOT))] == slots
            assert s.line_list() == want_lines and s.lines == r.lines
    finally:
        e.set_chunk(65536)
    if chunk == 0:
        assert _device_chain(e, batch, log) == want_lines


@pytest.mark.parametrize("slot_bytes", [0, SLOT])
@pytest.mark.parametrize("pinned", [True, False])
def test_batch_log_capacity(setup, slot_bytes, pinned):
    spec, stage2, e = setup
    n = 2000
    batch, log = M.mixed_requests(n, seed=5, stage2=stage2), M.log_records(n, seed=5)
    want_resp, want_meta, want_lines = M.expectation(spec, batch, log)
    need = sum(map(len, want_lines))
    e.set_chunk(256)
    try:
        r = e.serve_host_log(batch, M.DATE, log, M.LOG_NS, slot_bytes=slot_bytes, pinned=pinned, log_out_cap=need - 1,
                             raise_on_capacity=False)
        assert r.rc == 7
        assert r.lines == sum(1 for x in want_lines if x) and r.log_bytes == need
        assert (r.lines_out[need - 1:] == 0xAB).all()   # nothing written at or past the capacity
        assert (r.meta == want_meta).all()
        if not slot_bytes:
            assert r.responses() == want_resp
        else:
            assert all(x == want_resp[i] for i, x in enumerate(r.responses(SLOT)) if r.out_len[i] <= SLOT)
        ok = e.serve_host_log(batch, M.DATE, log, M.LOG_NS, slot_bytes=slot_bytes, pinned=pinned, log_out_cap=need)
        assert ok.rc == 0 and ok.line_list() == want_lines
    finally:
        e.set_chunk(65536)


def test_batch_log_argument_errors(setup):
    _, stage2, e = setup
    L = _abi.lib()
    batch, log = M.mixed_requests(10, stage2=stage2), M.log_records(10)

    def rc_of(desc, arena_bytes=None, null_out=False):
        lout, loff = np.zeros(1 << 16, np.uint8), np.zeros(11, np.uint32)
        out, off, meta = np.zeros(1 << 16, np.uint8), np.zeros(11, np.uint32), np.zeros(10, np.uint32)
        rb = _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data, arena=batch.arena.ctypes.data,
                           arena_bytes=batch.arena.size, n=10, date=M.DATE)
        ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out.size, out_off=off.ctypes.data, meta=meta.ctypes.data)
        lb = _abi.BatchLog(desc=desc.ctypes.data, arena=log.arena.ctypes.data,
                           arena_bytes=log.arena.size if arena_bytes is None else arena_bytes, log_unix_ns=M.LOG_NS,
                           out=None if null_out else lout.ctypes.data, out_cap=lout.size, log_off=loff.ctypes.data)
        t = C.c_uint64()
        rc = L.gofr_batch_submit_log(e._e, C.byref(rb), C.byref(ob), C.byref(lb), C.byref(t))
        return rc if rc else L.gofr_batch_wait(e._e, t.value)

    assert rc_of(log.desc) == 0
    bad = log.desc.copy()
    bad["kind"][3] = S.LOG_RPC
    assert rc_of(bad) == 1
    bad = log.desc.copy()
    bad["kind"][4] = 9
    assert rc_of(bad) == 1
    end = log.desc["arena_off"].astype(np.int64) + sum(log.desc[k].astype(np.int64) for k in
                                                         ("method_len", "ua_len", "xff_len", "remote_len", "uri_len"))
    assert rc_of(log.desc, arena_bytes=int(end.max()) - 1) == 1
    assert rc_of(log.desc, null_out=True) == 1
    assert rc_of(log.desc) == 0   # the engine keeps serving


def test_frontend_serve_log_threads(setup):
    from gofr_b200.frontend import Frontend
    spec, stage2, e = setup
    n = 600
    batch, log = M.mixed_requests(n, seed=21, stage2=stage2, long_every=41), M.log_records(n, seed=21)
    want_resp, want_meta, want_lines = M.expectation(spec, batch, log)
    desc = batch.desc
    recs = []
    for i in range(n):
        d = log.desc[i]
        a = int(d["arena_off"])
        k = [int(d[f]) for f in ("method_len", "ua_len", "xff_len", "remote_len", "uri_len")]
        s = log.arena[a:a + sum(k)].tobytes()
        parts, o = [], 0
        for x in k:
            parts.append(s[o:o + x])
            o += x
        recs.append(S.LogRec(int(d["start_unix_ns"]), 0, 0, parts[0], parts[1], parts[2], parts[3], parts[4], 0,
                             int(d["tz_offset_s"]), None, int(d["kind"])))
    f = Frontend(e, max_batch=64, max_wait_us=300, slot_bytes=SLOT, max_request_bytes=8192, max_log_bytes=4096)
    f.set_clock(1_700_000_000)
    f.set_log_clock(M.LOG_NS)
    got, errors = [None] * n, []

    def worker(w):
        try:
            for i in range(w, n, 8):
                dd = desc[i]
                a, pl, ql, dl = int(dd["arena_off"]), int(dd["path_len"]), int(dd["query_len"]), int(dd["data_len"])
                path = batch.arena[a:a + pl].tobytes()
                query = batch.arena[a + pl:a + pl + ql].tobytes()
                b0 = (a + pl + ql + 3) & ~3
                data = batch.arena[b0:b0 + dl].tobytes()
                tid = batch.trace_ids[i].tobytes()
                if i % 3 == 2:   # a plain caller rides along as GOFR_LOG_NONE
                    r, m = f.serve(int(dd["method"]), path, query, data, tid, flags=int(dd["flags"]), resp_cap=1 << 16)
                    got[i] = (r, m, None)
                else:
                    got[i] = f.serve(int(dd["method"]), path, query, data, tid, flags=int(dd["flags"]), resp_cap=1 << 16,
                                     log=recs[i])
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    th = [threading.Thread(target=worker, args=(w,)) for w in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    f.close()
    assert not errors, errors[:3]
    assert any(len(want_resp[i]) > SLOT for i in range(n))
    for i in range(n):
        r, m, line = got[i]
        assert r == want_resp[i] and m == want_meta[i], i
        if line is not None:
            assert line == want_lines[i], i


def test_frontend_line_capacity_and_plain_frontend(setup):
    from gofr_b200.frontend import Frontend
    spec, stage2, e = setup
    rec = S.LogRec(1_700_000_000_000_000_000, 0, 0, b"GET", b"ua", b"", b"10.0.0.1:5", b"/hello")
    f = Frontend(e, max_batch=4, max_wait_us=50, slot_bytes=SLOT, max_log_bytes=256)
    f.set_log_clock(M.LOG_NS)
    r, m, line = f.serve(S.M_GET, b"/hello", log=rec)
    assert m & 0xFFFF == 200 and line.startswith(b'{"Level":"INFO"') and line.endswith(b"}}\n")
    with pytest.raises(_abi.GofrError) as ex:
        f.serve(S.M_GET, b"/hello", log=rec, line_cap=len(line) - 1)
    assert ex.value.code == 7
    r2, m2, line2 = f.serve(S.M_GET, b"/hello", log=rec)   # the front-end keeps serving
    assert r2 == r and line2 == line
    f.close()
    plain = Frontend(e, max_batch=4, max_wait_us=50, slot_bytes=SLOT)
    with pytest.raises(_abi.GofrError) as ex:
        plain.serve(S.M_GET, b"/hello", log=rec)
    assert ex.value.code == 1
    plain.close()
