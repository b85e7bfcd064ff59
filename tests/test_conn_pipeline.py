"""The connection pipeline's shared parts (engine.cu: PackedOut::ship, the chunk loop conn_chunks) in the cases the per-call
tests do not reach: the outputs of one gofr_conn_batch_submit_log call in different kinds of host memory, and a bad offset in
a later chunk of gofr_conn_batch_route, refused while earlier chunks are in flight.

The models and streams are those of test_conn_batch, test_conn_log and test_conn_closures."""
import ctypes as C

import numpy as np
import pytest

from gofr_b200 import _abi, synth
from gofr_b200.table import Table
from tests import test_conn_batch as CB
from tests import test_conn_closures as CC
from tests import test_conn_log as CL

RESP = ("out", "out_off", "meta")             # the responses' packed output: pinned only when all three are
COLS = ("req_at", "trace_ids", "req_first", "consumed", "conn_status")
LOG = ("lout", "log_off", "log_req")
ALL = set(RESP + COLS + LOG)
# which buffers are pinned
MIXED = {"responses pinned, log lines pageable": set(RESP + COLS),
         "responses pageable, log lines pinned": set(LOG),
         "columns pageable": set(RESP + LOG)}


def _submit(eng, buf, off, remote, roff, start, pinned, req_cap, out_cap, line_cap, lout_cap, canary=64):
    """gofr_conn_batch_submit_log with each buffer named in `pinned` in pinned memory and the others pageable, `canary`
    guard bytes (0xA5, as every unwritten byte) behind each capacity → (rc, buffers, ConnResp, ConnLog)"""
    from gofr_b200.engine import pinned_array
    n = len(off) - 1
    counts = dict(out=(out_cap, np.uint8), out_off=(req_cap + 1, np.uint32), meta=(req_cap, np.uint32),
                  req_at=(req_cap, np.uint32), trace_ids=(req_cap * 16, np.uint8), req_first=(n + 1, np.uint32),
                  consumed=(n, np.uint32), conn_status=(n, np.uint32), lout=(lout_cap, np.uint8),
                  log_off=(line_cap + 1, np.uint32), log_req=(line_cap, np.uint32))
    a = {}
    for k, (count, dt) in counts.items():
        nbytes = (count + canary) * np.dtype(dt).itemsize
        a[k] = (pinned_array(nbytes) if k in pinned else np.empty(nbytes, np.uint8)).view(dt)
        a[k].view(np.uint8)[:] = 0xA5
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=CB.DATE, trace_seed=3)
    cr = _abi.ConnResp(out=a["out"].ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=a["out_off"].ctypes.data,
                       meta=a["meta"].ctypes.data, req_at=a["req_at"].ctypes.data, trace_ids=a["trace_ids"].ctypes.data,
                       req_first=a["req_first"].ctypes.data, consumed=a["consumed"].ctypes.data, conn_status=a["conn_status"].ctypes.data)
    cl = _abi.ConnLog(remote=remote.ctypes.data, remote_off=roff.ctypes.data, start_unix_ns=start.ctypes.data, log_unix_ns=CL.LOG_NS,
                      tz_offset_s=CL.TZ, line_cap=line_cap, out=a["lout"].ctypes.data, out_cap=lout_cap,
                      log_off=a["log_off"].ctypes.data, log_req=a["log_req"].ctypes.data)
    L = _abi.lib()
    t = C.c_uint64()
    rc = L.gofr_conn_batch_submit_log(eng._e, C.byref(cb), C.byref(cr), C.byref(cl), C.byref(t))
    if rc == 0:
        rc = L.gofr_batch_wait(eng._e, t.value)
    return rc, a, cr, cl


def _lines_equal(a, cl, want):
    lines = len(want["log_req"])
    assert a["lout"][:int(want["log_off"][-1])].tobytes() == want["log"].tobytes()
    assert np.array_equal(a["log_off"][:lines + 1], want["log_off"]) and np.array_equal(a["log_req"][:lines], want["log_req"])
    assert cl.lines == lines and cl.out_bytes == int(want["log_off"][-1])


def _lines_untouched(a, line_cap, lout_cap):
    return all((v.view(np.uint8)[k:] == 0xA5).all() for v, k in ((a["lout"], lout_cap), (a["log_off"], 4 * (line_cap + 1)),
                                                                  (a["log_req"], 4 * line_cap)))


@pytest.mark.gpu
def test_gpu_mixed_residency():
    """responses pinned with log lines pageable, the reverse, and pinned responses with pageable per-request and
    per-connection columns: each equals the model and the all-pinned call byte for byte, for chunk sizes 7, 700 and 65536.
    In the first two, a capacity one short on either output is GOFR_ERR_CAPACITY, writes nothing at or past that capacity,
    and leaves the other output and the per-connection columns complete"""
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(Table(spec), 0)
    buf, off = CL._streams(2000)
    remote, roff, start = CL._clients(len(off) - 1)
    want, _ = CL.model(spec, buf, off, 3, remote, roff, start)
    n_req, n_bytes = len(want["meta"]), int(want["out_off"][-1])
    lines, lbytes = len(want["log_req"]), int(want["log_off"][-1])
    caps = (n_req, n_bytes, lines, lbytes)
    for chunk in (7, 700, 65536):
        eng.set_chunk(chunk)
        rc, ref, cr, cl = _submit(eng, buf, off, remote, roff, start, ALL, *caps)
        assert rc == 0 and cr.out_bytes == n_bytes
        CL._responses_equal(ref, want)
        _lines_equal(ref, cl, want)
        ref = {k: v.copy() for k, v in ref.items()}
        for what, pinned in MIXED.items():
            rc, a, cr, cl = _submit(eng, buf, off, remote, roff, start, pinned, *caps)
            assert rc == 0 and cr.out_bytes == n_bytes, (chunk, what)
            for k in ref:                                                   # canaries included
                assert a[k].tobytes() == ref[k].tobytes(), (chunk, what, k)
            if what == "columns pageable":
                continue
            for k in range(4):                                              # one short: req_cap, out_cap, line_cap, log out_cap
                short = list(caps)
                short[k] -= 1
                rc, a, cr, cl = _submit(eng, buf, off, remote, roff, start, pinned, *short)
                case = (chunk, what, k)
                assert rc == 7, case                                        # GOFR_ERR_CAPACITY
                assert cr.out_bytes == n_bytes and int(a["req_first"][len(off) - 1]) == n_req, case
                for c in ("req_first", "consumed", "conn_status"):
                    assert np.array_equal(a[c][:len(want[c])], want[c]), case
                if k < 2:
                    assert CB._untouched(a, short[0], short[1]), case
                    _lines_equal(a, cl, want)
                else:
                    assert _lines_untouched(a, short[2], short[3]), case
                    assert cl.lines == lines and cl.out_bytes == lbytes, case
                    CL._responses_equal(a, want)
    eng.close()


@pytest.mark.gpu
def test_gpu_route_refuses_a_bad_offset_in_a_later_chunk():
    """chunks of 7 connections: a buf_off that decreases at a connection of the fifth chunk, or passes buf_bytes at the last
    one, is refused with GOFR_ERR_INVALID, and the next route_connections on the engine equals the model"""
    spec = CC.c2_spec()
    eng = CC._engine(spec)
    buf, off = CC._streams(3000)
    m1 = CC._model(spec, buf, off, CC.SEED)
    dec = off.copy()
    dec[30] = dec[29] - 1
    past = off.copy()
    past[-1] = buf.size + 1
    eng.set_chunk(7)
    for pinned in (True, False):
        for bad in (dec, past):
            with pytest.raises(_abi.GofrError) as ei:                       # (the bound would refuse dec before the call)
                eng.route_connections(buf, bad, CC.SEED, pinned=pinned, req_cap=len(m1["meta"]) + 100)
            assert ei.value.code == 1
            CC._check_stage1(eng.route_connections(buf, off, CC.SEED, pinned=pinned), m1, pinned)
    eng.close()
