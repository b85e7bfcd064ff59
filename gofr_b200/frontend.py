"""Batching front-ends: single records in from many threads, batches out to the GPU (include/gofr_b200.h).

The reference serves one request per goroutine (net/http conn.serve → Router.ServeHTTP, pkg/gofr/httpServer.go:29-33);
`Frontend.serve` is that per-request call (gofr_frontend_*): it blocks until the batch the request joined has come back.
grpc-go calls its codec once per message; `ProtoFrontend.call` is that call for the nested proto3 codec
(gofr_proto_frontend_*).  A connection goroutine reads raw bytes; `ConnFrontend.serve` takes one such read and answers it
through the device framer, parser and serve chain (gofr_conn_frontend_*); `ConnAppFrontend.route` / `.respond` take it
through the closure path, with the closures run by the caller between the two calls (gofr_conn_app_frontend_*).  ctypes drops the GIL for the duration of a
call, so Python threads can stand in for goroutines.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

from . import _abi
from . import spec as S
from .engine import ConnLogLines, ConnResponses, ConnRoute, Engine, conn_batch_bound, conn_log_bound, nested_bound


class Frontend:
    def __init__(self, engine: Engine, max_batch: int = 4096, max_wait_us: int = 200, slot_bytes: int = 1024,
                 max_request_bytes: int = 4096, max_log_bytes: Optional[int] = None):
        """max_log_bytes: log staging per request (gofr_frontend_create_log), so that serve takes log=; None: none."""
        self._f = C.c_void_p()
        self.engine = engine
        self.slot_bytes = slot_bytes
        self.max_log_bytes = max_log_bytes
        if max_log_bytes is None:
            _abi.check(_abi.lib().gofr_frontend_create(C.byref(self._f), engine._e, max_batch, max_wait_us, slot_bytes,
                                                       max_request_bytes), "gofr_frontend_create")
        else:
            _abi.check(_abi.lib().gofr_frontend_create_log(C.byref(self._f), engine._e, max_batch, max_wait_us, slot_bytes,
                                                           max_request_bytes, max_log_bytes), "gofr_frontend_create_log")

    def close(self):
        if self._f:
            _abi.lib().gofr_frontend_destroy(self._f)
            self._f = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_clock(self, unix_seconds: int) -> None:
        """pin the Date header of every batch (tests); 0 = wall clock"""
        _abi.check(_abi.lib().gofr_frontend_set_clock(self._f, unix_seconds), "gofr_frontend_set_clock")

    def set_log_clock(self, unix_ns: int) -> None:
        """pin the log time of every line (tests); 0 = wall clock"""
        _abi.check(_abi.lib().gofr_frontend_set_log_clock(self._f, unix_ns), "gofr_frontend_set_log_clock")

    def stats(self) -> Tuple[int, int]:
        b, r = C.c_uint64(), C.c_uint64()
        _abi.check(_abi.lib().gofr_frontend_stats(self._f, C.byref(b), C.byref(r)), "gofr_frontend_stats")
        return int(b.value), int(r.value)

    def serve(self, method: int, path: bytes, query: bytes = b"", data: bytes = b"", trace_id: bytes = b"\0" * 16,
              flags: int = 0, resp_cap: int = 0, log: Optional[S.LogRec] = None, line_cap: int = 0):
        """One request → (response bytes, meta).  Blocks until the batch it joined has been served.  resp_cap: size of
        the caller's buffer (default: one slot); a response longer than the slot but within resp_cap is served alone.
        With log (a LogRec: its start time, zone, strings and kind LOG_REQUEST / LOG_NONE; the rest is the call's) →
        (response bytes, meta, line) through gofr_frontend_serve_log; line_cap defaults to the bound of the record."""
        assert len(trace_id) == 16
        cap = resp_cap or self.slot_bytes
        buf = C.create_string_buffer(cap)
        n, meta = C.c_uint32(), C.c_uint32()
        if log is not None:
            lb = S.LogBatch.pack([log])
            strings = lb.arena.tobytes()
            lcap = line_cap or 320 + 6 * len(strings)
            line = C.create_string_buffer(max(lcap, 1))
            ln = C.c_uint32()
            _abi.check(_abi.lib().gofr_frontend_serve_log(self._f, method, path, len(path), query, len(query), flags, data,
                                                          len(data), trace_id, lb.desc.ctypes.data, strings, buf, cap,
                                                          C.byref(n), C.byref(meta), line, lcap, C.byref(ln)),
                       "gofr_frontend_serve_log")
            return buf.raw[:n.value], int(meta.value), line.raw[:ln.value]
        _abi.check(_abi.lib().gofr_frontend_serve(self._f, method, path, len(path), query, len(query), flags, data, len(data),
                                                  trace_id, buf, cap, C.byref(n), C.byref(meta)),
                   "gofr_frontend_serve")
        return buf.raw[:n.value], int(meta.value)


class ProtoFrontend:
    """One message type (spec.ProtoNField lists, as for Engine.proto_decode_batch) in one direction.  decode: call(message
    without the 5-byte prefix) → (row, status); encode: call(row) → (marshalled message without the prefix, status).
    max_log_bytes (encode only): log staging of that many method bytes per call (gofr_proto_frontend_create_log), so that
    call takes log=; None: none."""

    def __init__(self, engine: Engine, msgs, root: int, decode: bool, max_batch: int = 1024, max_wait_us: int = 200,
                 max_record_bytes: int = 4096, max_log_bytes: Optional[int] = None):
        self._f = C.c_void_p()
        self.engine = engine
        self.decode = bool(decode)
        self._nm, self._nf, k = S.proto_nested_tables(msgs)
        self._pr = S.proto_nested_presence(msgs)
        self.per_byte, self.per_record = nested_bound(msgs, root, self.decode)
        pr = None if self._pr is None else self._pr.ctypes.data
        if max_log_bytes is None:
            _abi.check(_abi.lib().gofr_proto_frontend_create(C.byref(self._f), engine._e, self._nm.ctypes.data, len(msgs),
                                                             self._nf.ctypes.data, k, root, pr, int(self.decode), max_batch,
                                                             max_wait_us, max_record_bytes),
                       "gofr_proto_frontend_create")
        else:
            _abi.check(_abi.lib().gofr_proto_frontend_create_log(C.byref(self._f), engine._e, self._nm.ctypes.data, len(msgs),
                                                                 self._nf.ctypes.data, k, root, pr, int(self.decode), max_batch,
                                                                 max_wait_us, max_record_bytes, max_log_bytes),
                       "gofr_proto_frontend_create_log")

    def close(self):
        if self._f:
            _abi.lib().gofr_proto_frontend_destroy(self._f)
            self._f = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stats(self) -> Tuple[int, int]:
        b, r = C.c_uint64(), C.c_uint64()
        _abi.check(_abi.lib().gofr_proto_frontend_stats(self._f, C.byref(b), C.byref(r)), "gofr_proto_frontend_stats")
        return int(b.value), int(r.value)

    def set_log_clock(self, unix_ns: int) -> None:
        """pin the log time of every line (tests); 0 = wall clock"""
        _abi.check(_abi.lib().gofr_proto_frontend_set_log_clock(self._f, unix_ns), "gofr_proto_frontend_set_log_clock")

    def call(self, data: bytes, out_cap: Optional[int] = None, log: Optional[S.LogRec] = None, trace_id: bytes = b"\0" * 16,
             line_cap: int = 0):
        """One record → (result bytes, GOFR_GRPC_* status).  Blocks until the batch it joined has come back.  out_cap: size
        of the caller's buffer, by default the bound of the record (never too small).  With log (a LogRec: its start time,
        elapsed time, zone, method and kind LOG_RPC / LOG_NONE; the rest is ignored) and the span's trace_id → (message,
        status, RPCLog line) through gofr_proto_frontend_call_log; data may be empty (the handler failed); line_cap
        defaults to the bound of the record."""
        if out_cap is None:
            out_cap = self.per_byte * (len(data) + 5) + self.per_record
        buf = C.create_string_buffer(max(out_cap, 1))
        n, status = C.c_uint32(), C.c_uint32()
        if log is not None:
            assert len(trace_id) == 16
            lb = S.LogBatch.pack([log])
            method = lb.arena.tobytes()[:int(lb.desc["method_len"][0])]
            lcap = line_cap or 320 + 7 * len(method)
            line = C.create_string_buffer(max(lcap, 1))
            ln = C.c_uint32()
            _abi.check(_abi.lib().gofr_proto_frontend_call_log(self._f, data, len(data), trace_id, lb.desc.ctypes.data, method,
                                                               buf, out_cap, C.byref(n), C.byref(status), line, lcap,
                                                               C.byref(ln)),
                       "gofr_proto_frontend_call_log")
            return buf.raw[:n.value], int(status.value), line.raw[:ln.value]
        _abi.check(_abi.lib().gofr_proto_frontend_call(self._f, data, len(data), buf, out_cap, C.byref(n), C.byref(status)),
                   "gofr_proto_frontend_call")
        return buf.raw[:n.value], int(status.value)


class ConnFrontend:
    """One read of one connection per call: serve(bytes held for the connection) → ConnResponses of that connection alone
    (n_conns = 1: req_first, consumed and conn_status have one connection's entries), with .log when the front-end was
    created with log.  On MORE keep buf[consumed[0]:] and append the next read; on DEFER write the responses, then hand
    buf[consumed[0]:] to net/http; a hole (status 0) is served from buf[req_at[k]:]."""

    def __init__(self, engine: Engine, max_batch: int = 1024, max_wait_us: int = 200, max_conn_bytes: int = 16384,
                 log: bool = False, tz_offset_s: int = 0, seed: int = 0):
        self._f = C.c_void_p()
        self.engine = engine
        self.log = bool(log)
        _abi.check(_abi.lib().gofr_conn_frontend_create(C.byref(self._f), engine._e, max_batch, max_wait_us, max_conn_bytes,
                                                        int(self.log), tz_offset_s, seed), "gofr_conn_frontend_create")

    def close(self):
        if self._f:
            _abi.lib().gofr_conn_frontend_destroy(self._f)
            self._f = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_clock(self, unix_ns: int) -> None:
        """pin the Date header and the log time of every batch (tests); 0 = wall clock"""
        _abi.check(_abi.lib().gofr_conn_frontend_set_clock(self._f, unix_ns), "gofr_conn_frontend_set_clock")

    def stats(self) -> Tuple[int, int, int]:
        """(batches, connection reads served, batches served again after their outputs grew)"""
        b, c, r = C.c_uint64(), C.c_uint64(), C.c_uint64()
        _abi.check(_abi.lib().gofr_conn_frontend_stats(self._f, C.byref(b), C.byref(c), C.byref(r)), "gofr_conn_frontend_stats")
        return int(b.value), int(c.value), int(r.value)

    def serve(self, buf: bytes, remote: bytes = b"", start_unix_ns: int = 0) -> ConnResponses:
        """Blocks until the batch this read joined has been served.  remote: the connection's req.RemoteAddr (at most 255
        bytes); start_unix_ns: Logging's start clock for this read.  The outputs are sized with gofr_conn_batch_bound /
        gofr_conn_log_bound on {0, len(buf)}, which always suffice; a read past max_conn_bytes raises
        GofrError(GOFR_ERR_CAPACITY)."""
        buf = bytes(buf)
        off = np.array([0, len(buf)], np.uint32)
        req_cap, out_cap = conn_batch_bound(self.engine.table, off)
        out, out_off, meta = np.zeros(max(out_cap, 1), np.uint8), np.zeros(req_cap + 1, np.uint32), np.zeros(max(req_cap, 1), np.uint32)
        req_at, ids = np.zeros(max(req_cap, 1), np.uint32), np.zeros(max(req_cap, 1) * 16, np.uint8)
        req_first, consumed, status = np.zeros(2, np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint32)
        cr = _abi.ConnResp(out=out.ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data,
                           req_at=req_at.ctypes.data, trace_ids=ids.ctypes.data, req_first=req_first.ctypes.data,
                           consumed=consumed.ctypes.data, conn_status=status.ctypes.data, out_bytes=0)
        cl = None
        if self.log:
            line_cap, log_out_cap = conn_log_bound(off, np.array([0, len(remote)], np.uint32))
            lout, log_off, log_req = np.zeros(max(log_out_cap, 1), np.uint8), np.zeros(line_cap + 1, np.uint32), np.zeros(max(line_cap, 1), np.uint32)
            cl = _abi.ConnLog(line_cap=line_cap, out=lout.ctypes.data, out_cap=log_out_cap, log_off=log_off.ctypes.data,
                              log_req=log_req.ctypes.data)
        _abi.check(_abi.lib().gofr_conn_frontend_serve(self._f, buf, len(buf), remote, len(remote), start_unix_ns, C.byref(cr),
                                                       C.byref(cl) if cl is not None else None), "gofr_conn_frontend_serve")
        k = int(req_first[1])
        lines = None
        if cl is not None:
            m = cl.lines
            lines = ConnLogLines(lout[:int(cl.out_bytes)], log_off[:m + 1], log_req[:m], m, int(cl.out_bytes))
        return ConnResponses(out[:int(cr.out_bytes)], out_off[:k + 1], meta[:k], req_at[:k], ids[:k * 16].reshape(k, 16), req_first,
                             consumed, status, lines)


@dataclass
class ConnAppRoute:
    """What ConnAppFrontend.route returns for one read: its requests as gofr_conn_batch_route gives them for a batch of one
    (.route, rebased to this read: req_at into the read, desc into route.arena), the binds of the routes that declared a
    schema (bind_status[k]: GOFR_BIND_*, 0xFFFFFFFF not bound; row k is rows[row_off[k]:row_off[k + 1]]) and the read's
    trace key, which respond takes."""
    route: ConnRoute
    bind_status: np.ndarray  # uint32[requests]
    row_off: np.ndarray      # uint32[requests + 1]
    rows: np.ndarray         # uint8
    trace_key: int


class ConnAppFrontend:
    """The closure path one read per call: route(read) → ConnAppRoute; the caller runs the closures of its status-0
    requests and encodes their records; respond(read, trace_key, rec, rec_off) → ConnResponses as ConnFrontend.serve
    returns them (gofr_conn_app_frontend_*).  route_schema: {route id: (schema id, field count)} of the routes whose
    closures call Context.Bind, bound for the whole route batch."""

    def __init__(self, engine: Engine, max_batch: int = 1024, max_wait_us: int = 200, max_conn_bytes: int = 16384,
                 log: bool = False, tz_offset_s: int = 0, seed: int = 0, route_schema: Optional[dict] = None):
        self._f = C.c_void_p()
        self.engine = engine
        self.log = bool(log)
        rs = route_schema or {}
        n_routes = max(rs) + 1 if rs else 0
        self._schema = np.zeros(max(n_routes, 1), np.uint32)
        self._fields = np.zeros(max(n_routes, 1), np.uint32)
        for r, (s, nf) in rs.items():
            self._schema[r], self._fields[r] = s, nf
        self.max_fields = int(self._fields.max())
        _abi.check(_abi.lib().gofr_conn_app_frontend_create(C.byref(self._f), engine._e, max_batch, max_wait_us, max_conn_bytes,
                                                            int(self.log), tz_offset_s, seed, self._schema.ctypes.data, n_routes,
                                                            self._fields.ctypes.data), "gofr_conn_app_frontend_create")

    def close(self):
        if self._f:
            _abi.lib().gofr_conn_app_frontend_destroy(self._f)
            self._f = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_clock(self, unix_ns: int) -> None:
        """pin the Date header and the log time of every respond batch (tests); 0 = wall clock"""
        _abi.check(_abi.lib().gofr_conn_app_frontend_set_clock(self._f, unix_ns), "gofr_conn_app_frontend_set_clock")

    def stats(self) -> dict:
        st = _abi.ConnAppStats()
        _abi.check(_abi.lib().gofr_conn_app_frontend_stats(self._f, C.byref(st)), "gofr_conn_app_frontend_stats")
        return {name: int(getattr(st, name)) for name, _ in _abi.ConnAppStats._fields_}

    def route(self, buf: bytes) -> ConnAppRoute:
        """Blocks until the route batch this read joined has been routed and bound.  The outputs are sized so that they
        always suffice; a read past max_conn_bytes raises GofrError(GOFR_ERR_CAPACITY)."""
        buf = bytes(buf)
        req_cap, _ = conn_batch_bound(self.engine.table, np.array([0, len(buf)], np.uint32))
        rc1 = max(req_cap, 1)
        desc, arena = np.zeros(rc1, S.DESC_DTYPE), np.zeros(len(buf) + 80, np.uint8)
        meta, vars_, req_at, ids = np.zeros(rc1, np.uint32), np.zeros(rc1 * 8, np.uint32), np.zeros(rc1, np.uint32), np.zeros(rc1 * 16, np.uint8)
        req_first, consumed, status = np.zeros(2, np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint32)
        # GOFR_BIND_ROW_BOUND without the schemas' names, which this wrapper does not know: a read whose error texts need
        # more is routed again with the rows it reported
        rows_cap = req_cap * (8 * self.max_fields + 70) + 3 * len(buf)
        bstat, row_off = np.zeros(rc1, np.uint32), np.zeros(rc1 + 1, np.uint32)
        cr = _abi.ConnRoute(req_cap=req_cap, desc=desc.ctypes.data, arena=arena.ctypes.data, meta=meta.ctypes.data,
                            vars=vars_.ctypes.data, req_at=req_at.ctypes.data, trace_ids=ids.ctypes.data,
                            req_first=req_first.ctypes.data, consumed=consumed.ctypes.data, conn_status=status.ctypes.data)
        key = C.c_uint64()
        while True:
            rows = np.zeros(max(rows_cap, 1), np.uint8)
            cb = _abi.ConnAppBind(status=bstat.ctypes.data, row_off=row_off.ctypes.data, rows=rows.ctypes.data, rows_cap=rows_cap)
            rc = _abi.lib().gofr_conn_app_frontend_route(self._f, buf, len(buf), C.byref(cr), C.byref(cb), C.byref(key))
            if rc != 7 or cb.rows_bytes <= rows_cap:   # GOFR_ERR_CAPACITY for anything else: the read is too long
                break
            rows_cap = int(cb.rows_bytes)
        _abi.check(rc, "gofr_conn_app_frontend_route")
        k = int(req_first[1])
        r = ConnRoute(desc[:k], arena, meta[:k], vars_[:k * 8].reshape(k, 8), req_at[:k], ids[:k * 16].reshape(k, 16), req_first,
                      consumed, status)
        return ConnAppRoute(r, bstat[:k], row_off[:k + 1], rows[:int(cb.rows_bytes)], int(key.value))

    def respond(self, buf: bytes, trace_key: int, rec: bytes, rec_off, remote: bytes = b"", start_unix_ns: int = 0) -> ConnResponses:
        """Blocks until the respond batch this read joined has been served: the same read as its route call, its trace key,
        and request k's record rec[rec_off[k]:rec_off[k + 1]] (empty: the request is answered as the batch call answers it).
        Returns ConnResponses as ConnFrontend.serve does."""
        buf, rec = bytes(buf), np.frombuffer(bytes(rec) or b"\0", np.uint8)
        roff = np.ascontiguousarray(rec_off, dtype=np.uint32)
        off = np.array([0, len(buf)], np.uint32)
        req_cap, out_cap = conn_batch_bound(self.engine.table, off)
        rb = lambda dl: _abi.lib().gofr_table_response_bound(self.engine.table.handle, 0, 0, dl)
        out_cap += (rb(1) - rb(0)) * int(roff[-1] if len(roff) else 0)   # a record byte grows a response by at most this much
        out, out_off, meta = np.zeros(max(out_cap, 1), np.uint8), np.zeros(req_cap + 1, np.uint32), np.zeros(max(req_cap, 1), np.uint32)
        req_at, ids = np.zeros(max(req_cap, 1), np.uint32), np.zeros(max(req_cap, 1) * 16, np.uint8)
        req_first, consumed, status = np.zeros(2, np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint32)
        cr = _abi.ConnResp(out=out.ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data,
                           req_at=req_at.ctypes.data, trace_ids=ids.ctypes.data, req_first=req_first.ctypes.data,
                           consumed=consumed.ctypes.data, conn_status=status.ctypes.data, out_bytes=0)
        res = _abi.ConnResults(rec=rec.ctypes.data, rec_off=roff.ctypes.data if len(roff) else None,
                               rec_bytes=int(roff[-1]) if len(roff) else 0, n_req=max(len(roff) - 1, 0))
        cl = None
        if self.log:
            line_cap, log_out_cap = conn_log_bound(off, np.array([0, len(remote)], np.uint32))
            lout, log_off, log_req = np.zeros(max(log_out_cap, 1), np.uint8), np.zeros(line_cap + 1, np.uint32), np.zeros(max(line_cap, 1), np.uint32)
            cl = _abi.ConnLog(line_cap=line_cap, out=lout.ctypes.data, out_cap=log_out_cap, log_off=log_off.ctypes.data,
                              log_req=log_req.ctypes.data)
        _abi.check(_abi.lib().gofr_conn_app_frontend_respond(self._f, buf, len(buf), trace_key, C.byref(res), remote, len(remote),
                                                             start_unix_ns, C.byref(cr), C.byref(cl) if cl is not None else None),
                   "gofr_conn_app_frontend_respond")
        k = int(req_first[1])
        lines = None
        if cl is not None:
            m = cl.lines
            lines = ConnLogLines(lout[:int(cl.out_bytes)], log_off[:m + 1], log_req[:m], m, int(cl.out_bytes))
        return ConnResponses(out[:int(cr.out_bytes)], out_off[:k + 1], meta[:k], req_at[:k], ids[:k * 16].reshape(k, 16), req_first,
                             consumed, status, lines)
