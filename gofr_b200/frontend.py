"""Batching front-ends: single records in from many threads, batches out to the GPU (include/gofr_b200.h).

The reference serves one request per goroutine (net/http conn.serve → Router.ServeHTTP, pkg/gofr/httpServer.go:29-33);
`Frontend.serve` is that per-request call (gofr_frontend_*): it blocks until the batch the request joined has come back.
grpc-go calls its codec once per message; `ProtoFrontend.call` is that call for the nested proto3 codec
(gofr_proto_frontend_*).  ctypes drops the GIL for the duration of a call, so Python threads can stand in for goroutines.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

from . import _abi
from . import spec as S
from .engine import Engine, nested_bound


class Frontend:
    def __init__(self, engine: Engine, max_batch: int = 4096, max_wait_us: int = 200, slot_bytes: int = 1024,
                 max_request_bytes: int = 4096):
        self._f = C.c_void_p()
        self.engine = engine
        self.slot_bytes = slot_bytes
        _abi.check(_abi.lib().gofr_frontend_create(C.byref(self._f), engine._e, max_batch, max_wait_us, slot_bytes,
                                                   max_request_bytes), "gofr_frontend_create")

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

    def stats(self) -> Tuple[int, int]:
        b, r = C.c_uint64(), C.c_uint64()
        _abi.check(_abi.lib().gofr_frontend_stats(self._f, C.byref(b), C.byref(r)), "gofr_frontend_stats")
        return int(b.value), int(r.value)

    def serve(self, method: int, path: bytes, query: bytes = b"", data: bytes = b"", trace_id: bytes = b"\0" * 16,
              flags: int = 0, resp_cap: int = 0) -> Tuple[bytes, int]:
        """One request → (response bytes, meta).  Blocks until the batch it joined has been served.  resp_cap: size of
        the caller's buffer (default: one slot); a response longer than the slot but within resp_cap is served alone."""
        assert len(trace_id) == 16
        cap = resp_cap or self.slot_bytes
        buf = C.create_string_buffer(cap)
        n, meta = C.c_uint32(), C.c_uint32()
        _abi.check(_abi.lib().gofr_frontend_serve(self._f, method, path, len(path), query, len(query), flags, data, len(data),
                                                  trace_id, buf, cap, C.byref(n), C.byref(meta)),
                   "gofr_frontend_serve")
        return buf.raw[:n.value], int(meta.value)


class ProtoFrontend:
    """One message type (spec.ProtoNField lists, as for Engine.proto_decode_batch) in one direction.  decode: call(message
    without the 5-byte prefix) → (row, status); encode: call(row) → (marshalled message without the prefix, status)."""

    def __init__(self, engine: Engine, msgs, root: int, decode: bool, max_batch: int = 1024, max_wait_us: int = 200,
                 max_record_bytes: int = 4096):
        self._f = C.c_void_p()
        self.engine = engine
        self.decode = bool(decode)
        self._nm, self._nf, k = S.proto_nested_tables(msgs)
        self._pr = S.proto_nested_presence(msgs)
        self.per_byte, self.per_record = nested_bound(msgs, root, self.decode)
        _abi.check(_abi.lib().gofr_proto_frontend_create(C.byref(self._f), engine._e, self._nm.ctypes.data, len(msgs),
                                                         self._nf.ctypes.data, k, root,
                                                         None if self._pr is None else self._pr.ctypes.data, int(self.decode),
                                                         max_batch, max_wait_us, max_record_bytes),
                   "gofr_proto_frontend_create")

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

    def call(self, data: bytes, out_cap: Optional[int] = None) -> Tuple[bytes, int]:
        """One record → (result bytes, GOFR_GRPC_* status).  Blocks until the batch it joined has come back.  out_cap: size
        of the caller's buffer, by default the bound of the record (never too small)."""
        if out_cap is None:
            out_cap = self.per_byte * (len(data) + 5) + self.per_record
        buf = C.create_string_buffer(max(out_cap, 1))
        n, status = C.c_uint32(), C.c_uint32()
        _abi.check(_abi.lib().gofr_proto_frontend_call(self._f, data, len(data), buf, out_cap, C.byref(n), C.byref(status)),
                   "gofr_proto_frontend_call")
        return buf.raw[:n.value], int(status.value)
