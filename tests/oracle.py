"""ctypes binding of the CPU oracle (oracle/libgofr_oracle.so) — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Tuple

import numpy as np

from gofr_b200 import spec as S

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB_PATH = os.path.join(_ROOT, "oracle", "libgofr_oracle.so")
_lib = None


def build() -> None:
    srcs = ["gofr_oracle.c", "orc_bind.c", "orc_grpc.c", "orc_reqlog.c", "orc_http.c", "orc_proto.c", "orc_proto_nested.c", "orc_value.c", "gofr_oracle.h", "orc_internal.h", "Makefile"]
    odir = os.path.join(_ROOT, "oracle")
    if os.path.exists(_LIB_PATH):
        so_m = os.path.getmtime(_LIB_PATH)
        if all(os.path.getmtime(os.path.join(odir, s)) <= so_m for s in srcs):
            return
    subprocess.check_call(["make", "-C", odir, "-s", "CC=gcc"])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.orc_table_new.restype = C.c_void_p
        L.orc_table_new.argtypes = [C.c_int]
        L.orc_table_free.argtypes = [C.c_void_p]
        L.orc_add_schema.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_char_p),
                                     C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.orc_schema_extend.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.orc_json_float64.argtypes = [C.c_double, C.c_char_p, C.c_int]
        L.orc_json_float32.argtypes = [C.c_float, C.c_char_p, C.c_int]
        L.orc_encode_row_json.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_int]
        L.orc_add_route.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int] + \
            [C.c_char_p, C.c_int] * 4 + [C.c_char_p, C.c_int]
        L.orc_add_default_routes.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        L.orc_serve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_void_p,
                                C.c_uint64, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_route_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_http_parse.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_request_log.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        L.orc_grpc_hello.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                     C.c_int]
        L.orc_proto_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                       C.c_void_p]
        L.orc_proto_decode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                       C.c_void_p]
        for name in ("orc_json_string", "orc_clean_path", "orc_escape_path"):
            getattr(L, name).argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int]
        L.orc_json_int.argtypes = [C.c_int64, C.c_char_p, C.c_int]
        L.orc_query_get.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_int]
        L.orc_match.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
        L.orc_bind.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_int]
        L.orc_rpclog_string.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_char_p, C.c_int]
        L.orc_format_http_date.argtypes = [C.c_int64, C.c_char_p]
        _lib = L
    return _lib


def set_strict_chunking(on: bool) -> None:
    """oracle only: frame JSON bodies beyond 2 KiB as the reference does (Transfer-Encoding: chunked) instead of as the product
    does (Content-Length) — see oracle/gofr_oracle.c rw_write and DESIGN.md §8"""
    lib().orc_set_strict_chunking(1 if on else 0)


def _buf_call(fn, *args, cap=1 << 16) -> bytes:
    out = C.create_string_buffer(cap)
    n = fn(*args, out, cap)
    if n < 0:
        raise RuntimeError(f"oracle call failed: {n}")
    return out.raw[:n]


def json_string(s: bytes) -> bytes:
    return _buf_call(lib().orc_json_string, s, len(s), cap=len(s) * 6 + 16)


def json_int(v: int) -> bytes:
    return _buf_call(lib().orc_json_int, v)


def clean_path(p: bytes) -> bytes:
    return _buf_call(lib().orc_clean_path, p, len(p), cap=len(p) + 16)


def escape_path(p: bytes) -> bytes:
    return _buf_call(lib().orc_escape_path, p, len(p), cap=len(p) * 3 + 16)


def query_get(q: bytes, key: bytes) -> bytes:
    return _buf_call(lib().orc_query_get, q, len(q), key, len(key), cap=len(q) + 16)


def rpclog_string(id_: str, start: str, rt: int, method: str) -> bytes:
    return _buf_call(lib().orc_rpclog_string, id_.encode(), start.encode(), rt, method.encode())


def http_date(unix_seconds: int) -> bytes:
    out = C.create_string_buffer(29)
    lib().orc_format_http_date(unix_seconds, out)
    return out.raw[:29]


class OracleTable:
    def __init__(self, spec: S.TableSpec):
        L = lib()
        self._t = L.orc_table_new(spec.frame_mode)
        self.spec = spec
        for sc in spec.schemas:
            n = len(sc.fields)
            go = (C.c_char_p * n)(*[f.go_name.encode() for f in sc.fields])
            js = (C.c_char_p * n)(*[f.json_name.encode() for f in sc.fields])
            kinds = (C.c_int * n)(*[f.kind for f in sc.fields])
            oe = (C.c_int * n)(*[1 if f.omitempty else 0 for f in sc.fields])
            L.orc_add_schema(self._t, sc.id, sc.go_type.encode(), n, go, js, kinds, oe)
            L.orc_schema_extend(self._t, (C.c_int * n)(*[f.container for f in sc.fields]), (C.c_int * n)(*[f.flags for f in sc.fields]),
                                (C.c_int * n)(*[f.elem_schema for f in sc.fields]))
        self.route_ids = []
        for r in spec.routes:
            p = r.pattern.encode()
            rid = L.orc_add_route(self._t, r.method, p, len(p), r.kind, r.schema_id, r.s0, len(r.s0), r.s1, len(r.s1),
                                  r.s2, len(r.s2), r.s3, len(r.s3), r.blob, len(r.blob))
            if rid < 0:
                raise ValueError(f"oracle refused route {r.pattern!r}")
            self.route_ids.append(rid)
        if spec.default_routes:
            L.orc_add_default_routes(self._t, spec.favicon, len(spec.favicon))

    def __del__(self):
        try:
            lib().orc_table_free(self._t)
        except Exception:
            pass

    def match(self, method: int, path: bytes) -> int:
        return lib().orc_match(self._t, method, path, len(path))

    def encode_row_json(self, schema_id: int, row: bytes):
        """JSON text of one handler-result row; None: malformed, b"": not encodable (NaN / Inf)"""
        out = C.create_string_buffer(64 + 8 * len(row))
        n = lib().orc_encode_row_json(self._t, schema_id, row, len(row), out, len(out))
        return None if n == -1 else b"" if n == -2 else out.raw[:n]

    def bind(self, schema_id: int, body: bytes):
        cap = len(body) * 4 + 4096
        while True:
            out = C.create_string_buffer(cap)
            n = lib().orc_bind(self._t, schema_id, body, len(body), out, len(out))
            if n != -1000000:   # -1000000: the row or error text did not fit (an error text names the type and the field)
                break
            cap *= 4
        if n >= 0:
            return True, out.raw[:n]
        return False, out.raw[:-n]

    def serve(self, batch: S.RequestBatch, date: bytes, out_cap: int | None = None,
              nthreads: int = 1) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        n = batch.n
        if out_cap is None:
            out_cap = max(4096, n * 640 + int(batch.arena.size) * 6 + len(self.spec.favicon) * n // 4)
        out = np.zeros(out_cap, dtype=np.uint8)
        off = np.zeros(n + 1, dtype=np.uint32)
        meta = np.zeros(n, dtype=np.uint32)
        rc = lib().orc_serve(self._t, batch.desc.ctypes.data, batch.trace_ids.ctypes.data, batch.arena.ctypes.data, n,
                             date, out.ctypes.data, out_cap, off.ctypes.data, meta.ctypes.data, nthreads)
        if rc != 0:
            raise RuntimeError("oracle output capacity too small")
        return out, off, meta


MAX_PATH_VARS = 8


def route(table: "OracleTable", batch) -> Tuple[np.ndarray, np.ndarray]:
    """Router.Match + mux.Vars for every request: (meta[n], vars[n, 8])."""
    n = batch.n
    meta = np.zeros(n, dtype=np.uint32)
    vars_ = np.zeros((n, MAX_PATH_VARS), dtype=np.uint32)
    lib().orc_route_batch(table._t, batch.desc.ctypes.data, batch.arena.ctypes.data, n, meta.ctypes.data, vars_.ctypes.data,
                    MAX_PATH_VARS)
    return meta, vars_


def responses(out: np.ndarray, off: np.ndarray):
    b = out.tobytes()
    return [b[int(off[i]):int(off[i + 1])] for i in range(len(off) - 1)]


def http_parse(raw: np.ndarray, raw_off: np.ndarray):
    """orc_http_parse → (desc[n] in gofr_req_desc layout, arena, status[n], spans[n, 6])."""
    n = len(raw_off) - 1
    desc = np.zeros(n, dtype=S.DESC_DTYPE)
    arena = np.zeros(int(raw.size) + 32, dtype=np.uint8)
    status = np.zeros(n, dtype=np.uint32)
    spans = np.zeros((n, 6), dtype=np.uint64)
    rawp = np.concatenate([raw, np.zeros(16, dtype=np.uint8)])
    lib().orc_http_parse(rawp.ctypes.data, raw_off.ctypes.data, n, desc.ctypes.data, arena.ctypes.data, status.ctypes.data,
                         spans.ctypes.data)
    return desc, arena, status, spans


def request_log(batch):
    """batch: gofr_b200.spec.LogBatch → (out, out_off): the packed RequestLog lines (orc_reqlog.c)."""
    n = batch.n
    cap = 400 * n + 6 * int(batch.arena.size) + 64
    out = np.zeros(cap, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    arena = batch.arena if batch.arena.size else np.zeros(1, dtype=np.uint8)
    rc = lib().orc_request_log(batch.desc.ctypes.data, batch.trace_ids.ctypes.data, arena.ctypes.data, n,
                               out.ctypes.data, cap, off.ctypes.data)
    if rc != 0:
        raise RuntimeError("oracle output capacity too small")
    return out, off


def grpc_hello(frames: np.ndarray, in_off: np.ndarray, nthreads: int = 1):
    n = len(in_off) - 1
    cap = int(frames.size) + 32 * n + 64
    out = np.zeros(cap, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(n, dtype=np.uint32)
    rc = lib().orc_grpc_hello(frames.ctypes.data, in_off.ctypes.data, n, out.ctypes.data, cap, off.ctypes.data,
                              meta.ctypes.data, nthreads)
    if rc != 0:
        raise RuntimeError("oracle output capacity too small")
    return out, off, meta


def proto_encode(fields, rows: np.ndarray, row_off: np.ndarray):
    """orc_proto_encode: proto.Marshal + gRPC length prefix per row → (out, out_off, meta)."""
    n = len(row_off) - 1
    ft = np.array([[f.number, f.type] for f in fields], dtype=np.uint32).reshape(-1)
    cap = int(rows.size) * 3 + 32 * n * max(len(fields), 1) + 64
    out = np.zeros(cap, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    rows = np.ascontiguousarray(rows)
    rc = lib().orc_proto_encode(ft.ctypes.data, len(fields), rows.ctypes.data, row_off.ctypes.data, n, out.ctypes.data, cap,
                                off.ctypes.data, meta.ctypes.data)
    assert rc == 0
    return out, off, meta[:n]


def proto_encode_nested(msgs, root: int, rows: np.ndarray, row_off: np.ndarray):
    """orc_proto_encode_nested: message types with nested / repeated fields → (out, out_off, meta)."""
    n = len(row_off) - 1
    mt, ft, k = [], [], 0
    for fields in msgs:
        mt += [k, len(fields)]
        for f in fields:
            ft += [f.number, f.type, 1 if f.repeated else 0, f.msg]
            k += 1
    mt, ft = np.array(mt, dtype=np.uint32), np.array(ft, dtype=np.uint32)
    cap = int(rows.size) * 4 + 64 * n + 64
    out = np.zeros(cap, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    rows = np.ascontiguousarray(rows)
    lib().orc_proto_encode_nested.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                              C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    rc = lib().orc_proto_encode_nested(mt.ctypes.data, len(msgs), ft.ctypes.data, k, root, rows.ctypes.data, row_off.ctypes.data, n,
                                       out.ctypes.data, cap, off.ctypes.data, meta.ctypes.data)
    assert rc == 0
    return out, off, meta[:n]


def proto_decode_nested(msgs, root: int, frames: np.ndarray, in_off: np.ndarray):
    """orc_proto_decode_nested: frames → rows of message types with nested / repeated fields → (rows, row_off, meta)."""
    n = len(in_off) - 1
    mt, ft, k = [], [], 0
    for fields in msgs:
        mt += [k, len(fields)]
        for f in fields:
            ft += [f.number, f.type, 1 if f.repeated else 0, f.msg]
            k += 1
    mt, ft = np.array(mt, dtype=np.uint32), np.array(ft, dtype=np.uint32)
    cap = int(frames.size) * 10 + 4096 * max(n, 1)
    rows = np.zeros(cap, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    frames = np.ascontiguousarray(frames)
    lib().orc_proto_decode_nested.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                              C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    rc = lib().orc_proto_decode_nested(mt.ctypes.data, len(msgs), ft.ctypes.data, k, root, frames.ctypes.data, in_off.ctypes.data, n,
                                       rows.ctypes.data, cap, off.ctypes.data, meta.ctypes.data)
    assert rc == 0
    return rows, off, meta[:n]


def proto_decode(fields, frames: np.ndarray, in_off: np.ndarray):
    """orc_proto_decode: gRPC frames → rows (proto.Unmarshal) → (rows, row_off, meta)."""
    n = len(in_off) - 1
    ft = np.array([[f.number, f.type] for f in fields], dtype=np.uint32).reshape(-1)
    cap = int(frames.size) + (8 * len(fields) + 8) * n + 64
    rows = np.zeros(cap, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    frames = np.ascontiguousarray(frames)
    rc = lib().orc_proto_decode(ft.ctypes.data, len(fields), frames.ctypes.data, in_off.ctypes.data, n, rows.ctypes.data, cap,
                                off.ctypes.data, meta.ctypes.data)
    assert rc == 0
    return rows, off, meta[:n]
