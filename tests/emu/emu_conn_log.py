"""TEST INFRASTRUCTURE ONLY: CPU execution of the connection batch's request-log gather (see emu_conn_log.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gofr_b200 import spec as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.environ.get("GOFR_EMU_CONN_LOG_LIB", os.path.join(HERE, "libgofr_emu_conn_log.so"))
SRCS = [os.path.join(HERE, "emu_conn_log.cpp"), os.path.join(ROOT, "gofr_b200", "csrc", "conn_log_device.cuh"),
        os.path.join(ROOT, "gofr_b200", "csrc", "conn_device.cuh"), os.path.join(ROOT, "gofr_b200", "csrc", "engine_internal.h"),
        os.path.join(ROOT, "include", "gofr_b200.h")]
_lib = None


def _build():
    if "GOFR_EMU_CONN_LOG_LIB" in os.environ:   # a build of the caller's (scratch/emu_asan.sh: AddressSanitizer)
        return
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in SRCS)):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-fsanitize=undefined",
                               "-fno-sanitize-recover=undefined", "-static-libubsan", "-o", LIB, SRCS[0]])


def lib():
    global _lib
    if _lib is None:
        _build()
        _lib = C.CDLL(LIB)
        vp = C.c_void_p
        _lib.emu_conn_log.argtypes = [vp] * 11 + [C.c_int64, C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32] + [vp] * 5
        _lib.emu_conn_log.restype = None
    return _lib


def gather(first, conn_status, req_first, rec_off, spans, meta, ids, buf, alo: int, remote, remote_off, start_ns,
           log_ns: int, tz_offset_s: int, req0: int):
    """conn_log_count + conn_log_put over a chunk, laid out as the engine lays it out: buf is the chunk's bytes from buffer
    byte alo (absolute offsets address buf[off - alo]), remote the whole remote buffer, meta / ids / req_first per the
    chunk's requests (req_first rebased by req0) → (desc[lines] gofr_log_desc, ids[lines, 16], log_req[lines],
    line_first[n + 1], arena)"""
    n = len(first) - 1
    u32 = lambda a: np.ascontiguousarray(a, dtype=np.uint32)
    first, conn_status, req_first, rec_off, meta, remote_off = map(u32, (first, conn_status, req_first, rec_off, meta, remote_off))
    spans = np.ascontiguousarray(spans, dtype=np.uint64)
    ids = np.ascontiguousarray(ids, dtype=np.uint8).reshape(-1)
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    remote = np.concatenate([np.ascontiguousarray(remote, dtype=np.uint8), np.zeros(1, np.uint8)])
    start_ns = np.ascontiguousarray(start_ns, dtype=np.int64)
    lens = np.diff(remote_off.astype(np.int64))
    rmax = int(lens.max()) if n else 0
    n_req = max(len(meta), 1)
    out = np.zeros(n_req, dtype=S.LOG_DESC_DTYPE)
    line_ids = np.zeros((n_req, 16), dtype=np.uint8)
    line_req = np.zeros(n_req, dtype=np.uint32)
    line_first = np.zeros(n + 1, dtype=np.uint32)
    arena = np.zeros(buf.size + n_req * rmax + 64, dtype=np.uint8)
    lib().emu_conn_log(first.ctypes.data, conn_status.ctypes.data, req_first.ctypes.data, rec_off.ctypes.data, spans.ctypes.data,
                       meta.ctypes.data, ids.ctypes.data, buf.ctypes.data - alo, remote.ctypes.data, remote_off.ctypes.data,
                       start_ns.ctypes.data, log_ns, tz_offset_s, alo, rmax, req0, n, out.ctypes.data, line_first.ctypes.data,
                       line_ids.ctypes.data, line_req.ctypes.data, arena.ctypes.data)
    m = int(line_first[n])
    return out[:m], line_ids[:m], line_req[:m], line_first, arena
