"""TEST INFRASTRUCTURE ONLY: CPU execution of the connection batch's compact step (see emu_conn.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gofr_b200 import spec as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libgofr_emu_conn.so")
SRCS = [os.path.join(HERE, "emu_conn.cpp"), os.path.join(ROOT, "gofr_b200", "csrc", "conn_device.cuh"),
        os.path.join(ROOT, "include", "gofr_b200.h")]
_lib = None


def _build():
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in SRCS)):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-fsanitize=undefined",
                               "-fno-sanitize-recover=undefined", "-static-libubsan", "-o", LIB, SRCS[0]])


def lib():
    global _lib
    if _lib is None:
        _build()
        _lib = C.CDLL(LIB)
        _lib.emu_conn_compact.argtypes = [C.c_void_p] * 4 + [C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4
        _lib.emu_conn_compact.restype = None
        _lib.emu_conn_trace_id.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p]
        _lib.emu_conn_trace_id.restype = None
    return _lib


def compact(first, conn_status, rec_off, desc, seed: int, conn0: int = 0, req0: int = 0):
    """conn_requests + conn_put over a framed chunk → (desc[requests], req_at[requests], ids[requests, 16], req_first[n + 1])"""
    n = len(first) - 1
    first = np.ascontiguousarray(first, dtype=np.uint32)
    conn_status = np.ascontiguousarray(conn_status, dtype=np.uint32)
    rec_off = np.ascontiguousarray(rec_off, dtype=np.uint32)
    desc = np.ascontiguousarray(desc).view(S.DESC_DTYPE)
    cap = max(int(first[-1]), 1)
    d_out = np.zeros(cap, dtype=S.DESC_DTYPE)
    req_at = np.zeros(cap, dtype=np.uint32)
    ids = np.zeros((cap, 16), dtype=np.uint8)
    req_first = np.zeros(n + 1, dtype=np.uint32)
    lib().emu_conn_compact(first.ctypes.data, conn_status.ctypes.data, rec_off.ctypes.data, desc.ctypes.data, n, seed, conn0, req0,
                           d_out.ctypes.data, req_at.ctypes.data, ids.ctypes.data, req_first.ctypes.data)
    k = int(req_first[n]) - req0
    return d_out[:k], req_at[:k], ids[:k], req_first


def trace_id(seed: int, c: int, j: int) -> bytes:
    out = (C.c_uint8 * 16)()
    lib().emu_conn_trace_id(seed, c, j, out)
    return bytes(out)
