"""ctypes binding of the CPU oracle of gofr_http_frame_device (tests/http_frame_oracle.c) — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__ and scratch/http_frame_bench.py may import this module."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "http_frame_oracle.c")
LIB = os.path.join(HERE, "libgofr_http_frame_oracle.so")
_lib = None


def build() -> None:
    if os.path.exists(LIB) and os.path.getmtime(SRC) <= os.path.getmtime(LIB):
        return
    subprocess.check_call(["gcc", "-O2", "-g", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", LIB, SRC])


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB)
        _lib.orc_http_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def http_frame(buf: np.ndarray, buf_off: np.ndarray, rec_cap: int | None = None):
    """orc_http_frame → (rec_off[total + 1], first[n + 1], consumed[n], status[n]): connection buffers cut into records."""
    n = len(buf_off) - 1
    cap = int(buf.size) // 16 + n + 1 if rec_cap is None else rec_cap
    rec = np.full(cap + 1, 0xEEEEEEEE, dtype=np.uint32)
    first = np.zeros(n + 1, dtype=np.uint32)
    consumed = np.zeros(max(n, 1), dtype=np.uint32)
    status = np.zeros(max(n, 1), dtype=np.uint32)
    bufp = np.concatenate([np.ascontiguousarray(buf, dtype=np.uint8), np.zeros(16, dtype=np.uint8)])
    off = np.ascontiguousarray(buf_off, dtype=np.uint32)
    if lib().orc_http_frame(bufp.ctypes.data, off.ctypes.data, n, rec.ctypes.data, cap, first.ctypes.data, consumed.ctypes.data,
                            status.ctypes.data):
        raise RuntimeError("oracle record capacity too small")
    return rec[:int(first[n]) + 1], first, consumed[:n], status[:n]
