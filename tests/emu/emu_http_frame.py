"""TEST INFRASTRUCTURE ONLY: CPU execution of the connection framer's per-connection code (see emu_http_frame.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libgofr_emu_http_frame.so")
CSRC = os.path.join(ROOT, "gofr_b200", "csrc")
_lib = None


def _build():
    srcs = [os.path.join(HERE, "emu_http_frame.cpp")] + [os.path.join(CSRC, h) for h in (
        "http_frame_device.cuh", "http_device.cuh", "serve_device.cuh", "value_device.cuh", "float_device.cuh", "bind_device.cuh",
        "table_format.h")]
    srcs = [s for s in srcs if os.path.exists(s)]
    if os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                           "-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-static-libubsan",
                           "-o", LIB, os.path.join(HERE, "emu_http_frame.cpp")])


def lib():
    global _lib
    if _lib is None:
        alt = os.environ.get("GOFR_EMU_HTTP_FRAME_LIB")   # a differently instrumented build (scratch/emu_asan.sh)
        if not alt:
            _build()
        _lib = C.CDLL(alt or LIB)
        _lib.emu_http_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def http_frame(buf: np.ndarray, buf_off: np.ndarray, rec_cap: int | None = None):
    """http_frame_count + http_frame_put (http_frame_device.cuh) on the CPU → (rec_off[total + 1], first[n + 1], consumed[n],
    status[n]); the buffer is handed over with exactly the 16 bytes of slack the ABI promises."""
    n = len(buf_off) - 1
    cap = int(buf.size) // 16 + n + 1 if rec_cap is None else rec_cap
    rec = np.full(cap + 1, 0xEEEEEEEE, dtype=np.uint32)
    first = np.zeros(n + 1, dtype=np.uint32)
    consumed = np.zeros(max(n, 1), dtype=np.uint32)
    status = np.zeros(max(n, 1), dtype=np.uint32)
    bufp = np.concatenate([np.ascontiguousarray(buf, dtype=np.uint8), np.zeros(16, dtype=np.uint8)])
    off = np.ascontiguousarray(buf_off, dtype=np.uint32)
    if lib().emu_http_frame(bufp.ctypes.data, off.ctypes.data, n, rec.ctypes.data, cap, first.ctypes.data, consumed.ctypes.data,
                            status.ctypes.data):
        raise RuntimeError("emu record capacity too small")
    return rec[:int(first[n]) + 1], first, consumed[:n], status[:n]
