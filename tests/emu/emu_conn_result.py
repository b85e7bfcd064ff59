"""TEST INFRASTRUCTURE ONLY: CPU execution of the connection results' splice step (see emu_conn_result.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gofr_b200 import spec as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.environ.get("GOFR_EMU_CONN_RESULT_LIB") or os.path.join(HERE, "libgofr_emu_conn_result.so")
CSRC = os.path.join(ROOT, "gofr_b200", "csrc")
_lib = None


def _build():
    if os.environ.get("GOFR_EMU_CONN_RESULT_LIB"):   # a prebuilt variant (scratch/emu_asan.sh)
        return
    srcs = [os.path.join(HERE, "emu_conn_result.cpp"), os.path.join(ROOT, "include", "gofr_b200.h")] + [
        os.path.join(CSRC, h) for h in ("conn_result_device.cuh", "serve_device.cuh", "value_device.cuh", "float_device.cuh",
                                        "bind_device.cuh", "engine_internal.h", "table_format.h")]
    srcs = [s for s in srcs if os.path.exists(s)]
    if os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                           "-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-static-libubsan",
                           "-o", LIB, os.path.join(HERE, "emu_conn_result.cpp")])


def lib():
    global _lib
    if _lib is None:
        _build()
        _lib = C.CDLL(LIB)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        _lib.emu_conn_result.argtypes = [vp, u32, vp, vp, u32, vp, u32, vp, u64, vp]
        _lib.emu_conn_result.restype = C.c_int
        _lib.emu_conn_result_any_mode.argtypes = [C.c_int]
        _lib.emu_conn_result_any_mode.restype = None
    return _lib


def _placed(data: bytes, slack: int, mis: int, fill: int = 0) -> np.ndarray:
    """data in a buffer whose first byte sits `mis` bytes past a 64-byte boundary, with `slack` readable bytes behind it"""
    raw = np.full(len(data) + slack + 128, fill, dtype=np.uint8)
    k = (-raw.ctypes.data) % 64 + mis
    a = raw[k:k + len(data) + slack]
    a[:len(data)] = np.frombuffer(data, np.uint8)
    return a


def splice(desc, arena, rec, rec_off, req0: int = 0, start: int = 0, mis: int = 0, any_mode: int = 0, canary=0xEE):
    """the splice of requests desc[i] (whose records are rec[rec_off[req0 + i]:rec_off[req0 + i + 1]]) from byte `start`
    of a 64-byte aligned output pre-filled with `canary` → (out, out_off, rewritten desc).  The parse arena and the records
    sit `mis` bytes past a 64-byte boundary; the records are staged from rec_off[req0] rounded down to 16, as the engine
    uploads them, and every source has 16 readable bytes behind it, as the device buffers do."""
    d = np.ascontiguousarray(desc).view(S.DESC_DTYPE).copy()
    n = len(d)
    ro = np.ascontiguousarray(rec_off[req0:req0 + n + 1], dtype=np.uint32)
    rec = bytes(rec)
    rlo = int(ro[0]) & ~15 if n else 0
    rchunk = _placed(rec[rlo:int(ro[-1]) if n else rlo], 16, mis)
    a = _placed(bytes(arena), 16, mis)
    size = sum(((int(x["path_len"]) + int(x["query_len"]) + 3) & ~3) for x in d)
    size += sum(((int(ro[i + 1]) - int(ro[i]) if ro[i + 1] > ro[i] else int(d[i]["data_len"])) + 3) & ~3 for i in range(n))
    out = _placed(b"", start + size + 64, 0, canary)
    out_off = np.zeros(n + 1, dtype=np.uint32)
    L = lib()
    L.emu_conn_result_any_mode(any_mode)
    try:
        rc = L.emu_conn_result(d.ctypes.data, n, a.ctypes.data, rchunk.ctypes.data, rlo, ro.ctypes.data, start, out.ctypes.data,
                               out.size, out_off.ctypes.data)
    finally:
        L.emu_conn_result_any_mode(0)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return out, out_off, d
