"""TEST INFRASTRUCTURE ONLY: CPU execution of the chunk pack kernel's per-record logic (see emu_pack.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libgofr_emu_pack.so")
CSRC = os.path.join(ROOT, "gofr_b200", "csrc")
_lib = None


def _build():
    srcs = [os.path.join(HERE, "emu_pack.cpp")] + [os.path.join(CSRC, h) for h in (
        "pack_device.cuh", "serve_device.cuh", "value_device.cuh", "float_device.cuh", "bind_device.cuh", "engine_internal.h",
        "table_format.h")]
    srcs = [s for s in srcs if os.path.exists(s)]
    if os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                           "-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-static-libubsan",
                           "-o", LIB, os.path.join(HERE, "emu_pack.cpp")])


def lib():
    global _lib
    if _lib is None:
        _build()
        _lib = C.CDLL(LIB)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        _lib.emu_pack.argtypes = [vp, vp, u64, vp, vp, u64, vp, u32, u32, vp, u64, vp]
        _lib.emu_pack_any_mode.argtypes = [C.c_int]
        _lib.emu_pack_any_mode.restype = None
    return _lib


def _aligned(nbytes: int, fill: int, mis: int = 0) -> np.ndarray:
    """a buffer of nbytes whose first byte sits `mis` bytes past a 64-byte boundary"""
    raw = np.full(nbytes + 128, fill, dtype=np.uint8)
    k = (-raw.ctypes.data) % 64 + mis
    return raw[k:k + nbytes]


def pack(a, a_off, b=None, b_off=None, sel=None, start=0, a_cap=None, b_cap=None, any_mode=0, canary=0xEE):
    """the records of source A (or B where sel[i] == GOFR_GRPC_DEFER) packed from byte `start` of a 64-byte aligned output
    pre-filled with `canary` → (out, out_off).  Sources get 8 readable bytes behind their last record, as the device
    buffers do."""
    n = len(a_off) - 1
    L = lib()
    src = []
    for buf in (a, b):
        if buf is None:
            src.append(None)
            continue
        s = _aligned(len(buf) + 8, 0)
        s[:len(buf)] = buf
        src.append(s)
    total = sum(int(o[i + 1]) - int(o[i]) for i in range(n) for o in [b_off if b is not None and sel[i] == 6 else a_off])
    out = _aligned(start + total + 64, canary)
    out_off = np.zeros(n + 1, dtype=np.uint32)
    a_off = np.ascontiguousarray(a_off, dtype=np.uint32)
    b_off = None if b_off is None else np.ascontiguousarray(b_off, dtype=np.uint32)
    sel = None if sel is None else np.ascontiguousarray(sel, dtype=np.uint32)
    L.emu_pack_any_mode(any_mode)
    try:
        rc = L.emu_pack(src[0].ctypes.data, a_off.ctypes.data, len(a) if a_cap is None else a_cap,
                        None if b is None else src[1].ctypes.data, None if b_off is None else b_off.ctypes.data,
                        0 if b is None else (len(b) if b_cap is None else b_cap), None if sel is None else sel.ctypes.data,
                        n, start, out.ctypes.data, out.size, out_off.ctypes.data)
    finally:
        L.emu_pack_any_mode(0)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return out, out_off
