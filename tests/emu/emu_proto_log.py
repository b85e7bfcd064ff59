"""TEST INFRASTRUCTURE ONLY: CPU execution of gofr_proto_batch_encode_log's line decision (see emu_proto_log.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gofr_b200 import spec as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libgofr_emu_proto_log.so")
SRCS = [os.path.join(HERE, "emu_proto_log.cpp"), os.path.join(ROOT, "gofr_b200", "csrc", "batch_log_device.cuh"),
        os.path.join(ROOT, "gofr_b200", "csrc", "engine_internal.h"), os.path.join(ROOT, "include", "gofr_b200.h")]
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
        _lib.emu_proto_log.argtypes = [C.c_void_p, C.c_int64, C.c_uint32, C.c_void_p]
        _lib.emu_proto_log.restype = None
    return _lib


def fill(desc: np.ndarray, log_ns: int):
    """proto_log_fill over every record → (the records as the log kernel sees them, has_line[n] bool)"""
    d = np.ascontiguousarray(desc, dtype=S.LOG_DESC_DTYPE).copy()
    has = np.zeros(max(len(d), 1), dtype=np.uint8)
    lib().emu_proto_log(d.ctypes.data, log_ns, len(d), has.ctypes.data)
    return d, has[:len(d)].astype(bool)
