"""TEST INFRASTRUCTURE ONLY: CPU execution of the nested decoder's second pass (see emu_deferred.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gofr_b200 import spec as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libgofr_emu_deferred.so")
CSRC = os.path.join(ROOT, "gofr_b200", "csrc")
_lib = None


def _build():
    srcs = [os.path.join(HERE, "emu_deferred.cpp")] + [os.path.join(CSRC, h) for h in (
        "proto_nested_deferred_device.cuh", "proto_nested_decode_device.cuh", "proto_nested_device.cuh", "grpc_device.cuh",
        "serve_device.cuh", "value_device.cuh", "float_device.cuh", "engine_internal.h", "table_format.h")]
    srcs = [s for s in srcs if os.path.exists(s)]
    if os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                           "-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-static-libubsan",
                           "-o", LIB, os.path.join(HERE, "emu_deferred.cpp")])


def lib():
    global _lib
    if _lib is None:
        _build()
        _lib = C.CDLL(LIB)
        _lib.emu_proto_decode_nested_deferred.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                                          C.c_uint64, C.c_void_p, C.c_void_p]
        _lib.emu_deferred_desc_bytes.restype = C.c_uint32
    return _lib


def _desc(msgs, root):
    """the descriptor the host hands to the kernel (gofr_proto_nested_describe_ex: the product's own validation, host code)"""
    from gofr_b200 import _abi
    nm, nf, n_fields = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    desc = np.zeros(int(lib().emu_deferred_desc_bytes()), dtype=np.uint8)
    _abi.check(_abi.lib().gofr_proto_nested_describe_ex(nm.ctypes.data, len(msgs), nf.ctypes.data, n_fields, root,
                                                        None if pr is None else pr.ctypes.data, desc.ctypes.data, desc.size),
               "gofr_proto_nested_describe_ex")
    return desc


def proto_decode_nested_deferred(msgs, root, frames, in_off, meta_in, rows_cap=None):
    """the second pass on the CPU: the frames whose meta_in status is DEFER decoded again by the walk with the sorted-list
    map step (lists sorted on the CPU by the device code) → (rows pre-filled with 0xEE, row_off, meta)"""
    n = len(in_off) - 1
    desc = _desc(msgs, root)
    cap = rows_cap if rows_cap is not None else int(frames.size) * 10 + 4096 * max(n, 1)
    rows = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    meta_in = np.ascontiguousarray(meta_in, dtype=np.uint32)
    frames = np.concatenate([np.ascontiguousarray(frames), np.zeros(16, np.uint8)])
    rc = lib().emu_proto_decode_nested_deferred(desc.ctypes.data, frames.ctypes.data, in_off.ctypes.data, n, meta_in.ctypes.data,
                                                rows.ctypes.data, cap, off.ctypes.data, meta.ctypes.data)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return rows, off, meta[:n]
