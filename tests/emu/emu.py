"""TEST INFRASTRUCTURE ONLY: CPU execution of the kernel's per-request device code (see emu_serve.cpp)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from gofr_b200 import spec as S

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libgofr_emu.so")
_lib = None


def _build():
    srcs = [os.path.join(HERE, "emu_serve.cpp"), os.path.join(ROOT, "gofr_b200", "csrc", "serve_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "bind_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "value_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "float_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "grpc_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "proto_nested_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "proto_nested_decode_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "engine_internal.h"),
            os.path.join(ROOT, "gofr_b200", "csrc", "reqlog_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "http_device.cuh"),
            os.path.join(ROOT, "gofr_b200", "csrc", "table_format.h")]
    srcs = [s for s in srcs if os.path.exists(s)]
    if os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                           "-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-static-libubsan",
                           "-o", LIB, os.path.join(HERE, "emu_serve.cpp")])


def _padded(arena: np.ndarray) -> np.ndarray:
    """the arena as the ABI promises it to the device code (include/gofr_b200.h: the allocation extends 16 bytes past the last
    request byte — copies read whole words) and not one byte more: under ASan this checks the promise is enough"""
    return np.concatenate([arena, np.zeros(16, dtype=np.uint8)])


def lib():
    global _lib
    if _lib is None:
        alt = os.environ.get("GOFR_EMU_LIB")   # a differently instrumented build of the same source (scratch/fuzz_long.py --asan)
        if not alt:
            _build()
        _lib = C.CDLL(alt or LIB)
        _lib.emu_serve.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p,
                                   C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32]
        _lib.emu_grpc_hello.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                        C.c_void_p, C.c_uint32]
        _lib.emu_proto_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64,
                                          C.c_void_p, C.c_void_p, C.c_uint32]
        _lib.emu_proto_decode.argtypes = _lib.emu_proto_encode.argtypes
        _lib.emu_serve_slots.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p,
                                         C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib.emu_route.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib.emu_http_parse.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.emu_reqlog.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p,
                                    C.c_uint32]
    return _lib


def float_text(bits: int) -> bytes:
    """json_float64_text of the device code (float_device.cuh): b"" for NaN / Inf."""
    out = C.create_string_buffer(40)
    lib().emu_float_text.argtypes = [C.c_uint64, C.c_char_p]
    n = lib().emu_float_text(bits, out)
    return out.raw[:n]


def float32_text(bits: int) -> bytes:
    """json_float32_text of the device code: the text encoding/json writes for a float32 member; b"" for NaN / Inf."""
    out = C.create_string_buffer(40)
    lib().emu_float32_text.argtypes = [C.c_uint32, C.c_char_p]
    n = lib().emu_float32_text(bits, out)
    return out.raw[:n]


def float32_check(first: int, step: int, count: int):
    """float32 bit patterns first, first + step, ... against the C library (round trip, shortest, nearest): (failures, first bad)"""
    lib().emu_float32_check.restype = C.c_uint64
    lib().emu_float32_check.argtypes = [C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint32)]
    bad = C.c_uint32(0)
    return int(lib().emu_float32_check(first, step, count, C.byref(bad))), int(bad.value)


def float_text_many(bits: np.ndarray):
    """the texts of many float64 bit patterns: (bytes, offsets[n + 1])"""
    bits = np.ascontiguousarray(bits, dtype=np.uint64)
    out = np.zeros(len(bits) * 32, dtype=np.uint8)
    off = np.zeros(len(bits) + 1, dtype=np.uint32)
    lib().emu_float_text_many.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib().emu_float_text_many(bits.ctypes.data, len(bits), out.ctypes.data, off.ctypes.data)
    return out, off


def fast_taken(reset: bool = True) -> int:
    """Requests the slot-layout emulation sized with size_fast (hence wrote with emit_fast) since the last reset."""
    lib().emu_fast_taken.restype = C.c_uint64
    return int(lib().emu_fast_taken(1 if reset else 0))


def set_stage_mode(mode: int):
    """Slot emulation: which requests count as staged in shared memory (0: every other one, 1: all, 2: none)."""
    lib().emu_set_stage_mode(mode)


def set_pair_stores(on: bool):
    """Slot emulation: write fast-path responses with the PairStores store policy of the wide instance (True) or with
    SoloStores (False, the default)."""
    lib().emu_set_pair_stores(1 if on else 0)


def set_flush_mode(mode: int):
    """0: flush decisions per request; 1: flush at every decision point; 2: pseudo-random extra flushes (on the GPU the
    other lanes of a warp impose theirs)."""
    lib().emu_set_flush_mode(mode)


def serve_slots(image: bytes, batch, date: bytes, slot_bytes: int):
    """Slot layout on the CPU: (out uint8[n, slot_bytes] pre-filled with 0xEE, out_len, meta)."""
    n = batch.n
    img = np.frombuffer(image, dtype=np.uint8).copy()
    base = np.full(n * slot_bytes + 64, 0xEE, dtype=np.uint8)
    shift = (-base.ctypes.data) % 16          # slots are 16-byte aligned, like cudaMalloc'ed memory
    out = base[shift:shift + n * slot_bytes]
    ln = np.zeros(n, dtype=np.uint32)
    meta = np.zeros(n, dtype=np.uint32)
    arena = _padded(batch.arena)
    lib().emu_serve_slots(img.ctypes.data, len(image), batch.desc.ctypes.data, batch.trace_ids.ctypes.data, arena.ctypes.data,
                          n, date, out.ctypes.data, slot_bytes, ln.ctypes.data, meta.ctypes.data)
    return out.reshape(n, slot_bytes), ln, meta


def bind_rows(image: bytes, schema_idx: int, batch, slot_bytes: int):
    """gofr_bind_device on the CPU: (out uint8[n, slot_bytes] pre-filled with 0xEE, len, status)."""
    n = batch.n
    img = np.frombuffer(image, dtype=np.uint8).copy()
    base = np.full(n * slot_bytes + 64, 0xEE, dtype=np.uint8)
    shift = (-base.ctypes.data) % 16
    out = base[shift:shift + n * slot_bytes]
    ln = np.zeros(n, dtype=np.uint32)
    st = np.zeros(n, dtype=np.uint32)
    arena = _padded(batch.arena)
    lib().emu_bind_rows.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib().emu_bind_rows(img.ctypes.data, schema_idx, batch.desc.ctypes.data, arena.ctypes.data, n, out.ctypes.data, slot_bytes,
                        ln.ctypes.data, st.ctypes.data)
    return out.reshape(n, slot_bytes), ln, st


def route(image: bytes, batch):
    n = batch.n
    img = np.frombuffer(image, dtype=np.uint8).copy()
    meta = np.zeros(n, dtype=np.uint32)
    vars_ = np.zeros((n, 8), dtype=np.uint32)
    arena = _padded(batch.arena)
    lib().emu_route(img.ctypes.data, batch.desc.ctypes.data, arena.ctypes.data, n, meta.ctypes.data,
                    vars_.ctypes.data)
    return meta, vars_


def http_parse(raw: np.ndarray, raw_off: np.ndarray):
    n = len(raw_off) - 1
    desc = np.zeros(n * 16, dtype=np.uint8)
    arena = np.zeros(int(raw.size) + 32, dtype=np.uint8)
    status = np.zeros(n, dtype=np.uint32)
    spans = np.zeros((n, 6), dtype=np.uint64)
    rawp = np.concatenate([raw, np.zeros(16, dtype=np.uint8)])
    lib().emu_http_parse(rawp.ctypes.data, raw_off.ctypes.data, n, desc.ctypes.data, arena.ctypes.data, status.ctypes.data,
                         spans.ctypes.data)
    return desc, arena, status, spans


def request_log(batch, misalign: int = 0):
    """batch: gofr_b200.spec.LogBatch.  Returns (out, out_off)."""
    n = batch.n
    cap = 400 * n + 6 * int(batch.arena.size) + 64
    out = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    arena = _padded(batch.arena)
    rc = lib().emu_reqlog(batch.desc.ctypes.data, batch.trace_ids.ctypes.data, arena.ctypes.data, n, out.ctypes.data,
                          cap, off.ctypes.data, misalign)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return out, off


def proto_encode(fields, rows, row_off, misalign: int = 0):
    """proto_size + proto_emit (grpc_device.cuh) on the CPU → (out, out_off, meta)"""
    n = len(row_off) - 1
    ft = np.array([[f.number, f.type] for f in fields], dtype=np.uint32).reshape(-1)
    cap = int(rows.size) * 3 + 32 * n * max(len(fields), 1) + 64 + misalign
    out = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    rows = np.ascontiguousarray(rows)
    rc = lib().emu_proto_encode(ft.ctypes.data, len(fields), rows.ctypes.data, row_off.ctypes.data, n, out.ctypes.data, cap,
                                off.ctypes.data, meta.ctypes.data, misalign)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return out, off, meta[:n]


def _pbn_desc(msgs, root, presence_instance):
    """the descriptor the host hands to the nested kernels, from the product's own validation (gofr_proto_nested_describe_ex
    with the description's presence bytes: host code, no GPU).  Its presence byte (byte 1) and maps half-word pick the
    instance the emulation runs, as they pick the kernels on the host.  presence_instance: that byte set whatever the
    description, so that the presence instance runs a presence-free description too."""
    from gofr_b200 import _abi
    nm, nf, n_fields = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    lib().emu_pbn_desc_bytes.restype = C.c_uint32
    desc = np.zeros(int(lib().emu_pbn_desc_bytes()), dtype=np.uint8)
    _abi.check(_abi.lib().gofr_proto_nested_describe_ex(nm.ctypes.data, len(msgs), nf.ctypes.data, n_fields, root,
                                                        None if pr is None else pr.ctypes.data, desc.ctypes.data, desc.size),
               "gofr_proto_nested_describe_ex")
    if presence_instance:
        desc[1] = 1
    return desc


def proto_encode_nested(msgs, root, rows, row_off, misalign: int = 0, presence_instance: bool = False):
    """pbn_size + pbn_emit (proto_nested_device.cuh) on the CPU → (out, out_off, meta)"""
    n = len(row_off) - 1
    desc = _pbn_desc(msgs, root, presence_instance)
    cap = int(rows.size) * 4 + 64 * n + 64 + misalign
    out = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    rows = np.concatenate([np.ascontiguousarray(rows), np.zeros(16, np.uint8)])
    lib().emu_proto_encode_nested.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32]
    rc = lib().emu_proto_encode_nested(desc.ctypes.data, rows.ctypes.data, row_off.ctypes.data, n, out.ctypes.data, cap, off.ctypes.data,
                                       meta.ctypes.data, misalign)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return out, off, meta[:n]


def proto_decode_nested(msgs, root, frames, in_off, presence_instance: bool = False):
    """pdn_decode_size + pdn_decode_emit (proto_nested_decode_device.cuh) on the CPU → (rows, row_off, meta)"""
    n = len(in_off) - 1
    desc = _pbn_desc(msgs, root, presence_instance)
    cap = int(frames.size) * 10 + 4096 * max(n, 1)
    rows = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    frames = np.concatenate([np.ascontiguousarray(frames), np.zeros(16, np.uint8)])
    lib().emu_proto_decode_nested.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    rc = lib().emu_proto_decode_nested(desc.ctypes.data, frames.ctypes.data, in_off.ctypes.data, n, rows.ctypes.data, cap, off.ctypes.data,
                                       meta.ctypes.data)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return rows, off, meta[:n]


def proto_decode(fields, frames, in_off, misalign: int = 0):
    """proto_decode_scan + proto_decode_emit (grpc_device.cuh) on the CPU → (rows, row_off, meta)"""
    n = len(in_off) - 1
    ft = np.array([[f.number, f.type] for f in fields], dtype=np.uint32).reshape(-1)
    cap = int(frames.size) + (8 * len(fields) + 8) * n + 64 + misalign
    rows = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    frames = np.concatenate([np.ascontiguousarray(frames), np.zeros(16, np.uint8)])
    rc = lib().emu_proto_decode(ft.ctypes.data, len(fields), frames.ctypes.data, in_off.ctypes.data, n, rows.ctypes.data, cap,
                                off.ctypes.data, meta.ctypes.data, misalign)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return rows, off, meta[:n]


def grpc_hello(frames, in_off, misalign: int = 0):
    n = len(in_off) - 1
    cap = int(frames.size) + 40 * n + 64
    out = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(n, dtype=np.uint32)
    rc = lib().emu_grpc_hello(frames.ctypes.data, in_off.ctypes.data, n, out.ctypes.data, cap, off.ctypes.data,
                              meta.ctypes.data, misalign)
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return out, off, meta


def serve(image: bytes, batch, date: bytes, out_cap: int | None = None, misalign: int = 0):
    n = batch.n
    if out_cap is None:
        out_cap = max(4096, n * 700 + int(batch.arena.size) * 6) + 64 + len(image) * max(1, n // 8)
    img = np.frombuffer(image, dtype=np.uint8).copy()
    out = np.full(out_cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(n, dtype=np.uint32)
    arena = _padded(batch.arena)
    rc = lib().emu_serve(img.ctypes.data, len(image), batch.desc.ctypes.data, batch.trace_ids.ctypes.data,
                         arena.ctypes.data, n, date, out.ctypes.data, out_cap, off.ctypes.data, meta.ctypes.data,
                         misalign)
    if rc == -2:
        raise AssertionError("hashed and linear route matchers disagree")
    if rc == -3:
        raise AssertionError("a response wrote bytes outside its own range")
    if rc != 0:
        raise RuntimeError("emu output capacity too small")
    return out, off, meta
