"""ctypes binding of the C ABI in include/gofr_b200.h (libgofr_b200.so).

The signatures carry plain pointers and sizes only; torch (or numpy) merely owns the memory behind them.
"""
from __future__ import annotations

import ctypes as C
import os

from . import _build

_lib = None


class FieldDesc(C.Structure):
    _fields_ = [("go_name", C.c_char_p), ("json_name", C.c_char_p), ("kind", C.c_uint8), ("omitempty", C.c_uint8),
                ("container", C.c_uint8), ("flags", C.c_uint8), ("elem_schema", C.c_uint16), ("reserved", C.c_uint8 * 2)]


class HandlerDesc(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("schema_id", C.c_uint32),
                ("s0", C.c_char_p), ("s0_len", C.c_uint32),
                ("s1", C.c_char_p), ("s1_len", C.c_uint32),
                ("s2", C.c_char_p), ("s2_len", C.c_uint32),
                ("s3", C.c_char_p), ("s3_len", C.c_uint32),
                ("blob", C.c_char_p), ("blob_len", C.c_uint32)]


class ReqBatch(C.Structure):
    _fields_ = [("desc", C.c_void_p), ("trace_ids", C.c_void_p), ("arena", C.c_void_p), ("arena_bytes", C.c_uint64),
                ("n", C.c_uint32), ("date", C.c_char * 29), ("pad", C.c_uint8 * 3)]


class SlotBatch(C.Structure):
    _fields_ = [("out", C.c_void_p), ("slot_bytes", C.c_uint32), ("reserved", C.c_uint32), ("out_len", C.c_void_p),
                ("meta", C.c_void_p)]


class RespBatch(C.Structure):
    _fields_ = [("out", C.c_void_p), ("out_cap", C.c_uint64), ("out_off", C.c_void_p), ("meta", C.c_void_p),
                ("out_bytes", C.c_uint64)]


ERR_NAMES = {0: "OK", 1: "INVALID", 2: "UNSUPPORTED", 3: "NOMEM", 4: "CUDA", 5: "SEALED", 6: "NOT_SEALED", 7: "CAPACITY",
             8: "NO_DEVICE"}


class ConnBatch(C.Structure):
    _fields_ = [("buf", C.c_void_p), ("buf_off", C.c_void_p), ("buf_bytes", C.c_uint64), ("n_conns", C.c_uint32),
                ("date", C.c_char * 29), ("pad", C.c_uint8 * 3), ("trace_seed", C.c_uint64)]


class ConnResp(C.Structure):
    _fields_ = [("out", C.c_void_p), ("out_cap", C.c_uint64), ("req_cap", C.c_uint32), ("reserved", C.c_uint32),
                ("out_off", C.c_void_p), ("meta", C.c_void_p), ("req_at", C.c_void_p), ("trace_ids", C.c_void_p),
                ("req_first", C.c_void_p), ("consumed", C.c_void_p), ("conn_status", C.c_void_p), ("out_bytes", C.c_uint64)]


class ConnLog(C.Structure):
    _fields_ = [("remote", C.c_void_p), ("remote_off", C.c_void_p), ("start_unix_ns", C.c_void_p), ("log_unix_ns", C.c_int64),
                ("tz_offset_s", C.c_int32), ("line_cap", C.c_uint32), ("out", C.c_void_p), ("out_cap", C.c_uint64),
                ("log_off", C.c_void_p), ("log_req", C.c_void_p), ("lines", C.c_uint32), ("reserved", C.c_uint32),
                ("out_bytes", C.c_uint64)]


class BatchLog(C.Structure):
    _fields_ = [("desc", C.c_void_p), ("arena", C.c_void_p), ("arena_bytes", C.c_uint64), ("log_unix_ns", C.c_int64),
                ("out", C.c_void_p), ("out_cap", C.c_uint64), ("log_off", C.c_void_p), ("lines", C.c_uint32),
                ("reserved", C.c_uint32), ("out_bytes", C.c_uint64)]


class ConnRoute(C.Structure):
    _fields_ = [("req_cap", C.c_uint32), ("reserved", C.c_uint32), ("desc", C.c_void_p), ("arena", C.c_void_p),
                ("meta", C.c_void_p), ("vars", C.c_void_p), ("req_at", C.c_void_p), ("trace_ids", C.c_void_p),
                ("req_first", C.c_void_p), ("consumed", C.c_void_p), ("conn_status", C.c_void_p)]


class ConnResults(C.Structure):
    _fields_ = [("rec", C.c_void_p), ("rec_off", C.c_void_p), ("rec_bytes", C.c_uint64), ("n_req", C.c_uint32),
                ("reserved", C.c_uint32)]


class ConnAppBind(C.Structure):
    _fields_ = [("status", C.c_void_p), ("row_off", C.c_void_p), ("rows", C.c_void_p), ("rows_cap", C.c_uint64),
                ("rows_bytes", C.c_uint64)]


class ConnAppStats(C.Structure):
    _fields_ = [("route_batches", C.c_uint64), ("route_reads", C.c_uint64), ("respond_batches", C.c_uint64),
                ("respond_reads", C.c_uint64), ("reruns", C.c_uint64), ("isolated", C.c_uint64), ("gather_ns", C.c_uint64)]


class ProtoBatch(C.Structure):
    _fields_ = [("data", C.c_void_p), ("data_bytes", C.c_uint64), ("off", C.c_void_p), ("n", C.c_uint32)]


class ProtoField(C.Structure):
    _fields_ = [("number", C.c_uint32), ("type", C.c_uint32)]


class GofrError(RuntimeError):
    def __init__(self, code: int, where: str):
        self.code = code
        msg = lib().gofr_last_error().decode("utf-8", "replace")
        super().__init__(f"{where}: GOFR_ERR_{ERR_NAMES.get(code, code)}: {msg}")


def check(code: int, where: str) -> None:
    if code != 0:
        raise GofrError(code, where)


def lib_path() -> str:
    return _build.LIB


def lib():
    """Loads (building first if stale) the CUDA library.  There is no fallback: if it cannot be built or loaded the
    import of anything that serves requests fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    # GOFR_LIB_PATH: load a prebuilt variant of the library instead (A/B measurements of two builds in one GPU session)
    path = os.environ.get("GOFR_LIB_PATH") or _build.build()
    L = C.CDLL(path)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.gofr_table_create.argtypes = [C.POINTER(vp), u32]
    L.gofr_table_destroy.argtypes = [vp]
    L.gofr_table_destroy.restype = None
    L.gofr_table_add_schema.argtypes = [vp, u32, C.c_char_p, C.POINTER(FieldDesc), u32]
    L.gofr_table_add_route.argtypes = [vp, u32, C.c_char_p, u32, C.POINTER(HandlerDesc), C.POINTER(u32)]
    L.gofr_table_add_default_routes.argtypes = [vp, C.c_char_p, u32]
    L.gofr_table_seal.argtypes = [vp]
    L.gofr_table_serialize.argtypes = [vp, vp, C.POINTER(u64)]
    L.gofr_table_deserialize.argtypes = [C.POINTER(vp), vp, u64]
    L.gofr_table_route_count.argtypes = [vp]
    L.gofr_table_route_count.restype = u32
    L.gofr_table_max_response_bytes.argtypes = [vp, u32]
    L.gofr_table_max_response_bytes.restype = u32
    L.gofr_engine_create.argtypes = [C.POINTER(vp), vp, i32]
    L.gofr_engine_destroy.argtypes = [vp]
    L.gofr_engine_destroy.restype = None
    L.gofr_serve_device.argtypes = [vp, vp, vp, vp, u32, C.c_char_p, vp, u64, vp, vp, vp]
    L.gofr_serve_device_slots.argtypes = [vp, vp, vp, vp, u32, C.c_char_p, vp, u32, vp, vp, vp]
    L.gofr_batch_submit.argtypes = [vp, C.POINTER(ReqBatch), C.POINTER(RespBatch), C.POINTER(u64)]
    L.gofr_batch_wait.argtypes = [vp, u64]
    L.gofr_batch_submit_slots.argtypes = [vp, C.POINTER(ReqBatch), C.POINTER(SlotBatch), C.POINTER(u64)]
    L.gofr_engine_set_chunk.argtypes = [vp, u32]
    L.gofr_engine_set_tile.argtypes = [vp, u32]
    L.gofr_engine_set_timing.argtypes = [vp, i32]
    L.gofr_engine_overflowed.argtypes = [vp, C.POINTER(i32), i32]
    L.gofr_proto_nested_describe.argtypes = [vp, u32, vp, u32, u32, vp, u32]
    L.gofr_proto_decode_nested_device.argtypes = [vp, vp, u32, vp, u32, u32, vp, vp, u32, vp, u64, vp, vp, vp]
    L.gofr_proto_encode_nested_device.argtypes = [vp, vp, u32, vp, u32, u32, vp, vp, u32, vp, u64, vp, vp, vp]
    L.gofr_proto_nested_describe_ex.argtypes = [vp, u32, vp, u32, u32, vp, vp, u32]
    L.gofr_proto_decode_nested_ex_device.argtypes = [vp, vp, u32, vp, u32, u32, vp, vp, vp, u32, vp, u64, vp, vp, vp]
    L.gofr_proto_encode_nested_ex_device.argtypes = [vp, vp, u32, vp, u32, u32, vp, vp, vp, u32, vp, u64, vp, vp, vp]
    L.gofr_proto_decode_nested_deferred_device.argtypes = [vp, vp, u32, vp, u32, u32, vp, vp, vp, u32, vp, vp, u64, vp, vp, vp]
    L.gofr_proto_batch_decode.argtypes = [vp, vp, u32, vp, u32, u32, vp, C.POINTER(ProtoBatch), C.POINTER(RespBatch), C.POINTER(u64)]
    L.gofr_proto_batch_encode.argtypes = [vp, vp, u32, vp, u32, u32, vp, C.POINTER(ProtoBatch), C.POINTER(RespBatch), C.POINTER(u64)]
    L.gofr_proto_nested_bound.argtypes = [vp, u32, vp, u32, u32, vp, i32, C.POINTER(u32), C.POINTER(u32)]
    L.gofr_table_slot_ctas.argtypes = [vp, C.POINTER(C.c_int)]
    L.gofr_engine_slot_ctas.argtypes = [vp, C.c_int, C.POINTER(C.c_int)]
    L.gofr_engine_geometry.argtypes = [vp, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)]
    L.gofr_bind_device.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, vp, C.c_uint32, vp, vp, vp]
    L.gofr_bind_device.restype = C.c_int
    L.gofr_bind_host_thread.argtypes = [C.c_int, C.POINTER(C.c_int)]
    L.gofr_bind_host_thread.restype = C.c_int
    L.gofr_alloc_pinned.argtypes = [C.c_size_t]
    L.gofr_alloc_pinned.restype = vp
    L.gofr_free_pinned.argtypes = [vp]
    L.gofr_free_pinned.restype = None
    L.gofr_grpc_hello_device.argtypes = [vp, vp, vp, u32, vp, u64, vp, vp, vp]
    L.gofr_route_device.argtypes = [vp, vp, vp, u32, vp, vp, vp]
    L.gofr_table_response_bound.argtypes = [vp, u32, u32, u32]
    L.gofr_table_response_bound.restype = u32
    L.gofr_proto_encode_device.argtypes = [vp, vp, u32, vp, vp, u32, vp, u64, vp, vp, vp]
    L.gofr_proto_decode_device.argtypes = [vp, vp, u32, vp, vp, u32, vp, u64, vp, vp, vp]
    L.gofr_batch_route.argtypes = [vp, C.POINTER(ReqBatch), vp, vp]
    L.gofr_batch_bind.argtypes = [vp, u32, C.POINTER(ReqBatch), vp, u32, vp, vp]
    L.gofr_frontend_create.argtypes = [C.POINTER(vp), vp, u32, u32, u32, u32]
    L.gofr_frontend_destroy.argtypes = [vp]
    L.gofr_frontend_destroy.restype = None
    L.gofr_frontend_set_clock.argtypes = [vp, C.c_int64]
    L.gofr_frontend_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    L.gofr_frontend_serve.argtypes = [vp, C.c_uint8, C.c_char_p, C.c_uint16, C.c_char_p, C.c_uint16, C.c_uint8, C.c_char_p, u32,
                                      C.c_char_p, C.c_char_p, u32, C.POINTER(u32), C.POINTER(u32)]
    L.gofr_proto_frontend_create.argtypes = [C.POINTER(vp), vp, vp, u32, vp, u32, u32, vp, i32, u32, u32, u32]
    L.gofr_proto_frontend_destroy.argtypes = [vp]
    L.gofr_proto_frontend_destroy.restype = None
    L.gofr_proto_frontend_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    L.gofr_proto_frontend_call.argtypes = [vp, C.c_char_p, u32, vp, u32, C.POINTER(u32), C.POINTER(u32)]
    L.gofr_proto_frontend_create_log.argtypes = [C.POINTER(vp), vp, vp, u32, vp, u32, u32, vp, i32, u32, u32, u32, u32]
    L.gofr_proto_frontend_set_log_clock.argtypes = [vp, C.c_int64]
    L.gofr_proto_frontend_call_log.argtypes = [vp, C.c_char_p, u32, C.c_char_p, vp, C.c_char_p, vp, u32, C.POINTER(u32),
                                               C.POINTER(u32), vp, u32, C.POINTER(u32)]
    L.gofr_conn_frontend_create.argtypes = [C.POINTER(vp), vp, u32, u32, u32, i32, C.c_int32, u64]
    L.gofr_conn_frontend_destroy.argtypes = [vp]
    L.gofr_conn_frontend_destroy.restype = None
    L.gofr_conn_frontend_set_clock.argtypes = [vp, C.c_int64]
    L.gofr_conn_frontend_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.gofr_conn_frontend_serve.argtypes = [vp, C.c_char_p, u32, C.c_char_p, u32, C.c_int64, C.POINTER(ConnResp), C.POINTER(ConnLog)]
    L.gofr_http_parse_device.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.gofr_http_frame_device.argtypes = [vp, vp, vp, u32, vp, u32, vp, vp, vp, vp]
    L.gofr_conn_batch_submit.argtypes = [vp, C.POINTER(ConnBatch), C.POINTER(ConnResp), C.POINTER(u64)]
    L.gofr_conn_batch_bound.argtypes = [vp, vp, u32, C.POINTER(u32), C.POINTER(u64)]
    L.gofr_conn_batch_submit_log.argtypes = [vp, C.POINTER(ConnBatch), C.POINTER(ConnResp), C.POINTER(ConnLog), C.POINTER(u64)]
    L.gofr_conn_log_bound.argtypes = [vp, vp, u32, C.POINTER(u32), C.POINTER(u64)]
    L.gofr_conn_batch_route.argtypes = [vp, C.POINTER(ConnBatch), C.POINTER(ConnRoute)]
    L.gofr_conn_batch_respond.argtypes = [vp, C.POINTER(ConnBatch), C.POINTER(ConnResults), C.POINTER(ConnResp), C.POINTER(ConnLog),
                                          C.POINTER(u64)]
    L.gofr_conn_respond_bound.argtypes = [vp, vp, u32, vp, C.POINTER(u64)]
    L.gofr_conn_batch_respond_ex.argtypes = [vp, C.POINTER(ConnBatch), vp, C.POINTER(ConnResults), C.POINTER(ConnResp),
                                             C.POINTER(ConnLog), C.POINTER(u64)]
    L.gofr_conn_app_frontend_create.argtypes = [C.POINTER(vp), vp, u32, u32, u32, i32, C.c_int32, u64, vp, u32, vp]
    L.gofr_conn_app_frontend_destroy.argtypes = [vp]
    L.gofr_conn_app_frontend_destroy.restype = None
    L.gofr_conn_app_frontend_set_clock.argtypes = [vp, C.c_int64]
    L.gofr_conn_app_frontend_stats.argtypes = [vp, C.POINTER(ConnAppStats)]
    L.gofr_conn_app_frontend_route.argtypes = [vp, C.c_char_p, u32, C.POINTER(ConnRoute), C.POINTER(ConnAppBind), C.POINTER(u64)]
    L.gofr_conn_app_frontend_respond.argtypes = [vp, C.c_char_p, u32, u64, C.POINTER(ConnResults), C.c_char_p, u32, C.c_int64,
                                                 C.POINTER(ConnResp), C.POINTER(ConnLog)]
    L.gofr_requestlog_device.argtypes = [vp, vp, vp, vp, u32, vp, u64, vp, vp]
    L.gofr_batch_submit_log.argtypes = [vp, C.POINTER(ReqBatch), C.POINTER(RespBatch), C.POINTER(BatchLog), C.POINTER(u64)]
    L.gofr_batch_submit_slots_log.argtypes = [vp, C.POINTER(ReqBatch), C.POINTER(SlotBatch), C.POINTER(BatchLog), C.POINTER(u64)]
    L.gofr_batch_log_bound.argtypes = [vp, u32, C.POINTER(u64)]
    L.gofr_proto_batch_encode_log.argtypes = [vp, vp, u32, vp, u32, u32, vp, C.POINTER(ProtoBatch), vp, C.POINTER(RespBatch),
                                              C.POINTER(BatchLog), C.POINTER(u64)]
    L.gofr_frontend_create_log.argtypes = [C.POINTER(vp), vp, u32, u32, u32, u32, u32]
    L.gofr_frontend_set_log_clock.argtypes = [vp, C.c_int64]
    L.gofr_frontend_serve_log.argtypes = [vp, C.c_uint8, C.c_char_p, C.c_uint16, C.c_char_p, C.c_uint16, C.c_uint8, C.c_char_p,
                                          u32, C.c_char_p, vp, C.c_char_p, C.c_char_p, u32, C.POINTER(u32), C.POINTER(u32),
                                          C.c_char_p, u32, C.POINTER(u32)]
    L.gofr_engine_launch_count.argtypes = [vp]
    L.gofr_engine_launch_count.restype = u64
    L.gofr_engine_kernel_time_ms.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(u64), i32]
    L.gofr_last_error.restype = C.c_char_p
    L.gofr_abi_version.restype = u32
    L.gofr_format_http_date.argtypes = [C.c_int64, C.c_char_p]
    L.gofr_format_http_date.restype = None
    _lib = L
    return L


# every symbol include/gofr_b200.h declares (tests check the library exports them all)
DECLARED_SYMBOLS = [
    "gofr_table_create", "gofr_table_destroy", "gofr_table_add_schema", "gofr_table_add_route",
    "gofr_table_add_default_routes", "gofr_table_seal", "gofr_table_serialize", "gofr_table_deserialize",
    "gofr_table_route_count", "gofr_table_max_response_bytes", "gofr_engine_create", "gofr_engine_destroy",
    "gofr_serve_device", "gofr_serve_device_slots", "gofr_batch_submit", "gofr_batch_wait", "gofr_batch_submit_slots", "gofr_engine_set_chunk", "gofr_engine_set_tile",
    "gofr_engine_set_timing", "gofr_engine_overflowed", "gofr_engine_geometry", "gofr_engine_slot_ctas", "gofr_table_slot_ctas", "gofr_alloc_pinned", "gofr_free_pinned", "gofr_bind_host_thread", "gofr_bind_device", "gofr_batch_bind",
    "gofr_grpc_hello_device", "gofr_requestlog_device", "gofr_batch_submit_log", "gofr_batch_submit_slots_log", "gofr_batch_log_bound", "gofr_http_parse_device", "gofr_http_frame_device", "gofr_conn_batch_submit", "gofr_conn_batch_bound", "gofr_conn_batch_submit_log", "gofr_conn_log_bound", "gofr_conn_batch_route", "gofr_conn_batch_respond", "gofr_conn_respond_bound", "gofr_conn_batch_respond_ex", "gofr_batch_route", "gofr_proto_encode_device", "gofr_proto_decode_device", "gofr_proto_encode_nested_device", "gofr_proto_decode_nested_device", "gofr_proto_nested_describe", "gofr_proto_encode_nested_ex_device", "gofr_proto_decode_nested_ex_device", "gofr_proto_nested_describe_ex", "gofr_proto_decode_nested_deferred_device", "gofr_proto_batch_decode", "gofr_proto_batch_encode", "gofr_proto_batch_encode_log", "gofr_proto_nested_bound", "gofr_table_response_bound", "gofr_frontend_create", "gofr_frontend_destroy", "gofr_frontend_set_clock",
    "gofr_frontend_stats", "gofr_frontend_serve", "gofr_frontend_create_log", "gofr_frontend_set_log_clock", "gofr_frontend_serve_log", "gofr_proto_frontend_create", "gofr_proto_frontend_destroy",
    "gofr_proto_frontend_stats", "gofr_proto_frontend_call", "gofr_proto_frontend_create_log", "gofr_proto_frontend_set_log_clock",
    "gofr_proto_frontend_call_log", "gofr_conn_frontend_create", "gofr_conn_frontend_destroy",
    "gofr_conn_frontend_set_clock", "gofr_conn_frontend_stats", "gofr_conn_frontend_serve",
    "gofr_conn_app_frontend_create", "gofr_conn_app_frontend_destroy", "gofr_conn_app_frontend_set_clock",
    "gofr_conn_app_frontend_stats", "gofr_conn_app_frontend_route", "gofr_conn_app_frontend_respond",
    "gofr_route_device", "gofr_engine_launch_count", "gofr_engine_kernel_time_ms", "gofr_last_error",
    "gofr_abi_version", "gofr_format_http_date",
]
