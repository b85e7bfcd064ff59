"""Per-GPU engine: thin wrapper over gofr_engine_* (include/gofr_b200.h).

torch is plumbing only: it owns device buffers and the CUDA stream whose raw handle is passed through the C ABI.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _abi
from . import spec as S
from .table import Table


@dataclass
class DeviceBatch:
    """A request batch resident in HBM (torch uint8 tensors)."""
    desc: "torch.Tensor"
    trace_ids: "torch.Tensor"
    arena: "torch.Tensor"
    n: int
    input_bytes: int


@dataclass
class DeviceResponses:
    out: "torch.Tensor"       # uint8[out_cap]
    out_off: "torch.Tensor"   # int32 view of uint32[n+1]
    meta: "torch.Tensor"      # int32 view of uint32[n]
    n: int

    def to_host(self):
        import torch
        off = self.out_off.cpu().numpy().view(np.uint32)
        meta = self.meta.cpu().numpy().view(np.uint32)
        total = int(off[self.n])
        out = self.out[:total].cpu().numpy()
        return out, off, meta


def nested_bound(msgs, root: int, decode: bool):
    """gofr_proto_nested_bound: (per_byte, per_record) such that no record of b bytes of the message types msgs yields more
    than per_byte * b + per_record bytes: a row when decoding, a frame with its 5-byte prefix when encoding.  The
    derivation is at the C function."""
    nm, nf, k = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    pb, prec = C.c_uint32(), C.c_uint32()
    _abi.check(_abi.lib().gofr_proto_nested_bound(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root,
                                                  None if pr is None else pr.ctypes.data, 1 if decode else 0,
                                                  C.byref(pb), C.byref(prec)), "gofr_proto_nested_bound")
    return pb.value, prec.value


def row_growth_bound(msgs, root: int):
    """(per_byte, per_frame): no frame of b bytes of the message types msgs decodes to a row longer than per_byte * b +
    per_frame (nested_bound when decoding)."""
    return nested_bound(msgs, root, True)


class Engine:
    def __init__(self, table: Table, device: int = 0):
        L = _abi.lib()
        self._e = C.c_void_p()
        self.table = table
        self.device = device
        _abi.check(L.gofr_engine_create(C.byref(self._e), table.handle, device), "gofr_engine_create")

    def close(self):
        if self._e:
            _abi.lib().gofr_engine_destroy(self._e)
            self._e = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- configuration ----
    def set_tile(self, in_bytes_per_req: int):
        _abi.check(_abi.lib().gofr_engine_set_tile(self._e, in_bytes_per_req), "gofr_engine_set_tile")

    def set_chunk(self, n: int):
        _abi.check(_abi.lib().gofr_engine_set_chunk(self._e, n), "gofr_engine_set_chunk")

    def set_timing(self, on: bool):
        _abi.check(_abi.lib().gofr_engine_set_timing(self._e, 1 if on else 0), "gofr_engine_set_timing")

    def slot_ctas(self, force: int = 0) -> int:
        """CTAs/SM of the slot-layout serve kernel in effect (4: wide instance, 5); force=4/5 overrides the engine's choice."""
        v = C.c_int(0)
        _abi.check(_abi.lib().gofr_engine_slot_ctas(self._e, int(force), C.byref(v)), "gofr_engine_slot_ctas")
        return v.value

    def geometry(self):
        g, b, s, m = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        _abi.check(_abi.lib().gofr_engine_geometry(self._e, C.byref(g), C.byref(b), C.byref(s), C.byref(m)),
                   "gofr_engine_geometry")
        return {"grid": g.value, "blocks_per_sm": b.value, "smem_bytes": s.value, "sm_count": m.value}

    def launch_count(self) -> int:
        return int(_abi.lib().gofr_engine_launch_count(self._e))

    def kernel_time_ms(self, reset: bool = False):
        ms, n = C.c_double(), C.c_uint64()
        _abi.check(_abi.lib().gofr_engine_kernel_time_ms(self._e, C.byref(ms), C.byref(n), 1 if reset else 0),
                   "gofr_engine_kernel_time_ms")
        return ms.value, n.value

    def overflowed(self, reset: bool = True) -> bool:
        f = C.c_int()
        _abi.check(_abi.lib().gofr_engine_overflowed(self._e, C.byref(f), 1 if reset else 0), "gofr_engine_overflowed")
        return bool(f.value)

    # ---- device-resident path ----
    def upload(self, batch: S.RequestBatch) -> DeviceBatch:
        import torch
        dev = torch.device("cuda", self.device)
        desc = torch.from_numpy(batch.desc.view(np.uint8).reshape(-1).copy()).to(dev)
        ids = torch.from_numpy(batch.trace_ids.reshape(-1).copy()).to(dev)
        pad = (-batch.arena.size) % 16 + 16
        arena = torch.from_numpy(np.concatenate([batch.arena, np.zeros(pad, dtype=np.uint8)])).to(dev)
        return DeviceBatch(desc, ids, arena, batch.n, batch.input_bytes())

    def alloc_responses(self, n: int, out_cap: int) -> DeviceResponses:
        import torch
        dev = torch.device("cuda", self.device)
        out = torch.empty(out_cap + 64, dtype=torch.uint8, device=dev)
        off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        meta = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        return DeviceResponses(out, off, meta, n)

    def serve_device(self, b: DeviceBatch, date: bytes, resp: DeviceResponses, stream=None) -> None:
        """One fused launch on torch's current stream (or `stream`).  Asynchronous."""
        import torch
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        assert len(date) == 29
        _abi.check(_abi.lib().gofr_serve_device(self._e, b.desc.data_ptr(), b.trace_ids.data_ptr(), b.arena.data_ptr(),
                                                b.n, date, resp.out.data_ptr(), resp.out.numel() - 64,
                                                resp.out_off.data_ptr(), resp.meta.data_ptr(), st.cuda_stream),
                   "gofr_serve_device")

    # ---- routing only: stage 1 of the split API for closures that stay on the host ----
    def route_device(self, b: DeviceBatch, stream=None):
        """gofr_route_device → (meta int32[n] = status | route << 16, vars int32[n, 8] = off | len << 16)."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        meta = torch.zeros(max(b.n, 1), dtype=torch.int32, device=dev)
        vars_ = torch.zeros((max(b.n, 1), 8), dtype=torch.int32, device=dev)
        _abi.check(_abi.lib().gofr_route_device(self._e, b.desc.data_ptr(), b.arena.data_ptr(), b.n, meta.data_ptr(),
                                                vars_.data_ptr(), st.cuda_stream), "gofr_route_device")
        return meta[:b.n], vars_[:b.n]

    def proto_encode_device(self, fields, rows: np.ndarray, row_off: np.ndarray, out_cap: Optional[int] = None, stream=None):
        """gofr_proto_encode_device: rows (spec.pack_proto_rows) → packed gRPC frames.  Returns (out uint8, out_off int32
        view of uint32[n+1], meta int32 view of uint32[n]) on the device."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        n = len(row_off) - 1
        ft = (_abi.ProtoField * max(len(fields), 1))(*[_abi.ProtoField(f.number, f.type) for f in fields])
        d_rows = torch.from_numpy(np.concatenate([np.ascontiguousarray(rows), np.zeros(16, np.uint8)])).to(dev)
        d_off = torch.from_numpy(row_off.view(np.int32)).to(dev)
        cap = out_cap if out_cap is not None else int(rows.size) * 3 + 32 * n * max(len(fields), 1) + 64
        out = torch.empty(cap, dtype=torch.uint8, device=dev)
        off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        meta = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        _abi.check(_abi.lib().gofr_proto_encode_device(self._e, ft, len(fields), d_rows.data_ptr(), d_off.data_ptr(), n,
                                                       out.data_ptr(), cap, off.data_ptr(), meta.data_ptr(), st.cuda_stream),
                   "gofr_proto_encode_device")
        return out, off, meta[:n]

    def proto_encode_nested_device(self, msgs, root: int, rows: np.ndarray, row_off: np.ndarray, out_cap: Optional[int] = None, stream=None):
        """gofr_proto_encode_nested_device: rows (spec.pack_proto_nested_rows) of message types with nested / repeated fields →
        packed gRPC frames.  Returns (out, out_off, meta) on the device."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        n = len(row_off) - 1
        nm, nf, k = S.proto_nested_tables(msgs)
        d_rows = torch.from_numpy(np.concatenate([np.ascontiguousarray(rows), np.zeros(16, np.uint8)])).to(dev)
        d_off = torch.from_numpy(row_off.view(np.int32)).to(dev)
        cap = out_cap if out_cap is not None else int(rows.size) * 4 + 64 * n + 64
        out = torch.empty(cap, dtype=torch.uint8, device=dev)
        off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        meta = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        pr = S.proto_nested_presence(msgs)   # None: no field has explicit presence, and the _ex call is the plain one
        _abi.check(_abi.lib().gofr_proto_encode_nested_ex_device(self._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, root,
                                                                 None if pr is None else pr.ctypes.data, d_rows.data_ptr(), d_off.data_ptr(), n,
                                                                 out.data_ptr(), cap, off.data_ptr(), meta.data_ptr(), st.cuda_stream),
                   "gofr_proto_encode_nested_ex_device")
        return out, off, meta[:n]

    def proto_decode_nested_device(self, msgs, root: int, frames: np.ndarray, in_off: np.ndarray, rows_cap: Optional[int] = None, stream=None):
        """gofr_proto_decode_nested_device: packed gRPC frames of message types with nested / repeated fields → rows.
        Returns (rows uint8, row_off, meta) on the device."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        n = len(in_off) - 1
        nm, nf, k = S.proto_nested_tables(msgs)
        d_in = torch.from_numpy(np.concatenate([np.ascontiguousarray(frames), np.zeros(16, np.uint8)])).to(dev)
        d_off = torch.from_numpy(in_off.view(np.int32)).to(dev)
        cap = rows_cap if rows_cap is not None else int(frames.size) * 10 + 4096 * max(n, 1)
        rows = torch.empty(cap, dtype=torch.uint8, device=dev)
        off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        meta = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        pr = S.proto_nested_presence(msgs)   # None: no field has explicit presence, and the _ex call is the plain one
        _abi.check(_abi.lib().gofr_proto_decode_nested_ex_device(self._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, root,
                                                                 None if pr is None else pr.ctypes.data, d_in.data_ptr(), d_off.data_ptr(), n,
                                                                 rows.data_ptr(), cap, off.data_ptr(), meta.data_ptr(), st.cuda_stream),
                   "gofr_proto_decode_nested_ex_device")
        return rows, off, meta[:n]

    def proto_decode_nested_deferred_device(self, msgs, root: int, frames: np.ndarray, in_off: np.ndarray, meta_in, rows_cap: Optional[int] = None,
                                            stream=None, meta_out=None):
        """gofr_proto_decode_nested_deferred_device: the second pass after proto_decode_nested_device on the same frames.
        meta_in: that call's status column (a contiguous int32 device tensor of n words).  Frames whose status is
        GOFR_GRPC_DEFER are decoded again with map fields of up to 4096 entries; the others get an empty row and keep their
        status.  Returns (rows uint8, row_off, meta) on the device; meta is the merged status column, written to meta_out
        when given (meta_in itself is allowed).  Row i of this call replaces the first call's when meta_in[i] was DEFER and
        meta[i] is OK.  The default capacity covers the longest rows the frames can decode to (row_growth_bound)."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        n = len(in_off) - 1
        nm, nf, k = S.proto_nested_tables(msgs)
        d_in = torch.from_numpy(np.concatenate([np.ascontiguousarray(frames), np.zeros(16, np.uint8)])).to(dev)
        d_off = torch.from_numpy(in_off.view(np.int32)).to(dev)
        if rows_cap is None:
            per_byte, per_frame = row_growth_bound(msgs, root)
            rows_cap = per_byte * int(in_off[-1] - in_off[0]) + per_frame * n
        cap = max(int(rows_cap), 0)
        rows = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        meta = meta_out if meta_out is not None else torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        for t in (meta_in, meta):
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() >= n
        pr = S.proto_nested_presence(msgs)
        _abi.check(_abi.lib().gofr_proto_decode_nested_deferred_device(self._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, root,
                                                                       None if pr is None else pr.ctypes.data, d_in.data_ptr(), d_off.data_ptr(), n,
                                                                       meta_in.data_ptr() if n else None, rows.data_ptr(), cap, off.data_ptr(),
                                                                       meta.data_ptr(), st.cuda_stream),
                   "gofr_proto_decode_nested_deferred_device")
        return rows, off, meta[:n]

    # ---- the nested codec on host buffers (gofr_proto_batch_decode / _encode) ----
    def _proto_batch(self, msgs, root: int, data: np.ndarray, off: np.ndarray, out_cap: Optional[int], pinned: bool, decode: bool):
        n = len(off) - 1
        data = np.ascontiguousarray(data, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.uint32)
        if out_cap is None:
            per_byte, per_record = nested_bound(msgs, root, decode)
            out_cap = per_byte * int(off[-1] - off[0]) + per_record * n if n else 0
        if pinned:
            out, out_off, meta = pinned_array(out_cap), pinned_array(4 * (n + 1), np.uint32), pinned_array(4 * max(n, 1), np.uint32)
        else:
            out, out_off, meta = np.empty(max(out_cap, 1), np.uint8), np.zeros(n + 1, np.uint32), np.zeros(max(n, 1), np.uint32)
        nm, nf, k = S.proto_nested_tables(msgs)
        pr = S.proto_nested_presence(msgs)
        L = _abi.lib()
        pb = _abi.ProtoBatch(data=data.ctypes.data, data_bytes=data.size, off=off.ctypes.data, n=n)
        ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out_cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data, out_bytes=0)
        t = C.c_uint64()
        fn = L.gofr_proto_batch_decode if decode else L.gofr_proto_batch_encode
        name = "gofr_proto_batch_decode" if decode else "gofr_proto_batch_encode"
        _abi.check(fn(self._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None if pr is None else pr.ctypes.data,
                      C.byref(pb), C.byref(ob), C.byref(t)), name)
        _abi.check(L.gofr_batch_wait(self._e, t.value), "gofr_batch_wait")
        return out[:int(ob.out_bytes)], out_off, meta[:n]

    def proto_decode_batch(self, msgs, root: int, frames: np.ndarray, in_off: np.ndarray, out_cap: Optional[int] = None,
                           pinned: bool = False):
        """gofr_proto_batch_decode: frames in host memory → (rows uint8, row_off uint32[n + 1], meta uint32[n]), both decode
        passes combined; a frame still GOFR_GRPC_DEFER, or failed, has an empty row.  out_cap defaults to the bound; pinned
        puts the outputs in pinned memory (device-driven egress)."""
        return self._proto_batch(msgs, root, frames, in_off, out_cap, pinned, True)

    def proto_encode_batch(self, msgs, root: int, rows: np.ndarray, row_off: np.ndarray, out_cap: Optional[int] = None,
                           pinned: bool = False):
        """gofr_proto_batch_encode: rows (spec.pack_proto_nested_rows) in host memory → (frames uint8, out_off uint32[n + 1],
        meta uint32[n]), what gofr_proto_encode_nested_ex_device gives."""
        return self._proto_batch(msgs, root, rows, row_off, out_cap, pinned, False)

    def proto_decode_device(self, fields, frames: np.ndarray, in_off: np.ndarray, rows_cap: Optional[int] = None, stream=None):
        """gofr_proto_decode_device: packed gRPC frames → rows.  Returns (rows uint8, row_off, meta) on the device."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        n = len(in_off) - 1
        ft = (_abi.ProtoField * max(len(fields), 1))(*[_abi.ProtoField(f.number, f.type) for f in fields])
        d_in = torch.from_numpy(np.concatenate([np.ascontiguousarray(frames), np.zeros(16, np.uint8)])).to(dev)
        d_off = torch.from_numpy(in_off.view(np.int32)).to(dev)
        cap = rows_cap if rows_cap is not None else int(frames.size) + (8 * len(fields) + 8) * n + 64
        rows = torch.empty(cap, dtype=torch.uint8, device=dev)
        off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        meta = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        _abi.check(_abi.lib().gofr_proto_decode_device(self._e, ft, len(fields), d_in.data_ptr(), d_off.data_ptr(), n,
                                                       rows.data_ptr(), cap, off.data_ptr(), meta.data_ptr(), st.cuda_stream),
                   "gofr_proto_decode_device")
        return rows, off, meta[:n]

    def route_host(self, batch: S.RequestBatch):
        """gofr_batch_route: the same for a batch in host memory → (meta uint32[n], vars uint32[n, 8])."""
        rb = _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data, arena=batch.arena.ctypes.data,
                           arena_bytes=batch.arena.size, n=batch.n, date=b"")
        meta = np.zeros(max(batch.n, 1), dtype=np.uint32)
        vars_ = np.zeros((max(batch.n, 1), 8), dtype=np.uint32)
        _abi.check(_abi.lib().gofr_batch_route(self._e, C.byref(rb), meta.ctypes.data, vars_.ctypes.data), "gofr_batch_route")
        return meta[:batch.n], vars_[:batch.n]

    # ---- HTTP/1.1 request heads → request descriptors (the step in front of the router) ----
    def http_parse_device(self, raw: np.ndarray, raw_off: np.ndarray, stream=None):
        """gofr_http_parse_device on host arrays (uploaded here).  Returns torch tensors (desc uint8[n*16], arena uint8,
        status int32[n], spans int64[n, 6]) — desc/arena can be fed to the serve calls as they are."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        n = len(raw_off) - 1
        d_raw = torch.from_numpy(np.concatenate([raw, np.zeros(32, dtype=np.uint8)])).to(dev)
        d_off = torch.from_numpy(raw_off.astype(np.uint32).view(np.int32)).to(dev)
        return self.http_parse_resident(d_raw, d_off, n, stream)

    def http_frame_device(self, buf: np.ndarray, buf_off: np.ndarray, rec_cap: Optional[int] = None, stream=None):
        """gofr_http_frame_device on host arrays (uploaded here): connection c's received bytes are
        buf[buf_off[c]:buf_off[c+1]].  Returns torch tensors (d_buf uint8 with its slack, rec_off int32[rec_cap+1],
        first int32[n+1], consumed int32[n], status int32[n]); first[n] is the record count, and (d_buf, rec_off, first[n])
        goes to http_parse_resident as it is.  rec_cap defaults to what always suffices: the shortest request of the subset is
        longer than 16 bytes, and a connection has at most one tail record."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        n = len(buf_off) - 1
        if rec_cap is None:
            rec_cap = int(buf.size) // 16 + n + 1
        d_buf = torch.from_numpy(np.concatenate([buf, np.zeros(32, dtype=np.uint8)])).to(dev)
        d_off = torch.from_numpy(np.ascontiguousarray(buf_off, dtype=np.uint32).view(np.int32)).to(dev)
        rec_off = torch.zeros(rec_cap + 1, dtype=torch.int32, device=dev)
        first = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        consumed = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        status = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        _abi.check(_abi.lib().gofr_http_frame_device(self._e, d_buf.data_ptr(), d_off.data_ptr(), n, rec_off.data_ptr(), rec_cap,
                                                     first.data_ptr(), consumed.data_ptr(), status.data_ptr(), st.cuda_stream),
                   "gofr_http_frame_device")
        return d_buf, rec_off, first, consumed[:n], status[:n]

    def http_parse_resident(self, d_raw, d_raw_off, n: int, stream=None):
        """gofr_http_parse_device on tensors already in HBM (d_raw with 16 bytes of slack, d_raw_off int32[n+1]): returns
        (desc uint8[n*16], arena uint8, status int32[n], spans int64[n, 6])."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        desc = torch.zeros(max(n, 1) * 16, dtype=torch.uint8, device=dev)
        arena = torch.zeros(int(d_raw.numel()) + 16, dtype=torch.uint8, device=dev)
        status = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        spans = torch.zeros((max(n, 1), 6), dtype=torch.int64, device=dev)
        _abi.check(_abi.lib().gofr_http_parse_device(self._e, d_raw.data_ptr(), d_raw_off.data_ptr(), n, desc.data_ptr(),
                                                     arena.data_ptr(), status.data_ptr(), spans.data_ptr(), st.cuda_stream),
                   "gofr_http_parse_device")
        return desc[:n * 16], arena, status[:n], spans[:n]

    # ---- RequestLog lines (middleware.Logging → logger.Log), device resident ----
    def request_log_device(self, batch: S.LogBatch, out_cap: Optional[int] = None, stream=None):
        """Uploads a LogBatch, runs gofr_requestlog_device, returns (out, out_off) torch tensors (uint8, int32 view)."""
        import torch
        dev = torch.device("cuda", self.device)
        n = batch.n
        d_desc = torch.from_numpy(batch.desc.view(np.uint8).reshape(-1).copy()).to(dev)
        d_ids = torch.from_numpy(batch.trace_ids.reshape(-1).copy()).to(dev)
        d_arena = torch.from_numpy(np.concatenate([batch.arena, np.zeros(48, dtype=np.uint8)])).to(dev)
        if out_cap is None:
            out_cap = 400 * n + 6 * int(batch.arena.size) + 64
        d_out = torch.empty(out_cap + 64, dtype=torch.uint8, device=dev)
        d_off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        self.request_log_resident(d_desc, d_ids, d_arena, n, d_out, out_cap, d_off, stream)
        return d_out, d_off

    def request_log_resident(self, d_desc, d_ids, d_arena, n: int, d_out, out_cap: int, d_off, stream=None) -> None:
        import torch
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        _abi.check(_abi.lib().gofr_requestlog_device(self._e, d_desc.data_ptr(), d_ids.data_ptr(), d_arena.data_ptr(), n,
                                                     d_out.data_ptr(), out_cap, d_off.data_ptr(), st.cuda_stream),
                   "gofr_requestlog_device")

    def serve_device_slots(self, b: DeviceBatch, date: bytes, slot_bytes: int, out=None, out_len=None, meta=None, stream=None):
        """gofr_serve_device_slots: response i at out[i * slot_bytes:], its length in out_len[i].  Returns
        (out uint8[n * slot_bytes], out_len int32[n], meta int32[n]); pass the buffers to reuse / pre-fill them."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        if out is None:
            out = torch.empty(max(b.n, 1) * slot_bytes, dtype=torch.uint8, device=dev)
        if out_len is None:
            out_len = torch.zeros(max(b.n, 1), dtype=torch.int32, device=dev)
        if meta is None:
            meta = torch.zeros(max(b.n, 1), dtype=torch.int32, device=dev)
        assert len(date) == 29
        _abi.check(_abi.lib().gofr_serve_device_slots(self._e, b.desc.data_ptr(), b.trace_ids.data_ptr(), b.arena.data_ptr(),
                                                      b.n, date, out.data_ptr(), slot_bytes, out_len.data_ptr(),
                                                      meta.data_ptr(), st.cuda_stream), "gofr_serve_device_slots")
        return out, out_len[:b.n], meta[:b.n]

    def bind_device(self, b: DeviceBatch, schema_id: int, slot_bytes: int, stream=None, rows=None):
        """gofr_bind_device: Context.Bind for host closures.  Returns (rows uint8[n * slot_bytes], len int32[n], status int32[n]);
        pass rows to pre-fill them."""
        import torch
        dev = torch.device("cuda", self.device)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        if rows is None:
            rows = torch.zeros(max(b.n, 1) * slot_bytes, dtype=torch.uint8, device=dev)
        ln = torch.zeros(max(b.n, 1), dtype=torch.int32, device=dev)
        status = torch.zeros(max(b.n, 1), dtype=torch.int32, device=dev)
        _abi.check(_abi.lib().gofr_bind_device(self._e, schema_id, b.desc.data_ptr(), b.arena.data_ptr(), b.n, rows.data_ptr(),
                                               slot_bytes, ln.data_ptr(), status.data_ptr(), st.cuda_stream), "gofr_bind_device")
        return rows, ln[:b.n], status[:b.n]

    # ---- host path (the call a user makes): host buffers in, host buffers out ----
    def serve_host(self, batch: S.RequestBatch, date: bytes, out: np.ndarray, out_off: np.ndarray, meta: np.ndarray) -> int:
        L = _abi.lib()
        rb = _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data,
                           arena=batch.arena.ctypes.data, arena_bytes=batch.arena.size, n=batch.n, date=date)
        ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out.size, out_off=out_off.ctypes.data, meta=meta.ctypes.data,
                            out_bytes=0)
        t = C.c_uint64()
        _abi.check(L.gofr_batch_submit(self._e, C.byref(rb), C.byref(ob), C.byref(t)), "gofr_batch_submit")
        _abi.check(L.gofr_batch_wait(self._e, t.value), "gofr_batch_wait")
        return int(ob.out_bytes)


@dataclass
class ConnResponses:
    """What gofr_conn_batch_submit returns for a batch of connection buffers (numpy arrays, sliced to what was written).
    Connection c's bytes to write are out[out_off[req_first[c]]:out_off[req_first[c + 1]]]."""
    out: np.ndarray          # uint8[out_bytes]
    out_off: np.ndarray      # uint32[requests + 1]
    meta: np.ndarray         # uint32[requests]
    req_at: np.ndarray       # uint32[requests]: the request's first byte in buf
    trace_ids: np.ndarray    # uint8[requests, 16]
    req_first: np.ndarray    # uint32[n_conns + 1]
    consumed: np.ndarray     # uint32[n_conns]
    conn_status: np.ndarray  # uint32[n_conns]: GOFR_HTTP_CONN_DONE / MORE / DEFER
    log: Optional["ConnLogLines"] = None  # the request-log lines, when serve_connections was given a ConnLog


@dataclass
class ConnLog:
    """The inputs of gofr_conn_batch_submit_log besides the connections' bytes: connection c's req.RemoteAddr is
    remote[remote_off[c]:remote_off[c + 1]] (at most 255 bytes) and its requests' start clock start_unix_ns[c]; every line
    is logged at log_unix_ns in a zone tz_offset_s east of UTC.  The capacities default to conn_log_bound."""
    remote: np.ndarray         # uint8
    remote_off: np.ndarray     # uint32[n_conns + 1]
    start_unix_ns: np.ndarray  # int64[n_conns]
    log_unix_ns: int
    tz_offset_s: int = 0
    line_cap: Optional[int] = None
    out_cap: Optional[int] = None


@dataclass
class ConnLogLines:
    """middleware.Logging's lines for the requests answered on the device, in request order: line m is
    out[log_off[m]:log_off[m + 1]] and belongs to batch request log_req[m].  lines / out_bytes: what the batch needed."""
    out: np.ndarray          # uint8[out_bytes]
    log_off: np.ndarray      # uint32[lines + 1]
    log_req: np.ndarray      # uint32[lines]
    lines: int
    out_bytes: int


def conn_batch_bound(table: Table, buf_off: np.ndarray):
    """gofr_conn_batch_bound: (req_cap, out_cap) that always suffice for connection buffers with these offsets."""
    off = np.ascontiguousarray(buf_off, dtype=np.uint32)
    rc, oc = C.c_uint32(), C.c_uint64()
    _abi.check(_abi.lib().gofr_conn_batch_bound(table.handle, off.ctypes.data, len(off) - 1, C.byref(rc), C.byref(oc)),
               "gofr_conn_batch_bound")
    return rc.value, oc.value


def conn_log_bound(buf_off: np.ndarray, remote_off: np.ndarray):
    """gofr_conn_log_bound: (line_cap, out_cap) that always suffice for the request-log lines of these connections."""
    off = np.ascontiguousarray(buf_off, dtype=np.uint32)
    roff = np.ascontiguousarray(remote_off, dtype=np.uint32)
    lc, oc = C.c_uint32(), C.c_uint64()
    _abi.check(_abi.lib().gofr_conn_log_bound(off.ctypes.data, roff.ctypes.data, len(off) - 1, C.byref(lc), C.byref(oc)),
               "gofr_conn_log_bound")
    return lc.value, oc.value


@dataclass
class ConnRoute:
    """What gofr_conn_batch_route returns (numpy arrays, sliced to the batch's requests): per request k its route decision
    (meta[k], vars[k]: as route_host gives them; status 0 = the closure of route meta[k] >> 16 runs), its first byte in buf,
    its trace id and its parsed form, desc[k] into arena; per connection req_first / consumed / conn_status.  .batch is the
    requests as a RequestBatch (desc, trace_ids, arena): what gofr_batch_bind takes and what Param / PathParam read."""
    desc: np.ndarray         # DESC_DTYPE[requests]
    arena: np.ndarray        # uint8[buf_bytes + 64]
    meta: np.ndarray         # uint32[requests]
    vars: np.ndarray         # uint32[requests, 8]: off | len << 16 inside the request's path, 0xFFFFFFFF unused
    req_at: np.ndarray       # uint32[requests]
    trace_ids: np.ndarray    # uint8[requests, 16]
    req_first: np.ndarray    # uint32[n_conns + 1]
    consumed: np.ndarray     # uint32[n_conns]
    conn_status: np.ndarray  # uint32[n_conns]

    @property
    def batch(self) -> S.RequestBatch:
        return S.RequestBatch(self.desc, self.trace_ids, self.arena)


def _alloc(pinned: bool):
    if pinned:
        return lambda count, dt: pinned_array(max(count, 1) * np.dtype(dt).itemsize).view(dt)
    return lambda count, dt: np.zeros(max(count, 1), dt)


def _route_connections(self, buf: np.ndarray, buf_off: np.ndarray, trace_seed: int, pinned: bool = True,
                       req_cap: Optional[int] = None) -> ConnRoute:
    """gofr_conn_batch_route: stage 1 of serving connection buffers with handler closures (frame, parse and route on the
    device).  Run the closures of the requests whose status is 0, then hand their GOFR_H_RESULT records to
    serve_connections(..., results=(rec, rec_off)) with the same buf, buf_off and trace_seed.  req_cap defaults to
    conn_batch_bound's; pinned puts the outputs in pinned memory, else in pageable numpy arrays."""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    off = np.ascontiguousarray(buf_off, dtype=np.uint32)
    n = len(off) - 1
    if req_cap is None:
        req_cap, _ = conn_batch_bound(self.table, off)
    alloc = _alloc(pinned)
    desc, arena = alloc(req_cap, S.DESC_DTYPE), alloc(buf.size + 64, np.uint8)
    meta, vars_, req_at = alloc(req_cap, np.uint32), alloc(req_cap * 8, np.uint32), alloc(req_cap, np.uint32)
    ids = alloc(req_cap * 16, np.uint8)
    req_first, consumed, status = alloc(n + 1, np.uint32), alloc(n, np.uint32), alloc(n, np.uint32)
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=b"", trace_seed=trace_seed)
    cr = _abi.ConnRoute(req_cap=req_cap, desc=desc.ctypes.data, arena=arena.ctypes.data, meta=meta.ctypes.data,
                        vars=vars_.ctypes.data, req_at=req_at.ctypes.data, trace_ids=ids.ctypes.data,
                        req_first=req_first.ctypes.data, consumed=consumed.ctypes.data, conn_status=status.ctypes.data)
    _abi.check(_abi.lib().gofr_conn_batch_route(self._e, C.byref(cb), C.byref(cr)), "gofr_conn_batch_route")
    k = int(req_first[n]) if n else 0
    return ConnRoute(desc[:k], arena[:buf.size + 64], meta[:k], vars_[:k * 8].reshape(k, 8), req_at[:k], ids[:k * 16].reshape(k, 16),
                     req_first[:n + 1] if n else np.zeros(1, np.uint32), consumed[:n], status[:n])


Engine.route_connections = _route_connections


def conn_respond_bound(table: Table, desc: np.ndarray, rec_off: np.ndarray) -> int:
    """gofr_conn_respond_bound: an out_cap that always suffices for serve_connections(..., results=(rec, rec_off)) on the
    requests stage 1 described (desc: ConnRoute.desc)."""
    d = np.ascontiguousarray(desc).view(S.DESC_DTYPE)
    ro = np.ascontiguousarray(rec_off, dtype=np.uint32)
    assert len(ro) == len(d) + 1
    oc = C.c_uint64()
    _abi.check(_abi.lib().gofr_conn_respond_bound(table.handle, d.ctypes.data, len(d), ro.ctypes.data, C.byref(oc)),
               "gofr_conn_respond_bound")
    return oc.value


def _serve_connections(self, buf: np.ndarray, buf_off: np.ndarray, date: bytes, trace_seed: int, pinned: bool = True,
                       req_cap: Optional[int] = None, out_cap: Optional[int] = None, log: Optional[ConnLog] = None,
                       results=None, trace_key: Optional[np.ndarray] = None):
    """gofr_conn_batch_submit + wait: connection c's received bytes are buf[buf_off[c]:buf_off[c + 1]] (host memory).
    Returns ConnResponses.  The capacities default to conn_batch_bound; pinned puts the outputs in pinned memory (egress
    driven by the device), else in pageable numpy arrays.  With log (a ConnLog), gofr_conn_batch_submit_log: the result's
    .log holds the request-log lines, in the same kind of memory.  With results = (rec uint8, rec_off uint32[requests + 1]),
    gofr_conn_batch_respond: stage 2 after route_connections on the same buffers and seed, request k's data section is its
    closure's record rec[rec_off[k]:rec_off[k + 1]] where that is not empty; out_cap then defaults to the larger of
    conn_batch_bound's and what the records need (conn_respond_bound over the requests the table's bound assumes).  With
    trace_key (uint64[n_conns]), gofr_conn_batch_respond_ex: connection c's ids come from trace_key[c], not (trace_seed, c)."""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    off = np.ascontiguousarray(buf_off, dtype=np.uint32)
    n = len(off) - 1
    rres = None
    if results is not None:
        rec = np.ascontiguousarray(results[0], dtype=np.uint8)
        roff = np.ascontiguousarray(results[1], dtype=np.uint32)
        rres = _abi.ConnResults(rec=rec.ctypes.data if rec.size else None, rec_off=roff.ctypes.data, rec_bytes=rec.size,
                                n_req=len(roff) - 1)
    if req_cap is None or out_cap is None:
        rc, oc = conn_batch_bound(self.table, off)
        if results is not None:   # every request's data section may be a record: per byte of a record, the table's bound
            rb = lambda dl: _abi.lib().gofr_table_response_bound(self.table.handle, 0, 0, dl)
            oc += (rb(1) - rb(0)) * rec.size
        req_cap = rc if req_cap is None else req_cap
        out_cap = oc if out_cap is None else out_cap
    alloc = _alloc(pinned)
    out, out_off, meta = alloc(out_cap, np.uint8), alloc(req_cap + 1, np.uint32), alloc(req_cap, np.uint32)
    req_at, ids = alloc(req_cap, np.uint32), alloc(req_cap * 16, np.uint8)
    req_first, consumed, status = alloc(n + 1, np.uint32), alloc(n, np.uint32), alloc(n, np.uint32)
    assert len(date) == 29
    cb = _abi.ConnBatch(buf=buf.ctypes.data, buf_off=off.ctypes.data, buf_bytes=buf.size, n_conns=n, date=date, trace_seed=trace_seed)
    cr = _abi.ConnResp(out=out.ctypes.data, out_cap=out_cap, req_cap=req_cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data,
                       req_at=req_at.ctypes.data, trace_ids=ids.ctypes.data, req_first=req_first.ctypes.data,
                       consumed=consumed.ctypes.data, conn_status=status.ctypes.data, out_bytes=0)
    L = _abi.lib()
    t = C.c_uint64()
    keys = None if trace_key is None else np.ascontiguousarray(trace_key, dtype=np.uint64)
    assert keys is None or len(keys) == n
    if keys is not None and log is None:
        _abi.check(L.gofr_conn_batch_respond_ex(self._e, C.byref(cb), keys.ctypes.data, None if rres is None else C.byref(rres),
                                                C.byref(cr), None, C.byref(t)), "gofr_conn_batch_respond_ex")
    elif results is not None and log is None:
        _abi.check(L.gofr_conn_batch_respond(self._e, C.byref(cb), C.byref(rres), C.byref(cr), None, C.byref(t)),
                   "gofr_conn_batch_respond")
    elif log is None:
        _abi.check(L.gofr_conn_batch_submit(self._e, C.byref(cb), C.byref(cr), C.byref(t)), "gofr_conn_batch_submit")
    else:
        remote = np.ascontiguousarray(log.remote, dtype=np.uint8)
        roff = np.ascontiguousarray(log.remote_off, dtype=np.uint32)
        start = np.ascontiguousarray(log.start_unix_ns, dtype=np.int64)
        assert len(roff) == n + 1 and len(start) == n
        line_cap, lout_cap = log.line_cap, log.out_cap
        if line_cap is None or lout_cap is None:
            lc, oc = conn_log_bound(off, roff)
            line_cap = lc if line_cap is None else line_cap
            lout_cap = oc if lout_cap is None else lout_cap
        lout, log_off, log_req = alloc(lout_cap, np.uint8), alloc(line_cap + 1, np.uint32), alloc(line_cap, np.uint32)
        cl = _abi.ConnLog(remote=remote.ctypes.data, remote_off=roff.ctypes.data, start_unix_ns=start.ctypes.data,
                          log_unix_ns=log.log_unix_ns, tz_offset_s=log.tz_offset_s, line_cap=line_cap, out=lout.ctypes.data,
                          out_cap=lout_cap, log_off=log_off.ctypes.data, log_req=log_req.ctypes.data)
        if keys is not None:
            _abi.check(L.gofr_conn_batch_respond_ex(self._e, C.byref(cb), keys.ctypes.data, None if rres is None else C.byref(rres),
                                                    C.byref(cr), C.byref(cl), C.byref(t)), "gofr_conn_batch_respond_ex")
        elif results is not None:
            _abi.check(L.gofr_conn_batch_respond(self._e, C.byref(cb), C.byref(rres), C.byref(cr), C.byref(cl), C.byref(t)),
                       "gofr_conn_batch_respond")
        else:
            _abi.check(L.gofr_conn_batch_submit_log(self._e, C.byref(cb), C.byref(cr), C.byref(cl), C.byref(t)),
                       "gofr_conn_batch_submit_log")
    _abi.check(L.gofr_batch_wait(self._e, t.value), "gofr_batch_wait")
    k = int(req_first[n]) if n else 0
    lines = None
    if log is not None:
        m = cl.lines
        lines = ConnLogLines(lout[:int(cl.out_bytes)], log_off[:m + 1] if n else np.zeros(1, np.uint32), log_req[:m], m,
                             int(cl.out_bytes))
    return ConnResponses(out[:int(cr.out_bytes)], out_off[:k + 1], meta[:k], req_at[:k], ids[:k * 16].reshape(k, 16),
                         req_first[:n + 1] if n else np.zeros(1, np.uint32), consumed[:n], status[:n], lines)


Engine.serve_connections = _serve_connections


def _serve_host_slots(self, batch: S.RequestBatch, date: bytes, slot_bytes: int, out: np.ndarray, out_len: np.ndarray,
                      meta: np.ndarray) -> None:
    """gofr_batch_submit_slots + wait: host buffers in, response i in out[i * slot_bytes:], its length in out_len[i]."""
    L = _abi.lib()
    rb = _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data, arena=batch.arena.ctypes.data,
                       arena_bytes=batch.arena.size, n=batch.n, date=date)
    sb = _abi.SlotBatch(out=out.ctypes.data, slot_bytes=slot_bytes, reserved=0, out_len=out_len.ctypes.data, meta=meta.ctypes.data)
    t = C.c_uint64()
    _abi.check(L.gofr_batch_submit_slots(self._e, C.byref(rb), C.byref(sb), C.byref(t)), "gofr_batch_submit_slots")
    _abi.check(L.gofr_batch_wait(self._e, t.value), "gofr_batch_wait")


Engine.serve_host_slots = _serve_host_slots


def batch_log_bound(log: S.LogBatch) -> int:
    """gofr_batch_log_bound: line bytes that always suffice for gofr_batch_submit_log on these records."""
    cap = C.c_uint64()
    _abi.check(_abi.lib().gofr_batch_log_bound(log.desc.ctypes.data, log.n, C.byref(cap)), "gofr_batch_log_bound")
    return int(cap.value)


@dataclass
class BatchLogResult:
    """What gofr_batch_submit_log / _slots_log return: the responses (packed: out[out_off[i]:out_off[i + 1]]; slots:
    out[i * slot_bytes:][:out_len[i]]), meta, and request i's line lines_out[log_off[i]:log_off[i + 1]] (empty when it has
    none).  lines / log_bytes: what the batch needed; rc: gofr_batch_wait's code (GOFR_ERR_CAPACITY = 7 when short)."""
    out: np.ndarray
    out_off: Optional[np.ndarray]   # packed layout
    out_len: Optional[np.ndarray]   # slot layout
    meta: np.ndarray
    lines_out: np.ndarray
    log_off: np.ndarray
    lines: int
    log_bytes: int
    out_bytes: int
    rc: int

    def responses(self, slot_bytes: int = 0):
        if self.out_off is not None:
            b = self.out.tobytes()
            return [b[int(self.out_off[i]):int(self.out_off[i + 1])] for i in range(len(self.meta))]
        return [self.out[i * slot_bytes:i * slot_bytes + int(self.out_len[i])].tobytes() for i in range(len(self.meta))]

    def line_list(self):
        b = self.lines_out.tobytes()
        return [b[int(self.log_off[i]):int(self.log_off[i + 1])] for i in range(len(self.log_off) - 1)]


def _serve_host_log(self, batch: S.RequestBatch, date: bytes, log: S.LogBatch, log_unix_ns: int, slot_bytes: int = 0,
                    pinned: bool = True, out_cap: Optional[int] = None, log_out_cap: Optional[int] = None,
                    raise_on_capacity: bool = True) -> BatchLogResult:
    """gofr_batch_submit_log (slot_bytes 0: packed layout) or gofr_batch_submit_slots_log + wait on a RequestBatch with
    one LogBatch record per request (kind LOG_REQUEST or LOG_NONE; status and the clock fields are the call's).  The log
    batch's trace ids are not used: a line's id is its request's.  Buffers are pinned (device-driven egress) or pageable."""
    L = _abi.lib()
    n = batch.n
    assert log.n == n
    alloc = _alloc(pinned)
    if out_cap is None:
        out_cap = sum(int(L.gofr_table_response_bound(self.table.handle, int(d["path_len"]), int(d["query_len"]),
                                                      int(d["data_len"]))) for d in batch.desc)
    if log_out_cap is None:
        log_out_cap = batch_log_bound(log)
    meta = alloc(n, np.uint32)
    lout = alloc(log_out_cap + 16, np.uint8)
    lout[log_out_cap:] = 0xAB   # 16 bytes past the capacity that the call must leave alone
    log_off = alloc(n + 1, np.uint32)
    rb = _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data, arena=batch.arena.ctypes.data,
                       arena_bytes=batch.arena.size, n=n, date=date)
    lb = _abi.BatchLog(desc=log.desc.ctypes.data, arena=log.arena.ctypes.data if log.arena.size else None,
                       arena_bytes=log.arena.size, log_unix_ns=log_unix_ns, out=lout.ctypes.data, out_cap=log_out_cap,
                       log_off=log_off.ctypes.data, lines=0, reserved=0, out_bytes=0)
    t = C.c_uint64()
    out_off = out_len = None
    if slot_bytes:
        out = alloc(n * slot_bytes, np.uint8)
        out_len = alloc(n, np.uint32)
        sb = _abi.SlotBatch(out=out.ctypes.data, slot_bytes=slot_bytes, reserved=0, out_len=out_len.ctypes.data,
                            meta=meta.ctypes.data)
        _abi.check(L.gofr_batch_submit_slots_log(self._e, C.byref(rb), C.byref(sb), C.byref(lb), C.byref(t)),
                   "gofr_batch_submit_slots_log")
    else:
        out = alloc(out_cap + 16, np.uint8)
        out_off = alloc(n + 1, np.uint32)
        ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out_cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data,
                            out_bytes=0)
        _abi.check(L.gofr_batch_submit_log(self._e, C.byref(rb), C.byref(ob), C.byref(lb), C.byref(t)), "gofr_batch_submit_log")
    rc = int(L.gofr_batch_wait(self._e, t.value))
    if rc and (raise_on_capacity or rc != 7):
        _abi.check(rc, "gofr_batch_wait")
    return BatchLogResult(out, out_off, out_len[:n] if slot_bytes else None, meta[:n], lout, log_off, int(lb.lines),
                          int(lb.out_bytes), 0 if slot_bytes else int(ob.out_bytes), rc)


Engine.serve_host_log = _serve_host_log


def _proto_encode_batch_log(self, msgs, root: int, rows: np.ndarray, row_off: np.ndarray, log: S.LogBatch, log_unix_ns: int,
                            pinned: bool = True, log_pinned: Optional[bool] = None, out_cap: Optional[int] = None,
                            log_out_cap: Optional[int] = None, raise_on_capacity: bool = True) -> BatchLogResult:
    """gofr_proto_batch_encode_log + wait: rows in host memory → the frames gofr_proto_batch_encode gives, and for every
    LogBatch record of kind LOG_RPC the gRPC LoggingInterceptor's RPCLog line (LOG_NONE: an empty line).  The log batch's
    trace ids are the lines' ids; its start, elapsed time, zone and method are the caller's, log_unix_ns the batch's.  The
    frames and lines go to pinned (device-driven egress) or pageable buffers, each its own (log_pinned defaults to pinned)."""
    L = _abi.lib()
    n = len(row_off) - 1
    assert log.n == n
    rows = np.ascontiguousarray(rows, dtype=np.uint8)
    row_off = np.ascontiguousarray(row_off, dtype=np.uint32)
    if out_cap is None:
        per_byte, per_record = nested_bound(msgs, root, False)
        out_cap = per_byte * int(row_off[-1] - row_off[0]) + per_record * n if n else 0
    if log_out_cap is None:
        log_out_cap = batch_log_bound(log)
    alloc, lalloc = _alloc(pinned), _alloc(pinned if log_pinned is None else log_pinned)
    out, out_off, meta = alloc(out_cap + 16, np.uint8), alloc(n + 1, np.uint32), alloc(n, np.uint32)
    out[out_cap:] = 0xAB        # 16 bytes past each capacity that the call must leave alone
    lout, log_off = lalloc(log_out_cap + 16, np.uint8), lalloc(n + 1, np.uint32)
    lout[log_out_cap:] = 0xAB
    nm, nf, k = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    pb = _abi.ProtoBatch(data=rows.ctypes.data, data_bytes=rows.size, off=row_off.ctypes.data, n=n)
    ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out_cap, out_off=out_off.ctypes.data, meta=meta.ctypes.data, out_bytes=0)
    lb = _abi.BatchLog(desc=log.desc.ctypes.data, arena=log.arena.ctypes.data if log.arena.size else None,
                       arena_bytes=log.arena.size, log_unix_ns=log_unix_ns, out=lout.ctypes.data, out_cap=log_out_cap,
                       log_off=log_off.ctypes.data, lines=0, reserved=0, out_bytes=0)
    t = C.c_uint64()
    _abi.check(L.gofr_proto_batch_encode_log(self._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, root,
                                             None if pr is None else pr.ctypes.data, C.byref(pb), log.trace_ids.ctypes.data,
                                             C.byref(ob), C.byref(lb), C.byref(t)), "gofr_proto_batch_encode_log")
    rc = int(L.gofr_batch_wait(self._e, t.value))
    if rc and (raise_on_capacity or rc != 7):
        _abi.check(rc, "gofr_batch_wait")
    return BatchLogResult(out, out_off, None, meta[:n], lout, log_off, int(lb.lines), int(lb.out_bytes), int(ob.out_bytes), rc)


Engine.proto_encode_batch_log = _proto_encode_batch_log


def pinned_array(nbytes: int, dtype=np.uint8) -> np.ndarray:
    """numpy view over cudaMallocHost memory (gofr_alloc_pinned).  The memory lives until process exit."""
    L = _abi.lib()
    p = L.gofr_alloc_pinned(max(nbytes, 1))
    if not p:
        raise MemoryError(L.gofr_last_error().decode())
    buf = (C.c_uint8 * max(nbytes, 1)).from_address(p)
    a = np.frombuffer(buf, dtype=np.uint8)[:nbytes]
    return a.view(dtype)


def pin_batch(batch: S.RequestBatch) -> S.RequestBatch:
    d = pinned_array(batch.desc.nbytes).view(S.DESC_DTYPE)
    d[:] = batch.desc
    i = pinned_array(batch.trace_ids.nbytes).reshape(-1, 16)
    i[:] = batch.trace_ids
    a = pinned_array(batch.arena.nbytes)
    a[:] = batch.arena
    return S.RequestBatch(d, i, a)
