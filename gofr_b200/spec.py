"""Plain-data description of a route table and of request batches (host side).

The numeric constants are the ones in include/gofr_b200.h.  A `TableSpec` is what `gofr.New()` + `app.GET(...)` calls
accumulate before `app.Run()` (pkg/gofr/gofr.go:152-177, :102-107); a `RequestBatch` is the SoA staging layout the
C ABI consumes (desc[n], trace_id[n][16], arena).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

# methods
M_GET, M_HEAD, M_POST, M_PUT, M_PATCH, M_DELETE, M_CONNECT, M_OPTIONS, M_TRACE = range(9)
M_OTHER = 15
M_ANY = 255
METHOD_BY_NAME = {"GET": M_GET, "HEAD": M_HEAD, "POST": M_POST, "PUT": M_PUT, "PATCH": M_PATCH, "DELETE": M_DELETE,
                  "CONNECT": M_CONNECT, "OPTIONS": M_OPTIONS, "TRACE": M_TRACE}

# frame modes
FRAME_WIRE, FRAME_INTENDED, FRAME_BODY = 0, 1, 2

# handler kinds
(H_HOST, H_STATIC_STRING, H_STATIC_ERROR, H_NIL, H_PARAM_FORMAT, H_ROW, H_BIND_ECHO, H_HEALTH, H_MISSING_FILE, H_FILE,
 H_PANIC, H_PATHPARAM_FORMAT, H_RESULT) = range(13)
(RESULT_DATA, RESULT_ERROR, RESULT_NIL, RESULT_MISSING, RESULT_BOTH, RESULT_STRING, RESULT_RAW_DATA, RESULT_RAW_STRING,
 RESULT_RAW_NIL) = range(9)
RAW_OK, RAW_ERR, RAW_MISSING = 0, 1, 2   # bits 8..15 of a RAW outcome word: which status the (ignored) error picks


def result_record(outcome: int, payload: bytes = b"", raw_err: int = RAW_OK) -> bytes:
    """Data section of a GOFR_H_RESULT request: outcome word, then a schema row (DATA / RAW_DATA) or len + bytes (ERROR / MISSING:
    err.Error(); STRING / RAW_STRING: the string the handler returned).  raw_err: for the RAW outcomes, the error the closure
    returned next to the response.Raw value (it only selects the status code)."""
    if outcome in (RESULT_ERROR, RESULT_MISSING, RESULT_STRING, RESULT_RAW_STRING):
        payload = len(payload).to_bytes(4, "little") + payload
    return (outcome | raw_err << 8).to_bytes(4, "little") + payload


def result_both(schema: "Schema", values: Sequence, message: bytes, lookup=None) -> bytes:
    """RESULT_BOTH record: (data, err) both non-nil — message length word + the row's fixed words, then the message
    bytes + the row's string bytes."""
    row = schema.encode_row(values, lookup)
    fixed = schema.fixed_bytes(lookup)
    return (RESULT_BOTH.to_bytes(4, "little") + len(message).to_bytes(4, "little") + row[:fixed] + message + row[fixed:])

# field kinds
F_INT64, F_INT32, F_BOOL, F_STRING, F_INT, F_FLOAT64, F_STRUCT = 1, 2, 3, 4, 5, 6, 7
F_UINT64, F_BYTES, F_FLOAT32 = 8, 9, 10   # uint64 / uint, []byte (base64, nil -> null), float32
F_TIME = 11   # time.Time: (unix seconds, nanoseconds, zone offset seconds)
# what a field holds of its kind T: T, *T, []T, map[string]T (include/gofr_b200.h GOFR_C_*)
C_VALUE, C_PTR, C_SLICE, C_MAP = 0, 1, 2, 3
C_SLICE_PTR = 4   # []*T: a presence word before every element (None elements are nil pointers)
FIELD_BARE = 1   # one-field schema standing for the field's own type (a handler returning []T, map[string]T, ...)
NIL_COUNT = 0xFFFFFFFF

REQ_FORCE_QUERY = 1
ROUTE_NONE = 0xFFFF

DESC_DTYPE = np.dtype([("arena_off", "<u4"), ("path_len", "<u2"), ("query_len", "<u2"), ("data_len", "<u4"),
                       ("method", "u1"), ("flags", "u1"), ("aux", "<u2")])
assert DESC_DTYPE.itemsize == 16


def method_code(name: str) -> int:
    """mux's methodMatcher compares exact strings: anything but the canonical upper-case names is OTHER."""
    return METHOD_BY_NAME.get(name, M_OTHER)


@dataclass
class Field:
    go_name: str
    kind: int
    json_name: str = ""
    omitempty: bool = False
    container: int = C_VALUE
    elem_schema: int = 0      # F_STRUCT: id of the struct's schema
    flags: int = 0

    @property
    def name(self) -> str:
        return self.json_name or self.go_name


def _str_bytes(v) -> bytes:
    return v.encode("utf-8", "surrogateescape") if isinstance(v, str) else bytes(v)


@dataclass
class Schema:
    id: int
    go_type: str  # reflect.Type.String(), e.g. "main.Person"
    fields: List[Field]

    def is_flat(self) -> bool:
        return all(f.container == C_VALUE and f.kind <= F_INT and not f.flags for f in self.fields)

    def fixed_bytes(self, lookup=None) -> int:
        return sum(self._field_fixed(f, lookup) for f in self.fields)

    @staticmethod
    def _scalar_bytes(kind: int) -> int:
        return 16 if kind == F_TIME else 8 if kind in (F_INT64, F_INT, F_FLOAT64, F_UINT64) else 4

    def _field_fixed(self, f: Field, lookup) -> int:
        if f.container in (C_SLICE, C_MAP, C_SLICE_PTR):
            return 4
        n = lookup(f.elem_schema).fixed_bytes(lookup) if f.kind == F_STRUCT else self._scalar_bytes(f.kind)
        return n + (4 if f.container == C_PTR else 0)

    @staticmethod
    def _scalar(kind: int, v) -> bytes:
        if kind in (F_INT64, F_INT):
            return int(v).to_bytes(8, "little", signed=True)
        if kind == F_INT32:
            return int(v).to_bytes(4, "little", signed=True)
        if kind == F_BOOL:
            return (1 if v else 0).to_bytes(4, "little")
        if kind == F_FLOAT64:
            import struct
            return v if isinstance(v, (bytes, bytearray)) else struct.pack("<d", float(v))   # bytes: raw IEEE bits (NaN payloads)
        if kind == F_FLOAT32:
            import struct
            return v if isinstance(v, (bytes, bytearray)) else struct.pack("<f", float(v))
        if kind == F_UINT64:
            return int(v).to_bytes(8, "little", signed=False)
        if kind == F_TIME:   # (unix seconds, nanoseconds, zone offset in seconds)
            return int(v[0]).to_bytes(8, "little", signed=True) + int(v[1]).to_bytes(4, "little") + int(v[2]).to_bytes(4, "little", signed=True)
        raise ValueError(f"bad field kind {kind}")

    def _plain(self, f: Field, v, lookup):
        """(fixed, variable) of a T"""
        if f.kind == F_STRING:
            b = _str_bytes(v)
            return len(b).to_bytes(4, "little"), b
        if f.kind == F_BYTES:   # []byte: None is the nil slice
            return (NIL_COUNT.to_bytes(4, "little"), b"") if v is None else (len(v).to_bytes(4, "little"), bytes(v))
        if f.kind == F_STRUCT:
            sub = lookup(f.elem_schema)
            row = sub.encode_row(v, lookup)
            fb = sub.fixed_bytes(lookup)
            return row[:fb], row[fb:]
        return self._scalar(f.kind, v), b""

    def _element(self, f: Field, v, lookup) -> bytes:
        if f.kind == F_STRING:
            b = _str_bytes(v)
            return len(b).to_bytes(4, "little") + b
        if f.kind == F_BYTES:
            return NIL_COUNT.to_bytes(4, "little") if v is None else len(v).to_bytes(4, "little") + bytes(v)
        if f.kind == F_STRUCT:
            return lookup(f.elem_schema).encode_row(v, lookup)
        return self._scalar(f.kind, v)

    def encode_row(self, values: Sequence, lookup=None) -> bytes:
        """Handler-result row (include/gofr_b200.h "Row format"): the fixed part — one LE u32 word per field (INT64 / INT /
        FLOAT64 two, nested structs inline, pointers a presence word first, slices and maps their count) — then the
        variable part.  values: one per field; a nested struct is a sequence, *T is None or the value, []T None or a list,
        map[string]T None or a dict (row order = dict order; the encoder sorts).  lookup(schema_id) resolves F_STRUCT."""
        words = bytearray()
        tail = bytearray()
        for f, v in zip(self.fields, values):
            if f.container == C_VALUE:
                fx, var = self._plain(f, v, lookup)
                words += fx
                tail += var
            elif f.container == C_PTR:
                if v is None:
                    words += bytes(self._field_fixed(f, lookup))
                else:
                    fx, var = self._plain(f, v, lookup)
                    words += (1).to_bytes(4, "little") + fx
                    tail += var
            elif f.container == C_SLICE:
                words += (NIL_COUNT if v is None else len(v)).to_bytes(4, "little")
                for e in (v or ()):
                    tail += self._element(f, e, lookup)
            elif f.container == C_SLICE_PTR:
                words += (NIL_COUNT if v is None else len(v)).to_bytes(4, "little")
                for e in (v or ()):
                    tail += (0).to_bytes(4, "little") if e is None else (1).to_bytes(4, "little") + self._element(f, e, lookup)
            elif f.container == C_MAP:
                words += (NIL_COUNT if v is None else len(v)).to_bytes(4, "little")
                for k, e in (v or {}).items():
                    kb = _str_bytes(k)
                    tail += len(kb).to_bytes(4, "little") + kb + self._element(f, e, lookup)
            else:
                raise ValueError(f"bad container {f.container}")
        return bytes(words + tail)


@dataclass
class Route:
    method: int
    pattern: str
    kind: int
    schema_id: int = 0
    s0: bytes = b""
    s1: bytes = b""
    s2: bytes = b""
    s3: bytes = b""
    blob: bytes = b""


@dataclass
class TableSpec:
    frame_mode: int = FRAME_WIRE
    schemas: List[Schema] = field(default_factory=list)
    routes: List[Route] = field(default_factory=list)
    default_routes: bool = True  # what App.Run() appends (gofr.go:102-107)
    favicon: bytes = b"\x89PNG\r\n\x1a\n" + bytes(range(48))  # stand-in blob with the PNG signature of the embedded one

    def schema(self, sid: int) -> Schema:
        for s in self.schemas:
            if s.id == sid:
                return s
        raise KeyError(sid)


@dataclass
class Req:
    method: int
    path: bytes
    query: bytes = b""
    data: bytes = b""
    flags: int = 0
    trace_id: Optional[bytes] = None


class RequestBatch:
    """desc[n] / trace_ids[n,16] / arena — contiguous numpy arrays in the ABI layout."""

    def __init__(self, desc: np.ndarray, trace_ids: np.ndarray, arena: np.ndarray):
        assert desc.dtype == DESC_DTYPE and trace_ids.dtype == np.uint8 and arena.dtype == np.uint8
        assert trace_ids.shape == (len(desc), 16)
        self.desc = np.ascontiguousarray(desc)
        self.trace_ids = np.ascontiguousarray(trace_ids)
        self.arena = np.ascontiguousarray(arena)

    @property
    def n(self) -> int:
        return len(self.desc)

    def slice(self, lo: int, hi: int) -> "RequestBatch":
        """A contiguous shard [lo, hi) that shares the arena (offsets stay absolute)."""
        return RequestBatch(self.desc[lo:hi].copy(), self.trace_ids[lo:hi].copy(), self.arena)

    def input_bytes(self) -> int:
        """Bytes the serve kernel must read: descriptors + trace ids + the arena bytes the descriptors cover."""
        return self.n * 32 + int(self.arena_span())

    def arena_span(self) -> int:
        if self.n == 0:
            return 0
        d = self.desc
        start = int(d["arena_off"][0])
        last = d[-1]
        end = ((int(last["arena_off"]) + int(last["path_len"]) + int(last["query_len"]) + 3) & ~3) + int(last["data_len"])
        return end - start

    @staticmethod
    def pack(reqs: Sequence[Req], seed: int = 0x60F2B200) -> "RequestBatch":
        n = len(reqs)
        desc = np.zeros(n, dtype=DESC_DTYPE)
        ids = np.zeros((n, 16), dtype=np.uint8)
        arena = bytearray()
        rng = np.random.default_rng(seed)
        rnd = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
        for i, r in enumerate(reqs):
            while len(arena) % 4:
                arena.append(0)
            off = len(arena)
            arena += r.path
            arena += r.query
            while len(arena) % 4:
                arena.append(0)
            arena += r.data
            desc[i] = (off, len(r.path), len(r.query), len(r.data), r.method, r.flags, 0)
            ids[i] = np.frombuffer(r.trace_id, dtype=np.uint8) if r.trace_id is not None else rnd[i]
        while len(arena) % 16:
            arena.append(0)
        return RequestBatch(desc, ids, np.frombuffer(bytes(arena), dtype=np.uint8).copy())


LOG_REQUEST, LOG_RPC, LOG_NONE = 0, 1, 2   # LOG_NONE: this request gets no line from gofr_batch_submit_log

# gofr_log_desc (include/gofr_b200.h): one RequestLog record (middleware/logger.go:24-33,41-70)
LOG_DESC_DTYPE = np.dtype([("start_unix_ns", "<i8"), ("elapsed_ns", "<i8"), ("log_unix_ns", "<i8"), ("arena_off", "<u4"),
                           ("method_len", "<u2"), ("ua_len", "<u2"), ("xff_len", "<u2"), ("remote_len", "<u2"),
                           ("uri_len", "<u2"), ("status", "<u2"), ("tz_offset_s", "<i4"), ("kind", "<u4")])
assert LOG_DESC_DTYPE.itemsize == 48


@dataclass
class LogRec:
    """What middleware.Logging reads from the clock and the request for one log line."""
    start_unix_ns: int
    elapsed_ns: int
    log_unix_ns: int
    method: bytes = b"GET"
    user_agent: bytes = b""
    xff: bytes = b""          # first X-Forwarded-For header value ("" if absent)
    remote_addr: bytes = b""
    uri: bytes = b"/"
    status: int = 200
    tz_offset_s: int = 0
    trace_id: Optional[bytes] = None
    kind: int = 0             # LOG_REQUEST, or LOG_RPC (the gRPC interceptor's RPCLog line; method = info.FullMethod)


class LogBatch:
    """desc[n] (gofr_log_desc) / trace_ids[n,16] / arena (method|user_agent|xff|remote_addr|uri per record)."""

    def __init__(self, desc: np.ndarray, trace_ids: np.ndarray, arena: np.ndarray):
        assert desc.dtype == LOG_DESC_DTYPE and trace_ids.dtype == np.uint8 and arena.dtype == np.uint8
        assert trace_ids.shape == (len(desc), 16)
        self.desc = np.ascontiguousarray(desc)
        self.trace_ids = np.ascontiguousarray(trace_ids)
        self.arena = np.ascontiguousarray(arena)

    @property
    def n(self) -> int:
        return len(self.desc)

    def input_bytes(self) -> int:
        return self.n * (48 + 16) + int(self.arena.size)

    @staticmethod
    def pack(recs: Sequence[LogRec], seed: int = 0x60F2B200) -> "LogBatch":
        n = len(recs)
        desc = np.zeros(n, dtype=LOG_DESC_DTYPE)
        ids = np.zeros((n, 16), dtype=np.uint8)
        rnd = np.random.default_rng(seed).integers(0, 256, size=(n, 16), dtype=np.uint8)
        arena = bytearray()
        for i, r in enumerate(recs):
            desc[i] = (r.start_unix_ns, r.elapsed_ns, r.log_unix_ns, len(arena), len(r.method), len(r.user_agent),
                       len(r.xff), len(r.remote_addr), len(r.uri), r.status, r.tz_offset_s, r.kind)
            arena += r.method + r.user_agent + r.xff + r.remote_addr + r.uri
            ids[i] = np.frombuffer(r.trace_id, dtype=np.uint8) if r.trace_id is not None else rnd[i]
        return LogBatch(desc, ids, np.frombuffer(bytes(arena), dtype=np.uint8).copy())


# protobuf field types (google.protobuf.FieldDescriptorProto.Type numbers) the proto3 encoder takes
(PB_DOUBLE, PB_FLOAT, PB_INT64, PB_UINT64, PB_INT32, PB_FIXED64, PB_FIXED32, PB_BOOL, PB_STRING) = range(1, 10)
PB_BYTES, PB_UINT32, PB_ENUM, PB_SFIXED32, PB_SFIXED64, PB_SINT32, PB_SINT64 = 12, 13, 14, 15, 16, 17, 18
PB_64BIT = (PB_DOUBLE, PB_INT64, PB_UINT64, PB_FIXED64, PB_SFIXED64, PB_SINT64)
GRPC_OK, GRPC_COMPRESSED, GRPC_BAD_LENGTH, GRPC_BAD_PROTO, GRPC_BAD_UTF8, GRPC_BAD_ROW, GRPC_DEFER = range(7)


@dataclass
class ProtoField:
    number: int
    type: int


def pack_proto_rows(fields: Sequence[ProtoField], messages: Sequence[Sequence]) -> "tuple[np.ndarray, np.ndarray]":
    """Rows for gofr_proto_encode_device: per field (in the order given = field-number order) 64-bit kinds two LE words,
    the others one (floats and doubles as their IEEE bits, strings / bytes as their length), then the string bytes.
    Values: ints (any sign, taken modulo the width), bools, floats, bytes / str.  Returns (rows uint8, row_off uint32);
    8 bytes of padding follow the last row (the device copies with aligned word loads)."""
    import struct
    blob = bytearray()
    off = [0]
    for msg in messages:
        words = bytearray()
        tail = bytearray()
        for f, v in zip(fields, msg):
            if f.type == PB_DOUBLE:
                words += struct.pack("<d", v) if isinstance(v, float) else int(v).to_bytes(8, "little")
            elif f.type == PB_FLOAT:
                words += struct.pack("<f", v) if isinstance(v, float) else int(v).to_bytes(4, "little")
            elif f.type in PB_64BIT:
                words += (int(v) & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little")
            elif f.type in (PB_STRING, PB_BYTES):
                b = v.encode("utf-8", "surrogateescape") if isinstance(v, str) else bytes(v)
                words += len(b).to_bytes(4, "little")
                tail += b
            elif f.type == PB_BOOL:
                words += (1 if v else 0).to_bytes(4, "little")
            else:
                words += (int(v) & 0xFFFFFFFF).to_bytes(4, "little")
        blob += words + tail
        blob += b"\0" * ((-len(blob)) % 4)
        off.append(len(blob))
    blob += b"\0" * 8
    return np.frombuffer(bytes(blob), dtype=np.uint8).copy(), np.array(off, dtype=np.uint32)


PB_MESSAGE = 11
PB_MAP = 32          # a map field: msg is its entry type (fields 1 key, 2 value); not repeated
PB_OPTIONAL = 0x80   # ProtoNField.presence: proto3 optional (1..7: a member of that oneof group)


@dataclass
class ProtoNField:
    """one field of a message type with nested / repeated fields (gofr_proto_nfield)"""
    number: int
    type: int            # PB_*, PB_MESSAGE or PB_MAP
    repeated: bool = False
    msg: int = 0         # PB_MESSAGE: index of the message type; PB_MAP: index of the entry type
    presence: int = 0    # 0 implicit presence, PB_OPTIONAL, or 1..7: a member of that oneof group of its message type


def _explicit(f: ProtoNField) -> bool:
    """a scalar / string / bytes field with a presence word of its own in the row"""
    return bool(f.presence) and f.type not in (PB_MESSAGE, PB_MAP) and not f.repeated


def proto_nested_presence(msgs: Sequence[Sequence[ProtoNField]]):
    """the presence bytes of the _ex calls (one per field, in the order of proto_nested_tables), or None when no field has
    explicit presence (then the calls without presence are the same)"""
    pr = [f.presence for fields in msgs for f in fields]
    return np.array(pr, dtype=np.uint8) if any(pr) else None


def proto_nested_tables(msgs: Sequence[Sequence[ProtoNField]]):
    """(gofr_proto_nmsg[n_msgs] as uint16 pairs, gofr_proto_nfield[n_fields] as 8-byte records, n_fields)"""
    nm = np.zeros((len(msgs), 2), dtype=np.uint16)
    recs = bytearray()
    k = 0
    for m, fields in enumerate(msgs):
        nm[m] = (k, len(fields))
        for f in fields:
            recs += int(f.number).to_bytes(4, "little") + bytes([f.type, 1 if f.repeated else 0]) + int(f.msg).to_bytes(2, "little")
            k += 1
    return nm, np.frombuffer(bytes(recs), dtype=np.uint8).copy(), k


def _pb_scalar_words(t: int, v) -> bytes:
    import struct
    if t == PB_DOUBLE:
        return struct.pack("<d", v) if isinstance(v, float) else int(v).to_bytes(8, "little")
    if t == PB_FLOAT:
        return struct.pack("<f", v) if isinstance(v, float) else int(v).to_bytes(4, "little")
    if t in PB_64BIT:
        return (int(v) & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little")
    if t == PB_BOOL:
        return (1 if v else 0).to_bytes(4, "little")
    return (int(v) & 0xFFFFFFFF).to_bytes(4, "little")


def map_key_order(key_type: int, k):
    """a sort key giving protobuf-go's Deterministic map order: bool false < true, signed kinds signed, unsigned kinds
    unsigned (both as the row words hold them), strings by their UTF-8 bytes with a shorter prefix first"""
    if key_type == PB_STRING:
        return k.encode("utf-8", "surrogateescape") if isinstance(k, str) else bytes(k)
    if key_type == PB_BOOL:
        return 1 if k else 0
    bits = 64 if key_type in PB_64BIT else 32
    v = int(k) & ((1 << bits) - 1)
    if key_type in (PB_INT32, PB_INT64, PB_SINT32, PB_SINT64, PB_SFIXED32, PB_SFIXED64) and v >> (bits - 1):
        v -= 1 << bits
    return v


def _pb_fixed_bytes(msgs, m: int) -> int:
    n = 0
    for f in msgs[m]:
        if f.repeated or f.type == PB_MAP:
            n += 4
        elif f.type == PB_MESSAGE:
            n += 4 + _pb_fixed_bytes(msgs, f.msg)
        else:
            n += (8 if f.type in PB_64BIT or f.type == PB_DOUBLE else 4) + (4 if _explicit(f) else 0)
    return n


def pack_proto_nested_message(msgs, m: int, value) -> "tuple[bytes, bytes]":
    """(fixed part, variable part) of one message of type m.  value: one entry per field — scalars as for pack_proto_rows, a
    singular message None (not set) or its own value list, a repeated field a list.  A map field takes a dict, whose
    entries are laid out in protobuf-go's Deterministic key order (map_key_order), or a list of (key, value) pairs laid
    out as given (unsorted or duplicate keys make a row the encoder refuses); a message value None is a nil message.  A
    scalar, string or bytes field with explicit presence (optional, a oneof member) takes None for "not set"."""
    def element(f, v) -> bytes:
        if f.type in (PB_STRING, PB_BYTES):
            b = v.encode("utf-8", "surrogateescape") if isinstance(v, str) else bytes(v)
            return len(b).to_bytes(4, "little") + b
        if f.type in (PB_MESSAGE, PB_MAP):
            fx, vr = pack_proto_nested_message(msgs, f.msg, v)
            return fx + vr
        return _pb_scalar_words(f.type, v)
    fixed, var = bytearray(), bytearray()
    for f, v in zip(msgs[m], value):
        if f.type == PB_MAP:
            if isinstance(v, dict):
                kt = msgs[f.msg][0].type
                v = sorted(v.items(), key=lambda kv: map_key_order(kt, kv[0]))
            v = [list(kv) for kv in v]
        if f.repeated or f.type == PB_MAP:
            fixed += len(v).to_bytes(4, "little")
            for e in v:
                var += element(f, e)
        elif f.type == PB_MESSAGE:
            if v is None:
                fixed += bytes(4 + _pb_fixed_bytes(msgs, f.msg))
            else:
                fx, vr = pack_proto_nested_message(msgs, f.msg, v)
                fixed += (1).to_bytes(4, "little") + fx
                var += vr
        elif _explicit(f) and v is None:
            fixed += bytes(4 + (8 if f.type in PB_64BIT or f.type == PB_DOUBLE else 4))
        elif _explicit(f):
            fixed += (1).to_bytes(4, "little")
            if f.type in (PB_STRING, PB_BYTES):
                b = v.encode("utf-8", "surrogateescape") if isinstance(v, str) else bytes(v)
                fixed += len(b).to_bytes(4, "little")
                var += b
            else:
                fixed += _pb_scalar_words(f.type, v)
        elif f.type in (PB_STRING, PB_BYTES):
            b = v.encode("utf-8", "surrogateescape") if isinstance(v, str) else bytes(v)
            fixed += len(b).to_bytes(4, "little")
            var += b
        else:
            fixed += _pb_scalar_words(f.type, v)
    return bytes(fixed), bytes(var)


def pack_proto_nested_rows(msgs, root: int, messages) -> "tuple[np.ndarray, np.ndarray]":
    """Rows for gofr_proto_encode_nested_device (4-byte aligned, 8 bytes of padding behind the last)."""
    blob = bytearray()
    off = [0]
    for v in messages:
        fx, vr = pack_proto_nested_message(msgs, root, v)
        blob += fx + vr
        blob += b"\0" * ((-len(blob)) % 4)
        off.append(len(blob))
    blob += b"\0" * 8
    return np.frombuffer(bytes(blob), dtype=np.uint8).copy(), np.array(off, dtype=np.uint32)


def http_date(unix_seconds: int) -> bytes:
    """net/http appendTime: IMF-fixdate, always 29 bytes."""
    import time
    t = time.gmtime(unix_seconds)
    days = ["Mon", "Tue", "Wed", "Thu", "Fri", "Sat", "Sun"]
    months = ["Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"]
    s = "%s, %02d %s %04d %02d:%02d:%02d GMT" % (days[t.tm_wday], t.tm_mday, months[t.tm_mon - 1], t.tm_year,
                                                  t.tm_hour, t.tm_min, t.tm_sec)
    b = s.encode()
    assert len(b) == 29
    return b
