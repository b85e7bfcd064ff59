"""The gRPC frame codecs on the GPU against protobuf: every scalar type and tag width, hostile wire input, exact capacities.

The device code of the five frame entry points (gofr_grpc_hello_device, gofr_proto_encode_device / _decode_device and the
nested gofr_proto_encode_nested_device / _decode_nested_device, with and without map fields) runs on the CPU in tests/emu and
is compared there with the oracle and python protobuf.  What exists only in the kernels is the tile loop they share
(frame_tiles.cuh): the TMA staging of a tile's bytes (up to 8 KiB) or the reads from HBM beyond that, the block scan and
the look-back that chain the packed offsets, the `fits` check that drops a whole tile when the output buffer is too small,
and the staging Writer's partial 16-byte windows at frame edges.  Each campaign below feeds one kernel seeded inputs that
reach those paths — all scalar types, tags of one to five bytes, hostile and mutated frames, lying headers, long strings —
and requires the GPU result to equal the oracle (or, for map fields, the model tests/proto_nested_model.py) byte for byte,
with 0xEE canaries behind every output.  The unmarked twin of each campaign checks on the CPU, on exactly the same inputs,
that the oracle equals the emulated device code and agrees with python protobuf, so that a GPU mismatch is a kernel finding.

The divergences from python protobuf that the twins allow are the documented ones: a tenth varint byte above 1 (protobuf-go
refuses it, upb truncates), unknown groups nested deeper than 16 (BAD_PROTO by design), and DEFER (a singular message sent
twice, more than 64 entries of one map field).

Each GPU campaign runs in a child process of its own: a fault in a kernel stays inside its test.
"""
import math
import os
import random
import struct
import subprocess
import sys
from functools import lru_cache

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from tests import oracle as O
from tests import proto_nested_harness as H
from tests import proto_nested_model as M
from tests import test_grpc as TG
from tests import test_proto as TP
from tests.emu import emu

ROOT_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 128                      # frames per tile (kServeThreads)
STAGE = 8192                 # bytes of a tile staged in shared memory (kGrpcStage); larger tiles are read from HBM
F = S.ProtoNField
OK, COMPRESSED, BAD_LENGTH, BAD_PROTO, BAD_UTF8, BAD_ROW, DEFER = (S.GRPC_OK, S.GRPC_COMPRESSED, S.GRPC_BAD_LENGTH, S.GRPC_BAD_PROTO,
                                                                   S.GRPC_BAD_UTF8, S.GRPC_BAD_ROW, S.GRPC_DEFER)
_varint, _frame, _pack = TP._varint, TP._frame, TP._pack_frames


# ---------------------------------------------------------------------------------------------------------------
# shared pieces
# ---------------------------------------------------------------------------------------------------------------
def _tile_paths(off):
    """(tiles staged, tiles read from HBM) by the kernels' rule: the span [off[t0] & ~15, (off[t1] + 15) & ~15) is staged when
    it is not empty and at most STAGE bytes"""
    staged = hbm = 0
    n = len(off) - 1
    for t0 in range(0, n, T):
        lo, hi = int(off[t0]) & ~15, (int(off[min(n, t0 + T)]) + 15) & ~15
        if hi > lo and hi - lo <= STAGE:
            staged += 1
        elif hi > lo:
            hbm += 1
    return staged, hbm


def _header_status(fr):
    """the status of a frame whose 5-byte header is wrong (None for a good header): too short, compressed, other flags,
    a length that disagrees with the frame"""
    if len(fr) < 5:
        return BAD_LENGTH
    if fr[0] == 1:
        return COMPRESSED
    if fr[0] != 0 or int.from_bytes(fr[1:5], "big") != len(fr) - 5:
        return BAD_LENGTH
    return None


_FRAGS = [b"\x08\x01", b"\x0b\x0c", b"\x12\x00", b"\xfa\x7f\x01\x00", b"\x0d\x00\x00\x00\x00", b"\x80", b"\x0a\x01\xff", b"\x0a\x02\x08\x01"]


def _mutate(rnd, body):
    """one to three of: a bit flipped, the tail cut, a fragment inserted, the tail moved in front"""
    body = bytearray(body)
    for _ in range(rnd.randint(1, 3)):
        r = rnd.randrange(4)
        if r == 0 and body:
            body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
        elif r == 1 and body:
            del body[rnd.randrange(len(body)):]
        elif r == 2:
            p = rnd.randrange(len(body) + 1)
            body[p:p] = rnd.choice(_FRAGS)
        else:
            p = rnd.randrange(len(body) + 1)
            body = body[p:] + body[:p]
    return bytes(body)


_TEXT = "aZ09 \t\x00é€日本\U0001F600"


def _text(rnd, n):
    s = "".join(rnd.choice(_TEXT) for _ in range(n))
    return s + "\udc80" if rnd.random() < 0.05 else s       # a lone surrogate: invalid UTF-8 once encoded (surrogatepass)


def _soup_frag(rnd, hi=14):
    """one wire fragment for field numbers 1..hi: varint, fixed64, fixed32, length-delimited (bytes or text), an empty group,
    or junk"""
    k, n = rnd.randrange(6), rnd.randint(1, hi)
    if k == 0:
        return _varint(n << 3) + _varint(rnd.getrandbits(rnd.choice([1, 7, 8, 32, 35, 63, 64])))
    if k == 1:
        return _varint(n << 3 | 1) + rnd.randbytes(8)
    if k == 2:
        return _varint(n << 3 | 5) + rnd.randbytes(4)
    if k == 3:
        b = rnd.randbytes(rnd.randint(0, 12)) if rnd.random() < 0.5 else _text(rnd, rnd.randint(0, 8)).encode("utf-8", "surrogatepass")
        return _varint(n << 3 | 2) + _varint(len(b)) + b
    if k == 4:
        return _varint(n << 3 | 3) + _varint(n << 3 | 4)
    return rnd.randbytes(rnd.randint(1, 3))


# ---------------------------------------------------------------------------------------------------------------
# the entry points through the C ABI, with buffers the caller owns
# ---------------------------------------------------------------------------------------------------------------
CANARY = 0xEE


def gpu_run(eng, kind, spec, data, off, cap):
    """one launch of `kind` ("hello", "enc", "dec", "nenc", "ndec"; spec: the fields, or (msgs, root)) over data[:off[-1]]
    followed by exactly the 16 bytes of slack the ABI asks for (0xEE: never looked at).  d_out has `cap` bytes and 64 more
    of 0xEE behind them; d_out_off and d_meta start as 0xEEEEEEEE.  Returns (out[cap + 64], out_off, meta, overflowed)."""
    import torch
    L = _abi.lib()
    n = len(off) - 1
    src = np.concatenate([np.ascontiguousarray(data[:int(off[-1])], dtype=np.uint8), np.full(16, CANARY, np.uint8)])
    d_in = torch.from_numpy(src).cuda()
    d_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.uint32).view(np.int32)).cuda()
    fill = int(np.array([0xEEEEEEEE], dtype=np.uint32).view(np.int32)[0])
    d_out = torch.full((cap + 64,), CANARY, dtype=torch.uint8, device="cuda")
    d_ooff = torch.full((n + 1,), fill, dtype=torch.int32, device="cuda")
    d_meta = torch.full((max(n, 1),), fill, dtype=torch.int32, device="cuda")
    args = (d_in.data_ptr(), d_off.data_ptr(), n, d_out.data_ptr(), cap, d_ooff.data_ptr(), d_meta.data_ptr(),
            torch.cuda.current_stream().cuda_stream)
    if kind == "hello":
        rc = L.gofr_grpc_hello_device(eng._e, *args)
    elif kind in ("enc", "dec"):
        ft = (_abi.ProtoField * max(len(spec), 1))(*[_abi.ProtoField(f.number, f.type) for f in spec])
        rc = (L.gofr_proto_encode_device if kind == "enc" else L.gofr_proto_decode_device)(eng._e, ft, len(spec), *args)
    else:
        msgs, root = spec
        nm, nf, k = S.proto_nested_tables(msgs)
        fn = L.gofr_proto_encode_nested_device if kind == "nenc" else L.gofr_proto_decode_nested_device
        rc = fn(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, *args)
    _abi.check(rc, kind)
    torch.cuda.synchronize()
    return d_out.cpu().numpy(), d_ooff.cpu().numpy().view(np.uint32), d_meta.cpu().numpy().view(np.uint32)[:n], eng.overflowed()


def reference(kind, spec, data, off):
    """what the launch must produce: (output bytes, out_off, meta) from the oracle — or, for message types with map fields,
    from the model"""
    n = len(off) - 1
    data = np.ascontiguousarray(data)
    if kind in ("nenc", "ndec") and any(f.type == S.PB_MAP for fs in spec[0] for f in fs):
        msgs, root = spec
        if kind == "nenc":
            items, meta = M.encode(msgs, root, data, off)
        else:
            items, meta = M.decode(msgs, root, [data[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)])
        return b"".join(items), np.cumsum([0] + [len(x) for x in items]).astype(np.uint32), np.array(meta, dtype=np.uint32)
    if kind == "hello":
        out, o, meta = O.grpc_hello(data, off)
    elif kind == "enc":
        out, o, meta = O.proto_encode(spec, data, off)
    elif kind == "dec":
        out, o, meta = O.proto_decode(spec, data, off)
    elif kind == "nenc":
        out, o, meta = O.proto_encode_nested(spec[0], spec[1], data, off)
    else:
        out, o, meta = O.proto_decode_nested(spec[0], spec[1], data, off)
    return out[:int(o[-1])].tobytes(), o, np.asarray(meta[:n], dtype=np.uint32)


def _first(a, b):
    d = np.flatnonzero(np.asarray(a) != np.asarray(b))
    return int(d[0]) if len(d) else None


def check_equal(got, want, what):
    """the GPU launch == the reference: offsets, statuses, bytes, and nothing written behind out_off[n]"""
    out, off, meta, ovf = got
    w_out, w_off, w_meta = want
    assert not ovf, what + ": overflow flag raised with a sufficient capacity"
    i = _first(off, w_off)
    assert i is None, "%s: out_off[%d] = %d, want %d" % (what, i, off[i], w_off[i])
    i = _first(meta, w_meta)
    assert i is None, "%s: meta[%d] = %d, want %d" % (what, i, meta[i], w_meta[i])
    total = int(w_off[-1])
    if out[:total].tobytes() != w_out:
        b = _first(out[:total], np.frombuffer(w_out, dtype=np.uint8))
        raise AssertionError("%s: output differs at byte %d (item %d)" % (what, b, int(np.searchsorted(w_off, b, side="right")) - 1))
    assert (out[total:] == CANARY).all(), what + ": bytes written behind out_off[n]"


# ---------------------------------------------------------------------------------------------------------------
# 1. flat encoder: random message types over every scalar type and ENUM, every tag width, bad rows, batch sizes
# ---------------------------------------------------------------------------------------------------------------
TAG_NUMBERS = [1, 15, 16, 2047, 2048, 262143, 262144, 2 ** 29 - 1]     # the last field number of tags of 1 .. 5 bytes and the first of the next
FLAT_TYPES = TP.ALL_TYPES + [S.PB_ENUM]
_INT_BITS = {S.PB_INT32: (32, True), S.PB_ENUM: (32, True), S.PB_SFIXED32: (32, True), S.PB_SINT32: (32, True),
             S.PB_INT64: (64, True), S.PB_SFIXED64: (64, True), S.PB_SINT64: (64, True),
             S.PB_UINT32: (32, False), S.PB_FIXED32: (32, False), S.PB_UINT64: (64, False), S.PB_FIXED64: (64, False)}
_EDGE = {S.PB_FLOAT: [0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-45, 3.4028234663852886e38, 1.5],
         S.PB_DOUBLE: [0.0, -0.0, float("inf"), float("-inf"), float("nan"), 5e-324, 1.7976931348623157e308, -1e300],
         S.PB_BOOL: [False, True], S.PB_STRING: ["", "a", "é", "x" * 127, "y" * 128, "z" * 300, "\U0001F600"],
         S.PB_BYTES: [b"", b"\x00", b"\xff\xfe", b"b" * 128]}


def _int_edges(bits, signed):
    if signed:
        return [0, 1, -1, 2 ** (bits - 1) - 1, -2 ** (bits - 1), 127, 128, -129, 16383, 16384]
    return [0, 1, 2 ** bits - 1, 2 ** (bits - 1), 127, 128, 16383, 16384]


def _flat_value(rnd, t):
    if t in _INT_BITS:
        bits, signed = _INT_BITS[t]
        if rnd.random() < 0.4:
            return rnd.choice(_int_edges(bits, signed))
        v = rnd.getrandbits(rnd.randint(1, bits))
        if signed:
            v = ((v if rnd.random() < 0.5 else -v) + 2 ** (bits - 1)) % 2 ** bits - 2 ** (bits - 1)
        return v
    if rnd.random() < 0.4:
        return rnd.choice(_EDGE[t])
    if t == S.PB_FLOAT:
        return struct.unpack("<f", struct.pack("<f", rnd.uniform(-1, 1) * 10.0 ** rnd.randint(-30, 30)))[0]
    if t == S.PB_DOUBLE:
        return rnd.uniform(-1, 1) * 10.0 ** rnd.randint(-300, 300)
    if t == S.PB_BOOL:
        return rnd.random() < 0.5
    n = rnd.choice([0, 1, 5, 40, 127, 128, 300])
    return _text(rnd, n).replace("\udc80", "") if t == S.PB_STRING else rnd.randbytes(n)


def _flat_schema(rnd, nf):
    pool = set(TAG_NUMBERS + [rnd.randint(2, 14), rnd.randint(17, 2046), rnd.randint(2049, 18999), rnd.randint(20000, 262142),
                              rnd.randint(262145, 2 ** 29 - 2)] + rnd.sample(range(1, 60), 12))
    return [S.ProtoField(n, rnd.choice(FLAT_TYPES)) for n in sorted(rnd.sample(sorted(pool), min(nf, len(pool))))]


SCHEMA_32 = [S.ProtoField(n, FLAT_TYPES[k % len(FLAT_TYPES)])
             for k, n in enumerate(sorted(TAG_NUMBERS + list(range(2, 15)) + list(range(17, 28))))]


def _py_fields(fields):
    return [S.ProtoField(f.number, S.PB_INT32 if f.type == S.PB_ENUM else f.type) for f in fields]


def _bad_rows(rnd):
    """a schema with three strings; rows of every malformed kind, each between good rows.  Returns (fields, blobs, values,
    want): values[i] is the row's message (None for a hand-made row), want[i] its required status (None: OK)"""
    fields = [S.ProtoField(1, S.PB_STRING), S.ProtoField(2, S.PB_INT64), S.ProtoField(16, S.PB_BYTES), S.ProtoField(2047, S.PB_STRING),
              S.ProtoField(2048, S.PB_FIXED32), S.ProtoField(2 ** 29 - 1, S.PB_STRING)]
    fixed = 4 + 8 + 4 + 4 + 4 + 4
    blobs, values, want = [], [], []

    def good():
        v = [_flat_value(rnd, f.type) for f in fields]
        r, o = S.pack_proto_rows(fields, [v])
        return v, r[:int(o[1])].tobytes()
    for k in range(400):
        v, row = good()
        kind = k % 8
        if kind == 0:                        # invalid UTF-8 in one of the three string positions
            pos = rnd.choice([0, 3, 5])
            v[pos] = rnd.choice([b"\xff", b"\xc3", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"ok\xe2\x82", "fine".encode() + b"\x80"])
            r, o = S.pack_proto_rows(fields, [v])
            blobs.append(r[:int(o[1])].tobytes()); values.append(None); want.append(BAD_UTF8)
        elif kind == 1:                      # shorter than its fixed part
            blobs.append(row[:4 * rnd.randrange(fixed // 4)]); values.append(None); want.append(BAD_ROW)
        elif kind == 2:                      # a string length that runs past the row
            slot = rnd.choice([0, 12, 16, 24])       # the length words of the string and bytes fields
            spos = fixed + sum(int.from_bytes(row[w:w + 4], "little") for w in (0, 12, 16, 24) if w < slot)
            over = len(row) - spos + rnd.choice([1, 2, 4, 1 << 20, 0xFFFFFFFF - (len(row) - spos)])
            blobs.append(row[:slot] + (over & 0xFFFFFFFF).to_bytes(4, "little") + row[slot + 4:]); values.append(None); want.append(BAD_ROW)
        elif kind == 3:                      # the row at an offset that is not a multiple of 4, two 2-byte rows around it
            blobs += [b"\x01\x02", row, b"\x03\x04"]; values += [None] * 3; want += [BAD_ROW] * 3
        else:
            blobs.append(row); values.append(v); want.append(None)
    return fields, blobs, values, want


def _assemble(blobs):
    body = b"".join(blobs)
    off = np.cumsum([0] + [len(b) for b in blobs]).astype(np.uint32)
    return np.frombuffer(body + b"\0" * 8, dtype=np.uint8).copy(), off


@lru_cache(maxsize=None)
def encoder_cases():
    """[(label, fields, rows, off, values, want)]: values[i] the message of row i (None for a hand-made one), want[i] a required
    status or None"""
    rnd = random.Random(0xE1C0)
    cases = []
    for n in (0, 1, 127, 128, 129, 5000):
        fields = _flat_schema(rnd, rnd.randint(1, 12))
        msgs = [[_flat_value(rnd, f.type) for f in fields] for _ in range(n)]
        cases.append(("n=%d" % n, fields, msgs))
    for k in range(16):
        fields = _flat_schema(rnd, rnd.randint(1, 16))
        cases.append(("random %d" % k, fields, [[_flat_value(rnd, f.type) for f in fields] for _ in range(300)]))
    cases.append(("32 fields", SCHEMA_32, [[_flat_value(rnd, f.type) for f in SCHEMA_32] for _ in range(1000)]))
    long_f = [S.ProtoField(1, S.PB_STRING), S.ProtoField(262144, S.PB_BYTES), S.ProtoField(2 ** 29 - 1, S.PB_SINT64)]
    cases.append(("long strings", long_f, [["é" * rnd.randint(0, 1500), rnd.randbytes(rnd.randint(0, 3000)), _flat_value(rnd, S.PB_SINT64)]
                                          for _ in range(400)]))
    out = []
    for label, fields, msgs in cases:
        rows, off = S.pack_proto_rows(fields, msgs)
        out.append((label, fields, rows, off, msgs, [None] * len(msgs)))
    fields, blobs, values, want = _bad_rows(rnd)
    rows, off = _assemble(blobs)
    out.append(("bad rows", fields, rows, off, values, want))
    return out


def test_encoder_cases_three_ways():
    """oracle == device code (CPU, output misalignments 0 and 3) on every encoder case; every OK frame == python's
    SerializeToString(); the hand-made bad rows get their status; the cases reach both tile paths"""
    paths = [0, 0]
    for label, fields, rows, off, values, want in encoder_cases():
        out, o, meta = O.proto_encode(fields, rows, off)
        for mis in (0, 3):
            e_out, e_off, e_meta = emu.proto_encode(fields, rows, off, mis)
            assert np.array_equal(e_meta, meta) and np.array_equal(e_off, o + mis), label
            assert e_out[mis:int(e_off[-1])].tobytes() == out[:int(o[-1])].tobytes(), label
        idx = [i for i, v in enumerate(values) if v is not None]
        py = TP._py_serialize(_py_fields(fields), [values[i] for i in idx])
        fr = TP._frames(out, o)
        for i, p in zip(idx, py):
            assert meta[i] == OK and fr[i] == p, (label, i, values[i])
        for i, w in enumerate(want):
            if w is not None:
                assert meta[i] == w and fr[i] == b"", (label, i)
        s, h = _tile_paths(off)
        paths[0] += s
        paths[1] += h
    assert paths[0] > 0 and paths[1] > 0, paths
    types = {f.type for c in encoder_cases() for f in c[1]}
    numbers = {f.number for c in encoder_cases() for f in c[1]}
    assert types == set(FLAT_TYPES) and set(TAG_NUMBERS) <= numbers


def _gpu_encoder(eng):
    rows_n = 0
    for label, fields, rows, off, _, _ in encoder_cases():
        want = reference("enc", fields, rows, off)
        check_equal(gpu_run(eng, "enc", fields, rows, off, len(want[0]) + 16), want, "encoder " + label)
        rows_n += len(off) - 1
    return "flat encoder: %d rows in %d launches equal to the oracle" % (rows_n, len(encoder_cases()))


# ---------------------------------------------------------------------------------------------------------------
# 2. flat decoder: hostile bodies, wire soup, mutated encoder output, lying headers, deep groups, long strings
# ---------------------------------------------------------------------------------------------------------------
def _deep(d):
    return b"".join(TP.T(60 + k, 3) for k in range(d)) + b"".join(TP.T(60 + k, 4) for k in reversed(range(d)))


@lru_cache(maxsize=None)
def decoder_cases():
    """[(label, fields, frames, want)]: want[i] a required status, or None where python protobuf decides"""
    rnd = random.Random(0xDEC0)
    cases = []
    bodies = TP.HOSTILE_BODIES
    want = [None] * (len(bodies) - 1) + [BAD_PROTO] + [_header_status(f) for f in TP.HOSTILE_HEADER_FRAMES]
    cases.append(("hostile", TP.HOSTILE_FIELDS, [_frame(b) for b in bodies] + TP.HOSTILE_HEADER_FRAMES, want))
    # groups 16 deep (accepted), 17 deep (BAD_PROTO: python accepts), unbalanced
    g = [_deep(16), _deep(16) + TP.T(1, 2) + b"\x01a", TP.T(59, 3) + _deep(16) + TP.T(59, 4), _deep(17), _deep(16)[:-1],
         _deep(15) + TP.T(2, 0) + b"\x05"]
    cases.append(("groups", TP.HOSTILE_FIELDS, [_frame(b) for b in g], [None, None, BAD_PROTO, BAD_PROTO, None, None]))
    for k in range(100):                     # wire soup
        fields = [S.ProtoField(n, rnd.choice(TP.ALL_TYPES)) for n in sorted(rnd.sample(range(1, 13), rnd.randint(1, 8)))]
        frames = [_frame(b"".join(_soup_frag(rnd) for _ in range(rnd.randint(0, 6)))) for _ in range(250)]
        cases.append(("soup %d" % k, fields, frames, [None] * len(frames)))
    for k in range(40):                      # encoder output, mutated four ways (every fourth frame left whole)
        fields = _py_fields(_flat_schema(rnd, rnd.randint(1, 10)))
        rows, off = S.pack_proto_rows(fields, [[_flat_value(rnd, f.type) for f in fields] for _ in range(250)])
        out, o, _ = O.proto_encode(fields, rows, off)
        frames = [fr for fr in TP._frames(out, o) if fr]
        frames = [fr if i % 4 == 0 else _frame(_mutate(rnd, fr[5:])) for i, fr in enumerate(frames)]
        cases.append(("mutated %d" % k, fields, frames, [None] * len(frames)))
    # headers that lie: flags 1 .. 255, lengths one off, frames shorter than a header
    fields = [S.ProtoField(1, S.PB_STRING), S.ProtoField(2, S.PB_INT32)]
    frames = []
    for flag in range(256):
        body = TP.T(1, 2) + b"\x03abc" + TP.T(2, 0) + _varint(flag)
        frames += [bytes([flag]) + len(body).to_bytes(4, "big") + body]
        frames += [b"\x00" + (len(body) + d).to_bytes(4, "big") + body for d in (1, -1)] if flag % 16 == 0 else []
        frames += [_frame(body)[:flag % 5]] if flag % 8 == 0 else []
    cases.append(("headers", fields, frames, [_header_status(f) for f in frames]))
    # strings of 9 .. 70 KiB: their tiles are read from HBM; some end in an invalid byte
    fields = [S.ProtoField(1, S.PB_STRING), S.ProtoField(2, S.PB_BYTES), S.ProtoField(3, S.PB_INT64), S.ProtoField(2 ** 29 - 1, S.PB_STRING)]
    frames = []
    for k in range(48):
        s = ("é€x" * 24000)[:rnd.randint(9 * 1024, 70 * 1024) // 2].encode()
        s = s + (b"\xc3" if k % 7 == 3 else b"")
        body = TP.T(1, 2) + _varint(len(s)) + s + TP.T(3, 0) + _varint(k) + TP.T(2 ** 29 - 1, 2) + b"\x02ok"
        if k % 5 == 1:
            body = TP.T(2, 2) + _varint(len(s)) + s + body
        frames += [_frame(body), _frame(TP.T(1, 2) + b"\x01z")]
    cases.append(("long strings", fields, frames, [None] * len(frames)))
    return cases


def _rows_agree(fields, got, want):
    """row equality, except that a float / double NaN matches any NaN: python's float quiets a signalling NaN (0xff800800
    comes back as 0xffc00800), protobuf-go and the codecs keep the bits"""
    if got == want:
        return True
    if len(got) != len(want):
        return False
    pos = 0
    for f in fields:
        w = 8 if f.type in S.PB_64BIT else 4
        a, b = got[pos:pos + w], want[pos:pos + w]
        fmt = {S.PB_FLOAT: "<f", S.PB_DOUBLE: "<d"}.get(f.type)
        if a != b and not (fmt and all(math.isnan(struct.unpack(fmt, x)[0]) for x in (a, b))):
            return False
        pos += w
    return got[pos:] == want[pos:]


def check_flat_decode(label, fields, frames, want, rows, roff, meta):
    """python protobuf decides frames with a good header: rows it parses are the rows of its values, frames it refuses are
    BAD_PROTO or BAD_UTF8 with an empty row (a tenth varint byte above 1 aside)"""
    got = TP._rows(rows, roff)
    good = [i for i, w in enumerate(want) if w is None]
    py = TP._py_parse_rows(fields, [frames[i] for i in good])
    for i, p in zip(good, py):
        assert _header_status(frames[i]) is None, (label, i)
        if p is None or (meta[i] == BAD_PROTO and TP._has_overflowing_varint(frames[i][5:])):
            assert meta[i] in (BAD_PROTO, BAD_UTF8) and got[i] == b"", (label, i, frames[i].hex())
        else:
            assert meta[i] == OK and _rows_agree(fields, got[i], p), (label, i, frames[i].hex())
    for i, w in enumerate(want):
        if w is not None:
            assert meta[i] == w and got[i] == b"", (label, i, frames[i].hex(), meta[i])


def test_decoder_cases_three_ways():
    paths, n = [0, 0], 0
    for label, fields, frames, want in decoder_cases():
        raw, off = _pack(frames)
        rows, roff, meta = O.proto_decode(fields, raw, off)
        e_rows, e_off, e_meta = emu.proto_decode(fields, raw, off, 5)
        assert np.array_equal(e_meta, meta) and np.array_equal(e_off, roff + 5), label
        assert e_rows[5:int(e_off[-1])].tobytes() == rows[:int(roff[-1])].tobytes(), label
        check_flat_decode(label, fields, frames, want, rows, roff, meta)
        s, h = _tile_paths(off)
        paths[0] += s
        paths[1] += h
        n += len(frames)
    assert paths[0] > 0 and paths[1] > 0 and n >= 20000, (paths, n)


def _gpu_decoder(eng):
    n = 0
    for label, fields, frames, _ in decoder_cases():
        raw, off = _pack(frames)
        want = reference("dec", fields, raw, off)
        check_equal(gpu_run(eng, "dec", fields, raw, off, len(want[0]) + 16), want, "decoder " + label)
        n += len(frames)
    return "flat decoder: %d frames in %d launches equal to the oracle" % (n, len(decoder_cases()))


# ---------------------------------------------------------------------------------------------------------------
# 3. Hello: random bytes, random flags, lying length prefixes
# ---------------------------------------------------------------------------------------------------------------
def _hello_body(rnd):
    parts = [_soup_frag(rnd) for _ in range(rnd.choice([0, 0, 1, 2]))]
    for _ in range(rnd.choice([1, 1, 1, 2])):
        name = _text(rnd, rnd.choice([0, 1, 5, 16, 40, 200])).encode("utf-8", "surrogatepass")
        if rnd.random() < 0.05:
            name = rnd.randbytes(len(name))
        parts.insert(rnd.randrange(len(parts) + 1), b"\x0a" + _varint(len(name)) + name)
    return b"".join(parts)


@lru_cache(maxsize=None)
def hello_frames():
    rnd = random.Random(0x4E110)
    frames = []
    for _ in range(200000):
        r = rnd.random()
        if r < 0.5:
            m = rnd.randbytes(rnd.randint(0, 300) if rnd.random() < 0.03 else rnd.randint(0, 64))
        else:
            m = _hello_body(rnd)
            if r > 0.8:
                m = _mutate(rnd, m)
        flag = 0 if rnd.random() < 0.97 else rnd.randint(1, 255)
        n = len(m)
        if rnd.random() < 0.03:
            n = max(0, n + rnd.choice([-2, -1, 1, 2, 256, 1 << 24]))
        fr = bytes([flag]) + n.to_bytes(4, "big") + m
        frames.append(fr[:rnd.randint(0, 4)] if rnd.random() < 0.005 else fr)
    return frames


def test_hello_frames_three_ways():
    """oracle == device code (CPU) on the Hello campaign; python's HelloRequest / HelloResponse decide every frame with a
    good header"""
    frames = hello_frames()
    raw, off = _pack(frames)
    out, o, meta = O.grpc_hello(raw, off)
    e_out, e_off, e_meta = emu.grpc_hello(raw, off, 7)
    assert np.array_equal(e_meta, meta) and np.array_equal(e_off, o + 7)
    assert e_out[7:int(e_off[-1])].tobytes() == out[:int(o[-1])].tobytes()
    Req, Resp = TG._hello_classes()
    res = TP._frames(out, o)
    accepted = 0
    for i, fr in enumerate(frames):
        h = _header_status(fr)
        if h is not None:
            assert meta[i] == h and res[i] == b"", (i, fr.hex())
            continue
        try:
            req, ok = Req.FromString(fr[5:]), True
        except Exception:
            ok = False
        if ok and meta[i] == BAD_PROTO and TP._has_overflowing_varint(fr[5:]):
            continue
        assert ok == (meta[i] == OK), (i, fr.hex(), meta[i])
        if ok:
            want = Resp(message="Hello %s!" % (req.name or "World")).SerializeToString()
            assert res[i] == b"\x00" + len(want).to_bytes(4, "big") + want, (i, fr.hex())
            accepted += 1
    assert accepted > 30000 and (meta == BAD_UTF8).any() and (meta == COMPRESSED).any()


def _gpu_hello(eng):
    raw, off = _pack(hello_frames())
    want = reference("hello", None, raw, off)
    check_equal(gpu_run(eng, "hello", None, raw, off, len(want[0]) + 16), want, "hello")
    return "hello: %d frames equal to the oracle (%d accepted)" % (len(off) - 1, int((want[2] == OK).sum()))


# ---------------------------------------------------------------------------------------------------------------
# 4. nested encoder: random types with tags 70000 and 2^29-1, invalid UTF-8 at every level, truncated rows, huge counts
# ---------------------------------------------------------------------------------------------------------------
def _with_field(fields, f):
    if any(x.number == f.number for x in fields):
        return fields
    return sorted(fields + [f], key=lambda x: x.number)


def _nested_types(rnd):
    msgs = H.rand_types(rnd)
    msgs[0] = _with_field(msgs[0], F(70000, rnd.choice(H.SCALARS), rnd.random() < 0.5))
    msgs[-1] = _with_field(msgs[-1], F(2 ** 29 - 1, rnd.choice([S.PB_STRING, S.PB_SINT64, S.PB_FIXED32]), rnd.random() < 0.5))
    return msgs


def _string_slots(msgs, m, value, depth, out):
    """(depth, container, index) of every string in a value"""
    for k, f in enumerate(msgs[m]):
        v = value[k]
        if f.type == S.PB_STRING:
            if f.repeated:
                out += [(depth, v, j) for j in range(len(v))]
            else:
                out.append((depth, value, k))
        elif f.type == S.PB_MESSAGE:
            for e in (v if f.repeated else [v] if v is not None else []):
                _string_slots(msgs, f.msg, e, depth + 1, out)
    return out


def _fixed_words(msgs, m):
    w = 0
    for f in msgs[m]:
        w += 1 if f.repeated or f.type == S.PB_MAP else 1 + _fixed_words(msgs, f.msg) if f.type == S.PB_MESSAGE else 2 if f.type in S.PB_64BIT else 1
    return w


NESTED_ROWS = 1500       # generated rows per type in nested_encoder_cases; the malformed rows follow them
# four levels, strings at every one, the widest tags at the bottom
DEEP_STRINGS = [[F(1, S.PB_STRING), F(2, S.PB_MESSAGE, True, 1), F(70000, S.PB_UINT64)],
                [F(1, S.PB_STRING, True), F(3, S.PB_MESSAGE, False, 2)],
                [F(5, S.PB_STRING), F(6, S.PB_MESSAGE, True, 3)],
                [F(1, S.PB_SINT32), F(262144, S.PB_BYTES), F(2 ** 29 - 1, S.PB_STRING, True)]]


@lru_cache(maxsize=None)
def nested_encoder_cases():
    """[(msgs, rows, off, values, depths)]: values[i] the row's value when python must agree (None otherwise); depths: the
    nesting levels at which a string was made invalid"""
    rnd = random.Random(0x7E57)
    cases = []
    for k in range(8):
        msgs = DEEP_STRINGS if k == 0 else _nested_types(rnd)
        values = [H.rand_value(rnd, msgs, 0) for _ in range(NESTED_ROWS)]
        depths = set()
        py = list(values)
        for i in range(0, len(values), 9):           # one string made invalid UTF-8
            slots = _string_slots(msgs, 0, values[i], 0, [])
            if slots:
                d, c, j = rnd.choice(slots)
                c[j] = rnd.choice([b"\xff", b"a\xc3", b"\xed\xa0\x80"])
                depths.add(d)
                py[i] = None
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        blobs = [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]
        # malformed rows: truncations (every 4th byte) of ten rows, and counts of the root's repeated fields past the row
        for i in range(10):
            r0 = blobs[i * 17]
            blobs += [r0[:k] for k in range(0, len(r0), 4)]
        w = 0                                        # the field's first word in the root's fixed part
        for f in msgs[0]:
            if f.repeated:
                for big in (0x00FFFFFF, 0x40000000, 0xFFFFFFFF):
                    r0 = bytearray(blobs[rnd.randrange(len(values))])
                    r0[4 * w:4 * w + 4] = big.to_bytes(4, "little")
                    blobs.append(bytes(r0))
            w += _fixed_words([[f]], 0) if f.type != S.PB_MESSAGE or f.repeated else 1 + _fixed_words(msgs, f.msg)
        rows, off = _assemble(blobs)
        cases.append((msgs, rows, off, py + [None] * (len(blobs) - len(values)), frozenset(depths)))
    return cases


def test_nested_encoder_cases_three_ways():
    depths = set()
    for msgs, rows, off, values, d in nested_encoder_cases():
        out, o, meta = O.proto_encode_nested(msgs, 0, rows, off)
        for mis in (0, 3):
            e_out, e_off, e_meta = emu.proto_encode_nested(msgs, 0, rows, off, mis)
            assert np.array_equal(e_meta, meta) and np.array_equal(e_off, o + mis)
            assert e_out[mis:int(e_off[-1])].tobytes() == out[:int(o[-1])].tobytes()
        idx = [i for i, v in enumerate(values) if v is not None]
        py = H.py_frames(msgs, 0, [values[i] for i in idx])
        fr = H.frames_of(out, o)
        for i, p in zip(idx, py):
            assert meta[i] == OK and fr[i] == p, i
        poisoned = np.array([v is None for v in values[:NESTED_ROWS]])
        assert (meta[:NESTED_ROWS][poisoned] == BAD_UTF8).all()
        assert (meta[NESTED_ROWS:] == BAD_ROW).sum() >= (len(meta) - NESTED_ROWS) // 2
        depths |= d
    assert depths == {0, 1, 2, 3}, depths


def _gpu_nested_encoder(eng):
    n = 0
    for msgs, rows, off, _, _ in nested_encoder_cases():
        want = reference("nenc", (msgs, 0), rows, off)
        check_equal(gpu_run(eng, "nenc", (msgs, 0), rows, off, len(want[0]) + 16), want, "nested encoder")
        n += len(off) - 1
    return "nested encoder: %d rows equal to the oracle" % n


# ---------------------------------------------------------------------------------------------------------------
# 5. nested decoder, map-free and with map fields: hostile and non-canonical lists, four-way mutations, 64 / 65 entries
# ---------------------------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def nested_decoder_cases():
    """[(label, msgs, frames)] map-free (oracle) and with map fields (model)"""
    rnd = random.Random(0xD0D0)
    cases = [("hostile", H.HOSTILE_MSGS, [_frame(b) for b in H.HOSTILE_BODIES] + H.HOSTILE_HEADER_FRAMES)]
    for k in range(12):
        msgs = _nested_types(rnd)
        rows, off = S.pack_proto_nested_rows(msgs, 0, [H.rand_value(rnd, msgs, 0) for _ in range(400)])
        out, o, _ = O.proto_encode_nested(msgs, 0, rows, off)
        frames = [fr if i % 4 == 0 else _frame(_mutate(rnd, fr[5:])) for i, fr in enumerate(H.frames_of(out, o))]
        cases.append(("mutated %d" % k, msgs, frames))
    entries = [b"".join(H._A(b"k%03d" % k, H._V1) for k in range(n)) for n in (64, 65)]
    cases.append(("maps: non-canonical", H.NONCANON_MSGS, [_frame(b) for b in H.NONCANON_OK + H.NONCANON_DEFER + H.NONCANON_BAD + entries]))
    for k in range(6):
        msgs = H.rand_map_types(rnd)
        rows, off = S.pack_proto_nested_rows(msgs, 0, [H.rand_map_value(rnd, msgs, 0) for _ in range(300)])
        frames, _ = M.encode(msgs, 0, rows, off)
        frames = [fr if i % 4 == 0 else _frame(_mutate(rnd, fr[5:])) for i, fr in enumerate(frames)]
        cases.append(("maps: mutated %d" % k, msgs, frames))
    return cases


def test_nested_decoder_cases_three_ways():
    """map-free: oracle == device code (CPU), python protobuf agrees on which frames parse and on their rows; with map
    fields: model == device code (CPU), pure-python protobuf agrees; 64 entries of one map field decode, 65 are DEFER"""
    for label, msgs, frames in nested_decoder_cases():
        if label.startswith("maps"):
            rows, meta = H.decode_model_emu(msgs, 0, frames)
            H.check_python_parse(msgs, 0, frames, rows, meta)
            if label == "maps: non-canonical":
                assert meta[-2:] == [OK, DEFER]
        else:
            H.decode_three_ways(msgs, 0, frames)


def _gpu_nested_decoder(eng):
    n = 0
    for label, msgs, frames in nested_decoder_cases():
        raw, off = _pack(frames)
        want = reference("ndec", (msgs, 0), raw, off)
        check_equal(gpu_run(eng, "ndec", (msgs, 0), raw, off, len(want[0]) + 16), want, "nested decoder " + label)
        n += len(frames)
    return "nested decoder: %d frames equal to the oracle / the model" % n


# ---------------------------------------------------------------------------------------------------------------
# 6. exact output capacities, every entry point and kernel instance
# ---------------------------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def capacity_inputs():
    """[(label, kind, spec, data, off)]: about a thousand items each, several tiles"""
    rnd = random.Random(0xCA9)
    h_raw, h_off = TG._frames(TG.EDGE_MSGS * 36)
    fields, msgs = TP._bulk(1000, seed=3)
    rows, off = S.pack_proto_rows(fields, msgs)
    out, o, _ = O.proto_encode(fields, rows, off)
    f_raw, f_off = _pack([fr for fr in TP._frames(out, o)])
    values = [H.rand_value(rnd, H.MSGS, 0) for _ in range(1000)]
    for v in values[7::50]:
        v[2] = b"\xff"                                  # PAGE.3, a string: BAD_UTF8, no frame
    n_rows, n_off = S.pack_proto_nested_rows(H.MSGS, 0, values)
    out, o, _ = O.proto_encode_nested(H.MSGS, 0, n_rows, n_off)
    nf_raw, nf_off = _pack(H.frames_of(out, o))
    mm = H.rand_map_types(rnd)
    values = [H.rand_map_value(rnd, mm, 0) for _ in range(800)]
    for v in values[::23]:                              # a duplicate key: BAD_ROW, no frame
        k = next((j for j, f in enumerate(mm[0]) if f.type == S.PB_MAP and v[j]), None)
        if k is not None:
            key = next(iter(v[k]))
            v[k] = [(key, v[k][key])] * 2
    m_rows, m_off = S.pack_proto_nested_rows(mm, 0, values)
    frames, _ = M.encode(mm, 0, m_rows, m_off)
    mf_raw, mf_off = _pack(frames)
    return [("hello", "hello", None, h_raw, h_off), ("flat encoder", "enc", fields, rows, off), ("flat decoder", "dec", fields, f_raw, f_off),
            ("nested encoder", "nenc", (H.MSGS, 0), n_rows, n_off), ("nested decoder", "ndec", (H.MSGS, 0), nf_raw, nf_off),
            ("maps encoder", "nenc", (mm, 0), m_rows, m_off), ("maps decoder", "ndec", (mm, 0), mf_raw, mf_off)]


def test_capacity_inputs_span_tiles():
    for label, kind, spec, data, off in capacity_inputs():
        w_out, w_off, w_meta = reference(kind, spec, data, off)
        n = len(off) - 1
        assert n > 4 * T and int(w_off[4 * T]) > int(w_off[3 * T]) > 0, label
        assert (w_meta == OK).any() and (w_meta != OK).any(), label


def check_short(got, want, cap, what):
    """a launch with out_cap < the total: the flag is raised; d_out_off and d_meta hold every offset and status as with room
    enough; the tiles before the first one that does not fit are written, nothing at or past that tile's first byte"""
    out, off, meta, ovf = got
    w_out, w_off, w_meta = want
    n = len(w_off) - 1
    assert ovf, what + ": no overflow flag"
    assert _first(off, w_off) is None and _first(meta, w_meta) is None, what + ": offsets / statuses differ after the overflow"
    k = next(t for t in range(0, n, T) if int(w_off[min(n, t + T)]) > cap)
    kept = int(w_off[k])
    assert out[:kept].tobytes() == w_out[:kept], what + ": the tiles that fit differ"
    assert (out[kept:] == CANARY).all(), what + ": bytes written at or past the first tile that does not fit"


def _gpu_capacity(eng):
    runs = 0
    for label, kind, spec, data, off in capacity_inputs():
        want = reference(kind, spec, data, off)
        total = int(want[1][-1])
        check_equal(gpu_run(eng, kind, spec, data, off, total), want, label + " (cap = total)")
        check_short(gpu_run(eng, kind, spec, data, off, total - 1), want, total - 1, label + " (cap = total - 1)")
        mid = int(want[1][3 * T]) + (int(want[1][4 * T]) - int(want[1][3 * T])) // 2
        check_short(gpu_run(eng, kind, spec, data, off, mid), want, mid, label + " (cap inside tile 3)")
        runs += 3
    return "capacity: %d launches at exact and short capacities" % runs


# ---------------------------------------------------------------------------------------------------------------
# the GPU campaigns, each in a process of its own
# ---------------------------------------------------------------------------------------------------------------
CAMPAIGNS = {"encoder": _gpu_encoder, "decoder": _gpu_decoder, "hello": _gpu_hello, "nested_encoder": _gpu_nested_encoder,
             "nested_decoder": _gpu_nested_decoder, "capacity": _gpu_capacity}


def _gpu_main(name):
    import time
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    t0 = time.perf_counter()
    eng = Engine(Table(synth.config1_spec()), 0)
    msg = CAMPAIGNS[name](eng)
    eng.close()
    print("%s (%.1f s)" % (msg, time.perf_counter() - t0))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CAMPAIGNS))
def test_gpu_campaign(name):
    r = subprocess.run([sys.executable, "-c", "import tests.test_gpu_proto_codecs as t; t._gpu_main(%r)" % name], cwd=ROOT_DIR,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip())
