"""gofr_proto_encode_nested_device — the proto3 encoder for message types with nested and repeated fields
(SURVEY.md §8f rank 4 widened; VERDICT r01 "missing" item 6).

Reference behaviour: proto.Marshal of the message a unary handler returns + grpc-go's 5-byte length prefix
(examples/grpc-server/grpc/hello_grpc.pb.go:73-89; protobuf-go v1.32.0, grpc-go v1.60.1).  Three statements compared:
  python google.protobuf with descriptors built at run time (independent implementation, deterministic field order)
  the oracle (oracle/orc_proto_nested.c: recursive, a message marshalled into its own buffer)
  the device code (proto_nested_device.cuh: explicit stack, nested lengths from a sizing walk) on the CPU via tests/emu,
  and the CUDA kernel with -m gpu."""
import random
import struct

import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200 import _abi
from tests import oracle as O
from tests.emu import emu

SCALARS = [S.PB_DOUBLE, S.PB_FLOAT, S.PB_INT64, S.PB_UINT64, S.PB_INT32, S.PB_FIXED64, S.PB_FIXED32, S.PB_BOOL, S.PB_STRING,
           S.PB_BYTES, S.PB_UINT32, S.PB_SFIXED32, S.PB_SFIXED64, S.PB_SINT32, S.PB_SINT64]
F = S.ProtoNField


def _py_classes(msgs):
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fdp = descriptor_pb2.FileDescriptorProto(name="n.proto", package="n", syntax="proto3")
    for m, fields in enumerate(msgs):
        mt = fdp.message_type.add(name="M%d" % m)
        for f in fields:
            # an enum field encodes exactly like int32 (and would need an enum type here)
            kw = dict(name="f%d" % f.number, number=f.number, type=S.PB_INT32 if f.type == S.PB_ENUM else f.type, label=3 if f.repeated else 1)
            if f.type == S.PB_MESSAGE:
                kw["type_name"] = ".n.M%d" % f.msg
            mt.field.add(**kw)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return [message_factory.GetMessageClass(pool.FindMessageTypeByName("n.M%d" % m)) for m in range(len(msgs))]


def _py_fill(classes, msgs, m, value):
    obj = classes[m]()
    for f, v in zip(msgs[m], value):
        name = "f%d" % f.number
        conv = (lambda x: x.decode("utf-8") if isinstance(x, (bytes, bytearray)) else x) if f.type == S.PB_STRING else (lambda x: x)
        if f.repeated:
            if f.type == S.PB_MESSAGE:
                for e in v:
                    getattr(obj, name).add().CopyFrom(_py_fill(classes, msgs, f.msg, e))
            else:
                getattr(obj, name).extend([conv(e) for e in v])
        elif f.type == S.PB_MESSAGE:
            if v is not None:
                getattr(obj, name).CopyFrom(_py_fill(classes, msgs, f.msg, v))
                getattr(obj, name).SetInParent()
        else:
            setattr(obj, name, conv(v))
    return obj


def _py_frames(msgs, root, values):
    classes = _py_classes(msgs)
    out = []
    for v in values:
        body = _py_fill(classes, msgs, root, v).SerializeToString(deterministic=True)
        out.append(b"\x00" + len(body).to_bytes(4, "big") + body)
    return out


def _frames(out, off):
    return [out[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def _three_ways(msgs, root, values):
    rows, off = S.pack_proto_nested_rows(msgs, root, values)
    o_out, o_off, o_meta = O.proto_encode_nested(msgs, root, rows, off)
    assert not o_meta.any(), o_meta
    want = _py_frames(msgs, root, values)
    got = _frames(o_out, o_off)
    for i in range(len(values)):
        assert got[i] == want[i], (i, values[i], got[i].hex(), want[i].hex())
    for mis in (0, 3):
        e_out, e_off, e_meta = emu.proto_encode_nested(msgs, root, rows, off, mis)
        assert not e_meta.any() and np.array_equal(e_off, o_off + mis)
        assert e_out[mis:int(e_off[-1])].tobytes() == o_out[:int(o_off[-1])].tobytes()
    return rows, off, o_out, o_off


# the shapes of a typical API: a page of items with tags, an optional owner, per-item attributes and histograms
ITEM = [F(1, S.PB_INT64), F(2, S.PB_STRING), F(3, S.PB_STRING, True), F(4, S.PB_DOUBLE, True), F(5, S.PB_MESSAGE, False, 2), F(7, S.PB_SINT32, True)]
PAGE = [F(1, S.PB_MESSAGE, True, 1), F(2, S.PB_UINT32), F(3, S.PB_STRING), F(15, S.PB_MESSAGE, False, 2), F(16, S.PB_BOOL, True), F(2047, S.PB_FIXED64, True)]
OWNER = [F(1, S.PB_STRING), F(2, S.PB_BYTES, True), F(3, S.PB_MESSAGE, False, 3)]
GEO = [F(1, S.PB_FLOAT), F(2, S.PB_FLOAT), F(9, S.PB_ENUM, True)]
MSGS = [PAGE, ITEM, OWNER, GEO]


def test_known_answers_and_python_protobuf():
    geo = [1.5, -2.25, [1, 0, -1]]
    owner = ["ann", [b"\x00\xff", b""], geo]
    item1 = [7, "first", ["a", "", "bb"], [0.0, -0.0, 1e300], owner, [-1, 0, 1, 2 ** 31 - 1, -2 ** 31]]
    item2 = [0, "", [], [], None, []]                                   # an element that encodes to nothing: tag + length 0
    page = [[item1, item2], 2, "next", [ "", [], None], [True, False, True], [1, 2 ** 64 - 1]]
    empty = [[], 0, "", None, [], []]
    rows, off, out, o = _three_ways(MSGS, 0, [page, empty, [[item2] * 3, 0, "", None, [], []]])
    fr = _frames(out, o)
    assert fr[1] == b"\x00\x00\x00\x00\x00"                             # nothing set: an empty message, still a frame
    assert fr[2] == b"\x00\x00\x00\x00\x06" + b"\x0a\x00" * 3           # three empty items: tag 1/LEN + length 0 each
    # a set but empty singular message is written (field 15 = tag 0x7a, length 0); packed bools; packed fixed64 under a
    # two-byte field number
    assert b"\x7a\x00" in fr[0] and b"\x82\x01\x03\x01\x00\x01" in fr[0]
    assert (2047 << 3 | 2).to_bytes(2, "little") != b"" and bytes([0xFA, 0x7F, 0x10]) in fr[0]


def _rand_types(rnd):
    """up to 5 acyclic message types (type m may use types > m), at most 4 levels deep from the root"""
    n = rnd.randint(1, 5)
    msgs = []
    depth_below = [1] * n
    for m in reversed(range(n)):
        fields, numbers = [], sorted(rnd.sample(range(1, 40), rnd.randint(1, 6)) + ([rnd.choice([100, 2047, 2048, 70000])] if rnd.random() < 0.3 else []))
        for num in sorted(set(numbers)):
            usable = [k for k in range(m + 1, n) if 1 + depth_below[k] <= 4 - 0]
            if usable and rnd.random() < 0.35:
                k = rnd.choice(usable)
                fields.append(F(num, S.PB_MESSAGE, rnd.random() < 0.5, k))
                depth_below[m] = max(depth_below[m], 1 + depth_below[k])
            else:
                fields.append(F(num, rnd.choice(SCALARS), rnd.random() < 0.4))
        msgs.insert(0, fields)
    # the indices used above refer to final positions m+1..n-1: types were built back to front into position m
    if depth_below[0] > 4:
        return _rand_types(rnd)
    return msgs


def _rand_scalar(rnd, t):
    if t == S.PB_DOUBLE:
        return rnd.choice([0.0, -0.0, 1.5, -1e300, 5e-324, float(rnd.randint(-5, 5))])
    if t == S.PB_FLOAT:
        return rnd.choice([0.0, -0.0, 1.5, -2.25, 3.0e38, float(rnd.randint(-5, 5))])
    if t in (S.PB_INT64, S.PB_SINT64, S.PB_SFIXED64):
        return rnd.choice([0, 1, -1, 2 ** 63 - 1, -2 ** 63, rnd.randint(-10 ** 6, 10 ** 6)])
    if t in (S.PB_UINT64, S.PB_FIXED64):
        return rnd.choice([0, 1, 2 ** 64 - 1, 127, 128, rnd.randint(0, 10 ** 12)])
    if t in (S.PB_INT32, S.PB_SINT32, S.PB_SFIXED32, S.PB_ENUM):
        return rnd.choice([0, 1, -1, 2 ** 31 - 1, -2 ** 31, rnd.randint(-1000, 1000)])
    if t in (S.PB_UINT32, S.PB_FIXED32):
        return rnd.choice([0, 1, 2 ** 32 - 1, 16383, 16384])
    if t == S.PB_BOOL:
        return rnd.random() < 0.5
    if t == S.PB_STRING:
        return rnd.choice(["", "a", "héllo", "x" * 130, "日本", "tab\t"])
    return rnd.choice([b"", b"\x00", b"\xff\xfe", b"b" * 200])


def _rand_value(rnd, msgs, m, depth=0):
    v = []
    for f in msgs[m]:
        one = (lambda: _rand_value(rnd, msgs, f.msg, depth + 1)) if f.type == S.PB_MESSAGE else (lambda: _rand_scalar(rnd, f.type))
        if f.repeated:
            v.append([one() for _ in range(rnd.choice([0, 0, 1, 2, 5]))])
        elif f.type == S.PB_MESSAGE:
            v.append(None if rnd.random() < 0.4 else one())
        else:
            v.append(one())
    return v


@pytest.mark.parametrize("seed", range(25))
def test_random_types_three_ways(seed):
    rnd = random.Random(500 + seed)
    msgs = _rand_types(rnd)
    values = [_rand_value(rnd, msgs, 0) for _ in range(60)]
    _three_ways(msgs, 0, values)


def test_invalid_utf8_and_malformed_rows():
    msgs = [[F(1, S.PB_STRING), F(2, S.PB_MESSAGE, True, 1), F(3, S.PB_INT32, True)], [F(1, S.PB_STRING, True), F(2, S.PB_BYTES)]]
    good = ["ok", [[["a", "b"], b"\xff"]], [1, 2]]
    vals = [good, [b"\xff", [], []], ["ok", [[[b"\xc3"], b""]], []], ["fine é", [[[], b""]] * 2, [0]]]
    rows, off = S.pack_proto_nested_rows(msgs, 0, vals)
    out, o, meta = O.proto_encode_nested(msgs, 0, rows, off)
    assert list(meta) == [S.GRPC_OK, S.GRPC_BAD_UTF8, S.GRPC_BAD_UTF8, S.GRPC_OK]
    # truncations of a valid row and counts that promise more than the row holds
    r0 = rows[int(off[0]):int(off[1])].tobytes()
    cut = [r0[:k] + b"\0" * ((-k) % 4) for k in range(0, len(r0), 3)]
    huge = (5).to_bytes(4, "little") + (0x00FFFFFF).to_bytes(4, "little") + (0).to_bytes(4, "little") + b"abcde" + b"\0" * 3
    huge2 = (0).to_bytes(4, "little") + (0).to_bytes(4, "little") + (0x40000000).to_bytes(4, "little")
    blobs = cut + [huge, huge2]
    body, offs = bytearray(), [0]
    for b in blobs:
        body += b
        offs.append(len(body))
    rows2 = np.frombuffer(bytes(body) + b"\0" * 16, dtype=np.uint8).copy()
    off2 = np.array(offs, dtype=np.uint32)
    out, o, meta = O.proto_encode_nested(msgs, 0, rows2, off2)
    e_out, e_off, e_meta = emu.proto_encode_nested(msgs, 0, rows2, off2)
    assert np.array_equal(meta, e_meta) and np.array_equal(o, e_off) and out[:int(o[-1])].tobytes() == e_out[:int(o[-1])].tobytes()
    assert (meta == S.GRPC_BAD_ROW).sum() >= len(cut) // 2 and meta[-1] == S.GRPC_BAD_ROW and meta[-2] == S.GRPC_BAD_ROW


def test_descriptions_outside_the_limits_are_refused():
    L = _abi.lib()

    def describe(msgs, root=0):
        nm, nf, k = S.proto_nested_tables(msgs)
        return L.gofr_proto_nested_describe(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None, 0)
    CAP = 7   # GOFR_ERR_CAPACITY: "valid, but no room to write the descriptor"
    assert describe(MSGS) == CAP
    assert describe([[F(1, S.PB_MESSAGE, False, 0)]]) != CAP                                   # recursive type
    assert describe([[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MESSAGE, True, 0)]]) != CAP    # mutually recursive
    assert describe([[F(2, S.PB_INT32), F(1, S.PB_INT32)]]) != CAP                             # not in field-number order
    assert describe([[F(1, S.PB_MESSAGE, False, 3)]]) != CAP                                   # unknown message type
    assert describe([[F(1, 10)]]) != CAP                                                       # TYPE_GROUP
    assert describe([[F(0, S.PB_INT32)]]) != CAP and describe([[F(19500, S.PB_INT32)]]) != CAP  # reserved numbers
    chain = [[F(1, S.PB_MESSAGE, False, m + 1)] for m in range(4)] + [[F(1, S.PB_INT32)]]
    assert describe(chain) != CAP and describe(chain[1:4] + [[F(1, S.PB_INT32)]]) != CAP - 99  # 5 levels: too deep
    ok4 = [[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MESSAGE, False, 2)], [F(1, S.PB_MESSAGE, False, 3)], [F(1, S.PB_INT32)]]
    assert describe(ok4) == CAP


@pytest.mark.gpu
def test_gpu_matches_oracle():
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(77)
    eng = Engine(Table(synth.config1_spec()), 0)
    for msgs in (MSGS, _rand_types(rnd), _rand_types(rnd)):
        values = [_rand_value(rnd, msgs, 0) for _ in range(5000)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        o_out, o_off, o_meta = O.proto_encode_nested(msgs, 0, rows, off)
        d_out, d_off, d_meta = eng.proto_encode_nested_device(msgs, 0, rows, off)
        torch.cuda.synchronize()
        assert np.array_equal(d_off.cpu().numpy().view(np.uint32), o_off)
        assert np.array_equal(d_meta.cpu().numpy().view(np.uint32), o_meta)
        assert d_out[:int(o_off[-1])].cpu().numpy().tobytes() == o_out[:int(o_off[-1])].tobytes()
    eng.close()


# ---------------------------------------------------------------------------------------------------------------
# the other direction: frames -> rows (gofr_proto_decode_nested_device)
# ---------------------------------------------------------------------------------------------------------------
def _py_to_value(msgs, m, obj):
    """the value list pack_proto_nested_rows takes, from a parsed python protobuf message"""
    v = []
    for f in msgs[m]:
        x = getattr(obj, "f%d" % f.number)
        conv = (lambda e: e.encode("utf-8")) if f.type == S.PB_STRING else (lambda e: e)
        if f.repeated:
            v.append([_py_to_value(msgs, f.msg, e) for e in x] if f.type == S.PB_MESSAGE else [conv(e) for e in x])
        elif f.type == S.PB_MESSAGE:
            v.append(_py_to_value(msgs, f.msg, x) if obj.HasField("f%d" % f.number) else None)
        else:
            v.append(conv(x))
    return v


def _frame(body: bytes) -> bytes:
    return b"\x00" + len(body).to_bytes(4, "big") + body


def _pack_frames(frames):
    blob, offs = bytearray(), [0]
    for fr in frames:
        blob += fr
        offs.append(len(blob))
    return np.frombuffer(bytes(blob) + b"\0" * 16, dtype=np.uint8).copy(), np.array(offs, dtype=np.uint32)


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _has_overlong_varint(body: bytes) -> bool:
    run = 0
    for b in body:
        if b >= 0x80:
            run += 1
        else:
            if run >= 9 and b > 1:
                return True
            run = 0
        if run >= 10:
            return True
    return False


def _decode_three_ways(msgs, root, frames):
    """oracle == device code on everything; python protobuf decides what the rows of well-formed frames must be"""
    raw, off = _pack_frames(frames)
    o_rows, o_off, o_meta = O.proto_decode_nested(msgs, root, raw, off)
    e_rows, e_off, e_meta = emu.proto_decode_nested(msgs, root, raw, off)
    assert np.array_equal(o_meta, e_meta), (o_meta, e_meta)
    assert np.array_equal(o_off, e_off)
    assert o_rows[:int(o_off[-1])].tobytes() == e_rows[:int(o_off[-1])].tobytes()
    classes = _py_classes(msgs)
    from google.protobuf.message import DecodeError
    for i, fr in enumerate(frames):
        body = fr[5:]
        try:
            obj = classes[root]()
            obj.ParseFromString(body)
            ok = True
        except DecodeError:
            ok = False
        if o_meta[i] in (S.GRPC_COMPRESSED, S.GRPC_BAD_LENGTH, S.GRPC_DEFER):
            continue
        if ok and o_meta[i] == S.GRPC_BAD_PROTO and _has_overlong_varint(body):
            continue      # protowire.ConsumeVarint refuses a tenth byte above 1; upb silently truncates it
        assert ok == (o_meta[i] == S.GRPC_OK), (i, fr.hex(), o_meta[i], ok)
        if ok:
            want, _ = S.pack_proto_nested_rows(msgs, root, [_py_to_value(msgs, root, obj)])
            got = o_rows[int(o_off[i]):int(o_off[i + 1])].tobytes()
            assert got == want[:len(got)].tobytes() and len(got) == (len(want) - 8 + 3) // 4 * 4, (i, fr.hex())
    return o_rows, o_off, o_meta


def test_decode_canonical_frames_round_trip():
    """decode(encode(row)) == row, and python protobuf parses the frames to the same values"""
    rnd = random.Random(9)
    for msgs in (MSGS, _rand_types(rnd), _rand_types(rnd), _rand_types(rnd)):
        values = [_rand_value(rnd, msgs, 0) for _ in range(80)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        out, o, meta = O.proto_encode_nested(msgs, 0, rows, off)
        frames = _frames(out, o)
        d_rows, d_off, d_meta = _decode_three_ways(msgs, 0, frames)
        assert not d_meta.any()
        for i in range(len(values)):
            a = rows[int(off[i]):int(off[i + 1])].tobytes()
            b = d_rows[int(d_off[i]):int(d_off[i + 1])].tobytes()
            # -0.0 and absent look the same on the wire only for... nothing: the encoder writes -0.0, so rows match exactly
            assert a == b, (i, values[i])


# message types and frames, well-formed but not canonical, or hostile: statuses as test_decode_noncanonical_and_hostile_frames
# states them (the singular message sent twice is DEFER; the four header frames come last)
HOSTILE_MSGS = [[F(1, S.PB_INT32), F(2, S.PB_STRING), F(3, S.PB_SINT64, True), F(4, S.PB_MESSAGE, False, 1), F(5, S.PB_MESSAGE, True, 1),
                 F(6, S.PB_FIXED32, True), F(7, S.PB_STRING, True), F(8, S.PB_DOUBLE, True), F(9, S.PB_BOOL)],
                [F(1, S.PB_STRING), F(2, S.PB_UINT64, True), F(3, S.PB_BYTES)]]
_SUB = b"\x0a\x02hi" + b"\x10\x05" + b"\x12\x02\x01\x02" + b"\x1a\x01\xff"         # name, unpacked + packed uint64, bytes
HOSTILE_BODIES = [
    b"",                                                           # nothing
    b"\x08\x01\x08\x02",                                           # singular scalar twice: last wins
    b"\x12\x01a\x12\x02bc",                                        # string twice: last wins
    b"\x18\x01\x18\x03" + b"\x1a\x02\x05\x07" + b"\x18\x09",       # repeated sint64: unpacked, packed, unpacked — wire order
    b"\x22" + _varint(len(_SUB)) + _SUB,                             # singular message
    b"\x2a\x00" + b"\x2a" + _varint(len(_SUB)) + _SUB + b"\x2a\x00",  # three elements, two empty
    b"\x35\x01\x00\x00\x00" + b"\x32\x08\x02\x00\x00\x00\x03\x00\x00\x00",  # fixed32 unpacked then packed
    b"\x3a\x00\x3a\x01x",                                          # repeated strings incl. an empty one
    b"\x42\x10" + struct.pack("<dd", 1.5, -0.0) + b"\x41" + struct.pack("<d", 2.5),  # doubles packed + unpacked
    b"\x48\x02",                                                   # bool from a varint that is not 0 / 1
    b"\x0d\x01\x00\x00\x00" + b"\x10\x07" + b"\xf8\x07\x01" + b"\x92\x03\x03abc",    # foreign wire types and unknown numbers: skipped
    b"\x0b\x08\x01\x13\x14\x0c" + b"\x08\x05",                      # unknown groups, nested, balanced
    b"\x22\x02\x0a\x00" + b"\x08\x03",                             # message with an explicit empty string
    b"\x22\x00\x22\x00",                                           # singular message twice: protobuf-go merges -> DEFER
    b"\x2a\x04\x22\x02\x08\x01",                                   # element with fields the sub-message does not know
    # malformed
    b"\x08", b"\x12\x05ab", b"\x22\x03\x0a\x05a", b"\x0b\x08\x01", b"\x0c", b"\x32\x03\x01\x00\x00", b"\x1a\x02\x80\x80",
    b"\x00\x01", b"\x0e\x01", b"\x42\x07" + b"\0" * 7, b"\x2a\x02\x12\x05",
    # invalid UTF-8: top level, in an element, in an occurrence that is overwritten later
    b"\x12\x01\xff", b"\x2a\x03\x0a\x01\xc3", b"\x12\x01\xff\x12\x01a", b"\x3a\x02\xed\xa0",
]
HOSTILE_HEADER_FRAMES = [b"\x01\x00\x00\x00\x00", b"\x00\x00\x00\x00\x05\x08", b"\x00\x00", b"\x02\x00\x00\x00\x00"]   # header problems


def test_decode_noncanonical_and_hostile_frames():
    msgs = HOSTILE_MSGS
    frames = [_frame(b) for b in HOSTILE_BODIES] + HOSTILE_HEADER_FRAMES
    rows, off, meta = _decode_three_ways(msgs, 0, frames)
    assert list(meta[:15]) == [S.GRPC_OK] * 13 + [S.GRPC_DEFER, S.GRPC_OK]
    assert all(m == S.GRPC_BAD_PROTO for m in meta[15:26]) and all(m == S.GRPC_BAD_UTF8 for m in meta[26:30])
    assert list(meta[30:]) == [S.GRPC_COMPRESSED, S.GRPC_BAD_LENGTH, S.GRPC_BAD_LENGTH, S.GRPC_BAD_LENGTH]
    # spot values: wire order of the repeated sint64 (zigzag: 1 -> -1, 3 -> -2, 5 -> -3, 7 -> -4, 9 -> -5)
    r3 = rows[int(off[3]):int(off[4])].tobytes()
    fixed = 4 + 4 + 4 + (4 + 12) + 4 + 4 + 4 + 4 + 4
    assert struct.unpack_from("<I", r3, 8)[0] == 5 and struct.unpack_from("<5q", r3, fixed) == (-1, -2, -3, -4, -5)


@pytest.mark.parametrize("seed", range(20))
def test_decode_mutated_frames_device_code_equals_oracle(seed):
    """frames of random message types with bytes flipped, inserted and cut: oracle == device code on status and row, and
    python protobuf agrees on which frames parse (DEFER aside)"""
    rnd = random.Random(800 + seed)
    msgs = _rand_types(rnd)
    values = [_rand_value(rnd, msgs, 0) for _ in range(60)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    out, o, meta = O.proto_encode_nested(msgs, 0, rows, off)
    frames = []
    for fr in _frames(out, o):
        body = bytearray(fr[5:])
        for _ in range(rnd.randint(0, 2)):
            r = rnd.random()
            if body and r < 0.4:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            elif body and r < 0.6:
                del body[rnd.randrange(len(body)):]
            elif r < 0.8:
                p = rnd.randrange(len(body) + 1)
                body[p:p] = rnd.choice([b"\x08\x01", b"\x0b\x0c", b"\x12\x00", b"\xfa\x7f\x01\x00", b"\x0d\x00\x00\x00\x00", b"\x80"])
            else:      # reorder: move the tail in front (fields may arrive in any order)
                p = rnd.randrange(len(body) + 1)
                body = body[p:] + body[:p]
        frames.append(_frame(bytes(body)))
    _decode_three_ways(msgs, 0, frames)


def _gpu_decode_check():
    """the body of test_gpu_decode_matches_oracle (run in a process of its own)"""
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(78)
    eng = Engine(Table(synth.config1_spec()), 0)
    for msgs in (MSGS, _rand_types(rnd), _rand_types(rnd)):
        values = [_rand_value(rnd, msgs, 0) for _ in range(4000)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        out, o, _ = O.proto_encode_nested(msgs, 0, rows, off)
        frames = _frames(out, o)
        for i in range(0, len(frames), 7):          # every seventh frame damaged: statuses and empty rows must agree too
            body = bytearray(frames[i][5:])
            if body:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            frames[i] = _frame(bytes(body))
        raw, in_off = _pack_frames(frames)
        o_rows, o_off, o_meta = O.proto_decode_nested(msgs, 0, raw, in_off)
        d_rows, d_off, d_meta = eng.proto_decode_nested_device(msgs, 0, raw, in_off)
        torch.cuda.synchronize()
        assert np.array_equal(d_meta.cpu().numpy().view(np.uint32), o_meta)
        assert np.array_equal(d_off.cpu().numpy().view(np.uint32), o_off)
        assert d_rows[:int(o_off[-1])].cpu().numpy().tobytes() == o_rows[:int(o_off[-1])].tobytes()
        good = ~o_meta.astype(bool)                  # undamaged frames decode back to the rows they were encoded from
        for i in np.flatnonzero(good)[:500]:
            if i % 7:
                assert o_rows[int(o_off[i]):int(o_off[i + 1])].tobytes() == rows[int(off[i]):int(off[i + 1])].tobytes()
    eng.close()


@pytest.mark.gpu
def test_gpu_decode_matches_oracle():
    """gofr_proto_decode_nested_device on the GPU == oracle (statuses, offsets, rows) — in a child process, so that a fault
    in the kernel cannot leave a sticky CUDA error in the process the other GPU tests run in"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import tests.test_proto_nested as t; t._gpu_decode_check()"], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
