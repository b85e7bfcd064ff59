"""gofr_proto_encode_device — proto3 message encoder + gRPC framing (SURVEY.md §8f rank 4).

Reference behaviour: proto.Marshal of the message a unary handler returns, then grpc-go's 5-byte length prefix
(examples/grpc-server/grpc/hello_grpc.pb.go:73-89; protobuf-go v1.32.0, grpc-go v1.60.1).  Three layers:
  oracle (oracle/orc_proto.c)  vs  python google.protobuf with a descriptor built at run time (independent implementation)
  device code on the CPU (tests/emu) vs oracle, hypothesis-generated message types and values
  CUDA kernel vs oracle (-m gpu)"""
import struct

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from gofr_b200 import spec as S
from tests import oracle as O
from tests.emu import emu

ALL_TYPES = [S.PB_DOUBLE, S.PB_FLOAT, S.PB_INT64, S.PB_UINT64, S.PB_INT32, S.PB_FIXED64, S.PB_FIXED32, S.PB_BOOL, S.PB_STRING,
             S.PB_BYTES, S.PB_UINT32, S.PB_SFIXED32, S.PB_SFIXED64, S.PB_SINT32, S.PB_SINT64]   # PB_ENUM encodes like INT32


def _py_class(fields):
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fdp = descriptor_pb2.FileDescriptorProto(name="t.proto", package="t", syntax="proto3")
    m = fdp.message_type.add(name="M")
    for f in fields:
        m.field.add(name="f%d" % f.number, number=f.number, type=f.type, label=1)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("t.M"))


def _py_serialize(fields, values):
    cls = _py_class(fields)
    out = []
    for msg in values:
        kw = {}
        for f, v in zip(fields, msg):
            if f.type == S.PB_STRING:
                v = v.decode("utf-8") if isinstance(v, (bytes, bytearray)) else v
            kw["f%d" % f.number] = v
        body = cls(**kw).SerializeToString()
        out.append(b"\x00" + len(body).to_bytes(4, "big") + body)
    return out


def _frames(out, off):
    return [out[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def _hello_fields():
    return [S.ProtoField(1, S.PB_STRING)]      # HelloResponse{message = 1} — examples/grpc-server/grpc/hello.proto:8-10


def test_hello_response_matches_the_hello_path():
    """the fused Hello kernel's response is this encoder applied to HelloResponse{message: "Hello <name>!"}"""
    f = _hello_fields()
    msgs = [["Hello World!"], ["Hello gofr!"], ["Hello " + "n" * 200 + "!"], [""]]
    rows, off = S.pack_proto_rows(f, msgs)
    out, o, meta = O.proto_encode(f, rows, off)
    fr = _frames(out, o)
    assert fr[0] == b"\x00\x00\x00\x00\x0e\x0a\x0cHello World!"
    assert fr[3] == b"\x00\x00\x00\x00\x00"                       # zero value: empty message, still a frame
    assert fr == _py_serialize(f, msgs) and not meta.any()
    # the Hello oracle on the matching requests produces the same frames
    req = b"".join(b"\x00" + (2 + len(n)).to_bytes(4, "big") + b"\x0a" + bytes([len(n)]) + n for n in (b"", b"gofr"))
    roff = np.array([0, 7, 7 + 7 + 4], dtype=np.uint32)
    h_out, h_off, _ = O.grpc_hello(np.frombuffer(req, dtype=np.uint8), roff)
    assert _frames(h_out, h_off) == fr[:2]


def test_oracle_matches_python_protobuf_on_edge_values():
    f = [S.ProtoField(1, S.PB_INT32), S.ProtoField(2, S.PB_INT64), S.ProtoField(3, S.PB_UINT32), S.ProtoField(4, S.PB_UINT64),
         S.ProtoField(5, S.PB_SINT32), S.ProtoField(6, S.PB_SINT64), S.ProtoField(7, S.PB_BOOL), S.ProtoField(8, S.PB_FIXED32),
         S.ProtoField(9, S.PB_FIXED64), S.ProtoField(10, S.PB_SFIXED32), S.ProtoField(11, S.PB_SFIXED64), S.ProtoField(12, S.PB_FLOAT),
         S.ProtoField(13, S.PB_DOUBLE), S.ProtoField(14, S.PB_STRING), S.ProtoField(15, S.PB_BYTES), S.ProtoField(16, S.PB_STRING),
         S.ProtoField(2047, S.PB_INT32), S.ProtoField(2048, S.PB_BOOL), S.ProtoField(536870911, S.PB_UINT32)]
    msgs = [
        [0] * 6 + [False, 0, 0, 0, 0, 0.0, 0.0, "", b"", "", 0, False, 0],
        [-1, -1, 2**32 - 1, 2**64 - 1, -1, -1, True, 2**32 - 1, 2**64 - 1, -1, -1, -0.0, -0.0, "é", b"\xff\x00", "x", -2**31, True, 1],
        [2**31 - 1, 2**63 - 1, 127, 128, 2**31 - 1, 2**63 - 1, True, 1, 1, 1, 1, 1.5, 1e300, "a" * 127, b"b" * 128, "c" * 300, 1, False, 300],
        [-2**31, -2**63, 16383, 16384, -2**31, -2**63, False, 0, 0, -2**31, -2**63, float("inf"), float("nan"), " ", b"", "", 0, False, 0],
        [1, 1, 1, 1, 1, 1, True, 0, 0, 0, 0, 1e-45, 5e-324, "", b"\x00", "", 0, False, 0],
    ]
    rows, off = S.pack_proto_rows(f, msgs)
    out, o, meta = O.proto_encode(f, rows, off)
    assert not meta.any()
    got, want = _frames(out, o), _py_serialize(f, msgs)
    for i in range(len(msgs)):
        assert got[i] == want[i], i


def test_invalid_utf8_and_malformed_rows():
    f = [S.ProtoField(1, S.PB_STRING), S.ProtoField(2, S.PB_BYTES), S.ProtoField(3, S.PB_INT64)]
    rows, off = S.pack_proto_rows(f, [["ok", b"\xff", 1], [b"\xff", b"", 1], [b"\xed\xa0\x80", b"", 0], [b"\xf4\x90\x80\x80", b"x", 0],
                                      [b"\xc3", b"", 0], ["fine é€\U0001F600", b"", 2]])
    bad = bytearray(rows.tobytes())
    o2 = off.copy()
    # two more rows, hand made: a string longer than the row, a row shorter than its fixed part
    extra1 = (100).to_bytes(4, "little") + (0).to_bytes(4, "little") + (0).to_bytes(8, "little") + b"abcd"
    extra2 = b"\x01\x00\x00\x00"
    body = bytes(bad[:int(off[-1])]) + extra1 + extra2 + b"\0" * 8
    o2 = np.concatenate([off, np.array([int(off[-1]) + len(extra1), int(off[-1]) + len(extra1) + len(extra2)], dtype=np.uint32)])
    rows2 = np.frombuffer(body, dtype=np.uint8).copy()
    out, o, meta = O.proto_encode(f, rows2, o2)
    assert list(meta) == [S.GRPC_OK, S.GRPC_BAD_UTF8, S.GRPC_BAD_UTF8, S.GRPC_BAD_UTF8, S.GRPC_BAD_UTF8, S.GRPC_OK, S.GRPC_BAD_ROW,
                          S.GRPC_BAD_ROW]
    fr = _frames(out, o)
    assert all(fr[i] == b"" for i in (1, 2, 3, 4, 6, 7))
    for mis in (0, 5):
        e_out, e_off, e_meta = emu.proto_encode(f, rows2, o2, mis)
        assert np.array_equal(e_meta, meta) and np.array_equal(e_off, o + mis)
        assert e_out[mis:int(e_off[-1])].tobytes() == out[:int(o[-1])].tobytes()


_value = {
    S.PB_DOUBLE: st.floats(allow_nan=False, width=64) | st.sampled_from([0.0, -0.0, float("inf")]),
    S.PB_FLOAT: st.floats(allow_nan=False, width=32) | st.sampled_from([0.0, -0.0]),
    S.PB_INT64: st.integers(-2**63, 2**63 - 1) | st.sampled_from([0, 1, -1]), S.PB_UINT64: st.integers(0, 2**64 - 1) | st.just(0),
    S.PB_INT32: st.integers(-2**31, 2**31 - 1) | st.sampled_from([0, -1]), S.PB_FIXED64: st.integers(0, 2**64 - 1) | st.just(0),
    S.PB_FIXED32: st.integers(0, 2**32 - 1) | st.just(0), S.PB_BOOL: st.booleans(),
    S.PB_STRING: st.text(max_size=40) | st.text(alphabet="ab", min_size=100, max_size=300),
    S.PB_BYTES: st.binary(max_size=40), S.PB_UINT32: st.integers(0, 2**32 - 1) | st.just(0),
    S.PB_SFIXED32: st.integers(-2**31, 2**31 - 1), S.PB_SFIXED64: st.integers(-2**63, 2**63 - 1),
    S.PB_SINT32: st.integers(-2**31, 2**31 - 1) | st.just(0), S.PB_SINT64: st.integers(-2**63, 2**63 - 1) | st.just(0),
}


@st.composite
def _typed_messages(draw):
    nf = draw(st.integers(1, 10))
    numbers = sorted(draw(st.sets(st.integers(1, 40) | st.integers(2040, 2060) | st.integers(2**29 - 3, 2**29 - 1), min_size=nf, max_size=nf)))
    fields = [S.ProtoField(n, draw(st.sampled_from(ALL_TYPES))) for n in numbers]
    n_msgs = draw(st.integers(1, 6))
    msgs = [[draw(_value[f.type]) for f in fields] for _ in range(n_msgs)]
    return fields, msgs


@settings(max_examples=150, deadline=None)
@given(_typed_messages(), st.integers(0, 15))
def test_random_message_types_three_way(tm, mis):
    """python protobuf == oracle == device code (CPU emulation), for random flat proto3 message types and values"""
    fields, msgs = tm
    msgs = [[v.encode("utf-8", "surrogatepass").decode("utf-8", "replace") if isinstance(v, str) else v for v in m] for m in msgs]
    rows, off = S.pack_proto_rows(fields, msgs)
    out, o, meta = O.proto_encode(fields, rows, off)
    assert not meta.any()
    assert _frames(out, o) == _py_serialize(fields, msgs)
    e_out, e_off, e_meta = emu.proto_encode(fields, rows, off, mis)
    assert np.array_equal(e_meta, meta) and np.array_equal(e_off, o + mis)
    assert e_out[mis:int(e_off[-1])].tobytes() == out[:int(o[-1])].tobytes()


def _bulk(n, seed=7):
    rng = np.random.default_rng(seed)
    fields = [S.ProtoField(1, S.PB_STRING), S.ProtoField(2, S.PB_INT64), S.ProtoField(3, S.PB_SINT32), S.ProtoField(4, S.PB_BOOL),
              S.ProtoField(5, S.PB_DOUBLE), S.ProtoField(7, S.PB_BYTES), S.ProtoField(9, S.PB_FIXED32), S.ProtoField(300, S.PB_INT32),
              S.ProtoField(301, S.PB_STRING)]
    names = [b"", b"a", b"caf\xc3\xa9", b"x" * 40, b"\xe2\x82\xac" * 5, b"y" * 200]
    msgs = []
    for k in range(n):
        r = rng.integers(0, 1 << 62, 6)
        msgs.append([names[int(r[0]) % 6], int(r[1]) - (1 << 61) if k % 3 else 0, int(r[2] % 2001) - 1000, bool(r[3] & 1),
                     float(int(r[4]) % 1000) / 8 if k % 4 else 0.0, bytes(int(b) & 0xFF for b in r[:int(r[5]) % 5]),
                     int(r[5]) & 0xFFFFFFFF if k % 5 else 0, -int(r[0] % 50000) if k % 2 else 7,
                     b"\xff" if k % 97 == 0 else names[int(r[1]) % 6]])
    return fields, msgs


def test_emu_bulk_matches_oracle():
    fields, msgs = _bulk(3000)
    rows, off = S.pack_proto_rows(fields, msgs)
    out, o, meta = O.proto_encode(fields, rows, off)
    assert (meta == S.GRPC_BAD_UTF8).sum() == len(range(0, 3000, 97))
    e_out, e_off, e_meta = emu.proto_encode(fields, rows, off, 3)
    assert np.array_equal(e_meta, meta) and np.array_equal(e_off, o + 3)
    assert e_out[3:int(e_off[-1])].tobytes() == out[:int(o[-1])].tobytes()


@pytest.mark.gpu
def test_gpu_matches_oracle():
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    eng = Engine(Table(synth.config1_spec()), 0)
    for fields, msgs in (_bulk(50000), ([S.ProtoField(1, S.PB_STRING)], [["Hello %d!" % k] for k in range(10000)]),
                         ([S.ProtoField(5, S.PB_UINT64)], [[k * 977] for k in range(1000)]), (_bulk(1)[0], [])):
        rows, off = S.pack_proto_rows(fields, msgs)
        out, o, meta = O.proto_encode(fields, rows, off)
        d_out, d_off, d_meta = eng.proto_encode_device(fields, rows, off)
        g_off = d_off.cpu().numpy().view(np.uint32)
        assert np.array_equal(g_off, o)
        if len(msgs):
            assert np.array_equal(d_meta.cpu().numpy().view(np.uint32), meta)
        assert d_out[:int(o[-1])].cpu().numpy().tobytes() == out[:int(o[-1])].tobytes()
    # argument checks: descending field numbers, unknown type, too many fields
    from gofr_b200 import _abi
    rows, off = S.pack_proto_rows([S.ProtoField(1, S.PB_BOOL)], [[True]])
    for bad in ([S.ProtoField(2, S.PB_BOOL), S.ProtoField(1, S.PB_BOOL)], [S.ProtoField(1, 11)], [S.ProtoField(0, S.PB_BOOL)],
                [S.ProtoField(k + 1, S.PB_BOOL) for k in range(33)]):
        with pytest.raises(_abi.GofrError):
            eng.proto_encode_device(bad, rows, off)
    eng.close()


# =====================================================================================================================
# the other direction: gofr_proto_decode_device — frames → rows (proto.Unmarshal of the request message)
# =====================================================================================================================

def _frame(body: bytes, flag: int = 0) -> bytes:
    return bytes([flag]) + len(body).to_bytes(4, "big") + body


def _pack_frames(frames):
    off = np.zeros(len(frames) + 1, dtype=np.uint32)
    off[1:] = np.cumsum([len(f) for f in frames])
    return np.frombuffer(b"".join(frames), dtype=np.uint8).copy(), off


def _py_parse_rows(fields, frames):
    """rows as python protobuf sees the messages: ParseFromString, then pack the reported field values (None on error)"""
    from google.protobuf.message import DecodeError
    cls = _py_class(fields)
    out = []
    for fr in frames:
        m = cls()
        try:
            m.ParseFromString(fr[5:])
        except DecodeError:
            out.append(None)
            continue
        vals = [getattr(m, "f%d" % f.number) for f in fields]
        rows, off = S.pack_proto_rows(fields, [vals])
        out.append(rows[:int(off[1])].tobytes())
    return out


def _rows(rows, off):
    return [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def _has_overflowing_varint(b: bytes) -> bool:
    """nine continuation bytes followed by a byte > 1: protobuf-go's protowire.ConsumeVarint rejects the overflow
    (errCodeOverflow); python's upb parser drops the extra bits instead — the one place the two parsers disagree"""
    run = 0
    for c in b:
        if run >= 9 and c > 1:
            return True
        run = run + 1 if c >= 0x80 else 0
    return False


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def test_decode_round_trip_and_python_protobuf():
    fields, msgs = _bulk(1500)
    rows, off = S.pack_proto_rows(fields, msgs)
    out, o, meta = O.proto_encode(fields, rows, off)
    ok = meta == 0
    r2, o2, m2 = O.proto_decode(fields, out[:int(o[-1])], o)
    want = _rows(rows, off)
    got = _rows(r2, o2)
    frames = _frames(out, o)
    py = _py_parse_rows(fields, frames)
    for i in range(len(msgs)):
        if ok[i]:
            assert m2[i] == 0 and got[i] == want[i] == py[i], i        # decode(encode(row)) == row == python's view
        else:
            assert m2[i] == S.GRPC_BAD_LENGTH and got[i] == b""          # encoder emitted no frame: an empty frame is too short
    for mis in (0, 6):
        e_rows, e_off, e_meta = emu.proto_decode(fields, out[:int(o[-1])], o, mis)
        assert np.array_equal(e_meta, m2) and np.array_equal(e_off, o2 + mis)
        assert e_rows[mis:int(e_off[-1])].tobytes() == r2[:int(o2[-1])].tobytes()


def T(num, wt):
    """a tag: varint(number << 3 | wire type)"""
    return _varint(num << 3 | wt)


# hostile message bodies for HOSTILE_FIELDS; the last one nests groups deeper than 16 (BAD_PROTO by design, python accepts)
HOSTILE_FIELDS = [S.ProtoField(1, S.PB_STRING), S.ProtoField(2, S.PB_INT32), S.ProtoField(3, S.PB_SINT32), S.ProtoField(4, S.PB_BOOL),
                  S.ProtoField(5, S.PB_FIXED32), S.ProtoField(6, S.PB_UINT64), S.ProtoField(7, S.PB_BYTES), S.ProtoField(8, S.PB_SINT64),
                  S.ProtoField(9, S.PB_DOUBLE)]
HOSTILE_BODIES = [
    b"",                                                                    # all defaults
    T(1, 2) + b"\x02hi" + T(1, 2) + b"\x03bye",                              # last occurrence wins
    T(2, 0) + _varint(2**64 - 1),                                           # int32 -1 as ten bytes
    T(2, 0) + _varint(2**35 + 7),                                           # int32 keeps the low 32 bits
    T(4, 0) + _varint(2**40),                                               # bool: any non-zero varint is true
    T(3, 0) + _varint(2**33 + 3),                                           # sint32: zigzag of the low 32 bits
    T(8, 0) + _varint(2**64 - 1) + T(6, 0) + _varint(2**64 - 1),
    T(2, 2) + b"\x01\x07",                                                  # int32 with a length-delimited wire type: unknown, skipped
    T(1, 0) + b"\x05",                                                      # string with a varint wire type: unknown, skipped
    T(5, 5) + b"\x01\x02\x03\x04" + T(9, 1) + struct.pack("<d", -0.0),
    T(99, 0) + b"\x01" + T(100, 2) + b"\x03abc" + T(101, 1) + b"\0" * 8 + T(102, 5) + b"\0" * 4 + T(1, 2) + b"\x01z",  # unknown fields
    T(50, 3) + T(1, 2) + b"\x01q" + T(50, 4) + T(1, 2) + b"\x01r",           # field 1 inside an unknown group belongs to the group
    T(50, 3) + T(51, 3) + T(51, 4) + T(50, 4),
    T(50, 3),                                                               # unterminated group
    T(50, 4),                                                               # end group without start
    T(50, 3) + T(51, 4),                                                    # mismatched end group
    T(1, 2) + b"\x05ab",                                                    # length runs past the message
    T(1, 2) + b"\x01\xff",                                                  # invalid UTF-8 in a string
    T(1, 2) + b"\x01\xff" + T(1, 2) + b"\x01a",                              # … even when overwritten later
    T(7, 2) + b"\x02\xff\xfe",                                              # bytes may hold anything
    b"\x00",                                                                # field number 0
    _varint((2**29) << 3),                                                  # field number 2^29
    T(1, 6), T(1, 7),                                                       # wire types 6 and 7
    T(2, 0) + b"\x80" * 10 + b"\x01",                                       # varint longer than ten bytes
    T(2, 0) + b"\xff" * 9 + b"\x02",                                        # tenth byte > 1
    T(2, 0) + b"\x80",                                                      # truncated varint
    T(5, 5) + b"\x01\x02",                                                  # truncated fixed32
    T(9, 1) + b"\0" * 7,                                                    # truncated fixed64
    b"".join(T(60 + d, 3) for d in range(17)),                              # groups nested deeper than 16
]
# frames whose 5-byte header is wrong: compressed flag, flag 2, shorter than a header, empty, length one too long / too short
HOSTILE_HEADER_FRAMES = [_frame(T(2, 0) + b"\x01", flag=1), _frame(b"", flag=2), b"\x00\x00\x00", b"",
                         b"\x00\x00\x00\x00\x05" + T(2, 0) + b"\x01", _frame(T(2, 0) + b"\x01") + b"\x00"]


def test_decode_hostile_frames():
    f, bodies = HOSTILE_FIELDS, HOSTILE_BODIES
    frames = [_frame(b) for b in bodies] + HOSTILE_HEADER_FRAMES
    raw, off = _pack_frames(frames)
    rows, roff, meta = O.proto_decode(f, raw, off)
    py = _py_parse_rows(f, frames[:len(bodies)])
    got = _rows(rows, roff)
    for i in range(len(bodies)):
        if i == len(bodies) - 1:
            assert meta[i] == S.GRPC_BAD_PROTO       # our 16-level group limit; python accepts deeper nesting
            continue
        if py[i] is None or _has_overflowing_varint(bodies[i]):
            assert meta[i] in (S.GRPC_BAD_PROTO, S.GRPC_BAD_UTF8) and got[i] == b"", (i, bodies[i])
        else:
            assert meta[i] == 0 and got[i] == py[i], (i, bodies[i])
    assert list(meta[len(bodies):]) == [S.GRPC_COMPRESSED, S.GRPC_BAD_LENGTH, S.GRPC_BAD_LENGTH, S.GRPC_BAD_LENGTH, S.GRPC_BAD_LENGTH,
                                        S.GRPC_BAD_LENGTH]
    assert meta[17] == meta[18] == S.GRPC_BAD_UTF8
    for mis in (0, 3):
        e_rows, e_off, e_meta = emu.proto_decode(f, raw, off, mis)
        assert np.array_equal(e_meta, meta) and np.array_equal(e_off, roff + mis)
        assert e_rows[mis:int(e_off[-1])].tobytes() == rows[:int(roff[-1])].tobytes()


@st.composite
def _wire_soup(draw):
    """a message type plus frames made of random well-formed and malformed wire fragments"""
    nf = draw(st.integers(1, 8))
    numbers = sorted(draw(st.sets(st.integers(1, 12), min_size=nf, max_size=nf)))
    fields = [S.ProtoField(n, draw(st.sampled_from(ALL_TYPES))) for n in numbers]
    frag = st.one_of(
        st.tuples(st.integers(1, 14), st.just(0), st.integers(0, 2**64 - 1)).map(lambda t: _varint(t[0] << 3) + _varint(t[2])),
        st.tuples(st.integers(1, 14), st.binary(min_size=8, max_size=8)).map(lambda t: _varint(t[0] << 3 | 1) + t[1]),
        st.tuples(st.integers(1, 14), st.binary(min_size=4, max_size=4)).map(lambda t: _varint(t[0] << 3 | 5) + t[1]),
        st.tuples(st.integers(1, 14), st.binary(max_size=12) | st.text(max_size=8).map(lambda s: s.encode("utf-8", "surrogatepass")))
        .map(lambda t: _varint(t[0] << 3 | 2) + _varint(len(t[1])) + t[1]),
        st.integers(1, 14).map(lambda n: _varint(n << 3 | 3) + _varint(n << 3 | 4)),
        st.binary(min_size=1, max_size=3),                                        # junk
    )
    frames = [_frame(b"".join(draw(st.lists(frag, max_size=6)))) for _ in range(draw(st.integers(1, 5)))]
    return fields, frames


@settings(max_examples=200, deadline=None)
@given(_wire_soup(), st.integers(0, 15))
def test_decode_random_wire_three_way(soup, mis):
    """python protobuf == oracle == device code (CPU emulation) on random wire fragments, accepted or rejected alike"""
    fields, frames = soup
    raw, off = _pack_frames(frames)
    rows, roff, meta = O.proto_decode(fields, raw, off)
    py = _py_parse_rows(fields, frames)
    got = _rows(rows, roff)
    for i in range(len(frames)):
        if py[i] is None or (meta[i] == S.GRPC_BAD_PROTO and _has_overflowing_varint(frames[i][5:])):
            assert meta[i] in (S.GRPC_BAD_PROTO, S.GRPC_BAD_UTF8) and got[i] == b"", frames[i]
        else:
            assert meta[i] == 0 and got[i] == py[i], frames[i]
    e_rows, e_off, e_meta = emu.proto_decode(fields, raw, off, mis)
    assert np.array_equal(e_meta, meta) and np.array_equal(e_off, roff + mis)
    assert e_rows[mis:int(e_off[-1])].tobytes() == rows[:int(roff[-1])].tobytes()


@pytest.mark.gpu
def test_gpu_decode_matches_oracle():
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    eng = Engine(Table(synth.config1_spec()), 0)
    fields, msgs = _bulk(40000, seed=11)
    rows, off = S.pack_proto_rows(fields, msgs)
    out, o, _ = O.proto_encode(fields, rows, off)
    raw = out[:int(o[-1])]
    r1, o1, m1 = O.proto_decode(fields, raw, o)
    d_rows, d_off, d_meta = eng.proto_decode_device(fields, raw, o)
    assert np.array_equal(d_off.cpu().numpy().view(np.uint32), o1)
    assert np.array_equal(d_meta.cpu().numpy().view(np.uint32), m1)
    assert d_rows[:int(o1[-1])].cpu().numpy().tobytes() == r1[:int(o1[-1])].tobytes()
    # the Hello request type through the general decoder: the same names the Hello kernel extracts
    frames, foff = synth.config5_frames(20000)
    hf = [S.ProtoField(1, S.PB_STRING)]
    r1, o1, m1 = O.proto_decode(hf, frames, foff)
    d_rows, d_off, d_meta = eng.proto_decode_device(hf, frames, foff)
    assert np.array_equal(d_off.cpu().numpy().view(np.uint32), o1) and np.array_equal(d_meta.cpu().numpy().view(np.uint32), m1)
    assert d_rows[:int(o1[-1])].cpu().numpy().tobytes() == r1[:int(o1[-1])].tobytes()
    eng.close()


# =====================================================================================================================
# a pin from the reference itself: the FileDescriptorProto protoc embedded in examples/grpc-server/grpc/hello.pb.go
# (file_hello_proto_rawDesc; extracted by tests/golden/make_descriptor_pin.py) is the one byte string in the reference
# that a real protobuf encoder wrote.  Its nested messages are flat at every level, so both directions can be pinned to it.
# =====================================================================================================================

def _rawdesc() -> bytes:
    import os
    p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hello_proto_rawdesc.hex")
    return bytes.fromhex([l for l in open(p).read().splitlines() if not l.startswith("#")][0])


def _decode_one(fields, body: bytes):
    raw, off = _pack_frames([_frame(body)])
    rows, roff, meta = O.proto_decode(fields, raw, off)
    e_rows, e_off, e_meta = emu.proto_decode(fields, raw, off, 5)
    assert np.array_equal(meta, e_meta) and rows[:int(roff[-1])].tobytes() == e_rows[5:int(e_off[-1])].tobytes()
    assert meta[0] == 0
    row = rows[:int(roff[1])].tobytes()
    # unpack the row: fixed words, then the string bytes in field order
    vals, pos, spos = [], 0, sum(8 if f.type in S.PB_64BIT else 4 for f in fields)
    for f in fields:
        if f.type in (S.PB_STRING, S.PB_BYTES):
            ln = int.from_bytes(row[pos:pos + 4], "little")
            vals.append(row[spos:spos + ln])
            spos += ln
            pos += 4
        elif f.type in S.PB_64BIT:
            vals.append(int.from_bytes(row[pos:pos + 8], "little"))
            pos += 8
        else:
            vals.append(int.from_bytes(row[pos:pos + 4], "little"))
            pos += 4
    return vals


def _encode_one(fields, values) -> bytes:
    rows, off = S.pack_proto_rows(fields, [values])
    out, o, meta = O.proto_encode(fields, rows, off)
    e_out, e_off, e_meta = emu.proto_encode(fields, rows, off, 3)
    assert meta[0] == 0 and e_meta[0] == 0 and out[:int(o[1])].tobytes() == e_out[3:int(e_off[1])].tobytes()
    return out[5:int(o[1])].tobytes()


def test_reference_descriptor_pin():
    from google.protobuf import descriptor_pb2
    raw = _rawdesc()
    fd = descriptor_pb2.FileDescriptorProto.FromString(raw)
    # ---- decoder: the top level of FileDescriptorProto (name=1, message_type=4, service=6, options=8, syntax=12); the
    # repeated message_type keeps its LAST element when read as a singular field
    FILE = [S.ProtoField(1, S.PB_STRING), S.ProtoField(4, S.PB_BYTES), S.ProtoField(6, S.PB_BYTES), S.ProtoField(8, S.PB_BYTES),
            S.ProtoField(12, S.PB_STRING)]
    name, last_msg, service, options, syntax = _decode_one(FILE, raw)
    assert name == b"hello.proto" and syntax == b"proto3"                       # hello.proto:1
    assert last_msg == fd.message_type[1].SerializeToString() and service == fd.service[0].SerializeToString()
    assert options == fd.options.SerializeToString()
    # one level down: DescriptorProto{name=1, field=2}, FieldDescriptorProto{name=1, number=3, label=4, type=5, json_name=10}
    MSG = [S.ProtoField(1, S.PB_STRING), S.ProtoField(2, S.PB_BYTES)]
    FIELD = [S.ProtoField(1, S.PB_STRING), S.ProtoField(3, S.PB_INT32), S.ProtoField(4, S.PB_ENUM), S.ProtoField(5, S.PB_ENUM),
             S.ProtoField(10, S.PB_STRING)]
    mname, mfield = _decode_one(MSG, last_msg)
    assert mname == b"HelloResponse"                                            # hello.proto:8-10
    assert _decode_one(FIELD, mfield) == [b"message", 1, 1, 9, b"message"]      # string message = 1 (LABEL_OPTIONAL, TYPE_STRING)
    OPTS = [S.ProtoField(11, S.PB_STRING)]                                       # FileOptions.go_package
    assert _decode_one(OPTS, options) == [fd.options.go_package.encode()]
    # ---- encoder: rebuild the nested pieces bottom-up and find each of them, byte for byte, inside protoc's output
    for msg_name, fld in (("HelloRequest", "name"), ("HelloResponse", "message")):
        fbytes = _encode_one(FIELD, [fld, 1, 1, 9, fld])
        mbytes = _encode_one(MSG, [msg_name, fbytes])
        assert b"\x22" + bytes([len(mbytes)]) + mbytes in raw, msg_name           # field 4 (message_type), length, payload
    obytes = _encode_one(OPTS, [fd.options.go_package])
    assert raw.endswith(b"\x42" + bytes([len(obytes)]) + obytes + b"\x62\x06proto3")
    assert raw.startswith(_encode_one([S.ProtoField(1, S.PB_STRING)], ["hello.proto"]))
