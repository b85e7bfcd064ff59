"""Field presence in the nested proto3 codec: proto3 `optional` fields and `oneof` groups (ProtoNField.presence), through
gofr_proto_encode_nested_ex_device / gofr_proto_decode_nested_ex_device / gofr_proto_nested_describe_ex.

Reference behaviour: protobuf-go v1.32.0 — proto.Marshal writes a set explicit-presence field even at its zero value or
empty, an unset one not at all, every oneof member at its own number in field-number order; proto.Unmarshal sets an
optional field iff it occurs, and sets the oneof member whose occurrence is last among the group's members.  A message
member occurring twice is GOFR_GRPC_DEFER (protobuf-go merges or replaces; either way the host decodes it).
Statements compared:
  tests/proto_nested_model.py recursive, list-first, the set member is the one holding the group's last wire position
  the device code             one pass per field — on the CPU via tests/emu's nested exports (the descriptor picks the
                              presence instance, as on the host; output misalignments 0 and 3) and, with -m gpu, in
                              proto_encode_nested_presence_kernel / proto_decode_nested_presence_kernel
  python google.protobuf      the pure-Python backend in a child process (map fields are mixed in: upb neither sorts map keys
                              under deterministic=True nor skips unknown fields inside an entry), classes built from
                              descriptor_pb2 with oneof_decl / oneof_index, and proto3_optional with its synthetic oneof."""
import dataclasses
import random
from functools import lru_cache

import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200 import _abi
from tests import proto_nested_harness as H
from tests import proto_nested_model as M
from tests.proto_nested_harness import CAP, INVALID

F = S.ProtoNField
OPT = S.PB_OPTIONAL


# ---------------------------------------------------------------------------------------------------------------
# known answers, derived by hand
# ---------------------------------------------------------------------------------------------------------------
# M0 { optional int32 a = 1; optional string s = 2; oneof o { int32 x = 3; M1 y = 4; } oneof p { int32 A = 5; string B = 6; }
#      optional M1 z = 7; optional sint64 q = 8; }
# M1 { int32 v = 1; }
KA_MSGS = [[F(1, S.PB_INT32, presence=OPT), F(2, S.PB_STRING, presence=OPT), F(3, S.PB_INT32, presence=1), F(4, S.PB_MESSAGE, False, 1, 1),
            F(5, S.PB_INT32, presence=2), F(6, S.PB_STRING, presence=2), F(7, S.PB_MESSAGE, False, 1, OPT), F(8, S.PB_SINT64, presence=OPT)],
           [F(1, S.PB_INT32)]]
_N = [None] * 8


def _v(**kw):
    v = list(_N)
    for k, x in kw.items():
        v["a s x y A B z q".split().index(k)] = x
    return v


KA_ENC = [(_v(a=0), "0800"),                              # optional int32 set to 0
          (_v(s=""), "1200"),                             # optional string set to ""
          (_v(x=0), "1800"),                              # a oneof scalar member at 0, the message member absent
          (_v(y=[0]), "2200"),                            # the message member set, empty
          (_v(B=""), "3200"),
          (_v(z=[0]), "3a00"),                            # optional on a message field: a set message, as always
          (_v(q=0), "4000"),
          (_v(q=-1), "4001"),
          (list(_N), ""),                                 # nothing set: nothing written
          (_v(a=-1, s="é", y=[5], A=7, q=1), "08ffffffffffffffffff01" "1202c3a9" "22020805" "2807" "4002")]
# (body, decoded value list) — None: not set
KA_DEC = [("280132017828" "02", _v(A=2)),                 # A=1, B="x", A=2: A wins with its last value
          ("2801320178", _v(B=b"x")),
          ("3201782801", _v(A=1)),
          ("1805220208" "01", _v(y=[1])),                 # x, then y: y set
          ("2202080118" "05", _v(x=5)),                   # y, then x: x set, y unset
          ("22001d00000000", _v(y=[0])),                  # x with a foreign wire type: unknown, the case stays y
          ("0a00" "0801", _v(a=1)),                       # a with wire type 2 first: unknown
          ("0800" "1200" "4000", _v(a=0, s=b"", q=0)),
          ("", list(_N)),
          ("3a00" "3a020801", None)]                      # an optional message twice: merged by Go -> DEFER
KA_DEC_STATUS = [(b"\x22\x00\x18\x05\x22\x00", S.GRPC_DEFER),         # message member, other member, message member again
                 (b"\x22\x00\x22\x00", S.GRPC_DEFER),
                 (b"\x32\x01\xff\x28\x01", S.GRPC_BAD_UTF8),          # invalid UTF-8 in a member that loses
                 (b"\x12\x01\xff\x12\x00", S.GRPC_BAD_UTF8),          # ... in an optional string's overwritten value
                 (b"\x22\x03\x08", S.GRPC_BAD_PROTO),                 # a malformed message member
                 (b"\x22\x02\x0a\x00\x22\x00\x32\x01\xff", S.GRPC_BAD_UTF8)]   # invalid UTF-8 beats DEFER


def test_known_answers_encode():
    values = [v for v, _ in KA_ENC]
    rows, off = S.pack_proto_nested_rows(KA_MSGS, 0, values)
    frames, meta = H.encode_model_emu(KA_MSGS, 0, rows, off)
    assert meta == [0] * len(values)
    for k, (_, hexs) in enumerate(KA_ENC):
        assert frames[k] == H.frame(bytes.fromhex(hexs)), (k, frames[k].hex())
    assert H.pure_python([("enc", KA_MSGS, 0, values)])[0] == frames
    d_rows, d_meta = H.decode_model_emu(KA_MSGS, 0, frames)
    assert d_meta == meta
    assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]


def test_known_answers_decode():
    frames = [H.frame(bytes.fromhex(h)) for h, _ in KA_DEC] + [H.frame(b) for b, _ in KA_DEC_STATUS]
    rows, meta = H.decode_model_emu(KA_MSGS, 0, frames)
    assert meta == [0 if v is not None else S.GRPC_DEFER for _, v in KA_DEC] + [s for _, s in KA_DEC_STATUS], meta
    for k, (h, v) in enumerate(KA_DEC):
        if v is not None:
            want, _ = S.pack_proto_nested_rows(KA_MSGS, 0, [v])
            assert rows[k] == want[:-8].tobytes(), (k, h, rows[k].hex())
    H.check_python_parse(KA_MSGS, 0, frames, rows, meta)


# ---------------------------------------------------------------------------------------------------------------
# random type sets with optional fields and oneofs, mixed with nested, repeated and map fields
# ---------------------------------------------------------------------------------------------------------------
ENC_SEEDS = range(26)


@lru_cache(maxsize=None)
def _enc_cases():
    cases = []
    for seed in ENC_SEEDS:
        rnd = random.Random(5100 + seed)
        msgs = H.rand_presence_types(rnd)
        cases.append((msgs, 0, [H.rand_presence_value(rnd, msgs, 0) for _ in range(40)]))
    return cases, H.pure_python([("enc", m, r, v) for m, r, v in cases])


@pytest.mark.parametrize("seed", ENC_SEEDS)
def test_random_presence_types_encode(seed):
    """model == device code == pure-Python deterministic bytes; the decoder gives the rows back"""
    cases, py = _enc_cases()
    msgs, root, values = cases[seed]
    desc = np.zeros(512, np.uint8)
    assert H.describe(msgs, root, desc) == 0 and desc[1] == 1
    rows, off = S.pack_proto_nested_rows(msgs, root, values)
    frames, meta = H.encode_model_emu(msgs, root, rows, off)
    assert meta == [0] * len(values)
    for i in range(len(values)):
        assert frames[i] == py[seed][i], (i, values[i], frames[i].hex(), py[seed][i].hex())
    # round trip: decode(encode(row)) == row (map message values present: a nil one comes back empty)
    d_rows, d_meta = H.decode_model_emu(msgs, root, frames)
    assert d_meta == meta
    if not H.entry_types(msgs):
        assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]


def test_decode_round_trip_and_python_parse():
    """decode(encode(row)) == row; python protobuf parses each frame to the same values"""
    rnd = random.Random(77)
    for msgs in [KA_MSGS] + [H.rand_presence_types(rnd) for _ in range(8)]:
        values = [H.rand_presence_value(rnd, msgs, 0) for _ in range(40)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = H.encode_model_emu(msgs, 0, rows, off)
        assert meta == [0] * len(values)
        d_rows, d_meta = H.decode_model_emu(msgs, 0, frames)
        assert d_meta == meta
        assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]
        H.check_python_parse(msgs, 0, frames, d_rows, d_meta)


def _shuffle_fields(rnd, body, msgs):
    """the top-level fields of a well-formed body in a random order (oneof members in every order)"""
    items, i = [], 0
    while i < len(body):
        j = i
        tag, j = M._get_varint(body, j, len(body))
        wt = tag & 7
        if wt == 0:
            _, j = M._get_varint(body, j, len(body))
        elif wt == 1:
            j += 8
        elif wt == 5:
            j += 4
        else:
            n, j = M._get_varint(body, j, len(body))
            j += n
        items.append(body[i:j])
        i = j
    rnd.shuffle(items)
    return b"".join(items)


MUT_SEEDS = range(12)


@pytest.mark.parametrize("seed", MUT_SEEDS)
def test_decode_mutated_frames(seed):
    """frames of random presence types, fields reordered and duplicated, then bytes flipped, inserted, cut and rotated:
    model == device code on status, offsets and rows; python protobuf agrees on what parses and on every value"""
    rnd = random.Random(6200 + seed)
    msgs = H.rand_presence_types(rnd)
    values = [H.rand_presence_value(rnd, msgs, 0) for _ in range(50)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, _ = M.encode(msgs, 0, rows, off)
    others, _ = M.encode(msgs, 0, *S.pack_proto_nested_rows(msgs, 0, [H.rand_presence_value(rnd, msgs, 0) for _ in range(50)]))
    out = []
    for fr, other in zip(frames, others):
        body = bytearray(_shuffle_fields(rnd, fr[5:] + (other[5:] if rnd.random() < 0.5 else b""), msgs))
        for _ in range(rnd.randint(0, 2)):
            r = rnd.random()
            if body and r < 0.3:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            elif body and r < 0.4:
                del body[rnd.randrange(len(body)):]
            elif r < 0.7:
                p = rnd.randrange(len(body) + 1)
                body[p:p] = rnd.choice([b"\x08\x00", b"\x10\x01", b"\x12\x00", b"\x1a\x00", b"\x0b\x0c", b"\x0d\x00\x00\x00\x00", b"\x80"])
            else:
                p = rnd.randrange(len(body) + 1)
                body = body[p:] + body[:p]
        out.append(H.frame(bytes(body)))
    d_rows, d_meta = H.decode_model_emu(msgs, 0, out)
    assert sum(m == 0 for m in d_meta) >= 10
    H.check_python_parse(msgs, 0, out, d_rows, d_meta)


def test_presence_instance_on_presence_free_types():
    """the presence kernels' instance answers as the others on descriptions without presence (maps and map-free)"""
    rnd = random.Random(8)
    for k in range(6):
        msgs = H.rand_map_types(rnd) if k % 2 else H.rand_types(rnd)
        values = [[None if f.type == S.PB_MESSAGE and not f.repeated and rnd.random() < 0.3 else x for f, x in zip(msgs[0], v)]
                  for v in [H.rand_presence_value(rnd, msgs, 0) for _ in range(30)]]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = H.encode_model_emu(msgs, 0, rows, off, presence_instance=True)
        assert meta == [0] * len(values)
        frames = [fr if i % 3 else H.frame(_shuffle_fields(rnd, fr[5:], msgs) + fr[5:]) for i, fr in enumerate(frames)]
        H.decode_model_emu(msgs, 0, frames, presence_instance=True)


# ---------------------------------------------------------------------------------------------------------------
# bad rows and descriptions
# ---------------------------------------------------------------------------------------------------------------
# M0 { optional int32 a = 1; oneof o { int32 x = 2; string y = 3; M1 z = 4; } repeated M0b r = 5 }  M1 { int32 v = 1; }
BR_MSGS = [[F(1, S.PB_INT32, presence=OPT), F(2, S.PB_INT32, presence=1), F(3, S.PB_STRING, presence=1), F(4, S.PB_MESSAGE, False, 1, 1),
            F(5, S.PB_MESSAGE, True, 2)],
           [F(1, S.PB_INT32)],
           [F(1, S.PB_STRING, presence=OPT), F(2, S.PB_DOUBLE, presence=3)]]


def _words(*w):
    return b"".join(int(x).to_bytes(4, "little") for x in w)


def test_bad_rows():
    """presence word not 0 / 1, an unset field with value words, two set members of one group: BAD_ROW; model == device"""
    # fixed part of M0: a [p, w] x [p, w] y [p, len] z [p, v] r [count] = 36 bytes
    blobs = [
        (_words(1, 0, 0, 0, 0, 0, 0, 0, 0), 0),                       # a = 0, set: fine
        (_words(2, 5, 0, 0, 0, 0, 0, 0, 0), S.GRPC_BAD_ROW),          # presence word 2
        (_words(0xFFFFFFFF, 0, 0, 0, 0, 0, 0, 0, 0), S.GRPC_BAD_ROW),
        (_words(0, 5, 0, 0, 0, 0, 0, 0, 0), S.GRPC_BAD_ROW),          # unset, value 5
        (_words(0, 0, 1, 1, 1, 0, 0, 0, 0), S.GRPC_BAD_ROW),          # x and y set
        (_words(0, 0, 1, 1, 0, 0, 1, 3, 0), S.GRPC_BAD_ROW),          # x and z set
        (_words(0, 0, 0, 0, 0, 1, 0, 0, 0) + b"a\0\0\0", S.GRPC_BAD_ROW),   # y unset with a length
        (_words(0, 0, 0, 0, 0, 0, 0, 3, 0), S.GRPC_BAD_ROW),          # z unset, its fixed part not zero
        (_words(0, 0, 0, 0, 2, 0, 0, 0, 0), S.GRPC_BAD_ROW),          # y: presence word 2
        (_words(0, 0, 0, 0, 0, 0, 2, 0, 0), S.GRPC_BAD_ROW),          # z: presence word 2
        (_words(0, 0, 0, 0, 1, 1, 0, 0, 0) + b"\xff\0\0\0", S.GRPC_BAD_UTF8),  # y set, invalid UTF-8
        (_words(0, 0, 0, 0, 1, 2, 0, 0, 0) + b"a", S.GRPC_BAD_ROW),   # y's bytes past the row
        (_words(0, 0, 0, 0, 1, 1, 1, 0, 0) + b"a\0\0\0", S.GRPC_BAD_ROW),   # y and z set
        (_words(0, 0, 0, 0, 0, 0, 1, 0, 0), 0),                       # z set, empty
        # one element of r: M2 { optional string s; oneof { double d } }: fixed [p, len] [p, lo, hi]
        (_words(0, 0, 0, 0, 0, 0, 0, 0, 1) + _words(0, 0, 1, 0, 0), 0),
        (_words(0, 0, 0, 0, 0, 0, 0, 0, 1) + _words(0, 0, 0, 0, 7), S.GRPC_BAD_ROW),   # d unset, high word set
        (_words(0, 0, 0, 0, 0, 0, 0, 0, 1) + _words(3, 0, 0, 0, 0), S.GRPC_BAD_ROW),
        (_words(0, 0, 0, 0, 0, 0, 0, 0, 1) + _words(1, 1, 0, 0, 0) + b"\xc3\0\0\0", S.GRPC_BAD_UTF8),
        (_words(2, 0, 0, 0, 0, 0, 1, 0, 0), S.GRPC_BAD_ROW),          # bad a before a fine z
    ]
    body, offs = bytearray(), [0]
    for b, _ in blobs:
        body += b
        offs.append(len(body))
    rows = np.frombuffer(bytes(body) + b"\0" * 16, dtype=np.uint8).copy()
    _, meta = H.encode_model_emu(BR_MSGS, 0, rows, np.array(offs, dtype=np.uint32))
    assert meta == [s for _, s in blobs], meta
    # the packer lays out such rows too
    r2, o2 = S.pack_proto_nested_rows(BR_MSGS, 0, [[None, None, None, None, []], [0, 1, "", None, []], [None, None, None, [0], [[None, None]]]])
    _, meta2 = H.encode_model_emu(BR_MSGS, 0, r2, o2)
    assert meta2 == [0, S.GRPC_BAD_ROW, 0]


def _last_error():
    return _abi.lib().gofr_last_error().decode()


PLAIN = [[F(1, S.PB_INT32), F(2, S.PB_MESSAGE, False, 1)], [F(1, S.PB_STRING)]]
PLAIN_OPT = [[PLAIN[0][0], dataclasses.replace(PLAIN[0][1], presence=OPT)], PLAIN[1]]   # optional on a message field
WITHMAP = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_INT32, presence=OPT)], [F(1, S.PB_STRING), F(2, S.PB_INT32)]]
SEVEN_GROUPS = [[[F(k, S.PB_INT32, presence=k) for k in range(1, 8)]],
                [[F(1, S.PB_MESSAGE, False, 1, 7), F(2, S.PB_BYTES, presence=7)], [F(1, S.PB_INT32, presence=OPT)]]]
BAD_DESCRIPTIONS = [
    ([[F(1, S.PB_INT32, presence=8)]], "presence byte 8"),
    ([[F(1, S.PB_INT32, presence=0x81)]], "presence byte 129"),
    ([[F(1, S.PB_INT32, presence=0x40)]], "presence byte 64"),
    ([[F(1, S.PB_INT32, True, presence=OPT)]], "a repeated or map field has no presence"),
    ([[F(1, S.PB_STRING, True, presence=2)]], "a repeated or map field has no presence"),
    ([[F(1, S.PB_MESSAGE, True, 1, 1)], [F(1, S.PB_INT32)]], "a repeated or map field has no presence"),
    ([[F(1, S.PB_MAP, False, 1, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], "a repeated or map field has no presence"),
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32, presence=OPT), F(2, S.PB_INT32)]], "its key and value carry no presence"),
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_MESSAGE, False, 2, OPT)], [F(1, S.PB_INT32)]],
     "its key and value carry no presence"),
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_STRING, presence=3)]], "its key and value carry no presence"),
]


def test_descriptions():
    desc = np.zeros(512, np.uint8)
    # no presence, and optional on a message field: the same descriptor as the call without presence
    nm, nf, k = S.proto_nested_tables(PLAIN)
    ref = np.zeros(512, np.uint8)
    assert _abi.lib().gofr_proto_nested_describe(nm.ctypes.data, 2, nf.ctypes.data, k, 0, ref.ctypes.data, ref.size) == 0
    for msgs in (PLAIN, PLAIN_OPT):
        desc[:] = 0
        assert H.describe(msgs, 0, desc) == 0
        assert desc.tobytes() == ref.tobytes()
    assert _abi.lib().gofr_proto_nested_describe_ex(nm.ctypes.data, 2, nf.ctypes.data, k, 0, None, desc.ctypes.data, desc.size) == 0
    assert desc.tobytes() == ref.tobytes()
    # with presence: the presence byte of the descriptor is set, the maps half-word says what it said
    assert H.describe(KA_MSGS, 0, desc) == 0 and desc[1] == 1 and desc[2] == 0
    assert H.describe(WITHMAP, 0, desc) == 0 and desc[1] == 1 and desc[2] == 1
    # fixed words of the root (PbnDesc::fixed_words[0], bytes 40..41): the presence words count
    # (a: 2, s: 2, x: 2, y: 1 + 1, A: 2, B: 2, z: 1 + 1, q: 3)
    assert H.describe(KA_MSGS, 0, desc) == 0
    assert int(desc[40]) | int(desc[41]) << 8 == 17
    # seven groups in one message type are fine
    for msgs in SEVEN_GROUPS:
        assert H.describe(msgs) == CAP
    for msgs, text in BAD_DESCRIPTIONS:
        assert H.describe(msgs) == INVALID, msgs
        assert text in _last_error(), (_last_error(), text)


def test_ex_calls_without_presence_bytes_are_the_plain_calls():
    """presence == NULL: the _ex call answers exactly as the call without presence, with and without room for the
    descriptor, on every description of the description tests (the nested limits, map fields, presence)"""
    L = _abi.lib()
    descriptions = [(m, r) for m, r, _ in H.LIMIT_DESCRIPTIONS + H.MAP_DESCRIPTIONS]
    descriptions += [(m, 0) for m in [PLAIN, PLAIN_OPT, KA_MSGS, WITHMAP] + SEVEN_GROUPS + [m for m, _ in BAD_DESCRIPTIONS]]
    for msgs, root in descriptions:
        nm, nf, k = S.proto_nested_tables(msgs)
        a = L.gofr_proto_nested_describe(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None, 0)
        b = L.gofr_proto_nested_describe_ex(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None, None, 0)
        assert a == b, msgs
        da, db = np.zeros(512, np.uint8), np.zeros(512, np.uint8)
        a = L.gofr_proto_nested_describe(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, da.ctypes.data, da.size)
        b = L.gofr_proto_nested_describe_ex(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None, db.ctypes.data, db.size)
        assert a == b and da.tobytes() == db.tobytes(), msgs


# ---------------------------------------------------------------------------------------------------------------
# the CUDA kernels
# ---------------------------------------------------------------------------------------------------------------
def _top_presence_offsets(msgs):
    """byte offsets of the presence words of the root's explicit-presence scalar / string fields in its fixed part"""
    offs, p = [], 0
    for f in msgs[0]:
        if M.explicit(f):
            offs.append(p)
        p += 4 + M.fixed_bytes(msgs, f.msg) if f.type == S.PB_MESSAGE and not f.repeated else M.fixed_bytes([[f]], 0)
    return offs


def _types(rnd):
    """presence types whose root has an explicit-presence scalar or string field"""
    msgs = H.rand_presence_types(rnd)
    while not _top_presence_offsets(msgs):
        msgs = H.rand_presence_types(rnd)
    return msgs


def _spoil(rnd, msgs, values):
    """rows with a presence word of 2 in one row of 53, which the encoder refuses (H.gpu_check)"""
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    po = _top_presence_offsets(msgs)
    spoiled = range(0, len(values), 53)
    for i in spoiled:
        rows[int(off[i]) + rnd.choice(po)] = 2
    return rows, off, len(spoiled)


@pytest.mark.gpu
def test_gpu_presence_matches_model():
    """both presence kernels == the model (statuses, offsets, frames, rows) — in a child process, so that a fault in a
    kernel cannot leave a sticky CUDA error in the process the other GPU tests run in"""
    out = H.run_child("import tests.proto_nested_harness as h, tests.test_proto_presence as t; "
                      "h.gpu_check(93, t._types, h.rand_presence_value, t._spoil)")
    print(out.strip().splitlines()[-1] if out.strip() else "")
