"""What the tests of the nested proto3 codec share: frame helpers, seeded generators of message types and values,
fixtures, python protobuf (in-process or pure-Python in a child), the statements side by side, descriptions, and the
body of the GPU checks against the model.  The statements: tests/proto_nested_model.py, the C oracle
(oracle/orc_proto_nested.c, map- and presence-free), the device code on the CPU (tests/emu), python google.protobuf."""
import dataclasses
import os
import pickle
import random
import struct
import subprocess
import sys

import numpy as np

from gofr_b200 import spec as S
from gofr_b200 import _abi
from tests import oracle as O
from tests import proto_nested_model as M
from tests.emu import emu

F = S.ProtoNField
OPT = S.PB_OPTIONAL
ROOT_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, UNSUPPORTED, CAP = 1, 2, 7   # GOFR_ERR_*; CAPACITY = "valid, but no room to write the descriptor"


# ---------------------------------------------------------------------------------------------------------------
# frames
# ---------------------------------------------------------------------------------------------------------------
def frame(body: bytes) -> bytes:
    return b"\x00" + len(body).to_bytes(4, "big") + body


def pack_frames(frames):
    blob, offs = bytearray(), [0]
    for fr in frames:
        blob += fr
        offs.append(len(blob))
    return np.frombuffer(bytes(blob) + b"\0" * 16, dtype=np.uint8).copy(), np.array(offs, dtype=np.uint32)


def frames_of(out, off):
    return [out[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def has_overlong_varint(body: bytes) -> bool:
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


# ---------------------------------------------------------------------------------------------------------------
# seeded generators: message types and their values
# ---------------------------------------------------------------------------------------------------------------
SCALARS = [S.PB_DOUBLE, S.PB_FLOAT, S.PB_INT64, S.PB_UINT64, S.PB_INT32, S.PB_FIXED64, S.PB_FIXED32, S.PB_BOOL, S.PB_STRING,
           S.PB_BYTES, S.PB_UINT32, S.PB_SFIXED32, S.PB_SFIXED64, S.PB_SINT32, S.PB_SINT64]
KEYS = [S.PB_INT32, S.PB_INT64, S.PB_UINT32, S.PB_UINT64, S.PB_SINT32, S.PB_SINT64, S.PB_FIXED32, S.PB_FIXED64, S.PB_SFIXED32,
        S.PB_SFIXED64, S.PB_BOOL, S.PB_STRING]


def entry_types(msgs):
    return {f.msg for fields in msgs for f in fields if f.type == S.PB_MAP}


def rand_types(rnd):
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
        return rand_types(rnd)
    return msgs


def rand_map_types(rnd):
    """up to 8 types with at most 48 fields, 4 levels: map fields of every key kind, message values that hold maps and
    repeated fields, entry types shared by two map fields"""
    msgs = []

    def new_msg(levels):
        idx = len(msgs)
        msgs.append(None)
        fields, mine = [], []
        for num in sorted(rnd.sample(range(1, 30), rnd.randint(1, 5))):
            r = rnd.random()
            if levels >= 2 and r < 0.5 and (mine and rnd.random() < 0.25):
                fields.append(F(num, S.PB_MAP, False, rnd.choice(mine)))          # a second map field of the same entry type
            elif levels >= 2 and r < 0.5 and len(msgs) <= 6:
                e = len(msgs)
                msgs.append(None)
                if levels >= 3 and rnd.random() < 0.5 and len(msgs) <= 7:
                    vf = F(2, S.PB_MESSAGE, False, new_msg(levels - 2))
                else:
                    vf = F(2, rnd.choice(SCALARS + [S.PB_ENUM]))
                msgs[e] = [F(1, rnd.choice(KEYS)), vf]
                mine.append(e)
                fields.append(F(num, S.PB_MAP, False, e))
            elif levels >= 2 and r < 0.65 and len(msgs) <= 7:
                fields.append(F(num, S.PB_MESSAGE, rnd.random() < 0.5, new_msg(levels - 1)))
            else:
                fields.append(F(num, rnd.choice(SCALARS), rnd.random() < 0.3))
        msgs[idx] = fields
        return idx
    new_msg(4)
    if not entry_types(msgs) or sum(len(f) for f in msgs) > 48:
        return rand_map_types(rnd)
    return msgs


def add_presence(rnd, msgs):
    """optional fields and up to three oneof groups per message type (never in a map entry type)"""
    entries = entry_types(msgs)
    out = []
    for m, fields in enumerate(msgs):
        if m in entries:
            out.append(list(fields))
            continue
        groups = rnd.sample(range(1, 8), rnd.randint(0, 3))
        new = []
        for f in fields:
            p = 0
            if not f.repeated and f.type != S.PB_MAP:
                r = rnd.random()
                if groups and r < 0.45:
                    p = rnd.choice(groups)
                elif r < 0.75:
                    p = OPT
            new.append(dataclasses.replace(f, presence=p))
        out.append(new)
    return out


def rand_presence_types(rnd):
    while True:
        msgs = add_presence(rnd, rand_map_types(rnd) if rnd.random() < 0.6 else rand_types(rnd))
        if any(M.explicit(f) or M.group(f) for f in msgs[0]):   # (optional on a message field alone marks nothing)
            return msgs


def rand_scalar(rnd, t):
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


def rand_key(rnd, t):
    if t == S.PB_STRING:
        return rnd.choice(["", "a", "b", "ab", "aa", "a\x00", "é", "日本", "zz" * 20, "k%d" % rnd.randint(0, 99)])
    return rand_scalar(rnd, t)


def rand_value(rnd, msgs, m, depth=0):
    v = []
    for f in msgs[m]:
        one = (lambda: rand_value(rnd, msgs, f.msg, depth + 1)) if f.type == S.PB_MESSAGE else (lambda: rand_scalar(rnd, f.type))
        if f.repeated:
            v.append([one() for _ in range(rnd.choice([0, 0, 1, 2, 5]))])
        elif f.type == S.PB_MESSAGE:
            v.append(None if rnd.random() < 0.4 else one())
        else:
            v.append(one())
    return v


def rand_map_value(rnd, msgs, m, nil_values=True):
    v = []
    for f in msgs[m]:
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            d = {}
            for _ in range(rnd.choice([0, 0, 1, 2, 3, 8])):
                if vf.type == S.PB_MESSAGE:
                    x = None if nil_values and rnd.random() < 0.2 else rand_map_value(rnd, msgs, vf.msg, nil_values)
                else:
                    x = rand_scalar(rnd, vf.type)
                d[rand_key(rnd, kf.type)] = x
            v.append(d)
        elif f.type == S.PB_MESSAGE:
            one = lambda: rand_map_value(rnd, msgs, f.msg, nil_values)  # noqa: E731
            v.append([one() for _ in range(rnd.choice([0, 1, 2]))] if f.repeated else None if rnd.random() < 0.4 else one())
        elif f.repeated:
            v.append([rand_scalar(rnd, f.type) for _ in range(rnd.choice([0, 1, 3]))])
        else:
            v.append(rand_scalar(rnd, f.type))
    return v


def rand_presence_value(rnd, msgs, m):
    """a value list with at most one set member per oneof group; explicit-presence fields unset about half the time"""
    fields = msgs[m]
    chosen = {}
    for g in {f.presence for f in fields if 1 <= f.presence <= 7}:
        members = [q for q, f in enumerate(fields) if f.presence == g]
        chosen[g] = rnd.choice(members + [None])
    v = []
    for q, f in enumerate(fields):
        one = (lambda: rand_presence_value(rnd, msgs, f.msg)) if f.type == S.PB_MESSAGE else (lambda: rand_scalar(rnd, f.type))
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            d = {}
            for _ in range(rnd.choice([0, 0, 1, 2, 4])):
                d[rand_key(rnd, kf.type)] = rand_presence_value(rnd, msgs, vf.msg) if vf.type == S.PB_MESSAGE else rand_scalar(rnd, vf.type)
            v.append(d)
        elif f.repeated:
            v.append([one() for _ in range(rnd.choice([0, 1, 2]))])
        elif 1 <= f.presence <= 7:
            v.append(one() if chosen[f.presence] == q else None)
        elif f.presence or f.type == S.PB_MESSAGE:
            v.append(None if rnd.random() < 0.5 else one())
        else:
            v.append(one())
    return v


# ---------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------
# the shapes of a typical API: a page of items with tags, an optional owner, per-item attributes and histograms
ITEM = [F(1, S.PB_INT64), F(2, S.PB_STRING), F(3, S.PB_STRING, True), F(4, S.PB_DOUBLE, True), F(5, S.PB_MESSAGE, False, 2), F(7, S.PB_SINT32, True)]
PAGE = [F(1, S.PB_MESSAGE, True, 1), F(2, S.PB_UINT32), F(3, S.PB_STRING), F(15, S.PB_MESSAGE, False, 2), F(16, S.PB_BOOL, True), F(2047, S.PB_FIXED64, True)]
OWNER = [F(1, S.PB_STRING), F(2, S.PB_BYTES, True), F(3, S.PB_MESSAGE, False, 3)]
GEO = [F(1, S.PB_FLOAT), F(2, S.PB_FLOAT), F(9, S.PB_ENUM, True)]
MSGS = [PAGE, ITEM, OWNER, GEO]

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
    b"\x22" + varint(len(_SUB)) + _SUB,                              # singular message
    b"\x2a\x00" + b"\x2a" + varint(len(_SUB)) + _SUB + b"\x2a\x00",   # three elements, two empty
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


def _entry(num, body):
    return varint(num << 3 | 2) + varint(len(body)) + body


def _s(num, b):
    return varint(num << 3 | 2) + varint(len(b)) + b


# M { map<string, V> a = 1; map<int32, int64> b = 2; map<bool, string> c = 3; int32 d = 4; }  V { int32 x = 1; map<uint64, bytes> y = 2; }
NONCANON_MSGS = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 2), F(3, S.PB_MAP, False, 3), F(4, S.PB_INT32)],
                 [F(1, S.PB_STRING), F(2, S.PB_MESSAGE, False, 4)], [F(1, S.PB_INT32), F(2, S.PB_INT64)], [F(1, S.PB_BOOL), F(2, S.PB_STRING)],
                 [F(1, S.PB_INT32), F(2, S.PB_MAP, False, 5)], [F(1, S.PB_UINT64), F(2, S.PB_BYTES)]]
_V1, _V2 = b"\x08\x01", b"\x08\x02" + _entry(2, b"\x08\x05\x12\x01z")


def _A(k, v):
    return _entry(1, _s(1, k) + _s(2, v))


def _B(k, v):
    return _entry(2, b"\x08" + varint(k & (2 ** 64 - 1)) + b"\x10" + varint(v & (2 ** 64 - 1)))


NONCANON_OK = [
    _A(b"b", _V1) + _A(b"a", _V2) + _A(b"", b""),                            # shuffled
    _A(b"a", _V1) + _A(b"a", _V2),                                         # duplicate key: the later value replaces
    _A(b"a", _V2) + _B(3, 1) + _A(b"a", _V1) + _B(-3, 2) + _B(3, 9),          # duplicates interleaved with another map
    _entry(1, _s(2, _V1) + _s(1, b"k")),                                # value before key
    _entry(1, _s(1, b"k")) + _entry(1, _s(2, _V2)) + _entry(2, b"") + _entry(3, b"\x12\x00"),   # missing value / key / both
    _entry(1, _s(1, b"x") + _s(1, b"k") + _s(2, _V1)),                  # key twice inside an entry: the last wins
    _entry(2, b"\x08\x01\x10\x05\x10\x07\x08\x02"),                    # scalar key and value twice
    _entry(1, _s(1, b"k") + b"\x18\x05" + b"\x2b\x08\x01\x2c" + _s(2, _V1) + b"\x25\x00\x00\x00\x00"),  # unknown fields and a group
    _entry(2, b"\x0d\x01\x00\x00\x00\x08\x04\x11" + bytes(8) + b"\x10\x06"),  # foreign wire types for key and value: unknown
    b"\x08\x03" + b"\x10\x05" + b"\x18\x01" + _entry(3, b"\x08\x02\x12\x01t") + b"\x20\x07",   # map fields with a foreign wire type
    _entry(3, b"\x08\x01\x12\x01t") + _entry(3, b"\x12\x01f"),          # bool keys: true first on the wire
    b"\x0b" + _A(b"g", _V1) + b"\x0c" + _A(b"h", _V1),                     # an entry inside an unknown group is skipped
    _entry(1, _s(1, b"n") + _s(2, _entry(2, b"\x08\x02") + _entry(2, b"\x08\x01\x12\x01a") + _entry(2, b"\x08\x02\x12\x01b"))),
    b"".join(_B(k, k) for k in range(63, -1, -1)),                      # exactly 64 entries
    b"".join(_B(k % 8, k) for k in range(64)),                          # 64 on the wire, 8 keys
]
NONCANON_DEFER = [
    b"".join(_B(k, k) for k in range(65)),                              # 65 entries
    b"".join(_B(k % 2, k) for k in range(65)),                          # 65 on the wire, duplicates counted
    _entry(1, _s(1, b"k") + _s(2, _V1) + _s(2, _V2)),                    # a value message twice in one entry (merged by Go)
    _A(b"a", _entry(2, b"") * 65),                                      # too many entries one level down
]
NONCANON_BAD = [
    _entry(1, _s(1, b"\xff") + _s(2, _V1)),                             # invalid UTF-8 key -> BAD_UTF8
    _A(b"a", _V1) + _A(b"\xc3", _V1) + _A(b"a", _V2),                        # ... in an entry that a later one replaces
    _entry(3, b"\x08\x01\x12\x01\xff"),                                # invalid UTF-8 value
    _entry(1, b"\x0a\x05ab"),                                          # malformed inside an entry -> BAD_PROTO
    _entry(1, b"\x0b"),                                                # open group inside an entry
    _entry(1, _s(2, b"\x12\x03\x08")),                                 # malformed inside a value's map
    b"".join(_B(k, k) for k in range(70)) + _entry(1, b"\x0a\x05ab"),   # malformed beats DEFER
    b"".join(_B(k, k) for k in range(70)) + _entry(1, _s(1, b"\xff")),  # invalid UTF-8 beats DEFER
]

# M { map<string,int32> s = 1; map<int32,string> i = 2; map<bool,V> b = 3; map<uint64,bytes> u = 4; map<sint64,double> z = 5; }
MAP_KA_MSGS = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 2), F(3, S.PB_MAP, False, 3), F(4, S.PB_MAP, False, 5), F(5, S.PB_MAP, False, 6)],
               [F(1, S.PB_STRING), F(2, S.PB_INT32)],
               [F(1, S.PB_INT32), F(2, S.PB_STRING)],
               [F(1, S.PB_BOOL), F(2, S.PB_MESSAGE, False, 4)],
               [F(1, S.PB_INT32)],                                     # V { int32 x = 1; }
               [F(1, S.PB_UINT64), F(2, S.PB_BYTES)],
               [F(1, S.PB_SINT64), F(2, S.PB_DOUBLE)]]


# ---------------------------------------------------------------------------------------------------------------
# descriptions: (msgs, root, the answer of describe() without room for the descriptor)
# ---------------------------------------------------------------------------------------------------------------
def describe(msgs, root=0, desc=None):
    """gofr_proto_nested_describe_ex with the description's presence bytes (NULL when no field has presence), the
    descriptor written to desc"""
    nm, nf, k = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    return _abi.lib().gofr_proto_nested_describe_ex(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None if pr is None else pr.ctypes.data,
                                                    None if desc is None else desc.ctypes.data, 0 if desc is None else desc.size)


_CHAIN = [[F(1, S.PB_MESSAGE, False, m + 1)] for m in range(4)] + [[F(1, S.PB_INT32)]]
# the limits of the nested codec (test_descriptions_outside_the_limits_are_refused)
LIMIT_DESCRIPTIONS = [
    (MSGS, 0, CAP),
    ([[F(1, S.PB_MESSAGE, False, 0)]], 0, UNSUPPORTED),                                  # recursive type
    ([[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MESSAGE, True, 0)]], 0, UNSUPPORTED),    # mutually recursive
    ([[F(2, S.PB_INT32), F(1, S.PB_INT32)]], 0, INVALID),                                 # not in field-number order
    ([[F(1, S.PB_MESSAGE, False, 3)]], 0, INVALID),                                       # unknown message type
    ([[F(1, 10)]], 0, UNSUPPORTED),                                                       # TYPE_GROUP
    ([[F(0, S.PB_INT32)]], 0, INVALID), ([[F(19500, S.PB_INT32)]], 0, INVALID),            # reserved numbers
    (_CHAIN, 0, UNSUPPORTED),                                                             # 5 levels: too deep
    (_CHAIN[1:4] + [[F(1, S.PB_INT32)]], 0, INVALID),                                     # types 2..4 of four: unknown type 4
    ([[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MESSAGE, False, 2)], [F(1, S.PB_MESSAGE, False, 3)], [F(1, S.PB_INT32)]], 0, CAP),
]


def _one_map(key, value=S.PB_INT32, vmsg=0, number1=1, number2=2, extra=()):
    return [[F(1, S.PB_MAP, False, 1)], [F(number1, key), F(number2, value, False, vmsg)] + list(extra)]


_MAP_CHAIN = [[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MESSAGE, False, 2)], [F(1, S.PB_MAP, False, 3)], [F(1, S.PB_STRING), F(2, S.PB_INT32)]]
# map fields (test_proto_maps.py::test_descriptions)
MAP_DESCRIPTIONS = [(MAP_KA_MSGS, 0, CAP)] + [(_one_map(k), 0, CAP) for k in KEYS] + [
    (_one_map(S.PB_STRING, S.PB_MESSAGE, 2) + [[F(1, S.PB_INT32)]], 0, CAP),
    # an entry type serving two map fields, two levels down
    ([[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MAP, False, 2), F(2, S.PB_MAP, False, 2)], [F(1, S.PB_INT64), F(2, S.PB_BOOL)]], 0, CAP),
] + [(_one_map(k), 0, INVALID) for k in (S.PB_FLOAT, S.PB_DOUBLE, S.PB_BYTES, S.PB_ENUM)] + [   # key types Go does not allow
    (_one_map(S.PB_MESSAGE, S.PB_INT32) + [[F(1, S.PB_INT32)]], 0, INVALID),              # message key (msg 0: the root)
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_MESSAGE, False, 2), F(2, S.PB_INT32)], [F(1, S.PB_INT32)]], 0, INVALID),
    (_one_map(S.PB_INT32, number1=2, number2=3), 0, INVALID),                             # entry numbers other than 1, 2
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32)]], 0, INVALID),                      # one field only
    (_one_map(S.PB_INT32, extra=[F(3, S.PB_INT32)]), 0, INVALID),                        # three fields
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32, True), F(2, S.PB_INT32)]], 0, INVALID),   # repeated key
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32, True)]], 0, INVALID),   # repeated value
    ([[F(1, S.PB_MAP, True, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], 0, INVALID),          # a repeated map
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], 1, INVALID),         # entry type as root
    ([[F(1, S.PB_MAP, False, 1), F(2, S.PB_MESSAGE, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], 0, INVALID),  # as a message
    ([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_MAP, False, 2)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], 0, INVALID),  # map-valued
    ([[F(1, S.PB_MAP, False, 5)]], 0, INVALID),                                           # unknown entry type
    # limits: map<string, M> is two levels
    (_MAP_CHAIN, 0, CAP),
    ([[F(1, S.PB_MESSAGE, False, 1)]] + [[F(1, f.type, f.repeated, f.msg + 1) for f in t] for t in _MAP_CHAIN], 0, INVALID),
]


# ---------------------------------------------------------------------------------------------------------------
# python google.protobuf: classes built from descriptor_pb2 with map entries, oneof_decl and proto3_optional
# ---------------------------------------------------------------------------------------------------------------
def py_classes(msgs):
    """{message type: class}; map entry types get no class of their own (one nested entry type per map field)"""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fdp = descriptor_pb2.FileDescriptorProto(name="nested.proto", package="pn", syntax="proto3")
    entries = entry_types(msgs)

    def add_field(mt, f, name, oneof_index=None, optional=False):
        # an enum field encodes exactly like int32 (and would need an enum type here)
        kw = dict(name=name, number=f.number, type=S.PB_INT32 if f.type == S.PB_ENUM else f.type, label=3 if f.repeated else 1)
        if f.type == S.PB_MESSAGE:
            kw["type_name"] = ".pn.M%d" % f.msg
        fd = mt.field.add(**kw)
        if oneof_index is not None:
            fd.oneof_index = oneof_index
        if optional:
            fd.proto3_optional = True
    for m, fields in enumerate(msgs):
        if m in entries:
            continue
        mt = fdp.message_type.add(name="M%d" % m)
        groups = sorted({f.presence for f in fields if 1 <= f.presence <= 7})
        for g in groups:                                   # real oneofs first, the synthetic ones of optional fields after
            mt.oneof_decl.add(name="o%d" % g)
        n_real = len(groups)
        for f in fields:
            if f.presence == OPT:
                mt.oneof_decl.add(name="_f%d" % f.number)
                add_field(mt, f, "f%d" % f.number, n_real, optional=True)
                n_real += 1
                continue
            if f.type != S.PB_MAP:
                add_field(mt, f, "f%d" % f.number, groups.index(f.presence) if f.presence else None)
                continue
            e = mt.nested_type.add(name="F%dEntry" % f.number)
            e.options.map_entry = True
            add_field(e, msgs[f.msg][0], "key")
            add_field(e, msgs[f.msg][1], "value")
            mt.field.add(name="f%d" % f.number, number=f.number, type=11, label=3, type_name=".pn.M%d.F%dEntry" % (m, f.number))
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return {m: message_factory.GetMessageClass(pool.FindMessageTypeByName("pn.M%d" % m)) for m in range(len(msgs)) if m not in entries}


def _py_conv(t):
    return (lambda x: x.decode("utf-8") if isinstance(x, (bytes, bytearray)) else x) if t == S.PB_STRING else (lambda x: x)


def py_fill(classes, msgs, m, value):
    """the python protobuf message of a value list (maps as dicts or lists of pairs; unset explicit-presence fields None)"""
    obj = classes[m]()
    for f, v in zip(msgs[m], value):
        name = "f%d" % f.number
        conv = _py_conv(f.type)
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            field = getattr(obj, name)
            for k, x in (v.items() if isinstance(v, dict) else v):
                k = _py_conv(kf.type)(k)
                if vf.type == S.PB_MESSAGE:
                    field[k].CopyFrom(py_fill(classes, msgs, vf.msg, x) if x is not None else classes[vf.msg]())
                else:
                    field[k] = _py_conv(vf.type)(x)
        elif f.repeated:
            if f.type == S.PB_MESSAGE:
                for e in v:
                    getattr(obj, name).add().CopyFrom(py_fill(classes, msgs, f.msg, e))
            else:
                getattr(obj, name).extend([conv(e) for e in v])
        elif f.type == S.PB_MESSAGE:
            if v is not None:
                getattr(obj, name).CopyFrom(py_fill(classes, msgs, f.msg, v))
                getattr(obj, name).SetInParent()
        elif v is not None or not f.presence:                # an explicit-presence field is set by any assignment
            setattr(obj, name, conv(v))
    return obj


def py_to_value(msgs, m, obj):
    """the value list pack_proto_nested_rows takes (maps as dicts, unset explicit-presence fields None), from a parsed
    python protobuf message"""
    def conv(t, e):
        return e.encode("utf-8") if t == S.PB_STRING else e
    v = []
    for f in msgs[m]:
        name = "f%d" % f.number
        x = getattr(obj, name)
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            v.append({conv(kf.type, k): (py_to_value(msgs, vf.msg, y) if vf.type == S.PB_MESSAGE else conv(vf.type, y)) for k, y in x.items()})
        elif f.repeated:
            v.append([py_to_value(msgs, f.msg, e) for e in x] if f.type == S.PB_MESSAGE else [conv(f.type, e) for e in x])
        elif f.type == S.PB_MESSAGE:
            v.append(py_to_value(msgs, f.msg, x) if obj.HasField(name) else None)
        elif f.presence and not obj.HasField(name):
            v.append(None)
        else:
            v.append(conv(f.type, x))
    return v


def py_frames(msgs, root, values):
    """frames of python protobuf's default backend (deterministic=True), in this process"""
    classes = py_classes(msgs)
    return [frame(py_fill(classes, msgs, root, v).SerializeToString(deterministic=True)) for v in values]


def _pure_python_main():
    """child process, jobs pickled on stdin: ("enc", msgs, root, [values]) -> frames (deterministic=True); ("dec", msgs, root,
    [frame]) -> the value list each frame parses to, None where parsing fails"""
    from google.protobuf.internal import api_implementation
    from google.protobuf.message import DecodeError
    assert api_implementation.Type() == "python"
    jobs = pickle.load(sys.stdin.buffer)
    out = []
    for kind, msgs, root, items in jobs:
        classes = py_classes(msgs)
        res = []
        for x in items:
            if kind == "enc":
                res.append(frame(py_fill(classes, msgs, root, x).SerializeToString(deterministic=True)))
                continue
            obj = classes[root]()
            try:
                obj.ParseFromString(x[5:])
                res.append(py_to_value(msgs, root, obj))
            except (DecodeError, UnicodeDecodeError):   # the pure-Python backend reports invalid UTF-8 as the latter
                res.append(None)
        out.append(res)
    pickle.dump(out, sys.stdout.buffer)


def pure_python(jobs):
    """runs _pure_python_main's jobs in one child process: the backend is chosen when protobuf is first imported.  The
    pure-Python backend is the one to compare maps with: like protobuf-go it sorts map keys under deterministic=True and
    skips unknown fields inside a map entry, where upb (the default backend) does neither."""
    env = dict(os.environ, PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION="python")
    r = subprocess.run([sys.executable, "-c", "import tests.proto_nested_harness as h; h._pure_python_main()"], cwd=ROOT_DIR, env=env,
                       input=pickle.dumps(jobs), capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr.decode()[-4000:]
    return pickle.loads(r.stdout)


# ---------------------------------------------------------------------------------------------------------------
# the statements side by side
# ---------------------------------------------------------------------------------------------------------------
def encode_model_emu(msgs, root, rows, off, presence_instance=False):
    """model == device code (misalignments 0 and 3) on statuses, offsets and bytes; returns (frames, meta)"""
    frames, meta = M.encode(msgs, root, rows, off)
    want_off = np.cumsum([0] + [len(f) for f in frames]).astype(np.uint32)
    for mis in (0, 3):
        e_out, e_off, e_meta = emu.proto_encode_nested(msgs, root, rows, off, mis, presence_instance)
        assert list(e_meta) == meta, [(i, a, b) for i, (a, b) in enumerate(zip(list(e_meta), meta)) if a != b][:5]
        assert np.array_equal(e_off, want_off + mis)
        assert e_out[mis:int(e_off[-1])].tobytes() == b"".join(frames)
    return frames, meta


def decode_model_emu(msgs, root, frames, presence_instance=False):
    """model == device code on statuses, offsets and rows; returns (rows, meta)"""
    raw, in_off = pack_frames(frames)
    rows, meta = M.decode(msgs, root, frames)
    e_rows, e_off, e_meta = emu.proto_decode_nested(msgs, root, raw, in_off, presence_instance)
    assert list(e_meta) == meta, [(i, a, b, frames[i].hex()) for i, (a, b) in enumerate(zip(list(e_meta), meta)) if a != b][:5]
    assert np.array_equal(e_off, np.cumsum([0] + [len(r) for r in rows]).astype(np.uint32))
    for i, r in enumerate(rows):
        got = e_rows[int(e_off[i]):int(e_off[i + 1])].tobytes()
        assert got == r, (i, frames[i].hex(), got.hex(), r.hex())
    return rows, meta


def check_python_parse(msgs, root, frames, rows, meta):
    """wherever python protobuf (pure-Python backend) and the codec both accept a frame, the row is what python parsed; they
    agree on what parses"""
    parsed = pure_python([("dec", msgs, root, frames)])[0]
    for i, fr in enumerate(frames):
        if meta[i] in (M.COMPRESSED, M.BAD_LENGTH, M.DEFER):
            continue
        ok = parsed[i] is not None
        if ok and meta[i] == M.BAD_PROTO and has_overlong_varint(fr[5:]):
            continue      # protowire.ConsumeVarint refuses a tenth byte above 1; python protobuf truncates it
        assert ok == (meta[i] == M.OK), (i, fr.hex(), meta[i])
        if ok:
            want, _ = S.pack_proto_nested_rows(msgs, root, [parsed[i]])
            assert rows[i] == want[:len(rows[i])].tobytes() and len(rows[i]) == len(want) - 8, (i, fr.hex(), parsed[i])


def decode_three_ways(msgs, root, frames):
    """map- and presence-free: oracle == device code on everything; python protobuf (the default backend, in this process)
    decides what the rows of well-formed frames must be"""
    raw, off = pack_frames(frames)
    o_rows, o_off, o_meta = O.proto_decode_nested(msgs, root, raw, off)
    e_rows, e_off, e_meta = emu.proto_decode_nested(msgs, root, raw, off)
    assert np.array_equal(o_meta, e_meta), (o_meta, e_meta)
    assert np.array_equal(o_off, e_off)
    assert o_rows[:int(o_off[-1])].tobytes() == e_rows[:int(o_off[-1])].tobytes()
    classes = py_classes(msgs)
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
        if ok and o_meta[i] == S.GRPC_BAD_PROTO and has_overlong_varint(body):
            continue      # protowire.ConsumeVarint refuses a tenth byte above 1; upb silently truncates it
        assert ok == (o_meta[i] == S.GRPC_OK), (i, fr.hex(), o_meta[i], ok)
        if ok:
            want, _ = S.pack_proto_nested_rows(msgs, root, [py_to_value(msgs, root, obj)])
            got = o_rows[int(o_off[i]):int(o_off[i + 1])].tobytes()
            assert got == want[:len(got)].tobytes() and len(got) == (len(want) - 8 + 3) // 4 * 4, (i, fr.hex())
    return o_rows, o_off, o_meta


# ---------------------------------------------------------------------------------------------------------------
# the CUDA kernels against the model
# ---------------------------------------------------------------------------------------------------------------
def gpu_check(seed, make_types, make_value, spoil):
    """both nested kernels == the model (statuses, offsets, frames, rows) on three random type sets of 4 200 messages:
    make_types(rnd) -> msgs, make_value(rnd, msgs, 0) -> a value list, spoil(rnd, msgs, values) -> (rows, off, n): the
    rows with one in 53 made a row the encoder refuses (n of them).  The frames go back through the decoder with one in
    seven damaged.  Run it in a child process, so that a fault in a kernel cannot leave a sticky CUDA error in the process
    the other GPU tests run in."""
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    eng = Engine(Table(synth.config1_spec()), 0)
    checked = 0
    for _ in range(3):
        msgs = make_types(rnd)
        values = [make_value(rnd, msgs, 0) for _ in range(4200)]
        rows, off, spoiled = spoil(rnd, msgs, values)
        frames, meta = M.encode(msgs, 0, rows, off)
        assert meta.count(S.GRPC_BAD_ROW) >= spoiled
        d_out, d_off, d_meta = eng.proto_encode_nested_device(msgs, 0, rows, off)
        torch.cuda.synchronize()
        want_off = np.cumsum([0] + [len(f) for f in frames]).astype(np.uint32)
        assert np.array_equal(d_meta.cpu().numpy().view(np.uint32), np.array(meta, dtype=np.uint32))
        assert np.array_equal(d_off.cpu().numpy().view(np.uint32), want_off)
        assert d_out[:int(want_off[-1])].cpu().numpy().tobytes() == b"".join(frames)
        frames = [fr for fr in frames if fr]
        for i in range(0, len(frames), 7):           # every seventh frame damaged
            body = bytearray(frames[i][5:])
            if body:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            frames[i] = frame(bytes(body))
        raw, in_off = pack_frames(frames)
        rows2, meta2 = M.decode(msgs, 0, frames)
        g_rows, g_off, g_meta = eng.proto_decode_nested_device(msgs, 0, raw, in_off)
        torch.cuda.synchronize()
        want_off = np.cumsum([0] + [len(r) for r in rows2]).astype(np.uint32)
        assert np.array_equal(g_meta.cpu().numpy().view(np.uint32), np.array(meta2, dtype=np.uint32))
        assert np.array_equal(g_off.cpu().numpy().view(np.uint32), want_off)
        assert g_rows[:int(want_off[-1])].cpu().numpy().tobytes() == b"".join(rows2)
        checked += len(values)
    eng.close()
    assert checked >= 12000
    print("%d messages on the GPU, encode and decode equal to the model" % checked)


def run_child(code, timeout=900):
    """python -c code from the repository root; fails the test with the end of its output"""
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT_DIR, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return r.stdout
