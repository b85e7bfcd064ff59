"""Map fields (GOFR_PB_MAP) in the nested proto3 codec: gofr_proto_encode_nested_device / gofr_proto_decode_nested_device.

Reference behaviour: protobuf-go v1.32.0 impl/codec_map.go — a map is a repeated entry message (1 key, 2 value); marshalling
writes key and value at their zero values too and a message value always; Deterministic marshalling sorts the keys;
unmarshalling lets the last key / value inside an entry win and a later entry replace an earlier one with an equal key.
Statements compared:
  tests/proto_maps_model.py   recursive; the decoder collects the entries, stable-sorts them and keeps the last of equal keys
  the device code             explicit stacks, the decoder selects the next key by rescanning — on the CPU via tests/emu
                              (output misalignments 0 and 3) and, with -m gpu, in the CUDA kernels
  python google.protobuf      the pure-Python backend for BYTES (its deterministic=True sorts keys like Go; upb does not),
                              the default backend for what a frame parses to (dict equality)."""
import os
import pickle
import random
import subprocess
import sys
from functools import lru_cache

import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200 import _abi
from tests import oracle as O
from tests import proto_maps_model as PM
from tests.emu import emu
from tests.test_proto_nested import (MSGS, SCALARS, _frame, _frames, _has_overlong_varint, _pack_frames, _rand_scalar, _rand_types,
                                     _rand_value, _varint)

F = S.ProtoNField
ROOT_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = [S.PB_INT32, S.PB_INT64, S.PB_UINT32, S.PB_UINT64, S.PB_SINT32, S.PB_SINT64, S.PB_FIXED32, S.PB_FIXED64, S.PB_SFIXED32,
        S.PB_SFIXED64, S.PB_BOOL, S.PB_STRING]


# ---------------------------------------------------------------------------------------------------------------
# python google.protobuf with map fields: one nested entry type per map field (options.map_entry)
# ---------------------------------------------------------------------------------------------------------------
def _entry_types(msgs):
    return {f.msg for fields in msgs for f in fields if f.type == S.PB_MAP}


def _py_classes(msgs):
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fdp = descriptor_pb2.FileDescriptorProto(name="maps.proto", package="mp", syntax="proto3")
    entries = _entry_types(msgs)

    def add_field(mt, f, name):
        kw = dict(name=name, number=f.number, type=S.PB_INT32 if f.type == S.PB_ENUM else f.type, label=3 if f.repeated else 1)
        if f.type == S.PB_MESSAGE:
            kw["type_name"] = ".mp.M%d" % f.msg
        mt.field.add(**kw)
    for m, fields in enumerate(msgs):
        if m in entries:
            continue
        mt = fdp.message_type.add(name="M%d" % m)
        for f in fields:
            if f.type != S.PB_MAP:
                add_field(mt, f, "f%d" % f.number)
                continue
            e = mt.nested_type.add(name="F%dEntry" % f.number)
            e.options.map_entry = True
            add_field(e, msgs[f.msg][0], "key")
            add_field(e, msgs[f.msg][1], "value")
            mt.field.add(name="f%d" % f.number, number=f.number, type=11, label=3, type_name=".mp.M%d.F%dEntry" % (m, f.number))
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return {m: message_factory.GetMessageClass(pool.FindMessageTypeByName("mp.M%d" % m)) for m in range(len(msgs)) if m not in entries}


def _py_conv(t):
    return (lambda x: x.decode("utf-8") if isinstance(x, (bytes, bytearray)) else x) if t == S.PB_STRING else (lambda x: x)


def _py_fill(classes, msgs, m, value):
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
                    field[k].CopyFrom(_py_fill(classes, msgs, vf.msg, x) if x is not None else classes[vf.msg]())
                else:
                    field[k] = _py_conv(vf.type)(x)
        elif f.repeated:
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


def _py_to_value(msgs, m, obj):
    """the value list pack_proto_nested_rows takes (maps as dicts), from a parsed python protobuf message"""
    def conv(t, e):
        return e.encode("utf-8") if t == S.PB_STRING else e
    v = []
    for f in msgs[m]:
        x = getattr(obj, "f%d" % f.number)
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            v.append({conv(kf.type, k): (_py_to_value(msgs, vf.msg, y) if vf.type == S.PB_MESSAGE else conv(vf.type, y)) for k, y in x.items()})
        elif f.repeated:
            v.append([_py_to_value(msgs, f.msg, e) for e in x] if f.type == S.PB_MESSAGE else [conv(f.type, e) for e in x])
        elif f.type == S.PB_MESSAGE:
            v.append(_py_to_value(msgs, f.msg, x) if obj.HasField("f%d" % f.number) else None)
        else:
            v.append(conv(f.type, x))
    return v


def _pure_python_main():
    """child process, jobs pickled on stdin: ("enc", msgs, root, [values]) -> frames (deterministic=True); ("dec", msgs, root,
    [frame]) -> the value list each frame parses to (maps as dicts), None where parsing fails"""
    from google.protobuf.internal import api_implementation
    from google.protobuf.message import DecodeError
    assert api_implementation.Type() == "python"
    jobs = pickle.load(sys.stdin.buffer)
    out = []
    for kind, msgs, root, items in jobs:
        classes = _py_classes(msgs)
        res = []
        for x in items:
            if kind == "enc":
                res.append(_frame(_py_fill(classes, msgs, root, x).SerializeToString(deterministic=True)))
                continue
            obj = classes[root]()
            try:
                obj.ParseFromString(x[5:])
                res.append(_py_to_value(msgs, root, obj))
            except (DecodeError, UnicodeDecodeError):   # the pure-Python backend reports invalid UTF-8 as the latter
                res.append(None)
        out.append(res)
    pickle.dump(out, sys.stdout.buffer)


def _pure_python(jobs):
    """runs _pure_python_main's jobs in one child process: the backend is chosen when protobuf is first imported"""
    env = dict(os.environ, PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION="python")
    r = subprocess.run([sys.executable, "-c", "import tests.test_proto_maps as t; t._pure_python_main()"], cwd=ROOT_DIR, env=env,
                       input=pickle.dumps(jobs), capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr.decode()[-4000:]
    return pickle.loads(r.stdout)


def _pure_python_frames(cases):
    """[(msgs, root, values)] -> [[frame]]"""
    return _pure_python([("enc", m, r, v) for m, r, v in cases])


# ---------------------------------------------------------------------------------------------------------------
# the statements side by side
# ---------------------------------------------------------------------------------------------------------------
def _encode_model_emu(msgs, root, rows, off):
    """model == device code (misalignments 0 and 3) on statuses, offsets and bytes; returns (frames, meta)"""
    frames, meta = PM.encode(msgs, root, rows, off)
    want_off = np.cumsum([0] + [len(f) for f in frames]).astype(np.uint32)
    for mis in (0, 3):
        e_out, e_off, e_meta = emu.proto_encode_nested(msgs, root, rows, off, mis)
        assert list(e_meta) == meta, (list(e_meta), meta)
        assert np.array_equal(e_off, want_off + mis)
        assert e_out[mis:int(e_off[-1])].tobytes() == b"".join(frames)
    return frames, meta


def _decode_model_emu(msgs, root, frames):
    """model == device code on statuses, offsets and rows; returns (rows, meta)"""
    raw, in_off = _pack_frames(frames)
    rows, meta = PM.decode(msgs, root, frames)
    e_rows, e_off, e_meta = emu.proto_decode_nested(msgs, root, raw, in_off)
    assert list(e_meta) == meta, [(i, a, b, frames[i].hex()) for i, (a, b) in enumerate(zip(list(e_meta), meta)) if a != b][:5]
    assert np.array_equal(e_off, np.cumsum([0] + [len(r) for r in rows]).astype(np.uint32))
    for i, r in enumerate(rows):
        got = e_rows[int(e_off[i]):int(e_off[i + 1])].tobytes()
        assert got == r, (i, frames[i].hex(), got.hex(), r.hex())
    return rows, meta


def _check_python_parse(msgs, root, frames, rows, meta):
    """wherever python protobuf and the codec both accept a frame, the row is the parsed map in canonical form.  The
    pure-Python backend parses: like protobuf-go it skips unknown fields inside a map entry, where upb (the default
    backend) keeps such an entry out of the map, as an unknown field of the parent."""
    parsed = _pure_python([("dec", msgs, root, frames)])[0]
    for i, fr in enumerate(frames):
        if meta[i] in (PM.COMPRESSED, PM.BAD_LENGTH, PM.DEFER):
            continue
        ok = parsed[i] is not None
        if ok and meta[i] == PM.BAD_PROTO and _has_overlong_varint(fr[5:]):
            continue      # protowire.ConsumeVarint refuses a tenth byte above 1; python protobuf truncates it
        assert ok == (meta[i] == PM.OK), (i, fr.hex(), meta[i])
        if ok:
            want, _ = S.pack_proto_nested_rows(msgs, root, [parsed[i]])
            assert rows[i] == want[:len(rows[i])].tobytes() and len(rows[i]) == len(want) - 8, (i, fr.hex())


# ---------------------------------------------------------------------------------------------------------------
# known answers
# ---------------------------------------------------------------------------------------------------------------
# M { map<string,int32> s = 1; map<int32,string> i = 2; map<bool,V> b = 3; map<uint64,bytes> u = 4; map<sint64,double> z = 5; }
KA_MSGS = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 2), F(3, S.PB_MAP, False, 3), F(4, S.PB_MAP, False, 5), F(5, S.PB_MAP, False, 6)],
           [F(1, S.PB_STRING), F(2, S.PB_INT32)],
           [F(1, S.PB_INT32), F(2, S.PB_STRING)],
           [F(1, S.PB_BOOL), F(2, S.PB_MESSAGE, False, 4)],
           [F(1, S.PB_INT32)],                                     # V { int32 x = 1; }
           [F(1, S.PB_UINT64), F(2, S.PB_BYTES)],
           [F(1, S.PB_SINT64), F(2, S.PB_DOUBLE)]]
KA = [({"b": 2, "a": 0, "": -1}, 0, "0a0d0a0010ffffffffffffffffff01" "0a050a01611000" "0a050a01621002"),
      ({7: "x", -1: ""}, 1, "120d08ffffffffffffffffff011200" "12050807120178"),
      ({True: [0]}, 2, "1a0408011200"),
      ({2 ** 64 - 1: b""}, 3, "220d08ffffffffffffffffff011200"),
      ({-1: -0.0}, 4, "2a0b0801110000000000000080")]


def test_known_answers():
    values = []
    for m, slot, _ in KA:
        v = [{}, {}, {}, {}, {}]
        v[slot] = m
        values.append(v)
    values.append([dict(KA[k][0]) for k in range(5)])
    rows, off = S.pack_proto_nested_rows(KA_MSGS, 0, values)
    frames, meta = _encode_model_emu(KA_MSGS, 0, rows, off)
    assert meta == [0] * len(values)
    for k, (_, _, hexs) in enumerate(KA):
        assert frames[k] == _frame(bytes.fromhex(hexs)), (k, frames[k].hex())
    assert frames[-1] == _frame(bytes.fromhex("".join(h for _, _, h in KA)))
    assert _pure_python_frames([(KA_MSGS, 0, values)])[0] == frames
    d_rows, d_meta = _decode_model_emu(KA_MSGS, 0, frames)
    assert d_meta == [0] * len(values)
    assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]


def test_model_equals_oracle_without_maps():
    """the model restates the nested codec as a whole: on map-free types it answers as the oracle does"""
    rnd = random.Random(4)
    for _ in range(6):
        msgs = _rand_types(rnd)
        values = [_rand_value(rnd, msgs, 0) for _ in range(40)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        o_out, o_off, o_meta = O.proto_encode_nested(msgs, 0, rows, off)
        frames, meta = PM.encode(msgs, 0, rows, off)
        assert list(o_meta) == meta and _frames(o_out, o_off) == frames
        raw, in_off = _pack_frames(frames)
        d_rows, d_off, d_meta = O.proto_decode_nested(msgs, 0, raw, in_off)
        rows2, meta2 = PM.decode(msgs, 0, frames)
        assert list(d_meta) == meta2 and [d_rows[int(d_off[i]):int(d_off[i + 1])].tobytes() for i in range(len(frames))] == rows2


# ---------------------------------------------------------------------------------------------------------------
# random type sets with map fields
# ---------------------------------------------------------------------------------------------------------------
def _rand_map_types(rnd):
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
    if not _entry_types(msgs) or sum(len(f) for f in msgs) > 48:
        return _rand_map_types(rnd)
    return msgs


def _rand_key(rnd, t):
    if t == S.PB_STRING:
        return rnd.choice(["", "a", "b", "ab", "aa", "a\x00", "é", "日本", "zz" * 20, "k%d" % rnd.randint(0, 99)])
    return _rand_scalar(rnd, t)


def _rand_map_value(rnd, msgs, m, nil_values=True):
    v = []
    for f in msgs[m]:
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            d = {}
            for _ in range(rnd.choice([0, 0, 1, 2, 3, 8])):
                if vf.type == S.PB_MESSAGE:
                    x = None if nil_values and rnd.random() < 0.2 else _rand_map_value(rnd, msgs, vf.msg, nil_values)
                else:
                    x = _rand_scalar(rnd, vf.type)
                d[_rand_key(rnd, kf.type)] = x
            v.append(d)
        elif f.type == S.PB_MESSAGE:
            one = lambda: _rand_map_value(rnd, msgs, f.msg, nil_values)  # noqa: E731
            v.append([one() for _ in range(rnd.choice([0, 1, 2]))] if f.repeated else None if rnd.random() < 0.4 else one())
        elif f.repeated:
            v.append([_rand_scalar(rnd, f.type) for _ in range(rnd.choice([0, 1, 3]))])
        else:
            v.append(_rand_scalar(rnd, f.type))
    return v


ENC_SEEDS = range(25)


@lru_cache(maxsize=None)
def _enc_cases():
    cases = []
    for seed in ENC_SEEDS:
        rnd = random.Random(1300 + seed)
        msgs = _rand_map_types(rnd)
        cases.append((msgs, 0, [_rand_map_value(rnd, msgs, 0) for _ in range(40)]))
    return cases, _pure_python_frames(cases)


@pytest.mark.parametrize("seed", ENC_SEEDS)
def test_random_map_types_encode(seed):
    """model == device code == pure-Python deterministic bytes"""
    cases, py = _enc_cases()
    msgs, root, values = cases[seed]
    assert _abi.lib().gofr_proto_nested_describe(*_tables(msgs), root, None, 0) == CAP
    rows, off = S.pack_proto_nested_rows(msgs, root, values)
    frames, meta = _encode_model_emu(msgs, root, rows, off)
    assert meta == [0] * len(values)
    for i in range(len(values)):
        assert frames[i] == py[seed][i], (i, values[i], frames[i].hex(), py[seed][i].hex())


def test_bad_rows():
    """unsorted and duplicate keys, truncations, invalid UTF-8 in keys and values: BAD_ROW / BAD_UTF8, model == device code"""
    msgs = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 2), F(3, S.PB_MAP, False, 3)],
            [F(1, S.PB_STRING), F(2, S.PB_STRING)], [F(1, S.PB_SINT64), F(2, S.PB_MESSAGE, False, 4)], [F(1, S.PB_BOOL), F(2, S.PB_UINT32)],
            [F(1, S.PB_MAP, False, 5), F(2, S.PB_INT32, True)], [F(1, S.PB_UINT32), F(2, S.PB_BYTES)]]
    V = lambda s=(), z=(), b=(): [list(s), list(z), list(b)]  # noqa: E731  (lists of pairs: laid out as given)
    inner = [[(2 ** 32 - 1, b"x"), (0, b"")], [1]]               # unsorted uint32 keys inside a message value
    vals = [V(s=[("a", "1"), ("b", "2")], z=[(-5, None), (3, [[(1, b"")], []])], b=[(False, 0), (True, 7)]),   # fine
            V(s=[("b", "1"), ("a", "2")]),                        # unsorted string keys
            V(s=[("a", "1"), ("a", "2")]),                        # duplicate
            V(s=[("ab", ""), ("a", "")]),                         # a longer key before its prefix
            V(z=[(3, None), (-5, None)]),                         # signed order
            V(z=[(-1, None), (-1, None)]),
            V(z=[(0, [inner[0], []])]),                           # nested map out of order
            V(b=[(True, 0), (False, 0)]),
            V(b=[(True, 0), (True, 0)]),
            V(s=[("\udcff", "v")]),                               # invalid UTF-8 key
            V(s=[("k", b"\xc3")]),                                # invalid UTF-8 value
            V(s=[("b", b"\xff"), ("a", "")]),                     # invalid UTF-8 before the disorder: BAD_UTF8 first
            V(s=[("b", ""), ("a", b"\xff")]),                     # disorder before the invalid UTF-8: BAD_ROW first
            V(s=[("", ""), ("a", "")], z=[(-(2 ** 63), None), (2 ** 63 - 1, None)])]  # fine: the extremes in order
    rows, off = S.pack_proto_nested_rows(msgs, 0, vals)
    _, meta = _encode_model_emu(msgs, 0, rows, off)
    R, U = S.GRPC_BAD_ROW, S.GRPC_BAD_UTF8
    assert meta == [0, R, R, R, R, R, R, R, R, U, U, U, R, 0], meta
    # truncations of a valid row, and entry counts that promise more than the row holds
    r0 = rows[int(off[0]):int(off[1])].tobytes()
    blobs = [r0[:k] + b"\0" * ((-k) % 4) for k in range(0, len(r0), 2)]
    blobs += [(0x00FFFFFF).to_bytes(4, "little") + bytes(8), (3).to_bytes(4, "little") + bytes(8) + bytes(12)]
    body, offs = bytearray(), [0]
    for b in blobs:
        body += b
        offs.append(len(body))
    rows2 = np.frombuffer(bytes(body) + b"\0" * 16, dtype=np.uint8).copy()
    _, meta2 = _encode_model_emu(msgs, 0, rows2, np.array(offs, dtype=np.uint32))
    assert meta2.count(R) >= len(blobs) // 2 and meta2[-2] == R


# ---------------------------------------------------------------------------------------------------------------
# the decoder
# ---------------------------------------------------------------------------------------------------------------
def test_decode_round_trip():
    """decode(encode(row)) == row for rows whose message values are present; python protobuf parses the same maps"""
    rnd = random.Random(21)
    for msgs in [KA_MSGS] + [_rand_map_types(rnd) for _ in range(6)]:
        values = [_rand_map_value(rnd, msgs, 0, nil_values=False) for _ in range(50)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = _encode_model_emu(msgs, 0, rows, off)
        assert meta == [0] * len(values)
        d_rows, d_meta = _decode_model_emu(msgs, 0, frames)
        assert d_meta == meta
        assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]
        _check_python_parse(msgs, 0, frames, d_rows, d_meta)


def _entry(num, body):
    return _varint(num << 3 | 2) + _varint(len(body)) + body


def _s(num, b):
    return _varint(num << 3 | 2) + _varint(len(b)) + b


# M { map<string, V> a = 1; map<int32, int64> b = 2; map<bool, string> c = 3; int32 d = 4; }  V { int32 x = 1; map<uint64, bytes> y = 2; }
NONCANON_MSGS = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 2), F(3, S.PB_MAP, False, 3), F(4, S.PB_INT32)],
                 [F(1, S.PB_STRING), F(2, S.PB_MESSAGE, False, 4)], [F(1, S.PB_INT32), F(2, S.PB_INT64)], [F(1, S.PB_BOOL), F(2, S.PB_STRING)],
                 [F(1, S.PB_INT32), F(2, S.PB_MAP, False, 5)], [F(1, S.PB_UINT64), F(2, S.PB_BYTES)]]
_V1, _V2 = b"\x08\x01", b"\x08\x02" + _entry(2, b"\x08\x05\x12\x01z")


def _A(k, v):
    return _entry(1, _s(1, k) + _s(2, v))


def _B(k, v):
    return _entry(2, b"\x08" + _varint(k & (2 ** 64 - 1)) + b"\x10" + _varint(v & (2 ** 64 - 1)))


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


def test_decode_noncanonical_frames():
    msgs, ok, defer, bad = NONCANON_MSGS, NONCANON_OK, NONCANON_DEFER, NONCANON_BAD
    frames = [_frame(b) for b in ok + defer + bad]
    rows, meta = _decode_model_emu(msgs, 0, frames)
    D, P, U = S.GRPC_DEFER, S.GRPC_BAD_PROTO, S.GRPC_BAD_UTF8
    assert meta == [0] * len(ok) + [D] * len(defer) + [U, U, U, P, P, P, P, U], meta
    _check_python_parse(msgs, 0, frames, rows, meta)
    # spot values: the shuffled map comes back in key order, message values always present
    want, _ = S.pack_proto_nested_rows(msgs, 0, [[{"": [0, {}], "a": [2, {5: b"z"}], "b": [1, {}]}, {}, {}, 0]])
    assert rows[0] == want[:len(rows[0])].tobytes()
    want, _ = S.pack_proto_nested_rows(msgs, 0, [[{"a": [1, {}]}, {-3: 2, 3: 9}, {}, 0]])
    assert rows[2] == want[:len(rows[2])].tobytes()
    want, _ = S.pack_proto_nested_rows(msgs, 0, [[{}, {k: k for k in range(64)}, {}, 0]])
    assert rows[13] == want[:len(rows[13])].tobytes()


MUT_SEEDS = range(20)


@pytest.mark.parametrize("seed", MUT_SEEDS)
def test_decode_mutated_frames(seed):
    """frames of random map types with bytes flipped, inserted, cut and rotated: model == device code on status, offsets
    and rows; python protobuf agrees where both parse"""
    rnd = random.Random(2100 + seed)
    msgs = _rand_map_types(rnd)
    values = [_rand_map_value(rnd, msgs, 0) for _ in range(50)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, _ = PM.encode(msgs, 0, rows, off)
    out = []
    for fr in frames:
        body = bytearray(fr[5:])
        for _ in range(rnd.randint(0, 3)):
            r = rnd.random()
            if body and r < 0.35:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            elif body and r < 0.5:
                del body[rnd.randrange(len(body)):]
            elif r < 0.75:
                p = rnd.randrange(len(body) + 1)
                body[p:p] = rnd.choice([b"\x08\x01", b"\x0b\x0c", b"\x12\x00", b"\x0a\x00", b"\x0a\x02\x08\x01", b"\x0d\x00\x00\x00\x00", b"\x80"])
            else:       # move the tail in front: entries and fields arrive in any order
                p = rnd.randrange(len(body) + 1)
                body = body[p:] + body[:p]
        out.append(_frame(bytes(body)))
    d_rows, d_meta = _decode_model_emu(msgs, 0, out)
    _check_python_parse(msgs, 0, out, d_rows, d_meta)


# ---------------------------------------------------------------------------------------------------------------
# descriptions
# ---------------------------------------------------------------------------------------------------------------
CAP = 7   # GOFR_ERR_CAPACITY: "valid, but no room to write the descriptor"


def _tables(msgs):
    nm, nf, k = S.proto_nested_tables(msgs)
    return nm.ctypes.data, len(msgs), nf.ctypes.data, k


def test_descriptions():
    L = _abi.lib()

    def describe(msgs, root=0):
        nm, nf, k = S.proto_nested_tables(msgs)
        return L.gofr_proto_nested_describe(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None, 0)

    def one_map(key, value=S.PB_INT32, vmsg=0, number1=1, number2=2, extra=()):
        return [[F(1, S.PB_MAP, False, 1)], [F(number1, key), F(number2, value, False, vmsg)] + list(extra)]
    assert describe(KA_MSGS) == CAP
    for k in KEYS:
        assert describe(one_map(k)) == CAP, k
    assert describe(one_map(S.PB_STRING, S.PB_MESSAGE, 2) + [[F(1, S.PB_INT32)]]) == CAP
    # an entry type serving two map fields, two levels down
    assert describe([[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MAP, False, 2), F(2, S.PB_MAP, False, 2)], [F(1, S.PB_INT64), F(2, S.PB_BOOL)]]) == CAP
    INV = 1   # GOFR_ERR_INVALID
    for k in (S.PB_FLOAT, S.PB_DOUBLE, S.PB_BYTES, S.PB_ENUM):
        assert describe(one_map(k)) == INV, k                                           # key types Go does not allow
    assert describe(one_map(S.PB_MESSAGE, S.PB_INT32) + [[F(1, S.PB_INT32)]]) == INV    # message key (msg 0: the root)
    assert describe([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_MESSAGE, False, 2), F(2, S.PB_INT32)], [F(1, S.PB_INT32)]]) == INV
    assert describe(one_map(S.PB_INT32, number1=2, number2=3)) == INV                   # entry numbers other than 1, 2
    assert describe([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32)]]) == INV            # one field only
    assert describe(one_map(S.PB_INT32, extra=[F(3, S.PB_INT32)])) == INV              # three fields
    assert describe([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32, True), F(2, S.PB_INT32)]]) == INV   # repeated key
    assert describe([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32, True)]]) == INV   # repeated value
    assert describe([[F(1, S.PB_MAP, True, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]]) == INV          # a repeated map
    assert describe([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], root=1) == INV  # entry type as root
    assert describe([[F(1, S.PB_MAP, False, 1), F(2, S.PB_MESSAGE, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]]) == INV  # as a message
    assert describe([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_MAP, False, 2)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]]) == INV  # map-valued
    assert describe([[F(1, S.PB_MAP, False, 5)]]) == INV                                 # unknown entry type
    # limits: map<string, M> is two levels
    chain = [[F(1, S.PB_MESSAGE, False, 1)], [F(1, S.PB_MESSAGE, False, 2)], [F(1, S.PB_MAP, False, 3)], [F(1, S.PB_STRING), F(2, S.PB_INT32)]]
    assert describe(chain) == CAP
    assert describe([[F(1, S.PB_MESSAGE, False, 1)]] + [[F(1, f.type, f.repeated, f.msg + 1) for f in t] for t in chain]) != CAP


def test_descriptor_size_unchanged():
    lib = emu.lib()
    import ctypes
    lib.emu_pbn_desc_bytes.restype = ctypes.c_uint32
    assert lib.emu_pbn_desc_bytes() == 440


# ---------------------------------------------------------------------------------------------------------------
# the CUDA kernels
# ---------------------------------------------------------------------------------------------------------------
def _gpu_check():
    """the body of test_gpu_maps_match_model (run in a process of its own)"""
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(91)
    eng = Engine(Table(synth.config1_spec()), 0)
    checked = 0
    for _ in range(3):
        msgs = _rand_map_types(rnd)
        values = [_rand_map_value(rnd, msgs, 0) for _ in range(4200)]
        for i in range(0, len(values), 53):          # a few rows the encoder refuses: a duplicate key
            for f, v in zip(msgs[0], values[i]):
                if f.type == S.PB_MAP and v:
                    k = next(iter(v))
                    values[i][msgs[0].index(f)] = [(k, v[k]), (k, v[k])]
                    break
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = PM.encode(msgs, 0, rows, off)
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
            frames[i] = _frame(bytes(body))
        raw, in_off = _pack_frames(frames)
        rows2, meta2 = PM.decode(msgs, 0, frames)
        g_rows, g_off, g_meta = eng.proto_decode_nested_device(msgs, 0, raw, in_off)
        torch.cuda.synchronize()
        want_off = np.cumsum([0] + [len(r) for r in rows2]).astype(np.uint32)
        assert np.array_equal(g_meta.cpu().numpy().view(np.uint32), np.array(meta2, dtype=np.uint32))
        assert np.array_equal(g_off.cpu().numpy().view(np.uint32), want_off)
        assert g_rows[:int(want_off[-1])].cpu().numpy().tobytes() == b"".join(rows2)
        checked += len(values)
    eng.close()
    assert checked >= 12000
    print("maps on the GPU: %d messages, encode and decode equal to the model" % checked)


@pytest.mark.gpu
def test_gpu_maps_match_model():
    """both kernels with map fields == the model (statuses, offsets, frames, rows) — in a child process, so that a fault in a
    kernel cannot leave a sticky CUDA error in the process the other GPU tests run in"""
    r = subprocess.run([sys.executable, "-c", "import tests.test_proto_maps as t; t._gpu_check()"], cwd=ROOT_DIR,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
