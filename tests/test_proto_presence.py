"""Field presence in the nested proto3 codec: proto3 `optional` fields and `oneof` groups (ProtoNField.presence), through
gofr_proto_encode_nested_ex_device / gofr_proto_decode_nested_ex_device / gofr_proto_nested_describe_ex.

Reference behaviour: protobuf-go v1.32.0 — proto.Marshal writes a set explicit-presence field even at its zero value or
empty, an unset one not at all, every oneof member at its own number in field-number order; proto.Unmarshal sets an
optional field iff it occurs, and sets the oneof member whose occurrence is last among the group's members.  A message
member occurring twice is GOFR_GRPC_DEFER (protobuf-go merges or replaces; either way the host decodes it).
Statements compared:
  tests/proto_presence_model.py   the maps model with presence: recursive, list-first, the set member is the one holding the
                              group's last wire position
  the device code             one pass per field — on the CPU via tests/emu's nested exports (the descriptor picks the
                              presence instance, as on the host; output misalignments 0 and 3) and, with -m gpu, in
                              proto_encode_nested_presence_kernel / proto_decode_nested_presence_kernel
  python google.protobuf      the pure-Python backend in a child process (map fields are mixed in: upb neither sorts map keys
                              under deterministic=True nor skips unknown fields inside an entry), classes built from
                              descriptor_pb2 with oneof_decl / oneof_index, and proto3_optional with its synthetic oneof."""
import ctypes
import dataclasses
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
from tests import proto_maps_model as PM
from tests import proto_presence_model as PP
from tests.emu import emu
from tests.test_proto_maps import _entry_types, _rand_key, _rand_map_types
from tests.test_proto_nested import _frame, _has_overlong_varint, _pack_frames, _rand_scalar, _rand_types

F = S.ProtoNField
OPT = S.PB_OPTIONAL
ROOT_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, CAP = 1, 7   # GOFR_ERR_INVALID; GOFR_ERR_CAPACITY = "valid, but no room to write the descriptor"


# ---------------------------------------------------------------------------------------------------------------
# python google.protobuf with presence (pure-Python backend, child process)
# ---------------------------------------------------------------------------------------------------------------
def _py_classes(msgs):
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fdp = descriptor_pb2.FileDescriptorProto(name="presence.proto", package="pp", syntax="proto3")
    entries = _entry_types(msgs)

    def add_field(mt, f, name, oneof_index=None, optional=False):
        kw = dict(name=name, number=f.number, type=S.PB_INT32 if f.type == S.PB_ENUM else f.type, label=3 if f.repeated else 1)
        if f.type == S.PB_MESSAGE:
            kw["type_name"] = ".pp.M%d" % f.msg
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
            mt.field.add(name="f%d" % f.number, number=f.number, type=11, label=3, type_name=".pp.M%d.F%dEntry" % (m, f.number))
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return {m: message_factory.GetMessageClass(pool.FindMessageTypeByName("pp.M%d" % m)) for m in range(len(msgs)) if m not in entries}


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
        elif v is not None or not f.presence:                # an explicit-presence field is set by any assignment
            setattr(obj, name, conv(v))
    return obj


def _py_to_value(msgs, m, obj):
    """the value list pack_proto_nested_rows takes (maps as dicts, unset explicit-presence fields None)"""
    def conv(t, e):
        return e.encode("utf-8") if t == S.PB_STRING else e
    v = []
    for f in msgs[m]:
        name = "f%d" % f.number
        x = getattr(obj, name)
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            v.append({conv(kf.type, k): (_py_to_value(msgs, vf.msg, y) if vf.type == S.PB_MESSAGE else conv(vf.type, y)) for k, y in x.items()})
        elif f.repeated:
            v.append([_py_to_value(msgs, f.msg, e) for e in x] if f.type == S.PB_MESSAGE else [conv(f.type, e) for e in x])
        elif f.type == S.PB_MESSAGE:
            v.append(_py_to_value(msgs, f.msg, x) if obj.HasField(name) else None)
        elif f.presence and not obj.HasField(name):
            v.append(None)
        else:
            v.append(conv(f.type, x))
    return v


def _pure_python_main():
    """child process, jobs pickled on stdin: ("enc", msgs, root, [values]) -> frames (deterministic=True); ("dec", msgs, root,
    [frame]) -> the value list each frame parses to, None where parsing fails"""
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
    env = dict(os.environ, PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION="python")
    r = subprocess.run([sys.executable, "-c", "import tests.test_proto_presence as t; t._pure_python_main()"], cwd=ROOT_DIR, env=env,
                       input=pickle.dumps(jobs), capture_output=True, timeout=600)
    assert r.returncode == 0, r.stderr.decode()[-4000:]
    return pickle.loads(r.stdout)


# ---------------------------------------------------------------------------------------------------------------
# the device code on the CPU: tests/emu's nested exports run the instance the descriptor picks (pbn_size /
# pdn_decode_size dispatch on PbnDesc::presence, then ::maps, as the host picks the kernels)
# ---------------------------------------------------------------------------------------------------------------
def _emu_desc(msgs, root, presence_instance):
    """the descriptor of gofr_proto_nested_describe_ex; presence_instance: its presence byte (byte 1) set whatever the
    description, so that the presence instance runs a presence-free description too"""
    desc = np.zeros(512, np.uint8)
    assert _describe(msgs, root, desc) == 0, _last_error()
    if presence_instance:
        desc[1] = 1
    return desc


def _emu_encode(msgs, root, rows, row_off, misalign, presence_instance):
    n = len(row_off) - 1
    desc = _emu_desc(msgs, root, presence_instance)
    cap = int(rows.size) * 4 + 64 * n + 64 + misalign
    out = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    rows = np.concatenate([np.ascontiguousarray(rows), np.zeros(16, np.uint8)])
    fn = emu.lib().emu_proto_encode_nested
    fn.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32]
    assert fn(desc.ctypes.data, rows.ctypes.data, row_off.ctypes.data, n, out.ctypes.data, cap, off.ctypes.data, meta.ctypes.data, misalign) == 0
    return out, off, meta[:n]


def _emu_decode(msgs, root, frames, in_off, presence_instance):
    n = len(in_off) - 1
    desc = _emu_desc(msgs, root, presence_instance)
    cap = int(frames.size) * 10 + 4096 * max(n, 1)
    rows = np.full(cap, 0xEE, dtype=np.uint8)
    off = np.zeros(n + 1, dtype=np.uint32)
    meta = np.zeros(max(n, 1), dtype=np.uint32)
    frames = np.concatenate([np.ascontiguousarray(frames), np.zeros(16, np.uint8)])
    fn = emu.lib().emu_proto_decode_nested
    fn.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
    assert fn(desc.ctypes.data, frames.ctypes.data, in_off.ctypes.data, n, rows.ctypes.data, cap, off.ctypes.data, meta.ctypes.data) == 0
    return rows, off, meta[:n]


# ---------------------------------------------------------------------------------------------------------------
# the statements side by side
# ---------------------------------------------------------------------------------------------------------------
def _encode_model_emu(msgs, root, rows, off, presence_instance=False):
    """model == device code (misalignments 0 and 3) on statuses, offsets and bytes; returns (frames, meta)"""
    frames, meta = PP.encode(msgs, root, rows, off)
    want_off = np.cumsum([0] + [len(f) for f in frames]).astype(np.uint32)
    for mis in (0, 3):
        e_out, e_off, e_meta = _emu_encode(msgs, root, rows, off, mis, presence_instance)
        assert list(e_meta) == meta, [(i, a, b) for i, (a, b) in enumerate(zip(list(e_meta), meta)) if a != b][:5]
        assert np.array_equal(e_off, want_off + mis)
        assert e_out[mis:int(e_off[-1])].tobytes() == b"".join(frames)
    return frames, meta


def _decode_model_emu(msgs, root, frames, presence_instance=False):
    """model == device code on statuses, offsets and rows; returns (rows, meta)"""
    raw, in_off = _pack_frames(frames)
    rows, meta = PP.decode(msgs, root, frames)
    e_rows, e_off, e_meta = _emu_decode(msgs, root, raw, in_off, presence_instance)
    assert list(e_meta) == meta, [(i, a, b, frames[i].hex()) for i, (a, b) in enumerate(zip(list(e_meta), meta)) if a != b][:5]
    assert np.array_equal(e_off, np.cumsum([0] + [len(r) for r in rows]).astype(np.uint32))
    for i, r in enumerate(rows):
        got = e_rows[int(e_off[i]):int(e_off[i + 1])].tobytes()
        assert got == r, (i, frames[i].hex(), got.hex(), r.hex())
    return rows, meta


def _check_python_parse(msgs, root, frames, rows, meta):
    """wherever python protobuf and the codec both accept a frame, the row is what python parsed; they agree on what parses"""
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
            assert rows[i] == want[:len(rows[i])].tobytes() and len(rows[i]) == len(want) - 8, (i, fr.hex(), parsed[i])


def _describe(msgs, root=0, desc=None):
    nm, nf, k = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    return _abi.lib().gofr_proto_nested_describe_ex(nm.ctypes.data, len(msgs), nf.ctypes.data, k, root, None if pr is None else pr.ctypes.data,
                                                    None if desc is None else desc.ctypes.data, 0 if desc is None else desc.size)


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
    frames, meta = _encode_model_emu(KA_MSGS, 0, rows, off)
    assert meta == [0] * len(values)
    for k, (_, hexs) in enumerate(KA_ENC):
        assert frames[k] == _frame(bytes.fromhex(hexs)), (k, frames[k].hex())
    assert _pure_python([("enc", KA_MSGS, 0, values)])[0] == frames
    d_rows, d_meta = _decode_model_emu(KA_MSGS, 0, frames)
    assert d_meta == meta
    assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]


def test_known_answers_decode():
    frames = [_frame(bytes.fromhex(h)) for h, _ in KA_DEC] + [_frame(b) for b, _ in KA_DEC_STATUS]
    rows, meta = _decode_model_emu(KA_MSGS, 0, frames)
    assert meta == [0 if v is not None else S.GRPC_DEFER for _, v in KA_DEC] + [s for _, s in KA_DEC_STATUS], meta
    for k, (h, v) in enumerate(KA_DEC):
        if v is not None:
            want, _ = S.pack_proto_nested_rows(KA_MSGS, 0, [v])
            assert rows[k] == want[:-8].tobytes(), (k, h, rows[k].hex())
    _check_python_parse(KA_MSGS, 0, frames, rows, meta)


# ---------------------------------------------------------------------------------------------------------------
# random type sets with optional fields and oneofs, mixed with nested, repeated and map fields
# ---------------------------------------------------------------------------------------------------------------
def _add_presence(rnd, msgs):
    """optional fields and up to three oneof groups per message type (never in a map entry type)"""
    entries = _entry_types(msgs)
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


def _rand_presence_types(rnd):
    while True:
        msgs = _add_presence(rnd, _rand_map_types(rnd) if rnd.random() < 0.6 else _rand_types(rnd))
        if any(PP.explicit(f) or PP.group(f) for f in msgs[0]):   # (optional on a message field alone marks nothing)
            return msgs


def _rand_presence_value(rnd, msgs, m):
    """a value list with at most one set member per oneof group; explicit-presence fields unset about half the time"""
    fields = msgs[m]
    chosen = {}
    for g in {f.presence for f in fields if 1 <= f.presence <= 7}:
        members = [q for q, f in enumerate(fields) if f.presence == g]
        chosen[g] = rnd.choice(members + [None])
    v = []
    for q, f in enumerate(fields):
        one = (lambda: _rand_presence_value(rnd, msgs, f.msg)) if f.type == S.PB_MESSAGE else (lambda: _rand_scalar(rnd, f.type))
        if f.type == S.PB_MAP:
            kf, vf = msgs[f.msg]
            d = {}
            for _ in range(rnd.choice([0, 0, 1, 2, 4])):
                d[_rand_key(rnd, kf.type)] = _rand_presence_value(rnd, msgs, vf.msg) if vf.type == S.PB_MESSAGE else _rand_scalar(rnd, vf.type)
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


ENC_SEEDS = range(26)


@lru_cache(maxsize=None)
def _enc_cases():
    cases = []
    for seed in ENC_SEEDS:
        rnd = random.Random(5100 + seed)
        msgs = _rand_presence_types(rnd)
        cases.append((msgs, 0, [_rand_presence_value(rnd, msgs, 0) for _ in range(40)]))
    return cases, _pure_python([("enc", m, r, v) for m, r, v in cases])


@pytest.mark.parametrize("seed", ENC_SEEDS)
def test_random_presence_types_encode(seed):
    """model == device code == pure-Python deterministic bytes; the decoder gives the rows back"""
    cases, py = _enc_cases()
    msgs, root, values = cases[seed]
    desc = np.zeros(512, np.uint8)
    assert _describe(msgs, root, desc) == 0 and desc[1] == 1
    rows, off = S.pack_proto_nested_rows(msgs, root, values)
    frames, meta = _encode_model_emu(msgs, root, rows, off)
    assert meta == [0] * len(values)
    for i in range(len(values)):
        assert frames[i] == py[seed][i], (i, values[i], frames[i].hex(), py[seed][i].hex())
    # round trip: decode(encode(row)) == row (map message values present: a nil one comes back empty)
    d_rows, d_meta = _decode_model_emu(msgs, root, frames)
    assert d_meta == meta
    if not _entry_types(msgs):
        assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]


def test_decode_round_trip_and_python_parse():
    """decode(encode(row)) == row; python protobuf parses each frame to the same values"""
    rnd = random.Random(77)
    for msgs in [KA_MSGS] + [_rand_presence_types(rnd) for _ in range(8)]:
        values = [_rand_presence_value(rnd, msgs, 0) for _ in range(40)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = _encode_model_emu(msgs, 0, rows, off)
        assert meta == [0] * len(values)
        d_rows, d_meta = _decode_model_emu(msgs, 0, frames)
        assert d_meta == meta
        assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]
        _check_python_parse(msgs, 0, frames, d_rows, d_meta)


def _shuffle_fields(rnd, body, msgs):
    """the top-level fields of a well-formed body in a random order (oneof members in every order)"""
    items, i = [], 0
    while i < len(body):
        j = i
        tag, j = PM._get_varint(body, j, len(body))
        wt = tag & 7
        if wt == 0:
            _, j = PM._get_varint(body, j, len(body))
        elif wt == 1:
            j += 8
        elif wt == 5:
            j += 4
        else:
            n, j = PM._get_varint(body, j, len(body))
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
    msgs = _rand_presence_types(rnd)
    values = [_rand_presence_value(rnd, msgs, 0) for _ in range(50)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, _ = PP.encode(msgs, 0, rows, off)
    others, _ = PP.encode(msgs, 0, *S.pack_proto_nested_rows(msgs, 0, [_rand_presence_value(rnd, msgs, 0) for _ in range(50)]))
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
        out.append(_frame(bytes(body)))
    d_rows, d_meta = _decode_model_emu(msgs, 0, out)
    assert sum(m == 0 for m in d_meta) >= 10
    _check_python_parse(msgs, 0, out, d_rows, d_meta)


def test_presence_instance_on_presence_free_types():
    """the presence kernels' instance answers as the others on descriptions without presence (maps and map-free)"""
    rnd = random.Random(8)
    for k in range(6):
        msgs = _rand_map_types(rnd) if k % 2 else _rand_types(rnd)
        values = [[None if f.type == S.PB_MESSAGE and not f.repeated and rnd.random() < 0.3 else x for f, x in zip(msgs[0], v)]
                  for v in [_rand_presence_value(rnd, msgs, 0) for _ in range(30)]]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = _encode_model_emu(msgs, 0, rows, off, presence_instance=True)
        assert meta == [0] * len(values)
        frames = [fr if i % 3 else _frame(_shuffle_fields(rnd, fr[5:], msgs) + fr[5:]) for i, fr in enumerate(frames)]
        _decode_model_emu(msgs, 0, frames, presence_instance=True)


def test_presence_model_equals_maps_model_without_presence():
    """the presence model restates the maps model: on presence-free types (maps and map-free) it answers as that one does,
    on rows and on shuffled, duplicated and damaged frames"""
    rnd = random.Random(12)
    for k in range(8):
        msgs = _rand_map_types(rnd) if k % 2 else _rand_types(rnd)
        values = [_rand_presence_value(rnd, msgs, 0) for _ in range(30)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = PM.encode(msgs, 0, rows, off)
        assert PP.encode(msgs, 0, rows, off) == (frames, meta)
        bad = [fr[:len(fr) - 1] for fr in frames[:5]]
        out = [_frame(_shuffle_fields(rnd, fr[5:] + fr[5:], msgs)) for fr in frames] + bad
        for i in range(0, len(out), 4):
            body = bytearray(out[i][5:])
            if body:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            out[i] = _frame(bytes(body))
        assert PP.decode(msgs, 0, frames + out) == PM.decode(msgs, 0, frames + out)


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
    _, meta = _encode_model_emu(BR_MSGS, 0, rows, np.array(offs, dtype=np.uint32))
    assert meta == [s for _, s in blobs], meta
    # the packer lays out such rows too
    r2, o2 = S.pack_proto_nested_rows(BR_MSGS, 0, [[None, None, None, None, []], [0, 1, "", None, []], [None, None, None, [0], [[None, None]]]])
    _, meta2 = _encode_model_emu(BR_MSGS, 0, r2, o2)
    assert meta2 == [0, S.GRPC_BAD_ROW, 0]


def _last_error():
    return _abi.lib().gofr_last_error().decode()


def test_descriptions():
    desc = np.zeros(512, np.uint8)
    plain = [[F(1, S.PB_INT32), F(2, S.PB_MESSAGE, False, 1)], [F(1, S.PB_STRING)]]
    # no presence, and optional on a message field: the same descriptor as the call without presence
    nm, nf, k = S.proto_nested_tables(plain)
    ref = np.zeros(512, np.uint8)
    assert _abi.lib().gofr_proto_nested_describe(nm.ctypes.data, 2, nf.ctypes.data, k, 0, ref.ctypes.data, ref.size) == 0
    for msgs in (plain, [[plain[0][0], dataclasses.replace(plain[0][1], presence=OPT)], plain[1]]):
        desc[:] = 0
        assert _describe(msgs, 0, desc) == 0
        assert desc.tobytes() == ref.tobytes()
    assert _abi.lib().gofr_proto_nested_describe_ex(nm.ctypes.data, 2, nf.ctypes.data, k, 0, None, desc.ctypes.data, desc.size) == 0
    assert desc.tobytes() == ref.tobytes()
    # with presence: the presence byte of the descriptor is set, the maps half-word says what it said
    assert _describe(KA_MSGS, 0, desc) == 0 and desc[1] == 1 and desc[2] == 0
    withmap = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_INT32, presence=OPT)], [F(1, S.PB_STRING), F(2, S.PB_INT32)]]
    assert _describe(withmap, 0, desc) == 0 and desc[1] == 1 and desc[2] == 1
    # fixed words of the root (PbnDesc::fixed_words[0], bytes 40..41): the presence words count
    # (a: 2, s: 2, x: 2, y: 1 + 1, A: 2, B: 2, z: 1 + 1, q: 3)
    assert _describe(KA_MSGS, 0, desc) == 0
    assert int(desc[40]) | int(desc[41]) << 8 == 17
    # seven groups in one message type are fine
    assert _describe([[F(k, S.PB_INT32, presence=k) for k in range(1, 8)]]) == CAP
    assert _describe([[F(1, S.PB_MESSAGE, False, 1, 7), F(2, S.PB_BYTES, presence=7)], [F(1, S.PB_INT32, presence=OPT)]]) == CAP
    bad = [
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
    for msgs, text in bad:
        assert _describe(msgs) == INVALID, msgs
        assert text in _last_error(), (_last_error(), text)


def test_ex_calls_without_presence_bytes_are_the_plain_calls():
    """presence == NULL: the _ex calls validate exactly as the calls without presence"""
    L = _abi.lib()
    for msgs in ([[F(1, S.PB_MAP, True, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], [[F(0, S.PB_INT32)]], [[F(1, 10)]]):
        nm, nf, k = S.proto_nested_tables(msgs)
        a = L.gofr_proto_nested_describe(nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, None, 0)
        b = L.gofr_proto_nested_describe_ex(nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, None, None, 0)
        assert a == b != CAP


def test_descriptor_size_unchanged():
    lib = emu.lib()
    lib.emu_pbn_desc_bytes.restype = ctypes.c_uint32
    assert lib.emu_pbn_desc_bytes() == 440


# ---------------------------------------------------------------------------------------------------------------
# the CUDA kernels
# ---------------------------------------------------------------------------------------------------------------
def _top_presence_offsets(msgs):
    """byte offsets of the presence words of the root's explicit-presence scalar / string fields in its fixed part"""
    offs, p = [], 0
    for f in msgs[0]:
        if PP.explicit(f):
            offs.append(p)
        p += 4 + PP.fixed_bytes(msgs, f.msg) if f.type == S.PB_MESSAGE and not f.repeated else PP.fixed_bytes([[f]], 0)
    return offs


def _gpu_check():
    """the body of test_gpu_presence_matches_model (run in a process of its own)"""
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(93)
    eng = Engine(Table(synth.config1_spec()), 0)
    checked = 0
    for _ in range(3):
        msgs = _rand_presence_types(rnd)
        while not _top_presence_offsets(msgs):
            msgs = _rand_presence_types(rnd)
        values = [_rand_presence_value(rnd, msgs, 0) for _ in range(4200)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        po = _top_presence_offsets(msgs)
        for i in range(0, len(values), 53):          # a few rows the encoder refuses: a presence word of 2
            rows[int(off[i]) + rnd.choice(po)] = 2
        frames, meta = PP.encode(msgs, 0, rows, off)
        assert meta.count(S.GRPC_BAD_ROW) >= len(values) // 53
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
        rows2, meta2 = PP.decode(msgs, 0, frames)
        g_rows, g_off, g_meta = eng.proto_decode_nested_device(msgs, 0, raw, in_off)
        torch.cuda.synchronize()
        want_off = np.cumsum([0] + [len(r) for r in rows2]).astype(np.uint32)
        assert np.array_equal(g_meta.cpu().numpy().view(np.uint32), np.array(meta2, dtype=np.uint32))
        assert np.array_equal(g_off.cpu().numpy().view(np.uint32), want_off)
        assert g_rows[:int(want_off[-1])].cpu().numpy().tobytes() == b"".join(rows2)
        checked += len(values)
    eng.close()
    assert checked >= 12000
    print("presence on the GPU: %d messages, encode and decode equal to the model" % checked)


@pytest.mark.gpu
def test_gpu_presence_matches_model():
    """both presence kernels == the model (statuses, offsets, frames, rows) — in a child process, so that a fault in a
    kernel cannot leave a sticky CUDA error in the process the other GPU tests run in"""
    r = subprocess.run([sys.executable, "-c", "import tests.test_proto_presence as t; t._gpu_check()"], cwd=ROOT_DIR,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    print(r.stdout.strip().splitlines()[-1] if r.stdout.strip() else "")
