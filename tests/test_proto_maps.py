"""Map fields (GOFR_PB_MAP) in the nested proto3 codec: gofr_proto_encode_nested_device / gofr_proto_decode_nested_device.

Reference behaviour: protobuf-go v1.32.0 impl/codec_map.go — a map is a repeated entry message (1 key, 2 value); marshalling
writes key and value at their zero values too and a message value always; Deterministic marshalling sorts the keys;
unmarshalling lets the last key / value inside an entry win and a later entry replace an earlier one with an equal key.
Statements compared:
  tests/proto_nested_model.py recursive; the decoder collects the entries, stable-sorts them and keeps the last of equal keys
  the device code             explicit stacks, the decoder selects the next key by rescanning — on the CPU via tests/emu
                              (output misalignments 0 and 3) and, with -m gpu, in the CUDA kernels
  python google.protobuf      the pure-Python backend, in a child process: its deterministic=True sorts keys like Go, and it
                              skips unknown fields inside an entry like Go (upb does neither)."""
import random
from functools import lru_cache

import numpy as np
import pytest

from gofr_b200 import spec as S
from tests import oracle as O
from tests import proto_nested_harness as H
from tests import proto_nested_model as M
from tests.emu import emu
from tests.proto_nested_harness import CAP, MAP_KA_MSGS as KA_MSGS

F = S.ProtoNField


# ---------------------------------------------------------------------------------------------------------------
# known answers
# ---------------------------------------------------------------------------------------------------------------
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
    frames, meta = H.encode_model_emu(KA_MSGS, 0, rows, off)
    assert meta == [0] * len(values)
    for k, (_, _, hexs) in enumerate(KA):
        assert frames[k] == H.frame(bytes.fromhex(hexs)), (k, frames[k].hex())
    assert frames[-1] == H.frame(bytes.fromhex("".join(h for _, _, h in KA)))
    assert H.pure_python([("enc", KA_MSGS, 0, values)])[0] == frames
    d_rows, d_meta = H.decode_model_emu(KA_MSGS, 0, frames)
    assert d_meta == [0] * len(values)
    assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]


def test_model_equals_oracle_without_maps():
    """the model restates the nested codec as a whole: on map-free types it answers as the oracle does"""
    rnd = random.Random(4)
    for _ in range(6):
        msgs = H.rand_types(rnd)
        values = [H.rand_value(rnd, msgs, 0) for _ in range(40)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        o_out, o_off, o_meta = O.proto_encode_nested(msgs, 0, rows, off)
        frames, meta = M.encode(msgs, 0, rows, off)
        assert list(o_meta) == meta and H.frames_of(o_out, o_off) == frames
        raw, in_off = H.pack_frames(frames)
        d_rows, d_off, d_meta = O.proto_decode_nested(msgs, 0, raw, in_off)
        rows2, meta2 = M.decode(msgs, 0, frames)
        assert list(d_meta) == meta2 and [d_rows[int(d_off[i]):int(d_off[i + 1])].tobytes() for i in range(len(frames))] == rows2


ENC_SEEDS = range(25)


@lru_cache(maxsize=None)
def _enc_cases():
    cases = []
    for seed in ENC_SEEDS:
        rnd = random.Random(1300 + seed)
        msgs = H.rand_map_types(rnd)
        cases.append((msgs, 0, [H.rand_map_value(rnd, msgs, 0) for _ in range(40)]))
    return cases, H.pure_python([("enc", m, r, v) for m, r, v in cases])


@pytest.mark.parametrize("seed", ENC_SEEDS)
def test_random_map_types_encode(seed):
    """model == device code == pure-Python deterministic bytes"""
    cases, py = _enc_cases()
    msgs, root, values = cases[seed]
    assert H.describe(msgs, root) == CAP
    rows, off = S.pack_proto_nested_rows(msgs, root, values)
    frames, meta = H.encode_model_emu(msgs, root, rows, off)
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
    _, meta = H.encode_model_emu(msgs, 0, rows, off)
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
    _, meta2 = H.encode_model_emu(msgs, 0, rows2, np.array(offs, dtype=np.uint32))
    assert meta2.count(R) >= len(blobs) // 2 and meta2[-2] == R


# ---------------------------------------------------------------------------------------------------------------
# the decoder
# ---------------------------------------------------------------------------------------------------------------
def test_decode_round_trip():
    """decode(encode(row)) == row for rows whose message values are present; python protobuf parses the same maps"""
    rnd = random.Random(21)
    for msgs in [KA_MSGS] + [H.rand_map_types(rnd) for _ in range(6)]:
        values = [H.rand_map_value(rnd, msgs, 0, nil_values=False) for _ in range(50)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = H.encode_model_emu(msgs, 0, rows, off)
        assert meta == [0] * len(values)
        d_rows, d_meta = H.decode_model_emu(msgs, 0, frames)
        assert d_meta == meta
        assert d_rows == [rows[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(values))]
        H.check_python_parse(msgs, 0, frames, d_rows, d_meta)


def test_decode_noncanonical_frames():
    msgs, ok, defer, bad = H.NONCANON_MSGS, H.NONCANON_OK, H.NONCANON_DEFER, H.NONCANON_BAD
    frames = [H.frame(b) for b in ok + defer + bad]
    rows, meta = H.decode_model_emu(msgs, 0, frames)
    D, P, U = S.GRPC_DEFER, S.GRPC_BAD_PROTO, S.GRPC_BAD_UTF8
    assert meta == [0] * len(ok) + [D] * len(defer) + [U, U, U, P, P, P, P, U], meta
    H.check_python_parse(msgs, 0, frames, rows, meta)
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
    msgs = H.rand_map_types(rnd)
    values = [H.rand_map_value(rnd, msgs, 0) for _ in range(50)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, _ = M.encode(msgs, 0, rows, off)
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
        out.append(H.frame(bytes(body)))
    d_rows, d_meta = H.decode_model_emu(msgs, 0, out)
    H.check_python_parse(msgs, 0, out, d_rows, d_meta)


# ---------------------------------------------------------------------------------------------------------------
# descriptions
# ---------------------------------------------------------------------------------------------------------------
def test_descriptions():
    """every key kind, shared entry types, the entry type's shape and use, depth (the table: H.MAP_DESCRIPTIONS)"""
    for msgs, root, want in H.MAP_DESCRIPTIONS:
        assert H.describe(msgs, root) == want, msgs


def test_descriptor_size_unchanged():
    lib = emu.lib()
    import ctypes
    lib.emu_pbn_desc_bytes.restype = ctypes.c_uint32
    assert lib.emu_pbn_desc_bytes() == 440


# ---------------------------------------------------------------------------------------------------------------
# the CUDA kernels
# ---------------------------------------------------------------------------------------------------------------
def _spoil(rnd, msgs, values):
    """rows with a duplicate key in one row of 53, which the encoder refuses (H.gpu_check)"""
    spoiled = 0
    for i in range(0, len(values), 53):
        for f, v in zip(msgs[0], values[i]):
            if f.type == S.PB_MAP and v:
                k = next(iter(v))
                values[i][msgs[0].index(f)] = [(k, v[k]), (k, v[k])]
                spoiled += 1
                break
    return (*S.pack_proto_nested_rows(msgs, 0, values), spoiled)


@pytest.mark.gpu
def test_gpu_maps_match_model():
    """both kernels with map fields == the model (statuses, offsets, frames, rows) — in a child process, so that a fault in a
    kernel cannot leave a sticky CUDA error in the process the other GPU tests run in"""
    H.run_child("import tests.proto_nested_harness as h, tests.test_proto_maps as t; "
                "h.gpu_check(91, h.rand_map_types, h.rand_map_value, t._spoil)")
