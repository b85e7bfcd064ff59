"""gofr_proto_encode_nested_device — the proto3 encoder for message types with nested and repeated fields
(SURVEY.md §8f rank 4 widened; VERDICT r01 "missing" item 6).

Reference behaviour: proto.Marshal of the message a unary handler returns + grpc-go's 5-byte length prefix
(examples/grpc-server/grpc/hello_grpc.pb.go:73-89; protobuf-go v1.32.0, grpc-go v1.60.1).  Three statements compared:
  python google.protobuf with descriptors built at run time (independent implementation, deterministic field order)
  the oracle (oracle/orc_proto_nested.c: recursive, a message marshalled into its own buffer)
  the device code (proto_nested_device.cuh: explicit stack, nested lengths from a sizing walk) on the CPU via tests/emu,
  and the CUDA kernel with -m gpu.
Generators, fixtures and the python protobuf classes are shared with the map and presence tests (tests/proto_nested_harness.py)."""
import random
import struct

import numpy as np
import pytest

from gofr_b200 import spec as S
from tests import oracle as O
from tests import proto_nested_harness as H
from tests.emu import emu

F = S.ProtoNField


def _three_ways(msgs, root, values):
    rows, off = S.pack_proto_nested_rows(msgs, root, values)
    o_out, o_off, o_meta = O.proto_encode_nested(msgs, root, rows, off)
    assert not o_meta.any(), o_meta
    want = H.py_frames(msgs, root, values)
    got = H.frames_of(o_out, o_off)
    for i in range(len(values)):
        assert got[i] == want[i], (i, values[i], got[i].hex(), want[i].hex())
    for mis in (0, 3):
        e_out, e_off, e_meta = emu.proto_encode_nested(msgs, root, rows, off, mis)
        assert not e_meta.any() and np.array_equal(e_off, o_off + mis)
        assert e_out[mis:int(e_off[-1])].tobytes() == o_out[:int(o_off[-1])].tobytes()
    return rows, off, o_out, o_off


def test_known_answers_and_python_protobuf():
    geo = [1.5, -2.25, [1, 0, -1]]
    owner = ["ann", [b"\x00\xff", b""], geo]
    item1 = [7, "first", ["a", "", "bb"], [0.0, -0.0, 1e300], owner, [-1, 0, 1, 2 ** 31 - 1, -2 ** 31]]
    item2 = [0, "", [], [], None, []]                                   # an element that encodes to nothing: tag + length 0
    page = [[item1, item2], 2, "next", [ "", [], None], [True, False, True], [1, 2 ** 64 - 1]]
    empty = [[], 0, "", None, [], []]
    rows, off, out, o = _three_ways(H.MSGS, 0, [page, empty, [[item2] * 3, 0, "", None, [], []]])
    fr = H.frames_of(out, o)
    assert fr[1] == b"\x00\x00\x00\x00\x00"                             # nothing set: an empty message, still a frame
    assert fr[2] == b"\x00\x00\x00\x00\x06" + b"\x0a\x00" * 3           # three empty items: tag 1/LEN + length 0 each
    # a set but empty singular message is written (field 15 = tag 0x7a, length 0); packed bools; packed fixed64 under a
    # two-byte field number
    assert b"\x7a\x00" in fr[0] and b"\x82\x01\x03\x01\x00\x01" in fr[0]
    assert (2047 << 3 | 2).to_bytes(2, "little") != b"" and bytes([0xFA, 0x7F, 0x10]) in fr[0]


@pytest.mark.parametrize("seed", range(25))
def test_random_types_three_ways(seed):
    rnd = random.Random(500 + seed)
    msgs = H.rand_types(rnd)
    values = [H.rand_value(rnd, msgs, 0) for _ in range(60)]
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
    """recursive types, field order, unknown types, groups, reserved numbers and depth (the table: H.LIMIT_DESCRIPTIONS)"""
    for msgs, root, want in H.LIMIT_DESCRIPTIONS:
        assert H.describe(msgs, root) == want, msgs


@pytest.mark.gpu
def test_gpu_matches_oracle():
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(77)
    eng = Engine(Table(synth.config1_spec()), 0)
    for msgs in (H.MSGS, H.rand_types(rnd), H.rand_types(rnd)):
        values = [H.rand_value(rnd, msgs, 0) for _ in range(5000)]
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
def test_decode_canonical_frames_round_trip():
    """decode(encode(row)) == row, and python protobuf parses the frames to the same values"""
    rnd = random.Random(9)
    for msgs in (H.MSGS, H.rand_types(rnd), H.rand_types(rnd), H.rand_types(rnd)):
        values = [H.rand_value(rnd, msgs, 0) for _ in range(80)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        out, o, meta = O.proto_encode_nested(msgs, 0, rows, off)
        frames = H.frames_of(out, o)
        d_rows, d_off, d_meta = H.decode_three_ways(msgs, 0, frames)
        assert not d_meta.any()
        for i in range(len(values)):
            a = rows[int(off[i]):int(off[i + 1])].tobytes()
            b = d_rows[int(d_off[i]):int(d_off[i + 1])].tobytes()
            # -0.0 and absent look the same on the wire only for... nothing: the encoder writes -0.0, so rows match exactly
            assert a == b, (i, values[i])


def test_decode_noncanonical_and_hostile_frames():
    msgs = H.HOSTILE_MSGS
    frames = [H.frame(b) for b in H.HOSTILE_BODIES] + H.HOSTILE_HEADER_FRAMES
    rows, off, meta = H.decode_three_ways(msgs, 0, frames)
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
    msgs = H.rand_types(rnd)
    values = [H.rand_value(rnd, msgs, 0) for _ in range(60)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    out, o, meta = O.proto_encode_nested(msgs, 0, rows, off)
    frames = []
    for fr in H.frames_of(out, o):
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
        frames.append(H.frame(bytes(body)))
    H.decode_three_ways(msgs, 0, frames)


def _gpu_decode_check():
    """the body of test_gpu_decode_matches_oracle (run in a process of its own)"""
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(78)
    eng = Engine(Table(synth.config1_spec()), 0)
    for msgs in (H.MSGS, H.rand_types(rnd), H.rand_types(rnd)):
        values = [H.rand_value(rnd, msgs, 0) for _ in range(4000)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        out, o, _ = O.proto_encode_nested(msgs, 0, rows, off)
        frames = H.frames_of(out, o)
        for i in range(0, len(frames), 7):          # every seventh frame damaged: statuses and empty rows must agree too
            body = bytearray(frames[i][5:])
            if body:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            frames[i] = H.frame(bytes(body))
        raw, in_off = H.pack_frames(frames)
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
    H.run_child("import tests.test_proto_nested as t; t._gpu_decode_check()", timeout=600)
