"""Config 5 — gRPC unary Hello at the message level: oracle vs python google.protobuf (independent implementation),
oracle vs the kernel's device code on the CPU (tests/emu), and — with -m gpu — the CUDA kernel through the C ABI."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from gofr_b200 import synth
from tests import oracle as O
from tests.emu import emu
from tests.conftest import has_gpu


def _frames(msgs, flags=None):
    buf, offs = bytearray(), [0]
    for k, m in enumerate(msgs):
        buf += bytes([flags[k] if flags else 0]) + len(m).to_bytes(4, "big") + m
        offs.append(len(buf))
    buf += b"\0" * 16
    return np.frombuffer(bytes(buf), dtype=np.uint8).copy(), np.array(offs, dtype=np.uint32)


def _hello_classes():
    """HelloRequest / HelloResponse built from the schema of examples/grpc-server/grpc/hello.proto:4-10."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fd = descriptor_pb2.FileDescriptorProto(name="hello_gofr_test.proto", syntax="proto3")
    for mname, fname in (("HelloRequest", "name"), ("HelloResponse", "message")):
        m = fd.message_type.add(name=mname)
        m.field.add(name=fname, number=1, type=descriptor_pb2.FieldDescriptorProto.TYPE_STRING,
                    label=descriptor_pb2.FieldDescriptorProto.LABEL_OPTIONAL)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return (message_factory.GetMessageClass(pool.FindMessageTypeByName("HelloRequest")),
            message_factory.GetMessageClass(pool.FindMessageTypeByName("HelloResponse")))


EDGE_MSGS = [
    b"", b"\x0a\x00", b"\x0a\x05world", b"\x0a\x03123", b"\x0a\x01a\x0a\x02bc",            # last occurrence wins
    b"\x10\x96\x01\x0a\x02hi", b"\x0a\x02hi\x15\x01\x02\x03\x04\x19" + b"\x00" * 8,       # unknown varint / fixed32 / fixed64
    b"\x12\x03abc\x0a\x01z", b"\x1b\x0a\x01q\x1c\x0a\x01k", b"\x0b\x0a\x01q\x0c",          # unknown bytes field, groups
    b"\x0a\x02\xc3\xa9", b"\x0a\x01\xff", b"\x0a\x02\xc3", b"\x0a\x03\xed\xa0\x80",        # utf-8 valid / invalid
    b"\x0a", b"\x0a\x05ab", b"\x80", b"\x00\x00", b"\x0f", b"\x0e\x01", b"\x0c", b"\x1b\x0a\x01q",  # malformed
    b"\xff\xff\xff\xff\xff\xff\xff\xff\xff\x02\x00", b"\x08" + b"\xff" * 9 + b"\x01", b"\x08" + b"\xff" * 9 + b"\x02",
    b"\x0a\x80\x01" + b"n" * 128, b"\x0a\xc8\x01" + b"m" * 200,                            # two-byte length varints
]


# python's upb parser silently drops the overflow bits of a 10-byte varint whose last byte is > 1; protobuf-go
# (protowire.ConsumeVarint) rejects it.  The oracle follows Go, so this vector is excluded from the cross-check.
GO_STRICTER_THAN_UPB = {b"\x08" + b"\xff" * 9 + b"\x02"}


def test_oracle_vs_python_protobuf():
    """Independent check of the oracle's wire arithmetic against upstream protobuf (python)."""
    Req, Resp = _hello_classes()
    frames, off = _frames(EDGE_MSGS)
    out, ooff, meta = O.grpc_hello(frames, off)
    res = O.responses(out, ooff)
    for m, r, st_ in zip(EDGE_MSGS, res, meta):
        if m in GO_STRICTER_THAN_UPB:
            assert st_ == 3  # protobuf-go: protowire.ConsumeVarint → errCodeOverflow
            continue
        try:
            req = Req.FromString(m)
            ok = True
        except Exception:
            ok = False
        assert ok == (st_ == 0), (m, st_)
        if ok:
            want = Resp(message="Hello %s!" % (req.name or "World")).SerializeToString()
            assert r == b"\x00" + len(want).to_bytes(4, "big") + want, m


def test_frame_level_errors():
    frames, off = _frames([b"\x0a\x01a", b"\x0a\x01a", b"\x0a\x01a"], flags=[1, 2, 0])
    out, ooff, meta = O.grpc_hello(frames, off)
    assert list(meta) == [1, 2, 0]
    # declared length disagrees with the frame
    bad = np.frombuffer(b"\x00\x00\x00\x00\x09\x0a\x01a" + b"\0" * 16, dtype=np.uint8).copy()
    _, _, meta = O.grpc_hello(bad, np.array([0, 8], dtype=np.uint32))
    assert meta[0] == 2
    _, _, meta = O.grpc_hello(bad, np.array([0, 3], dtype=np.uint32))
    assert meta[0] == 2


def _cmp(frames, off, impl, mis=0):
    o1, f1, m1 = O.grpc_hello(frames, off)
    o2, f2, m2 = impl(frames, off, mis) if mis is not None else impl(frames, off)
    assert np.array_equal(m1, m2)
    assert O.responses(o1, f1) == O.responses(o2, f2)


@pytest.mark.parametrize("mis", [0, 1, 2, 3, 7, 13])
def test_emu_edge_cases(mis):
    frames, off = _frames(EDGE_MSGS + [b"\x0a\x01a"] * 3, flags=[0] * len(EDGE_MSGS) + [1, 2, 0])
    _cmp(frames, off, emu.grpc_hello, mis)


def test_emu_config5_stream():
    frames, off = synth.config5_frames(20000)
    _cmp(frames, off, emu.grpc_hello, 5)


@settings(max_examples=200, deadline=None)
@given(st.lists(st.binary(min_size=0, max_size=24), min_size=1, max_size=16), st.integers(0, 15))
def test_emu_random_messages(msgs, mis):
    frames, off = _frames(msgs)
    _cmp(frames, off, emu.grpc_hello, mis)


def _gpu_hello(frames, off, eng=None):
    import ctypes as C
    import torch
    from gofr_b200 import _abi
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    eng = eng or Engine(Table(synth.config1_spec()), 0)
    n = len(off) - 1
    cap = int(frames.size) + 40 * n + 64
    d_in = torch.from_numpy(np.concatenate([frames, np.zeros(64, np.uint8)])).cuda()
    d_off = torch.from_numpy(off.view(np.int32)).cuda()
    d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
    d_ooff = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
    d_meta = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    _abi.check(_abi.lib().gofr_grpc_hello_device(eng._e, d_in.data_ptr(), d_off.data_ptr(), n, d_out.data_ptr(), cap,
                                                 d_ooff.data_ptr(), d_meta.data_ptr(),
                                                 torch.cuda.current_stream().cuda_stream), "gofr_grpc_hello_device")
    torch.cuda.synchronize()
    assert not eng.overflowed()
    return d_out.cpu().numpy(), d_ooff.cpu().numpy().view(np.uint32), d_meta.cpu().numpy().view(np.uint32)[:n]


@pytest.mark.gpu
def test_gpu_edge_cases():
    frames, off = _frames(EDGE_MSGS * 40 + [b"\x0a\x01a"] * 3, flags=[0] * (40 * len(EDGE_MSGS)) + [1, 2, 0])
    _cmp(frames, off, _gpu_hello, None)


@pytest.mark.gpu
def test_gpu_config5_full_size():
    """1 Mi frames: byte-identical to the oracle, and a 64 k sample re-checked against python protobuf."""
    n = 1 << 20
    frames, off = synth.config5_frames(n)
    o1, f1, m1 = O.grpc_hello(frames, off)
    o2, f2, m2 = _gpu_hello(frames, off)
    assert np.array_equal(m1, m2) and np.array_equal(f1, f2)
    assert np.array_equal(o1[:int(f1[n])], o2[:int(f1[n])])
    Req, Resp = _hello_classes()
    raw, res = frames.tobytes(), o2.tobytes()
    for i in range(0, 65536, 7):
        req = Req.FromString(raw[off[i] + 5:off[i + 1]])
        want = Resp(message="Hello %s!" % (req.name or "World")).SerializeToString()
        assert res[f2[i]:f2[i + 1]] == b"\x00" + len(want).to_bytes(4, "big") + want
