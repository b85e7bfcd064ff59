"""The nested proto3 codec on host buffers: gofr_proto_batch_decode / _encode (the chunk pipeline of gofr_batch_submit,
the codec kernels and the chunk pack kernel), gofr_proto_nested_bound, gofr::ProtoCodec and examples/cpp/grpc_hello.cpp.

Without a GPU: the bound against the model's exact output sizes, the pack kernel's per-record logic on the CPU (tests/emu)
against a restatement, and the C++ example's build.  On the GPU, in a child process (H.run_child): both calls against the
model and the resident calls across chunk sizes, pinned and pageable outputs, capacities, bad offsets and SayHello."""
import os
import random
import subprocess

import numpy as np
import pytest

from gofr_b200 import _build
from gofr_b200 import spec as S
from gofr_b200.engine import nested_bound
from tests import proto_nested_harness as H
from tests import proto_nested_model as M
from tests.emu import emu_pack

F = S.ProtoNField
OK, BAD_UTF8, BAD_ROW, DEFER = S.GRPC_OK, S.GRPC_BAD_UTF8, S.GRPC_BAD_ROW, S.GRPC_DEFER
ROOT = H.ROOT_DIR
TOP = 2 ** 29 - 1          # the largest field number: a five-byte tag
LIMIT = 4096               # map entries the two decode passes together take


def model_decode(msgs, frames):
    """what the two resident decode passes give combined: the model with its map entry limit at 4096"""
    saved = M.MAX_MAP_ENTRIES
    M.MAX_MAP_ENTRIES = LIMIT
    try:
        return M.decode(msgs, 0, frames)
    finally:
        M.MAX_MAP_ENTRIES = saved


# ---------------------------------------------------------------------------------------------------------------
# gofr_proto_nested_bound against the model's exact sizes
# ---------------------------------------------------------------------------------------------------------------
def check_encode_bound(msgs, values):
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, meta = M.encode(msgs, 0, rows, off)
    per_byte, per_record = nested_bound(msgs, 0, False)
    for i, fr in enumerate(frames):
        b = int(off[i + 1] - off[i])
        assert len(fr) <= per_byte * b + per_record, (i, len(fr), b, per_byte, per_record)
    return meta


def check_decode_bound(msgs, frames):
    rows, meta = model_decode(msgs, frames)
    per_byte, per_record = nested_bound(msgs, 0, True)
    for i, (r, fr) in enumerate(zip(rows, frames)):
        assert len(r) <= per_byte * len(fr) + per_record, (i, len(r), len(fr), per_byte, per_record)
    return meta


@pytest.mark.parametrize("seed", range(10))
def test_bound_on_random_types(seed):
    rnd = random.Random(5100 + seed)
    msgs = H.rand_map_types(rnd) if seed % 2 else H.rand_presence_types(rnd)
    make = H.rand_map_value if seed % 2 else H.rand_presence_value
    values = [make(rnd, msgs, 0) for _ in range(80)]
    meta = check_encode_bound(msgs, values)
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, _ = M.encode(msgs, 0, rows, off)
    check_decode_bound(msgs, [fr for fr, m in zip(frames, meta) if m == OK])


ENCODE_WORST = [
    # negative int32 / enum at the largest field number: a five-byte tag and a ten-byte varint per word
    ([[F(TOP, S.PB_INT32)]], [[-1]]),
    ([[F(TOP - 1, S.PB_ENUM), F(TOP, S.PB_SINT64)]], [[-5, -2 ** 63]]),
    # packed negative int32, repeated empty strings
    ([[F(TOP, S.PB_INT32, True)]], [[[-1] * 100]]),
    ([[F(TOP, S.PB_STRING, True)]], [[[""] * 100]]),
    # repeated messages, empty and with a negative int32, their element headers at the largest field number
    ([[F(TOP, S.PB_MESSAGE, True, 1)], [F(TOP, S.PB_INT32)]], [[[[0]] * 100]]),
    ([[F(TOP, S.PB_MESSAGE, True, 1)], [F(TOP, S.PB_INT32)]], [[[[-1]] * 100]]),
    ([[F(TOP, S.PB_MESSAGE, True, 1)], [F(TOP, S.PB_MESSAGE, False, 2)], [F(TOP, S.PB_INT32, True)]], [[[[[[-1]]]] * 50]]),
    # map entries written at zero values, negative keys, nil message values
    ([[F(TOP, S.PB_MAP, False, 1)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]], [[{-k: -k for k in range(200)}]]),
    ([[F(TOP, S.PB_MAP, False, 1)], [F(1, S.PB_INT64), F(2, S.PB_MESSAGE, False, 2)], [F(TOP, S.PB_INT32)]], [[{-k: None for k in range(100)}]]),
    ([[F(TOP, S.PB_MAP, False, 1)], [F(1, S.PB_STRING), F(2, S.PB_BYTES)]], [[{"": b""}]]),
    # singular messages nested to the limit, explicit presence at zero values
    ([[F(TOP, S.PB_MESSAGE, False, 1)], [F(TOP, S.PB_MESSAGE, False, 2)], [F(TOP, S.PB_MESSAGE, False, 3)], [F(TOP, S.PB_INT32)]], [[[[[-1]]]]]),
    ([[F(TOP - 2, S.PB_INT32, presence=S.PB_OPTIONAL), F(TOP - 1, S.PB_STRING, presence=1), F(TOP, S.PB_UINT64, presence=1)]], [[0, "", None]]),
    ([[F(1, S.PB_UINT64), F(2, S.PB_FIXED64), F(3, S.PB_DOUBLE), F(4, S.PB_FLOAT), F(5, S.PB_BOOL)]], [[2 ** 64 - 1, 1, -0.0, 1.5, True]]),
]


@pytest.mark.parametrize("k", range(len(ENCODE_WORST)))
def test_encode_bound_on_worst_cases(k):
    msgs, values = ENCODE_WORST[k]
    assert check_encode_bound(msgs, values) == [OK] * len(values)


def test_decode_bound_on_worst_cases():
    """the frames that grow most per wire byte: packed 1-byte varints of 64-bit kinds, empty repeated messages and map
    entries of wide types, absent singular messages inline"""
    wide = [F(k, S.PB_FIXED64) for k in range(1, 9)]
    msgs = [[F(1, S.PB_MESSAGE, True, 1), F(2, S.PB_MAP, False, 2), F(3, S.PB_INT64, True), F(4, S.PB_MESSAGE, False, 1)],
            wide, [F(1, S.PB_BOOL), F(2, S.PB_MESSAGE, False, 1)]]
    frames = [H.frame(b"\x0a\x00" * 50), H.frame(b"\x12\x00" * 70), H.frame(b"\x1a\x7f" + b"\x01" * 127),
              H.frame(b"\x18\x01" * 60), H.frame(b""), H.frame(b"\x22\x00")]
    assert check_decode_bound(msgs, frames) == [OK] * len(frames)
    per_byte, per_record = nested_bound(msgs, 0, True)
    assert per_byte == (S._pb_fixed_bytes(msgs, 2) + 1) // 2 and per_record == S._pb_fixed_bytes(msgs, 0) + 3


# ---------------------------------------------------------------------------------------------------------------
# the pack kernel's per-record logic on the CPU
# ---------------------------------------------------------------------------------------------------------------
def pack_restated(a, a_off, b=None, b_off=None, sel=None):
    """record i: the bytes of source B where the selector says DEFER, else of source A"""
    out = []
    for i in range(len(a_off) - 1):
        src, o = (b, b_off) if b is not None and sel[i] == DEFER else (a, a_off)
        out.append(bytes(src[int(o[i]):int(o[i + 1])]))
    return out


def rand_source(rnd, n, empty=0.2):
    lens = [0 if rnd.random() < empty else rnd.choice([1, 2, 3, 4, 5, 7, 15, 16, 17, 31, 33, 63, 64, 65, 200, 1000]) for _ in range(n)]
    off = np.cumsum([0] + lens).astype(np.uint32)
    return np.frombuffer(bytes(rnd.randrange(256) for _ in range(int(off[-1]))), dtype=np.uint8).copy(), off


@pytest.mark.parametrize("start", range(16))
def test_pack_logic_every_start(start):
    rnd = random.Random(77 + start)
    for any_mode in (0, 1, 2):
        n = 150
        a, a_off = rand_source(rnd, n)
        b, b_off = rand_source(rnd, n)
        sel = np.array([rnd.choice([OK, DEFER, DEFER, S.GRPC_BAD_PROTO]) for _ in range(n)], dtype=np.uint32)
        for two in (False, True):
            args = (a, a_off, b, b_off, sel) if two else (a, a_off)
            want = pack_restated(*args)
            out, off = emu_pack.pack(*args, start=start, any_mode=any_mode)
            assert np.array_equal(off, (start + np.cumsum([0] + [len(w) for w in want])).astype(np.uint32))
            assert out[:start].tobytes() == b"\xee" * start
            assert out[start:int(off[-1])].tobytes() == b"".join(want)
            assert (out[int(off[-1]):] == 0xEE).all()


def test_pack_logic_source_past_its_capacity_is_empty():
    """a codec buffer that overflowed (its kernel set the overflow flag) is never read past what was written"""
    a = np.arange(64, dtype=np.uint8)
    a_off = np.array([0, 8, 40, 64], dtype=np.uint32)
    out, off = emu_pack.pack(a, a_off, start=3, a_cap=40)
    assert list(off) == [3, 11, 43, 43] and out[3:43].tobytes() == a[:40].tobytes()


# ---------------------------------------------------------------------------------------------------------------
# the C++ example builds
# ---------------------------------------------------------------------------------------------------------------
def _compile_hello(exe):
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "cpp", "grpc_hello.cpp"), "-o", exe, _build.LIB,
                           "-Wl,-rpath," + os.path.dirname(_build.LIB)])


def test_grpc_hello_compiles(tmp_path):
    from gofr_b200 import _abi
    _abi.lib()
    _compile_hello(str(tmp_path / "grpc_hello"))


# ---------------------------------------------------------------------------------------------------------------
# the GPU (child processes)
# ---------------------------------------------------------------------------------------------------------------
LM_MSGS = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 3), F(3, S.PB_MESSAGE, False, 4), F(4, S.PB_STRING, presence=S.PB_OPTIONAL)],
           [F(1, S.PB_INT64), F(2, S.PB_MESSAGE, False, 2)],
           [F(1, S.PB_STRING), F(2, S.PB_DOUBLE, True), F(3, S.PB_MAP, False, 5)],
           [F(1, S.PB_STRING), F(2, S.PB_STRING)],
           [F(1, S.PB_INT32)],
           [F(1, S.PB_UINT32), F(2, S.PB_INT32)]]


def _lm_frames(rnd, n):
    """frames of LM_MSGS: ordinary ones, 65..4097 map entries on the wire, a singular message sent twice (still DEFER)"""
    def small():
        return [{rnd.randrange(-50, 50): ["n%d" % rnd.randrange(9), [0.5], {}] for _ in range(rnd.randint(0, 5))}, {}, [1], None]

    def large():
        items_ = {rnd.randrange(-10 ** 6, 10 ** 6): ["n", [1.0] * rnd.randint(0, 2), {k: 1 for k in range(rnd.choice([0, 70]))}]
                  for _ in range(rnd.randint(65, 400))}
        return [items_, {"k%d" % k: "v" for k in range(rnd.randint(0, 100))}, [rnd.randint(0, 5)], "o"]

    frames = []
    for _ in range(n):
        kind = rnd.random()
        if kind < 0.05:
            vals = [large()]
        elif kind < 0.07:
            frames.append(H.frame(b"".join(H._entry(2, H._s(1, b"%d" % k)) for k in range(rnd.choice([4096, 4097])))))
            continue
        else:
            vals = [small()]
        rows, off = S.pack_proto_nested_rows(LM_MSGS, 0, vals)
        fr, meta = M.encode(LM_MSGS, 0, rows, off)
        assert meta == [OK]
        if kind > 0.97:        # message field 3 sent twice
            fr = [H.frame(fr[0][5:] + b"\x1a\x02\x08\x01")]
        frames.append(fr[0])
    return frames


def _damage(rnd, frames):
    out = list(frames)
    for i in range(0, len(out), 7):       # every seventh frame damaged
        body = bytearray(out[i][5:])
        if body:
            body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
        out[i] = H.frame(bytes(body))
    return out


def _spoil(rnd, msgs, values):
    """rows of the values, one in 53 with a word overwritten (the encoder may refuse it: BAD_ROW)"""
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    rows = rows.copy()
    for i in range(0, len(values), 53):
        lo, hi = int(off[i]), int(off[i + 1])
        if hi > lo:
            w = lo + 4 * rnd.randrange((hi - lo) // 4)
            rows[w:w + 4] = 0xFF
    return rows, off


def _check_rows(got, want_rows, want_meta):
    out, off, meta = got
    n = len(want_rows)
    assert list(meta[:n]) == list(want_meta), [(i, a, b) for i, (a, b) in enumerate(zip(meta, want_meta)) if a != b][:5]
    want_off = np.cumsum([0] + [len(r) for r in want_rows]).astype(np.uint32)
    assert np.array_equal(np.asarray(off[:n + 1]), want_off)
    assert out[:int(want_off[-1])].tobytes() == b"".join(want_rows)


def _gpu_codec(seed):
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    eng = Engine(Table(synth.config1_spec()), 0)
    checked = 0
    # ---- decode: the large-map description, then three random map / presence type sets ----
    sets = [(LM_MSGS, _lm_frames(rnd, 1500))]
    for k in range(3):
        msgs = H.rand_map_types(rnd) if k != 1 else H.rand_presence_types(rnd)
        make = H.rand_map_value if k != 1 else H.rand_presence_value
        values = [make(rnd, msgs, 0) for _ in range(1500)]
        rows, off = S.pack_proto_nested_rows(msgs, 0, values)
        frames, meta = M.encode(msgs, 0, rows, off)
        sets.append((msgs, [f for f, m in zip(frames, meta) if m == OK]))
    for msgs, frames in sets:
        frames = _damage(rnd, frames)
        want_rows, want_meta = model_decode(msgs, frames)
        raw, in_off = H.pack_frames(frames)
        for chunk in (1, 127, 128, 129, 1000, 65536):
            eng.set_chunk(chunk)
            nb = len(frames) if chunk > 1 else 300     # (a chunk per frame: a shorter batch)
            for pinned in (False, True):
                got = eng.proto_decode_batch(msgs, 0, raw, in_off[:nb + 1], pinned=pinned)
                _check_rows(got, want_rows[:nb], want_meta[:nb])
                checked += nb
    lm_meta = model_decode(LM_MSGS, sets[0][1])[1]
    assert DEFER in lm_meta and OK in lm_meta          # the large-map set kept frames for the host
    # ---- encode: against the resident encoder and the model, BAD_ROW and BAD_UTF8 included; then the round trip ----
    utf = [[F(1, S.PB_STRING), F(2, S.PB_MESSAGE, True, 1)], [F(1, S.PB_STRING, True)]]
    for msgs, make in ((LM_MSGS, None), (utf, None), (H.rand_map_types(rnd), H.rand_map_value), (H.rand_presence_types(rnd), H.rand_presence_value)):
        if msgs is LM_MSGS:
            values = [[{rnd.randrange(99): ["x", [], {}] for _ in range(rnd.randint(0, 70))}, {}, None, None] for _ in range(900)]
        elif msgs is utf:
            values = [["ok" if rnd.random() < 0.8 else "\udcff", [["a", "\udcfe" if rnd.random() < 0.1 else "b"]]] for _ in range(900)]
        else:
            values = [make(rnd, msgs, 0) for _ in range(900)]
        rows, off = _spoil(rnd, msgs, values)
        frames, meta = M.encode(msgs, 0, rows, off)
        d_out, d_off, d_meta = eng.proto_encode_nested_device(msgs, 0, rows, off)
        torch.cuda.synchronize()
        res = (d_out.cpu().numpy(), d_off.cpu().numpy().view(np.uint32), d_meta.cpu().numpy().view(np.uint32))
        _check_rows(res, frames, meta)
        for chunk in (1, 128, 129, 65536):
            eng.set_chunk(chunk)
            for pinned in (False, True):
                got = eng.proto_encode_batch(msgs, 0, rows, off, pinned=pinned)
                _check_rows(got, frames, meta)
                checked += len(values)
        if msgs is utf:
            assert BAD_UTF8 in meta
        assert BAD_ROW in meta or msgs is utf
        # decode(encode(rows)) == rows through the two host calls
        good = [i for i in range(len(values)) if meta[i] == OK]
        rows_g, off_g = S.pack_proto_nested_rows(msgs, 0, [values[i] for i in good])
        fo, fo_off, fm = eng.proto_encode_batch(msgs, 0, rows_g, off_g)
        assert (fm == OK).all()
        ro, ro_off, rm = eng.proto_decode_batch(msgs, 0, fo, fo_off)
        assert (rm == OK).all()
        assert ro.tobytes() == rows_g[:int(off_g[-1])].tobytes()
    eng.set_chunk(65536)
    # ---- a record alone beyond the per-slot budget: its own chunk ----
    msgs = [[F(1, S.PB_STRING), F(2, S.PB_INT32)]]
    big = b"a" * (33 << 20)
    frames = [H.frame(b"\x10\x07"), H.frame(b"\x0a" + H.varint(len(big)) + big + b"\x10\x05"), H.frame(b"\x0a\x01b")]
    per_byte, per_record = nested_bound(msgs, 0, True)
    assert per_byte * len(frames[1]) + per_record > 256 << 20
    want = [b"\0" * 4 + (7).to_bytes(4, "little"), len(big).to_bytes(4, "little") + (5).to_bytes(4, "little") + big,
            (1).to_bytes(4, "little") + b"\0" * 4 + b"b\0\0\0"]
    raw, in_off = H.pack_frames(frames)
    for pinned in (False, True):
        _check_rows(eng.proto_decode_batch(msgs, 0, raw, in_off, pinned=pinned), want, [OK] * 3)
    eng.close()
    print("%d records through the host path on the GPU, equal to the model and the resident calls" % checked)


def _call(eng, msgs, data, off, out, out_cap, out_off, meta, decode, n=None):
    """the C call on caller buffers → (submit code, wait code or None, out_bytes)"""
    import ctypes as C
    from gofr_b200 import _abi
    nm, nf, k = S.proto_nested_tables(msgs)
    pr = S.proto_nested_presence(msgs)
    L = _abi.lib()
    n = len(off) - 1 if n is None else n
    pb = _abi.ProtoBatch(data=data.ctypes.data if data is not None else None, data_bytes=0 if data is None else data.size,
                         off=off.ctypes.data if off is not None else None, n=n)
    ob = _abi.RespBatch(out=None if out is None else out.ctypes.data, out_cap=out_cap, out_off=None if out_off is None else out_off.ctypes.data,
                        meta=None if meta is None else meta.ctypes.data, out_bytes=0)
    t = C.c_uint64()
    fn = L.gofr_proto_batch_decode if decode else L.gofr_proto_batch_encode
    rc = fn(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, None if pr is None else pr.ctypes.data, C.byref(pb), C.byref(ob), C.byref(t))
    if rc != 0:
        return rc, None, 0
    return rc, L.gofr_batch_wait(eng._e, t.value), int(ob.out_bytes)


def _gpu_edges(seed):
    import torch
    from gofr_b200 import synth
    from gofr_b200.engine import Engine, pinned_array
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    eng = Engine(Table(synth.config1_spec()), 0)
    INVALID, CAPACITY = 1, 7
    msgs = LM_MSGS
    frames = _damage(rnd, _lm_frames(rnd, 700))
    want_rows, want_meta = model_decode(msgs, frames)
    raw, in_off = H.pack_frames(frames)
    n = len(frames)
    total = sum(len(r) for r in want_rows)
    CANARY = 0xA5
    # ---- capacity: exact succeeds, one byte less is GOFR_ERR_CAPACITY with nothing past out_cap and meta complete ----
    for chunk in (128, 65536):
        eng.set_chunk(chunk)
        for pinned in (False, True):
            for cap in (total, total - 1):
                if pinned:
                    out, out_off, meta = pinned_array(cap + 256), pinned_array(4 * (n + 1), np.uint32), pinned_array(4 * n, np.uint32)
                    out[:] = CANARY
                else:
                    out, out_off, meta = np.full(cap + 256, CANARY, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.uint32)
                meta[:] = 0xFFFFFFFF
                rc, wrc, nbytes = _call(eng, msgs, raw, in_off, out, cap, out_off, meta, True)
                assert rc == 0
                assert list(meta) == list(want_meta)
                assert (out[cap:] == CANARY).all()
                if cap == total:
                    assert wrc == 0 and nbytes == total
                    _check_rows((out, out_off, meta), want_rows, want_meta)
                else:
                    assert wrc == CAPACITY and nbytes < total and int(out_off[n]) == nbytes
            # the same engine then serves a good batch correctly
            _check_rows(eng.proto_decode_batch(msgs, 0, raw, in_off, pinned=pinned), want_rows, want_meta)
    # ---- bad offsets in a later chunk: GOFR_ERR_INVALID, nothing in flight, the next batch right ----
    eng.set_chunk(128)
    rows, off = S.pack_proto_nested_rows(LM_MSGS, 0, [[{}, {}, [k], None] for k in range(1000)])
    enc_frames, enc_meta = M.encode(LM_MSGS, 0, rows, off)
    for pinned in (False, True):
        for decode, data, offs in ((True, raw, in_off), (False, rows, off)):
            cases = []
            o = offs.copy(); o[600] = o[599] - 1; cases.append(o)                  # decreasing
            o = offs.copy(); o[-1] = data.size + 1; cases.append(o)                # past data_bytes
            if not decode:
                o = offs.copy(); o[500] = o[500] + 2; cases.append(o)              # a row offset not a multiple of 4
            for o in cases:
                m = len(o) - 1
                if pinned:
                    out, out_off, meta = pinned_array(1 << 22), pinned_array(4 * (m + 1), np.uint32), pinned_array(4 * m, np.uint32)
                else:
                    out, out_off, meta = np.zeros(1 << 22, np.uint8), np.zeros(m + 1, np.uint32), np.zeros(m, np.uint32)
                rc, _, _ = _call(eng, msgs, data, o, out, out.size, out_off, meta, decode)
                assert rc == INVALID
            if decode:
                _check_rows(eng.proto_decode_batch(msgs, 0, raw, in_off, pinned=pinned), want_rows, want_meta)
            else:
                _check_rows(eng.proto_encode_batch(msgs, 0, rows, off, pinned=pinned), enc_frames, enc_meta)
    # ---- n == 0 with no buffers, and through the Engine calls ----
    for decode in (True, False):
        assert _call(eng, msgs, None, None, None, 0, None, None, decode, n=0)[:2] == (0, 0)
        z = (eng.proto_decode_batch if decode else eng.proto_encode_batch)(msgs, 0, np.zeros(0, np.uint8), np.zeros(1, np.uint32))
        assert z[0].size == 0 and list(z[1]) == [0] and z[2].size == 0
    eng.close()
    print("capacity, bad offsets and empty batches: as documented")


@pytest.mark.gpu
def test_gpu_host_path_matches_model_and_resident_calls():
    out = H.run_child("import tests.test_proto_batch as t; t._gpu_codec(6060)", timeout=1800)
    assert "equal to the model and the resident calls" in out


@pytest.mark.gpu
def test_gpu_capacity_bad_offsets_and_empty_batches():
    out = H.run_child("import tests.test_proto_batch as t; t._gpu_edges(6161)")
    assert "as documented" in out


@pytest.mark.gpu
def test_gpu_say_hello(tmp_path):
    """examples/cpp/grpc_hello.cpp answers the reference's three cases, with the bytes python protobuf marshals"""
    from gofr_b200 import _abi
    _abi.lib()
    exe = str(tmp_path / "grpc_hello")
    _compile_hello(exe)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln.split("\t") for ln in r.stdout.splitlines()]
    assert [m for m, _ in lines] == ["Hello world!", "Hello 123!", "Hello World!"]
    cls = H.py_classes([[F(1, S.PB_STRING)]])[0]
    for m, hx in lines:
        obj = cls()
        setattr(obj, obj.DESCRIPTOR.fields[0].name, m)
        assert bytes.fromhex(hx) == H.frame(obj.SerializeToString())
