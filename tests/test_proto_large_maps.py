"""The second pass of the nested proto3 decoder (gofr_proto_decode_nested_deferred_device): frames the first pass answered
DEFER are decoded again with map fields of up to 4096 entries, entries put in key order by sorted lists instead of
selection.  Statements compared: the model (tests/proto_nested_model.py) with its entry limit at 4096, the device code on
the CPU (tests/emu/emu_deferred: the walk with the sorted-list map step, the lists built, sorted and compacted by the same
code as a CTA of one thread), pure-Python protobuf, the first pass wherever it answers, and with -m gpu the CUDA kernel."""
import random

import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200.engine import row_growth_bound
from tests import proto_nested_harness as H
from tests import proto_nested_model as M
from tests.emu import emu, emu_deferred

F = S.ProtoNField
LIMIT = 4096
OK, BAD_PROTO, BAD_UTF8, DEFER = M.OK, M.BAD_PROTO, M.BAD_UTF8, M.DEFER


def _uvarint(b, i):
    v = s = 0
    while True:
        c = b[i]
        i += 1
        v |= (c & 0x7F) << s
        s += 7
        if c < 0x80:
            return v, i


def items(body: bytes):
    """the top-level items of a well-formed message body (tag through payload)"""
    out, i = [], 0
    while i < len(body):
        j = i
        tag, j = _uvarint(body, j)
        wt = tag & 7
        if wt == 0:
            _, j = _uvarint(body, j)
        elif wt == 1:
            j += 8
        elif wt == 5:
            j += 4
        else:
            ln, j = _uvarint(body, j)
            j += ln
        out.append(body[i:j])
        i = j
    return out


def encode(msgs, values):
    """frames of value lists, by the device encoder on the CPU (Deterministic bytes)"""
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    out, o, meta = emu.proto_encode_nested(msgs, 0, rows, off, presence_instance=True)
    assert list(meta) == [OK] * len(values)
    return H.frames_of(out, o)


def shuffled(rnd, *frames):
    """one frame of all the items of the given frames, in a random order"""
    its = [it for fr in frames for it in items(fr[5:])]
    rnd.shuffle(its)
    return H.frame(b"".join(its))


def second_pass(msgs, frames, meta_in=None):
    """both passes on the CPU.  The first equals the model (limit 64); the second equals the model with the limit at 4096
    where meta_in (default: the first pass's statuses) is DEFER, and passes every other status through with an empty row.
    Returns (first rows, first meta, second rows, second meta)."""
    rows1, meta1 = H.decode_model_emu(msgs, 0, frames, presence_instance=True)
    meta_in = list(meta1) if meta_in is None else list(meta_in)
    raw, in_off = H.pack_frames(frames)
    e_rows, e_off, e_meta = emu_deferred.proto_decode_nested_deferred(msgs, 0, raw, in_off, np.array(meta_in, dtype=np.uint32))
    want_rows, want_meta = model_decode(msgs, 0, frames)
    rows2 = [want_rows[i] if meta_in[i] == DEFER else b"" for i in range(len(frames))]
    meta2 = [want_meta[i] if meta_in[i] == DEFER else meta_in[i] for i in range(len(frames))]
    assert list(e_meta) == meta2, [(i, a, b) for i, (a, b) in enumerate(zip(list(e_meta), meta2)) if a != b][:5]
    assert np.array_equal(e_off, np.cumsum([0] + [len(r) for r in rows2]).astype(np.uint32))
    for i, r in enumerate(rows2):
        assert e_rows[int(e_off[i]):int(e_off[i + 1])].tobytes() == r, i
    assert (e_rows[int(e_off[-1]):] == 0xEE).all()
    return rows1, meta1, rows2, meta2


def model_decode(msgs, root, frames, max_map_entries=LIMIT):
    """the model's decode with its map entry limit at max_map_entries instead of the first pass's 64 (the model reads
    MAX_MAP_ENTRIES on every call)"""
    saved = M.MAX_MAP_ENTRIES
    M.MAX_MAP_ENTRIES = max_map_entries
    try:
        return M.decode(msgs, root, frames)
    finally:
        M.MAX_MAP_ENTRIES = saved


def check_python(msgs, frames, rows, meta):
    H.check_python_parse(msgs, 0, frames, rows, meta)


def rand_keys(rnd, t, n):
    """n keys of type t (fewer distinct ones for bool)"""
    if t == S.PB_BOOL:
        return [rnd.random() < 0.5 for _ in range(n)]
    if t == S.PB_STRING:
        stems = ["", "a", "ab", "abc", "abd", "é", "日本", "k\x00", "zz" * 10]
        return [rnd.choice(stems) + ("" if rnd.random() < 0.1 else str(rnd.randrange(4 * n))) for _ in range(n)]
    lo, hi = (-2 ** 31, 2 ** 31 - 1) if t in (S.PB_INT32, S.PB_SINT32, S.PB_SFIXED32) else \
        (0, 2 ** 32 - 1) if t in (S.PB_UINT32, S.PB_FIXED32) else \
        (0, 2 ** 64 - 1) if t in (S.PB_UINT64, S.PB_FIXED64) else (-2 ** 63, 2 ** 63 - 1)
    small = (-4 * n, 4 * n) if lo < 0 else (0, 8 * n)
    return [rnd.choice([lo, hi, 0, small[0]]) if rnd.random() < 0.1 else rnd.randint(lo, hi) if rnd.random() < 0.5 else rnd.randint(*small)
            for _ in range(n)]


def map_frame(rnd, msgs, kt, n, value=lambda rnd, k: rnd.randrange(1000)):
    """a frame of map field 1 with n entries on the wire in a random order: two maps' worth of keys, so keys repeat"""
    keys = rand_keys(rnd, kt, n)
    half = n // 2
    a = {k: value(rnd, k) for k in keys[:half]}
    b = {k: value(rnd, k) for k in keys[half:]}
    fa, fb = encode(msgs, [[a], [b]])
    fr = shuffled(rnd, fa, fb)
    have = len(items(fr[5:]))
    if have < n:      # equal keys inside one half collapsed: top up with copies of entries already there
        its = items(fr[5:])
        fr = H.frame(fr[5:] + b"".join(rnd.choice(its) for _ in range(n - have)))
    return fr


# ---------------------------------------------------------------------------------------------------------------
# the CPU: model with the limit at 4096, device code, python protobuf
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kt", H.KEYS)
def test_every_key_kind(kt):
    """map<K, string> and map<K, int64> with 65 and 300 entries on the wire, shuffled, duplicate keys"""
    rnd = random.Random(7000 + kt)
    for vt in (S.PB_STRING, S.PB_INT64):
        msgs = [[F(1, S.PB_MAP, False, 1)], [F(1, kt), F(2, vt)]]
        val = (lambda r, k: "v%d" % r.randrange(99)) if vt == S.PB_STRING else (lambda r, k: r.randint(-2 ** 63, 2 ** 63 - 1))
        frames = [map_frame(rnd, msgs, kt, n, val) for n in (65, 300, 65, 300)]
        _, meta1, rows2, meta2 = second_pass(msgs, frames)
        assert meta1 == [DEFER] * 4 and meta2 == [OK] * 4
        check_python(msgs, frames, rows2, meta2)


def test_entry_counts():
    """65, 1000 and 4096 entries decode; 4097 stay DEFER, duplicates counted"""
    rnd = random.Random(11)
    msgs = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_STRING)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]]
    ents = lambda keys: b"".join(H._entry(1, b"\x08" + H.varint(k & (2 ** 64 - 1)) + b"\x10" + H.varint(rnd.randrange(2 ** 31))) for k in keys)
    frames = []
    for n in (65, 1000, 4096, 4097):
        keys = rnd.sample(range(-5000, 5000), n)
        frames.append(H.frame(ents(keys) + H._s(2, b"tail")))
    frames.append(H.frame(ents([rnd.randrange(50) for _ in range(4096)])))    # 4096 on the wire, 50 keys
    frames.append(H.frame(ents([rnd.randrange(50) for _ in range(4097)])))    # 4097 on the wire, 50 keys
    _, meta1, rows2, meta2 = second_pass(msgs, frames)
    assert meta1 == [DEFER] * 6
    assert meta2 == [OK, OK, OK, DEFER, OK, DEFER]
    check_python(msgs, frames, rows2, meta2)
    assert int.from_bytes(rows2[2][:4], "little") == 4096


def test_duplicate_keys_last_wins():
    """of equal keys the last on the wire wins, wherever the copies are"""
    msgs = H.NONCANON_MSGS
    body = b"".join(H._B(k % 40, k) for k in range(200)) + H._A(b"x", H._V1) + b"".join(H._B(k, -k) for k in range(39, -1, -1))
    frames = [H.frame(body)]
    _, meta1, rows2, meta2 = second_pass(msgs, frames)
    assert meta1 == [DEFER] and meta2 == [OK]
    want, _ = S.pack_proto_nested_rows(msgs, 0, [[{"x": [1, {}]}, {k: -k for k in range(40)}, {}, 0]])
    assert rows2[0] == want[:len(rows2[0])].tobytes()
    check_python(msgs, frames, rows2, meta2)


def test_string_keys_shared_prefixes_and_empty():
    rnd = random.Random(13)
    msgs = [[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_STRING), F(2, S.PB_BYTES)]]
    keys = ["", "a", "a\x00", "aa", "ab", "abc", "abcd", "abcd" * 20, "b", "é", "日", "日本"] + ["p" * k for k in range(60)]
    frames = []
    for _ in range(4):
        ks = keys + [rnd.choice(keys) for _ in range(100)]
        rnd.shuffle(ks)
        frames.append(H.frame(b"".join(H._entry(1, H._s(1, k.encode()) + H._s(2, bytes([rnd.randrange(256)]))) for k in ks)))
    frames.append(H.frame(b"".join(H._entry(1, H._s(2, b"%d" % k)) for k in range(70))))   # 70 entries, all of key ""
    _, _, rows2, meta2 = second_pass(msgs, frames)
    assert meta2 == [OK] * 5
    check_python(msgs, frames, rows2, meta2)


def test_maps_inside_map_values():
    """map<string, V> with V { int32 x; map<int64, string> m }: both levels beyond 64 entries, and a third map beside"""
    rnd = random.Random(17)
    msgs = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 3)], [F(1, S.PB_STRING), F(2, S.PB_MESSAGE, False, 2)],
            [F(1, S.PB_INT32), F(2, S.PB_MAP, False, 4)], [F(1, S.PB_UINT32), F(2, S.PB_BOOL)], [F(1, S.PB_INT64), F(2, S.PB_STRING)]]
    frames = []
    for n_out, n_in in ((70, 70), (100, 3), (5, 300), (66, 66)):
        outer = {}
        for k in rand_keys(rnd, S.PB_STRING, n_out):
            inner = {x: "s%d" % rnd.randrange(9) for x in rand_keys(rnd, S.PB_INT64, n_in)}
            outer[k] = [rnd.randrange(100), inner]
        side = {rnd.randrange(2 ** 32): rnd.random() < 0.5 for _ in range(80)}
        fr = encode(msgs, [[outer, side]])[0]
        frames.append(shuffled(rnd, fr))
    _, meta1, rows2, meta2 = second_pass(msgs, frames)
    assert meta1 == [DEFER] * 4 and meta2 == [OK] * 4
    check_python(msgs, frames, rows2, meta2)


def test_presence_types():
    """optional fields and oneofs beside and inside large maps"""
    rnd = random.Random(19)
    msgs = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_STRING, presence=S.PB_OPTIONAL), F(3, S.PB_INT32, presence=1),
             F(4, S.PB_MESSAGE, False, 2, presence=1)],
            [F(1, S.PB_SINT64), F(2, S.PB_MESSAGE, False, 2)],
            [F(1, S.PB_DOUBLE, presence=S.PB_OPTIONAL), F(2, S.PB_BYTES, presence=2), F(3, S.PB_UINT64, presence=2)]]
    frames = []
    for n in (100, 200, 10):
        vals = [H.rand_presence_value(rnd, msgs, 2) for _ in range(n)]
        m = {k: v for k, v in zip(rand_keys(rnd, S.PB_SINT64, n), vals)}
        top = H.rand_presence_value(rnd, msgs, 0)
        top[0] = m
        frames.append(shuffled(rnd, encode(msgs, [top])[0]))
    rows1, meta1, rows2, meta2 = second_pass(msgs, frames, meta_in=[DEFER] * 3)
    assert meta1 == [DEFER, DEFER, OK] and meta2 == [OK, OK, OK]
    check_python(msgs, frames, rows2, meta2)
    assert rows2[2] == rows1[2]    # selected by mistake: the first pass's row


def test_still_deferred_and_precedence():
    """4097 entries and merges stay DEFER; malformed and invalid UTF-8 beat DEFER as in the first pass"""
    msgs = H.NONCANON_MSGS
    big = b"".join(H._B(k, k) for k in range(4097))
    frames = [H.frame(big),
              H.frame(b"".join(H._B(k, k) for k in range(100)) + H._entry(1, H._s(1, b"k") + H._s(2, H._V1) + H._s(2, H._V2))),
              H.frame(big + H._entry(1, b"\x0a\x05ab")),
              H.frame(big + H._entry(1, H._s(1, b"\xff"))),
              H.frame(b"".join(H._B(k, k) for k in range(100)) + H._entry(1, H._s(1, b"\xff")))]
    _, meta1, _, meta2 = second_pass(msgs, frames)
    assert meta1 == [DEFER, DEFER, BAD_PROTO, BAD_UTF8, BAD_UTF8]
    assert meta2 == [DEFER, DEFER, BAD_PROTO, BAD_UTF8, BAD_UTF8]
    # a singular message sent twice stays DEFER in a description without maps as well
    flat = H.HOSTILE_MSGS
    frames = [H.frame(b) for b in H.HOSTILE_BODIES]
    _, meta1, _, meta2 = second_pass(flat, frames, meta_in=[DEFER] * len(frames))
    assert meta2 == meta1 and DEFER in meta2


def test_status_pass_through():
    """frames not selected keep their status (whatever it is) and get an empty row; d_meta is the merged column"""
    rnd = random.Random(23)
    msgs = H.NONCANON_MSGS
    frames = [H.frame(b) for b in H.NONCANON_OK + H.NONCANON_DEFER + H.NONCANON_BAD] * 3
    meta_in = [rnd.choice([OK, DEFER, DEFER, BAD_PROTO, 77]) for _ in frames]
    second_pass(msgs, frames, meta_in)


@pytest.mark.parametrize("seed", range(12))
def test_equals_first_pass_on_random_campaigns(seed):
    """random map (and presence) types, frames mutated as test_proto_maps mutates them, every frame selected: wherever
    the first pass answers anything but DEFER, the second gives the same status and row"""
    rnd = random.Random(9100 + seed)
    msgs = H.rand_map_types(rnd) if seed % 3 else H.rand_presence_types(rnd)
    make = H.rand_map_value if seed % 3 else H.rand_presence_value
    values = [make(rnd, msgs, 0) for _ in range(60)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    frames, meta = M.encode(msgs, 0, rows, off)
    out = []
    for fr in (f for f, m in zip(frames, meta) if m == OK):
        body = bytearray(fr[5:])
        for _ in range(rnd.randint(0, 3)):
            r = rnd.random()
            if body and r < 0.35:
                body[rnd.randrange(len(body))] ^= 1 << rnd.randrange(8)
            elif body and r < 0.5:
                del body[rnd.randrange(len(body)):]
            elif r < 0.75:
                p = rnd.randrange(len(body) + 1)
                body[p:p] = rnd.choice([b"\x08\x01", b"\x0b\x0c", b"\x12\x00", b"\x0a\x00", b"\x0a\x02\x08\x01", b"\x80"])
            else:
                p = rnd.randrange(len(body) + 1)
                body = body[p:] + body[:p]
        out.append(H.frame(bytes(body)))
    rows1, meta1, rows2, meta2 = second_pass(msgs, out, meta_in=[DEFER] * len(out))
    for i in range(len(out)):
        if meta1[i] != DEFER:
            assert (meta2[i], rows2[i]) == (meta1[i], rows1[i]), i
    # the default capacity of Engine.proto_decode_nested_deferred_device covers every row
    per_byte, per_frame = row_growth_bound(msgs, 0)
    assert all(len(r) <= per_byte * len(fr) + per_frame for r, fr in zip(rows2, out))


def test_growth_bound_on_dense_elements():
    """the rows that grow most per wire byte: empty repeated messages with wide fixed parts, empty map entries, packed
    varints of 64-bit kinds"""
    wide = [F(k, S.PB_FIXED64) for k in range(1, 9)]
    msgs = [[F(1, S.PB_MESSAGE, True, 1), F(2, S.PB_MAP, False, 2), F(3, S.PB_INT64, True)], wide, [F(1, S.PB_BOOL), F(2, S.PB_MESSAGE, False, 1)]]
    body = b"\x0a\x00" * 50 + b"\x12\x00" * 70 + b"\x1a\x40" + b"\x01" * 64
    frames = [H.frame(body)]
    _, _, rows2, meta2 = second_pass(msgs, frames, meta_in=[DEFER])
    per_byte, per_frame = row_growth_bound(msgs, 0)
    assert meta2 == [OK] and len(rows2[0]) <= per_byte * len(frames[0]) + per_frame


# ---------------------------------------------------------------------------------------------------------------
# the CUDA kernel
# ---------------------------------------------------------------------------------------------------------------
def _gpu_check(seed):
    """the kernel against the model and the first pass, run in a child process (H.run_child)"""
    import torch
    from gofr_b200 import _abi, synth
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    assert torch.cuda.is_available()
    rnd = random.Random(seed)
    eng = Engine(Table(synth.config1_spec()), 0)
    dev = torch.device("cuda", 0)
    CANARY = 0xEEEEEEEE

    msgs = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 3), F(3, S.PB_MESSAGE, False, 4), F(4, S.PB_STRING, presence=S.PB_OPTIONAL)],
            [F(1, S.PB_INT64), F(2, S.PB_MESSAGE, False, 2)],
            [F(1, S.PB_STRING), F(2, S.PB_DOUBLE, True), F(3, S.PB_MAP, False, 5)],
            [F(1, S.PB_STRING), F(2, S.PB_STRING)],
            [F(1, S.PB_INT32)],
            [F(1, S.PB_UINT32), F(2, S.PB_INT32)]]
    nested = lambda r: {k: r.randint(0, 9) for k in rand_keys(r, S.PB_UINT32, r.choice([0, 2, 70]))}   # noqa: E731
    small = lambda r: [{k: ["n%d" % k, [0.5], {}] for k in rand_keys(r, S.PB_INT64, r.randint(0, 5))}, {}, [1], None]  # noqa: E731

    def large(r):
        items_ = {k: ["n%d" % r.randrange(9), [1.0] * r.randint(0, 2), nested(r) if r.random() < 0.2 else {}]
                  for k in rand_keys(r, S.PB_INT64, r.randint(65, 500))}
        labels = {k: "v" + k for k in rand_keys(r, S.PB_STRING, r.randint(0, 300))}
        return [items_, labels, [r.randint(0, 5)], "o"]

    def batch(n, kinds):
        frames = []
        for _ in range(n):
            kind = rnd.choice(kinds)
            if kind == "large":
                frames.append(shuffled(rnd, encode(msgs, [large(rnd)])[0]))
            elif kind == "normal":
                frames.append(encode(msgs, [small(rnd)])[0])
            elif kind == "merged":   # message field 3 sent twice
                frames.append(H.frame(encode(msgs, [small(rnd)])[0][5:] + b"\x1a\x02\x08\x01"))
            elif kind == "bad":
                frames.append(H.frame(encode(msgs, [large(rnd)])[0][5:] + b"\x0a\x05ab"))
            else:                    # 4097 entries
                frames.append(H.frame(b"".join(H._entry(2, H._s(1, b"%d" % k)) for k in range(4097))))
        return frames

    def run(frames, meta_in, rows_cap, alias):
        n = len(frames)
        raw, in_off = H.pack_frames(frames)
        d_in = torch.from_numpy(raw).to(dev)
        d_off = torch.from_numpy(in_off.view(np.int32)).to(dev)
        m_in = torch.full((n + 8,), CANARY - 2 ** 32, dtype=torch.int32, device=dev)
        m_in[:n] = torch.from_numpy(np.array(meta_in, dtype=np.uint32).view(np.int32)).to(dev)
        rows = torch.full((rows_cap + 64,), 0xEE, dtype=torch.uint8, device=dev)
        row_off = torch.full((n + 9,), CANARY - 2 ** 32, dtype=torch.int32, device=dev)
        meta = m_in if alias else torch.full((n + 8,), CANARY - 2 ** 32, dtype=torch.int32, device=dev)
        nm, nf, k = S.proto_nested_tables(msgs)
        pr = S.proto_nested_presence(msgs)
        _abi.check(_abi.lib().gofr_proto_decode_nested_deferred_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, pr.ctypes.data,
                                                                       d_in.data_ptr(), d_off.data_ptr(), n, m_in.data_ptr(), rows.data_ptr(),
                                                                       rows_cap, row_off.data_ptr(), meta.data_ptr(), None), "deferred")
        torch.cuda.synchronize()
        return (rows.cpu().numpy(), row_off.cpu().numpy().view(np.uint32), meta.cpu().numpy().view(np.uint32))

    def check(frames, meta_in, exact_cap=False, alias=False):
        n = len(frames)
        want_rows, want_meta = model_decode(msgs, 0, frames)
        rows2 = [want_rows[i] if meta_in[i] == DEFER else b"" for i in range(n)]
        meta2 = [want_meta[i] if meta_in[i] == DEFER else meta_in[i] for i in range(n)]
        want_off = np.cumsum([0] + [len(r) for r in rows2]).astype(np.uint32)
        total = int(want_off[-1])
        caps = [total, total - 1] if exact_cap and total else [total + 1000]
        for cap in caps:
            eng.overflowed(reset=True)
            g_rows, g_off, g_meta = run(frames, meta_in, cap, alias)
            assert list(g_meta[:n]) == meta2, [(i, a, b) for i, (a, b) in enumerate(zip(g_meta, meta2)) if a != b][:5]
            assert (g_meta[n:] == CANARY).all()
            assert np.array_equal(g_off[:n + 1], want_off) and (g_off[n + 1:] == CANARY).all()
            over = eng.overflowed(reset=True)
            assert over == (cap < total), (cap, total)
            if cap >= total:
                assert g_rows[:total].tobytes() == b"".join(rows2)
            else:                                      # whole tiles dropped: those written are right, nothing past cap
                for t0 in range(0, n, 128):
                    lo, hi = int(want_off[t0]), int(want_off[min(n, t0 + 128)])
                    if hi <= cap and lo < hi and (g_rows[lo:hi] != 0xEE).any():
                        assert g_rows[lo:hi].tobytes() == b"".join(rows2[t0:t0 + 128])
            assert (g_rows[min(cap, total):] == 0xEE).all()
        return rows2, meta2

    checked = 0
    # first pass on the GPU, then the second on its statuses, aliased and not
    for n, kinds in ((0, ["normal"]), (1, ["large"]), (127, ["normal", "large", "merged", "bad", "huge"]), (128, ["large"]),
                     (129, ["normal", "large"]), (3000, ["normal"] * 12 + ["large", "merged", "bad", "huge"])):
        frames = batch(n, kinds)
        raw, in_off = H.pack_frames(frames)
        _, _, g1 = eng.proto_decode_nested_device(msgs, 0, raw, in_off)
        meta1 = list(g1.cpu().numpy().view(np.uint32)) if n else []
        assert meta1 == M.decode(msgs, 0, frames)[1]
        if n > 128:                        # a tile with no selected frame (the 128 batch: a tile whose selected frames all are large)
            for i in range(128):
                if meta1[i] == DEFER:
                    meta1[i] = OK
        for alias in (False, True):
            check(frames, meta1, alias=alias)
        wrong = [DEFER if rnd.random() < 0.3 else m for m in meta1]       # a wrong selection
        check(frames, wrong, exact_cap=True)
        checked += n
    # the Engine call with its default capacity, and a round trip of 65..4096-entry rows through encoder and both passes
    values = [[{k: ["n", [], {}] for k in range(m)}, {str(k): "x" * (k % 7) for k in range(m // 2)}, None, None]
              for m in (65, 100, 1000, 4096)]
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    d_out, d_off, d_meta = eng.proto_encode_nested_device(msgs, 0, rows, off)
    torch.cuda.synchronize()
    assert (d_meta.cpu().numpy() == 0).all()
    o = d_off.cpu().numpy().view(np.uint32)
    frames = H.frames_of(d_out[:int(o[-1])].cpu().numpy(), o)
    raw, in_off = H.pack_frames(frames)
    _, _, m1 = eng.proto_decode_nested_device(msgs, 0, raw, in_off)
    assert (m1.cpu().numpy() == DEFER).all()
    g_rows, g_off, g_meta = eng.proto_decode_nested_deferred_device(msgs, 0, raw, in_off, m1, meta_out=m1)
    torch.cuda.synchronize()
    assert (g_meta.cpu().numpy() == OK).all() and (m1.cpu().numpy() == OK).all()
    go = g_off.cpu().numpy().view(np.uint32)
    for i in range(len(values)):
        assert g_rows[int(go[i]):int(go[i + 1])].cpu().numpy().tobytes() == rows[int(off[i]):int(off[i + 1])].tobytes(), i
    eng.close()
    print("%d frames through the second pass on the GPU, equal to the model" % checked)


@pytest.mark.gpu
def test_gpu_second_pass_matches_model():
    out = H.run_child("import tests.test_proto_large_maps as t; t._gpu_check(4242)")
    assert "equal to the model" in out
