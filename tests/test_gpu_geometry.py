"""The GPU-only serve machinery against the oracle, across batch sizes, tile budgets and arena layouts.

The CPU emulation runs the per-request device code; what only exists in the kernels is checked here: the TMA staging of a
tile's arena span (and the HBM path when the span is over the budget), the block scan and the look-back that chain packed
offsets, the slot layout's regrouping by shape class and its deferred general pass, the host-path chunk pipeline and the
VALUES kernel instances.  Every batch the other GPU tests serve comes from RequestBatch.pack: request bytes in index order,
contiguous, never shared.  The ABI (include/gofr_b200.h) asks less — arena_off a multiple of 4, and 16 readable bytes past
the last request byte — and the kernels take the min / max over a tile for any order, so `relayout` places the same requests
in other orders, with gaps, off 16-byte alignment, sharing bytes, at the arena's very end.

Each GPU result is checked three ways: equal to the oracle for every request (with an output capacity summed from
gofr_table_response_bound: shared bytes make the oracle's default capacity too small), byte for byte equal to the GPU run
of the packed layout of the same requests, and for VALUES rows the body equals `go_json`, the Python model.  The unmarked
tests show on the CPU that the oracle and the device code in the emulation give the same bytes for every layout, so a
layout-dependent GPU mismatch is a kernel finding.
"""
import random

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O
from tests import test_route as TR
from tests import test_values as TV
from tests.emu import emu as E

DATE = S.http_date(1_700_000_000)
T = 128                       # requests per tile (kServeT)
MODES = ["reversed", "shuffled", "gaps", "misaligned", "shared", "empty", "tight"]


# ---------------------------------------------------------------------------------------------------------------
# layouts
# ---------------------------------------------------------------------------------------------------------------
def _records(batch):
    """each request's bytes as the ABI lays them out from arena_off: path, query, zero padding to 4, data"""
    d, a = batch.desc, batch.arena
    recs = []
    for off, pl, ql, dl in zip(d["arena_off"].tolist(), d["path_len"].tolist(), d["query_len"].tolist(), d["data_len"].tolist()):
        doff = (off + pl + ql + 3) & ~3
        recs.append(a[off:off + pl + ql].tobytes() + bytes(doff - off - pl - ql) + a[doff:doff + dl].tobytes())
    return recs


def _assemble(batch, recs, offs, size):
    arena = np.zeros(size, dtype=np.uint8)
    for r, o in zip(recs, offs):
        if r:
            arena[o:o + len(r)] = np.frombuffer(r, dtype=np.uint8)
    desc = batch.desc.copy()
    desc["arena_off"] = np.asarray(offs, dtype=np.uint32)
    return S.RequestBatch(desc, batch.trace_ids.copy(), arena)


def relayout(batch, mode, rnd):
    """The same requests (descriptors apart from arena_off, trace ids) with their bytes placed
      reversed / shuffled:  in reverse or random order;
      gaps:                 in order, with random 4-aligned gaps between them;
      misaligned:           in order, every arena_off = 4, 8 or 12 (mod 16);
      shared:               identical requests point at one copy of their bytes;
      empty:                in order, and every zero-length request at one offset (inside another request's bytes);
      tight:                in order, and the arena ends with the last request's last byte (only the ABI's 16 bytes of
                            slack follow it on the device: see _upload)."""
    recs = _records(batch)
    n = len(recs)
    order = list(range(n))
    if mode == "reversed":
        order.reverse()
    elif mode == "shuffled":
        rnd.shuffle(order)
    offs, seen, cur = [0] * n, {}, 0
    for k, i in enumerate(order):
        r = recs[i]
        if mode == "shared" and r in seen:
            offs[i] = seen[r]
            continue
        if mode == "empty" and not r:
            offs[i] = -1
            continue
        cur = (cur + 3) & ~3
        if mode == "gaps":
            cur += 4 * rnd.randrange(16)
        elif mode == "misaligned":
            cur = ((cur + 15) & ~15) + 4 * (1 + k % 3)
        offs[i] = cur
        seen.setdefault(r, cur)
        cur += len(r)
    if mode == "empty":
        mid = next((o for o in offs[n // 2:] + offs if o >= 0), 0)
        offs = [mid if o < 0 else o for o in offs]
    size = cur if mode == "tight" else (cur + 15) & ~15
    return _assemble(batch, recs, offs, max(size, 0))


def tile_span_layout(batch, span):
    """Requests in index order, every tile of T starting on a 16-byte boundary with its last request moved so that the span
    the serve kernel stages, [min arena_off & ~15, (max end + 15) & ~15), is exactly `span` bytes — the request ends on a
    16-byte boundary whenever its length is a multiple of 4 (one with such a length is chosen where the tile has one).
    None when the tile's requests do not fit into `span`."""
    recs = _records(batch)
    n = len(recs)
    offs, cur = [0] * n, 0
    for t0 in range(0, n, T):
        idx = list(range(t0, min(n, t0 + T)))
        last = next((i for i in reversed(idx) if len(recs[i]) % 4 == 0 and recs[i]), idx[-1])
        lo = (cur + 15) & ~15
        cur = lo
        for i in idx:
            if i != last:
                cur = (cur + 3) & ~3
                offs[i] = cur
                cur += len(recs[i])
        o = (lo + span - len(recs[last])) & ~3
        if o < cur or o < lo:
            return None
        offs[last] = o
        cur = lo + span
    return _assemble(batch, recs, offs, cur)


def zero_length(batch, every):
    """every `every`-th request with no path, query or data (the input of the "empty" layout)"""
    recs = []
    d = batch.desc
    ar = batch.arena.tobytes()
    for i in range(batch.n):
        off, pl, ql, dl = int(d["arena_off"][i]), int(d["path_len"][i]), int(d["query_len"][i]), int(d["data_len"][i])
        if i % every == every - 1:
            recs.append(S.Req(int(d["method"][i]), b"", b"", b"", int(d["flags"][i]), batch.trace_ids[i].tobytes()))
        else:
            doff = (off + pl + ql + 3) & ~3
            recs.append(S.Req(int(d["method"][i]), ar[off:off + pl], ar[off + pl:off + pl + ql], ar[doff:doff + dl],
                              int(d["flags"][i]), batch.trace_ids[i].tobytes()))
    return S.RequestBatch.pack(recs)


def tile_of_copies(batch, tile):
    """the batch with every request of tile `tile` replaced by that tile's first request (under the "shared" layout the
    whole tile then points at one copy)"""
    lo, hi = tile * T, min(batch.n, tile * T + T)
    idx = np.arange(batch.n)
    idx[lo:hi] = lo
    b = S.RequestBatch(batch.desc[idx].copy(), batch.trace_ids.copy(), batch.arena)
    recs = _records(b)
    offs, cur = [], 0
    for r in recs:
        cur = (cur + 3) & ~3
        offs.append(cur)
        cur += len(r)
    return _assemble(b, recs, offs, (cur + 15) & ~15)


def replicate(batch, n):
    """n requests: the batch repeated (its arena once per repetition), cut at n"""
    k = -(-n // batch.n)
    size = int(batch.arena.size)
    desc = np.concatenate([batch.desc] * k)[:n].copy()
    desc["arena_off"] += (np.repeat(np.arange(k, dtype=np.uint32), batch.n)[:n] * np.uint32(size))
    return S.RequestBatch(desc, np.concatenate([batch.trace_ids] * k)[:n].copy(), np.concatenate([batch.arena] * k))


# ---------------------------------------------------------------------------------------------------------------
# tables and references
# ---------------------------------------------------------------------------------------------------------------
def _values_spec():
    return TV._spec(S.FRAME_WIRE, S.H_ROW, TV.LATE + [TV.USER])


def _values_batch(n, seed=21):
    """n VALUES rows (the LATE + USER table) and the Python model's body of each: 2 000 distinct rows, repeated"""
    spec = _values_spec()
    b, want = TV._batch(spec, min(n, 2000), seed, nan_rate=0.01, routed=TV.LATE + [TV.USER])
    return replicate(b, n), [want[i % b.n] for i in range(n)]


def _chain_spec():
    """an 8-level pointer chain (the walker's frame stack depth): L7 → *L6 → … → *L0 {V int64}"""
    chain = [S.Schema(100, "L0", [S.Field("V", S.F_INT64, "v")])]
    for k in range(1, 8):
        chain.append(S.Schema(100 + k, "L%d" % k, [S.Field("C", S.F_STRUCT, "c", container=S.C_PTR, elem_schema=99 + k)]))
    return S.TableSpec(schemas=chain, routes=[S.Route(S.M_GET, "/chain", S.H_ROW, schema_id=107)])


def _chain_batch(n, seed=3):
    spec = _chain_spec()
    rnd = random.Random(seed)
    reqs, want = [], []
    for i in range(min(n, 1000)):
        depth = rnd.randrange(9)                  # levels set below the top; 8: the int64 is reached
        v = [rnd.choice([0, -1, 2 ** 63 - 1, rnd.randrange(-10 ** 9, 10 ** 9)])]
        for _ in range(7):
            v = [v]
        def cut(x, k):
            return None if k == 0 else [cut(x[0], k - 1)] if isinstance(x[0], list) else x
        vals = cut(v, depth) if depth < 8 else v
        vals = vals if vals is not None else [None]
        sc = spec.schema(107)
        reqs.append(S.Req(S.M_GET, b"/chain", b"", sc.encode_row(vals, spec.schema)))
        want.append('{"data":%s}\n' % TV.go_json(spec, sc, vals))
    b = S.RequestBatch.pack(reqs, seed=seed)
    return replicate(b, n), [want[i % b.n] for i in range(n)]


TABLES = {
    "config2": (synth.config2_spec, lambda n: (synth.config2_batch(n, escape_every=13), None), 544),
    "config4": (synth.config4_spec, lambda n: (synth.config4_batch(n), None), 352),
    "config3": (synth.config3_spec, lambda n: (synth.config3_batch(n, variant_every=7), None), 1024),
    "values": (_values_spec, _values_batch, 2048),
}
_tables = {}


def _table(name):
    if name not in _tables:
        spec = TABLES[name][0]() if name in TABLES else name()
        _tables[name] = (spec, Table(spec), O.OracleTable(spec))
    return _tables[name]


def bound_total(table, batch):
    """Σ gofr_table_response_bound over the batch: what a host batcher sizes its output buffer from"""
    L, h = _abi.lib(), table.handle
    base = L.gofr_table_response_bound(h, 0, 0, 0)
    per_pq = L.gofr_table_response_bound(h, 1, 0, 0) - base
    per_data = L.gofr_table_response_bound(h, 0, 0, 1) - base
    d = batch.desc
    pq = d["path_len"].astype(np.int64) + d["query_len"].astype(np.int64)
    return int(batch.n * base + per_pq * pq.sum() + per_data * d["data_len"].astype(np.int64).sum())


def oracle(ot, table, batch):
    o, f, m = ot.serve(batch, DATE, out_cap=max(4096, bound_total(table, batch)))
    return o[:int(f[-1])], f, m


def _same(got, want, what):
    (o2, f2, m2), (o1, f1, m1) = got, want
    assert np.array_equal(m2, m1), f"{what}: status / route column differs at {np.flatnonzero(m2 != m1)[:5]}"
    assert np.array_equal(f2, f1), f"{what}: offsets differ from request {int(np.flatnonzero(f2 != f1)[0]) - 1}"
    if o2.tobytes() != o1.tobytes():
        bad = int(np.flatnonzero(o2 != o1)[0])
        i = int(np.searchsorted(f1, bad, side="right") - 1)
        raise AssertionError(f"{what}: request {i} differs: want {o1[f1[i]:f1[i + 1]].tobytes()[:300]!r} "
                             f"got {o2[f1[i]:f1[i + 1]].tobytes()[:300]!r}")


def _bodies_match_model(out, off, want, step=1):
    ob = out.tobytes()
    for i in range(0, len(want), step):
        if want[i] is not None:
            body = ob[int(off[i]):int(off[i + 1])].partition(b"\r\n\r\n")[2]
            assert body == want[i].encode(), (i, body[:200], want[i][:200])


# ---------------------------------------------------------------------------------------------------------------
# CPU: the references do not depend on the layout
# ---------------------------------------------------------------------------------------------------------------
def _cpu_input(name, n=300):
    batch, _ = TABLES[name][1](n)
    return zero_length(batch, 11)


@pytest.mark.parametrize("name", list(TABLES))
def test_references_ignore_layout(name):
    """oracle, emu.serve, emu.serve_slots and emu.route give every request the same bytes and meta whatever the layout"""
    spec, table, ot = _table(name)
    image = table.serialize()
    slot = TABLES[name][2]
    rnd = random.Random(7)
    base = _cpu_input(name)
    want = oracle(ot, table, base)
    e_cap = bound_total(table, base) + 64
    e_want = E.serve(image, base, DATE, out_cap=e_cap)
    _same((e_want[0][:int(e_want[1][-1])], e_want[1], e_want[2]), want, "emu packed")
    s_out, s_len, s_meta = E.serve_slots(image, base, DATE, slot)
    r_meta, r_vars = E.route(image, base)
    o_meta, o_vars = O.route(ot, base)
    assert np.array_equal(r_meta, o_meta) and np.array_equal(r_vars, o_vars)
    layouts = [relayout(base, m, rnd) for m in MODES] + [relayout(tile_of_copies(base, 1), "shared", rnd)]
    span = next(s for s in (4096, 8192, 16384, 32768) if tile_span_layout(base, s) is not None)
    layouts += [tile_span_layout(base, span), tile_span_layout(base, span + 16)]
    for k, b in enumerate(layouts):
        what = f"layout {k}"
        ref = want if k != len(MODES) else oracle(ot, table, tile_of_copies(base, 1))
        got = oracle(ot, table, b)
        _same(got, ref, "oracle " + what)
        o2, f2, m2 = E.serve(image, b, DATE, out_cap=e_cap)
        _same((o2[:int(f2[-1])], f2, m2), ref, "emu " + what)
        if k == len(MODES):
            continue
        so, sl, sm = E.serve_slots(image, b, DATE, slot)
        assert np.array_equal(sl, s_len) and np.array_equal(sm, s_meta), what
        assert np.array_equal(so, s_out), what
        check_slots(so, sl, sm, want, slot)
        rm, rv = E.route(image, b)
        om, ov = O.route(ot, b)
        assert np.array_equal(rm, r_meta) and np.array_equal(rv, r_vars) and np.array_equal(om, o_meta) and np.array_equal(ov, o_vars), what


def test_relayout_keeps_the_requests():
    base = _cpu_input("config4", 400)
    recs = _records(base)
    rnd = random.Random(1)
    for m in MODES:
        b = relayout(base, m, rnd)
        assert np.array_equal(b.trace_ids, base.trace_ids)
        for f in ("path_len", "query_len", "data_len", "method", "flags", "aux"):
            assert np.array_equal(b.desc[f], base.desc[f]), (m, f)
        assert _records(b) == recs, m
        assert (b.desc["arena_off"] % 4 == 0).all(), m
        ends = [int(o) + len(r) for o, r in zip(b.desc["arena_off"], recs)]
        assert max(ends) <= b.arena.size, m
    offs = relayout(base, "misaligned", rnd).desc["arena_off"]
    assert set((offs % 16).tolist()) == {4, 8, 12}
    b = relayout(base, "tight", rnd)
    assert max(int(o) + len(r) for o, r in zip(b.desc["arena_off"], recs)) == b.arena.size
    assert len(set(relayout(base, "empty", rnd).desc["arena_off"][base.desc["path_len"] == 0].tolist())) == 1
    sh = relayout(tile_of_copies(base, 1), "shared", rnd).desc["arena_off"]
    assert len(set(sh[T:2 * T].tolist())) == 1
    for span in (2048, 8192, 8208):
        b = tile_span_layout(base, span)
        if b is None:
            continue
        ends = np.array([int(o) + len(r) for o, r in zip(b.desc["arena_off"], recs)])
        for t0 in range(0, base.n, T):
            lo, hi = int(b.desc["arena_off"][t0:t0 + T].min()) & ~15, (int(ends[t0:t0 + T].max()) + 15) & ~15
            assert hi - lo == span, (span, t0)


def test_log_references_ignore_layout():
    lb = synth.reqlog_batch(700, hostile_every=5, rpc_every=7)
    o1, f1 = O.request_log(lb)
    for b in (_log_relayout(lb, "shuffled", random.Random(2)), _log_relayout(lb, "shared", random.Random(2)),
              _log_span(lb, 24576 - 16), _log_span(lb, 24576), _log_span(lb, 24576 + 16)):
        o2, f2 = O.request_log(b)
        o3, f3 = E.request_log(b)
        assert np.array_equal(f1, f2) and np.array_equal(f1, f3)
        assert o1[:f1[-1]].tobytes() == o2[:f2[-1]].tobytes() == o3[:f3[-1]].tobytes()


# ---- request-log layouts ----
def _log_recs(lb):
    d = lb.desc
    ln = (d["method_len"].astype(np.int64) + d["ua_len"] + d["xff_len"] + d["remote_len"] + d["uri_len"]).tolist()
    return [lb.arena[o:o + k].tobytes() for o, k in zip(d["arena_off"].tolist(), ln)]


def _log_build(lb, recs, offs, size):
    arena = np.zeros(size, dtype=np.uint8)
    for r, o in zip(recs, offs):
        arena[o:o + len(r)] = np.frombuffer(r, dtype=np.uint8)
    desc = lb.desc.copy()
    desc["arena_off"] = np.asarray(offs, dtype=np.uint32)
    return S.LogBatch(desc, lb.trace_ids.copy(), arena)


def _log_relayout(lb, mode, rnd):
    """records shuffled, or identical records at one copy (with a random permutation)"""
    recs = _log_recs(lb)
    order = list(range(len(recs)))
    rnd.shuffle(order)
    offs, seen, cur = [0] * len(recs), {}, 0
    for i in order:
        if mode == "shared" and recs[i] in seen:
            offs[i] = seen[recs[i]]
            continue
        offs[i] = seen.setdefault(recs[i], cur)
        cur += len(recs[i])
    return _log_build(lb, recs, offs, cur)


def _log_span(lb, span):
    """every tile of T records staged as exactly `span` bytes: [lo & ~15, (max end + 4 + 15) & ~15)"""
    recs = _log_recs(lb)
    offs, cur = [0] * len(recs), 0
    for t0 in range(0, len(recs), T):
        idx = list(range(t0, min(len(recs), t0 + T)))
        lo = cur = (cur + 15) & ~15
        for i in idx[:-1]:
            offs[i] = cur
            cur += len(recs[i])
        o = lo + span - 4 - len(recs[idx[-1]])
        assert o >= cur, "records too long for the span"
        offs[idx[-1]] = o
        cur = lo + span - 4
    return _log_build(lb, recs, offs, cur)


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "these tests need a GPU"
    return torch


def _engine(name, tile=None):
    from gofr_b200.engine import Engine
    eng = Engine(_table(name)[1], 0)
    if tile:
        eng.set_tile(tile)
    return eng


def _upload(eng, batch):
    """the batch on the device with exactly the ABI's 16 bytes of slack behind the arena"""
    import torch
    from gofr_b200.engine import DeviceBatch
    db = eng.upload(batch)
    arena = torch.from_numpy(np.concatenate([batch.arena, np.zeros(16, dtype=np.uint8)])).cuda()
    return DeviceBatch(db.desc, db.trace_ids, arena, batch.n, 0)


def gpu_packed(eng, table, batch):
    """gofr_serve_device with a 0xEE canary behind the capacity summed from the bounds: nothing may be written past out_off[n]"""
    import torch
    cap = bound_total(table, batch) + 64
    resp = eng.alloc_responses(batch.n, cap)
    resp.out.fill_(0xEE)
    eng.serve_device(_upload(eng, batch), DATE, resp)
    torch.cuda.synchronize()
    assert not eng.overflowed(), "the launch overflowed"
    off = resp.out_off.cpu().numpy().view(np.uint32)
    meta = resp.meta[:batch.n].cpu().numpy().view(np.uint32)
    out = resp.out.cpu().numpy()
    total = int(off[batch.n])
    assert (out[total:] == 0xEE).all(), "bytes written past out_off[n]"
    return out[:total], off, meta


def gpu_slots(eng, batch, slot, want, force=0):
    """gofr_serve_device_slots (force: 4 or 5 CTAs per SM, where the table allows) into a slot buffer filled with 0xEE"""
    import torch
    if force:
        eng.slot_ctas(force)
    n = batch.n
    canary = torch.full((max(n, 1) * slot,), 0xEE, dtype=torch.uint8, device="cuda")
    so, sl, sm = eng.serve_device_slots(_upload(eng, batch), DATE, slot, out=canary)
    torch.cuda.synchronize()
    out = so.cpu().numpy()[:n * slot].reshape(n, slot)
    check_slots(out, sl.cpu().numpy().view(np.uint32), sm.cpu().numpy().view(np.uint32), want, slot)


def check_slots(out, ln, meta, want, slot):
    """slot i holds response i of the packed result `want`, zero padded to 16 bytes, and the 0xEE it was filled with
    behind that; a response longer than the slot leaves the slot untouched"""
    o1, f1, m1 = want
    n = len(m1)
    assert np.array_equal(meta, m1), "slots: status / route column differs"
    assert np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32)), "slots: lengths differ"
    # every slot of a batch up to 16 Ki requests; of a larger one the first and last 2 Ki and every 13th in between
    rows = np.arange(n) if n <= 16384 else np.unique(np.concatenate([np.arange(2048), np.arange(2048, n, 13), np.arange(n - 2048, n)]))
    col = np.arange(slot)
    starts = f1[:-1].astype(np.int64)
    for b0 in range(0, len(rows), 4096):  # the expected slots, gathered from the packed bytes in blocks
        r = rows[b0:b0 + 4096]
        L = ln[r].astype(np.int64)
        src = np.minimum(starts[r, None] + col, max(len(o1) - 1, 0))
        body = col < L[:, None]
        pad = (col < ((L + 15) & ~15)[:, None]) & ~body
        exp = np.where(body, o1[src] if len(o1) else 0, np.where(pad, 0, 0xEE)).astype(np.uint8)
        exp[L > slot] = 0xEE
        got = out[r]
        if not np.array_equal(got, exp):
            k = int(np.flatnonzero((got != exp).any(axis=1))[0])
            raise AssertionError(f"slots: request {int(r[k])} (length {int(L[k])}) differs")


def gpu_host(eng, table, batch, pinned, chunk):
    from gofr_b200.engine import pin_batch, pinned_array
    eng.set_chunk(chunk)
    cap = bound_total(table, batch) + 64
    n = batch.n
    if pinned:
        batch = pin_batch(batch)
        out, off, meta = pinned_array(cap), pinned_array(4 * (n + 1), np.uint32), pinned_array(4 * max(n, 1), np.uint32)[:n]
    else:
        out, off, meta = np.zeros(cap, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.uint32)
    total = eng.serve_host(batch, DATE, out, off, meta)
    eng.set_chunk(65536)
    return out[:total].copy(), off.copy(), meta.copy()


_grid = {}


def _sizes():
    if "g" not in _grid:
        from gofr_b200.engine import Engine
        e = Engine(Table(synth.config2_spec()), 0)
        _grid["g"] = e.geometry()["grid"]
        e.close()
    g = _grid["g"]
    return [1, 31, 32, 127, 128, 129, g * T - 1, g * T, g * T + 1, 3 * g * T + 77]


def _modes_for(n, g):
    if n <= 129:
        return MODES
    if n <= g * T + 1:
        return ["reversed", "misaligned", "shared"] if n == g * T else ["shuffled", "gaps", "tight"]
    return ["shuffled"]


_base_cache = {}


def _base(name, n):
    """the geometry input: the table's stream, every 11th request zero-length; its oracle result; the model's bodies"""
    key = (name, n)
    if key not in _base_cache:
        if any(k[0] != name for k in _base_cache):
            _base_cache.clear()
        batch, want_bodies = TABLES[name][1](n)
        if n <= 4096:
            batch = zero_length(batch, 11)
            want_bodies = None if want_bodies is None else [None if i % 11 == 10 else w for i, w in enumerate(want_bodies)]
        spec, table, ot = _table(name)
        _base_cache[key] = (batch, oracle(ot, table, batch), want_bodies)
    return _base_cache[key]


@pytest.mark.gpu
@pytest.mark.parametrize("tile", [0, 16, 256])
@pytest.mark.parametrize("name", list(TABLES))
def test_gpu_serve_geometry(torch_cuda, name, tile):
    """every batch size from 1 to three tiles per CTA plus a partial tile, packed and slot layouts, for the table's own tile
    budget and for 16 and 256 staged bytes per request; each size in the packed layout and in several others"""
    spec, table, ot = _table(name)
    slot = TABLES[name][2]
    eng = _engine(name, tile)
    g = eng.geometry()["grid"]
    rnd = random.Random(tile * 7 + len(name))
    for k, n in enumerate(_sizes()):
        batch, want, bodies = _base(name, n)
        packed = gpu_packed(eng, table, batch)
        _same(packed, want, f"n={n} packed")
        if bodies is not None:
            _bodies_match_model(packed[0], packed[1], bodies, step=max(1, n // 3000))
        gpu_slots(eng, batch, slot, want, force=4 + k % 2)
        for mode in _modes_for(n, g):
            b = relayout(batch, mode, rnd)
            got = gpu_packed(eng, table, b)
            _same(got, packed, f"n={n} {mode} vs the packed GPU run")
            _same(got, oracle(ot, table, b) if n <= 4096 else want, f"n={n} {mode} vs the oracle")
            gpu_slots(eng, b, slot, want, force=4 + (k + 1) % 2)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["config4", "config2", "values"])
def test_gpu_tile_spans_at_the_staging_capacity(torch_cuda, name):
    """tiles whose staged span is exactly in_cap (staged, the last byte on a 16-byte boundary where the lengths allow) and
    in_cap + 16 (one step over: served from HBM), and a tile of 128 requests sharing one copy of their bytes"""
    spec, table, ot = _table(name)
    slot = TABLES[name][2]
    done = 0
    for tile in (16, 64, 256):
        in_cap = T * tile
        eng = _engine(name, tile)
        for n in (T - 1, T, 3 * T + 5, 1000):
            batch, want, _ = _base(name, n)
            for span in (in_cap, in_cap + 16):
                b = tile_span_layout(batch, span)
                if b is None:
                    continue
                done += 1
                got = gpu_packed(eng, table, b)
                _same(got, want, f"tile={tile} n={n} span={span}")
                gpu_slots(eng, b, slot, want, force=4 + done % 2)
        b = tile_of_copies(batch, 1)
        w = oracle(ot, table, b)
        _same(gpu_packed(eng, table, relayout(b, "shared", random.Random(0))), w, "one tile at one copy")
        eng.close()
    assert done >= 4


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False])
@pytest.mark.parametrize("name", ["config4", "values"])
def test_gpu_host_chunks_and_layouts(torch_cuda, name, pinned):
    """gofr_batch_submit with chunks of 1, 127, 128, 129 and 1000 requests over the packed, shuffled and shared layouts, and
    gofr_batch_submit_slots on the same engine"""
    spec, table, ot = _table(name)
    eng = _engine(name)
    batch, want, _ = _base(name, 1500)
    rnd = random.Random(5)
    for chunk in (1, 127, 128, 129, 1000):
        for mode in (None, "shuffled", "shared"):
            b = batch if mode is None else relayout(batch, mode, rnd)
            _same(gpu_host(eng, table, b, pinned, chunk), want, f"chunk={chunk} {mode}")
    slot = TABLES[name][2]
    n = batch.n
    out, ln, meta = np.full(n * slot, 0xEE, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    eng.set_chunk(129)
    eng.serve_host_slots(relayout(batch, "shuffled", rnd), DATE, slot, out, ln, meta)
    o1, f1, m1 = want
    assert np.array_equal(meta, m1) and np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32))
    out = out.reshape(n, slot)
    for i in range(n):
        if ln[i] <= slot:
            assert out[i, :ln[i]].tobytes() == o1[int(f1[i]):int(f1[i + 1])].tobytes(), i
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False])
def test_gpu_host_chunk_of_requests_sharing_one_row(torch_cuda, pinned):
    """Every request of a chunk points at one cached 2 KiB row.  The caller's buffer is sized from the response bounds; the
    chunk's device buffer must be too — sized from the arena span (2 KiB for the whole chunk) it could not hold the
    chunk's responses and the call reported GOFR_ERR_CAPACITY."""
    spec, table, ot = _table("config2")
    row = synth.C2_SCHEMA.encode_row([7, b"n" * 1024, b"e<" * 500, 1, 9])
    assert len(row) >= 2048
    base = S.RequestBatch.pack([S.Req(S.M_GET, b"/api/v1/r%02d" % (i % 16), b"", row) for i in range(3000)])
    b = relayout(base, "shared", random.Random(0))
    assert len(set(b.desc["arena_off"].tolist())) == 16
    want = oracle(ot, table, base)
    assert ((want[2] & 0xFFFF) == 200).all() and int(want[1][-1]) > 3000 * 2048
    eng = _engine("config2")
    for chunk in (65536, 1000):
        _same(gpu_host(eng, table, b, pinned, chunk), want, f"chunk={chunk}")
    eng.close()


@pytest.mark.gpu
def test_gpu_route_and_bind_layouts(torch_cuda):
    """gofr_route_device / gofr_batch_route on config4 and gofr_bind_device on config3, in every layout"""
    import torch
    spec, table, ot = _table("config4")
    eng = _engine("config4")
    rnd = random.Random(9)
    for n in (129, 5000):
        batch = zero_length(synth.config4_batch(n), 11)
        m1, v1 = O.route(ot, batch)
        for mode in [None] + MODES:
            b = batch if mode is None else relayout(batch, mode, rnd)
            meta, vars_ = eng.route_device(_upload(eng, b))
            assert np.array_equal(meta.cpu().numpy().view(np.uint32), m1) and np.array_equal(vars_.cpu().numpy().view(np.uint32), v1), mode
            eng.set_chunk(1000)
            m2, v2 = eng.route_host(b)
            assert np.array_equal(m2, m1) and np.array_equal(v2, v1), mode
    eng.close()
    spec, table, ot = _table("config3")
    eng = _engine("config3")
    batch = synth.config3_batch(3000, variant_every=7)
    sid = spec.schemas[0].id
    r0, l0, s0 = eng.bind_device(_upload(eng, batch), sid, 1024)
    torch.cuda.synchronize()
    r0, l0, s0 = r0.cpu().numpy(), l0.cpu().numpy(), s0.cpu().numpy()
    er, el, es = E.bind_rows(table.serialize(), 0, batch, 1024)
    assert np.array_equal(l0.view(np.uint32), el) and np.array_equal(s0.view(np.uint32), es)
    r2 = r0.reshape(batch.n, 1024)
    for i in range(batch.n):
        L = int(el[i])
        if L <= 1024:
            assert r2[i, :L].tobytes() == er[i, :L].tobytes(), i
    for mode in MODES:
        b = relayout(batch, mode, rnd)
        r, ln, st = eng.bind_device(_upload(eng, b), sid, 1024)
        torch.cuda.synchronize()
        assert np.array_equal(ln.cpu().numpy(), l0) and np.array_equal(st.cpu().numpy(), s0), mode
        assert np.array_equal(r.cpu().numpy(), r0), mode
    eng.close()


@pytest.mark.gpu
def test_gpu_interleaved_launches(torch_cuda):
    """one engine, calls of different sizes and entry points interleaved: the look-back state, the scratch and the chunk
    slots are reused across them"""
    spec, table, ot = _table("config4")
    eng = _engine("config4")
    g = eng.geometry()["grid"]
    rnd = random.Random(11)
    plan = [(g * T + 1, "packed"), (31, "slots"), (5000, "host"), (1, "packed"), (2 * g * T + 3, "packed"), (129, "host"),
            (g * T - 1, "slots"), (127, "packed"), (5000, "host_pageable"), (3000, "packed")]
    for n, what in plan:
        batch = relayout(synth.config4_batch(n, start=n), "shuffled", rnd)
        want = oracle(ot, table, batch)
        if what == "packed":
            _same(gpu_packed(eng, table, batch), want, f"{n} {what}")
        elif what == "slots":
            gpu_slots(eng, batch, 352, want)
        else:
            _same(gpu_host(eng, table, batch, what == "host", 700), want, f"{n} {what}")
    eng.close()


@pytest.mark.gpu
def test_gpu_checker_sees_a_broken_lookback(torch_cuda, monkeypatch):
    """Self-test of the packed checks: with the look-back off (GOFR_DEBUG_NO_LOOKBACK, a diagnostic that chains tiles as
    if every response had the same size) the config-4 offsets are wrong, and gpu_packed / _same say so."""
    monkeypatch.setenv("GOFR_DEBUG_NO_LOOKBACK", "1")
    spec, table, ot = _table("config4")
    eng = _engine("config4")
    batch, want, _ = _base("config4", 3 * T + 5)
    with pytest.raises(AssertionError, match="offsets differ|overflowed|written past"):
        _same(gpu_packed(eng, table, batch), want, "no look-back")
    eng.overflowed()
    eng.close()


# ---- randomized campaigns at two tiles per CTA and more ----
def _campaign_n():
    return 2 * _sizes()[7] + 77           # two tiles per CTA of the packed grid, and a partial tile


def _campaign_check(spec, batch, bodies=None, slot=2048, step=1):
    table, ot = Table(spec), O.OracleTable(spec)
    from gofr_b200.engine import Engine
    eng = Engine(table, 0)
    want = oracle(ot, table, batch)
    got = gpu_packed(eng, table, batch)
    _same(got, want, "packed")
    gpu_slots(eng, batch, slot, want)
    if bodies is not None:
        ob = got[0].tobytes()
        for i in range(0, len(bodies), step):
            r = ob[int(got[1][i]):int(got[1][i + 1])]
            body = r if spec.frame_mode == S.FRAME_BODY else r.partition(b"\r\n\r\n")[2]
            assert body.decode("utf-8") == (bodies[i] or ""), i
    eng.close()
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 7, 13, 20])
def test_gpu_random_schemas(torch_cuda, seed):
    """test_values' random schema campaign on the VALUES kernel instances: 400 random rows repeated to two tiles per CTA"""
    spec, routed, b, want = TV._random_schema_case(seed)
    n = _campaign_n()
    _campaign_check(spec, replicate(b, n), [want[i % b.n] for i in range(n)], step=97)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 12])
def test_gpu_mutated_rows(torch_cuda, seed):
    """rows with flipped bytes, overwritten counts, cut tails and appended garbage: 500 where the oracle answers 500"""
    rnd = random.Random(4000 + seed)
    structs, bare = TV._rand_schemas(rnd, rnd.randint(2, 5), late=seed >= 10)
    routed = structs + bare
    kind = S.H_RESULT if seed % 2 else S.H_ROW
    spec = S.TableSpec(schemas=routed, routes=[S.Route(S.M_GET, "/t/%d" % sc.id, kind, schema_id=sc.id) for sc in routed])
    b = S.RequestBatch.pack(TV._mutated_rows(rnd, spec, routed, kind, 600), seed=seed)
    o1, f1, m1 = _campaign_check(spec, replicate(b, _campaign_n()))
    assert ((m1 & 0xFFFF) == 500).any() and ((m1 & 0xFFFF) == 200).any()


@pytest.mark.gpu
def test_gpu_pointer_chain(torch_cuda):
    """an 8-level pointer chain, cut at every depth, through the VALUES instances"""
    spec = _chain_spec()
    batch, bodies = _chain_batch(_campaign_n())
    _campaign_check(spec, batch, bodies, step=89)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [3, 4, 5])
def test_gpu_random_route_tables(torch_cuda, seed):
    """random route tables (test_route's vocabulary) through gofr_route_device, gofr_batch_route and the serve kernel's
    route column"""
    from gofr_b200.engine import Engine
    rnd = random.Random(seed)
    routes = [S.Route(rnd.choice(TR.ROUTE_METHODS), TR._rename_vars("/" + "/".join(rnd.choice(TR.SEGMENTS + TR.VARIABLES)
                                                                                 for _ in range(rnd.randrange(5))), k), S.H_HOST)
              for k in range(rnd.randint(1, 10))]
    spec = S.TableSpec(default_routes=bool(seed % 2), routes=routes)
    reqs = [S.Req(rnd.choice(TR.REQ_METHODS), ("/" + "/".join(rnd.choice(TR.PATH_SEGMENTS) for _ in range(rnd.randrange(5)))).encode())
            for _ in range(3000)]
    batch = relayout(replicate(S.RequestBatch.pack(reqs, seed=seed), _campaign_n()), "shuffled", rnd)
    table, ot = Table(spec), O.OracleTable(spec)
    m1, v1 = O.route(ot, batch)
    eng = Engine(table, 0)
    meta, vars_ = eng.route_device(_upload(eng, batch))
    assert np.array_equal(meta.cpu().numpy().view(np.uint32), m1) and np.array_equal(vars_.cpu().numpy().view(np.uint32), v1)
    m2, v2 = eng.route_host(batch)
    assert np.array_equal(m2, m1) and np.array_equal(v2, v1)
    _, _, m3 = gpu_packed(eng, table, batch)
    assert np.array_equal(m3 >> 16, m1 >> 16)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0x1234, 99, 2 ** 31 - 5])
def test_gpu_mixed_stream_windows(torch_cuda, seed):
    """windows of the seeded mixed-traffic stream (test_slots' property) at two tiles per CTA, short slots included"""
    spec, table, ot = _table("config4")
    from gofr_b200.engine import Engine
    eng = Engine(table, 0)
    batch = synth.config4_batch(_campaign_n(), start=seed % 100000, seed=seed)
    want = oracle(ot, table, batch)
    _same(gpu_packed(eng, table, batch), want, "packed")
    for slot in (176, 352, 1024):
        gpu_slots(eng, batch, slot, want)
    eng.close()


# ---- the other TMA-staged kernels at their staging limits ----
@pytest.mark.gpu
def test_gpu_request_log_layouts_and_limit(torch_cuda):
    """kLogStage (24 KiB): permuted and shared record layouts, and tiles staged as 24576 - 16, 24576 and 24576 + 16 bytes"""
    from gofr_b200.engine import Engine
    eng = Engine(Table(synth.config1_spec()), 0)
    lb = synth.reqlog_batch(3 * T + 9, hostile_every=5, rpc_every=7)
    o1, f1 = O.request_log(lb)
    for b in (_log_relayout(lb, "shuffled", random.Random(2)), _log_relayout(lb, "shared", random.Random(2)),
              _log_span(lb, 24576 - 16), _log_span(lb, 24576), _log_span(lb, 24576 + 16)):
        d_out, d_off = eng.request_log_device(b)
        off = d_off.cpu().numpy().view(np.uint32)
        assert np.array_equal(off, f1)
        assert d_out[:int(off[-1])].cpu().numpy().tobytes() == o1[:f1[-1]].tobytes()
        assert not eng.overflowed()
    eng.close()


def _hello_frames(sizes):
    """Hello frames of the given total sizes (5-byte prefix + field 1 with a name filling the rest)"""
    msgs = []
    for k, s in enumerate(sizes):
        m = s - 5
        name_len = m - 2 if m - 2 < 128 else m - 3
        name = bytes(b"abcdefghijklmnopqrstuvwxyz"[(k + j) % 26] for j in range(name_len))
        lenb = bytes([name_len]) if name_len < 128 else bytes([0x80 | (name_len & 0x7F), name_len >> 7])
        msgs.append(b"\x0a" + lenb + name)
    from tests.test_grpc import _frames
    frames, off = _frames(msgs)
    assert list(np.diff(off)) == list(sizes)
    return frames, off


@pytest.mark.gpu
def test_gpu_frame_codecs_at_the_staging_limit(torch_cuda):
    """kGrpcStage (8 KiB): tiles of 128 frames spanning exactly 8192 bytes (staged) and 8208 (served from HBM)"""
    from tests.test_grpc import _gpu_hello
    sizes = [64] * T + [64] * 127 + [80] + [64] * 127 + [64 + 16] + [40] * 30
    frames, off = _hello_frames(sizes)
    assert off[T] - off[0] == 8192 and off[2 * T] - off[T] == 8208 and off[3 * T] - off[2 * T] == 8208
    o1, f1, m1 = O.grpc_hello(frames, off)
    o2, f2, m2 = _gpu_hello(frames, off)
    assert np.array_equal(m1, m2) and np.array_equal(f1, f2) and o1[:int(f1[-1])].tobytes() == o2[:int(f1[-1])].tobytes()
    from gofr_b200.engine import Engine
    eng = Engine(Table(synth.config1_spec()), 0)
    fields = [S.ProtoField(1, S.PB_STRING)]
    r1, ro1, rm1 = O.proto_decode(fields, frames, off)
    r2, ro2, rm2 = eng.proto_decode_device(fields, frames, off)
    ro2 = ro2.cpu().numpy().view(np.uint32)
    assert np.array_equal(rm2.cpu().numpy().view(np.uint32), rm1) and np.array_equal(ro2, ro1)
    assert r2[:int(ro1[-1])].cpu().numpy().tobytes() == r1[:int(ro1[-1])].tobytes()
    eng.close()


@pytest.mark.gpu
def test_gpu_http_parse_at_the_staging_limit(torch_cuda):
    """kHttpStage (26 KiB): tiles of 128 request heads spanning exactly 26624 bytes (staged) and 26640 (from HBM)"""
    from gofr_b200.engine import Engine

    def msg(k, size):
        head = b"GET /svc/%02d/ping?k=%d HTTP/1.1\r\nHost: h\r\nX-Pad: " % (k % 48, k)
        return head + b"p" * (size - len(head) - 4) + b"\r\n\r\n"
    sizes = [208] * T + [208] * 127 + [224] + [208] * 40
    msgs = [msg(k, s) for k, s in enumerate(sizes)]
    raw = np.frombuffer(b"".join(msgs), dtype=np.uint8).copy()
    off = np.zeros(len(msgs) + 1, dtype=np.uint32)
    np.cumsum([len(m) for m in msgs], out=off[1:])
    assert off[T] == 26624 and off[2 * T] - off[T] == 26640
    eng = Engine(Table(synth.config4_spec()), 0)
    d1, a1, s1, sp1 = O.http_parse(raw, off)
    desc, arena, status, spans = eng.http_parse_device(raw, off)
    assert np.array_equal(s1, status.cpu().numpy().view(np.uint32)) and (s1 == 0).all()
    assert np.array_equal(d1.view(np.uint8).reshape(-1), desc.cpu().numpy())
    assert np.array_equal(sp1, spans.cpu().numpy().view(np.uint64))
    assert np.array_equal(a1[:raw.size], arena.cpu().numpy()[:raw.size])
    eng.close()
