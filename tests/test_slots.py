"""gofr_serve_device_slots: the same responses as the packed call, one 16-byte aligned slot per request."""
import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O

DATE = S.http_date(1_700_000_000)


def _check(eng, spec, batch, slot):
    import torch
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    n = batch.n
    canary = torch.full((n * slot,), 0xEE, dtype=torch.uint8, device="cuda")
    out, out_len, meta = eng.serve_device_slots(eng.upload(batch), DATE, slot, out=canary)
    out = out.cpu().numpy().reshape(n, slot)
    ln = out_len.cpu().numpy().view(np.uint32)
    assert np.array_equal(meta.cpu().numpy().view(np.uint32), m1)
    want_len = np.diff(f1.astype(np.int64)).astype(np.uint32)
    assert np.array_equal(ln, want_len)
    ob = o1.tobytes()
    for i in range(n):
        L = int(ln[i])
        if L > slot:                                    # too long for the slot: reported, nothing written
            assert (out[i] == 0xEE).all()
            continue
        assert out[i, :L].tobytes() == ob[int(f1[i]):int(f1[i]) + L], i
        pad = (-L) % 16
        assert (out[i, L:L + pad] == 0).all() and (out[i, L + pad:] == 0xEE).all(), i
    return ln


def _check_slots(out, ln, meta, spec, batch, slot, untouched=True):
    """untouched=False: the host path copies whole slots back, so bytes behind a response are unspecified there"""
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    assert np.array_equal(meta, m1)
    assert np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32))
    ob = o1.tobytes()
    for i in range(batch.n):
        L = int(ln[i])
        if L > slot:
            assert not untouched or (out[i] == 0xEE).all()
            continue
        assert out[i, :L].tobytes() == ob[int(f1[i]):int(f1[i]) + L], i
        pad = (-L) % 16
        assert (out[i, L:L + pad] == 0).all() and (not untouched or (out[i, L + pad:] == 0xEE).all()), i


@pytest.mark.parametrize("which,slot", [("config1", 320), ("config2", 528), ("config2", 544), ("config4", 352), ("config3", 1024)])
def test_emu_slots_match_oracle(which, slot):
    """the slot-layout emit path (emit_request<true>, Writer::finish_padded) on the CPU, with the fast path's sectors
    stored under both store policies (SoloStores as in serve_slots_kernel, PairStores as in the wide instance)"""
    from tests.emu import emu
    spec, batch = {"config1": (synth.config1_spec(), synth.config1_batch(200)),
                   "config2": (synth.config2_spec(), synth.config2_batch(300, escape_every=5)),
                   "config3": (synth.config3_spec(), synth.config3_batch(300)),
                   "config4": (synth.config4_spec(), synth.config4_batch(1500))}[which]
    image = Table(spec).serialize()
    try:
        for pair in (False, True):
            emu.set_pair_stores(pair)
            out, ln, meta = emu.serve_slots(image, batch, DATE, slot)
            _check_slots(out, ln, meta, spec, batch, slot)
    finally:
        emu.set_pair_stores(False)


@pytest.mark.parametrize("mode", [S.FRAME_WIRE, S.FRAME_INTENDED, S.FRAME_BODY])
@pytest.mark.parametrize("flush_mode", [0, 1, 2])
def test_emu_fast_path(mode, flush_mode):
    """emit_fast (seal-time response templates + tail ops) against the oracle: every framing mode, the flush decisions
    other lanes impose on the GPU replayed (emu.set_flush_mode), both store policies (SoloStores; PairStores, whose
    lockstep paths the wide instance runs), and a check that the fast path really ran"""
    from tests.emu import emu
    emu.set_flush_mode(flush_mode)
    emu.set_stage_mode(1)
    try:
        for spec, batch, slot, min_fast in (
                (synth.config1_spec(mode), synth.config1_batch(300), 320, 0.9),          # template-only programs
                (synth.config2_spec(mode), synth.config2_batch(600), 528, 0.99),         # template + struct tail
                (synth.config2_spec(mode), synth.config2_batch(600, escape_every=4), 640, 0.7),
                (synth.config4_spec(mode), synth.config4_batch(2500), 704, 0.5),
                (synth.config3_spec(mode), synth.config3_batch(400), 1024, 0.5)):
            image = Table(spec).serialize()
            for pair in (False, True):
                emu.set_pair_stores(pair)
                emu.fast_taken()
                out, ln, meta = emu.serve_slots(image, batch, DATE, slot)
                taken = emu.fast_taken()
                _check_slots(out, ln, meta, spec, batch, slot)
                assert taken >= min_fast * batch.n, (taken, batch.n, pair)
    finally:
        emu.set_flush_mode(0)
        emu.set_stage_mode(0)
        emu.set_pair_stores(False)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [S.FRAME_WIRE, S.FRAME_INTENDED, S.FRAME_BODY])
def test_config2_slots(torch_cuda, mode):
    from gofr_b200.engine import Engine
    spec = synth.config2_spec(mode)
    eng = Engine(Table(spec), 0)
    _check(eng, spec, synth.config2_batch(5000, escape_every=7), 640)
    eng.close()


@pytest.mark.gpu
def test_mixed_traffic_and_short_slots(torch_cuda):
    from gofr_b200.engine import Engine
    spec = synth.config4_spec()
    eng = Engine(Table(spec), 0)
    ln = _check(eng, spec, synth.config4_batch(20000), 352)   # about half of the responses are longer than 352 bytes
    assert (ln > 352).sum() > 1000 and (ln <= 352).sum() > 1000
    _check(eng, spec, synth.config4_batch(3000), 4096)
    eng.close()


def test_slot_residency_choice():
    """the 128-register (4-CTA) instance serves tables that answer with one fast-path program shape (config 2), the 5-CTA
    instance every other table"""
    assert Table(synth.config2_spec()).slot_ctas() == 4
    for spec in (synth.config4_spec(), synth.config3_spec(), synth.config1_spec()):
        assert Table(spec).slot_ctas() == 5


@pytest.mark.gpu
def test_both_slot_residencies(torch_cuda):
    """The engine runs the instance the table asks for (Table.slot_ctas); either instance forced on any table gives the
    same bytes."""
    from gofr_b200.engine import Engine
    for spec, batch, slot, auto in ((synth.config2_spec(), synth.config2_batch(40000, escape_every=11), 544, 4),
                                    (synth.config4_spec(), synth.config4_batch(20000), 1024, 5),
                                    (synth.config3_spec(), synth.config3_batch(4096), 1024, 5)):
        eng = Engine(Table(spec), 0)
        assert eng.slot_ctas() == auto
        for force in (4, 5):
            assert eng.slot_ctas(force) == force
            _check(eng, spec, batch, slot)
        eng.close()


@pytest.mark.gpu
def test_bind_and_results_in_slots(torch_cuda):
    from gofr_b200.engine import Engine
    spec = synth.config3_spec()
    eng = Engine(Table(spec), 0)
    _check(eng, spec, synth.config3_batch(4096), 1024)
    eng.close()
    from tests.test_result import _spec, _batch
    eng = Engine(Table(_spec()), 0)
    _check(eng, _spec(), _batch(), 768)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False])
def test_host_batch_slots(torch_cuda, pinned):
    """gofr_batch_submit_slots: host buffers in, slots out, chunked over the engine's three device slots"""
    from gofr_b200.engine import Engine, pin_batch, pinned_array
    spec = synth.config4_spec()
    batch = synth.config4_batch(5000)
    eng = Engine(Table(spec), 0)
    eng.set_chunk(700)                                  # 8 chunks, the last one short
    slot, n = 512, batch.n
    if pinned:
        hb = pin_batch(batch)
        out, ln, meta = pinned_array(n * slot), pinned_array(4 * n, np.uint32), pinned_array(4 * n, np.uint32)
    else:
        hb = batch
        out, ln, meta = np.zeros(n * slot, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    for rep in range(2):                                # buffers are reused across batches
        out[:] = 0xEE
        eng.serve_host_slots(hb, DATE, slot, out, ln, meta)
        _check_slots(out.reshape(n, slot), ln, meta, spec, batch, slot, untouched=False)
    # and it alternates with the packed host path on the same engine
    po, pf, pm = np.zeros(n * 700, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.uint32)
    got = eng.serve_host(batch, DATE, po, pf, pm)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    assert got == int(f1[-1]) and po[:got].tobytes() == o1[:got].tobytes()
    eng.serve_host_slots(hb, DATE, slot, out, ln, meta)
    _check_slots(out.reshape(n, slot), ln, meta, spec, batch, slot, untouched=False)
    eng.close()


@pytest.mark.gpu
def test_tiny_slots_write_nothing(torch_cuda):
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(Table(spec), 0)
    _check(eng, spec, synth.config1_batch(300), 16)     # every response is longer than 16 bytes: lengths only
    eng.close()


@pytest.mark.gpu
def test_slot_argument_checks(torch_cuda):
    from gofr_b200 import _abi
    from gofr_b200.engine import Engine
    spec = synth.config1_spec()
    eng = Engine(Table(spec), 0)
    b = eng.upload(synth.config1_batch(10))
    with pytest.raises(_abi.GofrError):
        eng.serve_device_slots(b, DATE, 500)            # not a multiple of 16
    eng.close()


# ---- the slot-layout emit path on arbitrary inputs (CPU): every response equals the oracle's, is zero padded to the next
#      16-byte boundary and leaves the rest of its slot alone; a response longer than its slot writes nothing ----
from hypothesis import given, settings, strategies as st  # noqa: E402

_bytes40 = st.binary(min_size=0, max_size=40)


@settings(max_examples=120, deadline=None)
@given(st.lists(st.tuples(_bytes40, _bytes40, st.integers(-2 ** 63, 2 ** 63 - 1), st.booleans()), min_size=1, max_size=10),
       st.sampled_from([16, 208, 528, 1024]), st.sampled_from([S.FRAME_WIRE, S.FRAME_INTENDED, S.FRAME_BODY]))
def test_emu_slots_random_rows_property(rows, slot, mode):
    from tests.emu import emu
    sc = synth.C2_SCHEMA
    spec = S.TableSpec(schemas=[sc], routes=[S.Route(S.M_GET, "/p", S.H_ROW, schema_id=1)], frame_mode=mode)
    batch = S.RequestBatch.pack([S.Req(S.M_GET, b"/p", b"", sc.encode_row([i, a, b, f, i % 2 ** 31])) for a, b, i, f in rows])
    out, ln, meta = emu.serve_slots(Table(spec).serialize(), batch, DATE, slot)
    _check_slots(out, ln, meta, spec, batch, slot)


@settings(max_examples=120, deadline=None)
@given(st.lists(st.tuples(st.sampled_from([S.M_GET, S.M_POST, S.M_HEAD, S.M_OPTIONS, S.M_PUT]),
                          st.text(alphabet="/.abx%? ", min_size=0, max_size=14).map(lambda s: ("/" + s).encode()),
                          st.binary(min_size=0, max_size=24)), min_size=1, max_size=12),
       st.sampled_from([16, 176, 352, 1024]))
def test_emu_slots_random_requests_property(reqs, slot):
    """mixed dispositions (200 / 301 / 404 / 405 / OPTIONS / HEAD) of the 64-route table through the slot layout"""
    from tests.emu import emu
    spec = synth.config4_spec()
    batch = S.RequestBatch.pack([S.Req(m, p.split(b"?", 1)[0], (p.split(b"?", 1) + [b""])[1] + q if b"?" in p else q) for m, p, q in reqs])
    out, ln, meta = emu.serve_slots(Table(spec).serialize(), batch, DATE, slot)
    _check_slots(out, ln, meta, spec, batch, slot)


@settings(max_examples=60, deadline=None)
@given(st.integers(0, 2 ** 31 - 1), st.integers(1, 150), st.sampled_from([16, 176, 352, 1024]))
def test_emu_slots_mixed_stream_property(seed, n, slot):
    """any window of the seeded mixed-traffic stream (matching routes with rows, path variables, redirects, OPTIONS, HEAD,
    panics) through the slot layout, short slots included"""
    from tests.emu import emu
    spec = synth.config4_spec()
    batch = synth.config4_batch(n, seed=seed)
    out, ln, meta = emu.serve_slots(Table(spec).serialize(), batch, DATE, slot)
    _check_slots(out, ln, meta, spec, batch, slot)
