"""The wide slot instance (4 CTAs/SM, LineStores) stores the response templates of a warp's 32 lanes together: the warp
numbers the 16-byte template windows of its responses in request order and lane L stores windows L, L + 32, ... of that
sequence, straight from the literal pool, or from the owner's staging column for the windows the trace id touches
(serve_device.cuh LineStores::templates, stage_trace_id).  Only the tail after the template goes through the column.

Checked byte for byte against the oracle on an output buffer filled with a sentinel first: every response that fits is
the oracle's, zero padded to the next multiple of 16, and every byte past that padded end still holds the sentinel.
The cases:

  * batches that end in a partial warp (n not a multiple of 32);
  * slots of 528, 544 and 1024 bytes: with 528-byte slots each of the eight 16-byte leads within a 128-byte line occurs;
  * bodies that need escaping (escape_every): those lanes are left to the general pass and sit idle inside the warp;
  * a table whose warps mix programs: the table compiler gives every row program of a frame mode the same header, so
    templates of different lengths in one warp come from the template-only programs next to it (static strings of
    several lengths, a 500 error, the mux 404 for a path without a route); their trace ids start at byte offsets 2, 5
    and 9 of a 16-byte window, and the 404s are lanes with no tail.

The same cases run through the host emulation (tests/emu), which stores one lane at a time.
"""
import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O

DATE = S.http_date(1_700_000_000)
SENTINEL = 0xA5


def mixed_spec() -> S.TableSpec:
    """Row routes r00..r07 (config 2's program), template-only routes r08..r13, a POST-only r14 (405 for GET) and no
    route for r15 (404), over the paths config2_batch(n_routes=16) requests."""
    routes = [S.Route(S.M_GET, "/api/v1/r%02d" % k, S.H_ROW, schema_id=1) for k in range(8)]
    routes += [S.Route(S.M_GET, "/api/v1/r%02d" % (8 + j), S.H_STATIC_STRING, s0=b"x" * n) for j, n in enumerate((1, 7, 20, 45))]
    routes += [S.Route(S.M_GET, "/api/v1/r12", S.H_STATIC_ERROR, s0=b"backend unavailable"),
               S.Route(S.M_GET, "/api/v1/r13", S.H_NIL),
               S.Route(S.M_POST, "/api/v1/r14", S.H_ROW, schema_id=1)]
    return S.TableSpec(frame_mode=S.FRAME_WIRE, schemas=[synth.C2_SCHEMA], routes=routes)


CASES = {
    "config2": lambda n: (synth.config2_spec(S.FRAME_WIRE), synth.config2_batch(n)),
    "escaped": lambda n: (synth.config2_spec(S.FRAME_WIRE), synth.config2_batch(n, escape_every=3)),
    "mixed": lambda n: (mixed_spec(), synth.config2_batch(n, n_routes=16)),
    "mixed_escaped": lambda n: (mixed_spec(), synth.config2_batch(n, n_routes=16, escape_every=5)),
}
SLOTS = [528, 544, 1024]
SIZES = [1, 31, 33, 1000]


def _check(out, ln, meta, spec, batch, slot, sentinel=SENTINEL):
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    assert np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32))
    assert np.array_equal(meta, m1)
    bad = []
    for i in range(batch.n):
        L, row = int(ln[i]), out[i]
        if 0 < L <= slot:
            p = min(slot, (L + 15) & ~15)
            ok = (row[:L].tobytes() == o1[int(f1[i]):int(f1[i]) + L].tobytes() and not row[L:p].any()
                  and bool((row[p:] == sentinel).all()))
        else:
            ok = bool((row == sentinel).all())
        if not ok:
            bad.append(i)
    assert not bad, f"{len(bad)} of {batch.n} slots differ from the oracle, first {bad[:8]}"


def test_mixed_table_runs_the_wide_instance():
    # the template-only programs do not count against the one-shape rule: the engine picks the wide instance
    assert Table(mixed_spec()).slot_ctas() == 4


def test_mixed_table_has_the_template_variety():
    spec = mixed_spec()
    batch = synth.config2_batch(256, n_routes=16)
    o1, f1, _ = O.OracleTable(spec).serve(batch, DATE)
    lens, phases = set(), set()
    for i in range(batch.n):
        r = o1[int(f1[i]):int(f1[i + 1])].tobytes()
        lens.add(len(r))
        phases.add((r.index(b"X-Correlation-Id: ") + 18) & 15)
    assert len(lens) >= 6 and phases >= {2, 5, 9}, (lens, phases)


@pytest.mark.parametrize("slot", SLOTS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_emulation(case, slot):
    from tests.emu import emu
    try:
        emu.set_pair_stores(True)
        emu.set_stage_mode(1)
        for n in SIZES:
            spec, batch = CASES[case](n)
            out, ln, meta = emu.serve_slots(Table(spec).serialize(), batch, DATE, slot)
            _check(out, ln, meta, spec, batch, slot, sentinel=0xEE)  # the emulation's own fill byte
    finally:
        emu.set_pair_stores(False)
        emu.set_stage_mode(0)


@pytest.fixture(scope="module")
def engines():
    from gofr_b200.engine import Engine
    made = {}

    def get(case):
        key = case.replace("_escaped", "")
        if key not in made:
            spec = CASES[case](1)[0]
            eng = Engine(Table(spec), 0)
            assert eng.slot_ctas(4) == 4
            made[key] = eng
        return made[key]

    yield get
    for eng in made.values():
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("slot", SLOTS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_wide_instance(engines, case, slot):
    import torch
    eng = engines(case)
    for n in SIZES + [4097]:
        spec, batch = CASES[case](n)
        out = torch.full((n * slot,), SENTINEL, dtype=torch.uint8, device="cuda")
        out_len = torch.zeros(n, dtype=torch.int32, device="cuda")
        meta = torch.zeros(n, dtype=torch.int32, device="cuda")
        eng.serve_device_slots(eng.upload(batch), DATE, slot, out=out, out_len=out_len, meta=meta)
        torch.cuda.synchronize()
        _check(out.cpu().numpy().reshape(n, slot), out_len.cpu().numpy().view(np.uint32),
               meta.cpu().numpy().view(np.uint32), spec, batch, slot)
