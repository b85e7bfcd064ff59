"""The slot-layout fast path of the wide instance (4 CTAs/SM, the one config 2 runs) stores each whole 32-byte sector of a
response with two 16-byte warp stores shared by a lane pair: lanes 2k and 2k+1 each write one half of the even lane's
sector, then one half of the odd lane's (the PairStores store policy in serve_device.cuh).  A lane whose partner has no sector
in a round, every store outside the fast path and the 5-CTA instance write their own.  Mixed traffic (config 4) runs here
on both instances: forced onto the wide one, its warps pair lanes of different programs, template-only programs next to
tail ops, and lanes whose requests were deferred to the general pass.
The CPU emulation runs one lane at a time and cannot see the pairing, so it is checked here, byte for byte against the
oracle, on an output buffer filled with a sentinel first:

  * every response that fits its slot is the oracle's, zero padded to the next multiple of 16, and the rest of the slot
    still holds the sentinel;
  * the slot of a response longer than the slot, and of a request left to the host, is untouched;
  * batches that end in partial warps and tiles, slots that start on and off sector boundaries, a slot too small for
    some responses, and mixed traffic (divergent shape classes, deferred requests and the general pass);
  * the packed layout of the same requests, which runs through the same Writer.
"""
import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200 import synth
from tests import oracle as O

DATE = S.http_date(1_700_000_000)
SENTINEL = 0xA5

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    """one engine per table, shared by the tests of this file"""
    from gofr_b200.engine import Engine
    from gofr_b200.table import Table
    made = {}

    def get(name, ctas=0):
        """ctas: force the slot-layout instance (4: wide, paired; 5), 0: the engine's choice"""
        if (name, ctas) not in made:
            spec = synth.config2_spec(S.FRAME_WIRE) if name == "config2" else synth.config4_spec()
            eng = Engine(Table(spec), 0)
            if ctas:
                assert eng.slot_ctas(ctas) == ctas
            made[(name, ctas)] = (spec, eng)
        return made[(name, ctas)]

    yield get
    for _, eng in made.values():
        eng.close()


def _batch(name, n, escape_every=0):
    return synth.config2_batch(n, escape_every=escape_every) if name == "config2" else synth.config4_batch(n)


def _check_slots(eng, spec, batch, slot):
    import torch
    n = batch.n
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    out = torch.full((n * slot,), SENTINEL, dtype=torch.uint8, device="cuda")
    out_len = torch.zeros(n, dtype=torch.int32, device="cuda")
    meta = torch.zeros(n, dtype=torch.int32, device="cuda")
    eng.serve_device_slots(eng.upload(batch), DATE, slot, out=out, out_len=out_len, meta=meta)
    torch.cuda.synchronize()
    got = out.cpu().numpy().reshape(n, slot)
    ln = out_len.cpu().numpy().view(np.uint32)
    assert np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32))
    assert np.array_equal(meta.cpu().numpy().view(np.uint32), m1)
    bad = []
    fitted = 0
    for i in range(n):
        L = int(ln[i])
        row = got[i]
        if 0 < L <= slot:
            fitted += 1
            p = min(slot, (L + 15) & ~15)
            ok = (row[:L].tobytes() == o1[int(f1[i]):int(f1[i]) + L].tobytes() and not row[L:p].any()
                  and bool((row[p:] == SENTINEL).all()))
        else:  # too long for the slot, or nothing to write: the slot is untouched
            ok = bool((row == SENTINEL).all())
        if not ok:
            bad.append(i)
    assert not bad, f"{len(bad)} of {n} slots differ from the oracle, first {bad[:8]}"
    return fitted, n - fitted


def _check_packed(eng, spec, batch):
    import torch
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    total = int(f1[batch.n])
    resp = eng.alloc_responses(batch.n, total + 1024)
    resp.out.fill_(SENTINEL)
    eng.serve_device(eng.upload(batch), DATE, resp)
    torch.cuda.synchronize()
    out, off, meta = resp.to_host()
    assert np.array_equal(off, f1) and np.array_equal(meta, m1)
    assert out[:total].tobytes() == o1[:total].tobytes()
    assert bool((resp.out[total:total + 1024].cpu().numpy() == SENTINEL).all())


@pytest.mark.parametrize("slot", [528, 544, 1024])
@pytest.mark.parametrize("n", [1, 2, 31, 33, 4097])
def test_config2_slots(engines, n, slot):
    spec, eng = engines("config2")
    assert eng.slot_ctas() == 4  # the paired instance
    fitted, _ = _check_slots(eng, spec, _batch("config2", n), slot)
    assert fitted == n


@pytest.mark.parametrize("n", [33, 4097])
def test_config2_escaped_general_pass(engines, n):
    # every 3rd body has a byte that needs escaping: the fast path leaves those requests to the general pass, whose stores
    # are not paired, while their warp neighbours are written by the fast path
    spec, eng = engines("config2")
    assert eng.slot_ctas() == 4
    fitted, _ = _check_slots(eng, spec, _batch("config2", n, escape_every=3), 528)
    assert fitted == n


@pytest.mark.parametrize("ctas", [0, 4])
@pytest.mark.parametrize("n", [33, 4097])
def test_config4_mixed_slots(engines, n, ctas):
    spec, eng = engines("config4", ctas)
    _check_slots(eng, spec, _batch("config4", n), 1024)


@pytest.mark.parametrize("ctas", [0, 4])
def test_config4_slot_too_small_for_some(engines, ctas):
    spec, eng = engines("config4", ctas)
    batch = _batch("config4", 4097)
    _, f1, _ = O.OracleTable(spec).serve(batch, DATE)
    slot = (int(np.median(np.diff(f1.astype(np.int64)))) + 15) & ~15
    fitted, skipped = _check_slots(eng, spec, batch, slot)
    assert fitted and skipped


@pytest.mark.parametrize("name", ["config2", "config4"])
@pytest.mark.parametrize("n", [1, 31, 33, 4097])
def test_packed_same_inputs(engines, name, n):
    spec, eng = engines(name)
    _check_packed(eng, spec, _batch(name, n))
