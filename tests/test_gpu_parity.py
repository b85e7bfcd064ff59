"""GPU parity (run with -m gpu on an H100): the CUDA path, called through the C ABI, vs the CPU oracle."""
import os

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O

pytestmark = pytest.mark.gpu
DATE = S.http_date(1789974595)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "these tests need a GPU"
    return torch


def _engine(spec):
    from gofr_b200.engine import Engine
    return Engine(Table(spec), 0)


def _check(spec, batch, eng=None, host=False, chunk=None, pinned=True):
    import torch
    ot = O.OracleTable(spec)
    o1, f1, m1 = ot.serve(batch, DATE)
    total = int(f1[batch.n])
    eng = eng or _engine(spec)
    if host:
        if chunk:
            eng.set_chunk(chunk)
        if pinned:  # device-driven egress straight into pinned buffers
            from gofr_b200.engine import pin_batch, pinned_array
            batch = pin_batch(batch)
            out = pinned_array(total + 64)
            off = pinned_array(4 * (batch.n + 1), np.uint32)
            meta = pinned_array(4 * max(batch.n, 1), np.uint32)[:batch.n]
        else:       # pageable buffers: exact-size cudaMemcpy pipeline
            out = np.zeros(total + 64, dtype=np.uint8)
            off = np.zeros(batch.n + 1, dtype=np.uint32)
            meta = np.zeros(batch.n, dtype=np.uint32)
        nbytes = eng.serve_host(batch, DATE, out, off, meta)
        assert nbytes == total
    else:
        db = eng.upload(batch)
        resp = eng.alloc_responses(batch.n, total + 1024)
        eng.serve_device(db, DATE, resp)
        torch.cuda.synchronize()
        assert not eng.overflowed()
        out, off, meta = resp.to_host()
    assert int(off[batch.n]) == total
    assert np.array_equal(off, f1), "packed offsets differ"
    assert np.array_equal(meta, m1), "status/route column differs"
    if not np.array_equal(out[:total], o1[:total]):
        bad = int(np.nonzero(out[:total] != o1[:total])[0][0])
        i = int(np.searchsorted(f1, bad, side="right") - 1)
        raise AssertionError(f"first differing byte {bad} in request {i}: oracle={bytes(o1[f1[i]:f1[i+1]])!r} gpu={bytes(out[f1[i]:f1[i+1]])!r}")
    return eng


def test_native_library_is_the_one_running(torch_cuda):
    _abi.lib()
    assert os.path.exists(_abi.lib_path())
    with open("/proc/self/maps") as f:
        assert "libgofr_b200.so" in f.read()


@pytest.mark.parametrize("mode", [S.FRAME_WIRE, S.FRAME_INTENDED, S.FRAME_BODY])
def test_config1(torch_cuda, mode):
    _check(synth.config1_spec(mode), synth.config1_batch(1000))


@pytest.mark.parametrize("n", [1, 127, 128, 129, 5000, 70001])
def test_config2_sizes(torch_cuda, n):
    _check(synth.config2_spec(), synth.config2_batch(n))


@pytest.mark.parametrize("mode", [S.FRAME_INTENDED, S.FRAME_BODY])
def test_config2_modes(torch_cuda, mode):
    _check(synth.config2_spec(mode), synth.config2_batch(20000))


def test_config2_escape_heavy(torch_cuda):
    _check(synth.config2_spec(), synth.config2_batch(50000, escape_every=3))


def test_config4_mixed(torch_cuda):
    _check(synth.config4_spec(), synth.config4_batch(30000))


def test_empty_batch(torch_cuda):
    import torch
    eng = _engine(synth.config1_spec())
    resp = eng.alloc_responses(0, 64)
    b = S.RequestBatch.pack([])
    eng.serve_device(eng.upload(b), DATE, resp)
    torch.cuda.synchronize()
    assert int(resp.out_off.cpu()[0]) == 0


def test_oversized_tiles_fall_back_to_hbm(torch_cuda):
    """Rows longer than the shared-memory staging budget and a file blob larger than a tile: same bytes, no staging."""
    sc = synth.C2_SCHEMA
    spec = S.TableSpec(schemas=[sc], routes=[S.Route(S.M_GET, "/p", S.H_ROW, schema_id=1)],
                       favicon=b"\x89PNG\r\n\x1a\n" + bytes(range(256)) * 60)
    rng = np.random.default_rng(5)
    reqs = []
    for i in range(700):
        ln = int(rng.integers(0, 3000)) if i % 7 == 0 else int(rng.integers(0, 40))
        s = bytes(rng.integers(32, 127, size=ln, dtype=np.uint8))
        reqs.append(S.Req(S.M_GET, b"/p", b"", sc.encode_row([i, s, s[:5], i & 1, i])))
        if i % 50 == 0:
            reqs.append(S.Req(S.M_GET, b"/favicon.ico"))
    _check(spec, S.RequestBatch.pack(reqs))


def test_output_capacity_overflow_is_reported(torch_cuda):
    import torch
    spec = synth.config2_spec()
    eng = _engine(spec)
    b = synth.config2_batch(1000)
    resp = eng.alloc_responses(b.n, 1000)
    eng.serve_device(eng.upload(b), DATE, resp)
    torch.cuda.synchronize()
    assert eng.overflowed()


def test_repeated_launches_reuse_lookback_state(torch_cuda):
    spec = synth.config2_spec()
    eng = _engine(spec)
    for n in (3000, 100, 9000, 3000):
        _check(spec, synth.config2_batch(n, start=n), eng=eng)


@pytest.mark.parametrize("pinned", [True, False])
@pytest.mark.parametrize("chunk", [1000, 4096, 65536])
def test_host_path_chunked_pipeline(torch_cuda, chunk, pinned):
    _check(synth.config2_spec(), synth.config2_batch(20000), host=True, chunk=chunk, pinned=pinned)


def test_host_path_output_capacity(torch_cuda):
    """A caller buffer that is too small is reported as GOFR_ERR_CAPACITY, not overrun."""
    from gofr_b200 import _abi
    from gofr_b200.engine import Engine, pin_batch, pinned_array
    eng = Engine(Table(synth.config2_spec()), 0)
    eng.set_chunk(1000)
    b = pin_batch(synth.config2_batch(5000))
    out = pinned_array(2000 * synth.C2_WIRE_BYTES)
    off = pinned_array(4 * 5001, np.uint32)
    meta = pinned_array(4 * 5000, np.uint32)
    with pytest.raises(_abi.GofrError) as e:
        eng.serve_host(b, DATE, out, off, meta)
    assert e.value.code == 7


def test_host_path_mixed(torch_cuda):
    _check(synth.config4_spec(), synth.config4_batch(10000), host=True, chunk=3000)


def test_full_size_config2_is_byte_identical(torch_cuda):
    """BASELINE config 2 at full size (1 Mi requests): every response 521 bytes, packed, and memcmp-equal to the oracle."""
    import torch
    n = 1 << 20
    spec = synth.config2_spec()
    batch = synth.config2_batch(n)
    eng = _engine(spec)
    db = eng.upload(batch)
    resp = eng.alloc_responses(n, n * synth.C2_WIRE_BYTES + 4096)
    eng.serve_device(db, DATE, resp)
    torch.cuda.synchronize()
    out, off, meta = resp.to_host()
    assert int(off[n]) == n * synth.C2_WIRE_BYTES
    assert np.array_equal(off, np.arange(n + 1, dtype=np.uint64).astype(np.uint32) * np.uint32(synth.C2_WIRE_BYTES))
    assert (meta & 0xFFFF == 200).all()
    ot = O.OracleTable(spec)
    o1, f1, m1 = ot.serve(batch, DATE, out_cap=n * synth.C2_WIRE_BYTES + 4096, nthreads=1)
    assert np.array_equal(meta, m1)
    assert np.array_equal(out, o1[:int(f1[n])])


def test_shards_concatenate_to_the_unsharded_result(torch_cuda):
    """Multi-GPU partitioning rule on one GPU: serve 4 contiguous shards, concatenate, compare with the whole batch."""
    import torch
    spec = synth.config4_spec()
    batch = synth.config4_batch(8000)
    ot = O.OracleTable(spec)
    o1, f1, _ = ot.serve(batch, DATE)
    eng = _engine(spec)
    parts = []
    for k in range(4):
        sh = batch.slice(2000 * k, 2000 * (k + 1))
        db = eng.upload(sh)
        resp = eng.alloc_responses(sh.n, int(f1[-1]) + 1024)
        eng.serve_device(db, DATE, resp)
        torch.cuda.synchronize()
        out, off, _ = resp.to_host()
        parts.append(out[:int(off[sh.n])])
    assert np.array_equal(np.concatenate(parts), o1[:int(f1[-1])])


def test_lookback_epoch_wrap(torch_cuda, monkeypatch):
    """An engine created three look-back epochs before the 24-bit epoch wraps (GOFR_DEBUG_EPOCH_START): the wrap falls in
    the middle of a streamed host-path batch.  The packed serve, the host path, Hello, the flat proto encoder and the request
    log run across it, twice over, and each matches the oracle."""
    from tests.test_grpc import _gpu_hello
    from tests.test_proto import _bulk
    monkeypatch.setenv("GOFR_DEBUG_EPOCH_START", str((1 << 24) - 4))
    spec = synth.config2_spec()
    eng = _engine(spec)
    frames, foff = synth.config5_frames(3000)
    fields, msgs = _bulk(2000)
    rows, roff = S.pack_proto_rows(fields, msgs)
    lb = synth.reqlog_batch(3000, hostile_every=5, rpc_every=7)
    for _ in range(2):
        _check(spec, synth.config2_batch(3000), eng=eng)
        _check(spec, synth.config2_batch(5000, start=7), eng=eng, host=True, chunk=1000)
        o1, f1, m1 = O.grpc_hello(frames, foff)
        o2, f2, m2 = _gpu_hello(frames, foff, eng)
        assert np.array_equal(m1, m2) and np.array_equal(f1, f2) and np.array_equal(o1[:int(f1[-1])], o2[:int(f1[-1])])
        out, o, meta = O.proto_encode(fields, rows, roff)
        d_out, d_off, d_meta = eng.proto_encode_device(fields, rows, roff)
        assert np.array_equal(d_off.cpu().numpy().view(np.uint32), o)
        assert np.array_equal(d_meta.cpu().numpy().view(np.uint32), meta)
        assert d_out[:int(o[-1])].cpu().numpy().tobytes() == out[:int(o[-1])].tobytes()
        o1, f1 = O.request_log(lb)
        d_out, d_off = eng.request_log_device(lb)
        assert np.array_equal(d_off.cpu().numpy().view(np.uint32), f1)
        assert d_out[:int(f1[-1])].cpu().numpy().tobytes() == o1[:f1[-1]].tobytes()
        assert not eng.overflowed()
    eng.close()


def test_two_live_engines(torch_cuda):
    """Two engines alive at once on tables with hot parts of different size.  The one created first stages 256 request
    bytes per request, so its kernels need more dynamic shared memory than the 48 KB default and than the second engine's.
    Once the second exists it still serves a slot batch with each slot-layout instance and a packed batch (whose grid the
    two engines now share)."""
    from tests import test_slots
    big, small = synth.config4_spec(), synth.config2_spec()
    eng = _engine(big)
    eng.set_tile(256)
    other = _engine(small)
    assert eng.geometry()["smem_bytes"] > max(48 * 1024, other.geometry()["smem_bytes"])
    batch = synth.config4_batch(20000)
    for force in (4, 5):
        assert eng.slot_ctas(force) == force
        test_slots._check(eng, big, batch, 1024)
    _check(big, batch, eng=eng)
    _check(small, synth.config2_batch(5000), eng=other)
    other.close()
    eng.close()


def test_path_params(torch_cuda):
    spec = S.TableSpec(routes=[
        S.Route(S.M_GET, "/users/{id}", S.H_PATHPARAM_FORMAT, s0=b"id", s2=b"user ", s3=b"!"),
        S.Route(S.M_GET, "/x/{a}-{b}/y", S.H_PATHPARAM_FORMAT, s0=b"b", s2=b"b=", s3=b""),
        S.Route(S.M_GET, "/w/{rest:.*}", S.H_PATHPARAM_FORMAT, s0=b"rest", s2=b"[", s3=b"]")])
    paths = [b"/users/42", b"/users/a\"b<c", b"/users/\xc3\xa9", b"/users/\xff", b"/x/1-2-3/y", b"/w/a/b/c", b"/w/", b"/nope"]
    _check(spec, S.RequestBatch.pack([S.Req(S.M_GET, paths[i % len(paths)]) for i in range(5000)]))
