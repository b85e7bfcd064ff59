"""The packed output of a host-batch call past 4 GiB.  Offsets are 32-bit, so a chunk whose bytes would pass 0xFFFFFFFF is
not written and the call fails with GOFR_ERR_CAPACITY, with the offsets of what was written intact.  Pinned buffers have
always been handled so (advance_kernel); this checks the pageable path, which shares the rule with every host-batch call."""
import ctypes as C
import os

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table

pytestmark = pytest.mark.gpu
DATE = S.http_date(1789974595)
CAPACITY = 7      # GOFR_ERR_CAPACITY
N = 8_650_000     # config-2 responses of C2_WIRE_BYTES each: 4.5 GB, past 4 GiB
CANARY = 0xA5


def _host_memory() -> int:
    return os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES")


@pytest.mark.skipif(_host_memory() < 16 << 30, reason="needs about 16 GB of host memory")
def test_gpu_pageable_output_past_4gib_is_a_capacity_error():
    import torch
    from gofr_b200.engine import Engine
    assert torch.cuda.is_available(), "this test needs a GPU"
    W = synth.C2_WIRE_BYTES
    # every descriptor names the same arena row, so a chunk uploads one row; each response is W bytes
    one = synth.config2_batch(1)
    batch = S.RequestBatch(np.repeat(one.desc, N), np.repeat(one.trace_ids, N, axis=0), one.arena)
    # pageable (numpy) buffers, out_cap past 4 GiB and past what the whole batch needs
    out = np.full((1 << 32) + (256 << 20), CANARY, np.uint8)
    assert out.size > N * W
    off = np.full(N + 1, 0xFFFFFFFF, np.uint32)
    meta = np.full(N, 0xFFFFFFFF, np.uint32)
    eng = Engine(Table(synth.config2_spec()), 0)
    L = _abi.lib()
    rb = _abi.ReqBatch(desc=batch.desc.ctypes.data, trace_ids=batch.trace_ids.ctypes.data, arena=batch.arena.ctypes.data,
                       arena_bytes=batch.arena.size, n=batch.n, date=DATE)
    ob = _abi.RespBatch(out=out.ctypes.data, out_cap=out.size, out_off=off.ctypes.data, meta=meta.ctypes.data, out_bytes=0)
    t = C.c_uint64()
    assert L.gofr_batch_submit(eng._e, C.byref(rb), C.byref(ob), C.byref(t)) == 0
    assert L.gofr_batch_wait(eng._e, t.value) == CAPACITY
    eng.close()

    nbytes = int(ob.out_bytes)
    assert nbytes == int(off[N]) and 0 < nbytes <= 0xFFFFFFFF
    # the chunks written are whole responses from the start, their offsets rising by W (no wrap)
    assert nbytes % W == 0
    done = nbytes // W
    assert done < N
    assert np.array_equal(off[:done], np.arange(done, dtype=np.uint64).astype(np.uint32) * np.uint32(W))
    # every request was served, and each meta word is the same 200
    assert (meta == meta[0]).all() and int(meta[0]) & 0xFFFF == 200
    # the responses are identical; nothing at or past out_bytes was written
    first = out[:W].copy()
    assert first[:15].tobytes() == b"HTTP/1.1 200 OK"
    rows = out[:nbytes].reshape(done, W)
    for lo in range(0, done, 1 << 20):  # a window at a time: the whole comparison would take another 4 GB
        assert (rows[lo:lo + (1 << 20)] == first).all(), lo
    assert (out[nbytes:] == CANARY).all()
