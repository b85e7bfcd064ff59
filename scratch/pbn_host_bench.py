#!/usr/bin/env python
"""pbn_host_bench.py — the nested proto3 codec on host buffers (gofr_proto_batch_encode / _decode), pinned in and out:
   python scratch/pbn_host_bench.py [--n 1048576] [--steps 10] [--only a,b,d]
Workloads (a), (b) and (d) of scratch/pbn_bench.py (DESIGN §6), 1 Mi messages each.  Per workload and direction, one JSON
line with
   host_ms      submit + wait of the whole batch (host clock; the call ends in a device synchronise), after 2 warm-up calls;
   floor_ms     the link floor: the same H2D bytes (records + offsets) and D2H bytes (output + offsets + statuses) copied
                concurrently between pinned and device buffers by torch, no kernel (as pcie_probe.py measures it);
   resident_ms  the resident calls' own time on the same records already in HBM (CUDA events; decode: both passes).
The first line gives the card's name, power limit and max SM clock (nvidia-smi, read-only query)."""
import argparse
import ctypes as C
import json
import os
import random
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pbn_bench as B  # noqa: E402
from gofr_b200 import _abi, synth  # noqa: E402
from gofr_b200 import spec as S  # noqa: E402
from gofr_b200.engine import Engine, pinned_array  # noqa: E402
from gofr_b200.table import Table  # noqa: E402


def pinned_copy(a: np.ndarray) -> np.ndarray:
    p = pinned_array(a.nbytes, a.dtype)
    p[:] = a
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default="a,b,d")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"gpu": smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else "nvidia-smi failed"}), flush=True)
    rnd = random.Random(5)
    work = {"a": (B.MSGS, lambda: [B.rand_value(rnd, B.MSGS, 0) for _ in range(1024)]),
            "b": (B.MAP_MSGS, lambda: [B.map_value(rnd, 8) for _ in range(1024)]),
            "d": (B.EVENT_MSGS, lambda: [B.event_value(rnd, i) for i in range(1024)])}
    eng = Engine(Table(synth.config1_spec()), 0)
    L = _abi.lib()
    dev = torch.device("cuda", 0)
    for w in a.only.split(","):
        msgs, gen = work[w]
        rows, off = B.tiled_rows(msgs, gen(), a.n)
        n = len(off) - 1
        nm, nf, k = S.proto_nested_tables(msgs)
        pr = S.proto_nested_presence(msgs)
        prp = None if pr is None else pr.ctypes.data
        frames, f_off, f_meta = eng.proto_encode_batch(msgs, 0, rows, off)     # the decode direction's input
        assert (f_meta == 0).all()
        frames = np.concatenate([frames, np.zeros(16, np.uint8)])
        for direction, data, doff in (("encode", rows, off), ("decode", frames, f_off)):
            decode = direction == "decode"
            h_data, h_off = pinned_copy(data), pinned_copy(doff.astype(np.uint32))
            # the exact output size (the bound, summed over 1 Mi records, would ask for gigabytes of pinned memory)
            cap = int(off[-1]) if decode else int(f_off[-1])
            h_out, h_out_off, h_meta = pinned_array(cap), pinned_array(4 * (n + 1), np.uint32), pinned_array(4 * n, np.uint32)
            pb = _abi.ProtoBatch(data=h_data.ctypes.data, data_bytes=h_data.size, off=h_off.ctypes.data, n=n)
            ob = _abi.RespBatch(out=h_out.ctypes.data, out_cap=cap, out_off=h_out_off.ctypes.data, meta=h_meta.ctypes.data, out_bytes=0)
            fn = L.gofr_proto_batch_decode if decode else L.gofr_proto_batch_encode

            def host():
                t = C.c_uint64()
                _abi.check(fn(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, prp, C.byref(pb), C.byref(ob), C.byref(t)), direction)
                _abi.check(L.gofr_batch_wait(eng._e, t.value), "gofr_batch_wait")
            for _ in range(2):
                host()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                host()
            host_ms = (time.perf_counter() - t0) * 1e3 / a.steps
            out_bytes = int(ob.out_bytes)
            # the link floor for the same bytes
            h2d = int(doff[-1]) + 4 * (n + 1)
            d2h = out_bytes + 8 * n + 4
            src_h = torch.from_numpy(pinned_array(h2d))
            dst_h = torch.from_numpy(pinned_array(d2h))
            d_in = torch.empty(h2d, dtype=torch.uint8, device=dev)
            d_out = torch.empty(d2h, dtype=torch.uint8, device=dev)
            s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

            def link():
                with torch.cuda.stream(s1):
                    d_in.copy_(src_h, non_blocking=True)
                with torch.cuda.stream(s2):
                    dst_h.copy_(d_out, non_blocking=True)
                torch.cuda.synchronize()
            for _ in range(2):
                link()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                link()
            floor_ms = (time.perf_counter() - t0) * 1e3 / a.steps
            del src_h, dst_h, d_in, d_out
            # the resident calls on the same records in HBM
            d_data = torch.from_numpy(np.ascontiguousarray(data)).to(dev)
            d_doff = torch.from_numpy(doff.astype(np.uint32).view(np.int32)).to(dev)
            d_res = torch.empty(cap + 16, dtype=torch.uint8, device=dev)
            d_res2 = torch.empty(cap + 16, dtype=torch.uint8, device=dev)
            d_roff = torch.zeros(n + 1, dtype=torch.int32, device=dev)
            d_roff2 = torch.zeros(n + 1, dtype=torch.int32, device=dev)
            d_m1 = torch.zeros(n, dtype=torch.int32, device=dev)
            d_m2 = torch.zeros(n, dtype=torch.int32, device=dev)
            st = torch.cuda.current_stream().cuda_stream

            def resident():
                if decode:
                    _abi.check(L.gofr_proto_decode_nested_ex_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, prp, d_data.data_ptr(),
                                                                    d_doff.data_ptr(), n, d_res.data_ptr(), cap, d_roff.data_ptr(), d_m1.data_ptr(), st), "decode")
                    _abi.check(L.gofr_proto_decode_nested_deferred_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, prp, d_data.data_ptr(),
                                                                          d_doff.data_ptr(), n, d_m1.data_ptr(), d_res2.data_ptr(), cap, d_roff2.data_ptr(),
                                                                          d_m2.data_ptr(), st), "deferred")
                else:
                    _abi.check(L.gofr_proto_encode_nested_ex_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, prp, d_data.data_ptr(),
                                                                    d_doff.data_ptr(), n, d_res.data_ptr(), cap, d_roff.data_ptr(), d_m1.data_ptr(), st), "encode")
            resident_ms = B.timed(resident, a.steps)
            del d_data, d_doff, d_res, d_res2, d_roff, d_roff2, d_m1, d_m2
            torch.cuda.empty_cache()
            print(json.dumps({"workload": w, "direction": direction, "n": n, "in_bytes": int(doff[-1]), "out_bytes": out_bytes,
                              "host_ms": round(host_ms, 3), "floor_ms": round(floor_ms, 3), "resident_ms": round(resident_ms, 3),
                              "ok": bool((h_meta == 0).all())}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
