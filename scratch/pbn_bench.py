#!/usr/bin/env python
"""pbn_bench.py — kernel time of the nested proto3 codec (gofr_proto_encode_nested_device / gofr_proto_decode_nested_device):
   [GOFR_LIB_PATH=scratch/variants/libgofr_X.so] python scratch/pbn_bench.py [--n 1048576] [--steps 20] [--only a,b,c]
Workloads (1 Mi messages each; 1024 distinct rows repeated):
   a  the PAGE / ITEM type of tests/proto_nested_harness.py (no maps)
   b  M { map<string, string> labels = 1; map<int64, Item> items = 2; } with 8 labels and 8 items
   c  the same type with 64 labels and 64 items (short strings, no tags): the decoder's worst case (selection over 64
      entries per map)
   e  the type of b with 200..400 labels and 200..400 items per message (256 distinct rows, --n-large messages): beyond
      the first pass's 64 entries, so its frames are DEFER and the second pass
      (gofr_proto_decode_nested_deferred_device) decodes them
   d  Event { int64 id = 1; optional string note = 2; optional int64 parent = 3;
              oneof payload { Click click = 4; string text = 5; int64 code = 6; } repeated Tag tags = 7; }
      (field presence: the *_presence kernels through the _ex calls) with about half of the optional fields set and the
      oneof cases (none, click, text, code) spread evenly
A workload named twice in --only (a,d,a,d) runs again on the same rows: alternate two workloads to see the noise.
The decoder runs on the encoder's output, then the second pass on the decoder's status column ("deferred"; with
--select-all every frame is selected, as if the first pass had deferred them all).  CUDA events around `steps` launches after 3 warm-up launches; one JSON line per
workload and direction, after the card's name, power limit and max SM clock (nvidia-smi, read-only query)."""
import argparse
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gofr_b200 import _abi, synth  # noqa: E402
from gofr_b200 import spec as S  # noqa: E402
from gofr_b200.engine import Engine  # noqa: E402
from gofr_b200.table import Table  # noqa: E402
from tests.proto_nested_harness import MSGS, rand_value  # noqa: E402

F = S.ProtoNField
ITEM = [F(1, S.PB_INT64), F(2, S.PB_STRING), F(3, S.PB_STRING, True), F(4, S.PB_DOUBLE)]
MAP_MSGS = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MAP, False, 2)],
            [F(1, S.PB_STRING), F(2, S.PB_STRING)],
            [F(1, S.PB_INT64), F(2, S.PB_MESSAGE, False, 3)],
            ITEM]
OPT = S.PB_OPTIONAL
EVENT_MSGS = [[F(1, S.PB_INT64), F(2, S.PB_STRING, presence=OPT), F(3, S.PB_INT64, presence=OPT), F(4, S.PB_MESSAGE, False, 1, 1),
               F(5, S.PB_STRING, presence=1), F(6, S.PB_INT64, presence=1), F(7, S.PB_MESSAGE, True, 2)],
              [F(1, S.PB_INT32), F(2, S.PB_INT32)],        # Click { int32 x = 1; int32 y = 2; }
              [F(1, S.PB_STRING)]]                          # Tag { string name = 1; }


def event_value(rnd, i):
    case = i % 4                                            # the oneof: unset, click, text, code
    return [rnd.randint(1, 10 ** 12),
            "note-%d" % rnd.randint(0, 999) if rnd.random() < 0.5 else None,
            rnd.randint(0, 10 ** 9) if rnd.random() < 0.5 else None,
            [rnd.randint(0, 1920), rnd.randint(0, 1080)] if case == 1 else None,
            "text-%d" % rnd.randint(0, 10 ** 6) if case == 2 else None,
            rnd.randint(-10 ** 6, 10 ** 6) if case == 3 else None,
            [["tag-%d" % rnd.randint(0, 99)] for _ in range(rnd.randint(0, 3))]]


def map_value(rnd, n, compact=False):
    """compact: short strings and no tags, so that 1 Mi rows of 64 + 64 entries stay within 32-bit offsets"""
    if compact:
        labels = {"l%02d" % k: "v%d" % rnd.randint(0, 9) for k in range(n)}
    else:
        labels = {"label-%02d-%d" % (k, rnd.randint(0, 999)): "value-%d" % rnd.randint(0, 10 ** 6) for k in range(n)}
    items = {}
    while len(items) < n:
        items[rnd.randint(-10 ** 12, 10 ** 12)] = ([rnd.randint(0, 10 ** 9), "i", [], rnd.random()] if compact else
                                                   [rnd.randint(0, 10 ** 9), "item-%d" % rnd.randint(0, 999), ["t1", "t2"], rnd.random()])
    return [labels, items]


def tiled_rows(msgs, values, n):
    """rows of `values` repeated to n messages"""
    rows, off = S.pack_proto_nested_rows(msgs, 0, values)
    k, blen = len(values), int(off[-1])
    reps = (n + k - 1) // k
    all_rows = np.concatenate([np.tile(rows[:blen], reps), np.zeros(16, np.uint8)])
    j = np.arange(n + 1, dtype=np.int64)
    all_off = off.astype(np.int64)[j % k] + (j // k) * blen
    assert all_off[-1] < 1 << 32, "rows beyond 32-bit offsets"
    return all_rows, all_off.astype(np.uint32)


def timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--only", default="a,b,c")
    ap.add_argument("--n-large", type=int, default=32768)
    ap.add_argument("--select-all", action="store_true")
    ap.add_argument("--tag", default=os.environ.get("GOFR_LIB_PATH", "tree"))
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"gpu": smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else "nvidia-smi failed", "lib": a.tag}), flush=True)
    rnd = random.Random(5)
    work = {"a": (MSGS, lambda: [rand_value(rnd, MSGS, 0) for _ in range(1024)]),
            "b": (MAP_MSGS, lambda: [map_value(rnd, 8) for _ in range(1024)]),
            "c": (MAP_MSGS, lambda: [map_value(rnd, 64, compact=True) for _ in range(1024)]),
            "d": (EVENT_MSGS, lambda: [event_value(rnd, i) for i in range(1024)]),
            "e": (MAP_MSGS, lambda: [map_value(rnd, rnd.randint(200, 400)) for _ in range(256)])}
    cache = {}
    eng = Engine(Table(synth.config1_spec()), 0)
    L = _abi.lib()
    st = torch.cuda.current_stream().cuda_stream
    for w in a.only.split(","):
        msgs, gen = work[w]
        if w not in cache:
            cache[w] = tiled_rows(msgs, gen(), a.n_large if w == "e" else a.n)
        rows, off = cache[w]
        n = len(off) - 1
        nm, nf, k = S.proto_nested_tables(msgs)
        pr = S.proto_nested_presence(msgs)
        d_rows = torch.from_numpy(rows).cuda()
        d_off = torch.from_numpy(off.view(np.int32)).cuda()
        cap = int(off[-1]) * 2 + 64 * n
        d_out = torch.empty(cap + 16, dtype=torch.uint8, device="cuda")
        d_out_off = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
        d_meta = torch.zeros(n, dtype=torch.int32, device="cuda")

        def enc():
            if pr is not None:
                _abi.check(L.gofr_proto_encode_nested_ex_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, pr.ctypes.data,
                                                                d_rows.data_ptr(), d_off.data_ptr(), n, d_out.data_ptr(), cap,
                                                                d_out_off.data_ptr(), d_meta.data_ptr(), st), "encode")
                return
            _abi.check(L.gofr_proto_encode_nested_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, d_rows.data_ptr(),
                                                         d_off.data_ptr(), n, d_out.data_ptr(), cap, d_out_off.data_ptr(),
                                                         d_meta.data_ptr(), st), "encode")
        t_enc = timed(enc, a.steps)
        assert not d_meta.any().item()
        out_bytes = int(d_out_off[-1].item()) & 0xFFFFFFFF   # a u32 offset in an int32 tensor
        rows_cap = int(off[-1]) + 64 * n
        d_back = torch.empty(rows_cap, dtype=torch.uint8, device="cuda")
        d_back_off = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
        d_meta2 = torch.zeros(n, dtype=torch.int32, device="cuda")

        def dec():
            if pr is not None:
                _abi.check(L.gofr_proto_decode_nested_ex_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, pr.ctypes.data,
                                                                d_out.data_ptr(), d_out_off.data_ptr(), n, d_back.data_ptr(), rows_cap,
                                                                d_back_off.data_ptr(), d_meta2.data_ptr(), st), "decode")
                return
            _abi.check(L.gofr_proto_decode_nested_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0, d_out.data_ptr(),
                                                         d_out_off.data_ptr(), n, d_back.data_ptr(), rows_cap, d_back_off.data_ptr(),
                                                         d_meta2.data_ptr(), st), "decode")
        t_dec = timed(dec, a.steps)
        large = w == "e"
        assert bool((d_meta2 == 6).all().item()) if large else not d_meta2.any().item()
        same = large or bool(torch.equal(d_back[:int(off[-1])], d_rows[:int(off[-1])]))   # decode(encode(rows)) == rows
        # the second pass on the first pass's statuses (or every frame selected)
        d_sel = torch.full_like(d_meta2, 6) if a.select_all else d_meta2.clone()
        n_sel = int((d_sel == 6).sum().item())
        d_meta3 = torch.zeros(n, dtype=torch.int32, device="cuda")

        def dec2():
            _abi.check(L.gofr_proto_decode_nested_deferred_device(eng._e, nm.ctypes.data, len(msgs), nf.ctypes.data, k, 0,
                                                                  None if pr is None else pr.ctypes.data, d_out.data_ptr(),
                                                                  d_out_off.data_ptr(), n, d_sel.data_ptr(), d_back.data_ptr(), rows_cap,
                                                                  d_back_off.data_ptr(), d_meta3.data_ptr(), st), "deferred")
        t_dec2 = timed(dec2, a.steps)
        assert not d_meta3.any().item()
        if n_sel == n:
            same = same and bool(torch.equal(d_back[:int(off[-1])], d_rows[:int(off[-1])]))
        for direction, t in (("encode", t_enc), ("decode", t_dec), ("deferred", t_dec2)):
            print(json.dumps({"workload": w, "dir": direction, "n": n, "ms": round(t, 4), "Mmsg_per_s": round(n / t / 1e3, 1),
                              "frame_GBps": round(out_bytes / t / 1e6, 1), "row_bytes": int(off[-1]), "frame_bytes": out_bytes,
                              "round_trip_equal": same, "selected": n_sel if direction == "deferred" else None, "lib": a.tag}), flush=True)
        del d_rows, d_out, d_back
        torch.cuda.empty_cache()
    eng.close()


if __name__ == "__main__":
    main()
