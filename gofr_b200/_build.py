"""Builds libgofr_b200.so (CUDA, sm_90a) in-tree with nvcc.  No torch involvement: the library is a plain C ABI."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgofr_b200.so")
SOURCES = ["serve_kernel.cu", "serve_values_kernel.cu", "serve_slots_kernel.cu", "serve_slots_wide_kernel.cu", "serve_slots_values_kernel.cu", "grpc_kernel.cu", "proto_nested_kernel.cu", "proto_nested_decode_kernel.cu", "proto_nested_maps_kernel.cu", "proto_nested_presence_kernel.cu", "proto_nested_deferred_kernel.cu", "reqlog_kernel.cu", "batch_log_kernel.cu", "proto_log_kernel.cu", "route_kernel.cu", "bind_kernel.cu", "http_kernel.cu", "http_frame_kernel.cu", "conn_kernel.cu", "conn_log_kernel.cu", "conn_result_kernel.cu", "egress_kernel.cu", "pack_kernel.cu", "engine.cu", "table_build.cpp", "frontend.cpp", "proto_frontend.cpp", "conn_frontend.cpp", "conn_app_frontend.cpp"]
HEADERS = ["frontend_ring.h", "conn_staging.h","frame_tiles.cuh", "pack_device.cuh", "proto_nested_codecs.cuh", "proto_nested_device.cuh", "proto_nested_decode_device.cuh", "proto_nested_deferred_device.cuh", "serve_body.cuh", "serve_device.cuh", "value_device.cuh", "float_device.cuh", "ryu_tables.inc", "el_tables.inc", "bind_device.cuh", "grpc_device.cuh", "reqlog_device.cuh", "reqlog_tiles.cuh", "batch_log_device.cuh", "http_device.cuh", "http_frame_device.cuh", "conn_device.cuh", "conn_log_device.cuh", "conn_result_device.cuh","tile_common.cuh", "table_format.h", "engine_internal.h",
           "../../include/gofr_b200.h"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "-Xcompiler", "-Wall", "--expt-relaxed-constexpr"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    m = os.path.getmtime(LIB)
    files = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.exists(f) and os.path.getmtime(f) > m for f in files)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    srcs = [f for f in SOURCES if os.path.exists(os.path.join(CSRC, f))]
    extra = os.environ.get("GOFR_EXTRA_NVCC", "").split()  # experiments only, e.g. -DGOFR_SERVE_T=96
    flags = NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else [])
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    hdr_m = max(os.path.getmtime(f) for f in [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)] if os.path.exists(f))
    tag = os.path.join(objdir, ".flags")
    tag_text = " ".join(flags)
    flags_changed = not os.path.exists(tag) or open(tag).read() != tag_text

    # one translation unit per nvcc process, in parallel; objects are reused when neither the source, a header nor the
    # flags changed
    def compile_one(f: str):
        src, obj = os.path.join(CSRC, f), os.path.join(objdir, f + ".o")
        if not force and not flags_changed and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_m):
            return obj, 0, ""
        r = subprocess.run([nvcc] + flags + ["-c", "-o", obj, src], capture_output=True, text=True)
        log = r.stdout + r.stderr
        return obj, r.returncode, log

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=min(len(srcs), os.cpu_count() or 4)) as ex:
        results = list(ex.map(compile_one, srcs))
    log = "".join(o for _, _, o in results)
    if verbose or any(rc for _, rc, _ in results):
        sys.stderr.write(log)
    if any(rc for _, rc, _ in results):
        raise RuntimeError("nvcc failed building libgofr_b200.so")
    open(tag, "w").write(tag_text)
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB] + [o for o, _, _ in results] + ["-lcudart"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("linking libgofr_b200.so failed")
    return LIB


if __name__ == "__main__":
    build(force=True, verbose="-v" in sys.argv)
    print(LIB)
