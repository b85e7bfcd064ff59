// emu_conn_result.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the per-request logic of gofr_conn_batch_respond's splice step (gofr_b200/csrc/conn_result_device.cuh, the same
// __host__ __device__ functions conn_result_kernel.cu calls) on the CPU, request after request from `start` on: the running
// position stands in for the kernel's scan and look-back, which only exist on the device and are covered by the `-m gpu`
// tests.  Nothing in the product links or loads this file.
#include <cstdint>
#include <cstring>

#include "../../gofr_b200/csrc/conn_result_device.cuh"

using namespace gofr;

// desc[n] is rewritten in place, as on the device.  arena: the parse arena, addressed by the descriptors' offsets.  rec_chunk
// holds the chunk's records from the caller's byte rlo on (the slot buffer the engine uploads them to); rec_off[n + 1] are
// the caller's offsets of the chunk's requests.  Request i goes to out + out_off[i], out_off[0] = start (a multiple of 4).
// Returns -1 when out_cap is too small.
extern "C" int emu_conn_result(gofr_req_desc* desc, uint32_t n, const uint8_t* arena, const uint8_t* rec_chunk, uint32_t rlo,
                               const uint32_t* rec_off, uint32_t start, uint8_t* out, uint64_t out_cap, uint32_t* out_off) {
    ConnResultParams p;
    memset(&p, 0, sizeof p);
    p.desc = desc; p.arena = arena; p.rec = rec_chunk - rlo; p.rec_off = rec_off; p.n = n; p.out = out; p.out_cap = out_cap;
    uint64_t pos = start;
    for (uint32_t i = 0; i < n; i++) {
        const ConnSplice s = conn_splice(p, i);
        out_off[i] = (uint32_t)pos;
        if (pos + s.size > out_cap) return -1;
        uint32_t col[GOFR_STAGE_WORDS];
        conn_splice_emit(p, i, s, (uint32_t)pos, col);
        pos += s.size;
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}

// 0: flush decisions as one lane takes them; 1: a flush at every decision point; 2: pseudo-random extra flushes
extern "C" void emu_conn_result_any_mode(int mode) { emu_any_mode() = mode; }
