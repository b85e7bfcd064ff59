// emu_pack.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the per-record logic of the chunk pack kernel (gofr_b200/csrc/pack_device.cuh, the same __host__ __device__
// functions pack_kernel.cu calls) on the CPU: each record's source and size, and its copy through the Writer, one record
// after another from `start` on.  The tile loop, place_tile and the look-back only exist in the kernel and are covered by
// the `-m gpu` tests.  Nothing in the product links or loads this file.
#include <cstdint>
#include <cstring>

#include "../../gofr_b200/csrc/pack_device.cuh"

using namespace gofr;

// b may be null (one source).  Record i goes to out + out_off[i], out_off[0] = start.  Returns -1 when out_cap is too small.
extern "C" int emu_pack(const uint8_t* a, const uint32_t* a_off, uint64_t a_cap, const uint8_t* b, const uint32_t* b_off,
                        uint64_t b_cap, const uint32_t* sel, uint32_t n, uint32_t start, uint8_t* out, uint64_t out_cap,
                        uint32_t* out_off) {
    PackParams p;
    memset(&p, 0, sizeof p);
    p.a = a; p.a_off = a_off; p.a_cap = a_cap;
    p.b = b; p.b_off = b_off; p.b_cap = b_cap; p.sel = sel;
    p.n = n;
    uint64_t pos = start;
    for (uint32_t i = 0; i < n; i++) {
        const PackRec r = pack_record(p, i);
        out_off[i] = (uint32_t)pos;
        if (pos + r.len > out_cap) return -1;
        uint32_t col[GOFR_STAGE_WORDS];
        pack_emit(r, out + pos, col);
        pos += r.len;
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}

// 0: flush decisions as one lane takes them; 1: a flush at every decision point; 2: pseudo-random extra flushes (on the
// GPU a lane also flushes when another lane of its warp needs room)
extern "C" void emu_pack_any_mode(int mode) { emu_any_mode() = mode; }
