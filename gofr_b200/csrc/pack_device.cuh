// pack_device.cuh — per-record logic of the chunk pack kernel (pack_kernel.cu): which source a record's bytes come from, how
// many there are, and their copy to the packed output.  __host__ __device__ so tests/emu runs the same code on the CPU.
//
// The proto host path (gofr_proto_batch_decode / _encode) runs the codec kernels into buffers of their own, from byte 0.
// The pack step moves each record to its place in the chunk's packed output, which starts at the batch position mod 16
// so that egress_kernel can stream it to the caller with 16-byte stores.  When decoding it also merges the two passes'
// row columns by the rule of include/gofr_b200.h: row i is the second pass's when the first pass said GOFR_GRPC_DEFER.
// (The header's rule also asks for the final status to be OK; a first-pass DEFER row is empty, and a second-pass row is
// empty unless its status is OK, so the two rules pick the same bytes.)
#pragma once
#include "engine_internal.h"
#include "serve_device.cuh"

namespace gofr {

struct PackRec {
    const uint8_t* src;
    uint32_t len;
};

// Record i's bytes.  A source range that passes the bytes its codec could write (its buffer overflowed: the codec kernel has
// set the overflow flag, so the chunk is reported) packs as empty rather than reading past the buffer.
GOFR_HD PackRec pack_record(const PackParams& p, uint32_t i) {
    const bool use_b = p.b != nullptr && p.sel[i] == GOFR_GRPC_DEFER;
    const uint8_t* s = use_b ? p.b : p.a;
    const uint32_t* o = use_b ? p.b_off : p.a_off;
    const uint64_t cap = use_b ? p.b_cap : p.a_cap;
    const uint32_t lo = o[i], hi = o[i + 1];
    if (hi < lo || hi > cap) return PackRec{s, 0u};
    return PackRec{s + lo, hi - lo};
}

// The record's bytes at dst, any alignment of source and destination, through the Writer's staging column
GOFR_HD void pack_emit(const PackRec r, uint8_t* dst, uint32_t* stage_col) {
    if (!r.len) return;
    Writer w;
    w.init(dst, stage_col);
    w.copy<false>(r.src, r.len);
    w.finish();
}

}  // namespace gofr
