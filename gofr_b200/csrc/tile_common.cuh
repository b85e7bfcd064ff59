// tile_common.cuh — the tile skeleton of the batch kernels: serve_body.cuh (serve_*kernel.cu), frame_tiles.cuh (grpc_kernel.cu,
// proto_nested_*kernel.cu), reqlog_kernel.cu and http_kernel.cu.
//
// Execution model: persistent co-resident CTAs walk tiles blockIdx.x, blockIdx.x + gridDim.x, … with one thread per record.
// Each kernel keeps its own tile loop and shared-memory struct and calls these steps, in this order:
//   * tile_barrier_init by thread 0, once per CTA, then the caller's __syncthreads;
//   * the tile's input byte range, from an offset column (offset_range) or from each lane's [lo, hi) (warp_range, a
//     barrier, cta_range by thread 0);
//   * stage_start by thread 0, stage_wait by every thread: ONE TMA bulk copy of the range into shared memory when it fits,
//     and the base that addresses the staged copy (or the source in HBM when it does not fit);
//   * packed output only: place_tile scans the records' output sizes in the CTA and chains tiles by the decoupled
//     look-back, and put_offsets writes the offset column.  The packed-output contract (include/gofr_b200.h): when the
//     output does not fit, whole tiles are dropped and the overflow flag is set, while offsets (and meta) are still written
//     in full, out_off[n] included; no offset passes 2^32 - 1.
// It also holds the TMA bulk-copy and mbarrier wrappers and the look-back.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"

namespace gofr {

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
// global → shared bulk copy (TMA, 1-D): dst/src 16-byte aligned, bytes % 16 == 0
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_global, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_addr(dst_smem)),
                 "l"(src_global), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}
// The copy sources read staged bytes through NON-volatile `ld.shared` inline asm (the compiler may schedule them freely
// among themselves).  Such an asm has no memory operand, so neither a barrier nor a "memory" clobber orders it: only a
// data dependence does.  Every pointer to freshly staged shared memory (the TMA-filled tile after the mbarrier wait, the
// table copy after its __syncthreads) is therefore passed through this empty asm right after the synchronisation: all
// addresses derived from the result depend on it, so no load of the staged bytes can be hoisted above the wait.
// (Round 2: a build with a different store instruction hoisted literal-pool loads above the table barrier in the first
// tile of a CTA — zeros in the output, visible only on the GPU.)
template <typename T>
__device__ __forceinline__ T* launder_after_sync(T* p) {
    asm volatile("" : "+l"(p) : : "memory");
    return p;
}
__device__ __forceinline__ unsigned long long ld_state(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_state(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// decoupled look-back over tile totals.  state = epoch(24) | flag(2) | value(38); flag 1 = tile total, 2 = inclusive
// prefix.  Words written by earlier launches carry an older epoch and read as "not ready"; the host clears every state
// buffer when the epoch wraps (engine.cu, next_epoch).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kValBits = 38;
constexpr unsigned long long kValMask = (1ull << kValBits) - 1;
__device__ __forceinline__ unsigned long long pack_state(uint32_t epoch, uint32_t flag, unsigned long long v) {
    return ((unsigned long long)(epoch & kEpochMask) << (kValBits + 2)) | ((unsigned long long)flag << kValBits) | (v & kValMask);
}

// Called by warp 0.  Returns the exclusive prefix of `tile` (valid in every lane).
__device__ __forceinline__ unsigned long long lookback(unsigned long long* state, uint32_t epoch, uint32_t tile,
                                                       unsigned long long total, uint32_t lane) {
    if (lane == 0) st_state(&state[tile], pack_state(epoch, tile == 0 ? 2 : 1, total));
    unsigned long long excl = 0;
    if (tile > 0) {
        long long base = (long long)tile - 1;
        for (;;) {
            long long t = base - (long long)lane;
            unsigned long long s = t >= 0 ? ld_state(&state[t]) : pack_state(epoch, 2, 0);
            uint32_t flag = (uint32_t)(s >> kValBits) & 3u;
            bool ready = (uint32_t)(s >> (kValBits + 2)) == (epoch & kEpochMask) && flag != 0;
            uint32_t not_ready = __ballot_sync(0xFFFFFFFFu, !ready);
            uint32_t is_p = __ballot_sync(0xFFFFFFFFu, ready && flag == 2);
            uint32_t upto = is_p ? (uint32_t)__ffs((int)is_p) - 1 : 31u;  // lanes 0..upto contribute
            uint32_t need = upto == 31 ? 0xFFFFFFFFu : ((1u << (upto + 1)) - 1);
            if (not_ready & need) { __nanosleep(40); continue; }
            unsigned long long v = (lane <= upto) ? (s & kValMask) : 0ull;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
            excl += v;
            if (is_p) break;
            base -= 32;
        }
        if (lane == 0) st_state(&state[tile], pack_state(epoch, 2, excl + total));
    }
    return excl;
}

// ---------------------------------------------------------------------------------------------------------------
// the tile skeleton
// ---------------------------------------------------------------------------------------------------------------
// Thread 0: initialise the mbarrier of the tile input (one arrival: thread 0's expect_tx) and fence the initialisation;
// the caller's next __syncthreads publishes it.
__device__ __forceinline__ void tile_barrier_init(uint64_t* bar) {
    asm volatile(
        "mbarrier.init.shared::cta.b64 [%0], 1;\n\t"
        "fence.mbarrier_init.release.cluster;" ::"r"(smem_addr(bar))
        : "memory");
}

// A tile's input bytes [lo, hi), rounded out to 16 bytes (the bulk copy's granule)
struct ByteRange {
    uint32_t lo, hi;
};
__device__ __forceinline__ ByteRange round16(uint32_t lo, uint32_t hi) { return ByteRange{lo & ~15u, (hi + 15u) & ~15u}; }

// The range of records t0 .. t1 - 1 whose bytes lie back to back, record r at [off[r], off[r + 1])
__device__ __forceinline__ ByteRange offset_range(const uint32_t* off, uint32_t t0, uint32_t t1) {
    return round16(__ldg(off + t0), __ldg(off + t1));
}
// The range as the union of each lane's [lo, hi) (an idle lane passes [0xFFFFFFFF, 0)), in two steps around a barrier:
// warp_range leaves each warp's union in warp_lo / warp_hi; after a __syncthreads, cta_range (thread 0) takes their
// union, with `tail` bytes more after the last one, and leaves it in in_lo / in_hi for every thread to read after the next.
__device__ __forceinline__ void warp_range(uint32_t lo, uint32_t hi, uint32_t* warp_lo, uint32_t* warp_hi) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xFFFFFFFFu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xFFFFFFFFu, hi, o));
    }
    if ((threadIdx.x & 31) == 0) { warp_lo[threadIdx.x >> 5] = lo; warp_hi[threadIdx.x >> 5] = hi; }
}
template <int NW>
__device__ __forceinline__ ByteRange cta_range(const uint32_t (&warp_lo)[NW], const uint32_t (&warp_hi)[NW], uint32_t tail,
                                               uint32_t& in_lo, uint32_t& in_hi) {
    uint32_t l = warp_lo[0], h = warp_hi[0];
#pragma unroll
    for (int w = 1; w < NW; w++) { l = min(l, warp_lo[w]); h = max(h, warp_hi[w]); }
    const ByteRange r = round16(l, h + tail);
    in_lo = r.lo;
    in_hi = r.hi;
    return r;
}

// Does the range fit a staging buffer of `cap` bytes?  If not, the tile reads its input from HBM.
__device__ __forceinline__ bool stageable(ByteRange r, uint32_t cap) { return r.hi > r.lo && r.hi - r.lo <= cap; }
// Thread 0 copies src[r.lo, r.hi) to the staging buffer with one TMA bulk copy, if it fits; other callers do nothing.  The
// caller has made sure by a barrier that no thread still reads the previous tile's staged bytes.
__device__ __forceinline__ void stage_start(uint64_t* bar, uint8_t* stage, const uint8_t* src, ByteRange r, uint32_t cap) {
    if (stageable(r, cap) && threadIdx.x == 0) {
        mbar_expect_tx(bar, r.hi - r.lo);
        bulk_g2s(stage, src + r.lo, r.hi - r.lo, bar);
    }
}
// Every thread: wait for that copy and return the base at which base + x addresses byte x of src — in the staged copy when
// the range was staged, else src itself.  The staged pointer is laundered (see launder_after_sync) here and nowhere else.
__device__ __forceinline__ const uint8_t* stage_wait(uint64_t* bar, uint32_t& parity, const uint8_t* stage, const uint8_t* src,
                                                     ByteRange r, uint32_t cap) {
    if (!stageable(r, cap)) return src;
    mbar_wait(bar, parity);
    parity ^= 1;
    return launder_after_sync(stage) - r.lo;
}

// Inclusive prefix sum over the 32 lanes of a warp
__device__ __forceinline__ uint32_t warp_inclusive_sum(uint32_t v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, v, o);
        if (lane >= (uint32_t)o) v += u;
    }
    return v;
}

// Where a tile's packed output goes: the tile's first byte, this thread's offset inside the tile, and whether the whole tile
// fits the output (within out_cap, every offset within u32).
struct TilePlace {
    unsigned long long base;
    uint32_t excl;
    bool fits;
};
// Every thread of the CTA, with its record's output length `len` (0 for an idle thread): scans the lengths in the CTA
// through warp_sum, chains the tile behind the tiles before it (warp 0 runs the look-back, or takes tile * tile_total when
// no_lookback: GOFR_DEBUG_NO_LOOKBACK, valid for fixed-size outputs only), publishes the result in tile_base, offsets it by
// chain0 and sets p.overflow when the tile does not fit.  P is the kernel's parameter struct (tile_state, epoch, out_cap,
// overflow).  Contains two __syncthreads.
template <class P, int NW>
__device__ __forceinline__ TilePlace place_tile(const P& p, uint32_t tile, uint32_t len, uint32_t (&warp_sum)[NW],
                                                unsigned long long& tile_base, bool no_lookback = false,
                                                unsigned long long chain0 = 0) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t incl = warp_inclusive_sum(len, lane);
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    uint32_t warp_excl = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) {
        const uint32_t s = warp_sum[w];
        if ((uint32_t)w < warp) warp_excl += s;
        tile_total += s;
    }
    TilePlace t;
    t.excl = warp_excl + incl - len;
    if (warp == 0) {
        const unsigned long long b = no_lookback ? (unsigned long long)tile * tile_total
                                                 : lookback(p.tile_state, p.epoch, tile, tile_total, lane);
        if (lane == 0) tile_base = b;
    }
    __syncthreads();
    t.base = tile_base + chain0;
    t.fits = t.base + tile_total <= p.out_cap && t.base + tile_total <= 0xFFFFFFFFull;
    if (!t.fits && tid == 0) atomicExch(p.overflow, 1u);
    return t;
}
// The offset column of a valid record i: out_off[i], and out_off[n] after the batch's last record
__device__ __forceinline__ void put_offsets(uint32_t* out_off, uint32_t i, uint32_t n, const TilePlace& t, uint32_t len) {
    out_off[i] = (uint32_t)(t.base + t.excl);
    if (i == n - 1) out_off[n] = (uint32_t)(t.base + t.excl + len);
}

}  // namespace gofr
