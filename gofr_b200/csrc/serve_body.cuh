// serve_body.cuh — the fused, persistent serve kernel for sm_90a (body shared by the two kernels: serve_kernel.cu
// instantiates the packed layout, serve_slots_kernel.cu the slot layout).
//
// One launch replaces, for a whole batch, what the reference does per request on a goroutine:
// mux.Router.ServeHTTP → Tracer/Logging/CORS → handler.ServeHTTP → Responder.Respond → net/http framing
// (pkg/gofr/http/router.go:14, middleware/{tracer,logger,cors}.go, pkg/gofr/handler.go:32-36, pkg/gofr/http/responder.go:19-41).
//
// Execution model (HBM-bound integer/byte work; no tensor cores):
//   * grid = co-resident CTAs only (SMs × occupancy); CTA b walks tiles b, b+grid, … of 128 requests, one thread per
//     request;
//   * the tile's descriptors and trace ids are read with coalesced 16-byte loads; its contiguous arena byte range is
//     pulled into shared memory with ONE TMA bulk copy (cp.async.bulk.shared::cluster.global + mbarrier) when it
//     fits, so all per-request byte walking hits shared memory, not HBM;
//   * responses are packed back-to-back in request order: sizes are scanned inside the CTA and chained across CTAs
//     with a decoupled look-back (single pass — inputs are read from HBM exactly once);
//   * each thread streams its response through a funnel-shift word writer (serve_device.cuh) whose completed words
//     collect in a conflict-free shared-memory ring and leave for HBM as whole 32-byte sectors, two 16-byte
//     st.global.cs.v4 each; in the wide slot instance's fast path they leave as whole 128-byte lines, four lines per
//     warp store (the LineStores store policy).  No output tile lives in shared memory, which keeps 5 CTAs (20 warps)
//     resident per SM for this latency-bound byte work.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"
#include "serve_device.cuh"
#include "tile_common.cuh"

namespace gofr {

// ---------------------------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------------------------
constexpr int T = kServeT;
constexpr int NW = T / 32;

constexpr uint32_t kDeferred = 0xFFFFFFFFu;  // length-column mark of a request left for the general pass (never a length)

// RING: words of the Writer's staging ring — GOFR_SOLO_WORDS rows of T for SoloStores; the wide slot instance's
// LineStores columns need GOFR_LINE_WORDS rows of T + 1 (serve_device.cuh).  Only that instance has the larger ring.
template <uint32_t RING>
struct TileShared {
    uint64_t bar;  // mbarrier for the arena bulk load
    uint32_t warp_sum[NW];
    uint32_t warp_lo[NW], warp_hi[NW];
    uint32_t warp_cls[NW];  // slot layout: program shape class of each warp's lane 0
    unsigned long long tile_base;
    uint32_t in_lo, in_hi;
    uint32_t defer_n;         // slot layout: requests waiting for the general pass; their indices (at most 2 T: one tile's
                              // worth is added between two checks) live in the request staging area, which is idle once
                              // the tile loop is over — as static shared memory the list cost every instance its fifth CTA
    uint32_t ring[RING];  // word-major staging buffer of the Writer (serve_device.cuh)
};
constexpr uint32_t kSoloRing = GOFR_SOLO_WORDS * T, kLineRing = GOFR_LINE_WORDS * (T + 1);
static_assert(LineStores::kRowWords == T + 1, "LineStores rows are T + 1 words");

// Slot layout, general pass.  The tile loop of serve_slots_kernel runs only the fast path (size_fast / emit_fast); a request
// it cannot take — a program outside the fast path, a value that needs escaping or decoding, HEAD, an unstaged tile — is
// marked in the length column and served here after the loop, by the general interpreter, with ALL threads of the CTA
// working on such requests at once (128 at a time).  Slots make this legal: a response depends on nothing but its own request.
// Mixed traffic used to make every warp run both emitters, or — when the slow requests were sorted into one warp — made
// the other three wait for it at the next barrier (barrier stall 5.5 cycles per issue on the 64-route workload).  The
// request bytes are read from HBM here (the tile that staged them is gone); the code is out of line so that the tile loop
// keeps its registers and its instruction-cache footprint.
template <class TS>
static __device__ __noinline__ void general_pass(const ServeParams* pp, const TableView tv, const BatchRefs br, TS* sh,
                                          const uint32_t* defer, uint32_t first, uint32_t count) {
    const ServeParams& p = *pp;
    const uint32_t tid = threadIdx.x;
    if (tid >= count) return;
    const uint32_t r = defer[first + tid];
    const uint4 d = __ldg((const uint4*)p.desc + r);
    ReqCtx c;
    c.set(p.arena, d.x, d.y & 0xFFFFu, d.y >> 16, d.z, d.w & 0xFFu, (d.w >> 8) & 0xFFu, false, r);
    route_request(tv, br, c);
    size_routed_general(tv, br, c);
    p.out_off[r] = c.total_len;
    p.meta[r] = request_status(tv, c) | (c.route << 16);
    if (c.total_len <= p.slot_bytes && c.total_len)
        emit_request_general<true>(tv, br, c, p.out + (size_t)r * p.slot_bytes, &sh->ring[tid]);
}

// LINES (slot layout): the fast path stores whole 128-byte lines (emit_fast with LineStores).  Its votes and store rounds
// are warp-uniform, so a warp whose lanes run different programs makes every lane take part in every other lane's: on
// mixed traffic that costs more than whole lines gain (lane pairs, the earlier warp-uniform policy, took config 4 from
// 0.31 to 0.35 ms on an H100 SXM at 400 W).  Only the wide instance, which the engine runs for tables with one fast-path
// program shape, stores lines; it alone carries the larger staging ring.
template <bool SLOTS, bool LINES = false>
__device__ __forceinline__ void serve_body(const ServeParams& p) {
    // (p is a __grid_constant__ kernel parameter: its address can be handed to the out-of-line general pass)
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(16) TileShared<LINES ? kLineRing : kSoloRing> sh;

    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint8_t* tbl = smem;
    uint8_t* in_stage = smem + ((p.hot_bytes + 127u) & ~127u);

    // table → shared memory (once per CTA), then the batch's Date is patched into the literal pool
    {
        const uint4* src = (const uint4*)p.image;
        uint4* dst = (uint4*)tbl;
        for (uint32_t i = tid; i < p.hot_bytes / 16; i += T) dst[i] = src[i];
        if (tid == 0) {
            tile_barrier_init(&sh.bar);
            sh.defer_n = 0;
        }
    }
    __syncthreads();
    patch_dates(tbl, (const uint8_t*)p.date, tid, T);
    __syncthreads();
    tbl = launder_after_sync(tbl);
    TableView tv;
    tv.bind(tbl, p.image);
    BatchRefs br;
    br.ids = (const uint8_t*)p.ids; br.bind_scratch = p.bind_scratch; br.bind_row_words = p.bind_row_words;

    uint32_t parity = 0;
    const unsigned long long chain0 = p.chain_pos ? (*p.chain_pos & 15ull) : 0ull;

    // Static round-robin tile assignment over the co-resident grid: tile t only ever waits on tiles < t, all of which
    // belong to resident CTAs that process their tiles in increasing order, so the look-back cannot deadlock.
    // (A dynamic ticket counter was measured slower: the atomic's round trip sits on every tile's critical path.)
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * T + tid;
        const bool valid = i < p.n;
        uint4 d = make_uint4(0, 0, 0, 0);
        if (valid) d = __ldg((const uint4*)p.desc + i);
        // the trace ids are read only when the response is written: have the line in L1 by then (one lane per 128-byte line)
        if (valid && (lane & 7u) == 0) asm volatile("prefetch.global.L1 [%0];" ::"l"((const uint4*)p.ids + i));
        const uint32_t arena_off = d.x, path_len = d.y & 0xFFFFu, query_len = d.y >> 16, data_len = d.z;
        const uint32_t data_off = (arena_off + path_len + query_len + 3u) & ~3u;
        const uint32_t end = data_off + data_len;

        // ---- the tile's arena byte range ----
        warp_range(valid ? arena_off : 0xFFFFFFFFu, valid ? end : 0u, sh.warp_lo, sh.warp_hi);
        __syncthreads();  // also: every thread is done reading the previous tile's in_stage
        if (tid == 0) stage_start(&sh.bar, in_stage, p.arena, cta_range(sh.warp_lo, sh.warp_hi, 0u, sh.in_lo, sh.in_hi), p.in_cap);
        __syncthreads();
        const ByteRange in{sh.in_lo, sh.in_hi};
        const bool in_staged = stageable(in, p.in_cap);
        const uint8_t* abase = stage_wait(&sh.bar, parity, in_stage, p.arena, in, p.in_cap);  // abase + arena_off: the request

        // ---- stage 1: route ----
        ReqCtx c;
        c.set(abase, arena_off, path_len, query_len, data_len, d.w & 0xFFu, (d.w >> 8) & 0xFFu, in_staged, valid ? i : 0xFFFFFFFFu);
        if (valid) route_request(tv, br, c);

        if (SLOTS) {
            // Slot layout: response i owns out + i * slot_bytes.  No scan, no look-back, no dependence between tiles —
            // and every response starts 16-byte aligned.  Nothing ties a request to a particular thread either, so a
            // tile with mixed traffic is first regrouped by program shape: lanes of a warp then walk the same op
            // sequence instead of serialising over every shape present (the interpreter's only divergence).
            uint32_t cls = 31u;  // idle lanes sort last
            if (valid) {
                cls = 0u;
                if (c.prog != 0xFFFF) {
                    const ProgRec& PR = tv.progs()[c.prog];
                    // requests that are known to take the general interpreter (a program outside the fast path, a query
                    // value that needs decoding, HEAD) form one class of their own: they end up in the same warp instead
                    // of making every warp of the tile run both emitters
                    const bool general = !(PR.flags & PF_FAST) || (c.pv_flags & 2u) || c.method() == GOFR_M_HEAD || !c.staged();
                    cls = general ? 30u : PR.shape_class;
                }
            }
            const uint32_t cls0 = __shfl_sync(0xFFFFFFFFu, cls, 0);
            if (lane == 0) sh.warp_cls[warp] = cls0;
            bool mixed = __syncthreads_or(cls != cls0);
#pragma unroll
            for (int w = 1; w < NW; w++) mixed |= sh.warp_cls[w] != sh.warp_cls[0];
            if (mixed) {
                uint32_t* hist = sh.ring;  // the staging ring is idle until the first response is written
                if (tid < 32) hist[tid] = 0;
                __syncthreads();
                const uint32_t rank = atomicAdd(&hist[cls], 1u);
                __syncthreads();
                if (warp == 0) {
                    const uint32_t v = hist[lane];
                    hist[lane] = warp_inclusive_sum(v, lane) - v;
                }
                __syncthreads();
                const uint32_t pos = hist[cls] + rank;
                __syncthreads();
                uint32_t* x = sh.ring + pos;  // word-major exchange record of the request now owned by thread `pos`
                x[0 * T] = (uint32_t)(c.path - abase); x[1 * T] = c.path_len | c.query_len << 16; x[2 * T] = c.data_len;
                x[3 * T] = c.data_off; x[4 * T] = c.mflags; x[5 * T] = c.index; x[6 * T] = c.prog | c.route << 16;
                x[7 * T] = c.pv_off; x[8 * T] = c.pv_len; x[9 * T] = c.pv_flags; x[10 * T] = c.def_off; x[11 * T] = c.def_len;
                __syncthreads();
                const uint32_t* y = sh.ring + tid;
                c.path = abase + y[0 * T]; c.path_len = y[1 * T] & 0xFFFFu; c.query_len = y[1 * T] >> 16; c.data_len = y[2 * T];
                c.data_off = y[3 * T]; c.mflags = y[4 * T]; c.index = y[5 * T]; c.prog = y[6 * T] & 0xFFFFu; c.route = y[6 * T] >> 16;
                c.pv_off = y[7 * T]; c.pv_len = y[8 * T]; c.pv_flags = y[9 * T]; c.def_off = y[10 * T]; c.def_len = y[11 * T];
                __syncthreads();  // the ring is free again before any Writer stages into it
            }
            const uint32_t r = c.index;  // the request this thread serves now
            bool emit = false;
            if (r != 0xFFFFFFFFu) {
                if (c.prog == 0xFFFFu) {  // GOFR_H_HOST: nothing to emit, status 0 = pending on the host
                    p.out_off[r] = 0;
                    p.meta[r] = c.route << 16;
                } else if (size_fast(tv, br, c)) {
                    p.out_off[r] = c.total_len;  // the length column; > slot_bytes tells the host the slot was too small
                    p.meta[r] = request_status(tv, c) | (c.route << 16);
                    if (c.total_len <= p.slot_bytes && c.total_len) {
                        if (LINES) emit = true;
                        else emit_fast(tv, br, c, p.out + (size_t)r * p.slot_bytes, &sh.ring[tid], SoloStores{});
                    }
                } else {
                    p.out_off[r] = kDeferred;  // left for the general pass after the tile loop
                }
            }
            if (LINES) {
                // every thread of the CTA is here, and every lane of a warp runs the store rounds (eight lanes per line):
                // a lane without a response to write runs an empty one
                emit_fast(tv, br, c, emit ? p.out + (size_t)r * p.slot_bytes : p.out, &sh.ring[tid], LineStores{}, emit);
            }
            continue;
        }
        if (valid) size_routed(tv, br, c);
        // ---- place the tile: block scan of response sizes, chained by the look-back; on the host-batch path (chain0) the
        // chunk starts at the same offset mod 16 as its destination in the caller's buffer ----
        const TilePlace t = place_tile(p, tile, c.total_len, sh.warp_sum, sh.tile_base, p.debug_flags & 1u, chain0);
        if (valid) {
            put_offsets(p.out_off, i, p.n, t, c.total_len);
            p.meta[i] = request_status(tv, c) | (c.route << 16);
        }

        // ---- stage 3: emit straight to HBM in 16-byte chunks ----
        if (t.fits && valid && c.total_len) emit_request(tv, br, c, p.out + t.base + t.excl, &sh.ring[tid]);
        // the next iteration's first __syncthreads orders this tile's shared-memory reads before any overwrite
    }
    if (SLOTS) {
        // General pass: the requests the tile loop marked in the length column.  Every CTA rescans the columns of its own
        // tiles (one coalesced 4-byte load per request; the marks were stored by this CTA, so a barrier makes them
        // visible — read past L1, which may hold nothing newer than the launch), gathers the marked indices and serves
        // them 128 at a time.  Nothing of this is in the tile loop: no list, no atomics, no call site.
        __syncthreads();
        uint32_t* const defer = (uint32_t*)in_stage;  // >= 2 T words: the engine never stages less than 16 bytes per request
        for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
            const uint32_t i = tile * T + tid;
            const bool marked = i < p.n && __ldcg(p.out_off + i) == kDeferred;
            if (__syncthreads_or(marked)) {
                if (marked) defer[atomicAdd(&sh.defer_n, 1u)] = i;
                __syncthreads();
                const uint32_t dn = sh.defer_n;
                if (dn >= (uint32_t)T) {
                    general_pass(&p, tv, br, &sh, defer, dn - T, T);
                    __syncthreads();
                    if (tid == 0) sh.defer_n = dn - T;
                    __syncthreads();
                }
            }
        }
        const uint32_t dn = sh.defer_n;
        if (dn) general_pass(&p, tv, br, &sh, defer, 0, dn);
    }
}

}  // namespace gofr
