// serve_device.cuh — per-request device logic of the fused serve kernel.
//
// One thread owns one request.  Everything here is straight-line integer/byte work on generic pointers (the tile's
// request bytes live in shared memory when they fit the staging buffer, in HBM otherwise; the response is written into
// a shared-memory staging tile, or straight to HBM when a tile is too large).  Three stages per request:
//   route_request()  — mux cleanPath + Router.Match (gorilla/mux v1.8.1 semantics; pkg/gofr/http/router.go:14,30-33),
//                      CORS OPTIONS predicate (middleware/cors.go:10-13), handler kind → response program
//   run_prog<false>  — size pass: exact byte length of header block and body
//   run_prog<true>   — emit pass: writes the bytes through the word-stream Writer
// The functions are __host__ __device__ so tests/emu can run the very same code on the CPU per request (test
// infrastructure only; the product has no CPU path).
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/gofr_b200.h"
#include "table_format.h"

// (defaulted here, documented below at size_routed: 1 unless the translation unit says otherwise before including this)
#ifndef GOFR_TU_VALUES
#define GOFR_TU_VALUES 1
#endif

#if defined(__CUDACC__)
#define GOFR_HD __host__ __device__ __forceinline__
#define GOFR_HD_NOINLINE inline __host__ __device__ __noinline__
#else
#define GOFR_HD inline
#define GOFR_HD_NOINLINE inline
struct uint4 { uint32_t x, y, z, w; };  // host build (tests/emu) only
#endif

namespace gofr {

// ---------------------------------------------------------------------------------------------------------------
// bit helpers
// ---------------------------------------------------------------------------------------------------------------

// (hi:lo << sh) >> 32, sh in [0,31]
GOFR_HD uint32_t fsl(uint32_t lo, uint32_t hi, uint32_t sh) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, sh);
#else
    return sh ? (hi << sh) | (lo >> (32 - sh)) : hi;
#endif
}
// low 32 bits of (hi:lo >> sh), sh in [0,31]
GOFR_HD uint32_t fsr(uint32_t lo, uint32_t hi, uint32_t sh) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, sh);
#else
    return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}
GOFR_HD int clz64(uint64_t v) {
#if defined(__CUDA_ARCH__)
    return __clzll((long long)v);
#else
    return v ? __builtin_clzll(v) : 64;
#endif
}

// true if the predicate holds for ANY currently active lane: used so that lanes whose phases differ still take
// flush decisions together (flushing early is harmless, flushing at different times runs the flush code repeatedly)
#if !defined(__CUDACC__)
// host build (tests/emu): on the GPU a lane also flushes whenever ANOTHER lane of its warp needs room, i.e. at any of the
// decision points and in any state; the emulation can replay that (mode 1: always, mode 2: pseudo-randomly)
inline int& emu_any_mode() { static int m = 0; return m; }
inline bool emu_any_extra() {
    static uint32_t x = 0x9E3779B9u;
    if (emu_any_mode() == 1) return true;
    if (emu_any_mode() == 2) { x ^= x << 13; x ^= x >> 17; x ^= x << 5; return (x & 3u) == 0; }
    return false;
}
#endif
GOFR_HD bool warp_any(bool p) {
#if defined(__CUDA_ARCH__)
    return __any_sync(__activemask(), p);
#elif !defined(__CUDACC__)
    return p || emu_any_extra();
#else
    return p;
#endif
}

// ---------------------------------------------------------------------------------------------------------------
// output writer: appends bytes at an arbitrary byte address of the output; it stores whole, aligned 32-byte SECTORS —
// plus the few edge bytes a response shares with its neighbours.  sm_90 has no 256-bit store, so a sector is two 16-byte
// st.global.cs.v4.  When one lane issues both, a warp store touches 32 sectors 528 bytes apart (the config-2 slots) and
// fills half of each.  Storing 1 Mi such slots and nothing else, at full occupancy (scratch/experiments/sector_stores,
// H100 SXM at 400 W; the times rank store patterns, they are not the serve kernel's store cost), took 1.82 ms.  How
// bytes leave is the store policy the Writer is instantiated with (below): SoloStores, the default, stores each lane's
// sector as two back-to-back halves; LineStores (the fast path of the wide slot-layout instance, serve_body.cuh LINES)
// makes the destination alignment a 128-byte line and stores the complete lines of the warp's lanes four per warp store,
// eight lanes per line (0.333 ms for the same slots; lane pairs on 16 whole sectors per warp store 0.599 ms, fully
// coalesced rows 0.175 ms; H100 SXM at 700 W).
//
// Each thread owns a 16-word staging buffer in shared memory, laid out word-major (word k of thread t at
// [k * CTA + t]): whatever word index a lane is at, its bank is its lane id, so accesses never conflict.  The buffer is
// DESTINATION-ALIGNED: word 0 is the first word of the 32-byte sector at `chunk`.
//   produce: bytes are appended as whole words.  `pend` holds the nb (0..3) incomplete bytes in its TOP bytes, so
//            appending a word is one funnel shift + one STS + a pointer bump — no branches, no per-word flush test,
//            and the same code for every lane whatever its phase.  A memory source is streamed with the pending
//            bytes treated as a prefix of the source ("virtual source"): one aligned load + one funnel shift per
//            output word regardless of source and destination alignment.
//   flush:   decoupled from producing — between ops, when at least 8 words wait, whole sectors leave as
//            8 conflict-free LDS + two st.global.cs.v4; no shifting is needed because the buffer is already aligned.
//   edges:   the first sector's leading `lead` bytes and the last sector's tail belong to neighbouring responses
//            written by other threads; only this response's bytes are stored there.
// With LineStores the column holds one 128-byte line plus what is appended before the next flush vote (39 words), and
// its rows are T + 1 words apart: word k of thread t at [k * (T + 1) + t], so the bank of a word is (k + t) mod 32.
// Appends of one word index by the lanes of a warp stay conflict-free, and the eight lanes that load the eight 16-byte
// windows of one line (words 4w + j, w = 0..7) hit eight different banks (line_store_bank, tests/emu).
// ---------------------------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
#ifndef GOFR_RING_STRIDE_BYTES
#define GOFR_RING_STRIDE_BYTES 512u  /* word-major staging: one word of every thread that shares the buffer per row */
#endif
#define GOFR_LINE_STRIDE_BYTES 516u  /* LineStores: one padding word per row */
#else
#define GOFR_RING_STRIDE_BYTES 4u
#define GOFR_LINE_STRIDE_BYTES 4u
#endif
#define GOFR_SOLO_WORDS 16u  /* SoloStores column */
#define GOFR_LINE_WORDS 39u  /* LineStores column: < 32 words before an append of at most 8 */
// Words a caller's staging column must hold.  Device kernels stage only with SoloStores (the wide slot instance sizes its
// LineStores ring itself, serve_body.cuh); the host emulation (tests/emu) runs both policies through one column.
#if defined(__CUDACC__)
#define GOFR_STAGE_WORDS GOFR_SOLO_WORDS
#else
#define GOFR_STAGE_WORDS GOFR_LINE_WORDS
#endif

// ---- explicit address spaces -------------------------------------------------------------------------------------
// The staging buffer, the table's literal pool and (for staged tiles) the request bytes all live in shared memory.
// Going through generic pointers costs 64-bit address arithmetic, window checks and the slower LD.E/ST.E path, so on
// the device they are addressed with 32-bit shared-memory addresses and ld/st.shared; on the host (tests/emu) the
// same code runs on plain pointers.
#if defined(__CUDA_ARCH__)
typedef uint32_t saddr_t;
GOFR_HD saddr_t to_saddr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// Staging buffer accesses are read-after-write on the same addresses: `volatile` keeps them ordered among themselves.
// No "memory" clobber: nothing else ever touches the staging buffer, and a clobber would force every table value to be
// re-read after each store and forbid overlapping the next loads with these stores.
GOFR_HD void stg_st(saddr_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v)); }
GOFR_HD uint32_t stg_ld(saddr_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
// sources are read-only while a response is being written: let the compiler schedule these freely
GOFR_HD uint32_t src_ld(saddr_t a) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
GOFR_HD uint32_t stg_ld8(saddr_t a) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
GOFR_HD uint32_t salign(saddr_t a) { return a & 3u; }
// 16 aligned source bytes (response templates)
GOFR_HD uint4 src_ld128(saddr_t a) {
    uint4 v;
    asm("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
#else
typedef const uint8_t* saddr_t;
GOFR_HD saddr_t to_saddr(const void* p) { return (const uint8_t*)p; }
GOFR_HD void stg_st(saddr_t a, uint32_t v) { *(uint32_t*)a = v; }
GOFR_HD uint32_t stg_ld(saddr_t a) { return *(const uint32_t*)a; }
GOFR_HD uint32_t stg_ld8(saddr_t a) { return *a; }
GOFR_HD uint32_t src_ld(saddr_t a) { return *(const uint32_t*)a; }
GOFR_HD uint32_t salign(saddr_t a) { return (uint32_t)((uintptr_t)a & 3u); }
GOFR_HD uint4 src_ld128(saddr_t a) { uint4 v; memcpy(&v, a, 16); return v; }
#endif

// memory policy of a copy source: SH = shared-memory address, otherwise a generic pointer
template <bool SH> struct SrcMem;
template <> struct SrcMem<true> {
    typedef saddr_t A;
    GOFR_HD static A from(const uint8_t* p) { return to_saddr(p); }
    GOFR_HD static uint32_t ld(A a) { return src_ld(a); }
    GOFR_HD static uint32_t low2(A a) { return salign(a); }
};
template <> struct SrcMem<false> {
    typedef const uint8_t* A;
    GOFR_HD static A from(const uint8_t* p) { return p; }
    GOFR_HD static uint32_t ld(A a) { return *(const uint32_t*)a; }
    GOFR_HD static uint32_t low2(A a) { return (uint32_t)((uintptr_t)a & 3u); }
};

// load k (1..4) bytes at an arbitrary address as the low bytes of a word; reads only words that hold source bytes
GOFR_HD uint32_t load_bytes(const uint8_t* p, uint32_t k) {
    uintptr_t a = (uintptr_t)p;
    const uint32_t* q = (const uint32_t*)(a & ~(uintptr_t)3);
    uint32_t o = (uint32_t)(a & 3);
    uint32_t w0 = q[0];
    uint32_t w1 = o + k > 4 ? q[1] : 0u;
    return fsr(w0, w1, o * 8);
}

// 16 bytes at the 16-byte aligned addr: the one global store of a whole sector half
GOFR_HD void store16(uint8_t* addr, uint32_t v0, uint32_t v1, uint32_t v2, uint32_t v3) {
#if defined(__CUDA_ARCH__)
#if defined(GOFR_EXP_NO_STORE)  /* experiment: the kernel without its global stores (what is left is issue/latency bound) */
    if (v0 == 0x12345678u && v1 == 0x9ABCDEF0u && v2 == 0x0F1E2D3Cu)
#endif
    __stcs((uint4*)addr, make_uint4(v0, v1, v2, v3));
#else
    uint32_t v[4] = {v0, v1, v2, v3};
    memcpy(addr, v, 16);
#endif
}

// Store policies of the Writer: its staging geometry (kStride: bytes between the rows of the column, kWords: words a
// column holds, kLine: the destination alignment in bytes) and how the lanes that run flush, copy and finish_padded take
// a flush decision (vote) and how long a loop over the group runs (round).  kLockstep: every lane of the group makes
// every call of these routines together, also with nothing to store.
//
// SoloStores: each lane on its own, its 32-byte sector as two back-to-back 16-byte stores; a flush decision is taken by
// all active lanes of the warp.
struct SoloStores {
    static constexpr bool kLockstep = false;
    static constexpr uint32_t kStride = GOFR_RING_STRIDE_BYTES, kWords = GOFR_SOLO_WORDS, kLine = 32;
    GOFR_HD bool vote(bool p) const { return warp_any(p); }
    GOFR_HD bool round(bool have) const { return have; }
    // the sector v0..v7 at the 32-byte aligned addr, if `have`
    GOFR_HD void store32(bool have, uint8_t* addr, uint32_t v0, uint32_t v1, uint32_t v2, uint32_t v3, uint32_t v4,
                         uint32_t v5, uint32_t v6, uint32_t v7) const {
        if (have) { store16(addr, v0, v1, v2, v3); store16(addr + 16, v4, v5, v6, v7); }
    }
};
// LineStores (slot layout only: every response starts 16-byte aligned): all 32 lanes of the warp take every decision
// and run every round together — a line needs eight lanes, so a lane with no response to write takes part with an empty
// one (emit_fast, live false).  A flush stores the complete 128-byte lines of all of them in rounds of four: lane group
// g = lane >> 3 takes the g-th remaining lane with a line, and lane t = lane & 7 loads window t of that lane's column and
// stores it, so one warp store is four aligned lines.  `wins` (bit w: window w) says which windows of a line belong to
// the response: the first line skips the previous slot's, the last one ends at the zero-padded end.  On the host
// (tests/emu) lanes run one at a time: a lane stores its own line, and the vote is warp_any's so that the emulation
// replays extra flushes here too.
struct LineStores {
    static constexpr uint32_t wm = 0xFFFFFFFFu;
    static constexpr bool kLockstep = true;
    static constexpr uint32_t kStride = GOFR_LINE_STRIDE_BYTES, kWords = GOFR_LINE_WORDS, kLine = 128;
    static constexpr uint32_t kRowWords = 129;  // T + 1 (serve_body.cuh): the device row of the column
    GOFR_HD bool vote(bool p) const {
#if defined(__CUDA_ARCH__)
        return __any_sync(wm, p);
#else
        return warp_any(p);
#endif
    }
    GOFR_HD bool round(bool have) const {
#if defined(__CUDA_ARCH__)
        return __any_sync(wm, have);
#else
        return have;
#endif
    }
    // ring word that holds word j of window w of the column of thread s
    GOFR_HD static uint32_t window_word(uint32_t s, uint32_t w, uint32_t j) { return (4u * w + j) * kRowWords + s; }
    // store windows `wins` of the line at `line` (128-byte aligned) from the column at col
    GOFR_HD void lines(uint8_t* line, saddr_t col, uint32_t wins) const {
#if defined(__CUDA_ARCH__)
        const uint32_t lane = threadIdx.x & 31u, g = lane >> 3, t = lane & 7u;
        uint32_t rem = __ballot_sync(wm, wins != 0u);
        if (!rem) return;
        __syncwarp(wm);  // the owners' column stores before the other lanes' loads
        do {
            const uint32_t m1 = rem & (rem - 1u), m2 = m1 & (m1 - 1u), m3 = m2 & (m2 - 1u);
            const uint32_t sel = g == 0 ? rem : g == 1 ? m1 : g == 2 ? m2 : m3;
            const uint32_t s = sel ? __ffs(sel) - 1u : lane;
            uint8_t* const a = (uint8_t*)__shfl_sync(wm, (unsigned long long)line, s);
            const uint32_t ws = __shfl_sync(wm, wins, s);
            if (sel && ((ws >> t) & 1u)) {
                const saddr_t rp = col + 4u * (window_word(s, t, 0) - lane);
                store16(a + 16u * t, stg_ld(rp), stg_ld(rp + kStride), stg_ld(rp + 2u * kStride), stg_ld(rp + 3u * kStride));
            }
            rem = m3 & (m3 - 1u);
        } while (rem);
        __syncwarp(wm);  // every load of a column before its owner moves or overwrites words in it
#else
        for (uint32_t t = 0; t < 8; t++)
            if ((wins >> t) & 1u) {
                const saddr_t rp = col + 4u * t * kStride;
                store16(line + 16u * t, stg_ld(rp), stg_ld(rp + kStride), stg_ld(rp + 2u * kStride), stg_ld(rp + 3u * kStride));
            }
#endif
    }
    // Windows [0, nwin) of every lane's template into its slot at dst, straight from the literal pool (tp), except windows
    // [h0, h1), which the lane has staged from row 0 of its column at col (stage_trace_id).  The warp numbers the windows
    // of its 32 responses in request order (an exclusive sum of nwin) and lane L stores windows L, L + 32, ... of that
    // sequence, so consecutive lanes store consecutive windows of a response and one warp store covers the templates of
    // two or three whole responses.  The owner of window g is the lane whose range holds it: g / nwin when every lane has
    // the same count, else a search over the shuffled prefix.  A lane with nothing to write passes nwin 0.  On the host
    // (tests/emu) a lane stores its own windows.
    GOFR_HD void templates(uint8_t* dst, saddr_t tp, uint32_t nwin, uint32_t h0, uint32_t h1, saddr_t col) const {
#if defined(__CUDA_ARCH__)
        const uint32_t lane = threadIdx.x & 31u;
        uint32_t incl = nwin;
#pragma unroll
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(wm, incl, o);
            if (lane >= o) incl += u;
        }
        const uint32_t total = __shfl_sync(wm, incl, 31);
        if (!total) return;
        const uint32_t first = incl - nwin, n0 = __shfl_sync(wm, nwin, 0);
        const bool uniform = __all_sync(wm, nwin == n0);
        const uint32_t rec = first | h0 << 16 | h1 << 24;  // first < 32 * 256; h0 <= h1 <= nwin < 256
        __syncwarp(wm);  // the owners' staged windows before the other lanes' loads
#pragma unroll 1
        for (uint32_t g0 = 0; g0 < total; g0 += 32u) {
            const uint32_t g = g0 + lane;
            const bool have = g < total;
            uint32_t s = 0;
            if (uniform) {
                s = have ? g / n0 : lane;
            } else {
#pragma unroll
                for (uint32_t b = 16; b; b >>= 1)
                    if (__shfl_sync(wm, first, s + b) <= g) s += b;
            }
            const uint32_t r = __shfl_sync(wm, rec, s);
            const saddr_t src = __shfl_sync(wm, tp, s);
            uint8_t* const d = (uint8_t*)__shfl_sync(wm, (unsigned long long)dst, s);
            const uint32_t k = g - (r & 0xFFFFu), k0 = (r >> 16) & 0xFFu, k1 = r >> 24;
            const bool staged = k >= k0 && k < k1;
            const saddr_t rp = staged ? col + 4u * (s - lane) + (k - k0) * 4u * kStride : src + 16u * k;
            const uint32_t st = staged ? kStride : 4u;
            if (have) store16(d + 16u * k, stg_ld(rp), stg_ld(rp + st), stg_ld(rp + 2u * st), stg_ld(rp + 3u * st));
        }
        __syncwarp(wm);  // every load of a column before its owner appends the tail to it
#else
        for (uint32_t k = 0; k < nwin; k++) {
            const bool staged = k >= h0 && k < h1;
            const saddr_t rp = staged ? col + (k - h0) * 4u * kStride : tp + 16u * k;
            const uint32_t st = staged ? kStride : 4u;
            store16(dst + 16u * k, stg_ld(rp), stg_ld(rp + st), stg_ld(rp + 2u * st), stg_ld(rp + 3u * st));
        }
#endif
    }
};

#if !defined(__CUDACC__)
// The host emulation (tests/emu) selects the wide instance's policy by the name of the lane-pair policy LineStores
// replaced, with that policy's lane mask, which lines do not use.
struct PairStores : LineStores {
    explicit PairStores(uint32_t) {}
};
#endif

template <typename P>
struct WriterT {
    static constexpr uint32_t kStride = P::kStride, kWords = P::kWords, kLine = P::kLine;
    uint8_t* chunk;  // kLine-aligned global address that staging word 0 maps to
    saddr_t base;    // this thread's column of the staging buffer
    saddr_t wp;      // base + wl * stride: where the next complete word goes
    uint32_t wl;     // complete words staged (0 .. kWords)
    uint32_t pend, nb;
    uint32_t lead;   // bytes at the start of the first sector (line) owned by the previous response(s)

    GOFR_HD void init(uint8_t* dst, uint32_t* col) {
        uintptr_t x = (uintptr_t)dst;
        chunk = (uint8_t*)(x & ~(uintptr_t)(kLine - 1));
        lead = (uint32_t)(x & (kLine - 1));
        wl = lead >> 2;  // phantom words of the neighbour: never stored
        nb = lead & 3;
        base = to_saddr(col);
        wp = base + wl * kStride;
        pend = 0;
    }
    GOFR_HD uint32_t word(uint32_t k) const { return stg_ld(base + k * kStride); }

    // Write bytes [lo, hi) of the 32-byte sector at addr from the eight staging words at rp: a 16-byte half where one is
    // whole, else words, else single bytes.  Runs twice per response at most (first and last sector), so it is a loop,
    // not unrolled code.
    GOFR_HD static void st8(uint8_t* a, uint32_t v) { *a = (uint8_t)v; }
    GOFR_HD static void st32(uint8_t* a, uint32_t v) { *(uint32_t*)a = v; }
    GOFR_HD static void store_partial(uint8_t* addr, saddr_t rp, uint32_t lo, uint32_t hi) {
        uint32_t b = lo;
#pragma unroll 1
        for (; b < hi && (b & 3u); b++) st8(addr + b, stg_ld8(rp + (b >> 2) * kStride + (b & 3u)));
#pragma unroll 1
        for (; b + 4 <= hi && (b & 15u); b += 4) st32(addr + b, stg_ld(rp + (b >> 2) * kStride));
#pragma unroll 1
        for (; b + 16 <= hi; b += 16) {
            const saddr_t q = rp + (b >> 2) * kStride;
            store16(addr + b, stg_ld(q), stg_ld(q + kStride), stg_ld(q + 2 * kStride),
                    stg_ld(q + 3 * kStride));
        }
#pragma unroll 1
        for (; b + 4 <= hi; b += 4) st32(addr + b, stg_ld(rp + (b >> 2) * kStride));
#pragma unroll 1
        for (; b < hi; b++) st8(addr + b, stg_ld8(rp + (b >> 2) * kStride + (b & 3u)));
    }
    // store every complete sector (LineStores: line), move the (< 8) left-over words to the front
    GOFR_HD void flush(P p = P()) {
        if constexpr (P::kLockstep) {
            // a line is complete at 32 words; a column holds fewer than 40, so there is at most one
            const bool full = wl >= 32u;
            p.lines(chunk, base, full ? (0xFFu << (lead >> 4)) & 0xFFu : 0u);
            if (full) {
                const uint32_t r = wl - 32u;
#pragma unroll
                for (uint32_t j = 0; j < 7; j++)
                    if (r > j) stg_st(base + j * kStride, stg_ld(base + (32u + j) * kStride));
                wl = r;
                wp = base + r * kStride;
                chunk += 128;
                lead = 0;
            }
        } else {
            uint32_t n = wl >> 3;
            saddr_t rp = base;
            if (n && lead) {  // first sector of the response: skip the neighbour's bytes
                store_partial(chunk, rp, lead, 32);
                lead = 0;
                chunk += 32;
                rp += 8 * kStride;
                n--;
            }
#pragma unroll 1
            while (p.round(n != 0)) {
                const bool have = n != 0;
                uint8_t* const at = chunk;
                uint32_t v[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
                if (have) {
#pragma unroll
                    for (uint32_t j = 0; j < 8; j++) v[j] = stg_ld(rp + j * kStride);
                }
                p.store32(have, at, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
                if (have) {
                    chunk += 32;
                    rp += 8 * kStride;
                    n--;
                }
            }
            const uint32_t r = wl & 7;
            if (wl >= 8 && r) {
#pragma unroll
                for (uint32_t j = 0; j < 7; j++)
                    if (r > j) stg_st(base + j * kStride, stg_ld(rp + j * kStride));
            }
            wl = r;
            wp = base + r * kStride;
        }
    }
    // make room for n more words (n <= 8); the decision is taken together by all active lanes
    GOFR_HD void reserve(uint32_t n) {
        if (warp_any(wl + n > kWords)) flush();
    }
    GOFR_HD void store_word(uint32_t x) {
        stg_st(wp, x);
        wp += kStride;
        wl++;
    }
    GOFR_HD void put4(uint32_t v) {
        store_word(fsl(pend, v, nb * 8));
        pend = v;
    }
    // k in 1..3; bytes of v above k are ignored
    GOFR_HD void putk(uint32_t v, uint32_t k) {
        uint32_t c = fsl(pend, v, nb * 8);
        uint32_t t = nb + k;
        if (t >= 4) {
            store_word(c);
            pend = v << (8 * (4 - k));
            nb = t - 4;
        } else {
            pend = c << (8 * (4 - t));
            nb = t;
        }
    }
    GOFR_HD void put(uint32_t v, uint32_t k) {
        if (k == 4) put4(v);
        else if (k) putk(v, k);
    }
    // single bytes from slow paths: room is checked here because those loops are unbounded
    GOFR_HD void put1(uint32_t c);
    GOFR_HD void reserve_out(uint32_t n);
    // one byte from the hot path, where the caller has already made room
    GOFR_HD void putc(uint32_t c) { putk(c, 1); }

    // K consecutive words of a copy: output word i is the unaligned word at Y + 4i (cur holds the aligned word before Y)
    template <typename M, int K>
    GOFR_HD void stream_words(typename M::A& Y, uint32_t& cur, uint32_t sh) {
        uint32_t n[K];
#pragma unroll
        for (int i = 0; i < K; i++) n[i] = M::ld(Y + 4 * i);
#pragma unroll
        for (int i = 0; i < K; i++) stg_st(wp + i * kStride, fsr(i ? n[i - 1] : cur, n[i], sh));
        cur = n[K - 1];
        Y += 4 * K;
        wp += K * kStride;
        wl += K;
    }

    // Append len bytes from memory (any alignment).  With y = src - nb the stream "pending bytes ++ source" is
    // word-aligned with the destination, so output word k is the unaligned word at y + 4k: one aligned load (the
    // previous one is carried) and one funnel shift.  Only word 0 mixes in `pend`.
    // Sources must be readable up to the end of the aligned word following their last byte (literal pool, staged
    // arena and blobs are padded accordingly); no byte before the source is ever read.
    // With LineStores every lane of the write mask makes the call, also with len 0, and takes the flush votes and the
    // long-copy rounds below.
    template <bool SH>
    GOFR_HD void copy(typename SrcMem<SH>::A src, uint32_t len, P p = P()) {
        typedef SrcMem<SH> M;
        if (!P::kLockstep && !len) return;
        const uint32_t yo = (M::low2(src) - nb) & 3u, sh = yo * 8;
        typename M::A Y = src - nb - yo;  // aligned word that holds stream byte 0
        const uint32_t total = nb + len;
        uint32_t nwords = total >> 2;     // 0 when len is 0
        const uint32_t nn = total & 3;
        uint32_t cur = 0u, nxt = 0u, w0 = 0u;
        if (len) {
            // Y[0] holds source bytes iff the source starts inside it
            cur = (yo + nb < 4) ? M::ld(Y) : 0u;
            nxt = (yo + total > 4) ? M::ld(Y + 4) : 0u;  // second word needed only if the data reaches it
            w0 = fsr(cur, nxt, sh);
            if (nb) w0 = (w0 & (0xFFFFFFFFu << (8 * nb))) | (pend >> (8 * (4 - nb)));
        }
        const bool words = nwords != 0;
        if (!words) {  // still inside the same word (or nothing to copy)
            if (len) {
                pend = w0 << (8 * (4 - nn));
                nb = nn;
            }
            if (!P::kLockstep) return;
        }
        // at most 8 words staged from here on: this word + (head <= 7 | a short copy <= 7)
        if (p.vote(wl + 8 > kWords)) flush(p);
        if (words) {
            store_word(w0);
            cur = nxt;
            Y += 8;  // Y now points at the NEXT word to load
            nwords--;
        }
        if constexpr (P::kLockstep) {
            // Long copy: 8 words at a time through the column, a flush vote before each step and after the last one
            if (p.round(nwords >= 8)) {
#pragma unroll 1
                do {
                    if (p.vote(wl + 8 > kWords)) flush(p);
                    if (nwords >= 8) {
                        stream_words<M, 8>(Y, cur, sh);
                        nwords -= 8;
                    }
                } while (p.round(nwords >= 8));
                if (p.vote(wl + 8 > kWords)) flush(p);
            }
        } else if (p.round(nwords >= 8)) {
            if (nwords >= 8) {
                // Long copy.  Head: complete the sector under construction (<= 7 more words), store it; from then on
                // the staging buffer is empty and whole sectors go from registers straight to HBM.
                const uint32_t h = (8u - (wl & 7u)) & 7u;
                if (h & 4u) stream_words<M, 4>(Y, cur, sh);
                if (h & 2u) stream_words<M, 2>(Y, cur, sh);
                if (h & 1u) stream_words<M, 1>(Y, cur, sh);
                nwords -= h;
            }
            flush(p);  // a long copy's wl is a multiple of 8: nothing is left behind
#pragma unroll 1
            while (p.round(nwords >= 8)) {
                const bool have = nwords >= 8;
                uint32_t n0 = 0u, n1 = 0u, n2 = 0u, n3 = 0u, n4 = 0u, n5 = 0u, n6 = 0u, n7 = 0u;
                if (have) {
                    n0 = M::ld(Y); n1 = M::ld(Y + 4); n2 = M::ld(Y + 8); n3 = M::ld(Y + 12);
                    n4 = M::ld(Y + 16); n5 = M::ld(Y + 20); n6 = M::ld(Y + 24); n7 = M::ld(Y + 28);
                }
                p.store32(have, chunk, fsr(cur, n0, sh), fsr(n0, n1, sh), fsr(n1, n2, sh), fsr(n2, n3, sh),
                          fsr(n3, n4, sh), fsr(n4, n5, sh), fsr(n5, n6, sh), fsr(n6, n7, sh));
                if (have) {
                    chunk += 32;
                    cur = n7;
                    Y += 32;
                    nwords -= 8;
                }
            }
        }
        if (!words) return;
        // <= 7 words left: 4 + 2 + 1, each group with its loads issued together and immediate offsets (a word-at-a-time
        // loop spends more on its counters than on the words)
        if (nwords & 4u) stream_words<M, 4>(Y, cur, sh);
        if (nwords & 2u) stream_words<M, 2>(Y, cur, sh);
        if (nwords & 1u) stream_words<M, 1>(Y, cur, sh);
        if (nn) {
            // the partial last word: its bytes may or may not spill into the next aligned word
            nxt = (yo + nn > 4) ? M::ld(Y) : 0u;
            pend = fsr(cur, nxt, sh) << (8 * (4 - nn));
        }
        nb = nn;
    }
    // Slot layout (gofr_serve_device_slots): the response owns its 16-byte aligned slot, so the last 16-byte chunk is
    // stored whole, zero padded — no byte stores, nothing of a neighbour to preserve.  A slot starts either on a sector
    // boundary or in the middle of one (lead 0 or 16); with LineStores at any 16-byte window of a line, and the last line
    // is stored in whole windows up to the padded end.
    GOFR_HD void finish_padded(P p = P()) {
        flush(p);
        const uint32_t end = 4 * wl + nb;  // bytes of the last sector (line) in use, phantom lead included
        const bool some = end > lead;
        if constexpr (P::kLockstep) {
            uint32_t wins = 0u;
            if (some) {
                const uint32_t ew = (end + 15u) >> 4;  // windows in use: 1..8
                if (nb) stg_st(wp, pend >> (8 * (4 - nb)));
#pragma unroll 1
                for (uint32_t k = wl + (nb ? 1u : 0u); k < 4u * ew; k++) stg_st(base + k * kStride, 0u);
                wins = (0xFFu >> (8u - ew)) & (0xFFu << (lead >> 4));
            }
            p.lines(chunk, base, wins);
        } else {
            uint32_t v[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
            if (some) {
                const uint32_t tail = nb ? pend >> (8 * (4 - nb)) : 0u;
#pragma unroll
                for (uint32_t j = 0; j < 8; j++) v[j] = j < wl ? word(j) : (j == wl ? tail : 0u);
                if (lead) store16(chunk + 16, v[4], v[5], v[6], v[7]);  // upper half only: the lower one is the neighbour's
                else if (end > 16) p.store32(true, chunk, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
                else store16(chunk, v[0], v[1], v[2], v[3]);  // the upper half may be the next slot's
            }
        }
    }
    GOFR_HD void finish() {
        flush();
        if (4 * wl + nb > lead) {  // the last, partial sector; wl <= 7 after the flush
            if (nb) stg_st(wp, pend >> (8 * (4 - nb)));
            store_partial(chunk, base, lead, 4 * wl + nb);
        }
    }
};

typedef WriterT<SoloStores> Writer;

// The slow paths (rune-by-rune escapes, Location, Bind errors) share one out-of-line flush: they already work on a
// local-memory copy of the Writer, and inlining the flush into every byte loop made the kernel's code several times
// larger than its instruction cache.
GOFR_HD_NOINLINE void flush_out(Writer* w) { w->flush(); }
template <typename P>
GOFR_HD void WriterT<P>::reserve_out(uint32_t n) {
    if (warp_any(wl + n > GOFR_SOLO_WORDS)) flush_out(this);
}
template <typename P>
GOFR_HD void WriterT<P>::put1(uint32_t c) {
    if (warp_any(wl >= GOFR_SOLO_WORDS - 2)) flush_out(this);
    putk(c, 1);
}

// generic-pointer copy: out-of-line slow paths, file blobs, tiles too large for the shared-memory staging
GOFR_HD_NOINLINE void emit_bytes(Writer& w, const uint8_t* p, uint32_t len) { w.copy<false>(p, len); }

// ---------------------------------------------------------------------------------------------------------------
// encoding/json string contents (Go 1.21, escapeHTML on)
// ---------------------------------------------------------------------------------------------------------------

// 0x80 in every byte lane that needs the slow path: < 0x20, >= 0x80, or one of " & < > backslash
GOFR_HD uint32_t json_special_mask(uint32_t x) {
    uint32_t y = x & 0x7F7F7F7Fu;
    uint32_t ge20 = y + 0x60606060u;                          // bit7 set iff y >= 0x20
    uint32_t qa = ((y | 0x04040404u) ^ 0x26262626u) + 0x7F7F7F7Fu;  // bit7 clear iff y in {0x22 '"', 0x26 '&'}
    uint32_t lg = ((y | 0x02020202u) ^ 0x3E3E3E3Eu) + 0x7F7F7F7Fu;  // bit7 clear iff y in {0x3C '<', 0x3E '>'}
    uint32_t bs = (y ^ 0x5C5C5C5Cu) + 0x7F7F7F7Fu;                  // bit7 clear iff y == 0x5C
    return (~(ge20 & qa & lg & bs) | x) & 0x80808080u;
}
// the same test accumulated over many words: bit 7 of a byte lane of `acc` ends up set iff some word had a special byte
// there (two three-input logic ops per word instead of four; the final `& 0x80808080` is the caller's)
GOFR_HD uint32_t json_special_acc(uint32_t acc, uint32_t x) {
    const uint32_t y = x & 0x7F7F7F7Fu;
    const uint32_t ge20 = y + 0x60606060u;
    const uint32_t qa = ((y | 0x04040404u) ^ 0x26262626u) + 0x7F7F7F7Fu;
    const uint32_t lg = ((y | 0x02020202u) ^ 0x3E3E3E3Eu) + 0x7F7F7F7Fu;
    const uint32_t bs = (y ^ 0x5C5C5C5Cu) + 0x7F7F7F7Fu;
    const uint32_t t = ge20 & qa & lg;   // one LOP3
    acc |= x;                            // bytes >= 0x80 (folds into the next LOP3 on the device)
    return acc | ~(t & bs);              // one LOP3
}

// true if [p, p+len) contains a byte that encoding/json does not copy verbatim
template <bool SH>
GOFR_HD bool json_needs_escape(typename SrcMem<SH>::A p, uint32_t len) {
    typedef SrcMem<SH> M;
    if (!len) return false;
    const uint32_t lead = M::low2(p);
    typename M::A q = p - lead;
    const uint32_t total = lead + len;      // bytes from q to the end of the string
    const uint32_t last = (total - 1) >> 2; // index of the word holding the last byte
    const uint32_t keep = total & 3;        // valid bytes in that word (0 = all four)
    // bytes outside the string are replaced by 'a' so they can never flag
    uint32_t x = M::ld(q);
    if (lead) x = (x & (0xFFFFFFFFu << (8 * lead))) | (0x61616161u >> (8 * (4 - lead)));
    if (last == 0) {
        if (keep) x = (x & (0xFFFFFFFFu >> (8 * (4 - keep)))) | (0x61616161u << (8 * keep));
        return json_special_mask(x) != 0;
    }
    uint32_t acc = json_special_acc(0u, x);
    uint32_t i = 1;
#pragma unroll 1
    for (; i + 4 <= last; i += 4) {  // four words per trip: the loads go out together
        const uint32_t a = M::ld(q + 4 * i), b = M::ld(q + 4 * i + 4), c = M::ld(q + 4 * i + 8), d = M::ld(q + 4 * i + 12);
        acc = json_special_acc(json_special_acc(json_special_acc(json_special_acc(acc, a), b), c), d);
    }
#pragma unroll 1
    for (; i < last; i++) acc = json_special_acc(acc, M::ld(q + 4 * i));
    x = M::ld(q + 4 * last);
    if (keep) x = (x & (0xFFFFFFFFu >> (8 * (4 - keep)))) | (0x61616161u << (8 * keep));
    return (json_special_acc(acc, x) & 0x80808080u) != 0;
}

// Go utf8.DecodeRune acceptance on a plain byte range: length of the well-formed sequence at p (2..4) or 0.
GOFR_HD uint32_t utf8_len_at(const uint8_t* p, uint32_t n) {
    uint32_t a = p[0];
    uint32_t len = (a >= 0xC2 && a <= 0xDF) ? 2u : (a >= 0xE0 && a <= 0xEF) ? 3u : (a >= 0xF0 && a <= 0xF4) ? 4u : 0u;
    if (!len || n < len) return 0;
    uint32_t lo = a == 0xE0 ? 0xA0u : a == 0xF0 ? 0x90u : 0x80u;
    uint32_t hi = a == 0xED ? 0x9Fu : a == 0xF4 ? 0x8Fu : 0xBFu;
    uint32_t b = p[1];
    if (b < lo || b > hi) return 0;
    for (uint32_t k = 2; k < len; k++)
        if ((p[k] & 0xC0) != 0x80) return 0;
    return len;
}

GOFR_HD uint32_t hex_lc(uint32_t v) { return v < 10 ? '0' + v : 'a' + v - 10; }

// Slow path: escape [p, p+len) rune by rune.  EMIT=false only counts.  Kept out of line: it is rare and large, and
// the kernel is instruction-cache sensitive.
template <bool EMIT>
GOFR_HD_NOINLINE uint32_t json_escape_slow(Writer* w, const uint8_t* p, uint32_t len) {
    uint32_t out = 0;
    for (uint32_t i = 0; i < len;) {
        if (EMIT) w->reserve_out(4);
        uint32_t c = p[i];
        if (c < 0x80) {
            if (c >= 0x20 && c != '"' && c != '\\' && c != '<' && c != '>' && c != '&') {
                if (EMIT) w->put1(c);
                out += 1;
            } else if (c == '"' || c == '\\' || c == '\n' || c == '\r' || c == '\t') {
                uint32_t e = c == '\n' ? 'n' : c == '\r' ? 'r' : c == '\t' ? 't' : c;
                if (EMIT) w->putk('\\' | e << 8, 2);
                out += 2;
            } else {
                if (EMIT) { w->put4('\\' | 'u' << 8 | '0' << 16 | '0' << 24); w->putk(hex_lc(c >> 4) | hex_lc(c & 15) << 8, 2); }
                out += 6;
            }
            i++;
            continue;
        }
        uint32_t L = utf8_len_at(p + i, len - i);
        if (L == 0) {
            if (EMIT) { w->put4('\\' | 'u' << 8 | 'f' << 16 | 'f' << 24); w->putk('f' | 'd' << 8, 2); }
            out += 6;
            i++;
        } else if (L == 3 && c == 0xE2 && p[i + 1] == 0x80 && (p[i + 2] == 0xA8 || p[i + 2] == 0xA9)) {
            if (EMIT) { w->put4('\\' | 'u' << 8 | '2' << 16 | '0' << 24); w->putk('2' | (p[i + 2] == 0xA8 ? '8' : '9') << 8, 2); }
            out += 6;
            i += 3;
        } else {
            if (EMIT) for (uint32_t k = 0; k < L; k++) w->put1(p[i + k]);
            out += L;
            i += L;
        }
    }
    return out;
}

// ---------------------------------------------------------------------------------------------------------------
// integers (strconv.AppendInt base 10)
// ---------------------------------------------------------------------------------------------------------------

GOFR_HD uint32_t ndigits_u32_lt1e8(uint32_t v) {
    return v < 10000u ? (v < 100u ? (v < 10u ? 1u : 2u) : (v < 1000u ? 3u : 4u))
                      : (v < 1000000u ? (v < 100000u ? 5u : 6u) : (v < 10000000u ? 7u : 8u));
}
GOFR_HD uint32_t ndigits_u64(uint64_t v) {
    if (v < 100000000ull) return ndigits_u32_lt1e8((uint32_t)v);
    if (v < 10000000000000000ull) return 8 + ndigits_u32_lt1e8((uint32_t)(v / 100000000ull));
    return 16 + ndigits_u32_lt1e8((uint32_t)(v / 10000000000000000ull));
}

// four decimal digits of q (< 10000) as ASCII, most significant digit in the lowest byte
GOFR_HD uint32_t ascii4(uint32_t q) {
    uint32_t hi = q / 100, lo = q - hi * 100;
    uint32_t a = hi / 10, b = hi - a * 10, c = lo / 10, d = lo - c * 10;
    return (a | b << 8 | c << 16 | d << 24) + 0x30303030u;
}

// v < 10^8 with nd digits (nd = 1..8): at most two four-digit groups — what Content-Length, counters and most ids need
template <typename W>
GOFR_HD void emit_small_digits(W* w, uint32_t v, uint32_t nd) {
    const uint32_t hi = v / 10000u, lo = v - hi * 10000u;
    const uint32_t wlo = ascii4(lo);
    if (nd <= 4) {
        if (nd == 4) w->put4(wlo); else w->putk(wlo >> (8 * (4 - nd)), nd);
        return;
    }
    const uint32_t whi = ascii4(hi), part = nd - 4;
    if (part == 4) w->put4(whi); else w->putk(whi >> (8 * (4 - part)), part);
    w->put4(wlo);
}

// (WT: the Writer instance; the size pass passes a null Writer*)
template <typename X> struct NoDeduce { typedef X T; };
template <bool EMIT, typename WT = Writer>
GOFR_HD uint32_t emit_i64(typename NoDeduce<WT>::T* w, int64_t sv) {
    uint64_t v = sv < 0 ? (uint64_t)0 - (uint64_t)sv : (uint64_t)sv;
    uint32_t nd = ndigits_u64(v);
    uint32_t total = nd + (sv < 0 ? 1u : 0u);
    if (!EMIT) return total;
    if (sv < 0) w->putc('-');
    if (v < 100000000ull) { emit_small_digits(w, (uint32_t)v, nd); return total; }
    // zero-padded 20 digits as five words W[0..4], W[0] most significant
    uint32_t W[5];
    uint64_t top = v / 10000000000000000ull;           // < 1845
    uint64_t rest = v - top * 10000000000000000ull;    // < 1e16
    uint32_t mid = (uint32_t)(rest / 100000000ull), low = (uint32_t)(rest - (uint64_t)mid * 100000000ull);
    W[0] = ascii4((uint32_t)top);
    uint32_t mh = mid / 10000, ml = mid - mh * 10000, lh = low / 10000, ll = low - lh * 10000;
    W[1] = ascii4(mh); W[2] = ascii4(ml); W[3] = ascii4(lh); W[4] = ascii4(ll);
    uint32_t skip = 20 - nd;  // leading zeros to drop
    uint32_t wi = skip >> 2, part = 4 - (skip & 3);
#pragma unroll
    for (uint32_t k = 0; k < 5; k++) {
        if (k == wi) { if (part == 4) w->put4(W[k]); else w->putk(W[k] >> (8 * (4 - part)), part); }
        else if (k > wi) w->put4(W[k]);
    }
    return total;
}

template <bool EMIT, typename WT = Writer>
GOFR_HD uint32_t emit_u32(typename NoDeduce<WT>::T* w, uint32_t v) {
    uint32_t nd = v < 10 ? 1 : v < 100 ? 2 : v < 1000 ? 3 : v < 10000 ? 4 : v < 100000 ? 5 : v < 1000000 ? 6
                : v < 10000000 ? 7 : v < 100000000 ? 8 : v < 1000000000 ? 9 : 10;
    if (!EMIT) return nd;
    if (v < 100000000u) { emit_small_digits(w, v, nd); return nd; }
    uint32_t hi = v / 100000000u, rest = v - hi * 100000000u;
    uint32_t W[3] = {ascii4(hi), ascii4(rest / 10000), ascii4(rest % 10000)};
    uint32_t skip = 12 - nd, wi = skip >> 2, part = 4 - (skip & 3);
#pragma unroll
    for (uint32_t k = 0; k < 3; k++) {
        if (k == wi) { if (part == 4) w->put4(W[k]); else w->putk(W[k] >> (8 * (4 - part)), part); }
        else if (k > wi) w->put4(W[k]);
    }
    return nd;
}

// 4 id bytes → 8 lower-case hex chars (two words), byte order preserved
GOFR_HD void hex8(uint32_t x, uint32_t& w0, uint32_t& w1) {
    // nibble spread: byte b → (b >> 4) in one lane, (b & 15) in the next
    uint32_t b0 = x & 0xFF, b1 = (x >> 8) & 0xFF, b2 = (x >> 16) & 0xFF, b3 = x >> 24;
    uint32_t n0 = (b0 >> 4) | (b0 & 15) << 8 | (b1 >> 4) << 16 | (b1 & 15) << 24;
    uint32_t n1 = (b2 >> 4) | (b2 & 15) << 8 | (b3 >> 4) << 16 | (b3 & 15) << 24;
    // digit → '0'+d, or 'a'+d-10 when d > 9: add 39 where (d + 6) carries into bit 4
    uint32_t c0 = ((n0 + 0x06060606u) >> 4) & 0x01010101u, c1 = ((n1 + 0x06060606u) >> 4) & 0x01010101u;
    w0 = n0 + 0x30303030u + c0 * 39u;
    w1 = n1 + 0x30303030u + c1 * 39u;
}

// ---------------------------------------------------------------------------------------------------------------
// table view (pointers into the shared-memory copy of the image)
// ---------------------------------------------------------------------------------------------------------------
struct TableView {
    // Only two pointers are carried (the tile loop is register bound): every section is located through the header's
    // offsets when it is needed — a shared-memory load each, issued rarely.
    const uint8_t* base;  // hot part (shared memory on the device)
    const uint8_t* cold;  // file blobs (HBM)

    GOFR_HD void bind(const uint8_t* hot, const uint8_t* image_global) {
        base = hot;
        cold = image_global + ((const ImageHeader*)hot)->cold_off;
    }
    GOFR_HD const ImageHeader* hdr() const { return (const ImageHeader*)base; }
    GOFR_HD const RouteRec* routes() const { return (const RouteRec*)(base + hdr()->routes_off); }
    GOFR_HD const PieceRec* pieces() const { return (const PieceRec*)(base + hdr()->pieces_off); }
    GOFR_HD const ProgRec* progs() const { return (const ProgRec*)(base + hdr()->progs_off); }
    GOFR_HD const Op* ops() const { return (const Op*)(base + hdr()->ops_off); }
    GOFR_HD const SchemaRec* schemas() const { return (const SchemaRec*)(base + hdr()->schemas_off); }
    GOFR_HD const uint8_t* lits() const { return base + hdr()->lits_off; }
    GOFR_HD const uint16_t* hash_tab() const { return (const uint16_t*)(base + hdr()->hash_off); }
    GOFR_HD const uint16_t* tmpl_list() const { return (const uint16_t*)(base + hdr()->tmpl_off); }
    GOFR_HD const uint16_t* thash_tab() const { return (const uint16_t*)(base + hdr()->thash_off); }
    GOFR_HD const uint32_t* tmpl_keys() const { return (const uint32_t*)(base + hdr()->tmplkey_off); }
    GOFR_HD const uint16_t* last_method() const { return (const uint16_t*)(base + hdr()->last_method_off); }
    GOFR_HD const FastRec* fast() const { return (const FastRec*)(base + hdr()->fast_off); }
    GOFR_HD const uint16_t* rawprogs() const { return (const uint16_t*)(base + hdr()->rawprog_off); }
    GOFR_HD const uint32_t* lit_words(uint32_t off) const { return (const uint32_t*)(lits() + off); }
    GOFR_HD const uint8_t* lit_bytes(uint32_t off) const { return lits() + off; }
};

// Per-launch arrays a request reaches through its index (kernel parameters: they live in uniform registers)
struct BatchRefs {
    const uint8_t* ids;        // trace ids, 16 bytes per request
    uint32_t* bind_scratch;    // Bind span rows (bind_device.cuh), bind_row_words words per request
    uint32_t bind_row_words;
};

// ---------------------------------------------------------------------------------------------------------------
// per-request context
// ---------------------------------------------------------------------------------------------------------------
struct ReqCtx {
    const uint8_t* path;   // URL.Path; the query follows it, the data section starts at path + data_off
    uint32_t path_len, query_len, data_len, data_off;
    uint32_t mflags;       // method | flags << 8 | staged << 16  (staged: request bytes live in shared memory)
    uint32_t index;        // request index in the batch (trace id, Bind scratch row)
    uint32_t prog;         // program index, 0xFFFF = nothing to emit (GOFR_H_HOST)
    uint32_t route;        // matched route or GOFR_ROUTE_NONE
    uint32_t pv_off, pv_len, pv_flags;  // query value span; flags bit0 found&non-empty, bit1 needs decode/escape
    uint32_t body_len, total_len;
    uint32_t slow_mask;    // bit k: k-th OP_STR of the program needs the slow escape path
    uint32_t def_off, def_len;  // OP_PARAM default (pre-escaped literal)
    uint32_t str_base;     // fast path: byte offset of the row's string area inside the data section (size_fast)

    GOFR_HD const uint8_t* query() const { return path + path_len; }
    GOFR_HD const uint8_t* data() const { return path + data_off; }
    GOFR_HD uint32_t method() const { return mflags & 0xFFu; }
    GOFR_HD uint32_t flags() const { return (mflags >> 8) & 0xFFu; }
    GOFR_HD bool staged() const { return (mflags >> 16) & 1u; }
    GOFR_HD bool fast() const { return (mflags >> 17) & 1u; }  // sized by size_fast: emit_fast may write it
    GOFR_HD void set(const uint8_t* arena_base, uint32_t arena_off, uint32_t pl, uint32_t ql, uint32_t dl, uint32_t method_,
                     uint32_t flags_, bool staged_, uint32_t idx) {
        path = arena_base + arena_off;
        path_len = pl; query_len = ql; data_len = dl;
        data_off = ((arena_off + pl + ql + 3u) & ~3u) - arena_off;
        mflags = method_ | flags_ << 8 | (staged_ ? 1u << 16 : 0u);
        index = idx;
        prog = 0xFFFF; route = GOFR_ROUTE_NONE;
        pv_off = pv_len = pv_flags = 0;
        body_len = total_len = 0; slow_mask = 0; def_off = def_len = 0; str_base = 0;
    }
    GOFR_HD uint32_t* brow(const BatchRefs& br) const { return br.bind_scratch + (size_t)index * br.bind_row_words; }
};

// ---------------------------------------------------------------------------------------------------------------
// mux cleanPath
// ---------------------------------------------------------------------------------------------------------------

// cleanPath(p) == p  ⇔  p starts with '/', has no empty / "." / ".." segment (a single trailing slash is kept)
GOFR_HD bool path_is_clean(const uint8_t* p, uint32_t n) {
    if (n == 0 || p[0] != '/') return false;
    uint32_t i = 1;
    while (i < n) {
        uint32_t j = i;
        while (j < n && p[j] != '/') j++;
        uint32_t len = j - i;
        if (len == 0) return false;
        if (p[i] == '.' && (len == 1 || (len == 2 && p[i + 1] == '.'))) return false;
        i = j + 1;
    }
    return true;
}

GOFR_HD bool url_path_keep(uint32_t c) {
    return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '-' || c == '_' ||
           c == '.' || c == '~' || c == '$' || c == '&' || c == '+' || c == ',' || c == '/' || c == ':' || c == ';' ||
           c == '=' || c == '@';
}
GOFR_HD uint32_t hex_uc(uint32_t v) { return v < 10 ? '0' + v : 'A' + v - 10; }

template <bool EMIT>
GOFR_HD uint32_t put_url_escaped(Writer* w, uint32_t c) {
    if (url_path_keep(c)) { if (EMIT) w->put1(c); return 1; }
    if (EMIT) { w->reserve_out(2); w->putk('%' | hex_uc(c >> 4) << 8 | hex_uc(c & 15) << 16, 3); }
    return 3;
}

// Location of the 301: url.String() with Path = cleanPath(path) → escape(path, encodePath) + "?" + RawQuery.
// path.Clean's stack is replayed per segment: a normal segment survives iff no later ".." pops it.  Quadratic in the
// segment count, but only requests that are being redirected come here.
template <bool EMIT>
GOFR_HD_NOINLINE uint32_t emit_location(Writer* w, const ReqCtx c) {
    const uint8_t* p = c.path;
    uint32_t n = c.path_len;
    uint32_t out = 0;
    if (EMIT) w->put1('/');
    out += 1;
    uint32_t i = (n && p[0] == '/') ? 1 : 0;  // mux prepends '/' when missing
    bool any = false;
    while (i < n) {
        uint32_t j = i;
        while (j < n && p[j] != '/') j++;
        uint32_t len = j - i;
        bool dot = len == 1 && p[i] == '.';
        bool dotdot = len == 2 && p[i] == '.' && p[i + 1] == '.';
        if (len && !dot && !dotdot) {
            // survives?
            int depth = 1;
            uint32_t a = j < n ? j + 1 : n;
            while (a < n && depth > 0) {
                uint32_t b = a;
                while (b < n && p[b] != '/') b++;
                uint32_t l2 = b - a;
                if (l2 == 2 && p[a] == '.' && p[a + 1] == '.') depth--;
                else if (l2 && !(l2 == 1 && p[a] == '.')) depth++;
                a = b < n ? b + 1 : n;
            }
            if (depth > 0) {
                if (any) { if (EMIT) w->put1('/'); out += 1; }
                for (uint32_t k = i; k < j; k++) out += put_url_escaped<EMIT>(w, p[k]);
                any = true;
            }
        }
        i = j < n ? j + 1 : n;
    }
    // "put the trailing slash back if necessary": original ends in '/' and the cleaned path is not "/"
    if (n && p[n - 1] == '/' && any) { if (EMIT) w->put1('/'); out += 1; }
    if (c.query_len || (c.flags() & GOFR_REQ_FORCE_QUERY)) {
        if (EMIT) { w->put1('?'); emit_bytes(*w, c.query(), c.query_len); }
        out += 1 + c.query_len;
    }
    return out;
}

// ---------------------------------------------------------------------------------------------------------------
// route matching
// ---------------------------------------------------------------------------------------------------------------

GOFR_HD bool cls_has(const uint32_t* cls, uint32_t c) { return (cls[c >> 5] >> (c & 31)) & 1u; }

GOFR_HD bool bytes_equal(const uint8_t* a, const uint8_t* b, uint32_t n) {
    for (uint32_t i = 0; i < n; i++)
        if (a[i] != b[i]) return false;
    return true;
}

// both 4-byte aligned
GOFR_HD bool words_equal(const uint32_t* a, const uint32_t* b, uint32_t n) {
    uint32_t nw = n >> 2, diff = 0;
    for (uint32_t i = 0; i < nw; i++) diff |= a[i] ^ b[i];
    uint32_t r = n & 3;
    if (r) diff |= (a[nw] ^ b[nw]) & (0xFFFFFFFFu >> (8 * (4 - r)));
    return diff == 0;
}

// Anchored leftmost-first match of lit0 atom0 lit1 atom1 ... litN [$]: greedy atoms (a character class repeated
// min_rep..max_rep times) with backtracking — what Go's regexp reports for the regexp mux builds from a path template
// whose variables are concatenations of quantified classes (table_build.cpp parse_var_regexp).  A variable is one atom
// or several consecutive ones (PieceRec::var_idx / var_flags); its span runs from its first atom to its last.
// want_var >= 0: also report the span captured by that VARIABLE (mux.Vars, template order) in span_out[0..1] = (offset,
// length); want_var == -2: report every variable, span_out[2v], span_out[2v + 1] for variable v (other entries untouched)
GOFR_HD_NOINLINE bool template_match(const TableView tv, const RouteRec R, const uint8_t* p, uint32_t n, int want_var = -1,
                                     uint32_t* span_out = nullptr) {
    const PieceRec* pc = tv.pieces() + R.first_piece;
    uint32_t np = R.n_pieces;
    bool prefix = R.flags & RF_PREFIX;
    uint32_t start[kMaxPieces + 1], take[kMaxPieces + 1];
    uint32_t k = 0, pos = 0;
    for (;;) {
        // literal k at pos
        bool ok = n - pos >= pc[k].lit_len && bytes_equal(p + pos, tv.lit_bytes(pc[k].lit_off), pc[k].lit_len);
        if (ok) {
            pos += pc[k].lit_len;
            if (!pc[k].has_var) {
                if (prefix || pos == n) {
                    if (want_var != -1) {
                        uint32_t vs = 0;
                        for (uint32_t j = 0; j < k; j++) {
                            if (pc[j].var_flags & PV_FIRST) vs = start[j];
                            if (!(pc[j].var_flags & PV_LAST)) continue;
                            const uint32_t v = pc[j].var_idx, len = start[j] + take[j] - vs;
                            if (want_var == (int)v) { span_out[0] = vs; span_out[1] = len; }
                            if (want_var == -2 && v < (uint32_t)kMaxVars) { span_out[2 * v] = vs; span_out[2 * v + 1] = len; }
                        }
                    }
                    return true;
                }
                ok = false;
            } else {
                const uint32_t cap = pc[k].max_rep ? pc[k].max_rep : 0xFFFFFFFFu;
                uint32_t run = 0;
                while (pos + run < n && run < cap && cls_has(pc[k].cls, p[pos + run])) run++;
                if (run >= pc[k].min_rep) {
                    start[k] = pos;
                    take[k] = run;
                    pos += run;
                    k++;
                    if (k >= np) return prefix || pos == n;  // defensive: templates always end with a literal piece
                    continue;
                }
                ok = false;
            }
        }
        // backtrack: shorten the most recent atom that can still give a byte back
        for (;;) {
            if (k == 0) return false;
            k--;
            if (take[k] > pc[k].min_rep) {
                take[k]--;
                pos = start[k] + take[k];
                k++;
                break;
            }
        }
    }
}

GOFR_HD bool route_path_ok(const TableView& tv, const RouteRec& R, const uint8_t* p, uint32_t n) {
    if (R.flags & RF_LITERAL) {
        if (n != R.lit_len) return false;
        if (((uintptr_t)p & 3) == 0) return words_equal((const uint32_t*)p, tv.lit_words(R.lit_off), n);
        return bytes_equal(p, tv.lit_bytes(R.lit_off), n);
    }
    return template_match(tv, R, p, n);
}

// Router.Match over routes in registration order with mux v1.8.1's ErrMethodMismatch bookkeeping.
// Returns route index, or -1 (no route: 404) / -2 (405).  Reference formulation: every route is evaluated.
GOFR_HD_NOINLINE int mux_match_linear(const TableView tv, uint32_t method, const uint8_t* p, uint32_t n) {
    bool mismatch = false;
    uint32_t nr = tv.hdr()->n_routes;
    for (uint32_t r = 0; r < nr; r++) {
        const RouteRec& R = tv.routes()[r];
        if (R.flags & RF_DEAD) continue;
        bool has_m = R.method != GOFR_M_ANY;
        bool m_ok = !has_m || (R.method == method && method != GOFR_M_OTHER);
        // evaluation order inside Route.Match: method matcher, then path matcher; any matcher that succeeds clears
        // a stale ErrMethodMismatch; a failing path matcher returns without touching it
        if (has_m && m_ok) mismatch = false;
        bool p_ok = route_path_ok(tv, R, p, n);
        if (!p_ok) continue;
        mismatch = false;
        if (!m_ok) { mismatch = true; continue; }
        return (int)r;
    }
    return mismatch ? -2 : -1;
}

// Same result, evaluating only the routes whose path matcher can succeed: the literal routes in hash(path)'s bucket
// and the template / prefix routes, merged in registration order.  Skipped routes have a failing path matcher, so
// their only possible effect is a succeeding METHOD matcher clearing a stale ErrMethodMismatch; that is recovered at
// the end from last_method[] (index of the last live route registered for the request's method).
GOFR_HD int mux_match(const TableView& tv, uint32_t method, const uint8_t* p, uint32_t n) {
    if (((uintptr_t)p & 3) != 0) return mux_match_linear(tv, method, p, n);
    const uint32_t* pw = (const uint32_t*)p;
    uint32_t h = n, nw = n >> 2, r4 = n & 3;
    for (uint32_t i = 0; i < nw; i++) h = path_hash_step(h, pw[i]);
    if (r4) h = path_hash_step(h, pw[nw] & (0xFFFFFFFFu >> (8 * (4 - r4))));
    uint32_t lit = n ? tv.hash_tab()[h >> (32 - tv.hdr()->hash_bits)] : 0xFFFFu;
    uint32_t ti = 0, nt = tv.hdr()->n_tmpl;
    // the path's first eight bytes, zero beyond its end: a template whose leading literal bytes differ cannot match
    const uint32_t w0 = n >= 4 ? pw[0] : (n ? pw[0] & (0xFFFFFFFFu >> (8 * (4 - n))) : 0u);
    const uint32_t w1 = n >= 8 ? pw[1] : (n > 4 ? pw[1] & (0xFFFFFFFFu >> (8 * (8 - n))) : 0u);
    // templates with a leading literal of >= 8 bytes hang off a hash of those bytes
    uint32_t key = n >= 8 ? tv.thash_tab()[path_hash_step(path_hash_step(8u, w0), w1) >> (32 - tv.hdr()->thash_bits)] : 0xFFFFu;
    int a_last = -1;
    for (;;) {
        // three sources, each in registration order: the literal chain, the keyed-template chain, the short templates
        const uint32_t t = ti < nt ? tv.tmpl_list()[ti] : 0xFFFFu;
        uint32_t r = lit < t ? lit : t;
        r = key < r ? key : r;
        if (r == 0xFFFFu) break;
        const RouteRec& R = tv.routes()[r];
        bool p_ok;
        if (r == lit) {
            lit = R.next_lit;
            p_ok = n == R.lit_len && words_equal(pw, tv.lit_words(R.lit_off), n);
        } else if (r == key) {
            key = R.next_lit;
            p_ok = template_match(tv, R, p, n);  // a different template of the same bucket fails on its first literal
        } else {
            const uint32_t* k4 = tv.tmpl_keys() + 4 * ti;
            ti++;
            p_ok = (((w0 ^ k4[0]) & k4[2]) | ((w1 ^ k4[1]) & k4[3])) == 0 && template_match(tv, R, p, n);
        }
        if (!p_ok) continue;
        bool m_ok = R.method == GOFR_M_ANY || (R.method == method && method != GOFR_M_OTHER);
        if (m_ok) return (int)r;
        a_last = (int)r;
    }
    if (a_last < 0) return -1;
    int lm = method < 16 && method != GOFR_M_OTHER ? (int)tv.last_method()[method] - 1 : -1;
    return lm > a_last ? -1 : -2;
}

// ---------------------------------------------------------------------------------------------------------------
// query parameter: req.URL.Query().Get(key)  (pkg/gofr/http/request.go:28-30 → url.ParseQuery)
// ---------------------------------------------------------------------------------------------------------------

GOFR_HD int hexval(uint32_t c) {
    if (c >= '0' && c <= '9') return (int)c - '0';
    if (c >= 'a' && c <= 'f') return (int)c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return (int)c - 'A' + 10;
    return -1;
}

// does QueryUnescape(raw[0..n)) succeed and equal key?   (an invalid %-escape drops the pair)
GOFR_HD bool query_key_equals(const uint8_t* raw, uint32_t n, const uint8_t* key, uint32_t kn) {
    uint32_t j = 0;
    bool eq = true;
    for (uint32_t i = 0; i < n;) {
        uint32_t c = raw[i];
        if (c == '%') {
            if (i + 2 >= n) return false;
            int h = hexval(raw[i + 1]), l = hexval(raw[i + 2]);
            if (h < 0 || l < 0) return false;
            c = (uint32_t)(h << 4 | l);
            i += 3;
        } else {
            if (c == '+') c = ' ';
            i++;
        }
        if (j >= kn || key[j] != c) eq = false;
        j++;
    }
    return eq && j == kn;
}

// bit0: all %-escapes valid; bit1: contains '%' or '+' or a byte encoding/json would not copy verbatim
GOFR_HD uint32_t query_value_scan(const uint8_t* v, uint32_t n) {
    uint32_t special = 0;
    for (uint32_t i = 0; i < n;) {
        uint32_t c = v[i];
        if (c == '%') {
            if (i + 2 >= n || hexval(v[i + 1]) < 0 || hexval(v[i + 2]) < 0) return 0;
            special = 2;
            i += 3;
            continue;
        }
        if (c == '+' || c < 0x20 || c >= 0x80 || c == '"' || c == '\\' || c == '<' || c == '>' || c == '&') special = 2;
        i++;
    }
    return 1 | special;
}

struct ParamSpan { uint32_t off, len, flags; };
GOFR_HD_NOINLINE ParamSpan find_param(const uint8_t* q, uint32_t qn, const uint8_t* key, uint32_t kn) {
    ParamSpan r = {0, 0, 0};
    uint32_t i = 0;
    while (i < qn) {
        uint32_t j = i, eq = 0xFFFFFFFFu;
        bool semi = false;
        while (j < qn && q[j] != '&') {
            uint32_t ch = q[j];
            if (ch == ';') semi = true;
            if (ch == '=' && eq == 0xFFFFFFFFu) eq = j;
            j++;
        }
        uint32_t ps = i, pe = j;
        i = j < qn ? j + 1 : j;
        if (semi || pe == ps) continue;
        uint32_t kend = eq == 0xFFFFFFFFu ? pe : eq;
        if (!query_key_equals(q + ps, kend - ps, key, kn)) continue;
        uint32_t vs = eq == 0xFFFFFFFFu ? pe : eq + 1;
        uint32_t f = query_value_scan(q + vs, pe - vs);
        if (!(f & 1)) continue;
        // first successfully parsed pair for this key decides; an empty value makes the handler use its default
        if (pe > vs) { r.off = vs; r.len = pe - vs; r.flags = 1 | (f & 2); }
        return r;
    }
    return r;
}

// QueryUnescape + encoding/json escape of the value, rune by rune over the DECODED bytes
template <bool EMIT>
GOFR_HD_NOINLINE uint32_t emit_param_slow(Writer* w, const uint8_t* v, uint32_t n) {
    uint32_t out = 0;
    uint32_t i = 0;
    // decode one byte at raw position i → (byte, next position)
    auto dec = [&](uint32_t at, uint32_t& next) -> uint32_t {
        uint32_t c = v[at];
        if (c == '%') { next = at + 3; return (uint32_t)(hexval(v[at + 1]) << 4 | hexval(v[at + 2])); }
        next = at + 1;
        return c == '+' ? ' ' : c;
    };
    while (i < n) {
        uint32_t nx;
        uint32_t c = dec(i, nx);
        if (c < 0x80) {
            uint8_t one = (uint8_t)c;
            out += json_escape_slow<EMIT>(w, &one, 1);
            i = nx;
            continue;
        }
        // gather up to 4 decoded bytes to validate the UTF-8 sequence
        uint8_t buf[4];
        uint32_t pos[5];
        uint32_t cnt = 0, at = i;
        while (cnt < 4 && at < n) { uint32_t nn; buf[cnt] = (uint8_t)dec(at, nn); pos[cnt] = at; at = nn; cnt++; }
        pos[cnt] = at;
        uint32_t L = utf8_len_at(buf, cnt);
        if (L == 0) { out += json_escape_slow<EMIT>(w, buf, 1); i = pos[1]; }
        else { out += json_escape_slow<EMIT>(w, buf, L); i = pos[L]; }
    }
    return out;
}

// Bind (bind_device.cuh)
template <bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD_NOINLINE bool bind_request(const TableView tv, uint32_t schema_idx, const uint8_t* body, uint32_t n, uint32_t* row);
template <bool EMIT> GOFR_HD_NOINLINE uint32_t bind_string_slow(Writer* w, const uint8_t* s, uint32_t len);
template <bool EMIT, bool RAW>
GOFR_HD_NOINLINE uint32_t emit_bind_error(Writer* w, const TableView tv, uint32_t schema_idx, const uint8_t* body, const uint32_t* row);

// ---------------------------------------------------------------------------------------------------------------
// stage 1: route + handler kind → program
// ---------------------------------------------------------------------------------------------------------------
GOFR_HD void route_request(const TableView& tv, const BatchRefs& br, ReqCtx& c) {
    const ImageHeader& H = *tv.hdr();
    bool head = c.method() == GOFR_M_HEAD;
    if (!path_is_clean(c.path, c.path_len)) {  // mux redirects before routing and before any middleware
        c.prog = head ? H.prog_301_head : H.prog_301;
        return;
    }
    int m = mux_match(tv, c.method(), c.path, c.path_len);
    if (m == -2) { c.prog = head ? H.prog_405_head : H.prog_405; return; }
    if (m == -1) { c.prog = H.prog_404; return; }
    c.route = (uint32_t)m;
    const RouteRec& R = tv.routes()[m];
    if (c.method() == GOFR_M_OPTIONS) { c.prog = H.prog_options; return; }  // middleware/cors.go:10-13
    c.prog = R.prog_ok;
    if (R.hkind == GOFR_H_PARAM_FORMAT) {
        const ParamSpan ps = find_param(c.query(), c.query_len, tv.lit_bytes(R.key_off), R.key_len);
        c.pv_off = ps.off; c.pv_len = ps.len; c.pv_flags = ps.flags;
        c.def_off = R.def_off;
        c.def_len = R.def_len;
    } else if (R.hkind == GOFR_H_PATHPARAM_FORMAT) {
        // v := c.PathParam(name): the variable's span from the match (pkg/gofr/http/request.go:36-38)
        uint32_t sp[2] = {0, 0};
        if (R.key_len != 0xFFFF && template_match(tv, R, c.path, c.path_len, (int)R.key_len, sp) && sp[1]) {
            c.pv_off = sp[0];
            c.pv_len = sp[1];
            c.pv_flags = 1u | 4u | (json_needs_escape<false>(c.path + sp[0], sp[1]) ? 2u : 0u);  // bit2: source is the path
        }
        c.def_off = R.def_off;
        c.def_len = 0;
    } else if (R.hkind == GOFR_H_RESULT) {
        // the closure ran on the host; its outcome word selects what Responder.Respond does (responder.go:19-62)
        const uint32_t outcome = c.data_len >= 4 ? *(const uint32_t*)c.data() : 0xFFFFFFFFu;
        const uint32_t okind = outcome & 0xFFu, oerr = outcome >> 8;
        if (okind > GOFR_RESULT_RAW_NIL || (okind < GOFR_RESULT_RAW_DATA ? oerr != 0 : oerr > GOFR_RESULT_RAW_MISSING)) {
            c.prog = H.prog_panic;  // malformed record from the host shim
            return;
        }
        c.data_off += 4;
        c.data_len -= 4;
        if (okind >= GOFR_RESULT_RAW_DATA) {  // response.Raw: data encoded bare, the error picks the status (responder.go:21-26)
            c.prog = tv.rawprogs()[(uint32_t)m * 9u + (okind - GOFR_RESULT_RAW_DATA) * 3u + oerr];
            if (c.prog == 0xFFFFu) c.prog = H.prog_panic;  // RAW_DATA on a route registered without a schema
            return;
        }
        c.prog = outcome == GOFR_RESULT_DATA ? R.prog_ok : outcome == GOFR_RESULT_ERROR ? R.prog_err
               : outcome == GOFR_RESULT_NIL ? R.key_len : outcome == GOFR_RESULT_MISSING ? R.def_len
               : outcome == GOFR_RESULT_BOTH ? (R.key_off & 0xFFFFu) : (R.key_off >> 16);
        if (c.prog == 0xFFFFu) c.prog = H.prog_panic;  // DATA / BOTH on a route registered without a schema
    } else if (R.hkind == GOFR_H_BIND_ECHO) {
        // var v T; if err := c.Bind(&v); err != nil { return nil, err }; return v, nil
        uint32_t* brow = c.brow(br);
        if (!bind_request(tv, R.schema, c.data(), c.data_len, brow)) {
            // bodies nested deeper than the device scanner's 64-level stack are handed to the host like a
            // GOFR_H_HOST route (status 0) rather than answered differently from encoding/json (limit 10000)
            // (BE_DEFER = 5 exists only where float64 members do, i.e. in the VALUES instances: the others keep the very
            // compare they were validated with, so their binaries stay byte-identical)
            const bool to_host = (GOFR_TU_VALUES != 0) ? brow[0] >= 4u /* BE_DEPTH, BE_DEFER */ : brow[0] == 4u /* BE_DEPTH */;
            c.prog = to_host ? 0xFFFFu : R.prog_err;
        }
    }
}

// Routing only (gofr_route_device): what the router and the middlewares decide before any handler runs.
// Returns 301 (cleanPath redirect), 404 / 405 (mux's own handlers), 200 (CORS answers OPTIONS itself,
// middleware/cors.go:10-13) or 0 = "the handler of *route runs"; vars[k] = off | len << 16 of the k-th path variable
// (mux.Vars in template order), 0xFFFFFFFF for unused slots.
GOFR_HD uint32_t route_only(const TableView& tv, uint32_t method, const uint8_t* path, uint32_t n, uint32_t* route,
                            uint32_t vars[kMaxVars]) {
    *route = GOFR_ROUTE_NONE;
    for (int k = 0; k < kMaxVars; k++) vars[k] = 0xFFFFFFFFu;
    if (!path_is_clean(path, n)) return 301;
    const int m = mux_match(tv, method, path, n);
    if (m == -2) return 405;
    if (m == -1) return 404;
    *route = (uint32_t)m;
    const RouteRec R = tv.routes()[m];
    if (!(R.flags & RF_LITERAL) && R.n_pieces > 1) {
        uint32_t sp[2 * kMaxVars];
        for (int k = 0; k < 2 * kMaxVars; k++) sp[k] = 0xFFFFFFFFu;
        template_match(tv, R, path, n, -2, sp);
        for (int k = 0; k < kMaxVars; k++)
            if (sp[2 * k] != 0xFFFFFFFFu) vars[k] = sp[2 * k] | sp[2 * k + 1] << 16;
    }
    return method == GOFR_M_OPTIONS ? 200u : 0u;
}

// ---------------------------------------------------------------------------------------------------------------
// stages 2+3: interpret the response program.  EMIT=false: compute c.body_len / c.total_len / c.slow_mask and
// validate the row (returns false → caller switches to the panic program).  EMIT=true: write the bytes.
// ---------------------------------------------------------------------------------------------------------------
// Out-of-line slow paths work on a copy of the Writer so that the hot Writer never has its address taken (it stays in
// registers); the copy lives in local memory only while the rare path runs.
#define GOFR_SLOW_CALL(w, expr) do { Writer t_ = *(w); Writer* tw = &t_; (void)tw; expr; *(w) = t_; } while (0)

}  // namespace gofr
#include "value_device.cuh"  // float64 text and the generic encoder behind OP_F64 / OP_VALUE
namespace gofr {

// STATIC_N > 0: the program's ops are compile-time constants (static_ops, STATIC_N of them): the op loop is unrolled
// and every decision that depends only on the program folds away — what a table-specific build of the kernel runs for
// its hot programs.  STATIC_N == 0: the interpreter, ops fetched from the table in shared memory.
// VALUES: the instance that also knows OP_F64 / OP_VALUE and the emptiness test of their kinds (the wider data model,
// value_device.cuh).  Programs that contain such ops (PF_VALUES) run through out-of-line wrappers of that instance
// (size_values_call / emit_values_call); the inlined hot instance is compiled without them — one more call site inside
// its op loop cost the packed kernel 38 % (0.40 -> 0.555 ms per 1 Mi config-2 requests: registers live across the loop
// spilled, 176 -> 600 bytes of spill stores) although no config-2 program has such an op.
template <bool EMIT, int STATIC_N = 0, bool VALUES = false>
GOFR_HD bool run_prog(const TableView& tv, const BatchRefs& br, ReqCtx& c, Writer* w, const uint4* static_ops = nullptr) {
    const ProgRec P = tv.progs()[c.prog];  // by value: the staging stores below must not force re-reads of the table
    // the size pass visits only the ops whose length depends on the request
    const Op* ops = tv.ops() + (EMIT ? P.first_op : P.first_dyn);
    const bool head = c.method() == GOFR_M_HEAD;
    // chunkWriter eats the body of a HEAD response; body ops come last, so a HEAD emit simply stops before them
    const uint32_t n_ops = EMIT ? (head ? P.n_hdr_ops : P.n_ops) : P.n_dyn;
    const uint8_t* const lits = tv.lits();
    const uint32_t* row = (P.flags & PF_BIND) ? c.brow(br) : (const uint32_t*)c.data();
    uint32_t str_cursor = 0;  // byte offset of the next string in the row's string area
    uint32_t str_base = 0;
    if ((P.flags & PF_NEEDS_ROW) && !(P.flags & PF_BIND)) {
        str_base = P.row_words ? (uint32_t)P.row_words * 4 : (uint32_t)tv.schemas()[tv.routes()[c.route].schema].fixed_words * 4;
        if (!EMIT && str_base > c.data_len) return false;
    }
    uint32_t hdr_dyn = 0, body_dyn = 0, str_bit = 1;
    bool first = true, skip = false;
    auto do_op = [&](const uint4 raw) -> bool {
        const uint32_t code = raw.x & 0xFFu, oflags = (raw.x >> 16) & 0xFFu, okind = raw.x >> 24;
        const uint32_t olen = raw.y, ooff = raw.z, oaux = raw.w;
        const bool body = oflags & OPF_BODY;
        const bool governed = oflags & OPF_VALUE_OF_KEY;
        uint32_t produced = 0;
        // Everything that appends memory verbatim meets at the single copy() at the bottom of the two-step loop:
        // step 0 is the literal prefix folded into a value op (emit pass only), step 1 the op itself.
        const bool has_prefix = EMIT && code != OP_LIT && code != OP_KEY && code != OP_BLOB && olen;
        const uint8_t* csrc = lits + oaux;
        uint32_t clen = has_prefix ? olen : 0u;
        bool cshared = true;  // literals live in the shared-memory copy of the table
#pragma unroll 1
        for (uint32_t step = EMIT ? 0u : 1u; step < 2; step++) {
        if (step == 1) {
        csrc = nullptr;
        clen = 0;
        cshared = true;
        if (EMIT && warp_any(w->wl >= GOFR_SOLO_WORDS - 8)) w->flush();  // every non-copy action appends at most 8 words
        if (code == OP_LIT) {
            if (!(governed && skip)) {
                csrc = lits + ooff;
                clen = olen;
                if (governed) produced = olen;  // ungoverned literals are pre-summed in hdr_fixed / body_fixed
            }
        } else if (code == OP_STR) {
            const uint32_t len = row[ooff];
            if (!EMIT && (str_base + str_cursor + (uint64_t)len > c.data_len)) return false;
            const uint8_t* sp = c.data() + str_base + str_cursor;
            str_cursor += len;
            const uint32_t bit = str_bit;
            str_bit <<= 1;
            if (!(governed && skip)) {
                if (!EMIT) {
                    const bool esc = c.staged() ? json_needs_escape<true>(SrcMem<true>::from(sp), len) : json_needs_escape<false>(sp, len);
                    if (esc) { c.slow_mask |= bit; produced = json_escape_slow<false>(nullptr, sp, len); }
                    else produced = len;
                } else if (c.slow_mask & bit) {
                    GOFR_SLOW_CALL(w, json_escape_slow<true>(tw, sp, len));
                } else {
                    csrc = sp;
                    clen = len;
                    cshared = c.staged();
                }
            }
        } else if (code == OP_BSTR) {
            const uint32_t boff = row[ooff], lenw = row[ooff + 1], len = lenw & 0x7FFFFFFFu;
            if (!(governed && skip)) {
                const uint8_t* sp = c.data() + boff;
                if (lenw >> 31) {  // JSON escapes / non-ASCII in the request: decode and re-encode rune by rune
                    if (EMIT) GOFR_SLOW_CALL(w, bind_string_slow<true>(tw, sp, len));
                    else produced = bind_string_slow<false>(nullptr, sp, len);
                } else { csrc = sp; clen = len; produced = len; cshared = c.staged(); }
            }
        } else if (code == OP_ERRMSG) {
            const uint32_t sidx = tv.routes()[c.route].schema;
            if (EMIT) GOFR_SLOW_CALL(w, (emit_bind_error<true, false>(tw, tv, sidx, c.data(), c.brow(br))));
            else produced = emit_bind_error<false, false>(nullptr, tv, sidx, c.data(), c.brow(br));
        } else if (code == OP_I64 || code == OP_I32) {
            if (!(governed && skip)) {
                const int64_t v = code == OP_I64 ? (int64_t)((uint64_t)row[ooff] | (uint64_t)row[ooff + 1] << 32)
                                                 : (int64_t)(int32_t)row[ooff];
                produced = emit_i64<EMIT>(w, v);
            }
        } else if (code == OP_BOOL) {
            if (!(governed && skip)) {
                const bool t = row[ooff] != 0;
                if (EMIT) { if (t) w->put4('t' | 'r' << 8 | 'u' << 16 | 'e' << 24); else { w->put4('f' | 'a' << 8 | 'l' << 16 | 's' << 24); w->putc('e'); } }
                produced = t ? 4 : 5;
            }
        } else if (VALUES && code >= OP_F64) {  // OP_F64, OP_VALUE: one out-of-line call (value_device.cuh value_op)
            // an omitted field (OP_KEY found it empty) owns no bytes of the variable part: nothing to walk
            if (!(governed && skip)) {
                const uint32_t used = str_base + str_cursor;
                uint32_t consumed = 0, vstatus = 0;
                if (EMIT) GOFR_SLOW_CALL(w, (value_op<true>(tw, tv, raw, row, c.data(), c.data_len, used, &consumed, &vstatus)));
                else {
                    produced = value_op<false>(nullptr, tv, raw, row, c.data(), c.data_len, used, &consumed, &vstatus);
                    if (vstatus != VAL_OK) {
                        // NaN / Inf: the caller sizes the program's encfail companion instead; anything else: malformed row
                        if (vstatus == VAL_UNENCODABLE) c.prog = P.encfail;
                        return false;
                    }
                }
                str_cursor += consumed;
            }
        } else if (code == OP_HEXID) {
            if (EMIT) {
                const uint4 id = *(const uint4*)(br.ids + (size_t)c.index * 16);  // loaded here, not carried
                const uint32_t idw[4] = {id.x, id.y, id.z, id.w};
#pragma unroll
                for (int k = 0; k < 4; k++) { uint32_t a, b; hex8(idw[k], a, b); w->put4(a); w->put4(b); }
            }
        } else if (code == OP_CLEN) {
            if (EMIT) emit_u32<true>(w, c.body_len);  // sized after the loop
        } else if (code == OP_KEY) {
            bool empty = false;
            if (oflags & OPF_OMITEMPTY) {
                const uint32_t wv = row[oaux];
                if (okind == GOFR_F_INT64 || okind == GOFR_F_INT) empty = (wv | row[oaux + 1]) == 0;
                else if (VALUES && okind > GOFR_F_INT) empty = value_key_empty(okind, (const uint8_t*)(row + oaux));  // float64, struct, *T, []T, map
                else if (okind == GOFR_F_STRING && (P.flags & PF_BIND)) empty = (row[oaux + 1] & 0x7FFFFFFFu) == 0;
                else empty = wv == 0;
            }
            skip = empty;
            if (!empty) {
                if (!first) { if (EMIT) w->putc(','); produced += 1; }
                first = false;
                csrc = lits + ooff;
                clen = olen;
                produced += olen;
            }
        } else if (code == OP_PARAM) {
            if (c.pv_flags & 1) {
                const bool from_path = c.pv_flags & 4;  // PathParam: already decoded, no query unescaping
                const uint8_t* v = (from_path ? c.path : c.query()) + c.pv_off;
                if (c.pv_flags & 2) {
                    if (from_path) {
                        if (EMIT) GOFR_SLOW_CALL(w, json_escape_slow<true>(tw, v, c.pv_len));
                        else produced = json_escape_slow<false>(nullptr, v, c.pv_len);
                    } else if (EMIT) GOFR_SLOW_CALL(w, emit_param_slow<true>(tw, v, c.pv_len));
                    else produced = emit_param_slow<false>(nullptr, v, c.pv_len);
                } else { csrc = v; clen = c.pv_len; produced = c.pv_len; cshared = c.staged(); }
            } else {
                csrc = lits + c.def_off;
                clen = c.def_len;
                produced = c.def_len;
            }
        } else if (code == OP_LOCATION) {
            if (EMIT) GOFR_SLOW_CALL(w, emit_location<true>(tw, c));
            else produced = emit_location<false>(nullptr, c);
        } else if (code == OP_BLOB) {
            csrc = tv.cold + ooff;
            clen = olen;
            cshared = false;
        }
        }  // step == 1
        if (EMIT && clen) {
            if (cshared) w->copy<true>(SrcMem<true>::from(csrc), clen);
            else GOFR_SLOW_CALL(w, emit_bytes(*tw, csrc, clen));
        }
        }  // steps
        if (body) body_dyn += produced; else hdr_dyn += produced;
        return true;
    };
    if (STATIC_N > 0) {
#pragma unroll
        for (int oi = 0; oi < STATIC_N; oi++)
            if (!do_op(static_ops[oi])) return false;
    } else {
#pragma unroll 1
        for (uint32_t oi = 0; oi < n_ops; oi++)
            if (!do_op(*(const uint4*)(ops + oi))) return false;  // one 16-byte load per op
    }
    if (!EMIT) {
        c.body_len = P.body_fixed + body_dyn;
        uint32_t hl = P.hdr_fixed + hdr_dyn;
        if (P.flags & PF_HAS_CLEN) hl += emit_u32<false>(nullptr, c.body_len);
        c.total_len = hl + (head ? 0 : c.body_len);
    }
    return true;
}


// ---------------------------------------------------------------------------------------------------------------
// slot-layout fast path (table_format.h FastRec): programs made of literals and plain values, requests whose values
// need no escaping, tiles staged in shared memory.  Anything else takes run_prog — the general interpreter above.
// ---------------------------------------------------------------------------------------------------------------

// Row words of a staged request: the data section lives in shared memory, so it is read with ld.shared (a generic load
// of the same address takes the slow LD.E path and showed up as the second largest long-scoreboard stall); Bind span rows
// live in global scratch.
struct RowReader {
    saddr_t sh;           // data section in shared memory
    const uint32_t* gl;   // Bind span row (global), or null
    // stg_ld, not src_ld: a non-volatile asm is a pure function to the compiler, which hoisted these loads above the
    // op-code tests that guard them — with a literal-pool offset as the "row index" (memcheck: invalid __shared__ read)
    GOFR_HD uint32_t operator[](uint32_t k) const { return gl ? gl[k] : stg_ld(sh + 4 * k); }
};

// OP_KEY `raw` (op flags `oflags`): true if it has omitempty and its field holds the zero value, so that the key and the
// ops it governs are left out.  bind: the row is a Bind span row.
GOFR_HD bool key_omitted(const uint4& raw, uint32_t oflags, const RowReader& row, bool bind) {
    bool empty = false;
    if (oflags & OPF_OMITEMPTY) {
        const uint32_t okind = raw.x >> 24, wv = row[raw.w];
        if (okind == GOFR_F_INT64 || okind == GOFR_F_INT) empty = (wv | row[raw.w + 1]) == 0;
        else if (okind == GOFR_F_STRING && bind) empty = (row[raw.w + 1] & 0x7FFFFFFFu) == 0;
        else empty = wv == 0;
    }
    return empty;
}

// Lean size pass of a PF_FAST program (every dynamic op is a plain value of the body).  Returns false when the request
// needs something emit_fast does not do — a string encoding/json would escape, a query value that needs decoding, a
// malformed row, a tile that is not staged, HEAD — and the caller runs the general size pass instead.
GOFR_HD bool size_fast(const TableView& tv, const BatchRefs& br, ReqCtx& c) {
    const ProgRec P = tv.progs()[c.prog];
    if (!(P.flags & PF_FAST) || !c.staged() || c.method() == GOFR_M_HEAD) return false;
    const Op* ops = tv.ops() + P.first_dyn;
    RowReader row;
    row.sh = to_saddr(c.data());
    row.gl = (P.flags & PF_BIND) ? c.brow(br) : nullptr;
    uint32_t str_base = 0;
    if ((P.flags & PF_NEEDS_ROW) && !(P.flags & PF_BIND)) {
        str_base = P.row_words ? (uint32_t)P.row_words * 4 : (uint32_t)tv.schemas()[tv.routes()[c.route].schema].fixed_words * 4;
        if (str_base > c.data_len) return false;
    }
    uint32_t cursor = 0, dyn = 0;
    bool first = true, skip = false;  // struct keys with omitempty (OP_KEY) and the ops they govern
#pragma unroll 1
    for (uint32_t oi = 0; oi < P.n_dyn; oi++) {
        const uint4 raw = *(const uint4*)(ops + oi);
        const uint32_t code = raw.x & 0xFFu, oflags = (raw.x >> 16) & 0xFFu, ooff = raw.z;
        if (code == OP_KEY) {
            const bool empty = key_omitted(raw, oflags, row, P.flags & PF_BIND);
            skip = empty;
            if (!empty) { dyn += (first ? 0u : 1u) + raw.y; first = false; }
            continue;
        }
        const bool skipped = (oflags & OPF_VALUE_OF_KEY) && skip;
        if (code == OP_STR) {
            const uint32_t len = row[ooff];
            if (str_base + cursor + (uint64_t)len > c.data_len) return false;
            const uint8_t* sp = c.data() + str_base + cursor;
            cursor += len;
            if (skipped) continue;
            if (json_needs_escape<true>(SrcMem<true>::from(sp), len)) return false;
            dyn += len;
        } else if (skipped) {
            continue;
        } else if (code == OP_LIT) {  // a literal governed by a key (ungoverned ones are pre-summed)
            dyn += raw.y;
        } else if (code == OP_I64) {
            dyn += emit_i64<false>(nullptr, (int64_t)((uint64_t)row[ooff] | (uint64_t)row[ooff + 1] << 32));
        } else if (code == OP_I32) {
            dyn += emit_i64<false>(nullptr, (int64_t)(int32_t)row[ooff]);
        } else if (code == OP_BOOL) {
            dyn += row[ooff] ? 4u : 5u;
        } else if (code == OP_PARAM) {
            if (c.pv_flags & 1) {
                if (c.pv_flags & 2) return false;
                dyn += c.pv_len;
            } else dyn += c.def_len;
        } else if (code == OP_BSTR) {
            const uint32_t lenw = row[ooff + 1];
            if (lenw >> 31) return false;
            dyn += lenw;
        } else return false;
    }
    c.str_base = str_base;
    c.body_len = P.body_fixed + dyn;
    uint32_t hl = P.hdr_fixed;
    if (P.flags & PF_HAS_CLEN) hl += emit_u32<false>(nullptr, c.body_len);
    c.total_len = hl + c.body_len;
    c.mflags |= 1u << 17;
    return true;
}

// Windows [k0, k1) of a response into its slot, window k0 + i from window i of the template at src (16-byte aligned, in
// the literal pool): whole 32-byte sectors wherever the destination allows (a slot starts on a sector boundary or in the
// middle of one), single 16-byte windows at the ends.
GOFR_HD void copy_windows(uint8_t* dst, saddr_t src, uint32_t k0, uint32_t k1, SoloStores p) {
    const uint32_t n = k1 - k0;
    uint8_t* const d = dst + 16 * k0;
    uint32_t i = 0;
    if (n && ((uintptr_t)d & 16u)) {
        const uint4 v = src_ld128(src);
        store16(d, v.x, v.y, v.z, v.w);
        i = 1;
    }
#pragma unroll 1
    while (p.round(i + 2 <= n)) {
        const bool have = i + 2 <= n;
        uint4 a = {0u, 0u, 0u, 0u}, b = {0u, 0u, 0u, 0u};
        if (have) { a = src_ld128(src + 16 * i); b = src_ld128(src + 16 * (i + 1)); }
        p.store32(have, d + 16 * i, a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w);
        if (have) i += 2;
    }
    if (i < n) {
        const uint4 v = src_ld128(src + 16 * i);
        store16(d + 16 * i, v.x, v.y, v.z, v.w);
    }
}

// Windows [h0, h1) of the template at tp, the 2 or 3 that the 32 hex characters of the trace id touch, staged in the lane's
// (idle) Writer column at col, whose rows are S bytes apart: the template's words from row 0 on, then the 8 hex words of
// `id` shifted to byte hex_pos & 15 of window h0 on top.  The store policy stores the windows from there (emit_fast).
template <uint32_t S>
GOFR_HD void stage_trace_id(saddr_t col, saddr_t tp, uint32_t hex_pos, uint32_t h0, uint32_t h1, uint4 id) {
    const uint32_t nw = (h1 - h0) * 4;  // 8 or 12 words
#pragma unroll 1
    for (uint32_t k = 0; k < nw; k++) stg_st(col + k * S, src_ld(tp + 16 * h0 + 4 * k));
    uint32_t H[8];
    hex8(id.x, H[0], H[1]); hex8(id.y, H[2], H[3]); hex8(id.z, H[4], H[5]); hex8(id.w, H[6], H[7]);
    const uint32_t o = hex_pos & 15u, q = o >> 2, sh = (o & 3u) * 8;
    const saddr_t hp = col + q * S;
    if (sh == 0) {
#pragma unroll
        for (uint32_t j = 0; j < 8; j++) stg_st(hp + j * S, H[j]);
    } else {
        const uint32_t lowmask = (1u << sh) - 1u;
        stg_st(hp, (stg_ld(hp) & lowmask) | (H[0] << sh));
#pragma unroll
        for (uint32_t j = 1; j < 8; j++) stg_st(hp + j * S, fsr(H[j - 1], H[j], 32 - sh));
        stg_st(hp + 8 * S, (H[7] >> (32 - sh)) | (stg_ld(hp + 8 * S) & ~lowmask));
    }
}

// Writes a response sized by size_fast into its 16-byte aligned slot: the template as whole 16-byte windows from the
// literal pool, the windows the trace id touches staged in the lane's column first (stage_trace_id), then the tail ops
// through the Writer, which starts right after the template.  The store policies differ only in how the template windows
// leave.  SoloStores: each lane its own, the plain windows in whole sectors where the slot allows (copy_windows).
// LineStores: the warp stores the templates of all its lanes together (LineStores::templates), and every lane of the
// write mask runs every vote and store round of the tail, also when its program has no template or no tail: a lane past
// its last op, or on an op that writes nothing, copies 0 bytes.  Only the appending of words differs between lanes.
// live false (LineStores): the lane has no response and runs an empty one — votes and store rounds, no loads, no stores.
template <typename P>
GOFR_HD void emit_fast(const TableView& tv, const BatchRefs& br, ReqCtx& c, uint8_t* dst, uint32_t* ring_col, P p,
                       bool live = true) {
    const FastRec F = live ? *(tv.fast() + c.prog) : FastRec{0u, 0, 0, 0xFFFFu, 0, 0, 0u};
    const uint32_t nwin = F.tmpl_windows;
    // the trace id is needed after the template copy: ask for it now
    uint4 id = {0u, 0u, 0u, 0u};
    if (F.hex_pos != 0xFFFFu) id = *(const uint4*)(br.ids + (size_t)c.index * 16);
    WriterT<P> w;
    // the Writer's room check before a value: SoloStores flushes whole sectors once 8 words wait, LineStores has a line
    constexpr uint32_t kFull = P::kLockstep ? 32u : GOFR_SOLO_WORDS - 8;
    if (P::kLockstep || nwin) {
        const saddr_t tp = to_saddr(tv.lits() + F.tmpl_off);
        const saddr_t col = to_saddr(ring_col);
        uint32_t h0 = nwin, h1 = nwin;  // [h0, h1): windows the 32 hex characters touch
        if (F.hex_pos != 0xFFFFu) { h0 = (uint32_t)F.hex_pos >> 4; h1 = (((uint32_t)F.hex_pos + 31u) >> 4) + 1u; }
        if constexpr (P::kLockstep) {
            if (h0 < nwin) stage_trace_id<P::kStride>(col, tp, F.hex_pos, h0, h1, id);
            p.templates(dst, tp, nwin, h0, h1, col);
        } else {
            copy_windows(dst, tp, 0, h0, p);
            copy_windows(dst, tp + 16 * h1, h1, nwin, p);
            if (h0 < nwin) {
                // the 2 or 3 windows around the trace id go out whole, one at a time (as whole sectors the 5-CTA slot
                // instance took 4 % longer on config 4, well outside the run-to-run spread: DESIGN §6)
                stage_trace_id<P::kStride>(col, tp, F.hex_pos, h0, h1, id);
#pragma unroll 1
                for (uint32_t k = h0; k < h1; k++) {
                    const saddr_t rp = col + (k - h0) * 4 * P::kStride;
                    store16(dst + 16 * k, stg_ld(rp), stg_ld(rp + P::kStride), stg_ld(rp + 2 * P::kStride), stg_ld(rp + 3 * P::kStride));
                }
            }
        }
    }
    if (!P::kLockstep && (F.flags & FR_COMPLETE)) return;
    w.init(dst + 16 * nwin, ring_col);
    // a template-only program: with LineStores its Writer runs the tail with no ops, appending nothing but taking part in
    // the votes and store rounds
    const uint32_t n_ops = (F.flags & FR_COMPLETE) ? 0u : F.n_tail_ops;
    const Op* ops = tv.ops() + F.tail_op;
    const uint8_t* const lits = tv.lits();
    RowReader row;
    row.sh = to_saddr(c.data());
    row.gl = (F.flags & FR_BIND) ? c.brow(br) : nullptr;
    uint32_t str_cursor = 0;
    bool first = true, skip = false;
#pragma unroll 1
    for (uint32_t oi = 0; p.round(oi < n_ops); oi++) {
        bool live = oi < n_ops;  // false: this op writes nothing (a lane past its last op, an omitted key or value)
        uint4 raw = {0u, 0u, 0u, 0u};
        if (live) raw = *(const uint4*)(ops + oi);
        const uint32_t code = raw.x & 0xFFu, oflags = (raw.x >> 16) & 0xFFu, ooff = raw.z;
        bool comma = false;
        if (live && code == OP_KEY) {
            skip = key_omitted(raw, oflags, row, F.flags & FR_BIND);
            if (skip) live = false;
            else {
                comma = !first;
                first = false;
            }
        } else if (live && (oflags & OPF_VALUE_OF_KEY) && skip) {
            if (code == OP_STR) str_cursor += row[ooff];
            live = false;
        }
        if (!P::kLockstep && !live) continue;
        if ((P::kLockstep || comma) && p.vote(w.wl >= kFull)) w.flush(p);  // room for the comma
        if (comma) w.putc(',');
        const bool lit_only = code == OP_LIT || code == OP_KEY;
        // step 0: the op's literal bytes (OP_LIT / OP_KEY: the literal itself, else the folded prefix); step 1: its value
        const uint8_t* csrc = lits + (lit_only ? raw.z : raw.w);
        uint32_t clen = live ? raw.y : 0u;
#pragma unroll 1
        for (uint32_t step = 0; step < 2; step++) {
            if (step == 1) {
                if (!P::kLockstep && lit_only) break;
                clen = 0;
                if (p.vote(w.wl >= kFull)) w.flush(p);  // a generated value appends at most 8 words
                if (!live || lit_only) {
                    // no value: the copy below stores nothing
                } else if (code == OP_STR) {
                    clen = row[ooff];
                    csrc = c.data() + c.str_base + str_cursor;
                    str_cursor += clen;
                } else if (code == OP_I64) {
                    emit_i64<true, WriterT<P>>(&w, (int64_t)((uint64_t)row[ooff] | (uint64_t)row[ooff + 1] << 32));
                } else if (code == OP_I32) {
                    emit_i64<true, WriterT<P>>(&w, (int64_t)(int32_t)row[ooff]);
                } else if (code == OP_BOOL) {
                    if (row[ooff]) w.put4('t' | 'r' << 8 | 'u' << 16 | 'e' << 24);
                    else { w.put4('f' | 'a' << 8 | 'l' << 16 | 's' << 24); w.putc('e'); }
                } else if (code == OP_CLEN) {
                    emit_u32<true, WriterT<P>>(&w, c.body_len);
                } else if (code == OP_HEXID) {
                    const uint4 id = *(const uint4*)(br.ids + (size_t)c.index * 16);
                    const uint32_t idw[4] = {id.x, id.y, id.z, id.w};
#pragma unroll
                    for (int k = 0; k < 4; k++) { uint32_t a, b; hex8(idw[k], a, b); w.put4(a); w.put4(b); }
                } else if (code == OP_PARAM) {
                    if (c.pv_flags & 1) { csrc = ((c.pv_flags & 4) ? c.path : c.query()) + c.pv_off; clen = c.pv_len; }
                    else { csrc = lits + c.def_off; clen = c.def_len; }
                } else {  // OP_BSTR
                    csrc = c.data() + row[ooff];
                    clen = row[ooff + 1];
                }
            }
            if (P::kLockstep || clen) w.template copy<true>(SrcMem<true>::from(csrc), clen, p);
        }
    }
    w.finish_padded(p);
}

// Full size stage for one request: route, size; a malformed handler-result row is answered like a handler panic.
#if defined(GOFR_STATIC_PROG)
#include GOFR_STATIC_PROG  /* experiment: one program of one table as compile-time constants */
#if defined(__CUDA_ARCH__)
#define GOFR_IS_STATIC(c) ((c).prog == GOFR_STATIC_PROG_ID && (c).method() != GOFR_M_HEAD)
#endif
#endif

// GOFR_TU_VALUES: whether this translation unit's inlined size / emit functions know about PF_VALUES programs at all.  The
// packed kernel exists twice (serve_kernel.cu without, serve_values_kernel.cu with): the engine launches the second one
// only for tables that contain such a program, so tables without them run exactly the code they ran before the wider
// data model existed.  It is a template argument (VO), not an #if, so that the two variants are different functions.

// programs with OP_F64 / OP_VALUE ops: the VALUES instance of the interpreter, out of line (see run_prog)
GOFR_HD_NOINLINE bool size_values_call(const TableView tv, const BatchRefs br, ReqCtx* c) { return run_prog<false, 0, true>(tv, br, *c, nullptr); }
template <bool SLOTS>
GOFR_HD_NOINLINE void emit_values_call(const TableView tv, const BatchRefs br, ReqCtx* c, uint8_t* dst, uint32_t* ring_col) {
    Writer w;
    w.init(dst, ring_col);
    run_prog<true, 0, true>(tv, br, *c, &w);
    if (SLOTS) w.finish_padded(); else w.finish();
}

// sizes a routed request (route_request has run) with the general interpreter
template <bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD void size_routed_general(const TableView& tv, const BatchRefs& br, ReqCtx& c) {
    if (c.prog == 0xFFFF) {  // GOFR_H_HOST: nothing to emit, status 0 = pending on the host
        c.body_len = c.total_len = 0;
        return;
    }
    bool ok;
    const uint32_t asked = c.prog;
#ifdef GOFR_IS_STATIC
    if (GOFR_IS_STATIC(c)) ok = run_prog<false, GOFR_STATIC_N_DYN>(tv, br, c, nullptr, kStaticDyn);
    else
#endif
    if (VO && (tv.progs()[c.prog].flags & PF_VALUES)) {
        ReqCtx t = c;  // a copy: taking the address of `c` itself would move the request context to local memory (size_routed)
        ok = size_values_call(tv, br, &t);
        c.prog = t.prog; c.body_len = t.body_len; c.total_len = t.total_len; c.slow_mask = t.slow_mask;
    } else
    ok = run_prog<false>(tv, br, c, nullptr);
    if (!ok) {
        // a malformed row is answered like a handler panic; a float that encoding/json cannot write (run_prog switched
        // c.prog to the program's encfail companion) keeps its status and headers and loses its body
        if (c.prog == asked || c.prog == 0xFFFF) c.prog = tv.hdr()->prog_panic;
        c.slow_mask = 0;
        run_prog<false>(tv, br, c, nullptr);
    }
}
// The slot-layout kernel keeps the general interpreter OUT of line: its hot path is size_fast / emit_fast, and two more
// inlined copies of run_prog cost it registers and instruction-cache room (measured: no gain from the fast path until the
// general path became a call).
template <bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD_NOINLINE void size_routed_call(const TableView tv, const BatchRefs br, ReqCtx* c) { size_routed_general<VO>(tv, br, *c); }

// FAST: the slot-layout kernel — the lean size pass where it applies (the response is then written by emit_fast)
template <bool FAST = false, bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD void size_routed(const TableView& tv, const BatchRefs& br, ReqCtx& c) {
    if (FAST) {
        if (c.prog == 0xFFFF) { c.body_len = c.total_len = 0; return; }
        if (size_fast(tv, br, c)) return;
        // the call works on a copy: taking the address of `c` itself would move the whole request context to local
        // memory for the hot path too (it did: 568 LDL/STL in the kernel, and no gain from the fast path)
        ReqCtx t = c;
        size_routed_call<VO>(tv, br, &t);
        c.prog = t.prog; c.body_len = t.body_len; c.total_len = t.total_len; c.slow_mask = t.slow_mask;
        return;
    }
    size_routed_general<VO>(tv, br, c);
}

template <bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD void size_request(const TableView& tv, const BatchRefs& br, ReqCtx& c) {
    route_request(tv, br, c);
    size_routed<false, VO>(tv, br, c);
}

// HTTP status of a sized request (0: GOFR_H_HOST, the closure runs on the host)
GOFR_HD uint32_t request_status(const TableView& tv, const ReqCtx& c) { return c.prog == 0xFFFF ? 0u : tv.progs()[c.prog].status; }

template <bool SLOTS, bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD void emit_request_general(const TableView& tv, const BatchRefs& br, ReqCtx& c, uint8_t* dst, uint32_t* ring_col) {
    if (VO && (tv.progs()[c.prog].flags & PF_VALUES)) {
        ReqCtx t = c;
        emit_values_call<SLOTS>(tv, br, &t, dst, ring_col);
        return;
    }
    Writer w;
    w.init(dst, ring_col);
#ifdef GOFR_IS_STATIC
    if (GOFR_IS_STATIC(c)) run_prog<true, GOFR_STATIC_N_EMIT>(tv, br, c, &w, kStaticEmit);
    else
#endif
    run_prog<true>(tv, br, c, &w);
    if (SLOTS) w.finish_padded(); else w.finish();
}
template <bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD_NOINLINE void emit_request_slots_call(const TableView tv, const BatchRefs br, ReqCtx* c, uint8_t* dst, uint32_t* ring_col) {
    emit_request_general<true, VO>(tv, br, *c, dst, ring_col);
}

template <bool SLOTS = false, bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD void emit_request(const TableView& tv, const BatchRefs& br, ReqCtx& c, uint8_t* dst, uint32_t* ring_col) {
    if (c.total_len == 0) return;
    if (SLOTS) {
        if (c.fast()) emit_fast(tv, br, c, dst, ring_col, SoloStores{});
        else { ReqCtx t = c; emit_request_slots_call<VO>(tv, br, &t, dst, ring_col); }  // a copy: see size_routed
        return;
    }
    emit_request_general<false, VO>(tv, br, c, dst, ring_col);
}

// Patch the batch's Date into a private copy of the table's hot part (the kernel does this on its shared-memory
// copy right after loading it; `idx`/`step` spread the work over the CTA).
GOFR_HD void patch_dates(uint8_t* hot, const uint8_t* date29, uint32_t idx, uint32_t step) {
    const ImageHeader* H = (const ImageHeader*)hot;
    const uint32_t* fix = (const uint32_t*)(hot + H->fixups_off);
    uint8_t* lits = hot + H->lits_off;
    for (uint32_t k = idx; k < H->n_fixups * 29u; k += step) lits[fix[k / 29u] + k % 29u] = date29[k % 29u];
}

}  // namespace gofr

#include "bind_device.cuh"
