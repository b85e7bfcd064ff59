// proto_nested_deferred_device.cuh — the map step of the nested proto3 decoder for maps beyond kPbnMaxMapEntries entries
// (gofr_proto_decode_nested_deferred_device): the frames the first pass answered GOFR_GRPC_DEFER are decoded again, one at
// a time by a whole CTA, with the walks of proto_nested_decode_device.cuh and PdnSorted as their MapStep.
//
// PdnSorted puts a map field's entries in canonical order with a sorted entry list in shared memory instead of selection:
//   collect   every thread scans the message's items; entry k is keyed (pdn_entry_key) by thread k % threads and stored at
//             index k with its payload (offset << 32 | length): that number ascends with the wire position
//   sort      bitonic, over the next power of two of the count (padded with entries that sort last), by (key, wire
//             position): integer keys as pbn_key_order numbers, string keys by pbn_bytes_cmp on the frame's bytes
//   compact   of each run of equal keys the last entry is kept (a later equal key replaces an earlier entry); the kept
//             payloads go to the front of the list, in key order, and the walk takes them by index
// Every thread of the CTA runs the same walk on the same frame, so control flow is uniform and begin() holds barriers; only
// thread 0 stores (store()).  One list per active map level: a map inside a map's value is the second level, and the depth
// limit allows no third (root > entry > value > entry).  Up to kPdnMaxSortedEntries entries of one map field in one message,
// duplicates counted; more stay DEFER, as do the merges the first pass defers.
// __host__ __device__: on the CPU (tests/emu) the same code runs as a CTA of one thread, lists in pdn_host_sort_mem.
#pragma once
#include <stddef.h>

#include "proto_nested_decode_device.cuh"

namespace gofr {

struct PdnList {
    uint64_t key[kPdnMaxSortedEntries];  // the entries' keys; after compaction the kept payloads, in key order
    uint64_t ent[kPdnMaxSortedEntries];  // payload offset << 32 | length; ~0 pads the sort and marks a replaced entry
};
// The dynamic shared memory of the kernel: the head, then one list per map level the description has (the host sizes it
// with pdn_sort_bytes, engine_internal.h; a level beyond those is never touched)
struct PdnSortMem {
    uint32_t part[32];               // per-warp counts of the compaction scan
    uint32_t n[kPdnMaxMapLevels];    // distinct keys in the list of each level
    uint32_t pad[2];
    PdnList list[kPdnMaxMapLevels];
};
static_assert(offsetof(PdnSortMem, list) == kPdnSortHeadBytes && sizeof(PdnList) == kPdnMaxSortedEntries * 16u, "pdn_sort_bytes");

#if defined(__CUDACC__)
extern __shared__ __align__(16) uint8_t pdn_sort_smem[];
#endif
inline PdnSortMem* pdn_host_sort_mem = nullptr;  // the CPU's lists (tests/emu)

GOFR_HD PdnSortMem* pdn_sort_mem() {
#ifdef __CUDA_ARCH__
    return reinterpret_cast<PdnSortMem*>(pdn_sort_smem);
#else
    return pdn_host_sort_mem;
#endif
}
GOFR_HD uint32_t pdn_tid() {
#ifdef __CUDA_ARCH__
    return threadIdx.x;
#else
    return 0;
#endif
}
GOFR_HD uint32_t pdn_threads() {
#ifdef __CUDA_ARCH__
    return blockDim.x;
#else
    return 1;
#endif
}
GOFR_HD void pdn_sync() {
#ifdef __CUDA_ARCH__
    __syncthreads();
#endif
}
// exclusive prefix of v over the CTA's threads in thread order, *total the sum; one barrier (whole warps)
GOFR_HD uint32_t pdn_cta_excl(uint32_t v, uint32_t* part, uint32_t* total) {
#ifdef __CUDA_ARCH__
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= (uint32_t)o) incl += u;
    }
    if (lane == 31) part[warp] = incl;
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (uint32_t w = 0; w < nw; w++) { if (w < warp) before += part[w]; all += part[w]; }
    *total = all;
    return before + incl - v;
#else
    (void)part;
    *total = v;
    return 0;
#endif
}

// list order: (key, wire position); the padding last
GOFR_HD bool pdn_entry_less(const PdnList& L, const uint8_t* f, bool str, uint32_t a, uint32_t b) {
    const uint64_t ea = L.ent[a], eb = L.ent[b];
    if (ea == ~0ull || eb == ~0ull) return ea < eb;
    const uint64_t ka = L.key[a], kb = L.key[b];
    if (ka != kb) {
        if (!str) return ka < kb;
        const int c = pbn_bytes_cmp(f + (ka >> 32), (uint32_t)ka, f + (kb >> 32), (uint32_t)kb);
        if (c) return c < 0;
    }
    return ea < eb;
}
GOFR_HD bool pdn_same_key(const PdnList& L, const uint8_t* f, bool str, uint32_t a, uint32_t b) {
    const uint64_t ka = L.key[a], kb = L.key[b];
    return ka == kb || (str && pbn_bytes_cmp(f + (ka >> 32), (uint32_t)ka, f + (kb >> 32), (uint32_t)kb) == 0);
}

struct PdnSorted {
    static constexpr uint32_t kMaxEntries = kPdnMaxSortedEntries;
    static GOFR_HD uint32_t begin(const PbnDesc& D, const uint8_t* f, uint32_t lo, uint32_t hi, uint32_t mt, uint32_t q, uint32_t E,
                                  int level, PdnItem*) {
        PdnSortMem& S = *pdn_sort_mem();
        PdnList& L = S.list[level];
        const uint32_t tid = pdn_tid(), nt = pdn_threads();
        const bool str = (D.f[D.first[E]].cls & PC_WIRE) == 2;
        pdn_sync();  // every thread is done with the list of this level that this one replaces
        uint32_t n = 0, i = lo, g = 0;
        while (i < hi) {
            PdnItem it;
            pdn_next(f, &i, hi, &it);
            if (it.wt == 3) { g++; continue; }
            if (it.wt == 4) { g--; continue; }
            if (g || pdn_field_of(D, mt, it.num, it.wt) != (int)q) continue;
            if (n % nt == tid) {
                L.key[n] = pdn_entry_key(D, f, it.poff, it.poff + it.plen, E);
                L.ent[n] = (uint64_t)it.poff << 32 | it.plen;
            }
            n++;
        }
        if (!n) return 0;
        uint32_t p2 = 1;
        while (p2 < n) p2 <<= 1;
        for (uint32_t k = n + tid; k < p2; k += nt) { L.key[k] = 0; L.ent[k] = ~0ull; }
        pdn_sync();
        for (uint32_t k = 2; k <= p2; k <<= 1) {
            for (uint32_t j = k >> 1; j; j >>= 1) {
                for (uint32_t t = tid; t < p2 / 2; t += nt) {
                    const uint32_t a = ((t & ~(j - 1)) << 1) | (t & (j - 1)), b = a + j;
                    const bool swap = (a & k) == 0 ? pdn_entry_less(L, f, str, b, a) : pdn_entry_less(L, f, str, a, b);
                    if (swap) {
                        const uint64_t ka = L.key[a], ea = L.ent[a];
                        L.key[a] = L.key[b]; L.ent[a] = L.ent[b];
                        L.key[b] = ka; L.ent[b] = ea;
                    }
                }
                pdn_sync();
            }
        }
        // each thread a contiguous chunk: mark the entries a later equal key replaces, count the kept ones, then (after
        // the scan's barrier: no key is read any more) move the kept payloads to the front
        const uint32_t c = (n + nt - 1) / nt, c0 = tid * c < n ? tid * c : n, c1 = c0 + c < n ? c0 + c : n;
        uint32_t kept = 0;
        for (uint32_t k = c0; k < c1; k++) {
            if (k + 1 < n && pdn_same_key(L, f, str, k, k + 1)) L.ent[k] = ~0ull;
            else kept++;
        }
        uint32_t total;
        uint32_t at = pdn_cta_excl(kept, S.part, &total);
        for (uint32_t k = c0; k < c1; k++)
            if (L.ent[k] != ~0ull) L.key[at++] = L.ent[k];
        if (tid == 0) S.n[level] = total;
        pdn_sync();
        return total;
    }
    static GOFR_HD bool next(const PbnDesc&, const uint8_t*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, int level, bool have,
                             uint64_t* cursor, PdnItem* out) {
        const PdnSortMem& S = *pdn_sort_mem();
        const uint64_t k = have ? *cursor + 1 : 0;
        if (k >= S.n[level]) return false;
        *cursor = k;
        const uint64_t e = S.list[level].key[k];
        out->poff = (uint32_t)(e >> 32);
        out->plen = (uint32_t)e;
        return true;
    }
    static GOFR_HD bool store() { return pdn_tid() == 0; }
};

// the size and emit passes of one deferred frame, by every thread of the CTA (the instance with maps and presence: it
// decodes presence-free descriptions too)
GOFR_HD PdnRow pdn_deferred_size(const PbnDesc& D, const uint8_t* f, uint32_t fn) {
    return pdn_decode_size_as<true, true, PdnSorted>(D, f, fn);
}
GOFR_HD void pdn_deferred_emit(const PbnDesc& D, const uint8_t* f, uint32_t fn, const PdnRow r, uint8_t* dst) {
    pdn_decode_emit_as<true, true, PdnSorted>(D, f, fn, r, dst);
}

}  // namespace gofr
