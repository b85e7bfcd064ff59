// sector_stores.cu — what the store shape of the slot-layout serve kernel costs on its own.
//
// Writes N responses of LEN bytes (zero padded to a multiple of 16) into slots of SLOT bytes, one thread per response,
// and nothing else: no request bytes are read, each word is a cheap function of its address.  Patterns:
//   a  one lane per slot, each whole 32-byte sector as two back-to-back 16-byte st.global.cs.v4 of that lane (the
//      Writer before lane pairing): a warp store touches 32 sectors and fills half of each
//   b  lane pairs: in one instruction lanes 2k and 2k+1 write the two halves of one sector, first of the even lane's
//      slot, then of the odd lane's; a warp store covers 16 whole sectors
//   c  the warp's 32 slots as one contiguous row, 512 bytes per warp store (the floor: fully coalesced)
//   d  lane quads: four lanes write two whole sectors (64 bytes) of one slot per instruction
//   e  line rounds: one lane per slot stages its bytes in a line-aligned shared-memory column; the lanes holding a whole
//      128-byte line store four such lines per warp store, eight lanes per line (the LineStores policy of the serve
//      kernel's wide slot instance)
// Every pattern must produce the same bytes (checked against pattern a).  Prints one JSON line per pattern: CUDA-event
// time per launch over `steps` launches after a warm-up.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o sector_stores sector_stores.cu && ./sector_stores [steps]
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#define CK(x)                                                                                    \
    do {                                                                                         \
        cudaError_t e_ = (x);                                                                    \
        if (e_ != cudaSuccess) {                                                                 \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));   \
            exit(1);                                                                             \
        }                                                                                        \
    } while (0)

constexpr uint32_t N = 1u << 20, SLOT = 528, LEN = 521, PADDED = (LEN + 15) & ~15u, T = 128;

// the 16 bytes at byte offset o (16-aligned) of response r; zero past LEN
__device__ __forceinline__ uint4 val(uint32_t r, uint32_t o) {
    if (o >= PADDED) return make_uint4(0, 0, 0, 0);
    const uint32_t x = r * 0x9E3779B9u ^ o;
    uint4 v = make_uint4(x, x + 1, x + 2, x + 3);
    if (o + 16 > LEN) {  // the last window: bytes past LEN are zero
        const uint32_t k = LEN - o;  // 1..15
        uint32_t* w = &v.x;
#pragma unroll
        for (uint32_t j = 0; j < 4; j++) {
            const uint32_t b = 4 * j;
            w[j] = b >= k ? 0u : (k - b >= 4 ? w[j] : w[j] & (0xFFFFFFFFu >> (8 * (4 - (k - b)))));
        }
    }
    return v;
}
__device__ __forceinline__ void st16(uint8_t* a, uint4 v) { __stcs((uint4*)a, v); }

// a: one lane per slot
__global__ void __launch_bounds__(T) pat_a(uint8_t* out) {
    const uint32_t r = blockIdx.x * T + threadIdx.x;
    if (r >= N) return;
    uint8_t* s = out + (size_t)r * SLOT;
    uint32_t o = 0;
    if ((uintptr_t)s & 16u) { st16(s, val(r, 0)); o = 16; }
#pragma unroll 1
    for (; o + 32 <= PADDED; o += 32) { st16(s + o, val(r, o)); st16(s + o + 16, val(r, o + 16)); }
    if (o < PADDED) st16(s + o, val(r, o));
}

// b: lane pairs.  The even lane's slot and the odd lane's slot each have a head window (if it starts mid-sector), whole
// sectors and a tail window; the sectors go out paired, the edges from their own lane.
__global__ void __launch_bounds__(T) pat_b(uint8_t* out) {
    const uint32_t r = blockIdx.x * T + threadIdx.x, half = threadIdx.x & 1u;
    const bool valid = r < N;
    uint8_t* s = out + (size_t)r * SLOT;
    const uint32_t head = ((uintptr_t)s & 16u) ? 16u : 0u;
    const uint32_t nsec = valid ? (PADDED - head) / 32 : 0u;
    if (valid && head) st16(s, val(r, 0));
    // the partner's slot, sector count and head
    const uint32_t pr = r ^ 1u;
    uint8_t* ps = out + (size_t)pr * SLOT;
    const uint32_t phead = ((uintptr_t)ps & 16u) ? 16u : 0u;
    const uint32_t pn = __shfl_xor_sync(0xFFFFFFFFu, nsec, 1);
    const uint32_t both = min(nsec, pn);
    // round j: first the even lane's sector j, then the odd lane's; this lane writes half `half` of each
    uint8_t* s0 = half ? ps : s;  const uint32_t r0 = half ? pr : r, h0 = half ? phead : head;
    uint8_t* s1 = half ? s : ps;  const uint32_t r1 = half ? r : pr, h1 = half ? head : phead;
#pragma unroll 1
    for (uint32_t j = 0; j < both; j++) {
        const uint32_t o0 = h0 + 32 * j + 16 * half, o1 = h1 + 32 * j + 16 * half;
        st16(s0 + o0, val(r0, o0));
        st16(s1 + o1, val(r1, o1));
    }
#pragma unroll 1
    for (uint32_t j = both; j < nsec; j++) {  // sectors the partner has no counterpart for: alone, as in pattern a
        st16(s + head + 32 * j, val(r, head + 32 * j));
        st16(s + head + 32 * j + 16, val(r, head + 32 * j + 16));
    }
    const uint32_t o = head + 32 * nsec;
    if (valid && o < PADDED) st16(s + o, val(r, o));
}

// c: the warp's slots as one contiguous row (SLOT * 32 bytes, 16 bytes per lane per instruction)
__global__ void __launch_bounds__(T) pat_c(uint8_t* out) {
    const uint32_t w0 = (blockIdx.x * T + (threadIdx.x & ~31u));
    const uint32_t lane = threadIdx.x & 31u;
    if (w0 >= N) return;
    uint8_t* row = out + (size_t)w0 * SLOT;
#pragma unroll 1
    for (uint32_t b = 16 * lane; b < 32 * SLOT; b += 512) {
        const uint32_t r = b / SLOT, o = b - r * SLOT;
        if (o < PADDED) st16(row + b, val(w0 + r, o));
    }
}

// d: lane quads, two whole sectors (64 bytes) of one slot per instruction; four slots per quad in turn
__global__ void __launch_bounds__(T) pat_d(uint8_t* out) {
    const uint32_t r = blockIdx.x * T + threadIdx.x, q = threadIdx.x & 3u;
    uint8_t* s = out + (size_t)r * SLOT;
    const uint32_t head = ((uintptr_t)s & 16u) ? 16u : 0u;
    const uint32_t nsec = (PADDED - head) / 32;  // the same for every lane of a quad up to the head: 16 here
    if (head) st16(s, val(r, 0));
    const uint32_t nw = (nsec * 32) / 64;        // 64-byte rounds per slot (8)
#pragma unroll 1
    for (uint32_t j = 0; j < nw; j++) {
#pragma unroll
        for (uint32_t t = 0; t < 4; t++) {
            const uint32_t rr = (r & ~3u) + t;
            uint8_t* ss = out + (size_t)rr * SLOT;
            const uint32_t hh = ((uintptr_t)ss & 16u) ? 16u : 0u, o = hh + 64 * j + 16 * q;
            st16(ss + o, val(rr, o));
        }
    }
    const uint32_t o = head + 64 * nw;
    for (uint32_t b = o; b + 32 <= head + 32 * nsec; b += 32) { st16(s + b, val(r, b)); st16(s + b + 16, val(r, b + 16)); }
    const uint32_t t0 = head + 32 * nsec;
    if (t0 < PADDED) st16(s + t0, val(r, t0));
}

// e: one lane per slot, its bytes staged 8 words at a time in a line-aligned shared-memory column (word k of thread t at
//    [k * LS + t]; LS = T + 1 keeps the appends and a group's window loads conflict-free), then a vote; the lanes with a
//    complete 128-byte line are stored in rounds of four lines per warp store: lane group g = lane >> 3 takes the g-th
//    remaining ready lane, lane t = lane & 7 its 16-byte window t.  Edge lines store only the windows of the response.
constexpr uint32_t LW = 39, LS = T + 1;  // column words (< 32 before an append of at most 8), row stride in words

__device__ __forceinline__ void line_rounds(const uint32_t* ring, bool ready, uint8_t* chunk, uint32_t lo, uint32_t hi) {
    const uint32_t lane = threadIdx.x & 31u, g = lane >> 3, t = lane & 7u, warp0 = threadIdx.x & ~31u;
    uint32_t rem = __ballot_sync(~0u, ready);
    __syncwarp();  // the owners' column stores before the other lanes' loads
#pragma unroll 1
    while (rem) {
        const uint32_t m1 = rem & (rem - 1u), m2 = m1 & (m1 - 1u), m3 = m2 & (m2 - 1u);
        const uint32_t sel = g == 0 ? rem : g == 1 ? m1 : g == 2 ? m2 : m3;
        const uint32_t s = sel ? __ffs(sel) - 1u : lane;
        uint8_t* const c = (uint8_t*)__shfl_sync(~0u, (unsigned long long)chunk, s);
        const uint32_t l = __shfl_sync(~0u, lo, s), h = __shfl_sync(~0u, hi, s);
        if (sel && t >= l && t < h) {
            const uint32_t* p = ring + 4u * t * LS + warp0 + s;
            st16(c + 16u * t, make_uint4(p[0], p[LS], p[2 * LS], p[3 * LS]));
        }
        rem = m3 & (m3 - 1u);
    }
    __syncwarp();  // every load of a column before its owner moves or overwrites it
}

__global__ void __launch_bounds__(T) pat_e(uint8_t* out) {
    __shared__ uint32_t ring[LW * LS];
    const uint32_t r = blockIdx.x * T + threadIdx.x;  // N is a multiple of T: every lane has a slot
    uint32_t* const col = ring + threadIdx.x;
    uint8_t* const s = out + (size_t)r * SLOT;
    uint8_t* chunk = (uint8_t*)((uintptr_t)s & ~(uintptr_t)127);
    uint32_t lead = (uint32_t)((uintptr_t)s & 127u), wl = lead >> 2, o = 0;
#pragma unroll 1
    while (__any_sync(~0u, o < PADDED)) {
        if (o < PADDED) {
            const uint4 a = val(r, o);
            col[wl * LS] = a.x; col[(wl + 1) * LS] = a.y; col[(wl + 2) * LS] = a.z; col[(wl + 3) * LS] = a.w;
            wl += 4; o += 16;
            if (o < PADDED) {
                const uint4 b = val(r, o);
                col[wl * LS] = b.x; col[(wl + 1) * LS] = b.y; col[(wl + 2) * LS] = b.z; col[(wl + 3) * LS] = b.w;
                wl += 4; o += 16;
            }
        }
        const bool ready = wl >= 32u;
        if (__any_sync(~0u, ready)) {
            line_rounds(ring, ready, chunk, lead >> 4, 8u);
            if (ready) {
#pragma unroll 1
                for (uint32_t k = 32; k < wl; k++) col[(k - 32) * LS] = col[k * LS];
                wl -= 32; chunk += 128; lead = 0;
            }
        }
    }
    line_rounds(ring, 4 * wl > lead, chunk, lead >> 4, (wl + 3) >> 2);  // the last, partial line
}

int main(int argc, char** argv) {
    const int steps = argc > 1 ? atoi(argv[1]) : 50;
    const size_t bytes = (size_t)N * SLOT;
    uint8_t* out;
    CK(cudaMalloc(&out, bytes));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    std::vector<uint8_t> ref(bytes), got(bytes);
    void (*kern[5])(uint8_t*) = {pat_a, pat_b, pat_c, pat_d, pat_e};
    const char* names[5] = {"a_lane_per_slot", "b_lane_pairs", "c_coalesced_rows", "d_lane_quads", "e_line_rounds"};
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const uint32_t grid = (N + T - 1) / T;
    for (int rep = 0; rep < 2; rep++)
        for (int k = 0; k < 5; k++) {
            CK(cudaMemset(out, 0xA5, bytes));
            kern[k]<<<grid, T>>>(out);
            CK(cudaGetLastError());
            CK(cudaDeviceSynchronize());
            CK(cudaMemcpy(k == 0 ? ref.data() : got.data(), out, bytes, cudaMemcpyDeviceToHost));
            // bytes of a slot past PADDED are never written (sentinel), so all four must agree everywhere
            const bool same = k == 0 || memcmp(ref.data(), got.data(), bytes) == 0;
            for (int i = 0; i < 5; i++) kern[k]<<<grid, T>>>(out);
            CK(cudaEventRecord(e0));
            for (int i = 0; i < steps; i++) kern[k]<<<grid, T>>>(out);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            const double per = ms / steps;
            printf("{\"pattern\": \"%s\", \"rep\": %d, \"gpu\": \"%s\", \"n\": %u, \"slot\": %u, \"len\": %u, \"ms\": %.5f, "
                   "\"TB_s\": %.3f, \"same_bytes_as_a\": %s}\n",
                   names[k], rep, prop.name, N, SLOT, LEN, per, (double)N * PADDED / (per * 1e-3) / 1e12, same ? "true" : "false");
        }
    CK(cudaFree(out));
    return 0;
}
