// http_kernel.cu — HTTP/1.1 request heads for a batch of raw messages (gofr_http_parse_device), sm_90a.
//
// One thread per message on the tile skeleton of tile_common.cuh, staged from the offset column (messages are back to back
// in d_raw).  No scan and no look-back: the parsed form of message i is written inside the byte range the message itself
// occupies in an equally sized arena, so nothing depends on the other messages.  Per-message logic: http_device.cuh.
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"
#include "http_device.cuh"
#include "tile_common.cuh"

namespace gofr {

constexpr int HT = kServeThreads;
constexpr uint32_t kHttpStage = 26 * 1024;  // bytes of raw messages staged per tile (128 messages × 208 B): 8 CTAs per SM

struct HttpShared {
    uint64_t bar;
    __align__(16) uint8_t in[kHttpStage + 32];
};

__global__ void __launch_bounds__(HT, 8) http_parse_kernel(const HttpParams p) {
    __shared__ __align__(16) HttpShared sh;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) tile_barrier_init(&sh.bar);
    __syncthreads();
    uint32_t parity = 0;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * HT + tid;
        const bool valid = i < p.n;
        const ByteRange in = offset_range(p.raw_off, tile * HT, min(p.n, tile * HT + HT));
        __syncthreads();  // previous tile's reads of sh.in are done
        stage_start(&sh.bar, sh.in, p.raw, in, kHttpStage);
        uint32_t mo = 0, mn = 0;
        if (valid) { mo = __ldg(p.raw_off + i); mn = __ldg(p.raw_off + i + 1) - mo; }
        const uint8_t* base = stage_wait(&sh.bar, parity, sh.in, p.raw, in, kHttpStage);
        if (!valid) continue;
        const uint32_t a = (mo + 3u) & ~3u;
        HttpOut o;
        http_parse(base + mo, mn, p.arena + a, &o);
        p.status[i] = o.status;
        uint4 d = make_uint4(0, 0, 0, 0);
        if (o.status == GOFR_HTTP_OK) d = make_uint4(a, o.path_len | o.query_len << 16, o.data_len, o.method | o.flags << 8);
        ((uint4*)p.desc)[i] = d;
#pragma unroll
        for (int k = 0; k < GOFR_HTTP_SPANS; k++) {
            const unsigned long long s = o.spans[k];
            p.spans[(size_t)i * GOFR_HTTP_SPANS + k] = o.status == GOFR_HTTP_OK ? s + mo : 0ull;  // offsets into d_raw
        }
    }
}

}  // namespace gofr
