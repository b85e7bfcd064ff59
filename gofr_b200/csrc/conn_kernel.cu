// conn_kernel.cu — the compact step of gofr_conn_batch_submit, sm_90a: every connection's whole requests, without its tail
// record, to consecutive places of the request columns the serve kernel reads.
//
// One thread per connection on the tile skeleton of tile_common.cuh.  The inputs are word columns read once, so there is
// nothing to stage: a connection's length is its number of whole requests (conn_requests), place_tile scans the lengths in
// the CTA and chains the tiles by the look-back, and the connection copies its requests (conn_put, conn_device.cuh).
#include <cuda_runtime.h>
#include <stdint.h>

#include "conn_device.cuh"
#include "engine_internal.h"
#include "tile_common.cuh"

namespace gofr {

constexpr int CT = kServeThreads;
constexpr int CNW = CT / 32;

__global__ void __launch_bounds__(CT) conn_compact_kernel(const ConnParams p) {
    __shared__ uint32_t warp_sum[CNW];
    __shared__ unsigned long long tile_base;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * CT + threadIdx.x;
        const bool valid = i < p.n;
        const uint32_t count = valid ? conn_requests(p.first, p.conn_status, i) : 0u;
        const TilePlace t = place_tile(p, tile, count, warp_sum, tile_base);
        if (!valid) continue;
        const uint32_t k0 = (uint32_t)(t.base + t.excl);
        p.out_off[i] = p.req0 + k0;
        if (i == p.n - 1) p.out_off[p.n] = p.req0 + k0 + count;
        if (!t.fits) continue;
        conn_put((const gofr_req_desc*)p.desc_in, p.rec_off, p.first[i], count, conn_key(p.trace_key, p.trace_seed, p.conn0, i),
                 (gofr_req_desc*)p.out, p.req_at, p.ids, k0);
    }
}

}  // namespace gofr
