// conn_log_kernel.cu — the gather step of gofr_conn_batch_submit_log, sm_90a: every logged request of a chunk to its line,
// the input of reqlog_kernel.
//
// One thread per connection on the tile skeleton of tile_common.cuh, as conn_kernel.cu.  The inputs are word columns read
// once, so there is nothing to stage: a connection's length is its number of logged requests (conn_log_count), place_tile
// scans the lengths in the CTA and chains the tiles by the look-back, and the connection writes its lines (conn_log_put,
// conn_log_device.cuh).
#include <cuda_runtime.h>
#include <stdint.h>

#include "conn_log_device.cuh"
#include "engine_internal.h"
#include "tile_common.cuh"

namespace gofr {

constexpr int GT_LOG = kServeThreads;
constexpr int GNW_LOG = GT_LOG / 32;

__global__ void __launch_bounds__(GT_LOG) conn_log_kernel(const ConnLogParams p) {
    __shared__ uint32_t warp_sum[GNW_LOG];
    __shared__ unsigned long long tile_base;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * GT_LOG + threadIdx.x;
        const bool valid = i < p.n;
        uint32_t count = 0, k0 = 0, lines = 0;
        if (valid) {
            count = conn_requests(p.first, p.conn_status, i);
            k0 = p.req_first[i] - p.req0;
            lines = conn_log_count(p, p.first[i], k0, count);
        }
        const TilePlace t = place_tile(p, tile, lines, warp_sum, tile_base);
        if (!valid) continue;
        put_offsets(p.out_off, i, p.n, t, lines);
        if (t.fits && lines) conn_log_put(p, i, p.first[i], k0, count, (uint32_t)(t.base + t.excl));
    }
}

}  // namespace gofr
