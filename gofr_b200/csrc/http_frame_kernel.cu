// http_frame_kernel.cu — connection byte streams cut into HTTP/1.1 request records (gofr_http_frame_device), sm_90a.
//
// One thread per connection on the tile skeleton of tile_common.cuh, staged from the offset column like http_kernel.cu
// (connections are back to back in d_buf).  Packed output, but a column of words instead of bytes through the Writer: a
// connection's length is its number of records, the lengths are scanned in the CTA and chained across CTAs by the look-back
// (place_tile), and the connection's record offsets go to its place in d_rec_off.  The count walk keeps the first record
// starts; a connection with more records walks again from the last kept one.  Per-connection logic: http_frame_device.cuh.
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"
#include "http_frame_device.cuh"
#include "tile_common.cuh"

namespace gofr {

constexpr int FT = kServeThreads;
constexpr int FNW = FT / 32;
constexpr uint32_t kFrameStage = 26 * 1024;  // bytes of connection buffers staged per tile, as http_kernel.cu's kHttpStage

struct FrameShared {
    uint64_t bar;
    uint32_t warp_sum[FNW];
    unsigned long long tile_base;
    __align__(16) uint8_t in[kFrameStage + 32];
};

__global__ void __launch_bounds__(FT, 8) http_frame_kernel(const HttpFrameParams p) {
    __shared__ __align__(16) FrameShared sh;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) tile_barrier_init(&sh.bar);
    __syncthreads();
    uint32_t parity = 0;
    uint32_t* const rec_off = (uint32_t*)p.out;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * FT + tid;
        const bool valid = i < p.n;
        const ByteRange in = offset_range(p.buf_off, tile * FT, min(p.n, tile * FT + FT));
        __syncthreads();  // previous tile's reads of sh.in are done
        stage_start(&sh.bar, sh.in, p.buf, in, kFrameStage);
        uint32_t co = 0, cn = 0;
        if (valid) { co = __ldg(p.buf_off + i); cn = __ldg(p.buf_off + i + 1) - co; }
        const uint8_t* conn = stage_wait(&sh.bar, parity, sh.in, p.buf, in, kFrameStage) + co;
        HttpFrameConn c;
        c.count = 0;
        if (valid) http_frame_count(conn, cn, c);
        const TilePlace t = place_tile(p, tile, c.count, sh.warp_sum, sh.tile_base);
        if (!valid) continue;
        put_offsets(p.out_off, i, p.n, t, c.count);
        p.consumed[i] = c.consumed;
        p.status[i] = c.status;
        if (!t.fits) continue;
        uint32_t* rec = rec_off + t.base + t.excl;
        http_frame_put(conn, cn, c, co, rec);
        if (i == p.n - 1) rec[c.count] = co + cn;  // the column's last entry: the end of the buffer
    }
}

}  // namespace gofr
