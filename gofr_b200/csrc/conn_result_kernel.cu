// conn_result_kernel.cu — the splice step of gofr_conn_batch_respond, sm_90a: every request of a chunk, with the closure's
// record as its data section where it has one, into a packed arena in request order (conn_result_device.cuh).
//
// One thread per request on the tile skeleton of tile_common.cuh, shaped like chunk_pack_kernel: each thread sizes its
// request's spliced form, place_tile scans the sizes and chains the tiles by the look-back (from byte 0: the arena is the
// serve kernel's input, not a caller's output), and each thread copies its bytes and rewrites its descriptor.  Sources are
// read from HBM: the parse arena and the records were written just before on the same stream.
#include <cuda_runtime.h>
#include <stdint.h>

#include "conn_result_device.cuh"
#include "tile_common.cuh"

namespace gofr {

constexpr int RT = kServeThreads;
constexpr int RNW = RT / 32;

struct ConnResultShared {
    uint32_t warp_sum[RNW];
    unsigned long long tile_base;
    uint32_t stage[GOFR_STAGE_WORDS * RT];
};

__global__ void __launch_bounds__(RT) conn_result_kernel(const ConnResultParams p) {
    __shared__ ConnResultShared sh;
    const uint32_t tid = threadIdx.x;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * RT + tid;
        const bool valid = i < p.n;
        ConnSplice s;
        s.size = 0u;
        if (valid) s = conn_splice(p, i);
        const TilePlace t = place_tile(p, tile, s.size, sh.warp_sum, sh.tile_base);
        if (valid) put_offsets(p.out_off, i, p.n, t, s.size);
        if (t.fits && valid) conn_splice_emit(p, i, s, (uint32_t)(t.base + t.excl), &sh.stage[tid]);
    }
}

}  // namespace gofr
