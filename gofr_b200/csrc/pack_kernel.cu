// pack_kernel.cu — the chunk pack kernel of the proto host path (gofr_proto_batch_decode / _encode, engine.cu).
//
// Tiles of GT records on the tile skeleton of tile_common.cuh: each thread sizes its record (pack_device.cuh), place_tile
// scans the sizes and chains the tiles by the decoupled look-back, starting at *chain_pos & 15 on the pinned-buffer path
// (the serve kernel's convention, so advance_kernel and egress_kernel run unchanged), and each thread copies its record.
// Sources are read from HBM: they were written by the kernel just before on the same stream.
#include "frame_tiles.cuh"
#include "pack_device.cuh"

namespace gofr {

struct PackShared {
    uint32_t warp_sum[GNW];
    unsigned long long tile_base;
    uint32_t stage[GOFR_STAGE_WORDS * GT];
};

__global__ void __launch_bounds__(GT) chunk_pack_kernel(const PackParams p) {
    __shared__ PackShared sh;
    const uint32_t tid = threadIdx.x;
    const unsigned long long chain0 = p.chain_pos ? (*p.chain_pos & 15ull) : 0ull;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * GT + tid;
        const bool valid = i < p.n;
        PackRec r = {nullptr, 0u};
        if (valid) r = pack_record(p, i);
        const TilePlace t = place_tile(p, tile, r.len, sh.warp_sum, sh.tile_base, false, chain0);
        if (valid) put_offsets(p.out_off, i, p.n, t, r.len);
        if (t.fits && r.len) pack_emit(r, p.out + t.base + t.excl, &sh.stage[tid]);
    }
}

}  // namespace gofr
