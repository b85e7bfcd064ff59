// proto_nested_deferred_kernel.cu — the second pass of the nested proto3 decoder (gofr_proto_decode_nested_deferred_device):
// the frames whose status in the first pass's meta column is GOFR_GRPC_DEFER are decoded again, each by a whole CTA, with
// map fields of up to kPdnMaxSortedEntries entries put in key order by sorted lists in dynamic shared memory
// (proto_nested_deferred_device.cuh).  Every other frame keeps its status and gets an empty row.
//
// Tiles of GT frames on the tile skeleton of tile_common.cuh, packed output in frame order:
//   1. each thread reads its frame's first-pass status; the selected frames are listed in frame order;
//   2. the CTA decodes them one at a time — a size pass per selected frame (lengths and statuses kept in shared memory),
//      place_tile over those lengths (the decoupled look-back), offsets and statuses written, then an emit pass per frame
//      at its offset.  A tile without a selected frame only scans and writes its offsets and statuses.
// The input frames are read from HBM: a frame worth a second pass is rarely small enough to stage.
#include "frame_tiles.cuh"
#include "proto_nested_deferred_device.cuh"

namespace gofr {

struct PdnDeferredShared {
    uint32_t warp_sel[GNW];
    uint32_t warp_sum[GNW];
    unsigned long long tile_base;
    uint32_t sel[GT];     // the selected frames of the tile (thread indices), in frame order
    uint32_t len[GT];     // row length of each frame of the tile (0 unless selected and OK)
    uint32_t status[GT];  // its status
    uint32_t excl[GT];    // its row's offset inside the tile
};

__global__ void __launch_bounds__(GT, 3) proto_decode_nested_deferred_kernel(const GrpcParams p, const uint32_t* meta_in,
                                                                              const __grid_constant__ PbnDesc D) {
    __shared__ PdnDeferredShared sh;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * GT + tid;
        const bool valid = i < p.n;
        // (meta may be meta_in: each thread reads its own word here and writes it below, no one else's)
        const uint32_t m_in = valid ? meta_in[i] : GOFR_GRPC_OK;
        const bool selected = valid && m_in == GOFR_GRPC_DEFER;
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, selected);
        __syncthreads();  // the previous tile's reads of sh are done
        if (lane == 0) sh.warp_sel[warp] = __popc(ballot);
        sh.len[tid] = 0;
        sh.status[tid] = m_in;
        __syncthreads();
        uint32_t before = 0, n_sel = 0;
#pragma unroll
        for (int w = 0; w < GNW; w++) { if ((uint32_t)w < warp) before += sh.warp_sel[w]; n_sel += sh.warp_sel[w]; }
        if (selected) sh.sel[before + __popc(ballot & ((1u << lane) - 1u))] = tid;
        __syncthreads();
        for (uint32_t k = 0; k < n_sel; k++) {  // uniform: every thread walks the same frame
            const uint32_t j = sh.sel[k], fo = __ldg(p.in_off + tile * GT + j), fn = __ldg(p.in_off + tile * GT + j + 1) - fo;
            const PdnRow r = pdn_deferred_size(D, p.in + fo, fn);
            if (tid == 0) { sh.len[j] = r.out_len; sh.status[j] = r.status; }
        }
        __syncthreads();
        const uint32_t len = sh.len[tid];
        const TilePlace t = place_tile(p, tile, len, sh.warp_sum, sh.tile_base);
        if (valid) {
            put_offsets(p.out_off, i, p.n, t, len);
            p.meta[i] = sh.status[tid];
        }
        sh.excl[tid] = t.excl;
        __syncthreads();
        if (!t.fits) continue;  // (the same for every thread)
        for (uint32_t k = 0; k < n_sel; k++) {
            const uint32_t j = sh.sel[k];
            if (!sh.len[j]) continue;
            const uint32_t fo = __ldg(p.in_off + tile * GT + j), fn = __ldg(p.in_off + tile * GT + j + 1) - fo;
            pdn_deferred_emit(D, p.in + fo, fn, PdnRow{GOFR_GRPC_OK, sh.len[j]}, p.out + t.base + sh.excl[j]);
        }
    }
}

}  // namespace gofr
