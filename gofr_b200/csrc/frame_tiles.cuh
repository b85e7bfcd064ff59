// frame_tiles.cuh — the tile loop shared by the frame codecs of the gRPC message path (grpc_kernel.cu: Hello, proto3 encoder /
// decoder for flat messages; proto_nested_*kernel.cu: the nested codecs), one thread per frame, on the tile skeleton of
// tile_common.cuh; frames are packed in order through the staging Writer.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"
#include "grpc_device.cuh"
#include "tile_common.cuh"

namespace gofr {

constexpr int GT = kServeThreads;
constexpr int GNW = GT / 32;
constexpr uint32_t kGrpcStage = 8 * 1024;  // bytes of input frames staged per tile (128 frames × ≤ 64 B)

struct GrpcShared {
    uint64_t bar;
    uint32_t warp_sum[GNW];
    unsigned long long tile_base;
    uint32_t stage[GOFR_STAGE_WORDS * GT];
    __align__(16) uint8_t in[kGrpcStage + 32];
};

// The tile loop shared by the two frame codecs (Hello request → response, row → proto3 message).
template <class Codec>
__device__ __forceinline__ void frame_tiles(const GrpcParams& p, const Codec& cd, GrpcShared& sh) {
    const uint32_t tid = threadIdx.x;
    if (tid == 0) tile_barrier_init(&sh.bar);
    __syncthreads();
    uint32_t parity = 0;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * GT + tid;
        const bool valid = i < p.n;
        const ByteRange in = offset_range(p.in_off, tile * GT, min(p.n, tile * GT + GT));
        __syncthreads();  // previous tile's reads of sh.in are done
        stage_start(&sh.bar, sh.in, p.in, in, kGrpcStage);
        uint32_t fo = 0, fn = 0;
        if (valid) { fo = __ldg(p.in_off + i); fn = __ldg(p.in_off + i + 1) - fo; }
        const uint8_t* base = stage_wait(&sh.bar, parity, sh.in, p.in, in, kGrpcStage);
        typename Codec::R r = cd.none();
        if (valid) r = cd.parse(base + fo, fn, fo);

        const TilePlace t = place_tile(p, tile, r.out_len, sh.warp_sum, sh.tile_base);
        if (valid) {
            put_offsets(p.out_off, i, p.n, t, r.out_len);
            p.meta[i] = r.status;
        }
        if (t.fits && valid && r.out_len) cd.emit(base + fo, r, p.out + t.base + t.excl, &sh.stage[tid]);
    }
}

}  // namespace gofr
