// grpc_kernel.cu — the gRPC message path over batches of length-prefixed frames, sm_90a: the unary Hello of config 5
// (request frame → response frame) and the proto3 encoder / decoder for any flat message type (rows ↔ frames).
// The tile loop is frame_tiles.cuh, on the skeleton of tile_common.cuh.  Per-frame logic: grpc_device.cuh.
#include "frame_tiles.cuh"

namespace gofr {

struct HelloCodec {
    typedef HelloReq R;
    __device__ R none() const { return HelloReq{GOFR_GRPC_OK, 0, 0, 0}; }
    __device__ R parse(const uint8_t* f, uint32_t fn, uint32_t) const { return hello_parse(f, fn); }
    __device__ void emit(const uint8_t* f, const R& r, uint8_t* dst, uint32_t* col) const { hello_emit(f, r, dst, col); }
};

struct ProtoCodec {
    typedef ProtoMsg R;
    const ProtoSchema& S;
    __device__ R none() const { return ProtoMsg{GOFR_GRPC_OK, 0}; }
    __device__ R parse(const uint8_t* row, uint32_t rn, uint32_t off) const { return proto_size(S, row, rn, (off & 3u) == 0); }
    __device__ void emit(const uint8_t* row, const R& r, uint8_t* dst, uint32_t* col) const { proto_emit(S, row, r, dst, col); }
};

struct ProtoDecodeCodec {
    typedef ProtoRow R;
    const ProtoSchema& S;
    __device__ R none() const { ProtoRow r; r.status = GOFR_GRPC_OK; r.out_len = 0; return r; }
    __device__ R parse(const uint8_t* f, uint32_t fn, uint32_t) const { ProtoRow r; proto_decode_scan(S, f, fn, r); return r; }
    __device__ void emit(const uint8_t* f, const R& r, uint8_t* dst, uint32_t* col) const { proto_decode_emit(S, f, r, dst, col); }
};

__global__ void __launch_bounds__(GT, 12) grpc_hello_kernel(const GrpcParams p) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, HelloCodec{}, sh);
}

// rows → proto3 messages (gofr_proto_encode_device): the same pipeline, the row in place of the request frame
__global__ void __launch_bounds__(GT, 8) proto_encode_kernel(const GrpcParams p, const __grid_constant__ ProtoSchema S) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, ProtoCodec{S}, sh);
}

// frames → rows (gofr_proto_decode_device)
__global__ void __launch_bounds__(GT, 8) proto_decode_kernel(const GrpcParams p, const __grid_constant__ ProtoSchema S) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, ProtoDecodeCodec{S}, sh);
}

}  // namespace gofr
