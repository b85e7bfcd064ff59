// proto_nested_presence_kernel.cu — the nested proto3 encoder and decoder for descriptions WITH explicit-presence fields
// (PbnDesc::presence: proto3 optional, oneof members), with map code as well.  A translation unit of its own, so that the
// kernels of the other nested units contain no presence code and are register-allocated as before presence existed.
#include "proto_nested_codecs.cuh"

namespace gofr {

__global__ void __launch_bounds__(GT, 6) proto_encode_nested_presence_kernel(const GrpcParams p, const __grid_constant__ PbnDesc D) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, PbnCodec<true, true>{D}, sh);
}

__global__ void __launch_bounds__(GT, 6) proto_decode_nested_presence_kernel(const GrpcParams p, const __grid_constant__ PbnDesc D) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, PdnCodec<true, true>{D}, sh);
}

}  // namespace gofr
