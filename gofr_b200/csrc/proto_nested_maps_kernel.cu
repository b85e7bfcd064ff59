// proto_nested_maps_kernel.cu — the nested proto3 encoder and decoder for descriptions WITH map fields (PbnDesc::maps).  A
// translation unit of their own, so that the map-free kernels (proto_nested_kernel.cu, proto_nested_decode_kernel.cu)
// contain no map code and are register-allocated as before maps existed.
#include "proto_nested_codecs.cuh"

namespace gofr {

__global__ void __launch_bounds__(GT, 6) proto_encode_nested_maps_kernel(const GrpcParams p, const __grid_constant__ PbnDesc D) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, PbnCodec<true>{D}, sh);
}

__global__ void __launch_bounds__(GT, 6) proto_decode_nested_maps_kernel(const GrpcParams p, const __grid_constant__ PbnDesc D) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, PdnCodec<true>{D}, sh);
}

}  // namespace gofr
