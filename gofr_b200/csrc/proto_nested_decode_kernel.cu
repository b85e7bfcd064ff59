// proto_nested_decode_kernel.cu — length-prefixed frames -> rows for message types with nested and repeated fields
// (gofr_proto_decode_nested_device): the tile loop of the gRPC message path (frame_tiles.cuh) around the three walks of
// proto_nested_decode_device.cuh.  Its own translation unit, like the encoder's.  This kernel takes map-free
// descriptions; those with map fields run proto_decode_nested_maps_kernel.
#include "proto_nested_codecs.cuh"

namespace gofr {

__global__ void __launch_bounds__(GT, 6) proto_decode_nested_kernel(const GrpcParams p, const __grid_constant__ PbnDesc D) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, PdnCodec<false>{D}, sh);
}

}  // namespace gofr
