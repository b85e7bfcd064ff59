// proto_nested_kernel.cu — rows -> proto3 messages with nested and repeated fields (gofr_proto_encode_nested_device): the
// tile loop of the gRPC message path (frame_tiles.cuh) around the walker of proto_nested_device.cuh.  Its own translation
// unit, so that the flat encoder / decoder and the Hello kernel (grpc_kernel.cu) stay the binaries that were measured.
// This kernel takes map-free descriptions; those with map fields run proto_encode_nested_maps_kernel.
#include "proto_nested_codecs.cuh"

namespace gofr {

__global__ void __launch_bounds__(GT, 6) proto_encode_nested_kernel(const GrpcParams p, const __grid_constant__ PbnDesc D) {
    __shared__ __align__(16) GrpcShared sh;
    frame_tiles(p, PbnCodec<false>{D}, sh);
}

}  // namespace gofr
