// proto_nested_codecs.cuh — the nested proto3 encoder and decoder as codecs of the gRPC message path's tile loop
// (frame_tiles.cuh), for the kernels of proto_nested_kernel.cu, proto_nested_decode_kernel.cu, proto_nested_maps_kernel.cu
// and proto_nested_presence_kernel.cu.  MAPS is PbnDesc::maps and PRES PbnDesc::presence (with MAPS), chosen on the host
// per launch: map-free descriptions run kernels that contain no map code, presence-free ones kernels without presence code.
#pragma once
#include "frame_tiles.cuh"
#include "proto_nested_decode_device.cuh"

namespace gofr {

template <bool MAPS, bool PRES = false>
struct PbnCodec {
    typedef PbnMsg R;
    const PbnDesc& D;
    __device__ R none() const { return PbnMsg{GOFR_GRPC_OK, 0}; }
    __device__ R parse(const uint8_t* row, uint32_t rn, uint32_t) const { R r = pbn_size_as<MAPS, PRES>(D, row, rn); rn_of = rn; return r; }
    __device__ void emit(const uint8_t* row, const R& r, uint8_t* dst, uint32_t* col) const { pbn_emit_as<MAPS, PRES>(D, row, rn_of, r, dst, col); }
    mutable uint32_t rn_of = 0;  // the row's length, from parse to emit (one codec object per thread)
};

template <bool MAPS, bool PRES = false>
struct PdnCodec {
    typedef PdnRow R;
    const PbnDesc& D;
    __device__ R none() const { return PdnRow{GOFR_GRPC_OK, 0}; }
    __device__ R parse(const uint8_t* f, uint32_t fn, uint32_t) const { fn_of = fn; return pdn_decode_size_as<MAPS, PRES>(D, f, fn); }
    __device__ void emit(const uint8_t* f, const R& r, uint8_t* dst, uint32_t*) const { pdn_decode_emit_as<MAPS, PRES>(D, f, fn_of, r, dst); }
    mutable uint32_t fn_of = 0;  // the frame's length, from parse to emit (one codec object per thread)
};

}  // namespace gofr
