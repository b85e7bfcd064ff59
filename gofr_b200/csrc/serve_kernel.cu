// serve_kernel.cu — packed-layout instance of the serve kernel (serve_body.cuh); engine.cu launches it.
//
// This instance does not know the programs of the wider data model (PF_VALUES: float64, pointers, slices, maps ...): the
// packed layout has the interpreter inlined in its tile loop, and the two extra call sites cost every table registers
// (serve_device.cuh GOFR_TU_VALUES).  Tables that contain such a program are served by serve_values_kernel.cu.
#define GOFR_TU_VALUES 0
#include "serve_body.cuh"

namespace gofr {

__global__ void __launch_bounds__(T, kServeCtas) serve_kernel(const __grid_constant__ ServeParams p) { serve_body<false>(p); }

}  // namespace gofr
