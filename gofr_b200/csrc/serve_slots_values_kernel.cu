// serve_slots_values_kernel.cu — slot-layout instance of the serve kernel for tables with programs of the wider data model
// (PF_VALUES); see serve_slots_kernel.cu and serve_device.cuh GOFR_TU_VALUES.
#define GOFR_TU_VALUES 1
#include "serve_body.cuh"

namespace gofr {

__global__ void __launch_bounds__(T, kServeCtas) serve_slots_kernel_values(const __grid_constant__ ServeParams p) { serve_body<true>(p); }

}  // namespace gofr
