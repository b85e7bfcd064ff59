// serve_values_kernel.cu — packed-layout instance of the serve kernel for tables with programs of the wider data model
// (PF_VALUES); see serve_kernel.cu.
#define GOFR_TU_VALUES 1
#include "serve_body.cuh"

namespace gofr {

__global__ void __launch_bounds__(T, kServeCtas) serve_kernel_values(const __grid_constant__ ServeParams p) { serve_body<false>(p); }

}  // namespace gofr
