// serve_slots_wide_kernel.cu — slot-layout instance of the serve kernel with the 128-register budget (4 CTAs/SM); see
// serve_slots_kernel.cu for when the engine uses it.  Its tables answer with one fast-path program shape, so the lanes of
// a warp walk the same ops and this instance stores whole 128-byte lines (LINES: serve_body.cuh).
#define GOFR_TU_VALUES 0
#include "serve_body.cuh"

namespace gofr {

__global__ void __launch_bounds__(T, kServeCtasWide) serve_slots_kernel_wide(const __grid_constant__ ServeParams p) { serve_body<true, true>(p); }

}  // namespace gofr
