// serve_slots_kernel.cu — slot-layout instance of the serve kernel (serve_body.cuh): the resident headline kernel.
//
// Two register budgets of the same body exist: this one (5 CTAs/SM, 96 registers) and serve_slots_wide_kernel.cu (4 CTAs/SM,
// 128 registers, for tables that answer with one fast-path program shape: engine.cu choose_slot_residency).  The kernel is
// issue/latency bound; the staging budget keeps each instance's CTAs really resident (occupancy calculator, engine.cu).
// Each register budget is its own translation unit, as __launch_bounds__ applies to a whole kernel.
// Like the packed instance of serve_kernel.cu, this one and the wide one are compiled without the programs of the wider
// data model (GOFR_TU_VALUES 0); tables that have such programs run serve_slots_values_kernel.cu.
#define GOFR_TU_VALUES 0
#include "serve_body.cuh"

namespace gofr {

__global__ void __launch_bounds__(T, kServeCtas) serve_slots_kernel(const __grid_constant__ ServeParams p) { serve_body<true>(p); }

}  // namespace gofr
