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

int serve_slots_wide_blocks_per_sm(uint32_t smem_bytes);
int launch_serve_slots_wide(const ServeParams& p, int grid, uint32_t smem_bytes, void* stream);
int serve_slots_values_blocks_per_sm(uint32_t smem_bytes);
int launch_serve_slots_values(const ServeParams& p, int grid, uint32_t smem_bytes, void* stream);

int serve_slots_blocks_per_sm(uint32_t smem_bytes, bool wide) {
    if (wide) return serve_slots_wide_blocks_per_sm(smem_bytes);
    const int nv = serve_slots_values_blocks_per_sm(smem_bytes);
    if (nv < 0) return -1;
    if (cudaFuncSetAttribute(serve_slots_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes) != cudaSuccess) return -1;
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, serve_slots_kernel, T, smem_bytes) != cudaSuccess) return -1;
    return nb < nv ? nb : nv;
}

int launch_serve_slots(const ServeParams& p, int grid, uint32_t smem_bytes, void* stream, bool wide, bool values) {
    if (values) return launch_serve_slots_values(p, grid, smem_bytes, stream);
    if (wide) return launch_serve_slots_wide(p, grid, smem_bytes, stream);
    serve_slots_kernel<<<grid, T, smem_bytes, (cudaStream_t)stream>>>(p);
    return (int)cudaGetLastError();
}

}  // namespace gofr
