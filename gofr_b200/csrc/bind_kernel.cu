// bind_kernel.cu — gofr_bind_device: Request.Bind as a stage of the split API.
//
// Replaces, for closures that stay on the host, the json.Unmarshal inside Context.Bind (pkg/gofr/context.go:52-54,
// pkg/gofr/http/request.go:40-47): the GPU decodes every request body of a batch into the typed row of a registered struct
// (or into err.Error()), the host closure's Bind then only copies fields out of its row.  One thread per request; result i
// in its own slot (no scan, no dependence between requests); the scanner and decoder are bind_device.cuh — the very code
// the fused GOFR_H_BIND_ECHO routes run.
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"
#include "serve_device.cuh"

namespace gofr {

constexpr int BT = kBindThreads;

__global__ void __launch_bounds__(BT) bind_kernel(const BindParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ uint32_t ring[GOFR_STAGE_WORDS * BT];
    {
        const uint4* src = (const uint4*)p.image;
        uint4* dst = (uint4*)smem;
        for (uint32_t i = threadIdx.x; i < p.hot_bytes / 16; i += BT) dst[i] = src[i];
    }
    __syncthreads();
    TableView tv;
    tv.bind(smem, p.image);
    uint32_t row[BR_FIELDS + 2 * kMaxFields];
    for (uint32_t i = blockIdx.x * BT + threadIdx.x; i < p.n; i += gridDim.x * BT) {
        const uint4 d = __ldg((const uint4*)p.desc + i);
        const uint32_t data_off = (d.x + (d.y & 0xFFFFu) + (d.y >> 16) + 3u) & ~3u;
        const uint8_t* body = p.arena + data_off;
        bind_request(tv, p.schema_idx, body, d.z, row);
        const uint32_t st = bind_row_status(row);
        uint32_t len = 0;
        if (st != 2u) {
            len = bind_row_out<false>(nullptr, tv, p.schema_idx, body, row);
            if (len && len <= p.slot_bytes) {
                Writer w;
                w.init(p.out + (size_t)i * p.slot_bytes, &ring[threadIdx.x]);
                bind_row_out<true>(&w, tv, p.schema_idx, body, row);
                w.finish_padded();
            }
        }
        p.len[i] = len;
        p.status[i] = st;
    }
}

}  // namespace gofr
