// route_kernel.cu — stage 1 of the split API for routes whose closure runs on the host (GOFR_H_HOST), sm_90a.
//
// What mux.Router.ServeHTTP and the middleware chain decide before handler.ServeHTTP is reached
// (pkg/gofr/http/router.go:14,30-33; middleware/cors.go:10-13; pkg/gofr/handler.go:32-36): cleanPath redirect, the
// matched route (mux first-match with the ErrMethodMismatch bookkeeping) and the path variables mux.Vars would hold
// (pkg/gofr/http/request.go:36-38).  One thread per request; only descriptors and path bytes are read, so the kernel
// moves ~50 bytes per request and is bound by the latency of the short per-request walks, not by HBM.
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"
#include "serve_device.cuh"

namespace gofr {

constexpr int RT = kRouteThreads;

__global__ void __launch_bounds__(RT) route_kernel(const RouteParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    {
        const uint4* src = (const uint4*)p.image;
        uint4* dst = (uint4*)smem;
        for (uint32_t i = threadIdx.x; i < p.hot_bytes / 16; i += RT) dst[i] = src[i];
    }
    __syncthreads();
    TableView tv;
    tv.bind(smem, p.image);
    for (uint32_t i = blockIdx.x * RT + threadIdx.x; i < p.n; i += gridDim.x * RT) {
        const uint4 d = __ldg((const uint4*)p.desc + i);
        const uint32_t path_len = d.y & 0xFFFFu, method = d.w & 0xFFu;
        uint32_t route, vars[kMaxVars];
        const uint32_t status = route_only(tv, method, p.arena + d.x, path_len, &route, vars);
        p.meta[i] = status | route << 16;
        uint4* v = (uint4*)(p.vars + (size_t)i * kMaxVars);
        v[0] = make_uint4(vars[0], vars[1], vars[2], vars[3]);
        v[1] = make_uint4(vars[4], vars[5], vars[6], vars[7]);
    }
}
static_assert(kMaxVars == 8, "two 16-byte stores per request");

}  // namespace gofr
