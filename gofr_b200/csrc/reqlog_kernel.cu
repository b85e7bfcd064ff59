// reqlog_kernel.cu — the RequestLog JSON line of middleware.Logging for a whole batch (sm_90a): every record has its
// line.  The tile loop is reqlog_tiles.cuh.
#include "reqlog_tiles.cuh"

namespace gofr {

struct EveryRecord {
    static constexpr bool kEvery = true;
    __device__ __forceinline__ bool operator()(uint32_t, LogDesc&) const { return true; }
};

__global__ void __launch_bounds__(LT, 5) reqlog_kernel(const LogParams p) {
    reqlog_tiles(p, EveryRecord());
}

}  // namespace gofr
