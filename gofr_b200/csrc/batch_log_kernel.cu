// batch_log_kernel.cu — the serve-fed instance of the request-log kernel (sm_90a), the log step of gofr_batch_submit_log:
// record i of a chunk takes its status from the serve kernel's meta[i] and the batch's clock (batch_log_device.cuh), and a
// request the middleware does not wrap gets an empty line.  The tile loop is reqlog_tiles.cuh, as for reqlog_kernel.cu.
// Each warp adds its lines to *lines, the batch's line count, so that it never has to come back mid-batch.
#include "batch_log_device.cuh"
#include "reqlog_tiles.cuh"

namespace gofr {

struct ServeFed {
    static constexpr bool kEvery = false;
    const uint32_t* meta;
    int64_t log_ns;
    unsigned long long* lines;
    __device__ __forceinline__ bool operator()(uint32_t i, LogDesc& d) const {
        static_assert(sizeof(LogDesc) == sizeof(gofr_log_desc), "LogDesc is gofr_log_desc");
        gofr_log_desc g;
        memcpy(&g, &d, sizeof g);
        const bool line = batch_log_fill(g, __ldg(meta + i), log_ns);
        memcpy(&d, &g, sizeof g);
        return count_line(line, lines);
    }
};

__global__ void __launch_bounds__(LT, 5) batch_log_kernel(const LogParams p, const uint32_t* meta, int64_t log_ns,
                                                          unsigned long long* lines) {
    reqlog_tiles(p, ServeFed{meta, log_ns, lines});
}

}  // namespace gofr
