// proto_log_kernel.cu — the proto-fed instance of the request-log kernel (sm_90a), the log step of
// gofr_proto_batch_encode_log: record i of a chunk gets the gRPC LoggingInterceptor's RPCLog line when its kind is
// GOFR_LOG_RPC, with the batch's clock (batch_log_device.cuh), and an empty line otherwise.  The tile loop is
// reqlog_tiles.cuh, as for reqlog_kernel.cu; each warp adds its lines to *lines, the batch's line count.
#include "batch_log_device.cuh"
#include "reqlog_tiles.cuh"

namespace gofr {

struct ProtoFed {
    static constexpr bool kEvery = false;
    int64_t log_ns;
    unsigned long long* lines;
    __device__ __forceinline__ bool operator()(uint32_t, LogDesc& d) const {
        static_assert(sizeof(LogDesc) == sizeof(gofr_log_desc), "LogDesc is gofr_log_desc");
        gofr_log_desc g;
        memcpy(&g, &d, sizeof g);
        const bool line = proto_log_fill(g, log_ns);
        memcpy(&d, &g, sizeof g);
        return count_line(line, lines);
    }
};

__global__ void __launch_bounds__(LT, 5) proto_log_kernel(const LogParams p, int64_t log_ns, unsigned long long* lines) {
    reqlog_tiles(p, ProtoFed{log_ns, lines});
}

}  // namespace gofr
