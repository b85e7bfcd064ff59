// emu_proto_log.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs gofr_proto_batch_encode_log's per-call line decision (gofr_b200/csrc/batch_log_device.cuh, the same __host__
// __device__ function proto_log_kernel.cu calls) on the CPU, record after record.  Nothing in the product links or loads
// this file.
#include <cstdint>

#include "../../gofr_b200/csrc/batch_log_device.cuh"

using namespace gofr;

extern "C" void emu_proto_log(gofr_log_desc* desc, int64_t log_ns, uint32_t n, uint8_t* has_line) {
    for (uint32_t i = 0; i < n; i++) has_line[i] = proto_log_fill(desc[i], log_ns) ? 1 : 0;
}
