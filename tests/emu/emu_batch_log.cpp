// emu_batch_log.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs gofr_batch_submit_log's per-request line decision (gofr_b200/csrc/batch_log_device.cuh, the same __host__ __device__
// function batch_log_kernel.cu calls) on the CPU, request after request.  Nothing in the product links or loads this file.
#include <cstdint>

#include "../../gofr_b200/csrc/batch_log_device.cuh"

using namespace gofr;

extern "C" void emu_batch_log(gofr_log_desc* desc, const uint32_t* meta, int64_t log_ns, uint32_t n, uint8_t* has_line) {
    for (uint32_t i = 0; i < n; i++) has_line[i] = batch_log_fill(desc[i], meta[i], log_ns) ? 1 : 0;
}
