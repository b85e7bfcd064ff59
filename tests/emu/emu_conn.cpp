// emu_conn.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the compact step's per-connection code (gofr_b200/csrc/conn_device.cuh, the same __host__ __device__ functions
// conn_kernel.cu calls) on the CPU, connection after connection: the running request count stands in for the kernel's scan
// and look-back, which only exist on the device and are covered by the `-m gpu` tests.  Nothing in the product links or
// loads this file.
#include <cstdint>
#include <cstring>

#include "../../gofr_b200/csrc/conn_device.cuh"

using namespace gofr;

extern "C" void emu_conn_compact(const uint32_t* first, const uint32_t* conn_status, const uint32_t* rec_off, const gofr_req_desc* desc_in,
                                 uint32_t n_conns, uint64_t seed, uint32_t conn0, uint32_t req0, gofr_req_desc* desc_out,
                                 uint32_t* req_at, uint8_t* ids, uint32_t* req_first) {
    uint32_t k = 0;
    for (uint32_t c = 0; c < n_conns; c++) {
        const uint32_t count = conn_requests(first, conn_status, c);
        req_first[c] = req0 + k;
        conn_put(desc_in, rec_off, first[c], count, conn_trace_key(seed, conn0 + c), desc_out, req_at, ids, k);
        k += count;
    }
    req_first[n_conns] = req0 + k;
}

extern "C" void emu_conn_trace_id(uint64_t seed, uint32_t c, uint32_t j, uint8_t* out16) {
    conn_trace_id(conn_trace_key(seed, c), j, out16);
}
