// emu_http_frame.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the framer's per-connection code (gofr_b200/csrc/http_frame_device.cuh, the same __host__ __device__ functions
// http_frame_kernel.cu calls: the count walk, then the walk that stores the record starts) on the CPU, connection after
// connection, against the oracle.  Tile staging, the scan and the look-back only exist in the kernel and are covered by the
// `-m gpu` tests.  Returns 1 when rec_cap records do not hold the column (first is still complete).  Nothing in the product
// links or loads this file.
#include <cstdint>
#include <cstring>

#include "../../gofr_b200/csrc/http_frame_device.cuh"

using namespace gofr;

extern "C" int emu_http_frame(const uint8_t* buf, const uint32_t* buf_off, uint32_t n_conns, uint32_t* rec_off, uint32_t rec_cap,
                              uint32_t* first, uint32_t* consumed, uint32_t* status) {
    uint64_t total = 0;
    for (uint32_t c = 0; c < n_conns; c++) {
        const uint32_t co = buf_off[c], cn = buf_off[c + 1] - co;
        HttpFrameConn f;
        http_frame_count(buf + co, cn, f);
        first[c] = (uint32_t)total;
        consumed[c] = f.consumed;
        status[c] = f.status;
        if (total + f.count <= rec_cap) http_frame_put(buf + co, cn, f, co, rec_off + total);
        total += f.count;
    }
    if (n_conns) {
        first[n_conns] = (uint32_t)total;
        if (total <= rec_cap) rec_off[total] = buf_off[n_conns];
    }
    return total > rec_cap;
}
