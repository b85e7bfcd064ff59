// emu_conn_log.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the request-log gather's per-connection code (gofr_b200/csrc/conn_log_device.cuh, the same __host__ __device__
// functions conn_log_kernel.cu calls) on the CPU, connection after connection: the running line count stands in for the
// kernel's scan and look-back, which only exist on the device and are covered by the `-m gpu` tests.  Nothing in the product
// links or loads this file.
#include <cstdint>
#include <cstring>

#include "../../gofr_b200/csrc/conn_log_device.cuh"

using namespace gofr;

extern "C" void emu_conn_log(const uint32_t* first, const uint32_t* conn_status, const uint32_t* req_first, const uint32_t* rec_off,
                             const unsigned long long* spans, const uint32_t* meta, const uint8_t* ids, const uint8_t* buf,
                             const uint8_t* remote, const uint32_t* remote_off, const int64_t* start_ns, int64_t log_ns,
                             int32_t tz_offset_s, uint32_t alo, uint32_t remote_max, uint32_t req0, uint32_t n_conns,
                             gofr_log_desc* out, uint32_t* line_first, uint8_t* line_ids, uint32_t* line_req, uint8_t* arena) {
    ConnLogParams p;
    memset(&p, 0, sizeof p);
    p.first = first; p.conn_status = conn_status; p.req_first = req_first; p.rec_off = rec_off; p.spans = spans; p.meta = meta;
    p.ids = ids; p.buf = buf; p.remote = remote; p.remote_off = remote_off; p.start_ns = start_ns; p.log_ns = log_ns;
    p.tz_offset_s = tz_offset_s; p.alo = alo; p.remote_max = remote_max; p.req0 = req0; p.n = n_conns;
    p.out = (uint8_t*)out; p.line_ids = line_ids; p.line_req = line_req; p.arena = arena;
    uint32_t m = 0;
    for (uint32_t c = 0; c < n_conns; c++) {
        const uint32_t count = conn_requests(first, conn_status, c), k0 = req_first[c] - req0;
        const uint32_t lines = conn_log_count(p, first[c], k0, count);
        line_first[c] = m;
        conn_log_put(p, c, first[c], k0, count, m);
        m += lines;
    }
    line_first[n_conns] = m;
}
