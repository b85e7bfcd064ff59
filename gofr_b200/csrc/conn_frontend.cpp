// conn_frontend.cpp — per-read front-end of the connection pipeline: net/http runs one goroutine per connection (conn.serve
// looping readRequest, pkg/gofr/httpServer.go:29-33), and each holds only its own received bytes; gofr_conn_batch_submit_log
// wants a batch of connections.  Callers hand in one read each (a connection's kept tail plus its new bytes) and block on
// frontend_ring.h's ring; its dispatcher runs each closed batch through gofr_conn_batch_submit_log and every caller copies
// its own connection's responses, columns and log lines out, rebased to its own buffers.
//
// Written against the public ABI only (gofr_conn_batch_submit_log, gofr_batch_wait, the pinned allocator,
// gofr_format_http_date), as proto_frontend.cpp is, so that tests/emu/conn_frontend_stress.cpp runs it against stub batch
// calls under ThreadSanitizer.
//
// Staging, output growth and fan-out are conn_staging.h's, shared with conn_app_frontend.cpp.
#include "../../include/gofr_b200.h"
#include "conn_staging.h"
#include "engine_internal.h"
#include "frontend_ring.h"

using Staging = ConnStaging;

struct gofr_conn_frontend {
    gofr_conn_frontend(uint32_t max_batch, uint32_t max_wait_us) : ring(max_batch, max_wait_us) {}
    gofr_engine* eng = nullptr;
    uint32_t max_conn_bytes = 0;
    bool log = false;
    int32_t tz_offset_s = 0;
    uint64_t seed = 0, batch_no = 0;       // batch_no: the dispatcher's alone
    std::atomic<int64_t> fixed_clock{0};   // tests: Date and log time of every batch, in ns; 0 = wall clock
    std::atomic<uint64_t> reruns{0};
    Staging b[gofr_ring::kBatches];
    gofr_ring::Ring ring;
};
using ConnFrontend = gofr_conn_frontend;

// the dispatcher's step: batch k's n reads (arena_bytes in all) through gofr_conn_batch_submit_log
static int serve_batch(ConnFrontend* f, int k, uint32_t n, uint32_t arena_bytes) {
    const ConnServe s{f->eng, f->log, f->tz_offset_s, batch_seed(f->seed, f->batch_no++), batch_clock(f->fixed_clock), &f->reruns,
                      "gofr_conn_frontend"};
    return serve_staged(f->b[k], n, arena_bytes, s, [f](const gofr_conn_batch* in, gofr_conn_resp* out, gofr_conn_log* lg, gofr_ticket* t) {
        return gofr_conn_batch_submit_log(f->eng, in, out, lg, t);
    });
}

extern "C" {

int gofr_conn_frontend_create(gofr_conn_frontend** out, gofr_engine* e, uint32_t max_batch, uint32_t max_wait_us,
                              uint32_t max_conn_bytes, int log, int32_t tz_offset_s, uint64_t seed) {
    if (!out || !e || max_batch == 0 || max_batch > 0x7FFFFFFFu) return GOFR_ERR_INVALID;
    // the ring claims arena bytes in 32 bits, and buf_off is 32-bit
    const uint64_t arena = (uint64_t)max_batch * max_conn_bytes;
    if (arena > 0xFFFFFFF0ull) {
        set_last_error("gofr_conn_frontend_create: %u reads of %u bytes exceed 32-bit offsets", max_batch, max_conn_bytes);
        return GOFR_ERR_CAPACITY;
    }
    ConnFrontend* f = new ConnFrontend(max_batch, max_wait_us);
    f->eng = e;
    f->max_conn_bytes = max_conn_bytes;
    f->log = log != 0;
    f->tz_offset_s = tz_offset_s;
    f->seed = seed;
    for (auto& x : f->b) {
        if (!alloc_staging(x, max_batch, arena)) {
            for (auto& y : f->b) free_staging(y);
            delete f;
            return GOFR_ERR_NOMEM;
        }
    }
    f->ring.start([f](int k, uint32_t n, uint32_t arena_bytes) { return serve_batch(f, k, n, arena_bytes); });
    *out = f;
    return GOFR_OK;
}

void gofr_conn_frontend_destroy(gofr_conn_frontend* f) {
    if (!f) return;
    f->ring.stop();
    for (auto& x : f->b) free_staging(x);
    delete f;
}

int gofr_conn_frontend_set_clock(gofr_conn_frontend* f, int64_t unix_ns) {
    if (!f) return GOFR_ERR_INVALID;
    f->fixed_clock.store(unix_ns, std::memory_order_relaxed);
    return GOFR_OK;
}

int gofr_conn_frontend_stats(gofr_conn_frontend* f, uint64_t* batches, uint64_t* conns, uint64_t* reruns) {
    if (!f) return GOFR_ERR_INVALID;
    if (batches) *batches = f->ring.batches.load(std::memory_order_relaxed);
    if (conns) *conns = f->ring.records.load(std::memory_order_relaxed);
    if (reruns) *reruns = f->reruns.load(std::memory_order_relaxed);
    return GOFR_OK;
}

int gofr_conn_frontend_serve(gofr_conn_frontend* f, const uint8_t* buf, uint32_t len, const uint8_t* remote, uint32_t remote_len,
                             int64_t start_unix_ns, gofr_conn_resp* out, gofr_conn_log* log) {
    if (!f) return GOFR_ERR_INVALID;
    if (int rc = check_read(len, buf, remote, remote_len, out, &log, f->log)) return rc;
    if (len > f->max_conn_bytes) {
        set_last_error("a read of %u bytes exceeds the front-end's max_conn_bytes", len);
        return GOFR_ERR_CAPACITY;
    }
    if (len == 0) {  // nothing to frame: done without joining a batch
        no_requests(out, log, 0, GOFR_HTTP_CONN_DONE);
        return GOFR_OK;
    }
    gofr_ring::Seat s;
    if (!f->ring.claim(len, &s)) return GOFR_ERR_INVALID;
    Staging& x = f->b[s.k];
    memcpy(x.arena + s.a, buf, len);
    x.buf_off[s.i] = s.a;
    if (remote_len) memcpy(x.remote_at + (size_t)s.i * kRemoteMax, remote, remote_len);
    x.remote_len[s.i] = remote_len;
    x.start[s.i] = start_unix_ns;
    f->ring.filled(s);

    const uint32_t n = f->ring.wait(s);
    int rc = f->ring.b[s.k].rc;
    if (rc == GOFR_OK) rc = fan_out(x, s.i, s.a, out, log);
    f->ring.leave(s, n);
    return rc;
}

}  // extern "C"
