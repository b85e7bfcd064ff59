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
// The ring's claim word reserves slot i and arena range [a, a + len), so the reads lie back to back in slot order — exactly
// the batch call's buf_off contract:
//   caller      stores buf_off[i] = a, its read, its remote string (in a 255-byte place of its own) and its start clock;
//   dispatcher  stores buf_off[n], packs the remote strings back to back, pins the batch's trace seed, Date and log clock,
//               and grows the per-request columns to one request per 16 bytes plus one per connection (what the framer can
//               produce at most), so they never run short.  The response and log byte outputs start small and grow to what
//               the batch call reports when it returns GOFR_ERR_CAPACITY; the batch is then served again.  That is sound
//               because the call writes nothing past a capacity and the rerun sees the same bytes, seed, Date and clocks;
//               the always-sufficient bound is not allocated up front (for 64 KiB reads it is hundreds of MiB).
#include <algorithm>
#include <cstring>
#include <time.h>

#include "../../include/gofr_b200.h"
#include "engine_internal.h"
#include "frontend_ring.h"

static constexpr uint32_t kRemoteMax = 255;            // gofr_conn_batch_submit_log's limit on a remote string
static constexpr uint64_t kFirstOut = 64u << 10;        // the byte outputs' first capacity

struct gofr_conn_frontend_batch {
    // per connection (max_batch, + 1 for the offset columns)
    uint8_t* arena = nullptr;      // the reads back to back
    uint32_t* buf_off = nullptr;
    uint8_t* remote_at = nullptr;  // slot i's remote string at 255 * i, its length in remote_len[i]
    uint32_t* remote_len = nullptr;
    uint8_t* remote = nullptr;     // packed by the dispatcher
    uint32_t* remote_off = nullptr;
    int64_t* start = nullptr;
    uint32_t *req_first = nullptr, *consumed = nullptr, *conn_status = nullptr;
    // per request, grown by the dispatcher, never shrunk
    uint32_t req_cap = 0;
    uint32_t *out_off = nullptr, *meta = nullptr, *req_at = nullptr, *log_off = nullptr, *log_req = nullptr;
    uint8_t* ids = nullptr;
    // bytes, grown by the dispatcher, never shrunk
    uint8_t* out = nullptr;
    uint64_t out_cap = 0;
    uint8_t* log_out = nullptr;
    uint64_t log_cap = 0;
    uint32_t lines = 0;            // the batch's log lines
};
using Staging = gofr_conn_frontend_batch;

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

static uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

static void free_staging(Staging& x) {
    for (void* p : {(void*)x.arena, (void*)x.buf_off, (void*)x.remote_at, (void*)x.remote_len, (void*)x.remote, (void*)x.remote_off,
                    (void*)x.start, (void*)x.req_first, (void*)x.consumed, (void*)x.conn_status, (void*)x.out_off, (void*)x.meta,
                    (void*)x.req_at, (void*)x.log_off, (void*)x.log_req, (void*)x.ids, (void*)x.out, (void*)x.log_out})
        gofr_free_pinned(p);
    x = Staging();
}

// replaces *p by a pinned buffer of `bytes` (the old contents are not kept)
static bool regrow(void** p, size_t bytes) {
    gofr_free_pinned(*p);
    *p = gofr_alloc_pinned(bytes);
    return *p != nullptr;
}

static bool grow_requests(Staging& x, uint32_t req_cap) {
    if (req_cap <= x.req_cap) return true;
    const size_t n = (size_t)req_cap;
    x.req_cap = 0;
    bool ok = regrow((void**)&x.out_off, (n + 1) * 4) && regrow((void**)&x.meta, n * 4) && regrow((void**)&x.req_at, n * 4) &&
              regrow((void**)&x.ids, n * 16) && regrow((void**)&x.log_off, (n + 1) * 4) && regrow((void**)&x.log_req, n * 4);
    if (ok) x.req_cap = req_cap;
    return ok;
}

static bool grow_bytes(uint8_t** p, uint64_t* cap, uint64_t need) {
    if (need <= *cap) return true;
    const uint64_t c = std::max<uint64_t>((need + 0xFFFFu) & ~(uint64_t)0xFFFFu, kFirstOut);
    *cap = 0;
    if (!regrow((void**)p, (size_t)c)) return false;
    *cap = c;
    return true;
}

// the dispatcher's step: batch k's n reads (arena_bytes in all) through gofr_conn_batch_submit_log
static int serve_batch(ConnFrontend* f, int k, uint32_t n, uint32_t arena_bytes) {
    Staging& x = f->b[k];
    x.buf_off[n] = arena_bytes;
    x.remote_off[0] = 0;
    for (uint32_t i = 0; i < n; i++) {
        memcpy(x.remote + x.remote_off[i], x.remote_at + (size_t)i * kRemoteMax, x.remote_len[i]);
        x.remote_off[i + 1] = x.remote_off[i] + x.remote_len[i];
    }
    const uint32_t req_cap = arena_bytes / 16 + n;  // the framer's most: one request per 16 bytes plus one per connection
    if (!grow_requests(x, req_cap) || !grow_bytes(&x.out, &x.out_cap, kFirstOut) ||
        (f->log && !grow_bytes(&x.log_out, &x.log_cap, kFirstOut))) {
        set_last_error("gofr_conn_frontend: no pinned outputs for %u requests", req_cap);
        return GOFR_ERR_NOMEM;
    }
    gofr_conn_batch in;
    memset(&in, 0, sizeof in);
    in.buf = x.arena; in.buf_off = x.buf_off; in.buf_bytes = arena_bytes; in.n_conns = n;
    // the seed is mixed before the batch number is added: with splitmix64(seed + b), batch b's slot c and batch c's slot b
    // would get the same ids whenever seed + b and seed + c are slot numbers, as the id function mixes c the same way
    in.trace_seed = splitmix64(splitmix64(f->seed) + f->batch_no++);
    int64_t now = f->fixed_clock.load(std::memory_order_relaxed);
    if (!now) { struct timespec ts; clock_gettime(CLOCK_REALTIME, &ts); now = (int64_t)ts.tv_sec * 1000000000 + ts.tv_nsec; }
    gofr_format_http_date(now / 1000000000, in.date);
    for (;;) {
        gofr_conn_resp out;
        memset(&out, 0, sizeof out);
        out.out = x.out; out.out_cap = x.out_cap; out.req_cap = req_cap; out.out_off = x.out_off; out.meta = x.meta;
        out.req_at = x.req_at; out.trace_ids = x.ids; out.req_first = x.req_first; out.consumed = x.consumed;
        out.conn_status = x.conn_status;
        gofr_conn_log lg;
        memset(&lg, 0, sizeof lg);
        lg.remote = x.remote; lg.remote_off = x.remote_off; lg.start_unix_ns = x.start; lg.log_unix_ns = now;
        lg.tz_offset_s = f->tz_offset_s; lg.line_cap = req_cap; lg.out = x.log_out; lg.out_cap = x.log_cap;
        lg.log_off = x.log_off; lg.log_req = x.log_req;
        gofr_ticket t = 0;
        int rc = gofr_conn_batch_submit_log(f->eng, &in, &out, f->log ? &lg : nullptr, &t);
        if (rc == GOFR_OK) rc = gofr_batch_wait(f->eng, t);
        x.lines = f->log ? lg.lines : 0;
        if (rc != GOFR_ERR_CAPACITY) return rc;
        // the call reported what the batch needs: grow to it and serve the same batch again (a need the outputs already
        // hold is one no capacity fixes, such as log offsets past 32 bits)
        const bool more = out.out_bytes > x.out_cap || (f->log && lg.out_bytes > x.log_cap);
        if (!more) return rc;
        if (!grow_bytes(&x.out, &x.out_cap, out.out_bytes) || (f->log && !grow_bytes(&x.log_out, &x.log_cap, lg.out_bytes))) {
            set_last_error("gofr_conn_frontend: no pinned output of %llu response and %llu log bytes",
                           (unsigned long long)out.out_bytes, (unsigned long long)lg.out_bytes);
            return GOFR_ERR_NOMEM;
        }
        f->reruns.fetch_add(1, std::memory_order_relaxed);
    }
}

// what a call returns for a connection without requests or bytes
static void no_requests(gofr_conn_resp* out, gofr_conn_log* log, uint32_t consumed, uint32_t status) {
    out->out_off[0] = 0;
    out->req_first[0] = out->req_first[1] = 0;
    out->consumed[0] = consumed;
    out->conn_status[0] = status;
    out->out_bytes = 0;
    if (log) {
        log->lines = 0;
        log->out_bytes = 0;
        if (log->log_off) log->log_off[0] = 0;
    }
}

// slot i's share of batch x, rebased to the caller's buffers; GOFR_ERR_CAPACITY when one of the caller's capacities is short
static int fan_out(const Staging& x, uint32_t i, uint32_t a, gofr_conn_resp* out, gofr_conn_log* log) {
    const uint32_t k0 = x.req_first[i], k1 = x.req_first[i + 1], nreq = k1 - k0;
    const uint32_t o0 = nreq ? x.out_off[k0] : 0, bytes = nreq ? x.out_off[k1] - o0 : 0;
    int rc = GOFR_OK;
    no_requests(out, log, x.consumed[i], x.conn_status[i]);
    out->req_first[1] = nreq;
    out->out_bytes = bytes;
    if (nreq > out->req_cap || bytes > out->out_cap) {
        rc = GOFR_ERR_CAPACITY;
    } else {
        if (bytes) memcpy(out->out, x.out + o0, bytes);
        for (uint32_t j = 0; j < nreq; j++) {
            out->out_off[j + 1] = x.out_off[k0 + j + 1] - o0;
            out->meta[j] = x.meta[k0 + j];
            out->req_at[j] = x.req_at[k0 + j] - a;
        }
        if (out->trace_ids && nreq) memcpy(out->trace_ids, x.ids + (size_t)k0 * 16, (size_t)nreq * 16);
    }
    if (!log) return rc;
    // the connection's lines: log_req holds batch request indices in ascending order, so they are one run
    const uint32_t m0 = (uint32_t)(std::lower_bound(x.log_req, x.log_req + x.lines, k0) - x.log_req);
    const uint32_t m1 = (uint32_t)(std::lower_bound(x.log_req + m0, x.log_req + x.lines, k1) - x.log_req);
    const uint32_t lines = m1 - m0, l0 = lines ? x.log_off[m0] : 0, lbytes = lines ? x.log_off[m1] - l0 : 0;
    log->lines = lines;
    log->out_bytes = lbytes;
    if (lines > log->line_cap || lbytes > log->out_cap) return GOFR_ERR_CAPACITY;
    if (lbytes) memcpy(log->out, x.log_out + l0, lbytes);
    for (uint32_t m = 0; m < lines; m++) {
        log->log_off[m + 1] = x.log_off[m0 + m + 1] - l0;
        log->log_req[m] = x.log_req[m0 + m] - k0;
    }
    return rc;
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
    const size_t n = max_batch;
    for (auto& x : f->b) {
        x.arena = (uint8_t*)gofr_alloc_pinned((size_t)arena + 16);
        x.buf_off = (uint32_t*)gofr_alloc_pinned((n + 1) * 4);
        x.remote_at = (uint8_t*)gofr_alloc_pinned(n * kRemoteMax);
        x.remote_len = (uint32_t*)gofr_alloc_pinned(n * 4);
        x.remote = (uint8_t*)gofr_alloc_pinned(n * kRemoteMax + 16);
        x.remote_off = (uint32_t*)gofr_alloc_pinned((n + 1) * 4);
        x.start = (int64_t*)gofr_alloc_pinned(n * 8);
        x.req_first = (uint32_t*)gofr_alloc_pinned((n + 1) * 4);
        x.consumed = (uint32_t*)gofr_alloc_pinned(n * 4);
        x.conn_status = (uint32_t*)gofr_alloc_pinned(n * 4);
        if (!x.arena || !x.buf_off || !x.remote_at || !x.remote_len || !x.remote || !x.remote_off || !x.start || !x.req_first ||
            !x.consumed || !x.conn_status) {
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
    if (!f || !out || (len && !buf) || (remote_len && !remote) || remote_len > kRemoteMax || !out->out_off || !out->req_first ||
        !out->consumed || !out->conn_status || (out->out_cap && !out->out) || (out->req_cap && (!out->meta || !out->req_at)))
        return GOFR_ERR_INVALID;
    if (log && !f->log) {  // a front-end without lines
        log->lines = 0;
        log->out_bytes = 0;
        log = nullptr;
    }
    if (log && (!log->log_off || (log->line_cap && !log->log_req) || (log->out_cap && !log->out))) return GOFR_ERR_INVALID;
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
