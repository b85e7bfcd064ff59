// conn_staging.h — one batch's staging and outputs for the per-read connection front-ends (conn_frontend.cpp,
// conn_app_frontend.cpp), and the steps they share: allocate and grow it, serve it through a connection batch call (growing
// the byte outputs and serving the batch again on GOFR_ERR_CAPACITY), and hand one slot's share to its caller.
//
// Public ABI and the standard library only, so that the front-ends build against stub batch calls under ThreadSanitizer
// (tests/emu/conn_frontend_stress.cpp, tests/emu/conn_app_frontend_stress.cpp).
//
// The ring's claim word (frontend_ring.h) reserves slot i and arena range [a, a + len), so the reads lie back to back in slot
// order — exactly the batch calls' buf_off contract:
//   caller      stores buf_off[i] = a, its read, its remote string (in a 255-byte place of its own) and its start clock;
//   dispatcher  stores buf_off[n], packs the remote strings back to back, pins the batch's trace seed, Date and log clock,
//               and grows the per-request columns to one request per 16 bytes plus one per connection (what the framer can
//               produce at most), so they never run short.  The response and log byte outputs start small and grow to what
//               the batch call reports when it returns GOFR_ERR_CAPACITY; the batch is then served again.  That is sound
//               because the call writes nothing past a capacity and the rerun sees the same bytes, seed, Date and clocks;
//               the always-sufficient bound is not allocated up front (for 64 KiB reads it is hundreds of MiB).
#pragma once

#include <algorithm>
#include <atomic>
#include <cstring>
#include <time.h>

#include "../../include/gofr_b200.h"

void set_last_error(const char* fmt, ...);  // engine_internal.h

static constexpr uint32_t kRemoteMax = 255;            // gofr_conn_batch_submit_log's limit on a remote string
static constexpr uint64_t kFirstOut = 64u << 10;        // the byte outputs' first capacity

struct ConnStaging {
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

static uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// Batch number b's trace seed.  The seed is mixed before the batch number is added: with splitmix64(seed + b), batch b's
// slot c and batch c's slot b would get the same ids whenever seed + b and seed + c are slot numbers, as the id function
// mixes c the same way.
static uint64_t batch_seed(uint64_t seed, uint64_t b) { return splitmix64(splitmix64(seed) + b); }

// The Date and log clock of a batch: the pinned one, else the wall clock, in ns
static int64_t batch_clock(const std::atomic<int64_t>& fixed) {
    int64_t now = fixed.load(std::memory_order_relaxed);
    if (!now) { struct timespec ts; clock_gettime(CLOCK_REALTIME, &ts); now = (int64_t)ts.tv_sec * 1000000000 + ts.tv_nsec; }
    return now;
}

static void free_staging(ConnStaging& x) {
    for (void* p : {(void*)x.arena, (void*)x.buf_off, (void*)x.remote_at, (void*)x.remote_len, (void*)x.remote, (void*)x.remote_off,
                    (void*)x.start, (void*)x.req_first, (void*)x.consumed, (void*)x.conn_status, (void*)x.out_off, (void*)x.meta,
                    (void*)x.req_at, (void*)x.log_off, (void*)x.log_req, (void*)x.ids, (void*)x.out, (void*)x.log_out})
        gofr_free_pinned(p);
    x = ConnStaging();
}

// the per-connection staging of max_batch reads of `arena` bytes in all; false when a pinned allocation failed.  Without
// `served` (a batch that is only routed) the remote strings and start clocks, which only serving reads, are left out.
static bool alloc_staging(ConnStaging& x, uint32_t max_batch, uint64_t arena, bool served = true) {
    const size_t n = max_batch;
    x.arena = (uint8_t*)gofr_alloc_pinned((size_t)arena + 16);
    x.buf_off = (uint32_t*)gofr_alloc_pinned((n + 1) * 4);
    x.req_first = (uint32_t*)gofr_alloc_pinned((n + 1) * 4);
    x.consumed = (uint32_t*)gofr_alloc_pinned(n * 4);
    x.conn_status = (uint32_t*)gofr_alloc_pinned(n * 4);
    if (!(x.arena && x.buf_off && x.req_first && x.consumed && x.conn_status)) return false;
    if (!served) return true;
    x.remote_at = (uint8_t*)gofr_alloc_pinned(n * kRemoteMax);
    x.remote_len = (uint32_t*)gofr_alloc_pinned(n * 4);
    x.remote = (uint8_t*)gofr_alloc_pinned(n * kRemoteMax + 16);
    x.remote_off = (uint32_t*)gofr_alloc_pinned((n + 1) * 4);
    x.start = (int64_t*)gofr_alloc_pinned(n * 8);
    return x.remote_at && x.remote_len && x.remote && x.remote_off && x.start;
}

// replaces *p by a pinned buffer of `bytes` (the old contents are not kept)
static bool regrow(void** p, size_t bytes) {
    gofr_free_pinned(*p);
    *p = gofr_alloc_pinned(bytes);
    return *p != nullptr;
}

// the per-request columns for req_cap requests; without `served` only those a route call writes (meta, req_at, ids)
static bool grow_requests(ConnStaging& x, uint32_t req_cap, bool served = true) {
    if (req_cap <= x.req_cap) return true;
    const size_t n = (size_t)req_cap;
    x.req_cap = 0;
    bool ok = regrow((void**)&x.meta, n * 4) && regrow((void**)&x.req_at, n * 4) && regrow((void**)&x.ids, n * 16);
    if (served)
        ok = ok && regrow((void**)&x.out_off, (n + 1) * 4) && regrow((void**)&x.log_off, (n + 1) * 4) && regrow((void**)&x.log_req, n * 4);
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

// The requests a batch of n reads of arena_bytes in all can hold at most: one per 16 bytes plus one per connection
static uint32_t staged_req_cap(uint32_t n, uint32_t arena_bytes) { return arena_bytes / 16 + n; }

// What one run of a staged batch needs besides its staging.
struct ConnServe {
    gofr_engine* eng;
    bool log;
    int32_t tz_offset_s;
    uint64_t trace_seed;
    int64_t now;                    // Date and log time, ns
    std::atomic<uint64_t>* reruns;  // counts each run after an output grew
    const char* who;                // names the front-end in errors
};

// Closes the staging of batch x's n reads (arena_bytes in all) and serves it through `call` — a connection batch call
// (in, out, log or null, ticket) whose result gofr_batch_wait reports — growing the byte outputs and serving the batch again
// while the call reports GOFR_ERR_CAPACITY for a need they do not hold yet.
template <class Call>
static int serve_staged(ConnStaging& x, uint32_t n, uint32_t arena_bytes, const ConnServe& s, Call call) {
    x.buf_off[n] = arena_bytes;
    x.remote_off[0] = 0;
    for (uint32_t i = 0; i < n; i++) {
        memcpy(x.remote + x.remote_off[i], x.remote_at + (size_t)i * kRemoteMax, x.remote_len[i]);
        x.remote_off[i + 1] = x.remote_off[i] + x.remote_len[i];
    }
    const uint32_t req_cap = staged_req_cap(n, arena_bytes);
    if (!grow_requests(x, req_cap) || !grow_bytes(&x.out, &x.out_cap, kFirstOut) ||
        (s.log && !grow_bytes(&x.log_out, &x.log_cap, kFirstOut))) {
        set_last_error("%s: no pinned outputs for %u requests", s.who, req_cap);
        return GOFR_ERR_NOMEM;
    }
    gofr_conn_batch in;
    memset(&in, 0, sizeof in);
    in.buf = x.arena; in.buf_off = x.buf_off; in.buf_bytes = arena_bytes; in.n_conns = n;
    in.trace_seed = s.trace_seed;
    gofr_format_http_date(s.now / 1000000000, in.date);
    for (;;) {
        gofr_conn_resp out;
        memset(&out, 0, sizeof out);
        out.out = x.out; out.out_cap = x.out_cap; out.req_cap = req_cap; out.out_off = x.out_off; out.meta = x.meta;
        out.req_at = x.req_at; out.trace_ids = x.ids; out.req_first = x.req_first; out.consumed = x.consumed;
        out.conn_status = x.conn_status;
        gofr_conn_log lg;
        memset(&lg, 0, sizeof lg);
        lg.remote = x.remote; lg.remote_off = x.remote_off; lg.start_unix_ns = x.start; lg.log_unix_ns = s.now;
        lg.tz_offset_s = s.tz_offset_s; lg.line_cap = req_cap; lg.out = x.log_out; lg.out_cap = x.log_cap;
        lg.log_off = x.log_off; lg.log_req = x.log_req;
        gofr_ticket t = 0;
        int rc = call(&in, &out, s.log ? &lg : nullptr, &t);
        if (rc == GOFR_OK) rc = gofr_batch_wait(s.eng, t);
        x.lines = s.log ? lg.lines : 0;
        if (rc != GOFR_ERR_CAPACITY) return rc;
        // the call reported what the batch needs: grow to it and serve the same batch again (a need the outputs already
        // hold is one no capacity fixes, such as log offsets past 32 bits)
        const bool more = out.out_bytes > x.out_cap || (s.log && lg.out_bytes > x.log_cap);
        if (!more) return rc;
        if (!grow_bytes(&x.out, &x.out_cap, out.out_bytes) || (s.log && !grow_bytes(&x.log_out, &x.log_cap, lg.out_bytes))) {
            set_last_error("%s: no pinned output of %llu response and %llu log bytes", s.who, (unsigned long long)out.out_bytes,
                           (unsigned long long)lg.out_bytes);
            return GOFR_ERR_NOMEM;
        }
        s.reruns->fetch_add(1, std::memory_order_relaxed);
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

// the caller's side of a read: the checks gofr_conn_frontend_serve and the respond round make before anything is queued
// (GOFR_OK: go on); a log that the front-end does not write is answered with no lines and dropped
static int check_read(uint32_t len, const uint8_t* buf, const uint8_t* remote, uint32_t remote_len, const gofr_conn_resp* out,
                      gofr_conn_log** log, bool front_end_logs) {
    if (!out || (len && !buf) || (remote_len && !remote) || remote_len > kRemoteMax || !out->out_off || !out->req_first ||
        !out->consumed || !out->conn_status || (out->out_cap && !out->out) || (out->req_cap && (!out->meta || !out->req_at)))
        return GOFR_ERR_INVALID;
    gofr_conn_log* lg = *log;
    if (lg && !front_end_logs) {
        lg->lines = 0;
        lg->out_bytes = 0;
        *log = lg = nullptr;
    }
    if (lg && (!lg->log_off || (lg->line_cap && !lg->log_req) || (lg->out_cap && !lg->out))) return GOFR_ERR_INVALID;
    return GOFR_OK;
}

// slot i's share of batch x, rebased to the caller's buffers; GOFR_ERR_CAPACITY when one of the caller's capacities is short
static int fan_out(const ConnStaging& x, uint32_t i, uint32_t a, gofr_conn_resp* out, gofr_conn_log* log) {
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
