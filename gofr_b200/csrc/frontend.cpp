// frontend.cpp — batching front-end over gofr_batch_submit_slots (SURVEY.md §8f rank 3: "collect in-flight requests from
// conn goroutines into the ring, fan results back").
//
// The reference serves one request per goroutine (net/http conn.serve → router.ServeHTTP, pkg/gofr/httpServer.go:29-33);
// the GPU path wants batches.  This is the piece in between, host C++ only: any number of producer threads (connection
// goroutines through cgo, or the threads of the C++ stand-in) hand in single requests and block until their response is
// ready; the dispatcher of frontend_ring.h closes a batch, this file runs it through the engine's slot-layout host path,
// and each producer copies its own slot out.  The ring (claim, close, timer, wake tree, recycle) is shared with the gRPC
// front-end, proto_frontend.cpp; what is here is the HTTP payload: the pinned staging in the ABI layout, the Date of a
// batch and the re-serve of a response too long for its slot.  A front-end made by gofr_frontend_create_log also stages a
// log record and its strings per request (seat i's strings at i * max_log_bytes) and takes the batch's lines back: a batch
// in which some caller logs runs through gofr_batch_submit_slots_log, the other callers' records saying GOFR_LOG_NONE.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <time.h>

#include "../../include/gofr_b200.h"
#include "engine_internal.h"
#include "frontend_ring.h"

// A weak reference: frontend.cpp also links into harnesses whose stub engine has only the calls of a front-end without
// log staging (tests/emu/frontend_stress.cpp); the library defines it.
#pragma weak gofr_batch_submit_slots_log

struct gofr_frontend_batch {
    // pinned staging in the ABI layout (gofr_req_batch / gofr_slot_batch)
    gofr_req_desc* desc = nullptr;
    uint8_t* ids = nullptr;
    uint8_t* arena = nullptr;
    uint8_t* out = nullptr;
    uint32_t* out_len = nullptr;
    uint32_t* meta = nullptr;
    char date[29] = {0};                  // the round's Date header (a response too long for its slot is served again, alone)
    // log staging (gofr_frontend_create_log)
    gofr_log_desc* log_desc = nullptr;
    uint8_t* log_arena = nullptr;
    uint8_t* log_out = nullptr;
    uint32_t* log_off = nullptr;
    std::atomic<bool> logs{false};        // some caller of the filling batch asked for its line
};
using Batch = gofr_frontend_batch;

struct gofr_frontend {
    gofr_frontend(uint32_t max_batch, uint32_t max_wait_us) : ring(max_batch, max_wait_us) {}
    gofr_engine* eng = nullptr;
    uint32_t max_batch = 0, slot_bytes = 0, per_request = 0;
    uint32_t max_log_bytes = 0;           // log staging per request (0: gofr_frontend_create, no log staging)
    uint64_t log_cap = 0;                 // line bytes of a batch
    bool log = false;
    std::atomic<int64_t> fixed_clock{0};  // tests: the Date of every batch; 0 = wall clock
    std::atomic<int64_t> log_clock{0};    // tests: the log time of every line (ns); 0 = wall clock
    Batch b[gofr_ring::kBatches];
    gofr_ring::Ring ring;                 // GOFR_FRONTEND_DEBUG=1: where the dispatcher's time goes (printed at destroy)
};

static void free_batch(Batch& x) {
    gofr_free_pinned(x.desc); gofr_free_pinned(x.ids); gofr_free_pinned(x.arena);
    gofr_free_pinned(x.out); gofr_free_pinned(x.out_len); gofr_free_pinned(x.meta);
    gofr_free_pinned(x.log_desc); gofr_free_pinned(x.log_arena); gofr_free_pinned(x.log_out); gofr_free_pinned(x.log_off);
}

// the dispatcher's step: batch k's n requests (arena_bytes of path, query and body) through the slot-layout host path
static int serve_batch(gofr_frontend* f, int k, uint32_t n, uint32_t arena_bytes) {
    Batch& x = f->b[k];
    gofr_req_batch in;
    memset(&in, 0, sizeof in);
    in.desc = x.desc; in.trace_ids = x.ids; in.arena = x.arena; in.arena_bytes = (arena_bytes + 15u) & ~15u; in.n = n;
    int64_t now = f->fixed_clock.load(std::memory_order_relaxed);
    if (!now) { struct timespec ts; clock_gettime(CLOCK_REALTIME, &ts); now = (int64_t)ts.tv_sec; }
    gofr_format_http_date(now, in.date);
    memcpy(x.date, in.date, sizeof x.date);
    gofr_slot_batch out;
    memset(&out, 0, sizeof out);
    out.out = x.out; out.slot_bytes = f->slot_bytes; out.out_len = x.out_len; out.meta = x.meta;
    gofr_ticket t = 0;
    int rc;
    if (x.logs.exchange(false, std::memory_order_acquire)) {  // the batch is closed: no caller sets it until it reopens
        gofr_batch_log log;
        memset(&log, 0, sizeof log);
        log.desc = x.log_desc; log.arena = x.log_arena; log.arena_bytes = (uint64_t)n * f->max_log_bytes;
        int64_t ns = f->log_clock.load(std::memory_order_relaxed);
        if (!ns) { struct timespec ts; clock_gettime(CLOCK_REALTIME, &ts); ns = (int64_t)ts.tv_sec * 1000000000ll + ts.tv_nsec; }
        log.log_unix_ns = ns;
        log.out = x.log_out; log.out_cap = f->log_cap; log.log_off = x.log_off;
        rc = gofr_batch_submit_slots_log(f->eng, &in, &out, &log, &t);
    } else {
        rc = gofr_batch_submit_slots(f->eng, &in, &out, &t);
    }
    if (rc == GOFR_OK) rc = gofr_batch_wait(f->eng, t);
    return rc;
}

static int frontend_create(gofr_frontend** out, gofr_engine* e, uint32_t max_batch, uint32_t max_wait_us, uint32_t slot_bytes,
                           uint32_t max_request_bytes, bool log, uint32_t max_log_bytes) {
    if (!out || !e || max_batch == 0 || max_batch > 0x7FFFFFFFu || slot_bytes == 0 || (slot_bytes & 15u)) return GOFR_ERR_INVALID;
    const uint64_t per = ((uint64_t)max_request_bytes + 7u) & ~(uint64_t)3u;  // path|query and body are each padded to 4
    const uint64_t cap = (uint64_t)max_batch * per + 64;
    if (cap > 0xFFFFFFF0ull) return GOFR_ERR_CAPACITY;
    // a batch's lines: gofr_batch_log_bound's rule for max_batch requests of max_log_bytes string bytes
    const uint64_t log_cap = log ? (uint64_t)max_batch * (320u + 6ull * max_log_bytes) : 0;
    if (log_cap > 0xFFFFFFF0ull || (uint64_t)max_batch * max_log_bytes > 0xFFFFFFF0ull) return GOFR_ERR_CAPACITY;
    gofr_frontend* f = new gofr_frontend(max_batch, max_wait_us);
    f->eng = e;
    f->max_batch = max_batch;
    f->slot_bytes = slot_bytes;
    f->per_request = (uint32_t)per;
    f->log = log;
    f->max_log_bytes = max_log_bytes;
    f->log_cap = log_cap;
    for (auto& x : f->b) {
        if (log) {
            x.log_desc = (gofr_log_desc*)gofr_alloc_pinned((size_t)max_batch * sizeof(gofr_log_desc));
            x.log_arena = (uint8_t*)gofr_alloc_pinned((size_t)max_batch * max_log_bytes + 64);
            x.log_out = (uint8_t*)gofr_alloc_pinned((size_t)log_cap + 64);
            x.log_off = (uint32_t*)gofr_alloc_pinned(((size_t)max_batch + 1) * 4);
            if (!x.log_desc || !x.log_arena || !x.log_out || !x.log_off) {
                for (auto& y : f->b) free_batch(y);
                delete f;
                return GOFR_ERR_NOMEM;
            }
        }
        x.desc = (gofr_req_desc*)gofr_alloc_pinned((size_t)max_batch * sizeof(gofr_req_desc));
        x.ids = (uint8_t*)gofr_alloc_pinned((size_t)max_batch * 16);
        x.arena = (uint8_t*)gofr_alloc_pinned((size_t)cap);
        x.out = (uint8_t*)gofr_alloc_pinned((size_t)max_batch * slot_bytes);
        x.out_len = (uint32_t*)gofr_alloc_pinned((size_t)max_batch * 4);
        x.meta = (uint32_t*)gofr_alloc_pinned((size_t)max_batch * 4);
        if (!x.desc || !x.ids || !x.arena || !x.out || !x.out_len || !x.meta) {
            for (auto& y : f->b) free_batch(y);
            delete f;
            return GOFR_ERR_NOMEM;
        }
    }
    { const char* dbg = getenv("GOFR_FRONTEND_DEBUG"); f->ring.debug = dbg && dbg[0] == '1'; }
    f->ring.start([f](int k, uint32_t n, uint32_t arena_bytes) { return serve_batch(f, k, n, arena_bytes); });
    *out = f;
    return GOFR_OK;
}

extern "C" {

int gofr_frontend_create(gofr_frontend** out, gofr_engine* e, uint32_t max_batch, uint32_t max_wait_us, uint32_t slot_bytes,
                         uint32_t max_request_bytes) {
    return frontend_create(out, e, max_batch, max_wait_us, slot_bytes, max_request_bytes, false, 0);
}

int gofr_frontend_create_log(gofr_frontend** out, gofr_engine* e, uint32_t max_batch, uint32_t max_wait_us, uint32_t slot_bytes,
                             uint32_t max_request_bytes, uint32_t max_log_bytes) {
    return frontend_create(out, e, max_batch, max_wait_us, slot_bytes, max_request_bytes, true, max_log_bytes);
}

void gofr_frontend_destroy(gofr_frontend* f) {
    if (!f) return;
    gofr_ring::Ring& r = f->ring;
    r.stop();
    if (r.debug) {
        const double nb = (double)(r.batches.load() ? r.batches.load() : 1);
        fprintf(stderr, "[gofr frontend] batches %llu  fill-spin avg %.1f max %.1f us  engine avg %.1f max %.1f us (>5ms: %llu)  publish+wake avg %.1f max %.1f us\n",
                (unsigned long long)r.batches.load(), r.dbg_spin_ns / nb / 1e3, r.dbg_spin_max / 1e3, r.dbg_eng_ns / nb / 1e3,
                r.dbg_eng_max / 1e3, (unsigned long long)r.dbg_eng_slow, r.dbg_wake_ns / nb / 1e3, r.dbg_wake_max / 1e3);
    }
    for (auto& x : f->b) free_batch(x);
    delete f;
}

int gofr_frontend_set_clock(gofr_frontend* f, int64_t unix_seconds) {
    if (!f) return GOFR_ERR_INVALID;
    f->fixed_clock.store(unix_seconds, std::memory_order_relaxed);
    return GOFR_OK;
}

int gofr_frontend_set_log_clock(gofr_frontend* f, int64_t unix_ns) {
    if (!f) return GOFR_ERR_INVALID;
    f->log_clock.store(unix_ns, std::memory_order_relaxed);
    return GOFR_OK;
}

int gofr_frontend_stats(gofr_frontend* f, uint64_t* batches, uint64_t* requests) {
    if (!f) return GOFR_ERR_INVALID;
    if (batches) *batches = f->ring.batches.load(std::memory_order_relaxed);
    if (requests) *requests = f->ring.records.load(std::memory_order_relaxed);
    return GOFR_OK;
}

}  // extern "C"

// One caller's request, with its log record (log == NULL: a plain gofr_frontend_serve, GOFR_LOG_NONE on a log front-end).
static int frontend_serve(gofr_frontend* f, uint8_t method, const uint8_t* path, uint16_t path_len, const uint8_t* query,
                          uint16_t query_len, uint8_t flags, const uint8_t* data, uint32_t data_len, const uint8_t trace_id[16],
                          const gofr_log_desc* log, const uint8_t* strings, uint8_t* resp, uint32_t resp_cap, uint32_t* resp_len,
                          uint32_t* meta, uint8_t* line, uint32_t line_cap, uint32_t* line_len) {
    if (!f || !resp_len || !trace_id || (path_len && !path) || (query_len && !query) || (data_len && !data)) return GOFR_ERR_INVALID;
    uint32_t log_bytes = 0;
    if (log) {
        log_bytes = (uint32_t)log->method_len + log->ua_len + log->xff_len + log->remote_len + log->uri_len;
        if (!f->log || !line_len || (log_bytes && !strings) || (log->kind != GOFR_LOG_REQUEST && log->kind != GOFR_LOG_NONE)) {
            set_last_error(!f->log ? "the front-end was made without log staging (gofr_frontend_create_log)" : "bad log record");
            return GOFR_ERR_INVALID;
        }
        if (log_bytes > f->max_log_bytes) {
            set_last_error("log strings of %u bytes exceed the front-end's max_log_bytes", log_bytes);
            return GOFR_ERR_CAPACITY;
        }
        *line_len = 0;
    }
    const uint64_t need64 = (((uint64_t)path_len + query_len + 3u) & ~(uint64_t)3u) + (((uint64_t)data_len + 3u) & ~(uint64_t)3u);
    if (need64 > f->per_request) {
        set_last_error("request of %llu bytes exceeds the front-end's max_request_bytes", (unsigned long long)need64);
        return GOFR_ERR_CAPACITY;
    }
    const uint32_t need = (uint32_t)need64;
    // ---- claim slot i and `need` arena bytes in the filling batch (arena bytes never run out first: the arena holds
    //      max_batch requests of the largest admissible size) ----
    gofr_ring::Seat s;
    if (!f->ring.claim(need, &s)) return GOFR_ERR_INVALID;
    Batch& x = f->b[s.k];
    const uint32_t i = s.i, a = s.a;
    gofr_req_desc d;
    memset(&d, 0, sizeof d);
    d.arena_off = a; d.path_len = path_len; d.query_len = query_len; d.data_len = data_len; d.method = method; d.flags = flags;
    if (path_len) memcpy(x.arena + a, path, path_len);
    if (query_len) memcpy(x.arena + a + path_len, query, query_len);
    const uint32_t body_at = (a + path_len + query_len + 3u) & ~3u;
    if (data_len) memcpy(x.arena + body_at, data, data_len);
    x.desc[i] = d;
    memcpy(x.ids + (size_t)i * 16, trace_id, 16);
    if (f->log) {
        gofr_log_desc r;
        memset(&r, 0, sizeof r);
        if (log) r = *log;
        else r.kind = GOFR_LOG_NONE;
        r.arena_off = i * f->max_log_bytes;
        if (log_bytes) memcpy(x.log_arena + r.arena_off, strings, log_bytes);
        x.log_desc[i] = r;
        if (log) x.logs.store(true, std::memory_order_relaxed);
    }
    f->ring.filled(s);

    // ---- wait for the round to come back ----
    const uint32_t n = f->ring.wait(s);
    int rc = f->ring.b[s.k].rc;
    const uint32_t len = x.out_len[i];
    if (meta) *meta = x.meta[i];
    *resp_len = len;
    bool alone = false;
    char date[29];
    if (rc == GOFR_OK) {
        if (len > resp_cap) rc = GOFR_ERR_CAPACITY;
        else if (len > f->slot_bytes) { alone = true; memcpy(date, x.date, sizeof date); }  // did not fit its slot: see below
        else if (len) memcpy(resp, x.out + (size_t)i * f->slot_bytes, len);
    }
    int line_rc = GOFR_OK;
    if (log && f->ring.b[s.k].rc == GOFR_OK) {
        const uint32_t l0 = x.log_off[i], ll = x.log_off[i + 1] - l0;
        *line_len = ll;
        if (ll > line_cap) line_rc = GOFR_ERR_CAPACITY;
        else if (ll) memcpy(line, x.log_out + l0, ll);
    }
    // ---- the last producer to leave reopens the batch ----
    f->ring.leave(s, n);
    if (alone) {
        // The slot layout reports the length of a response that does not fit but writes nothing: serve this one request
        // again through the packed call, straight into the caller's buffer, with the Date of the batch it belonged to.
        std::vector<uint8_t> arena((size_t)need + 64, 0);
        if (path_len) memcpy(arena.data(), path, path_len);
        if (query_len) memcpy(arena.data() + path_len, query, query_len);
        if (data_len) memcpy(arena.data() + (((size_t)path_len + query_len + 3u) & ~(size_t)3u), data, data_len);
        d.arena_off = 0;
        gofr_req_batch in;
        memset(&in, 0, sizeof in);
        in.desc = &d; in.trace_ids = trace_id; in.arena = arena.data(); in.arena_bytes = arena.size(); in.n = 1;
        memcpy(in.date, date, sizeof date);
        uint32_t off2[2] = {0, 0}, meta1 = 0;
        gofr_resp_batch out;
        memset(&out, 0, sizeof out);
        out.out = resp; out.out_cap = resp_cap; out.out_off = off2; out.meta = &meta1;
        gofr_ticket t = 0;
        rc = gofr_batch_submit(f->eng, &in, &out, &t);
        if (rc == GOFR_OK) rc = gofr_batch_wait(f->eng, t);
        if (rc == GOFR_OK) { *resp_len = off2[1]; if (meta) *meta = meta1; }
    }
    if (rc == GOFR_OK && line_rc != GOFR_OK) set_last_error("a log line of %u bytes does not fit line_cap %u", *line_len, line_cap);
    return rc != GOFR_OK ? rc : line_rc;
}

extern "C" {

int gofr_frontend_serve(gofr_frontend* f, uint8_t method, const uint8_t* path, uint16_t path_len, const uint8_t* query,
                        uint16_t query_len, uint8_t flags, const uint8_t* data, uint32_t data_len, const uint8_t trace_id[16],
                        uint8_t* resp, uint32_t resp_cap, uint32_t* resp_len, uint32_t* meta) {
    return frontend_serve(f, method, path, path_len, query, query_len, flags, data, data_len, trace_id, nullptr, nullptr, resp,
                          resp_cap, resp_len, meta, nullptr, 0, nullptr);
}

int gofr_frontend_serve_log(gofr_frontend* f, uint8_t method, const uint8_t* path, uint16_t path_len, const uint8_t* query,
                            uint16_t query_len, uint8_t flags, const uint8_t* data, uint32_t data_len, const uint8_t trace_id[16],
                            const gofr_log_desc* log, const uint8_t* strings, uint8_t* resp, uint32_t resp_cap, uint32_t* resp_len,
                            uint32_t* meta, uint8_t* line, uint32_t line_cap, uint32_t* line_len) {
    if (!log) return GOFR_ERR_INVALID;
    return frontend_serve(f, method, path, path_len, query, query_len, flags, data, data_len, trace_id, log, strings, resp,
                          resp_cap, resp_len, meta, line, line_cap, line_len);
}

}  // extern "C"
