// conn_app_frontend.cpp — per-read front-end of the closure path: net/http runs one goroutine per connection and the user's
// closure runs on that goroutine (pkg/gofr/httpServer.go:29-33, handler.go:32-36).  A caller hands in one read and gets its
// connection's routed requests (gofr_conn_batch_route, with Context.Bind done for the batch); it runs the closures on its own
// thread, as long as they take; then it hands in the same read with the closures' records and gets its responses and log
// lines (gofr_conn_batch_respond_ex).
//
// Two independent rounds of frontend_ring.h's ring, not one two-phase batch: a connection's response never waits for
// another connection's closure, and a closure may call back into the server.  A respond batch holds connections from any
// route batches; each carries the trace key its route round handed out, so its ids are the ones its closures saw.
//
// Written against the public ABI only (gofr_conn_batch_route, gofr_batch_bind, gofr_conn_batch_respond_ex, gofr_batch_wait,
// the pinned allocator, gofr_format_http_date), so that tests/emu/conn_app_frontend_stress.cpp runs it against stub calls
// under ThreadSanitizer.  Staging, output growth and fan-out are conn_staging.h's, shared with conn_frontend.cpp.
//
// Route round: the ring's claim tiles the reads (buf_off); the dispatcher draws the batch's trace seed as conn_frontend.cpp
// does, hands slot i the key splitmix64(seed_b ^ splitmix64(i)), routes the batch, and binds the status-0 requests of every
// route that declared a schema with one gofr_batch_bind per schema.  Nothing is kept once the callers have copied out.
// Respond round: the claim tiles the reads again; each caller leaves its key and a pointer to its records (validated
// first: offsets within its record bytes, never decreasing), and the dispatcher gathers the records back to back in slot
// order at close.  A batch whose records do not match its connections' requests (a caller stated a wrong count, or its bytes
// changed since its route call) is served once without records to learn each connection's count; the callers whose count
// differs get GOFR_ERR_INVALID and the batch is served again with empty records in their place.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/gofr_b200.h"
#include "conn_staging.h"
#include "frontend_ring.h"

static constexpr uint32_t kUnbound = 0xFFFFFFFFu;  // bind status of a request no schema was bound for

// one route batch: the reads (ConnStaging's arena, buf_off, req_first, consumed, conn_status, meta, req_at, ids; its
// serving columns are not allocated) and what the route call and the binds add
struct RouteStaging {
    ConnStaging x;
    uint64_t* key = nullptr;       // per connection
    uint8_t* parsed = nullptr;     // the route call's arena: the batch's arena bytes + 64
    uint32_t req_cap = 0;          // of the columns below
    gofr_req_desc* desc = nullptr;
    uint32_t *vars = nullptr, *bstat = nullptr, *blen = nullptr;
    uint64_t* brow = nullptr;      // per request: its row's place in rows
    uint8_t* rows = nullptr;
    uint64_t rows_cap = 0;
    std::vector<uint32_t> who;     // the dispatcher's scratch
    std::vector<gofr_req_desc> bd;
};

// one respond batch: the reads and, per slot, the caller's key and records; the gathered records
struct RespondStaging {
    ConnStaging x;
    uint64_t* key = nullptr;
    const uint8_t** rec_at = nullptr;       // slot i's records (the caller's memory: it waits until the batch is served)
    const uint32_t** rec_off_at = nullptr;
    uint32_t* n_req = nullptr;              // slot i's stated request count
    int* rc = nullptr;                      // slot i's own result: GOFR_ERR_INVALID when its records did not match
    uint32_t* fix = nullptr;                // slot i's counted requests (a batch whose records did not match)
    uint8_t* rec = nullptr;
    uint64_t rec_cap = 0;
    uint32_t* rec_off = nullptr;
    uint32_t rec_off_cap = 0;
};

struct gofr_conn_app_frontend {
    gofr_conn_app_frontend(uint32_t max_batch, uint32_t max_wait_us) : route(max_batch, max_wait_us), respond(max_batch, max_wait_us) {}
    gofr_engine* eng = nullptr;
    uint32_t max_conn_bytes = 0;
    bool log = false;
    int32_t tz_offset_s = 0;
    uint64_t seed = 0, batch_no = 0;                   // batch_no: the route dispatcher's alone
    std::vector<uint32_t> route_schema, schema_fields; // per route: its bind schema (0: none) and that schema's field count
    std::vector<uint32_t> schemas;                     // the distinct bind schemas
    std::atomic<int64_t> fixed_clock{0};
    std::atomic<uint64_t> reruns{0}, isolated{0}, gather_ns{0};
    RouteStaging rb[gofr_ring::kBatches];
    RespondStaging pb[gofr_ring::kBatches];
    gofr_ring::Ring route, respond;
};
using AppFrontend = gofr_conn_app_frontend;

static bool grow_route(RouteStaging& r, uint32_t req_cap) {
    if (req_cap <= r.req_cap) return grow_requests(r.x, req_cap, false);
    const size_t n = req_cap;
    r.req_cap = 0;
    bool ok = grow_requests(r.x, req_cap, false) && regrow((void**)&r.desc, n * sizeof(gofr_req_desc)) &&
              regrow((void**)&r.vars, n * 4 * GOFR_MAX_PATH_VARS) && regrow((void**)&r.bstat, n * 4) && regrow((void**)&r.blen, n * 4) &&
              regrow((void**)&r.brow, n * 8);
    if (ok) r.req_cap = req_cap;
    return ok;
}

// the route dispatcher's step: batch k's n reads through gofr_conn_batch_route, then Context.Bind per schema
static int route_batch(AppFrontend* f, int k, uint32_t n, uint32_t arena_bytes) {
    RouteStaging& r = f->rb[k];
    ConnStaging& x = r.x;
    x.buf_off[n] = arena_bytes;
    const uint64_t seed_b = batch_seed(f->seed, f->batch_no++);
    for (uint32_t i = 0; i < n; i++) r.key[i] = splitmix64(seed_b ^ splitmix64(i));
    const uint32_t req_cap = staged_req_cap(n, arena_bytes);
    if (!grow_route(r, req_cap)) {
        set_last_error("gofr_conn_app_frontend: no pinned outputs for %u requests", req_cap);
        return GOFR_ERR_NOMEM;
    }
    gofr_conn_batch in;
    memset(&in, 0, sizeof in);
    in.buf = x.arena; in.buf_off = x.buf_off; in.buf_bytes = arena_bytes; in.n_conns = n; in.trace_seed = seed_b;
    gofr_conn_route rt;
    memset(&rt, 0, sizeof rt);
    rt.req_cap = req_cap; rt.desc = r.desc; rt.arena = r.parsed; rt.meta = x.meta; rt.vars = r.vars; rt.req_at = x.req_at;
    rt.trace_ids = x.ids; rt.req_first = x.req_first; rt.consumed = x.consumed; rt.conn_status = x.conn_status;
    int rc = gofr_conn_batch_route(f->eng, &in, &rt);
    if (rc) return rc;
    const uint32_t nreq = x.req_first[n];
    for (uint32_t q = 0; q < nreq; q++) r.bstat[q] = kUnbound, r.blen[q] = 0, r.brow[q] = 0;
    // Context.Bind for the batch: one gofr_batch_bind per schema over its routes' status-0 requests, rows in slots of
    // GOFR_BIND_ROW_SLOT
    uint64_t at = 0;
    auto reserve = [&](uint64_t need) {  // rows holds `need` bytes; the rows of the binds so far move along
        if (need <= r.rows_cap) return true;
        uint8_t* grown = (uint8_t*)gofr_alloc_pinned((size_t)need + (need >> 2));
        if (!grown) { set_last_error("gofr_conn_app_frontend: no pinned rows of %llu bytes", (unsigned long long)need); return false; }
        if (at) memcpy(grown, r.rows, (size_t)at);
        gofr_free_pinned(r.rows);
        r.rows = grown;
        r.rows_cap = need + (need >> 2);
        return true;
    };
    for (uint32_t s : f->schemas) {
        r.who.clear();
        r.bd.clear();
        uint32_t fields = 0, longest = 0;
        for (uint32_t q = 0; q < nreq; q++) {
            const uint32_t status = GOFR_META_STATUS(x.meta[q]), route = GOFR_META_ROUTE(x.meta[q]);
            if (status || route >= f->route_schema.size() || f->route_schema[route] != s) continue;
            r.who.push_back(q);
            r.bd.push_back(r.desc[q]);
            fields = f->schema_fields[route];
            longest = std::max(longest, r.desc[q].data_len);
        }
        if (r.who.empty()) continue;
        const uint32_t slot = (uint32_t)GOFR_BIND_ROW_SLOT(fields, longest);
        if (!reserve(at + (uint64_t)r.who.size() * slot)) return GOFR_ERR_NOMEM;
        gofr_req_batch b;
        memset(&b, 0, sizeof b);
        b.desc = r.bd.data(); b.arena = r.parsed; b.arena_bytes = (uint64_t)arena_bytes + 64; b.n = (uint32_t)r.who.size();
        std::vector<uint32_t> len(r.who.size()), st(r.who.size());
        rc = gofr_batch_bind(f->eng, s, &b, r.rows + at, slot, len.data(), st.data());
        if (rc) return rc;
        std::vector<uint32_t> over;  // rows the slot did not hold: the bind reported their exact length
        uint32_t wide = 0;
        for (size_t j = 0; j < r.who.size(); j++) {
            const uint32_t q = r.who[j];
            r.bstat[q] = st[j];
            r.blen[q] = len[j];
            r.brow[q] = at + (uint64_t)j * slot;
            if (len[j] > slot && st[j] != GOFR_BIND_HOST) { over.push_back(q); wide = std::max(wide, len[j]); }
        }
        at += (uint64_t)r.who.size() * slot;
        if (over.empty()) continue;
        // invalid UTF-8 triples a string, a long literal or name lengthens an error text: bind those requests once more in
        // slots of the longest
        const uint32_t slot2 = (wide + 15u) & ~15u;
        if (!reserve(at + (uint64_t)over.size() * slot2)) return GOFR_ERR_NOMEM;
        r.bd.clear();
        for (uint32_t q : over) r.bd.push_back(r.desc[q]);
        b.desc = r.bd.data(); b.n = (uint32_t)over.size();
        rc = gofr_batch_bind(f->eng, s, &b, r.rows + at, slot2, len.data(), st.data());
        if (rc) return rc;
        for (size_t j = 0; j < over.size(); j++) {
            // a bind that reports exact lengths always fits here; a row that does not is left to the host, alone
            const bool host = len[j] > slot2;
            r.bstat[over[j]] = host ? (uint32_t)GOFR_BIND_HOST : st[j];
            r.blen[over[j]] = host ? 0 : len[j];
            r.brow[over[j]] = at + (uint64_t)j * slot2;
        }
        at += (uint64_t)over.size() * slot2;
    }
    return GOFR_OK;
}

// slot i's share of route batch r (its reads from arena byte a, len bytes), rebased to the caller's buffers.  The parsed
// forms are rebased by a rounded down to 16, so each keeps its alignment.
static int route_out(const RouteStaging& r, uint32_t i, uint32_t a, uint32_t len, gofr_conn_route* out, gofr_conn_app_bind* bind,
                     uint64_t* trace_key) {
    const ConnStaging& x = r.x;
    const uint32_t k0 = x.req_first[i], nreq = x.req_first[i + 1] - k0, base = a & ~15u;
    out->req_first[0] = 0;
    out->req_first[1] = nreq;
    out->consumed[0] = x.consumed[i];
    out->conn_status[0] = x.conn_status[i];
    *trace_key = r.key[i];
    uint64_t rows = 0;
    for (uint32_t j = 0; j < nreq; j++) rows += r.blen[k0 + j];
    if (bind) bind->rows_bytes = rows;
    if (nreq > out->req_cap || (bind && rows > bind->rows_cap)) return GOFR_ERR_CAPACITY;
    memcpy(out->arena, r.parsed + base, a + len - base);
    for (uint32_t j = 0; j < nreq; j++) {
        out->desc[j] = r.desc[k0 + j];
        out->desc[j].arena_off -= base;
        out->meta[j] = x.meta[k0 + j];
        out->req_at[j] = x.req_at[k0 + j] - a;
    }
    memcpy(out->vars, r.vars + (size_t)k0 * GOFR_MAX_PATH_VARS, (size_t)nreq * 4 * GOFR_MAX_PATH_VARS);
    memcpy(out->trace_ids, x.ids + (size_t)k0 * 16, (size_t)nreq * 16);
    if (!bind) return GOFR_OK;
    uint64_t p = 0;
    bind->row_off[0] = 0;
    for (uint32_t j = 0; j < nreq; j++) {
        const uint32_t q = k0 + j;
        bind->status[j] = r.bstat[q];
        if (r.blen[q]) memcpy(bind->rows + p, r.rows + r.brow[q], r.blen[q]);
        p += r.blen[q];
        bind->row_off[j + 1] = (uint32_t)p;
    }
    return GOFR_OK;
}

// gathers respond batch p's records back to back in slot order, slot i's counted as `fix[i]` empty records when it was
// refused (rc[i] != GOFR_OK); false when no pinned memory was left
static bool gather(RespondStaging& p, uint32_t n, uint32_t* n_req_out, uint64_t* bytes_out) {
    uint64_t reqs = 0, bytes = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (p.rc[i]) { reqs += p.fix[i]; continue; }
        reqs += p.n_req[i];
        bytes += p.rec_off_at[i][p.n_req[i]] - p.rec_off_at[i][0];
    }
    if (reqs + 1 > p.rec_off_cap) {
        const uint64_t c = reqs + 1 + (reqs >> 2);
        p.rec_off_cap = 0;
        if (!regrow((void**)&p.rec_off, (size_t)c * 4)) return false;
        p.rec_off_cap = (uint32_t)c;
    }
    if (!grow_bytes(&p.rec, &p.rec_cap, bytes + 1)) return false;
    uint32_t k = 0;
    uint64_t at = 0;
    p.rec_off[0] = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (p.rc[i]) {
            for (uint32_t j = 0; j < p.fix[i]; j++) p.rec_off[++k] = (uint32_t)at;
            continue;
        }
        const uint32_t* ro = p.rec_off_at[i];
        const uint32_t m = p.n_req[i], b0 = ro[0];
        if (ro[m] > b0) memcpy(p.rec + at, p.rec_at[i] + b0, ro[m] - b0);
        for (uint32_t j = 0; j < m; j++) p.rec_off[++k] = (uint32_t)(at + ro[j + 1] - b0);
        at += ro[m] - b0;
    }
    *n_req_out = k;
    *bytes_out = at;
    return true;
}

// The record bytes a respond batch of n reads (arena_bytes in all) may gather: with the batch's bytes and 8 bytes per possible
// request they stay below 4 GiB, so rec_off fits 32 bits and no chunk of the batch call can pass its 32-bit spliced arena
static uint64_t record_budget(uint32_t n, uint32_t arena_bytes) {
    const uint64_t fixed = (uint64_t)arena_bytes + 8ull * staged_req_cap(n, arena_bytes) + 64;
    return fixed < 0xFFFFFFF0ull ? 0xFFFFFFF0ull - fixed : 0;
}

// the respond dispatcher's step: gather batch k's records and serve its n reads through gofr_conn_batch_respond_ex
static int respond_batch(AppFrontend* f, int k, uint32_t n, uint32_t arena_bytes) {
    RespondStaging& p = f->pb[k];
    const ConnServe s{f->eng, f->log, f->tz_offset_s, 0, batch_clock(f->fixed_clock), &f->reruns, "gofr_conn_app_frontend"};
    uint32_t nreq = 0;
    uint64_t rec_bytes = 0;
    auto with = [&](bool records) {
        return [&, records](const gofr_conn_batch* in, gofr_conn_resp* out, gofr_conn_log* lg, gofr_ticket* t) {
            gofr_conn_results res;
            memset(&res, 0, sizeof res);
            res.rec = p.rec; res.rec_off = p.rec_off; res.rec_bytes = rec_bytes; res.n_req = nreq;
            return gofr_conn_batch_respond_ex(f->eng, in, p.key, records ? &res : nullptr, out, lg, t);
        };
    };
    // Serves the batch once without records, so that each connection's request count is known: the callers whose records
    // are not for that many requests are refused, and every refused caller's place gets that many empty records
    auto count = [&]() -> int {
        f->isolated.fetch_add(1, std::memory_order_relaxed);
        const int rc = serve_staged(p.x, n, arena_bytes, s, with(false));
        if (rc != GOFR_OK && rc != GOFR_ERR_CAPACITY) return rc;
        uint32_t refused = 0;
        for (uint32_t i = 0; i < n; i++) {
            p.fix[i] = p.x.req_first[i + 1] - p.x.req_first[i];
            if (!p.rc[i] && p.fix[i] != p.n_req[i]) p.rc[i] = GOFR_ERR_INVALID;
            refused += p.rc[i] != GOFR_OK;
        }
        return refused ? GOFR_OK : GOFR_ERR_INVALID;  // nothing any one caller did: the batch call's own refusal
    };
    auto serve = [&]() -> int {
        const int64_t t0 = gofr_ring::mono_ns();
        const bool ok = gather(p, n, &nreq, &rec_bytes);
        f->gather_ns.fetch_add((uint64_t)(gofr_ring::mono_ns() - t0), std::memory_order_relaxed);
        if (!ok) { set_last_error("gofr_conn_app_frontend: no pinned records"); return GOFR_ERR_NOMEM; }
        return serve_staged(p.x, n, arena_bytes, s, with(true));
    };
    // the callers whose records, with the ones before them, would pass the batch's record budget are refused
    const uint64_t budget = record_budget(n, arena_bytes);
    uint64_t total = 0;
    bool over = false;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t b = p.rec_off_at[i][p.n_req[i]] - p.rec_off_at[i][0];
        p.rc[i] = total + b > budget ? GOFR_ERR_CAPACITY : GOFR_OK;
        if (p.rc[i]) over = true;
        else total += b;
    }
    int rc = over ? count() : GOFR_OK;
    if (rc) return rc;
    rc = serve();
    bool mismatch = rc == GOFR_ERR_INVALID;
    for (uint32_t i = 0; i < n && !mismatch && (rc == GOFR_OK || rc == GOFR_ERR_CAPACITY); i++)
        mismatch = p.x.req_first[i + 1] - p.x.req_first[i] != (p.rc[i] ? p.fix[i] : p.n_req[i]);
    if (!mismatch) return rc;
    // the records do not match the connections' requests (a caller stated a wrong count, or its bytes changed since its
    // route call): refuse the callers whose count differs and serve the others again
    if ((rc = count()) != GOFR_OK) return rc;
    return serve();
}

static void free_route(RouteStaging& r) {
    free_staging(r.x);
    for (void* q : {(void*)r.key, (void*)r.parsed, (void*)r.desc, (void*)r.vars, (void*)r.bstat, (void*)r.blen, (void*)r.brow, (void*)r.rows})
        gofr_free_pinned(q);
    r.key = nullptr; r.parsed = nullptr; r.desc = nullptr; r.vars = r.bstat = r.blen = nullptr; r.brow = nullptr; r.rows = nullptr;
    r.req_cap = 0; r.rows_cap = 0;
}

static void free_respond(RespondStaging& p) {
    free_staging(p.x);
    for (void* q : {(void*)p.key, (void*)p.rec_at, (void*)p.rec_off_at, (void*)p.n_req, (void*)p.rc, (void*)p.fix, (void*)p.rec, (void*)p.rec_off})
        gofr_free_pinned(q);
    p.key = nullptr; p.rec_at = nullptr; p.rec_off_at = nullptr; p.n_req = p.fix = p.rec_off = nullptr; p.rc = nullptr; p.rec = nullptr;
    p.rec_cap = 0; p.rec_off_cap = 0;
}

extern "C" {

int gofr_conn_app_frontend_create(gofr_conn_app_frontend** out, gofr_engine* e, uint32_t max_batch, uint32_t max_wait_us,
                                  uint32_t max_conn_bytes, int log, int32_t tz_offset_s, uint64_t seed, const uint32_t* route_schema,
                                  uint32_t n_routes, const uint32_t* schema_fields) {
    if (!out || !e || max_batch == 0 || max_batch > 0x7FFFFFFFu || (n_routes && (!route_schema || !schema_fields)))
        return GOFR_ERR_INVALID;
    const uint64_t arena = (uint64_t)max_batch * max_conn_bytes;
    if (arena > 0xFFFFFFF0ull) {
        set_last_error("gofr_conn_app_frontend_create: %u reads of %u bytes exceed 32-bit offsets", max_batch, max_conn_bytes);
        return GOFR_ERR_CAPACITY;
    }
    AppFrontend* f = new AppFrontend(max_batch, max_wait_us);
    f->eng = e;
    f->max_conn_bytes = max_conn_bytes;
    f->log = log != 0;
    f->tz_offset_s = tz_offset_s;
    f->seed = seed;
    f->route_schema.assign(route_schema, route_schema + n_routes);
    f->schema_fields.assign(schema_fields, schema_fields + n_routes);
    for (uint32_t s : f->route_schema)
        if (s && std::find(f->schemas.begin(), f->schemas.end(), s) == f->schemas.end()) f->schemas.push_back(s);
    const size_t n = max_batch;
    bool ok = true;
    for (auto& r : f->rb) {
        ok = ok && alloc_staging(r.x, max_batch, arena, false);
        r.key = (uint64_t*)gofr_alloc_pinned(n * 8);
        r.parsed = (uint8_t*)gofr_alloc_pinned((size_t)arena + 64);
        ok = ok && r.key && r.parsed;
    }
    for (auto& p : f->pb) {
        ok = ok && alloc_staging(p.x, max_batch, arena);
        p.key = (uint64_t*)gofr_alloc_pinned(n * 8);
        p.rec_at = (const uint8_t**)gofr_alloc_pinned(n * sizeof(void*));
        p.rec_off_at = (const uint32_t**)gofr_alloc_pinned(n * sizeof(void*));
        p.n_req = (uint32_t*)gofr_alloc_pinned(n * 4);
        p.rc = (int*)gofr_alloc_pinned(n * sizeof(int));
        p.fix = (uint32_t*)gofr_alloc_pinned(n * 4);
        ok = ok && p.key && p.rec_at && p.rec_off_at && p.n_req && p.rc && p.fix;
    }
    if (!ok) {
        for (auto& r : f->rb) free_route(r);
        for (auto& p : f->pb) free_respond(p);
        delete f;
        return GOFR_ERR_NOMEM;
    }
    f->route.start([f](int k, uint32_t n, uint32_t a) { return route_batch(f, k, n, a); });
    f->respond.start([f](int k, uint32_t n, uint32_t a) { return respond_batch(f, k, n, a); });
    *out = f;
    return GOFR_OK;
}

void gofr_conn_app_frontend_destroy(gofr_conn_app_frontend* f) {
    if (!f) return;
    f->route.stop();
    f->respond.stop();
    for (auto& r : f->rb) free_route(r);
    for (auto& p : f->pb) free_respond(p);
    delete f;
}

int gofr_conn_app_frontend_set_clock(gofr_conn_app_frontend* f, int64_t unix_ns) {
    if (!f) return GOFR_ERR_INVALID;
    f->fixed_clock.store(unix_ns, std::memory_order_relaxed);
    return GOFR_OK;
}

int gofr_conn_app_frontend_stats(gofr_conn_app_frontend* f, gofr_conn_app_stats* st) {
    if (!f || !st) return GOFR_ERR_INVALID;
    st->route_batches = f->route.batches.load(std::memory_order_relaxed);
    st->route_reads = f->route.records.load(std::memory_order_relaxed);
    st->respond_batches = f->respond.batches.load(std::memory_order_relaxed);
    st->respond_reads = f->respond.records.load(std::memory_order_relaxed);
    st->reruns = f->reruns.load(std::memory_order_relaxed);
    st->isolated = f->isolated.load(std::memory_order_relaxed);
    st->gather_ns = f->gather_ns.load(std::memory_order_relaxed);
    return GOFR_OK;
}

int gofr_conn_app_frontend_route(gofr_conn_app_frontend* f, const uint8_t* buf, uint32_t len, gofr_conn_route* out,
                                 gofr_conn_app_bind* bind, uint64_t* trace_key) {
    if (!f || !out || !trace_key || (len && !buf) || !out->req_first || !out->consumed || !out->conn_status ||
        (len && !out->arena) || (out->req_cap && (!out->desc || !out->meta || !out->vars || !out->req_at || !out->trace_ids)))
        return GOFR_ERR_INVALID;
    if (bind && (!bind->row_off || (out->req_cap && !bind->status) || (bind->rows_cap && !bind->rows))) return GOFR_ERR_INVALID;
    if (len > f->max_conn_bytes) {
        set_last_error("a read of %u bytes exceeds the front-end's max_conn_bytes", len);
        return GOFR_ERR_CAPACITY;
    }
    if (bind) { bind->rows_bytes = 0; bind->row_off[0] = 0; }
    if (len == 0) {  // nothing to frame: done without joining a batch
        out->req_first[0] = out->req_first[1] = 0;
        out->consumed[0] = 0;
        out->conn_status[0] = GOFR_HTTP_CONN_DONE;
        *trace_key = 0;
        return GOFR_OK;
    }
    gofr_ring::Seat s;
    if (!f->route.claim(len, &s)) return GOFR_ERR_INVALID;
    RouteStaging& r = f->rb[s.k];
    memcpy(r.x.arena + s.a, buf, len);
    r.x.buf_off[s.i] = s.a;
    f->route.filled(s);

    const uint32_t n = f->route.wait(s);
    int rc = f->route.b[s.k].rc;
    if (rc == GOFR_OK) rc = route_out(r, s.i, s.a, len, out, bind, trace_key);
    f->route.leave(s, n);
    return rc;
}

int gofr_conn_app_frontend_respond(gofr_conn_app_frontend* f, const uint8_t* buf, uint32_t len, uint64_t trace_key,
                                   const gofr_conn_results* res, const uint8_t* remote, uint32_t remote_len, int64_t start_unix_ns,
                                   gofr_conn_resp* out, gofr_conn_log* log) {
    if (!f || !res) return GOFR_ERR_INVALID;
    if (int rc = check_read(len, buf, remote, remote_len, out, &log, f->log)) return rc;
    // the caller's records, checked before they are queued: n_req + 1 offsets within its record bytes, never decreasing,
    // and no more requests than its bytes can hold
    if ((res->n_req && !res->rec_off) || (res->rec_bytes && !res->rec) || res->n_req > staged_req_cap(1, len)) return GOFR_ERR_INVALID;
    for (uint32_t j = 0; j < res->n_req; j++)
        if (res->rec_off[j + 1] < res->rec_off[j] || res->rec_off[j + 1] > res->rec_bytes) {
            set_last_error("rec_off[%u] decreases or passes rec_bytes", j + 1);
            return GOFR_ERR_INVALID;
        }
    if (len > f->max_conn_bytes) {
        set_last_error("a read of %u bytes exceeds the front-end's max_conn_bytes", len);
        return GOFR_ERR_CAPACITY;
    }
    if (len == 0) {  // nothing to frame: done without joining a batch
        if (res->n_req) return GOFR_ERR_INVALID;
        no_requests(out, log, 0, GOFR_HTTP_CONN_DONE);
        return GOFR_OK;
    }
    static const uint32_t kNoRecords[1] = {0};
    gofr_ring::Seat s;
    if (!f->respond.claim(len, &s)) return GOFR_ERR_INVALID;
    RespondStaging& p = f->pb[s.k];
    memcpy(p.x.arena + s.a, buf, len);
    p.x.buf_off[s.i] = s.a;
    if (remote_len) memcpy(p.x.remote_at + (size_t)s.i * kRemoteMax, remote, remote_len);
    p.x.remote_len[s.i] = remote_len;
    p.x.start[s.i] = start_unix_ns;
    p.key[s.i] = trace_key;
    p.rec_at[s.i] = res->rec;
    p.rec_off_at[s.i] = res->n_req ? res->rec_off : kNoRecords;
    p.n_req[s.i] = res->n_req;
    f->respond.filled(s);

    const uint32_t n = f->respond.wait(s);
    int rc = f->respond.b[s.k].rc;
    if (rc == GOFR_OK && p.rc[s.i]) {
        rc = p.rc[s.i];
        if (rc == GOFR_ERR_INVALID) set_last_error("the records are for %u requests, the read holds %u", res->n_req, p.fix[s.i]);
        else set_last_error("the records of this read, with its batch-mates', pass the respond batch's 4 GiB of record offsets");
    } else if (rc == GOFR_OK) {
        rc = fan_out(p.x, s.i, s.a, out, log);
    }
    f->respond.leave(s, n);
    return rc;
}

}  // extern "C"
