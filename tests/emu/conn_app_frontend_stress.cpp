// TEST INFRASTRUCTURE ONLY: the closure-path front-end's two rounds (gofr_b200/csrc/conn_app_frontend.cpp) on the CPU, under
// ThreadSanitizer, with stubs in place of gofr_conn_batch_route, gofr_batch_bind, gofr_conn_batch_respond_ex and
// gofr_batch_wait.  The stubs check every batch as the engine does (buf_off tiles the arena, records tile rec_off, the
// record count equals the batch's request count) and answer connection c from ITS bytes only: requests, routes, parsed
// forms, binds, and responses and log lines that also mix in its records, remote string, start clock and trace key.  The
// route stub remembers which bytes each key was handed out for; the respond stub checks that every connection comes back
// with the key its route call returned, and counts the respond batches that mix connections from different route batches.
//   conn_app_frontend_stress <threads> <reads_per_thread> <max_batch> <max_wait_us> <max_conn_bytes> <log 0|1> <seed>
//                            <park 0|1> <bad 0|1>
// park: thread 0 routes once and responds only after every other thread has finished all its reads (a one-batch design
// would deadlock); bad: every eleventh read responds with one record too many and must get GOFR_ERR_INVALID alone.
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../gofr_b200/csrc/conn_app_frontend.cpp"

static std::atomic<uint64_t> g_violations{0}, g_largest{0}, g_refused{0}, g_mixed{0}, g_route_calls{0}, g_respond_calls{0};
static int g_wait_rc = 0;  // the respond dispatcher's alone
static const int64_t kClock = 1700000000123456789ll;
static const int32_t kTz = 5400;
static std::mutex g_mu;
static std::map<uint64_t, std::pair<uint64_t, uint64_t>> g_keys;  // key → (hash of the read, route batch)

void set_last_error(const char*, ...) {}

static uint64_t mix(uint64_t h, const void* p, size_t n) {
    for (size_t j = 0; j < n; j++) h = (h ^ ((const uint8_t*)p)[j]) * 0x100000001B3ull;
    return h;
}
static uint64_t hash_of(const uint8_t* r, uint32_t len) { return mix(0xCBF29CE484222325ull, r, len); }

// what the route stub answers for one connection's bytes
struct Routed {
    uint32_t consumed = 0, status = 0;
    std::vector<uint32_t> meta, at;  // per request
};
static Routed routed(const uint8_t* r, uint32_t len) {
    Routed a;
    const uint64_t h = hash_of(r, len);
    const uint32_t nreq = len ? std::min(r[0] % 5u, len / 16 + 1) : 0;  // at most the framer's bound
    a.status = len ? (uint32_t)(h % 3) : (uint32_t)GOFR_HTTP_CONN_DONE;
    a.consumed = a.status == GOFR_HTTP_CONN_DONE ? len : (uint32_t)((h >> 8) % (len + 1));
    for (uint32_t j = 0; j < nreq; j++) {
        const uint64_t hj = splitmix64(h + j);
        a.meta.push_back((hj % 3 == 0 ? 200u : 0u) | (uint32_t)(hj >> 8) % 4u << 16);  // routes 0-3, a third answered by mux
        a.at.push_back(len * j / nreq);
    }
    return a;
}
static const uint32_t kRouteSchema[4] = {1, 1, 2, 0}, kFields[4] = {2, 2, 3, 0};

// the respond stub's answer for one connection: its responses and lines from its bytes, records, key, remote and clock
struct Answer {
    std::vector<std::string> resp;
    std::vector<std::pair<uint32_t, std::string>> lines;
};
static Answer answer(const uint8_t* r, uint32_t len, uint64_t key, const std::vector<std::string>& recs, const uint8_t* rem,
                     uint32_t rlen, int64_t start, const char* date, bool log) {
    Answer a;
    uint64_t h = mix(hash_of(r, len), &key, 8);
    h = mix(h, rem, rlen);
    h = mix(h, &start, 8);
    h = mix(h, date, 29);
    for (uint32_t j = 0; j < recs.size(); j++) {
        const uint64_t hj = splitmix64(mix(h + j, recs[j].data(), recs[j].size()));
        std::string o;
        const uint32_t size = (uint32_t)(hj >> 16) % (3000u + 16u * len);
        for (uint32_t m = 0; m < size; m++) o += (char)((uint8_t)(hj >> (8 * (m % 8))) ^ (uint8_t)m);
        a.resp.push_back(o);
        if (log && (hj >> 24) % 2 == 0) a.lines.push_back({j, "{\"line\":" + std::to_string(hj % 100000) + std::string((hj >> 32) % 500, 'l') + "}\n"});
    }
    return a;
}
static void id_of(uint64_t key, uint32_t j, uint8_t* out16) {
    const uint64_t id[2] = {splitmix64(key + 2ull * j), splitmix64(key + 2ull * j + 1)};
    memcpy(out16, id, 16);
}

static bool tiles(const gofr_conn_batch* in) {
    const uint32_t n = in->n_conns;
    bool bad = n == 0 || in->buf_off[0] != 0 || in->buf_off[n] != in->buf_bytes;
    for (uint32_t c = 0; c < n && !bad; c++) bad = in->buf_off[c + 1] <= in->buf_off[c];
    uint64_t l = g_largest.load();
    while (n > l && !g_largest.compare_exchange_weak(l, n)) {}
    return !bad;
}

extern "C" {
void* gofr_alloc_pinned(size_t n) { return calloc(1, n ? n : 1); }
void gofr_free_pinned(void* p) { free(p); }
void gofr_format_http_date(int64_t s, char out29[29]) {
    char tmp[40];
    snprintf(tmp, sizeof tmp, "Date-%024lld", (long long)s);
    memcpy(out29, tmp, 29);
}
int gofr_conn_batch_route(gofr_engine*, const gofr_conn_batch* in, gofr_conn_route* out) {
    const uint64_t b = g_route_calls++;
    const uint32_t n = in->n_conns;
    if (!tiles(in) || out->req_cap < in->buf_bytes / 16 + n) { g_violations++; return GOFR_ERR_INVALID; }
    uint32_t k = 0;
    for (uint32_t c = 0; c < n; c++) {
        const uint8_t* r = in->buf + in->buf_off[c];
        const uint32_t len = in->buf_off[c + 1] - in->buf_off[c];
        const Routed a = routed(r, len);
        const uint64_t key = splitmix64(in->trace_seed ^ splitmix64(c));  // the header's function of (trace_seed, c)
        {
            std::lock_guard<std::mutex> g(g_mu);
            g_keys[key] = {hash_of(r, len), b};
        }
        out->req_first[c] = k;
        out->consumed[c] = a.consumed;
        out->conn_status[c] = a.status;
        for (uint32_t x = in->buf_off[c]; x < in->buf_off[c + 1]; x++) out->arena[x] = in->buf[x] ^ 0x5A;
        for (uint32_t j = 0; j < a.meta.size(); j++, k++) {
            out->meta[k] = a.meta[j];
            out->req_at[k] = in->buf_off[c] + a.at[j];
            memset(&out->desc[k], 0, sizeof out->desc[k]);
            out->desc[k].arena_off = out->req_at[k];  // the parsed form: the stub's is the request's own first byte
            out->desc[k].data_len = j;
            for (uint32_t v = 0; v < GOFR_MAX_PATH_VARS; v++) out->vars[(size_t)k * GOFR_MAX_PATH_VARS + v] = a.meta[j] + v;
            id_of(key, j, out->trace_ids + (size_t)k * 16);
        }
    }
    out->req_first[n] = k;
    return GOFR_OK;
}
// row of a bound request: the schema, its parsed form's first byte and data_len bytes; data_len 3 passes any slot (a bind
// that does not keep to the length it reported), data_len 1 has 1024 bytes more (longer than the first slot of any batch
// these reads make: the front-end binds it again in a wider one)
int gofr_batch_bind(gofr_engine*, uint32_t schema, const gofr_req_batch* in, uint8_t* rows, uint32_t slot, uint32_t* len,
                    uint32_t* status) {
    for (uint32_t i = 0; i < in->n; i++) {
        const gofr_req_desc& d = in->desc[i];
        if (d.arena_off >= in->arena_bytes) { g_violations++; return GOFR_ERR_INVALID; }
        const uint32_t l = d.data_len == 3 ? slot + 1 : 2 + d.data_len + (d.data_len == 1 ? 1024u : 0u);
        len[i] = l;
        status[i] = d.data_len == 2 ? GOFR_BIND_ERROR : GOFR_BIND_OK;
        if (l > slot) continue;
        uint8_t* row = rows + (size_t)i * slot;
        row[0] = (uint8_t)schema;
        row[1] = in->arena[d.arena_off];
        memset(row + 2, 'r', l - 2);
    }
    return GOFR_OK;
}
int gofr_conn_batch_respond_ex(gofr_engine*, const gofr_conn_batch* in, const uint64_t* trace_key, const gofr_conn_results* res,
                               gofr_conn_resp* out, gofr_conn_log* log, gofr_ticket* t) {
    g_respond_calls++;
    const uint32_t n = in->n_conns;
    const uint32_t need_req = (uint32_t)(in->buf_bytes / 16 + n);
    if (!tiles(in) || !trace_key || out->req_cap < need_req ||
        (log && (log->remote_off[0] != 0 || log->line_cap < need_req || log->log_unix_ns != kClock || log->tz_offset_s != kTz))) {
        g_violations++;
        return GOFR_ERR_INVALID;
    }
    // every connection carries the key its route call handed out for these bytes
    std::set<uint64_t> from;
    for (uint32_t c = 0; c < n; c++) {
        const uint32_t len = in->buf_off[c + 1] - in->buf_off[c];
        std::lock_guard<std::mutex> g(g_mu);
        auto it = g_keys.find(trace_key[c]);
        if (it == g_keys.end() || it->second.first != hash_of(in->buf + in->buf_off[c], len)) { g_violations++; return GOFR_ERR_INVALID; }
        from.insert(it->second.second);
    }
    if (from.size() > 1) g_mixed++;
    std::vector<Routed> rt;
    uint32_t total = 0;
    for (uint32_t c = 0; c < n; c++) {
        rt.push_back(routed(in->buf + in->buf_off[c], in->buf_off[c + 1] - in->buf_off[c]));
        total += (uint32_t)rt.back().meta.size();
    }
    if (res) {  // the engine's check: as many records as requests, offsets that tile rec
        if (res->n_req != total) return GOFR_ERR_INVALID;
        for (uint32_t k = 0; k < total; k++)
            if (res->rec_off[k + 1] < res->rec_off[k] || res->rec_off[k + 1] > res->rec_bytes) { g_violations++; return GOFR_ERR_INVALID; }
    }
    std::vector<Answer> ans;
    uint64_t bytes = 0, lbytes = 0, lines = 0;
    uint32_t k0 = 0;
    for (uint32_t c = 0; c < n; c++) {
        std::vector<std::string> recs;
        for (uint32_t j = 0; j < rt[c].meta.size(); j++)
            recs.push_back(res ? std::string((const char*)res->rec + res->rec_off[k0 + j], res->rec_off[k0 + j + 1] - res->rec_off[k0 + j])
                               : std::string());
        k0 += (uint32_t)rt[c].meta.size();
        const uint8_t* rem = log ? log->remote + log->remote_off[c] : nullptr;
        const uint32_t rlen = log ? log->remote_off[c + 1] - log->remote_off[c] : 0;
        ans.push_back(answer(in->buf + in->buf_off[c], in->buf_off[c + 1] - in->buf_off[c], trace_key[c], recs, rem, rlen,
                             log ? log->start_unix_ns[c] : 0, in->date, log != nullptr));
        for (auto& s : ans.back().resp) bytes += s.size();
        for (auto& s : ans.back().lines) lbytes += s.second.size();
        lines += ans.back().lines.size();
    }
    out->out_bytes = bytes;
    if (log) { log->lines = (uint32_t)lines; log->out_bytes = lbytes; }
    uint32_t k = 0, m = 0;
    uint64_t pos = 0, lpos = 0;
    out->out_off[0] = 0;
    if (log) log->log_off[0] = 0;
    for (uint32_t c = 0; c < n; c++) {
        out->req_first[c] = k;
        out->consumed[c] = rt[c].consumed;
        out->conn_status[c] = rt[c].status;
        for (uint32_t j = 0; j < rt[c].meta.size(); j++, k++) {
            out->meta[k] = rt[c].meta[j] | 7u;
            out->req_at[k] = in->buf_off[c] + rt[c].at[j];
            id_of(trace_key[c], j, out->trace_ids + (size_t)k * 16);
            if (bytes <= out->out_cap) memcpy(out->out + pos, ans[c].resp[j].data(), ans[c].resp[j].size());
            pos += ans[c].resp[j].size();
            out->out_off[k + 1] = (uint32_t)pos;
        }
        for (auto& ln : ans[c].lines) {
            if (lbytes <= log->out_cap) memcpy(log->out + lpos, ln.second.data(), ln.second.size());
            lpos += ln.second.size();
            log->log_req[m] = out->req_first[c] + ln.first;
            log->log_off[++m] = (uint32_t)lpos;
        }
    }
    out->req_first[n] = k;
    g_wait_rc = bytes > out->out_cap || (log && lbytes > log->out_cap) ? GOFR_ERR_CAPACITY : GOFR_OK;
    if (g_wait_rc) g_refused++;
    *t = 1;
    return GOFR_OK;
}
int gofr_batch_wait(gofr_engine*, gofr_ticket) { return g_wait_rc; }
}

int main(int argc, char** argv) {
    if (argc < 10) return 2;
    const int T = atoi(argv[1]), R = atoi(argv[2]);
    const uint32_t max_batch = (uint32_t)atoi(argv[3]), wait_us = (uint32_t)atoi(argv[4]), max_len = (uint32_t)atoi(argv[5]);
    const bool log = atoi(argv[6]) != 0, park = atoi(argv[8]) != 0, bad_mode = atoi(argv[9]) != 0;
    const uint64_t seed = strtoull(argv[7], nullptr, 0);
    gofr_conn_app_frontend* fe = nullptr;
    if (gofr_conn_app_frontend_create(&fe, (gofr_engine*)0x1, max_batch, wait_us, max_len, log, kTz, seed, kRouteSchema, 4, kFields))
        return 2;
    gofr_conn_app_frontend_set_clock(fe, kClock);
    char date[29];
    gofr_format_http_date(kClock / 1000000000, date);
    std::atomic<uint64_t> bad{0}, queued{0}, empty{0}, over{0}, invalid_got{0}, bound{0}, rebound{0}, hosts{0}, finished{0}, parked_ok{0};
    std::vector<std::vector<uint64_t>> keys(T);

    // one read through both calls; false when anything differs from what the stubs say this read must get
    auto one_read = [&](int t, int r, bool wait_for_others) -> bool {
        const uint32_t len = r % 13 == 0 ? 0 : r % 13 == 1 ? max_len : r % 17 == 5 ? max_len + 1 : 1 + (uint32_t)((t * 977u + r * 131u) % max_len);
        std::vector<uint8_t> buf(len);
        for (uint32_t j = 0; j < len; j++) buf[j] = (uint8_t)(t * 31 + r * 7 + j * 13);
        const bool refuse = len > max_len;
        const Routed want = routed(buf.data(), refuse ? 0 : len);
        const uint32_t nreq = (uint32_t)want.meta.size(), rc1 = nreq + 1;
        // ---- route ----
        std::vector<gofr_req_desc> desc(rc1);
        std::vector<uint8_t> arena(len + 80), ids(rc1 * 16), rows(rc1 * 600 + len + 1024);
        std::vector<uint32_t> meta(rc1), vars(rc1 * GOFR_MAX_PATH_VARS), at(rc1), bstat(rc1), row_off(rc1 + 1);
        uint32_t first[2] = {9, 9}, consumed = 9, status = 9;
        gofr_conn_route ro;
        memset(&ro, 0, sizeof ro);
        ro.req_cap = nreq; ro.desc = desc.data(); ro.arena = arena.data(); ro.meta = meta.data(); ro.vars = vars.data(); ro.req_at = at.data();
        ro.trace_ids = ids.data(); ro.req_first = first; ro.consumed = &consumed; ro.conn_status = &status;
        gofr_conn_app_bind bd{bstat.data(), row_off.data(), rows.data(), rows.size(), 0};
        uint64_t key = 1;
        int rc = gofr_conn_app_frontend_route(fe, buf.data(), len, &ro, &bd, &key);
        if (refuse) { over++; return rc == GOFR_ERR_CAPACITY && first[0] == 9; }
        bool ok = rc == GOFR_OK && first[0] == 0 && first[1] == nreq && consumed == want.consumed && status == want.status;
        for (uint32_t j = 0; ok && j < nreq; j++) {
            uint8_t id[16];
            id_of(key, j, id);
            const uint32_t route = want.meta[j] >> 16, st = want.meta[j] & 0xFFFF;
            ok = meta[j] == want.meta[j] && at[j] == want.at[j] && memcmp(ids.data() + 16 * j, id, 16) == 0 && vars[j * GOFR_MAX_PATH_VARS + 3] == want.meta[j] + 3;
            ok = ok && desc[j].data_len == j && arena[desc[j].arena_off] == (buf[at[j]] ^ 0x5A) && desc[j].arena_off - at[j] < 16;
            const bool binds = st == 0 && kRouteSchema[route] != 0;
            const uint32_t rlen = row_off[j + 1] - row_off[j];
            if (!binds) ok = ok && bstat[j] == 0xFFFFFFFFu && rlen == 0;
            else if (j == 3) { ok = ok && bstat[j] == GOFR_BIND_HOST && rlen == 0; hosts++; }
            else {
                ok = ok && bstat[j] == (j == 2 ? (uint32_t)GOFR_BIND_ERROR : (uint32_t)GOFR_BIND_OK) && rlen == 2 + j + (j == 1 ? 1024u : 0u) &&
                     rows[row_off[j]] == kRouteSchema[route] && rows[row_off[j] + 1] == (buf[at[j]] ^ 0x5A) && (j == 0 || rows[row_off[j + 1] - 1] == 'r');
                bound++;
                if (j == 1) rebound++;
            }
        }
        if (len) keys[t].push_back(key);
        if (!ok) return false;
        if (wait_for_others)  // the parked caller: everybody else runs all its reads before it responds
            while (finished.load() + 1 < (uint64_t)T) std::this_thread::sleep_for(std::chrono::milliseconds(1));
        // ---- the closures: one record per request, some empty ----
        std::vector<std::string> recs;
        std::string rec;
        std::vector<uint32_t> rec_off{0};
        for (uint32_t j = 0; j < nreq; j++) {
            recs.push_back(std::string((t + r + j) % 3 ? (size_t)(5 + (t * 7 + j) % 40) : 0, (char)('A' + j)));
            rec += recs.back();
            rec_off.push_back((uint32_t)rec.size());
        }
        const bool wrong = bad_mode && len && r % 11 == 4;  // one record too many
        if (wrong) { rec += "extra"; rec_off.push_back((uint32_t)rec.size()); }
        // ---- respond ----
        std::string remote((size_t)((t * 7 + r) % 256), (char)('0' + r % 10));
        const int64_t start = 1000000ll * t + r;
        const Answer a = answer(buf.data(), len, key, recs, (const uint8_t*)remote.data(), log ? (uint32_t)remote.size() : 0, log ? start : 0, date, log);
        uint64_t want_bytes = 0, want_lbytes = 0;
        for (auto& s : a.resp) want_bytes += s.size();
        for (auto& s : a.lines) want_lbytes += s.second.size();
        std::vector<uint8_t> o(want_bytes + 16, 0xEE), lo(want_lbytes + 16, 0xEE), tid(rc1 * 16);
        std::vector<uint32_t> off(rc1 + 1), meta2(rc1), at2(rc1), loff(a.lines.size() + 1), lreq(a.lines.size() + 1);
        gofr_conn_resp cr;
        memset(&cr, 0, sizeof cr);
        cr.out = o.data(); cr.out_cap = want_bytes; cr.req_cap = nreq; cr.out_off = off.data(); cr.meta = meta2.data(); cr.req_at = at2.data();
        cr.trace_ids = tid.data(); cr.req_first = first; cr.consumed = &consumed; cr.conn_status = &status;
        gofr_conn_log cl;
        memset(&cl, 0, sizeof cl);
        cl.line_cap = (uint32_t)a.lines.size(); cl.out = lo.data(); cl.out_cap = want_lbytes; cl.log_off = loff.data(); cl.log_req = lreq.data();
        gofr_conn_results res{(const uint8_t*)rec.data(), rec_off.data(), rec.size(), (uint32_t)rec_off.size() - 1, 0};
        rc = gofr_conn_app_frontend_respond(fe, buf.data(), len, key, &res, (const uint8_t*)remote.data(), (uint32_t)remote.size(), start, &cr, &cl);
        if (wrong) { invalid_got += rc == GOFR_ERR_INVALID; return rc == GOFR_ERR_INVALID; }
        ok = rc == GOFR_OK && first[0] == 0 && first[1] == nreq && consumed == want.consumed && status == want.status && cr.out_bytes == want_bytes;
        ok = ok && (!log || (cl.lines == a.lines.size() && cl.out_bytes == want_lbytes));
        uint64_t p = 0;
        for (uint32_t j = 0; ok && j < nreq; j++) {
            uint8_t id[16];
            id_of(key, j, id);
            ok = memcmp(o.data() + p, a.resp[j].data(), a.resp[j].size()) == 0 && off[j + 1] == p + a.resp[j].size() &&
                 meta2[j] == (want.meta[j] | 7u) && at2[j] == want.at[j] && memcmp(tid.data() + 16 * j, id, 16) == 0;
            p += a.resp[j].size();
        }
        p = 0;
        for (uint32_t m = 0; ok && log && m < a.lines.size(); m++) {
            ok = memcmp(lo.data() + p, a.lines[m].second.data(), a.lines[m].second.size()) == 0 && lreq[m] == a.lines[m].first;
            p += a.lines[m].second.size();
        }
        ok = ok && o[want_bytes] == 0xEE && lo[want_lbytes] == 0xEE;
        if (len == 0) empty++;
        else queued++;
        return ok;
    };

    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            if (park && t == 0) {
                if (!one_read(0, 3, true)) bad++;  // routes, waits for all the others, responds
                else parked_ok++;
                return;
            }
            for (int r = 0; r < R; r++)
                if (!one_read(t, r, false)) { bad++; if (getenv("DBG")) fprintf(stderr, "bad t=%d r=%d\n", t, r); }
            finished++;
        });
    for (auto& x : th) x.join();
    gofr_conn_app_stats st;
    gofr_conn_app_frontend_stats(fe, &st);
    std::set<uint64_t> seen;
    uint64_t n_keys = 0;
    for (auto& v : keys) for (uint64_t k : v) { seen.insert(k); n_keys++; }
    if (seen.size() != n_keys) bad++;  // every read of every route batch got its own key
    // argument checks after the run
    {
        uint32_t f2[2], c2, s2, o2[1];
        gofr_conn_resp cr;
        memset(&cr, 0, sizeof cr);
        cr.out_off = o2; cr.req_first = f2; cr.consumed = &c2; cr.conn_status = &s2;
        gofr_conn_results none{nullptr, nullptr, 0, 0, 0};
        uint8_t b = 'G';
        uint32_t dec[3] = {0, 4, 2};
        gofr_conn_results decreasing{(const uint8_t*)"abcd", dec, 4, 2, 0};
        if (gofr_conn_app_frontend_respond(fe, &b, 1, 1, nullptr, nullptr, 0, 0, &cr, nullptr) != GOFR_ERR_INVALID) bad++;
        if (gofr_conn_app_frontend_respond(fe, &b, 1, 1, &decreasing, nullptr, 0, 0, &cr, nullptr) != GOFR_ERR_INVALID) bad++;
        if (gofr_conn_app_frontend_respond(fe, nullptr, 0, 1, &none, nullptr, 0, 0, &cr, nullptr) != GOFR_OK || f2[1] != 0) bad++;
        uint64_t key = 0;
        gofr_conn_route ro;
        memset(&ro, 0, sizeof ro);
        ro.req_first = f2; ro.consumed = &c2; ro.conn_status = &s2;
        if (gofr_conn_app_frontend_route(fe, &b, 1, &ro, nullptr, nullptr) != GOFR_ERR_INVALID) bad++;
        if (gofr_conn_app_frontend_route(fe, nullptr, 0, &ro, nullptr, &key) != GOFR_OK || f2[1] != 0 || s2 != GOFR_HTTP_CONN_DONE) bad++;
        gofr_conn_app_stats st2;
        gofr_conn_app_frontend_stats(fe, &st2);
        if (st2.route_batches != st.route_batches || st2.respond_batches != st.respond_batches) bad++;
    }
    gofr_conn_app_frontend_destroy(fe);
    printf("{\"queued\": %llu, \"empty\": %llu, \"over\": %llu, \"route_batches\": %llu, \"route_reads\": %llu, \"respond_batches\": %llu, "
           "\"respond_reads\": %llu, \"reruns\": %llu, \"isolated\": %llu, \"refused\": %llu, \"mixed\": %llu, \"largest\": %llu, "
           "\"respond_calls\": %llu, \"invalid_got\": %llu, \"bound\": %llu, \"rebound\": %llu, \"hosts\": %llu, \"keys\": %llu, \"parked_ok\": %llu, "
           "\"violations\": %llu, \"bad\": %llu}\n",
           (unsigned long long)queued.load(), (unsigned long long)empty.load(), (unsigned long long)over.load(),
           (unsigned long long)st.route_batches, (unsigned long long)st.route_reads, (unsigned long long)st.respond_batches,
           (unsigned long long)st.respond_reads, (unsigned long long)st.reruns, (unsigned long long)st.isolated,
           (unsigned long long)g_refused.load(), (unsigned long long)g_mixed.load(), (unsigned long long)g_largest.load(),
           (unsigned long long)g_respond_calls.load(), (unsigned long long)invalid_got.load(), (unsigned long long)bound.load(),
           (unsigned long long)rebound.load(), (unsigned long long)hosts.load(), (unsigned long long)n_keys, (unsigned long long)parked_ok.load(),
           (unsigned long long)g_violations.load(), (unsigned long long)bad.load());
    return bad.load() || g_violations.load() ? 1 : 0;
}
