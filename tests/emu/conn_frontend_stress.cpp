// TEST INFRASTRUCTURE ONLY: the connection front-end's fan-in / fan-out (gofr_b200/csrc/conn_frontend.cpp) on the CPU, under
// ThreadSanitizer, with stubs in place of gofr_conn_batch_submit_log and gofr_batch_wait.  The stub checks every batch as
// the engine does (buf_off tiles the arena from 0 to buf_bytes, remote strings back to back and at most 255 bytes, the
// per-request capacities at least one per 16 bytes plus one per connection) and "serves" connection c with requests,
// responses, a state and log lines derived from ITS bytes, remote string and start clock (and the batch's Date and log
// clock), so every caller can tell whether it got its own answer back.  When out_cap or the log's out_cap is short it
// writes nothing past them, reports what the batch needed and returns GOFR_ERR_CAPACITY from the wait, as the engine does;
// the front-end's first capacities are small enough that large batches take that path.
//   conn_frontend_stress <threads> <reads_per_thread> <max_batch> <max_wait_us> <max_conn_bytes> <log 0|1>
#include <cstdio>
#include <cstdlib>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../gofr_b200/csrc/conn_frontend.cpp"

static std::atomic<uint64_t> g_batches{0}, g_largest{0}, g_violations{0}, g_refused{0};
static int g_wait_rc = 0;               // the dispatcher's alone, as the engine's tickets are
static const int64_t kClock = 1700000000123456789ll;
static const int32_t kTz = 5400;

void set_last_error(const char*, ...) {}

static uint64_t mix(uint64_t h, const uint8_t* p, size_t n) {
    for (size_t j = 0; j < n; j++) h = (h ^ p[j]) * 0x100000001B3ull;
    return h;
}

// the stub's answer for one connection
struct Answer {
    uint32_t consumed = 0, status = 0;
    std::vector<uint32_t> meta, at;     // per request: meta, first byte within the connection
    std::vector<std::string> resp;
    std::vector<std::pair<uint32_t, std::string>> lines;  // (request, line)
};
static Answer answer(const uint8_t* r, uint32_t len, const uint8_t* rem, uint32_t rlen, int64_t start, const char* date, bool log) {
    Answer a;
    uint64_t h = mix(0xCBF29CE484222325ull, r, len);
    h = mix(h, rem, rlen);
    h = mix(h, (const uint8_t*)&start, 8);
    h = mix(h, (const uint8_t*)date, 29);
    const uint32_t nreq = len ? r[0] % 4u : 0;
    a.status = len ? (uint32_t)(h % 3) : (uint32_t)GOFR_HTTP_CONN_DONE;
    a.consumed = a.status == GOFR_HTTP_CONN_DONE ? len : (uint32_t)((h >> 8) % (len + 1));
    for (uint32_t j = 0; j < nreq; j++) {
        const uint64_t hj = splitmix64(h + j);
        const bool hole = hj % 5 == 0;
        a.meta.push_back(hole ? 0u : (200u | (uint32_t)(hj >> 40 & 0xFF) << 16));
        a.at.push_back(a.consumed * j / nreq);
        std::string o;
        const uint32_t size = hole ? 0 : (uint32_t)(hj >> 16) % (3000u + 16u * len);
        for (uint32_t m = 0; m < size; m++) o += (char)(r[m % len] ^ (uint8_t)(hj >> (8 * (m % 8))) ^ (uint8_t)m);
        a.resp.push_back(o);
        if (log && !hole && (hj >> 24) % 2 == 0) {
            std::string l = "{\"start\":" + std::to_string(start) + ",\"time\":" + std::to_string(kClock) + ",\"tz\":" +
                            std::to_string(kTz) + ",\"ip\":\"" + std::string((const char*)rem, rlen) + "\",\"x\":\"";
            for (uint32_t m = 0; m < (hj >> 32) % (400u + 8u * len); m++) l += (char)('a' + (hj + m) % 26);
            a.lines.push_back({j, l + "\"}\n"});
        }
    }
    return a;
}

extern "C" {
void* gofr_alloc_pinned(size_t n) { return calloc(1, n ? n : 1); }
void gofr_free_pinned(void* p) { free(p); }
void gofr_format_http_date(int64_t s, char out29[29]) {
    char tmp[40];
    snprintf(tmp, sizeof tmp, "Date-%024lld", (long long)s);
    memcpy(out29, tmp, 29);
}
int gofr_conn_batch_submit_log(gofr_engine*, const gofr_conn_batch* in, gofr_conn_resp* out, gofr_conn_log* log, gofr_ticket* t) {
    g_batches++;
    const uint32_t n = in->n_conns;
    uint64_t l = g_largest.load();
    while (n > l && !g_largest.compare_exchange_weak(l, n)) {}
    // the engine's checks, and the front-end's own promises: reads tile the arena, no read is empty, remote strings packed
    bool bad = n == 0 || in->buf_off[0] != 0 || in->buf_off[n] != in->buf_bytes;
    for (uint32_t c = 0; c < n && !bad; c++)
        bad = in->buf_off[c + 1] <= in->buf_off[c] || (log && (log->remote_off[c + 1] < log->remote_off[c] ||
                                                              log->remote_off[c + 1] - log->remote_off[c] > 255));
    const uint32_t need_req = (uint32_t)(in->buf_bytes / 16 + n);
    if (bad || out->req_cap < need_req || (log && (log->remote_off[0] != 0 || log->line_cap < need_req ||
                                                   log->log_unix_ns != kClock || log->tz_offset_s != kTz))) {
        g_violations++;
        return GOFR_ERR_INVALID;
    }
    std::vector<Answer> ans;
    uint64_t bytes = 0, lbytes = 0, reqs = 0, lines = 0;
    for (uint32_t c = 0; c < n; c++) {
        const uint8_t* rem = log ? log->remote + log->remote_off[c] : nullptr;
        const uint32_t rlen = log ? log->remote_off[c + 1] - log->remote_off[c] : 0;
        ans.push_back(answer(in->buf + in->buf_off[c], in->buf_off[c + 1] - in->buf_off[c], rem, rlen,
                             log ? log->start_unix_ns[c] : 0, in->date, log != nullptr));
        for (auto& s : ans.back().resp) bytes += s.size();
        for (auto& s : ans.back().lines) lbytes += s.second.size();
        reqs += ans.back().meta.size();
        lines += ans.back().lines.size();
    }
    out->out_bytes = bytes;
    if (log) { log->lines = (uint32_t)lines; log->out_bytes = lbytes; }
    uint32_t k = 0, m = 0;
    uint64_t pos = 0, lpos = 0;
    out->out_off[0] = 0;
    if (log) log->log_off[0] = 0;
    for (uint32_t c = 0; c < n; c++) {
        const Answer& a = ans[c];
        out->req_first[c] = k;
        out->consumed[c] = a.consumed;
        out->conn_status[c] = a.status;
        for (uint32_t j = 0; j < a.meta.size(); j++, k++) {
            out->meta[k] = a.meta[j];
            out->req_at[k] = in->buf_off[c] + a.at[j];
            const uint64_t key = splitmix64(in->trace_seed ^ splitmix64(c));  // the header's function of (trace_seed, c, j)
            const uint64_t id[2] = {splitmix64(key + 2ull * j), splitmix64(key + 2ull * j + 1)};
            memcpy(out->trace_ids + (size_t)k * 16, id, 16);
            if (bytes <= out->out_cap) memcpy(out->out + pos, a.resp[j].data(), a.resp[j].size());
            pos += a.resp[j].size();
            out->out_off[k + 1] = (uint32_t)pos;
        }
        for (auto& ln : a.lines) {
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
    if (argc < 7) return 2;
    const int T = atoi(argv[1]), R = atoi(argv[2]);
    const uint32_t max_batch = (uint32_t)atoi(argv[3]), wait_us = (uint32_t)atoi(argv[4]), max_len = (uint32_t)atoi(argv[5]);
    const bool log = atoi(argv[6]) != 0;
    gofr_conn_frontend* fe = nullptr;
    if (gofr_conn_frontend_create(&fe, (gofr_engine*)0x1, max_batch, wait_us, max_len, log, kTz, 0)) return 2;
    gofr_conn_frontend_set_clock(fe, kClock);
    char date[29];
    gofr_format_http_date(kClock / 1000000000, date);
    std::atomic<uint64_t> bad{0}, queued{0}, short_calls{0}, empty{0}, at_max{0}, over{0};
    std::vector<std::vector<std::string>> ids(T);
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            std::vector<uint8_t> buf;
            for (int r = 0; r < R; r++) {
                const uint32_t len = r % 13 == 0 ? 0 : r % 13 == 1 ? max_len : r % 17 == 5 ? max_len + 1
                                   : 1 + (uint32_t)((t * 977u + r * 131u) % max_len);
                buf.resize(len);
                for (uint32_t j = 0; j < len; j++) buf[j] = (uint8_t)(t * 31 + r * 7 + j * 13);
                std::string remote((size_t)((t * 7 + r) % 256), (char)('0' + r % 10));
                const int64_t start = 1000000ll * t + r;
                const bool refuse = len > max_len;
                // without lines the batch call sees no remote string and no clock
                Answer a = answer(buf.data(), refuse ? 0 : len, (const uint8_t*)remote.data(), log ? (uint32_t)remote.size() : 0,
                                  log ? start : 0, date, log);
                uint64_t want_bytes = 0, want_lbytes = 0;
                for (auto& s : a.resp) want_bytes += s.size();
                for (auto& s : a.lines) want_lbytes += s.second.size();
                const uint32_t nreq = (uint32_t)a.meta.size();
                // every fifth caller one byte short of its responses, every seventh one short of its log bytes
                const bool short_out = r % 5 == 2 && want_bytes > 0, short_log = log && r % 7 == 3 && want_lbytes > 0;
                const uint32_t req_cap = nreq + r % 3, line_cap = (uint32_t)a.lines.size() + r % 2;
                const uint64_t out_cap = short_out ? want_bytes - 1 : want_bytes + (r % 3) * 17;
                const uint64_t lcap = short_log ? want_lbytes - 1 : want_lbytes + (r % 2) * 5;
                const uint32_t canary = 16;
                std::vector<uint8_t> o(out_cap + canary, 0xEE), lo(lcap + canary, 0xEE), tid((req_cap + 1) * 16, 0xEE);
                std::vector<uint32_t> off(req_cap + 1 + canary, 0xEEEEEEEEu), meta(req_cap + canary, 0xEEEEEEEEu), at(req_cap + canary),
                                      loff(line_cap + 1 + canary, 0xEEEEEEEEu), lreq(line_cap + canary, 0xEEEEEEEEu);
                uint32_t first[2] = {9, 9}, consumed = 9, status = 9;
                gofr_conn_resp cr;
                memset(&cr, 0, sizeof cr);
                cr.out = o.data(); cr.out_cap = out_cap; cr.req_cap = req_cap; cr.out_off = off.data(); cr.meta = meta.data();
                cr.req_at = at.data(); cr.trace_ids = tid.data(); cr.req_first = first; cr.consumed = &consumed; cr.conn_status = &status;
                gofr_conn_log cl;
                memset(&cl, 0, sizeof cl);
                cl.line_cap = line_cap; cl.out = lo.data(); cl.out_cap = lcap; cl.log_off = loff.data(); cl.log_req = lreq.data();
                const int rc = gofr_conn_frontend_serve(fe, buf.data(), len, (const uint8_t*)remote.data(), (uint32_t)remote.size(), start,
                                                        &cr, &cl);
                bool ok;
                if (refuse) {
                    ok = rc == GOFR_ERR_CAPACITY && first[0] == 9;
                    over++;
                } else {
                    ok = first[0] == 0 && first[1] == nreq && consumed == a.consumed && status == a.status && cr.out_bytes == want_bytes;
                    ok = ok && (!log || (cl.lines == a.lines.size() && cl.out_bytes == want_lbytes));
                    ok = ok && rc == (short_out || short_log ? GOFR_ERR_CAPACITY : GOFR_OK);
                    if (!short_out) {  // the responses, rebased to this call's buffers
                        std::string all;
                        for (auto& s : a.resp) all += s;
                        ok = ok && memcmp(o.data(), all.data(), all.size()) == 0 && off[0] == 0;
                        uint32_t p = 0;
                        for (uint32_t j = 0; j < nreq; j++) {
                            p += (uint32_t)a.resp[j].size();
                            ok = ok && off[j + 1] == p && meta[j] == a.meta[j] && at[j] == a.at[j];
                            std::string id((const char*)tid.data() + 16 * j, 16);
                            ids[t].push_back(id);
                        }
                    } else {
                        ok = ok && o[0] == 0xEE;
                        short_calls++;
                    }
                    if (log && !short_log) {
                        std::string all;
                        uint32_t p = 0;
                        ok = ok && loff[0] == 0;
                        for (uint32_t m = 0; m < a.lines.size(); m++) {
                            all += a.lines[m].second;
                            p += (uint32_t)a.lines[m].second.size();
                            ok = ok && loff[m + 1] == p && lreq[m] == a.lines[m].first;
                        }
                        ok = ok && memcmp(lo.data(), all.data(), all.size()) == 0;
                    } else if (short_log) {
                        ok = ok && lo[0] == 0xEE;
                        short_calls++;
                    }
                    // nothing at or past a capacity
                    ok = ok && o[out_cap] == 0xEE && lo[lcap] == 0xEE && off[req_cap + 1] == 0xEEEEEEEEu && meta[req_cap] == 0xEEEEEEEEu &&
                         loff[line_cap + 1] == 0xEEEEEEEEu && lreq[line_cap] == 0xEEEEEEEEu;
                    if (len == 0) empty++;
                    else queued++;
                    if (len == max_len) at_max++;
                }
                if (!ok) bad++;
            }
        });
    for (auto& x : th) x.join();
    uint64_t batches = 0, conns = 0, reruns = 0;
    gofr_conn_frontend_stats(fe, &batches, &conns, &reruns);
    // every trace id the callers got is distinct: each batch draws its own seed
    std::set<std::string> seen;
    uint64_t n_ids = 0;
    for (auto& v : ids) for (auto& s : v) { seen.insert(s); n_ids++; }
    if (seen.size() != n_ids) bad++;
    // argument checks after the run: the front-end keeps its state
    {
        uint32_t first[2], consumed, status, off[1];
        gofr_conn_resp cr;
        memset(&cr, 0, sizeof cr);
        cr.out_off = off; cr.req_first = first; cr.consumed = &consumed; cr.conn_status = &status;
        uint8_t b = 'G';
        if (gofr_conn_frontend_serve(fe, nullptr, 1, nullptr, 0, 0, &cr, nullptr) != GOFR_ERR_INVALID) bad++;
        if (gofr_conn_frontend_serve(fe, &b, 1, nullptr, 0, 0, nullptr, nullptr) != GOFR_ERR_INVALID) bad++;
        std::string rem(256, 'x');
        if (gofr_conn_frontend_serve(fe, &b, 1, (const uint8_t*)rem.data(), 256, 0, &cr, nullptr) != GOFR_ERR_INVALID) bad++;
        if (gofr_conn_frontend_serve(fe, nullptr, 0, nullptr, 0, 0, &cr, nullptr) != GOFR_OK || first[1] != 0 ||
            status != GOFR_HTTP_CONN_DONE)
            bad++;
        uint64_t b2 = 0, c2 = 0;
        gofr_conn_frontend_stats(fe, &b2, &c2, nullptr);
        if (c2 != conns || b2 != batches) bad++;
    }
    gofr_conn_frontend_destroy(fe);
    printf("{\"conns\": %llu, \"queued\": %llu, \"batches\": %llu, \"stub_batches\": %llu, \"largest\": %llu, \"reruns\": %llu, "
           "\"refused\": %llu, \"short\": %llu, \"empty\": %llu, \"at_max\": %llu, \"over\": %llu, \"ids\": %llu, \"violations\": %llu, "
           "\"bad\": %llu}\n",
           (unsigned long long)conns, (unsigned long long)queued.load(), (unsigned long long)batches, (unsigned long long)g_batches.load(),
           (unsigned long long)g_largest.load(), (unsigned long long)reruns, (unsigned long long)g_refused.load(),
           (unsigned long long)short_calls.load(), (unsigned long long)empty.load(), (unsigned long long)at_max.load(),
           (unsigned long long)over.load(), (unsigned long long)n_ids, (unsigned long long)g_violations.load(), (unsigned long long)bad.load());
    return bad.load() || g_violations.load() || conns != queued.load() ? 1 : 0;
}
