// TEST INFRASTRUCTURE ONLY: the log front-end's fan-in / fan-out (gofr_b200/csrc/frontend.cpp, gofr_frontend_create_log)
// on the CPU, under ThreadSanitizer, with a stub engine: request i's response is built from ITS path and trace id, and its
// line, when its record asks for one, from ITS trace id and log strings, so every producer can tell whether it got its own
// answer and line back.  Every third producer call is a plain gofr_frontend_serve riding along as GOFR_LOG_NONE.
//   frontend_log_stress <threads> <requests_per_thread> <max_batch> <max_wait_us>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <vector>

#include "../../gofr_b200/csrc/frontend.cpp"

static std::atomic<uint64_t> g_plain{0}, g_logged{0};

void set_last_error(const char*, ...) {}
extern "C" {
void* gofr_alloc_pinned(size_t n) { return calloc(1, n ? n : 1); }
void gofr_free_pinned(void* p) { free(p); }
void gofr_format_http_date(int64_t t, char out[29]) { snprintf(out, 29, "%028lld", (long long)t); }
static uint32_t stub_response(const gofr_req_batch* in, uint32_t i, uint8_t* o) {
    const gofr_req_desc& d = in->desc[i];
    memcpy(o, in->trace_ids + (size_t)i * 16, 16);
    memcpy(o + 16, in->arena + d.arena_off, d.path_len);
    return 16u + d.path_len;
}
static void stub_slots(const gofr_req_batch* in, gofr_slot_batch* out) {
    for (uint32_t i = 0; i < in->n; i++) {
        uint8_t tmp[512];
        const uint32_t w = stub_response(in, i, tmp);
        out->out_len[i] = w;
        if (w <= out->slot_bytes) memcpy(out->out + (size_t)i * out->slot_bytes, tmp, w);
        out->meta[i] = 200u;
    }
}
int gofr_batch_submit_slots(gofr_engine*, const gofr_req_batch* in, gofr_slot_batch* out, gofr_ticket* t) {
    g_plain++;
    stub_slots(in, out);
    *t = 1;
    return 0;
}
// line of request i: its log_unix_ns (8 bytes), trace id, then its strings — or nothing for GOFR_LOG_NONE
int gofr_batch_submit_slots_log(gofr_engine*, const gofr_req_batch* in, gofr_slot_batch* out, gofr_batch_log* log, gofr_ticket* t) {
    g_logged++;
    stub_slots(in, out);
    uint32_t pos = 0;
    for (uint32_t i = 0; i < in->n; i++) {
        const gofr_log_desc& d = log->desc[i];
        log->log_off[i] = pos;
        if (d.kind != GOFR_LOG_REQUEST) continue;
        const uint32_t len = (uint32_t)d.method_len + d.ua_len + d.xff_len + d.remote_len + d.uri_len;
        if (d.arena_off + len > log->arena_bytes || pos + 24 + len > log->out_cap) return GOFR_ERR_INVALID;
        memcpy(log->out + pos, &log->log_unix_ns, 8);
        memcpy(log->out + pos + 8, in->trace_ids + (size_t)i * 16, 16);
        memcpy(log->out + pos + 24, log->arena + d.arena_off, len);
        pos += 24 + len;
    }
    log->log_off[in->n] = pos;
    *t = 1;
    return 0;
}
int gofr_batch_submit(gofr_engine*, const gofr_req_batch*, gofr_resp_batch*, gofr_ticket*) { return GOFR_ERR_INVALID; }
int gofr_batch_wait(gofr_engine*, gofr_ticket) { return 0; }
}

int main(int argc, char** argv) {
    const int T = argc > 1 ? atoi(argv[1]) : 16, R = argc > 2 ? atoi(argv[2]) : 200;
    const uint32_t max_batch = argc > 3 ? (uint32_t)atoi(argv[3]) : 8, wait_us = argc > 4 ? (uint32_t)atoi(argv[4]) : 100;
    gofr_frontend* fe = nullptr;
    if (gofr_frontend_create_log(&fe, (gofr_engine*)0x1, max_batch, wait_us, 256, 128, 64)) return 2;
    const int64_t clock = 1700000000123456789ll;
    gofr_frontend_set_log_clock(fe, clock);
    std::atomic<uint64_t> bad{0};
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            for (int r = 0; r < R; r++) {
                char path[64], strs[64];
                uint8_t id[16], resp[256], line[256];
                const int pl = snprintf(path, sizeof path, "/t%d/r%d", t, r);
                const int sl = snprintf(strs, sizeof strs, "GETua%d-%d", t, r);
                for (int k = 0; k < 16; k++) id[k] = (uint8_t)(t * 31 + r * 7 + k);
                uint32_t len = 0, meta = 0, ll = 12345;
                int rc;
                const int mode = r % 3;  // 0: logged, 1: GOFR_LOG_NONE through serve_log, 2: plain serve
                if (mode == 2) {
                    rc = gofr_frontend_serve(fe, 0, (const uint8_t*)path, (uint16_t)pl, nullptr, 0, 0, nullptr, 0, id, resp,
                                             sizeof resp, &len, &meta);
                    ll = 0;
                } else {
                    gofr_log_desc d;
                    memset(&d, 0, sizeof d);
                    d.method_len = 3; d.ua_len = (uint16_t)(sl - 3); d.kind = mode == 0 ? GOFR_LOG_REQUEST : GOFR_LOG_NONE;
                    rc = gofr_frontend_serve_log(fe, 0, (const uint8_t*)path, (uint16_t)pl, nullptr, 0, 0, nullptr, 0, id, &d,
                                                 (const uint8_t*)strs, resp, sizeof resp, &len, &meta, line, sizeof line, &ll);
                }
                bool ok = rc == 0 && len == 16u + (uint32_t)pl && memcmp(resp, id, 16) == 0 && memcmp(resp + 16, path, pl) == 0 &&
                          meta == 200u;
                if (mode == 0)
                    ok = ok && ll == 24u + (uint32_t)sl && memcmp(line, &clock, 8) == 0 && memcmp(line + 8, id, 16) == 0 &&
                         memcmp(line + 24, strs, sl) == 0;
                else
                    ok = ok && ll == 0;
                if (!ok) bad++;
            }
        });
    for (auto& x : th) x.join();
    uint64_t batches = 0, reqs = 0;
    gofr_frontend_stats(fe, &batches, &reqs);
    {   // a line longer than line_cap: reported with its length, the response delivered
        uint8_t id[16] = {0}, resp[64], line[8];
        uint32_t len = 0, ll = 0;
        gofr_log_desc d;
        memset(&d, 0, sizeof d);
        d.method_len = 3;
        int rc = gofr_frontend_serve_log(fe, 0, (const uint8_t*)"/x", 2, nullptr, 0, 0, nullptr, 0, id, &d, (const uint8_t*)"GET",
                                         resp, sizeof resp, &len, nullptr, line, sizeof line, &ll);
        if (rc != GOFR_ERR_CAPACITY || ll != 27 || len != 18) bad++;
        d.method_len = 65;  // past max_log_bytes
        rc = gofr_frontend_serve_log(fe, 0, (const uint8_t*)"/x", 2, nullptr, 0, 0, nullptr, 0, id, &d, (const uint8_t*)"GET",
                                     resp, sizeof resp, &len, nullptr, line, sizeof line, &ll);
        if (rc != GOFR_ERR_CAPACITY) bad++;
    }
    gofr_frontend_destroy(fe);
    printf("{\"requests\": %llu, \"batches\": %llu, \"plain_batches\": %llu, \"log_batches\": %llu, \"bad\": %llu}\n",
           (unsigned long long)reqs, (unsigned long long)batches, (unsigned long long)g_plain.load(),
           (unsigned long long)g_logged.load(), (unsigned long long)bad.load());
    return bad.load() || reqs != (uint64_t)T * R ? 1 : 0;
}
