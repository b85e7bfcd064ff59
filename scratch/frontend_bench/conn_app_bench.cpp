// conn_app_bench.cpp — closed-loop load on the closure-path front-end (gofr_conn_app_frontend_route / _respond): T threads
// ("connections"), each loops read → route → its closures → respond, sending its next read as soon as the previous one is
// answered.  A read holds 1–8 pipelined config-2 requests (synth.http_streams); the closures are trivial (every request's
// record is empty, so the route's own handler answers it), which leaves the two batching rounds as the cost.  Reports reads/s,
// requests/s, per-read latency percentiles, the mean route and respond batch sizes and the respond dispatcher's record-gather
// time; then gofr_conn_frontend_serve on the same reads and threads (one round per read); then, as the floor, batches of the
// mean respond batch size through gofr_conn_batch_route + gofr_conn_batch_respond_ex called directly, back to back.
//   conn_app_bench <table.img> <buf.bin> <off.bin> <threads> <max_batch> <max_wait_us> <seconds>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#include "../../include/gofr_b200.h"

static std::vector<uint8_t> slurp(const char* p) {
    FILE* f = fopen(p, "rb");
    if (!f) { perror(p); exit(2); }
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<uint8_t> v((size_t)n);
    if (n && fread(v.data(), 1, (size_t)n, f) != (size_t)n) { perror(p); exit(2); }
    fclose(f);
    return v;
}
#define CK(x) do { int rc_ = (x); if (rc_) { fprintf(stderr, "%s -> %d: %s\n", #x, rc_, gofr_last_error()); exit(1); } } while (0)
using Clock = std::chrono::steady_clock;

// T threads run `one(t, c)` on connection reads c = t, t + T, ... for `secs`; returns (reads/s, requests/s, p50, p99 µs)
struct Load { double reads_s, reqs_s; float p50, p99; uint64_t bad; };
static Load closed_loop(int T, uint32_t n, double secs, const std::function<uint32_t(int, uint32_t, bool*)>& one) {
    std::atomic<bool> stop{false};
    std::atomic<uint64_t> bad{0}, reqs{0};
    std::vector<std::vector<float>> lat((size_t)T);
    std::vector<std::thread> th;
    const auto t0 = Clock::now();
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            for (uint32_t c = (uint32_t)t % n; !stop.load(std::memory_order_relaxed); c = (c + (uint32_t)T) % n) {
                bool ok = true;
                const auto s = Clock::now();
                reqs += one(t, c, &ok);
                lat[(size_t)t].push_back(std::chrono::duration<float, std::micro>(Clock::now() - s).count());
                if (!ok) bad++;
            }
        });
    std::this_thread::sleep_for(std::chrono::duration<double>(secs));
    stop = true;
    for (auto& x : th) x.join();
    const double el = std::chrono::duration<double>(Clock::now() - t0).count();
    std::vector<float> all;
    for (auto& v : lat) all.insert(all.end(), v.begin(), v.end());
    std::sort(all.begin(), all.end());
    auto pct = [&](double p) { return all.empty() ? 0.f : all[(size_t)(p * (all.size() - 1))]; };
    return Load{all.size() / el, reqs.load() / el, pct(0.5), pct(0.99), bad.load()};
}

int main(int argc, char** argv) {
    if (argc < 8) { fprintf(stderr, "usage: conn_app_bench <table.img> <buf.bin> <off.bin> <threads> <max_batch> <max_wait_us> <seconds>\n"); return 2; }
    auto img = slurp(argv[1]), buf = slurp(argv[2]), offb = slurp(argv[3]);
    const int T = atoi(argv[4]);
    const uint32_t max_batch = (uint32_t)atoi(argv[5]), wait_us = (uint32_t)atoi(argv[6]);
    const double secs = atof(argv[7]);
    const uint32_t* off = (const uint32_t*)offb.data();
    const uint32_t n = (uint32_t)(offb.size() / 4 - 1);
    uint32_t max_len = 0;
    for (uint32_t c = 0; c < n; c++) max_len = std::max(max_len, off[c + 1] - off[c]);
    gofr_table* tab = nullptr;
    CK(gofr_table_deserialize(&tab, img.data(), img.size()));
    gofr_engine* eng = nullptr;
    CK(gofr_engine_create(&eng, tab, 0));
    const uint32_t req_cap = max_len / 16 + 1, cap = 1u << 20;

    // ---- the closure path: route, trivial closures, respond ----
    gofr_conn_app_frontend* af = nullptr;
    CK(gofr_conn_app_frontend_create(&af, eng, max_batch, wait_us, max_len, 0, 0, 7, nullptr, 0, nullptr));
    struct Bufs {
        std::vector<gofr_req_desc> desc;
        std::vector<uint8_t> arena, ids, out;
        std::vector<uint32_t> meta, vars, at, out_off, rec_off;
    };
    std::vector<Bufs> bufs((size_t)T);
    for (auto& b : bufs) {
        b.desc.resize(req_cap); b.arena.resize(max_len + 80); b.ids.resize(16 * (size_t)req_cap); b.out.resize(cap);
        b.meta.resize(req_cap); b.vars.resize((size_t)req_cap * GOFR_MAX_PATH_VARS); b.at.resize(req_cap);
        b.out_off.resize(req_cap + 1); b.rec_off.resize(req_cap + 1);
    }
    const Load app = closed_loop(T, n, secs, [&](int t, uint32_t c, bool* ok) -> uint32_t {
        Bufs& b = bufs[(size_t)t];
        const uint8_t* r = buf.data() + off[c];
        const uint32_t len = off[c + 1] - off[c];
        uint32_t first[2], consumed, status;
        gofr_conn_route rt{};
        rt.req_cap = req_cap; rt.desc = b.desc.data(); rt.arena = b.arena.data(); rt.meta = b.meta.data(); rt.vars = b.vars.data();
        rt.req_at = b.at.data(); rt.trace_ids = b.ids.data(); rt.req_first = first; rt.consumed = &consumed; rt.conn_status = &status;
        uint64_t key = 0;
        if (gofr_conn_app_frontend_route(af, r, len, &rt, nullptr, &key)) { *ok = false; return 0; }
        const uint32_t k = first[1];
        std::fill(b.rec_off.begin(), b.rec_off.begin() + k + 1, 0u);  // the closures: every record empty
        gofr_conn_results res{nullptr, b.rec_off.data(), 0, k, 0};
        gofr_conn_resp o{};
        o.out = b.out.data(); o.out_cap = cap; o.req_cap = req_cap; o.out_off = b.out_off.data(); o.meta = b.meta.data();
        o.req_at = b.at.data(); o.trace_ids = b.ids.data(); o.req_first = first; o.consumed = &consumed; o.conn_status = &status;
        const int rc = gofr_conn_app_frontend_respond(af, r, len, key, &res, nullptr, 0, 0, &o, nullptr);
        *ok = rc == 0 && status == GOFR_HTTP_CONN_DONE && consumed == len && first[1] == k && k > 0;
        return k;
    });
    gofr_conn_app_stats st{};
    CK(gofr_conn_app_frontend_stats(af, &st));
    gofr_conn_app_frontend_destroy(af);
    const double route_batch = st.route_batches ? (double)st.route_reads / st.route_batches : 0;
    const double respond_batch = st.respond_batches ? (double)st.respond_reads / st.respond_batches : 0;

    // ---- the same reads through gofr_conn_frontend_serve (fused routes, one round) ----
    gofr_conn_frontend* fe = nullptr;
    CK(gofr_conn_frontend_create(&fe, eng, max_batch, wait_us, max_len, 0, 0, 7));
    const Load fused = closed_loop(T, n, secs, [&](int t, uint32_t c, bool* ok) -> uint32_t {
        Bufs& b = bufs[(size_t)t];
        const uint32_t len = off[c + 1] - off[c];
        uint32_t first[2], consumed, status;
        gofr_conn_resp o{};
        o.out = b.out.data(); o.out_cap = cap; o.req_cap = req_cap; o.out_off = b.out_off.data(); o.meta = b.meta.data();
        o.req_at = b.at.data(); o.trace_ids = b.ids.data(); o.req_first = first; o.consumed = &consumed; o.conn_status = &status;
        const int rc = gofr_conn_frontend_serve(fe, buf.data() + off[c], len, nullptr, 0, 0, &o, nullptr);
        *ok = rc == 0 && status == GOFR_HTTP_CONN_DONE && consumed == len;
        return first[1];
    });
    uint64_t fb = 0, fc = 0;
    gofr_conn_frontend_stats(fe, &fb, &fc, nullptr);
    gofr_conn_frontend_destroy(fe);

    // ---- the floor: batches of the mean respond batch size through route + respond_ex, back to back ----
    const uint32_t B = std::min(n, std::max<uint32_t>(1, (uint32_t)(respond_batch + 0.5)));
    std::vector<uint32_t> boff(B + 1);
    uint32_t breq = 0;
    uint64_t bout = 0;
    for (uint32_t c0 = 0; c0 + B <= n; c0 += B) {
        for (uint32_t k = 0; k <= B; k++) boff[k] = off[c0 + k] - off[c0];
        uint32_t rq = 0;
        uint64_t oc = 0;
        CK(gofr_conn_batch_bound(tab, boff.data(), B, &rq, &oc));
        breq = std::max(breq, rq);
        bout = std::max(bout, oc);
    }
    uint8_t* pbuf = (uint8_t*)gofr_alloc_pinned(buf.size());
    memcpy(pbuf, buf.data(), buf.size());
    uint8_t* out = (uint8_t*)gofr_alloc_pinned(bout);
    uint8_t* ids = (uint8_t*)gofr_alloc_pinned(16 * (size_t)breq);
    uint8_t* parsed = (uint8_t*)gofr_alloc_pinned((size_t)max_len * B + 64);
    gofr_req_desc* desc = (gofr_req_desc*)gofr_alloc_pinned(sizeof(gofr_req_desc) * (size_t)breq);
    uint32_t* cols = (uint32_t*)gofr_alloc_pinned(4 * ((4 + GOFR_MAX_PATH_VARS) * ((size_t)breq + 1) + 3 * ((size_t)B + 1)));
    std::vector<uint64_t> keys(B);
    std::vector<float> floor_us;
    const auto f0 = Clock::now();
    for (uint32_t it = 0, c0 = 0; Clock::now() - f0 < std::chrono::duration<double>(std::min(secs, 2.0)) || it < 20; it++) {
        if (c0 + B > n) c0 = 0;
        for (uint32_t k = 0; k <= B; k++) boff[k] = off[c0 + k] - off[c0];
        gofr_conn_batch in{};
        in.buf = pbuf + off[c0]; in.buf_off = boff.data(); in.buf_bytes = boff[B]; in.n_conns = B; in.trace_seed = it;
        gofr_format_http_date(1700000000, in.date);
        uint32_t* p = cols;
        gofr_conn_route rt{};
        rt.req_cap = breq; rt.desc = desc; rt.arena = parsed; rt.meta = p; p += breq + 1; rt.vars = p; p += (size_t)(breq + 1) * GOFR_MAX_PATH_VARS;
        rt.req_at = p; p += breq + 1; rt.trace_ids = ids; rt.req_first = p; p += B + 1; rt.consumed = p; p += B + 1; rt.conn_status = p; p += B + 1;
        uint32_t* rec_off = p;
        const auto s = Clock::now();
        CK(gofr_conn_batch_route(eng, &in, &rt));
        const uint32_t k = rt.req_first[B];
        std::fill(rec_off, rec_off + k + 1, 0u);
        for (uint32_t c = 0; c < B; c++) keys[c] = it * 0x9E3779B97F4A7C15ull + c;
        gofr_conn_results res{nullptr, rec_off, 0, k, 0};
        gofr_conn_resp o{};
        o.out = out; o.out_cap = bout; o.req_cap = breq; o.out_off = rt.vars; o.meta = rt.meta; o.req_at = rt.req_at; o.trace_ids = ids;
        o.req_first = rt.req_first; o.consumed = rt.consumed; o.conn_status = rt.conn_status;
        gofr_ticket t = 0;
        CK(gofr_conn_batch_respond_ex(eng, &in, keys.data(), &res, &o, nullptr, &t));
        CK(gofr_batch_wait(eng, t));
        floor_us.push_back(std::chrono::duration<float, std::micro>(Clock::now() - s).count());
        c0 += B;
    }
    std::sort(floor_us.begin(), floor_us.end());
    const float floor_med = floor_us[floor_us.size() / 2];
    printf("{\"threads\": %d, \"max_batch\": %u, \"max_wait_us\": %u, \"reads_per_s\": %.0f, \"req_per_s\": %.0f, \"lat_us_p50\": %.1f, "
           "\"lat_us_p99\": %.1f, \"route_batch\": %.1f, \"respond_batch\": %.1f, \"gather_us_per_batch\": %.2f, "
           "\"reruns\": %llu, \"isolated\": %llu, \"fused_reads_per_s\": %.0f, \"fused_lat_us_p50\": %.1f, \"fused_lat_us_p99\": %.1f, "
           "\"fused_batch\": %.1f, \"floor_batch\": %u, \"floor_us_per_batch_p50\": %.1f, \"floor_reads_per_s\": %.0f, \"bad\": %llu}\n",
           T, max_batch, wait_us, app.reads_s, app.reqs_s, app.p50, app.p99, route_batch, respond_batch,
           st.respond_batches ? st.gather_ns / 1e3 / st.respond_batches : 0.0, (unsigned long long)st.reruns,
           (unsigned long long)st.isolated, fused.reads_s, fused.p50, fused.p99, fb ? (double)fc / fb : 0.0, B, floor_med,
           B / (floor_med * 1e-6), (unsigned long long)(app.bad + fused.bad));
    gofr_free_pinned(pbuf); gofr_free_pinned(out); gofr_free_pinned(ids); gofr_free_pinned(parsed); gofr_free_pinned(desc); gofr_free_pinned(cols);
    gofr_engine_destroy(eng);
    gofr_table_destroy(tab);
    return app.bad + fused.bad ? 1 : 0;
}
