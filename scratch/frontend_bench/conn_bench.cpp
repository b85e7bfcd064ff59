// conn_bench.cpp — closed-loop load on gofr_conn_frontend_serve: T threads ("connections"), each sends its next read as soon
// as the previous one is answered.  A read holds 1–8 pipelined config-2 requests (synth.http_streams).  Reports connection
// reads/s, requests/s, per-call latency percentiles and the mean batch size; then, as the floor, batches of that mean size
// through gofr_conn_batch_submit called directly, back to back.
//   conn_bench <table.img> <buf.bin> <off.bin> <threads> <max_batch> <max_wait_us> <seconds> [log 0|1]
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
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

int main(int argc, char** argv) {
    if (argc < 8) { fprintf(stderr, "usage: conn_bench <table.img> <buf.bin> <off.bin> <threads> <max_batch> <max_wait_us> <seconds> [log]\n"); return 2; }
    auto img = slurp(argv[1]), buf = slurp(argv[2]), offb = slurp(argv[3]);
    const int T = atoi(argv[4]);
    const uint32_t max_batch = (uint32_t)atoi(argv[5]), wait_us = (uint32_t)atoi(argv[6]);
    const double secs = atof(argv[7]);
    const int log = argc > 8 ? atoi(argv[8]) : 0;
    const uint32_t* off = (const uint32_t*)offb.data();
    const uint32_t n = (uint32_t)(offb.size() / 4 - 1);
    uint32_t max_len = 0;
    for (uint32_t c = 0; c < n; c++) max_len = std::max(max_len, off[c + 1] - off[c]);
    gofr_table* tab = nullptr;
    CK(gofr_table_deserialize(&tab, img.data(), img.size()));
    gofr_engine* eng = nullptr;
    CK(gofr_engine_create(&eng, tab, 0));
    gofr_conn_frontend* fe = nullptr;
    CK(gofr_conn_frontend_create(&fe, eng, max_batch, wait_us, max_len, log, 0, 7));
    std::atomic<bool> stop{false};
    std::atomic<uint64_t> bad{0}, reqs{0};
    std::vector<std::vector<float>> lat((size_t)T);
    std::vector<std::thread> th;
    auto t0 = std::chrono::steady_clock::now();
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            const uint32_t cap = 1u << 20, req_cap = max_len / 16 + 1;
            std::vector<uint8_t> out(cap), ids(16 * (size_t)req_cap), lout(log ? cap : 1);
            std::vector<uint32_t> out_off(req_cap + 1), meta(req_cap), at(req_cap), loff(req_cap + 1), lreq(req_cap);
            uint32_t first[2], consumed, status;
            gofr_conn_resp o{};
            o.out = out.data(); o.out_cap = cap; o.req_cap = req_cap; o.out_off = out_off.data(); o.meta = meta.data();
            o.req_at = at.data(); o.trace_ids = ids.data(); o.req_first = first; o.consumed = &consumed; o.conn_status = &status;
            gofr_conn_log l{};
            l.line_cap = req_cap; l.out = lout.data(); l.out_cap = log ? cap : 0; l.log_off = loff.data(); l.log_req = lreq.data();
            const char remote[] = "192.0.2.1:50000";
            for (uint32_t c = (uint32_t)t % n; !stop.load(std::memory_order_relaxed); c = (c + (uint32_t)T) % n) {
                const uint32_t len = off[c + 1] - off[c];
                auto s = std::chrono::steady_clock::now();
                const int rc = gofr_conn_frontend_serve(fe, buf.data() + off[c], len, (const uint8_t*)remote, sizeof remote - 1, 0, &o,
                                                        log ? &l : nullptr);
                auto e = std::chrono::steady_clock::now();
                if (rc || status != GOFR_HTTP_CONN_DONE || consumed != len || first[1] == 0) bad++;
                reqs += first[1];
                lat[(size_t)t].push_back(std::chrono::duration<float, std::micro>(e - s).count());
            }
        });
    std::this_thread::sleep_for(std::chrono::duration<double>(secs));
    stop = true;
    for (auto& x : th) x.join();
    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    std::vector<float> all;
    for (auto& v : lat) all.insert(all.end(), v.begin(), v.end());
    std::sort(all.begin(), all.end());
    uint64_t batches = 0, conns = 0, reruns = 0;
    gofr_conn_frontend_stats(fe, &batches, &conns, &reruns);
    gofr_conn_frontend_destroy(fe);
    const double mean_batch = batches ? (double)conns / batches : 1.0;
    auto pct = [&](double p) { return all.empty() ? 0.f : all[(size_t)(p * (all.size() - 1))]; };

    // the floor: batches of the same mean size (consecutive connections) through gofr_conn_batch_submit, back to back
    const uint32_t B = std::min(n, std::max<uint32_t>(1, (uint32_t)(mean_batch + 0.5)));
    std::vector<uint32_t> boff(B + 1);
    uint32_t req_cap = 0;
    uint64_t out_cap = 0;
    for (uint32_t c0 = 0; c0 + B <= n; c0 += B) {  // capacities for every window the loop below serves
        for (uint32_t k = 0; k <= B; k++) boff[k] = off[c0 + k] - off[c0];
        uint32_t rq = 0;
        uint64_t oc = 0;
        CK(gofr_conn_batch_bound(tab, boff.data(), B, &rq, &oc));
        req_cap = std::max(req_cap, rq);
        out_cap = std::max(out_cap, oc);
    }
    uint8_t* pbuf = (uint8_t*)gofr_alloc_pinned(buf.size());
    memcpy(pbuf, buf.data(), buf.size());
    uint8_t* out = (uint8_t*)gofr_alloc_pinned(out_cap);
    uint8_t* ids = (uint8_t*)gofr_alloc_pinned(16 * (size_t)req_cap);
    uint32_t* cols = (uint32_t*)gofr_alloc_pinned(4 * (3 * ((size_t)req_cap + 1) + 3 * ((size_t)B + 1)));
    std::vector<float> floor_us;
    const auto f0 = std::chrono::steady_clock::now();
    uint64_t floor_reqs = 0;
    for (uint32_t it = 0, c0 = 0; std::chrono::steady_clock::now() - f0 < std::chrono::duration<double>(std::min(secs, 2.0)) || it < 20; it++) {
        if (c0 + B > n) c0 = 0;
        for (uint32_t k = 0; k <= B; k++) boff[k] = off[c0 + k] - off[c0];
        gofr_conn_batch in{};
        in.buf = pbuf + off[c0]; in.buf_off = boff.data(); in.buf_bytes = boff[B]; in.n_conns = B; in.trace_seed = it;
        gofr_format_http_date(1700000000, in.date);
        gofr_conn_resp o{};
        uint32_t* p = cols;
        o.out = out; o.out_cap = out_cap; o.req_cap = req_cap; o.out_off = p; p += req_cap + 1; o.meta = p; p += req_cap + 1;
        o.req_at = p; p += req_cap + 1; o.trace_ids = ids; o.req_first = p; p += B + 1; o.consumed = p; p += B + 1; o.conn_status = p;
        auto s = std::chrono::steady_clock::now();
        gofr_ticket t = 0;
        CK(gofr_conn_batch_submit(eng, &in, &o, &t));
        CK(gofr_batch_wait(eng, t));
        floor_us.push_back(std::chrono::duration<float, std::micro>(std::chrono::steady_clock::now() - s).count());
        floor_reqs += o.req_first[B];
        c0 += B;
    }
    std::sort(floor_us.begin(), floor_us.end());
    const float floor_med = floor_us[floor_us.size() / 2];
    const double floor_req_per_batch = (double)floor_reqs / floor_us.size();
    printf("{\"threads\": %d, \"max_batch\": %u, \"max_wait_us\": %u, \"log\": %d, \"calls\": %zu, \"conn_per_s\": %.0f, "
           "\"req_per_s\": %.0f, \"batches\": %llu, \"reruns\": %llu, \"mean_batch\": %.1f, \"lat_us_p50\": %.1f, \"lat_us_p99\": %.1f, "
           "\"floor_batch\": %u, \"floor_us_per_batch_p50\": %.1f, \"floor_conn_per_s\": %.0f, \"floor_req_per_s\": %.0f, \"bad\": %llu}\n",
           T, max_batch, wait_us, log, all.size(), all.size() / el, reqs.load() / el, (unsigned long long)batches,
           (unsigned long long)reruns, mean_batch, pct(0.5), pct(0.99), B, floor_med, B / (floor_med * 1e-6),
           floor_req_per_batch / (floor_med * 1e-6), (unsigned long long)bad.load());
    gofr_free_pinned(pbuf); gofr_free_pinned(out); gofr_free_pinned(ids); gofr_free_pinned(cols);
    gofr_engine_destroy(eng);
    gofr_table_destroy(tab);
    return bad.load() ? 1 : 0;
}
