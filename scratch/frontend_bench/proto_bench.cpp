// proto_bench.cpp — closed-loop load on the gRPC front-ends: T threads, each runs unary SayHello RPCs back to back, each
// RPC = gofr_proto_frontend_call (decode) → SayHello on the host → gofr_proto_frontend_call (encode).  Reports RPCs/s and
// per-RPC latency percentiles; then, as the floor, the same mean batch size through gofr_proto_batch_decode / _encode
// called directly (one decode batch, the handler, one encode batch, back to back).
//   proto_bench <threads> <max_batch> <max_wait_us> <seconds>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/gofr_b200.h"

#define CK(x) do { int rc_ = (x); if (rc_) { fprintf(stderr, "%s -> %d: %s\n", #x, rc_, gofr_last_error()); exit(1); } } while (0)

static const gofr_proto_nmsg kMsg{0, 1};
static const gofr_proto_nfield kField{1, GOFR_PB_STRING, 0, 0};  // HelloRequest.name / HelloResponse.message

static std::string name_of(size_t i) { return "caller-" + std::to_string(i % 100000); }
static std::string request_message(const std::string& name) { return std::string("\x0a", 1) + (char)name.size() + name; }
static std::string hello_row(const uint8_t* row) {  // SayHello on a decoded HelloRequest row → a HelloResponse row
    uint32_t n = 0;
    memcpy(&n, row, 4);
    std::string name((const char*)row + 4, n);
    if (name.empty()) name = "World";
    const std::string msg = "Hello " + name + "!";
    std::string out(4, '\0');
    const uint32_t m = (uint32_t)msg.size();
    memcpy(&out[0], &m, 4);
    return out + msg;
}

int main(int argc, char** argv) {
    if (argc < 5) { fprintf(stderr, "usage: proto_bench <threads> <max_batch> <max_wait_us> <seconds>\n"); return 2; }
    const int T = atoi(argv[1]);
    const uint32_t max_batch = (uint32_t)atoi(argv[2]), wait_us = (uint32_t)atoi(argv[3]);
    const double secs = atof(argv[4]);
    gofr_table* tab = nullptr;
    CK(gofr_table_create(&tab, GOFR_FRAME_WIRE));
    CK(gofr_table_add_default_routes(tab, nullptr, 0));
    CK(gofr_table_seal(tab));
    gofr_engine* eng = nullptr;
    CK(gofr_engine_create(&eng, tab, 0));
    gofr_proto_frontend *dec = nullptr, *enc = nullptr;
    CK(gofr_proto_frontend_create(&dec, eng, &kMsg, 1, &kField, 1, 0, nullptr, 1, max_batch, wait_us, 256));
    CK(gofr_proto_frontend_create(&enc, eng, &kMsg, 1, &kField, 1, 0, nullptr, 0, max_batch, wait_us, 256));
    std::atomic<bool> stop{false};
    std::atomic<uint64_t> bad{0};
    std::vector<std::vector<float>> lat((size_t)T);
    std::vector<std::thread> th;
    auto t0 = std::chrono::steady_clock::now();
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            uint8_t row[512], msg[512];
            size_t i = (size_t)t;
            while (!stop.load(std::memory_order_relaxed)) {
                const std::string name = name_of(i), in = request_message(name);
                uint32_t n = 0, st = 0, n2 = 0, st2 = 0;
                auto s = std::chrono::steady_clock::now();
                int rc = gofr_proto_frontend_call(dec, (const uint8_t*)in.data(), (uint32_t)in.size(), row, sizeof row, &n, &st);
                if (rc == 0 && st == GOFR_GRPC_OK) {
                    const std::string resp = hello_row(row);
                    rc = gofr_proto_frontend_call(enc, (const uint8_t*)resp.data(), (uint32_t)resp.size(), msg, sizeof msg, &n2, &st2);
                }
                auto e = std::chrono::steady_clock::now();
                const std::string want = "Hello " + name + "!";
                if (rc || st || st2 || n2 != want.size() + 2 || memcmp(msg + 2, want.data(), want.size()) != 0) bad++;
                lat[(size_t)t].push_back(std::chrono::duration<float, std::micro>(e - s).count());
                i += (size_t)T;
            }
        });
    std::this_thread::sleep_for(std::chrono::duration<double>(secs));
    stop = true;
    for (auto& x : th) x.join();
    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    std::vector<float> all;
    for (auto& v : lat) all.insert(all.end(), v.begin(), v.end());
    std::sort(all.begin(), all.end());
    uint64_t batches = 0, recs = 0;
    gofr_proto_frontend_stats(dec, &batches, &recs);
    const double mean_batch = batches ? (double)recs / batches : 1.0;
    auto pct = [&](double p) { return all.empty() ? 0.f : all[(size_t)(p * (all.size() - 1))]; };

    // the floor: batches of the same mean size through the host-batch calls directly, decode → handler → encode
    const uint32_t B = std::max<uint32_t>(1, (uint32_t)(mean_batch + 0.5));
    std::string frames;
    std::vector<uint32_t> foff{0};
    for (uint32_t k = 0; k < B; k++) {
        const std::string m = request_message(name_of(k));
        frames += '\0';
        for (int s = 3; s >= 0; s--) frames += (char)((m.size() >> (8 * s)) & 0xFF);
        frames += m;
        foff.push_back((uint32_t)frames.size());
    }
    uint8_t* out = (uint8_t*)gofr_alloc_pinned(1 << 20);
    uint32_t* out_off = (uint32_t*)gofr_alloc_pinned(4 * (B + 1));
    uint32_t* meta = (uint32_t*)gofr_alloc_pinned(4 * B);
    uint8_t* out2 = (uint8_t*)gofr_alloc_pinned(1 << 20);
    uint32_t* out_off2 = (uint32_t*)gofr_alloc_pinned(4 * (B + 1));
    uint32_t* meta2 = (uint32_t*)gofr_alloc_pinned(4 * B);
    std::vector<float> floor_us;
    const auto f0 = std::chrono::steady_clock::now();
    for (int it = 0; std::chrono::steady_clock::now() - f0 < std::chrono::duration<double>(std::min(secs, 2.0)) || it < 20; it++) {
        auto s = std::chrono::steady_clock::now();
        gofr_proto_batch in{(const uint8_t*)frames.data(), frames.size(), foff.data(), B};
        gofr_resp_batch rb{out, 1 << 20, out_off, meta, 0};
        gofr_ticket t = 0;
        CK(gofr_proto_batch_decode(eng, &kMsg, 1, &kField, 1, 0, nullptr, &in, &rb, &t));
        CK(gofr_batch_wait(eng, t));
        std::string rows;
        std::vector<uint32_t> roff{0};
        for (uint32_t k = 0; k < B; k++) {
            rows += hello_row(out + out_off[k]);
            rows.append((4 - rows.size() % 4) % 4, '\0');
            roff.push_back((uint32_t)rows.size());
        }
        gofr_proto_batch in2{(const uint8_t*)rows.data(), rows.size(), roff.data(), B};
        gofr_resp_batch rb2{out2, 1 << 20, out_off2, meta2, 0};
        CK(gofr_proto_batch_encode(eng, &kMsg, 1, &kField, 1, 0, nullptr, &in2, &rb2, &t));
        CK(gofr_batch_wait(eng, t));
        floor_us.push_back(std::chrono::duration<float, std::micro>(std::chrono::steady_clock::now() - s).count());
    }
    std::sort(floor_us.begin(), floor_us.end());
    const float floor_med = floor_us[floor_us.size() / 2];
    printf("{\"threads\": %d, \"max_batch\": %u, \"max_wait_us\": %u, \"rpcs\": %zu, \"rpc_per_s\": %.0f, \"batches\": %llu, "
           "\"mean_batch\": %.1f, \"lat_us_p50\": %.1f, \"lat_us_p99\": %.1f, \"floor_batch\": %u, \"floor_us_per_batch_p50\": %.1f, "
           "\"floor_rpc_per_s\": %.0f, \"bad\": %llu}\n",
           T, max_batch, wait_us, all.size(), all.size() / el, (unsigned long long)batches, mean_batch, pct(0.5), pct(0.99), B,
           floor_med, B / (floor_med * 1e-6), (unsigned long long)bad.load());
    gofr_proto_frontend_destroy(dec);
    gofr_proto_frontend_destroy(enc);
    gofr_engine_destroy(eng);
    gofr_table_destroy(tab);
    return bad.load() ? 1 : 0;
}
