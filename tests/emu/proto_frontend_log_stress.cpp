// TEST INFRASTRUCTURE ONLY: the gRPC encode front-end's log staging (gofr_b200/csrc/proto_frontend.cpp,
// gofr_proto_frontend_create_log) on the CPU, under ThreadSanitizer, with stubs in place of the engine's batch calls.  The
// stubs check every batch as the engine does and "encode" row i as its own bytes behind a 5-byte prefix (an empty row: no
// frame, GOFR_GRPC_BAD_ROW); a record of kind GOFR_LOG_RPC gets the line log_unix_ns | trace id | elapsed_ns | method, so
// every caller can tell whether it got its own message and line back.  Callers mix plain calls, logged calls, logged
// calls whose handler failed (an empty row) and logged calls that ask for no line.
//   proto_frontend_log_stress <threads> <calls_per_thread> <max_batch> <max_wait_us>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include "../../gofr_b200/csrc/proto_frontend.cpp"

static constexpr uint32_t kMaxRow = 64, kMaxMethod = 48;
static constexpr int64_t kLogNs = 1700000000123456789ll;
static std::atomic<uint64_t> g_plain{0}, g_logged{0}, g_violations{0};

void set_last_error(const char*, ...) {}

static std::string stub_frame(const uint8_t* r, uint32_t len) {
    if (!len) return std::string();
    std::string o(1, '\0');
    for (int k = 3; k >= 0; k--) o += (char)((len >> (8 * k)) & 0xFF);
    return o + std::string(reinterpret_cast<const char*>(r), len);
}
static std::string stub_line(int64_t log_ns, const uint8_t* id, int64_t elapsed, const uint8_t* method, uint32_t len) {
    std::string o(reinterpret_cast<const char*>(&log_ns), 8);
    o.append(reinterpret_cast<const char*>(id), 16);
    o.append(reinterpret_cast<const char*>(&elapsed), 8);
    return o.append(reinterpret_cast<const char*>(method), len);
}

static int stub_encode(const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* t) {
    uint64_t pos = 0;
    for (uint32_t i = 0; i < in->n; i++) {
        const uint64_t a = in->off[i], b = in->off[i + 1];
        if (b < a || b > in->data_bytes || ((a | b) & 3u)) { g_violations++; return GOFR_ERR_INVALID; }
        const std::string f = stub_frame(in->data + a, (uint32_t)(b - a));
        if (pos + f.size() > out->out_cap) { g_violations++; return GOFR_ERR_CAPACITY; }
        out->out_off[i] = (uint32_t)pos;
        memcpy(out->out + pos, f.data(), f.size());
        out->meta[i] = f.empty() ? GOFR_GRPC_BAD_ROW : GOFR_GRPC_OK;
        pos += f.size();
    }
    out->out_off[in->n] = (uint32_t)pos;
    out->out_bytes = pos;
    *t = 1;
    return 0;
}

extern "C" {
void* gofr_alloc_pinned(size_t n) { return calloc(1, n ? n : 1); }
void gofr_free_pinned(void* p) { free(p); }
int gofr_proto_nested_bound(const gofr_proto_nmsg* msgs, uint32_t, const gofr_proto_nfield*, uint32_t, uint32_t, const uint8_t*, int,
                            uint32_t* per_byte, uint32_t* per_record) {
    if (!msgs) return GOFR_ERR_INVALID;
    *per_byte = 1;
    *per_record = 5;
    return GOFR_OK;
}
int gofr_proto_batch_decode(gofr_engine*, const gofr_proto_nmsg*, uint32_t, const gofr_proto_nfield*, uint32_t, uint32_t, const uint8_t*,
                            const gofr_proto_batch*, gofr_resp_batch*, gofr_ticket*) {
    g_violations++;  // an encode front-end never decodes
    return GOFR_ERR_INVALID;
}
int gofr_proto_batch_encode(gofr_engine*, const gofr_proto_nmsg*, uint32_t, const gofr_proto_nfield*, uint32_t, uint32_t, const uint8_t*,
                            const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* t) {
    g_plain++;
    return stub_encode(in, out, t);
}
int gofr_proto_batch_encode_log(gofr_engine*, const gofr_proto_nmsg*, uint32_t, const gofr_proto_nfield*, uint32_t, uint32_t,
                                const uint8_t*, const gofr_proto_batch* in, const uint8_t* trace_ids, gofr_resp_batch* out,
                                gofr_batch_log* log, gofr_ticket* t) {
    g_logged++;
    if (log->log_unix_ns != kLogNs) g_violations++;
    int rc = stub_encode(in, out, t);
    if (rc) return rc;
    uint32_t pos = 0, lines = 0;
    for (uint32_t i = 0; i < in->n; i++) {
        const gofr_log_desc& d = log->desc[i];
        log->log_off[i] = pos;
        if (d.kind != GOFR_LOG_RPC && d.kind != GOFR_LOG_NONE) { g_violations++; return GOFR_ERR_INVALID; }
        if (d.kind != GOFR_LOG_RPC) continue;
        if (d.arena_off + d.method_len > log->arena_bytes) { g_violations++; return GOFR_ERR_INVALID; }
        const std::string l = stub_line(log->log_unix_ns, trace_ids + (size_t)i * 16, d.elapsed_ns, log->arena + d.arena_off, d.method_len);
        if (pos + l.size() > log->out_cap) { g_violations++; return GOFR_ERR_CAPACITY; }
        memcpy(log->out + pos, l.data(), l.size());
        pos += (uint32_t)l.size();
        lines++;
    }
    log->log_off[in->n] = pos;
    log->lines = lines;
    log->out_bytes = pos;
    return 0;
}
int gofr_batch_wait(gofr_engine*, gofr_ticket) { return 0; }
}

int main(int argc, char** argv) {
    if (argc < 5) return 2;
    const int T = atoi(argv[1]), R = atoi(argv[2]);
    const uint32_t max_batch = (uint32_t)atoi(argv[3]), wait_us = (uint32_t)atoi(argv[4]);
    const gofr_proto_nmsg msg{0, 1};
    const gofr_proto_nfield field{1, GOFR_PB_STRING, 0, 0};
    gofr_proto_frontend* fe = nullptr;
    if (gofr_proto_frontend_create_log(&fe, (gofr_engine*)0x1, &msg, 1, &field, 1, 0, nullptr, 0, max_batch, wait_us, kMaxRow, kMaxMethod))
        return 2;
    gofr_proto_frontend_set_log_clock(fe, kLogNs);
    std::atomic<uint64_t> bad{0}, lines{0}, failed{0}, short_lines{0};
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            std::vector<uint8_t> row, out(kMaxRow + 8), line(512);
            for (int r = 0; r < R; r++) {
                // 0: plain call; 1: logged; 2: logged, the handler failed (empty row); 3: logged, no line asked
                const int mode = (t + r) % 4;
                const uint32_t len = mode == 2 ? 0 : 4u * (1u + (uint32_t)(t * 7 + r) % (kMaxRow / 4));
                row.resize(len);
                for (uint32_t j = 0; j < len; j++) row[j] = (uint8_t)(t * 31 + r * 7 + j * 13);
                uint8_t id[16];
                for (int k = 0; k < 16; k++) id[k] = (uint8_t)(t * 17 + r * 3 + k);
                std::string method = "/svc" + std::to_string(t) + "/M" + std::to_string(r);
                method.resize(std::min<size_t>(method.size(), kMaxMethod));
                gofr_log_desc d;
                memset(&d, 0, sizeof d);
                d.start_unix_ns = 1000 + r; d.elapsed_ns = t * 1000003ll + r; d.method_len = (uint16_t)method.size();
                d.kind = mode == 3 ? (uint32_t)GOFR_LOG_NONE : (uint32_t)GOFR_LOG_RPC;
                d.arena_off = 12345;  // ignored: the front-end places the method
                uint32_t n = 0xFFFFFFFFu, status = 0xFFFFFFFFu, ln = 0xFFFFFFFFu;
                const std::string want = stub_frame(row.data(), len);
                const std::string want_msg = want.empty() ? want : want.substr(kPrefix);
                int rc;
                std::string want_line;
                // every seventh logged caller passes a line buffer one byte short
                const bool one_short = mode == 1 && r % 7 == 3;
                if (mode == 0) {
                    rc = gofr_proto_frontend_call(fe, row.data(), len, out.data(), (uint32_t)out.size(), &n, &status);
                } else {
                    if (mode != 3) want_line = stub_line(kLogNs, id, d.elapsed_ns, (const uint8_t*)method.data(), d.method_len);
                    const uint32_t cap = one_short ? (uint32_t)want_line.size() - 1 : (uint32_t)line.size();
                    rc = gofr_proto_frontend_call_log(fe, row.data(), len, id, &d, (const uint8_t*)method.data(), out.data(),
                                                      (uint32_t)out.size(), &n, &status, line.data(), cap, &ln);
                }
                bool ok = n == want_msg.size() && memcmp(out.data(), want_msg.data(), want_msg.size()) == 0 &&
                          status == (want.empty() ? GOFR_GRPC_BAD_ROW : GOFR_GRPC_OK);
                if (mode != 0) ok = ok && ln == want_line.size();
                if (one_short) {
                    ok = ok && rc == GOFR_ERR_CAPACITY;
                    short_lines++;
                } else {
                    ok = ok && rc == GOFR_OK && (mode == 0 || memcmp(line.data(), want_line.data(), want_line.size()) == 0);
                }
                if (mode == 1 || mode == 2) lines++;
                if (mode == 2) failed++;
                if (!ok) bad++;
            }
        });
    for (auto& x : th) x.join();
    uint64_t batches = 0, recs = 0;
    gofr_proto_frontend_stats(fe, &batches, &recs);
    {
        // a method over max_log_bytes is refused before it is queued; a bad kind and a missing trace id are invalid
        std::string big(kMaxMethod + 1, 'm');
        uint8_t out[64], line[64], id[16] = {0};
        uint32_t n = 0, status = 0, ln = 0;
        gofr_log_desc d;
        memset(&d, 0, sizeof d);
        d.kind = GOFR_LOG_RPC; d.method_len = (uint16_t)big.size();
        if (gofr_proto_frontend_call_log(fe, nullptr, 0, id, &d, (const uint8_t*)big.data(), out, 64, &n, &status, line, 64, &ln) !=
            GOFR_ERR_CAPACITY) bad++;
        d.method_len = 1;
        d.kind = GOFR_LOG_REQUEST;
        if (gofr_proto_frontend_call_log(fe, nullptr, 0, id, &d, (const uint8_t*)"m", out, 64, &n, &status, line, 64, &ln) != GOFR_ERR_INVALID) bad++;
        d.kind = GOFR_LOG_RPC;
        if (gofr_proto_frontend_call_log(fe, nullptr, 0, nullptr, &d, (const uint8_t*)"m", out, 64, &n, &status, line, 64, &ln) != GOFR_ERR_INVALID) bad++;
        if (gofr_proto_frontend_call_log(fe, nullptr, 0, id, nullptr, nullptr, out, 64, &n, &status, line, 64, &ln) != GOFR_ERR_INVALID) bad++;
        uint64_t b2 = 0, r2 = 0;
        gofr_proto_frontend_stats(fe, &b2, &r2);
        if (r2 != recs) bad++;
    }
    gofr_proto_frontend_destroy(fe);
    // a decode front-end takes no log staging
    gofr_proto_frontend* dec = nullptr;
    if (gofr_proto_frontend_create_log(&dec, (gofr_engine*)0x1, &msg, 1, &field, 1, 0, nullptr, 1, max_batch, wait_us, kMaxRow, kMaxMethod) !=
        GOFR_ERR_INVALID) bad++;
    printf("{\"calls\": %llu, \"batches\": %llu, \"plain_batches\": %llu, \"log_batches\": %llu, \"lines\": %llu, \"failed\": %llu, "
           "\"short\": %llu, \"violations\": %llu, \"bad\": %llu}\n",
           (unsigned long long)recs, (unsigned long long)batches, (unsigned long long)g_plain.load(), (unsigned long long)g_logged.load(),
           (unsigned long long)lines.load(), (unsigned long long)failed.load(), (unsigned long long)short_lines.load(),
           (unsigned long long)g_violations.load(), (unsigned long long)bad.load());
    return bad.load() || g_violations.load() || recs != (uint64_t)T * R ? 1 : 0;
}
