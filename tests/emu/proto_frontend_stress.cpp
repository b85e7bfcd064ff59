// TEST INFRASTRUCTURE ONLY: the gRPC front-end's fan-in / fan-out (gofr_b200/csrc/proto_frontend.cpp) on the CPU, under
// ThreadSanitizer, with stubs in place of the engine's host-batch calls.  The stubs check every batch as the engine does
// (offsets non-decreasing and within the data, multiples of 4 for rows, the 5-byte prefix of a frame, out_cap at least the
// batch's bound) and "serve" record i with bytes and a status derived from ITS bytes alone, of any size from 0 up to the
// record's bound, so every caller can tell whether it got its own answer back.
//   proto_frontend_stress <decode 0|1> <threads> <records_per_thread> <max_batch> <max_wait_us> <max_record_bytes>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include "../../gofr_b200/csrc/proto_frontend.cpp"

static const uint32_t kPerByte[2] = {2, 3}, kPerRecord[2] = {5, 7};  // [encode, decode]
static std::atomic<uint64_t> g_batches{0}, g_largest{0}, g_violations{0};

void set_last_error(const char*, ...) {}

// the stub's answer for one record of the batch call (decode: the whole frame, prefix included; encode: the padded row)
static uint32_t stub_status(bool decode, const uint8_t* r, uint32_t len) {
    const uint32_t skip = decode ? kPrefix : 0;
    const uint32_t c = len > skip ? r[skip] % 5u : 0u;
    if (decode) return c == 1 ? GOFR_GRPC_BAD_PROTO : c == 2 ? GOFR_GRPC_BAD_UTF8 : c == 3 ? GOFR_GRPC_DEFER : GOFR_GRPC_OK;
    return c == 1 ? GOFR_GRPC_BAD_UTF8 : c == 2 ? GOFR_GRPC_BAD_ROW : GOFR_GRPC_OK;
}
static std::string stub_output(bool decode, const uint8_t* r, uint32_t len) {
    if (stub_status(decode, r, len) != GOFR_GRPC_OK) return std::string();
    const uint64_t bound = (uint64_t)kPerByte[decode] * len + kPerRecord[decode];
    uint64_t h = len;
    for (uint32_t j = 0; j < len; j++) h = h * 131 + r[j];
    std::string o;
    if (decode) {
        const uint32_t size = (uint32_t)(h % (bound + 1));
        for (uint32_t j = 0; j < size; j++) o += (char)((len ? r[j % len] : 0) ^ (uint8_t)(j * 7));
    } else {  // a frame: its own prefix, then a body of 0 .. bound - 5 bytes
        const uint32_t size = (uint32_t)(h % (bound - kPrefix + 1));
        o += '\0';
        for (int k = 3; k >= 0; k--) o += (char)((size >> (8 * k)) & 0xFF);
        for (uint32_t j = 0; j < size; j++) o += (char)((len ? r[j % len] : 0) ^ (uint8_t)(j * 7));
    }
    return o;
}

static int stub_batch(bool decode, const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* t) {
    g_batches++;
    uint64_t l = g_largest.load();
    while (in->n > l && !g_largest.compare_exchange_weak(l, in->n)) {}
    uint64_t bound = 0;
    for (uint32_t i = 0; i < in->n; i++) {
        const uint64_t a = in->off[i], b = in->off[i + 1];
        bool bad = b < a || b > in->data_bytes || (!decode && ((a | b) & 3u));
        if (!bad && decode) {  // 00 | len_be32 | message
            const uint8_t* p = in->data + a;
            bad = b - a < kPrefix || p[0] != 0 ||
                  (((uint32_t)p[1] << 24) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 8) | p[4]) != b - a - kPrefix;
        }
        if (bad) { g_violations++; return GOFR_ERR_INVALID; }
        bound += (uint64_t)kPerByte[decode] * (b - a) + kPerRecord[decode];
    }
    if (in->off[0] != 0 || out->out_cap < bound) { g_violations++; return GOFR_ERR_CAPACITY; }
    uint64_t pos = 0;
    for (uint32_t i = 0; i < in->n; i++) {
        const uint8_t* r = in->data + in->off[i];
        const uint32_t len = in->off[i + 1] - in->off[i];
        const std::string o = stub_output(decode, r, len);
        out->out_off[i] = (uint32_t)pos;
        memcpy(out->out + pos, o.data(), o.size());
        out->meta[i] = stub_status(decode, r, len);
        pos += o.size();
    }
    out->out_off[in->n] = (uint32_t)pos;
    out->out_bytes = pos;
    *t = 1;
    return 0;
}

extern "C" {
void* gofr_alloc_pinned(size_t n) { return calloc(1, n ? n : 1); }
void gofr_free_pinned(void* p) { free(p); }
int gofr_proto_nested_bound(const gofr_proto_nmsg* msgs, uint32_t, const gofr_proto_nfield*, uint32_t, uint32_t, const uint8_t*,
                            int decode, uint32_t* per_byte, uint32_t* per_record) {
    if (!msgs) return GOFR_ERR_INVALID;
    *per_byte = kPerByte[decode != 0];
    *per_record = kPerRecord[decode != 0];
    return GOFR_OK;
}
int gofr_proto_batch_decode(gofr_engine*, const gofr_proto_nmsg*, uint32_t, const gofr_proto_nfield*, uint32_t, uint32_t, const uint8_t*,
                            const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* t) {
    return stub_batch(true, in, out, t);
}
int gofr_proto_batch_encode(gofr_engine*, const gofr_proto_nmsg*, uint32_t, const gofr_proto_nfield*, uint32_t, uint32_t, const uint8_t*,
                            const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* t) {
    return stub_batch(false, in, out, t);
}
int gofr_batch_wait(gofr_engine*, gofr_ticket) { return 0; }
}

int main(int argc, char** argv) {
    if (argc < 7) return 2;
    const bool decode = atoi(argv[1]) != 0;
    const int T = atoi(argv[2]), R = atoi(argv[3]);
    const uint32_t max_batch = (uint32_t)atoi(argv[4]), wait_us = (uint32_t)atoi(argv[5]), max_rec = (uint32_t)atoi(argv[6]);
    const gofr_proto_nmsg msg{0, 1};
    const gofr_proto_nfield field{1, GOFR_PB_STRING, 0, 0};
    gofr_proto_frontend* fe = nullptr;
    if (gofr_proto_frontend_create(&fe, (gofr_engine*)0x1, &msg, 1, &field, 1, 0, nullptr, decode, max_batch, wait_us, max_rec)) return 2;
    std::atomic<uint64_t> bad{0}, short_calls{0}, empty{0}, at_max{0};
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t] {
            std::vector<uint8_t> rec, out;
            for (int r = 0; r < R; r++) {
                // lengths: empty, at max_record_bytes, and in between; contents from (t, r), so every record is its own
                const uint32_t len = r % 11 == 0 ? 0 : r % 11 == 1 ? max_rec : (uint32_t)((t * 977u + r * 131u) % (max_rec + 1));
                rec.resize(len);
                for (uint32_t j = 0; j < len; j++) rec[j] = (uint8_t)(t * 31 + r * 7 + j * 13);
                // what the stubs make of it: the frame or the padded row the front-end stages
                std::string staged;
                if (decode) {
                    staged += '\0';
                    for (int k = 3; k >= 0; k--) staged += (char)((len >> (8 * k)) & 0xFF);
                }
                staged.append(rec.begin(), rec.end());
                if (!decode) staged.append((4 - len % 4) % 4, '\0');
                std::string want = stub_output(decode, (const uint8_t*)staged.data(), (uint32_t)staged.size());
                if (!decode && !want.empty()) want.erase(0, kPrefix);
                const uint32_t want_status = stub_status(decode, (const uint8_t*)staged.data(), (uint32_t)staged.size());
                // every fifth caller with a buffer one byte short of its result
                const bool one_short = r % 5 == 2 && !want.empty();
                const uint32_t cap = one_short ? (uint32_t)want.size() - 1 : (uint32_t)want.size() + (r % 3) * 17;
                out.assign(cap + 1, 0xEE);
                uint32_t n = 0xFFFFFFFFu, status = 0xFFFFFFFFu;
                const int rc = gofr_proto_frontend_call(fe, rec.data(), len, out.data(), cap, &n, &status);
                bool ok = n == want.size() && status == want_status;
                if (one_short) {
                    ok = ok && rc == GOFR_ERR_CAPACITY && out[0] == 0xEE;
                    short_calls++;
                } else {
                    ok = ok && rc == GOFR_OK && memcmp(out.data(), want.data(), want.size()) == 0 && out[cap] == 0xEE;
                }
                if (len == 0) empty++;
                if (len == max_rec) at_max++;
                if (!ok) bad++;
            }
        });
    for (auto& x : th) x.join();
    uint64_t batches = 0, recs = 0;
    gofr_proto_frontend_stats(fe, &batches, &recs);
    // a record over max_record_bytes is refused before it is queued; the front-end keeps serving afterwards
    {
        std::vector<uint8_t> big(max_rec + 1, 1), out(64);
        uint32_t n = 0, status = 0;
        if (gofr_proto_frontend_call(fe, big.data(), max_rec + 1, out.data(), (uint32_t)out.size(), &n, &status) != GOFR_ERR_CAPACITY) bad++;
        uint64_t b2 = 0, r2 = 0;
        gofr_proto_frontend_stats(fe, &b2, &r2);
        if (r2 != recs) bad++;
        if (gofr_proto_frontend_call(fe, nullptr, 0, out.data(), (uint32_t)out.size(), &n, &status) != GOFR_OK) bad++;
        if (gofr_proto_frontend_call(fe, nullptr, 0, nullptr, 0, nullptr, &status) != GOFR_ERR_INVALID) bad++;
    }
    gofr_proto_frontend_destroy(fe);
    printf("{\"records\": %llu, \"batches\": %llu, \"stub_batches\": %llu, \"largest\": %llu, \"short\": %llu, \"empty\": %llu, "
           "\"at_max\": %llu, \"violations\": %llu, \"bad\": %llu}\n",
           (unsigned long long)recs, (unsigned long long)batches, (unsigned long long)g_batches.load(), (unsigned long long)g_largest.load(),
           (unsigned long long)short_calls.load(), (unsigned long long)empty.load(), (unsigned long long)at_max.load(),
           (unsigned long long)g_violations.load(), (unsigned long long)bad.load());
    return bad.load() || g_violations.load() || recs != (uint64_t)T * R ? 1 : 0;
}
