// emu_serve.cpp — TEST INFRASTRUCTURE ONLY.
//
// Runs the serve kernel's per-request code (gofr_b200/csrc/serve_device.cuh, the very same __host__ __device__
// functions the CUDA kernel calls) on the CPU, one request after another, packing the output the way the kernel does.
// Purpose: this container has no GPU, so kernel *logic* bugs (routing, sizing, the funnel-shift word writer) are caught
// here against the oracle; tile staging, the block scan and the look-back only exist in serve_kernel.cu and are
// covered by the `-m gpu` tests.  Nothing in the product links or loads this file.
#include <cstdint>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../gofr_b200/csrc/serve_device.cuh"
#include "../../gofr_b200/csrc/proto_nested_device.cuh"
#include "../../gofr_b200/csrc/proto_nested_decode_device.cuh"

using namespace gofr;

// 0: a lane flushes only when it needs room itself; 1: at every decision point; 2: pseudo-randomly (what the other lanes
// of a warp impose on it on the GPU)
extern "C" void emu_set_flush_mode(int mode) { emu_any_mode() = mode; }

extern "C" int emu_serve(const uint8_t* image, uint64_t image_len, const uint8_t* desc, const uint8_t* ids,
                         const uint8_t* arena, uint32_t n, const char* date29, uint8_t* out, uint64_t out_cap,
                         uint32_t* out_off, uint32_t* meta, uint32_t start_misalign) {
    (void)image_len;
    // the kernel works on a 16-byte aligned shared-memory copy of the hot part
    ImageHeader H;
    memcpy(&H, image, sizeof H);
    std::vector<uint32_t> hot((H.hot_bytes + 3) / 4 + 4);
    memcpy(hot.data(), image, H.hot_bytes);
    patch_dates((uint8_t*)hot.data(), (const uint8_t*)date29, 0, 1);
    TableView tv;
    tv.bind((const uint8_t*)hot.data(), image);
    uint32_t ring[GOFR_STAGE_WORDS];
    std::vector<uint32_t> bind_scratch((size_t)H.bind_row_words + 8);
    BatchRefs br;
    br.bind_scratch = bind_scratch.data(); br.bind_row_words = H.bind_row_words; br.ids = ids;
    uint64_t pos = start_misalign;  // lets the test exercise every head alignment
    for (uint32_t i = 0; i < n; i++) {
        uint32_t d[4];
        memcpy(d, desc + (size_t)i * 16, 16);
        ReqCtx c;
        uint32_t arena_off = d[0], path_len = d[1] & 0xFFFF, query_len = d[1] >> 16, data_len = d[2];
        // alternate the "staged" flag so both source policies of the Writer are exercised
        c.set(arena, arena_off, path_len, query_len, data_len, d[3] & 0xFF, (d[3] >> 8) & 0xFF, (i & 1) != 0, 0);
        br.ids = ids + (size_t)i * 16;  // index 0 of a one-request view
        size_request(tv, br, c);
        if (c.prog != 0xFFFF && path_is_clean(c.path, c.path_len)) {  // both matchers must always agree
            int a = mux_match(tv, c.method(), c.path, c.path_len), b = mux_match_linear(tv, c.method(), c.path, c.path_len);
            if (a != b) return -2;
        }
        out_off[i] = (uint32_t)pos;
        meta[i] = request_status(tv, c) | (c.route << 16);
        if (pos + c.total_len + 32 > out_cap) return -1;
        // a response may only touch its own bytes: on the GPU its neighbours are written concurrently by other threads
        uint8_t before[32], after[32];
        const uint64_t b0 = pos >= 32 ? pos - 32 : 0;
        memcpy(before, out + b0, (size_t)(pos - b0));
        memcpy(after, out + pos + c.total_len, 32);
        emit_request(tv, br, c, out + pos, ring);
        if (memcmp(before, out + b0, (size_t)(pos - b0)) != 0 || memcmp(after, out + pos + c.total_len, 32) != 0) return -3;
        pos += c.total_len;
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}

// ---- slot layout (gofr_serve_device_slots): same per-request code, emit_request<true> + finish_padded ----
static int g_stage_mode = 0;  // which requests of the slot emulation count as staged: 0 every other one, 1 all, 2 none
extern "C" int emu_float_text(uint64_t bits, uint8_t* out) { return (int)json_float64_text(bits, out); }
extern "C" int emu_float32_text(uint32_t bits, uint8_t* out) { return (int)json_float32_text(bits, out); }
// float32 text of the bit patterns first, first + step, … (count of them) checked against the C library, which rounds
// correctly: the text parses back to the same float32 (strtof), one digit fewer does not (shortest), and the digits are the
// correctly rounded ones of that length (printf on the exact value: closest, ties to even) — unless those do not parse back
// (at a power of two the interval below the value is half as wide as the one above: three float32 values have a shortest
// decimal that is not the nearest one of its length).  Returns the number of bit
// patterns that fail, the first one in *bad.  Exhaustive with first = 0, step = 1, count = 2^31 (sign bit aside).
extern "C" uint64_t emu_float32_check(uint32_t first, uint32_t step, uint64_t count, uint32_t* bad) {
    uint64_t fails = 0;
    uint32_t b = first;
    for (uint64_t k = 0; k < count; k++, b += step) {
        if (((b >> 23) & 0xFFu) == 0xFFu || (b & 0x7FFFFFFFu) == 0) continue;
        float x;
        memcpy(&x, &b, 4);
        uint8_t t[40];
        const uint32_t n = json_float32_text(b, t);
        t[n] = 0;
        bool ok = n > 0 && strtof((const char*)t, nullptr) == x;
        // digits of the text
        char dg[24];
        int nd = 0;
        bool lead = true;
        for (uint32_t i = 0; i < n && t[i] != 'e'; i++) {
            if (t[i] < '0' || t[i] > '9') continue;
            if (lead && t[i] == '0') continue;
            lead = false;
            dg[nd++] = (char)t[i];
        }
        while (nd > 1 && dg[nd - 1] == '0') nd--;  // 'f' format pads integers with zeros
        dg[nd] = 0;
        char ref[48];
        snprintf(ref, sizeof ref, "%.*e", nd - 1, (double)x);  // float -> double is exact
        char rd[24];
        int rn = 0;
        for (const char* p = ref; *p && *p != 'e'; p++) if (*p >= '0' && *p <= '9') rd[rn++] = *p;
        while (rn > 1 && rd[rn - 1] == '0') rn--;
        rd[rn] = 0;
        ok = ok && (strcmp(rd, dg) == 0 || strtof(ref, nullptr) != x);
        if (ok && nd > 1) {
            snprintf(ref, sizeof ref, "%.*e", nd - 2, (double)x);
            ok = strtof(ref, nullptr) != x;
        }
        if (!ok) { if (!fails && bad) *bad = b; fails++; }
    }
    return fails;
}
// bd_parse_float (Bind into float64 members) against the C library's correctly rounded strtod on `count` generated
// literals.  mode 0: random 1..19-digit mantissas with exponents over the whole range; 1: the 17-digit text of random
// doubles (what encoders emit) and its 16 / 18 / 19 / 25-digit variants; 2: integers around 2^53 .. 2^64 incl. the exact
// half-way points between doubles, with small exponents; 3: random doubles' neighbourhood written with 19 digits plus a
// tail of more digits (the truncated-mantissa path).  out[0] decided, out[1] deferred, out[2] mismatches (must be 0),
// out[3] overflow verdicts; *bad_len / bad = the first mismatching literal.
extern "C" void emu_parse_float_check(uint64_t seed, uint64_t count, int mode, uint64_t* out, char* bad, uint32_t bad_cap) {
    uint64_t s = seed * 0x9E3779B97F4A7C15ull + 1;
    auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
    out[0] = out[1] = out[2] = out[3] = 0;
    char lit[512];
    for (uint64_t k = 0; k < count; k++) {
        int n = 0;
        if (mode == 0) {
            const int nd = 1 + (int)(rnd() % 19);
            uint64_t m = rnd();
            uint64_t lim = 1;
            for (int i = 0; i < nd; i++) lim *= 10;
            m %= lim;
            const int e = (int)(rnd() % 700) - 350;
            n = snprintf(lit, sizeof lit, "%s%llue%d", (rnd() & 1) ? "-" : "", (unsigned long long)m, e);
        } else if (mode == 1) {
            uint64_t b = rnd();
            if (((b >> 52) & 0x7FF) == 0x7FF) b &= ~(1ull << 62);
            double d;
            memcpy(&d, &b, 8);
            static const int prec[] = {17, 16, 18, 19, 25, 17, 17, 15};
            n = snprintf(lit, sizeof lit, "%.*e", prec[rnd() % 8] - 1, d);
        } else if (mode == 2) {
            const int sh = (int)(rnd() % 11);                       // doubles in [2^(53+sh), 2^(54+sh)) are 2^(sh+1) apart
            uint64_t base = ((1ull << 53) | (rnd() & ((1ull << 53) - 1))) << sh;
            const uint64_t half = 1ull << sh;                       // base + half: exactly between two doubles
            const int64_t delta[] = {0, 1, -1, 2, -2};
            uint64_t v = base + half + (uint64_t)delta[rnd() % 5] * (rnd() % 3 == 0 ? 0 : 1);
            const int e = (int)(rnd() % 5);
            if (e == 0) n = snprintf(lit, sizeof lit, "%llu", (unsigned long long)v);
            else if (e == 1) n = snprintf(lit, sizeof lit, "%llu.0", (unsigned long long)v);
            else if (e == 2) n = snprintf(lit, sizeof lit, "%llu000e-3", (unsigned long long)v);
            else if (e == 3) n = snprintf(lit, sizeof lit, "%llu.%03llue0", (unsigned long long)(v / 1000), (unsigned long long)(v % 1000));
            else n = snprintf(lit, sizeof lit, "%llue%d", (unsigned long long)v, (int)(rnd() % 40) - 20);
        } else {
            uint64_t b = rnd();
            if (((b >> 52) & 0x7FF) == 0x7FF) b &= ~(1ull << 62);
            double d;
            memcpy(&d, &b, 8);
            n = snprintf(lit, sizeof lit, "%.18e", d);               // 19 digits d.dddddddddddddddddde+XX
            char* e = strchr(lit, 'e');
            char tail[64];
            snprintf(tail, sizeof tail, "%s", e);
            int extra = (int)(rnd() % 12);
            char* p = e;
            for (int i = 0; i < extra; i++) *p++ = (char)('0' + (rnd() % 4 == 0 ? rnd() % 10 : (rnd() & 1 ? 0 : 9)));
            n = (int)(p - lit) + snprintf(p, sizeof lit - (size_t)(p - lit), "%s", tail);
        }
        // JSON number grammar: no '+' after the mantissa sign position, exponent sign allowed
        uint64_t bits = 0;
        const uint32_t pf = bd_parse_float((const uint8_t*)lit, (uint32_t)n, &bits);
        const double want = strtod(lit, nullptr);
        if (pf == PF_DEFER) { out[1]++; continue; }
        bool ok;
        if (pf == PF_OVERFLOW) { out[3]++; ok = want == HUGE_VAL || want == -HUGE_VAL; }
        else { uint64_t wb; memcpy(&wb, &want, 8); ok = wb == bits; }
        out[0]++;
        if (!ok) { if (!out[2] && bad) snprintf(bad, bad_cap, "%s", lit); out[2]++; }
    }
}
extern "C" void emu_float_text_many(const uint64_t* bits, uint32_t n, uint8_t* out, uint32_t* off) {
    uint32_t o = 0;
    for (uint32_t i = 0; i < n; i++) { off[i] = o; o += json_float64_text(bits[i], out + o); }
    off[n] = o;
}
extern "C" void emu_set_stage_mode(int m) { g_stage_mode = m; }
static uint64_t g_fast_taken = 0;  // requests sized by size_fast (and therefore written by emit_fast) since the last reset
extern "C" uint64_t emu_fast_taken(int reset) { const uint64_t v = g_fast_taken; if (reset) g_fast_taken = 0; return v; }
// store policy of the fast path: 0 SoloStores (serve_slots_kernel), 1 PairStores (the wide instance): its lockstep code
// paths — zero-length copies through the flush votes, trace-id windows through copy_windows, an empty tail for a
// template-only program, the last sector stored after the per-lane branches — run here one lane at a time
static int g_pair_stores = 0;
extern "C" void emu_set_pair_stores(int on) { g_pair_stores = on; }
extern "C" int emu_serve_slots(const uint8_t* image, uint64_t image_len, const uint8_t* desc, const uint8_t* ids,
                               const uint8_t* arena, uint32_t n, const char* date29, uint8_t* out, uint32_t slot_bytes,
                               uint32_t* out_len, uint32_t* meta) {
    (void)image_len;
    ImageHeader H;
    memcpy(&H, image, sizeof H);
    std::vector<uint32_t> hot((H.hot_bytes + 3) / 4 + 4);
    memcpy(hot.data(), image, H.hot_bytes);
    patch_dates((uint8_t*)hot.data(), (const uint8_t*)date29, 0, 1);
    TableView tv;
    tv.bind((const uint8_t*)hot.data(), image);
    uint32_t ring[GOFR_STAGE_WORDS];
    std::vector<uint32_t> bind_scratch((size_t)H.bind_row_words + 8);
    BatchRefs br;
    br.bind_scratch = bind_scratch.data(); br.bind_row_words = H.bind_row_words; br.ids = ids;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t d[4];
        memcpy(d, desc + (size_t)i * 16, 16);
        ReqCtx c;
        c.set(arena, d[0], d[1] & 0xFFFF, d[1] >> 16, d[2], d[3] & 0xFF, (d[3] >> 8) & 0xFF,
              g_stage_mode == 1 || (g_stage_mode == 0 && (i & 1) != 0), 0);
        br.ids = ids + (size_t)i * 16;
        route_request(tv, br, c);
        size_routed<true>(tv, br, c);  // as serve_slots_kernel does: the lean size pass where it applies, then emit_fast
        out_len[i] = c.total_len;
        meta[i] = request_status(tv, c) | (c.route << 16);
        if (c.fast()) g_fast_taken++;
        if (c.total_len && c.total_len <= slot_bytes) {
            uint8_t* const dst = out + (size_t)i * slot_bytes;
            if (g_pair_stores && c.fast()) emit_fast(tv, br, c, dst, ring, PairStores{~0u});
            else emit_request<true>(tv, br, c, dst, ring);
        }
    }
    return 0;
}

// ---- Bind as a split-API stage (gofr_bind_device): bind_device.cuh's bind_request + bind_row_out on the CPU ----
extern "C" int emu_bind_rows(const uint8_t* image, uint32_t schema_idx, const uint8_t* desc, const uint8_t* arena, uint32_t n,
                             uint8_t* out, uint32_t slot_bytes, uint32_t* len, uint32_t* status) {
    ImageHeader H;
    memcpy(&H, image, sizeof H);
    std::vector<uint32_t> hot((H.hot_bytes + 3) / 4 + 4);
    memcpy(hot.data(), image, H.hot_bytes);
    TableView tv;
    tv.bind((const uint8_t*)hot.data(), image);
    uint32_t ring[GOFR_STAGE_WORDS];
    std::vector<uint32_t> row(BR_FIELDS + 2 * kMaxFields);
    for (uint32_t i = 0; i < n; i++) {
        uint32_t d[4];
        memcpy(d, desc + (size_t)i * 16, 16);
        const uint32_t data_off = (d[0] + (d[1] & 0xFFFF) + (d[1] >> 16) + 3u) & ~3u;
        const uint8_t* body = arena + data_off;
        bind_request(tv, schema_idx, body, d[2], row.data());
        const uint32_t st = bind_row_status(row.data());
        uint32_t L = 0;
        if (st != 2u) {
            L = bind_row_out<false>(nullptr, tv, schema_idx, body, row.data());
            if (L && L <= slot_bytes) {
                Writer w;
                w.init(out + (size_t)i * slot_bytes, ring);
                bind_row_out<true>(&w, tv, schema_idx, body, row.data());
                w.finish_padded();
            }
        }
        len[i] = L;
        status[i] = st;
    }
    return 0;
}

// ---- routing only (gofr_route_device): serve_device.cuh's route_only on the CPU ----
extern "C" int emu_route(const uint8_t* image, const uint8_t* desc, const uint8_t* arena, uint32_t n, uint32_t* meta,
                         uint32_t* vars) {
    ImageHeader H;
    memcpy(&H, image, sizeof H);
    std::vector<uint32_t> hot((H.hot_bytes + 3) / 4 + 4);
    memcpy(hot.data(), image, H.hot_bytes);
    TableView tv;
    tv.bind((const uint8_t*)hot.data(), image);
    for (uint32_t i = 0; i < n; i++) {
        uint32_t d[4];
        memcpy(d, desc + (size_t)i * 16, 16);
        uint32_t route;
        const uint32_t status = route_only(tv, d[3] & 0xFF, arena + d[0], d[1] & 0xFFFF, &route, vars + (size_t)i * kMaxVars);
        meta[i] = status | route << 16;
    }
    return 0;
}

// ---- HTTP/1.1 request heads (gofr_http_parse_device): http_device.cuh on the CPU ----
#include "../../gofr_b200/csrc/http_device.cuh"

extern "C" int emu_http_parse(const uint8_t* raw, const uint32_t* raw_off, uint32_t n, uint8_t* desc, uint8_t* arena,
                              uint32_t* status, uint64_t* spans) {
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t mo = raw_off[i], mn = raw_off[i + 1] - mo, a = (mo + 3u) & ~3u;
        HttpOut o;
        http_parse(raw + mo, mn, arena + a, &o);
        status[i] = o.status;
        uint32_t d[4] = {0, 0, 0, 0};
        if (o.status == GOFR_HTTP_OK) { d[0] = a; d[1] = o.path_len | o.query_len << 16; d[2] = o.data_len; d[3] = o.method | o.flags << 8; }
        memcpy(desc + (size_t)i * 16, d, 16);
        for (int k = 0; k < GOFR_HTTP_SPANS; k++) spans[(size_t)i * GOFR_HTTP_SPANS + k] = o.status == GOFR_HTTP_OK ? o.spans[k] + mo : 0;
    }
    return 0;
}

// ---- RequestLog line (SURVEY §8f rank 1): the same reqlog_device.cuh code the CUDA kernel runs ----
#include "../../gofr_b200/csrc/reqlog_device.cuh"

extern "C" int emu_reqlog(const uint8_t* desc, const uint8_t* ids, const uint8_t* arena, uint32_t n, uint8_t* out,
                          uint64_t out_cap, uint32_t* out_off, uint32_t start_misalign) {
    uint32_t stage[GOFR_STAGE_WORDS];
    uint64_t pos = start_misalign;
    for (uint32_t i = 0; i < n; i++) {
        LogDesc d;
        memcpy(&d, desc + (size_t)i * sizeof(LogDesc), sizeof d);
        uint32_t id[4];
        memcpy(id, ids + (size_t)i * 16, 16);
        LogCtx c;
        c.ip_off = c.ip_len = c.esc_mask = c.total_len = 0;
        const bool staged = (i & 1) != 0;  // exercise both source policies of the Writer
        reqlog_size(d, arena + d.arena_off, staged, c);
        out_off[i] = (uint32_t)pos;
        if (pos + c.total_len > out_cap) return -1;
        reqlog_emit(d, arena + d.arena_off, staged, id, c, out + pos, stage);
        pos += c.total_len;
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}

// ---- program inspection (scratch/prog_stats.py): the op list of program `prog` of a sealed image ----
extern "C" int emu_prog_ops(const uint8_t* image, uint32_t prog, uint8_t* ops_out, uint32_t cap_ops, uint32_t* hdr_fixed,
                            uint32_t* body_fixed, uint32_t* shape_class) {
    TableView tv;
    tv.bind(image, image);
    if (prog >= tv.hdr()->n_progs) return -1;
    const ProgRec P = tv.progs()[prog];
    if (P.n_ops > cap_ops) return -2;
    memcpy(ops_out, tv.ops() + P.first_op, (size_t)P.n_ops * sizeof(Op));
    *hdr_fixed = P.hdr_fixed;
    *body_fixed = P.body_fixed;
    *shape_class = P.shape_class;
    return (int)P.n_ops;
}

// ---- proto3 encoder (gofr_proto_encode_device): proto_size / proto_emit as the CUDA kernel runs them; the schema is
// built the way engine.cu builds it ----
#include "../../gofr_b200/csrc/grpc_device.cuh"

extern "C" int emu_proto_encode(const uint32_t* fields, uint32_t n_fields, const uint8_t* rows, const uint32_t* row_off, uint32_t n,
                                uint8_t* out, uint64_t out_cap, uint32_t* out_off, uint32_t* meta, uint32_t start_misalign) {
    ProtoSchema S;
    memset(&S, 0, sizeof S);
    S.n_fields = n_fields;
    for (uint32_t k = 0; k < n_fields; k++) {
        const uint32_t t = fields[2 * k + 1];
        S.tag[k] = fields[2 * k] << 3 | proto_wire(t);
        S.cls[k] = (uint8_t)proto_class(t);
        S.fixed_bytes += proto_is64(t) ? 8u : 4u;
    }
    uint32_t stage[GOFR_STAGE_WORDS];
    uint64_t pos = start_misalign;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* r = rows + row_off[i];
        ProtoMsg m = proto_size(S, r, row_off[i + 1] - row_off[i], (row_off[i] & 3u) == 0);
        out_off[i] = (uint32_t)pos;
        meta[i] = m.status;
        if (pos + m.out_len > out_cap) return -1;
        proto_emit(S, r, m, out + pos, stage);
        pos += m.out_len;
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}

// rows -> frames for message types with nested / repeated fields (proto_nested_device.cuh); desc = the PbnDesc the product's
// gofr_proto_nested_describe built
extern "C" int emu_proto_encode_nested(const void* desc, const uint8_t* rows, const uint32_t* row_off, uint32_t n, uint8_t* out,
                                       uint64_t out_cap, uint32_t* out_off, uint32_t* meta, uint32_t start_misalign) {
    PbnDesc D;
    memcpy(&D, desc, sizeof D);
    uint32_t stage[GOFR_STAGE_WORDS];
    uint64_t pos = start_misalign;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* r = rows + row_off[i];
        const uint32_t rn = row_off[i + 1] - row_off[i];
        PbnMsg m = pbn_size(D, r, rn);
        out_off[i] = (uint32_t)pos;
        meta[i] = m.status;
        if (pos + m.out_len > out_cap) return -1;
        pbn_emit(D, r, rn, m, out + pos, stage);
        pos += m.out_len;
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}
// frames -> rows for the same message types (proto_nested_decode_device.cuh)
extern "C" int emu_proto_decode_nested(const void* desc, const uint8_t* in, const uint32_t* in_off, uint32_t n, uint8_t* rows,
                                       uint64_t rows_cap, uint32_t* row_off, uint32_t* meta) {
    PbnDesc D;
    memcpy(&D, desc, sizeof D);
    uint64_t pos = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* f = in + in_off[i];
        const uint32_t fn = in_off[i + 1] - in_off[i];
        PdnRow r = pdn_decode_size(D, f, fn);
        row_off[i] = (uint32_t)pos;
        meta[i] = r.status;
        if (pos + r.out_len > rows_cap) return -1;
        pdn_decode_emit(D, f, fn, r, rows + pos);
        pos += r.out_len;
    }
    row_off[n] = (uint32_t)pos;
    return 0;
}
extern "C" uint32_t emu_pbn_desc_bytes() { return (uint32_t)sizeof(PbnDesc); }

extern "C" int emu_proto_decode(const uint32_t* fields, uint32_t n_fields, const uint8_t* in, const uint32_t* in_off, uint32_t n,
                                uint8_t* rows, uint64_t rows_cap, uint32_t* row_off, uint32_t* meta, uint32_t start_misalign) {
    ProtoSchema S;
    memset(&S, 0, sizeof S);
    S.n_fields = n_fields;
    for (uint32_t k = 0; k < n_fields; k++) {
        const uint32_t t = fields[2 * k + 1];
        S.tag[k] = fields[2 * k] << 3 | proto_wire(t);
        S.cls[k] = (uint8_t)proto_class(t);
        S.fixed_bytes += proto_is64(t) ? 8u : 4u;
    }
    uint32_t stage[GOFR_STAGE_WORDS];
    uint64_t pos = start_misalign;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* f = in + in_off[i];
        ProtoRow r;
        proto_decode_scan(S, f, in_off[i + 1] - in_off[i], r);
        row_off[i] = (uint32_t)pos;
        meta[i] = r.status;
        if (pos + r.out_len > rows_cap) return -1;
        proto_decode_emit(S, f, r, rows + pos, stage);
        pos += r.out_len;
    }
    row_off[n] = (uint32_t)pos;
    return 0;
}

// ---- gRPC Hello (config 5): the same grpc_device.cuh code the CUDA kernel runs ----

extern "C" int emu_grpc_hello(const uint8_t* in, const uint32_t* in_off, uint32_t n, uint8_t* out, uint64_t out_cap,
                              uint32_t* out_off, uint32_t* meta, uint32_t start_misalign) {
    uint32_t stage[GOFR_STAGE_WORDS];
    uint64_t pos = start_misalign;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* f = in + in_off[i];
        HelloReq r = hello_parse(f, in_off[i + 1] - in_off[i]);
        out_off[i] = (uint32_t)pos;
        meta[i] = r.status;
        if (pos + r.out_len > out_cap) return -1;
        hello_emit(f, r, out + pos, stage);
        pos += r.out_len;
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}
