// proto_frontend.cpp — per-message front-end of the nested proto3 codec: grpc-go calls its codec once per message
// (encoding.Codec.Unmarshal for the request, Marshal for the response, on the RPC's own goroutine; the reference's unary
// handler dec(in) runs between them, examples/grpc-server/grpc/hello_grpc.pb.go:73-89), the GPU codec wants batches.
// Callers hand in one message (decode) or one row (encode) each and block on frontend_ring.h's ring; its dispatcher runs
// each closed batch through gofr_proto_batch_decode / _encode and every caller copies its own record out.
//
// Written against the public ABI only (the batch calls, gofr_batch_wait, gofr_proto_nested_bound, the pinned allocator),
// as frontend.cpp is, so that tests/emu/proto_frontend_stress.cpp runs it against stub batch calls under ThreadSanitizer.
//
// The ring's claim word reserves slot i and arena range [a, a + need), so records lie back to back in slot order — exactly
// the batch call's off[] contract:
//   decode  the caller stores off[i] = a and the frame 00 | len_be32(m) | m, which the batch call requires;
//   encode  the caller stores off[i] = a and the row zero padded to a multiple of 4, so every offset stays one;
//   close   the dispatcher stores off[n] = the claimed arena bytes, sums the records' bounds (gofr_proto_nested_bound:
//           per_byte * bytes + per_record) and grows the batch's pinned output to that sum when it is larger, so the batch
//           call never runs out of room.  The output never shrinks: the worst case can be hundreds of MiB, so it is not
//           allocated up front.
//
// An encode front-end made by gofr_proto_frontend_create_log also stages a log record, a trace id and the method per call
// (seat i's method at i * max_log_bytes) and takes the batch's RPCLog lines back: a batch in which some caller logs runs
// through gofr_proto_batch_encode_log, the other callers' records saying GOFR_LOG_NONE.
#include <cstring>
#include <vector>
#include <time.h>

#include "../../include/gofr_b200.h"
#include "engine_internal.h"
#include "frontend_ring.h"

// A weak reference: this file also links into harnesses whose stub engine has only the calls of a front-end without log
// staging (tests/emu/proto_frontend_stress.cpp); the library defines it.
#pragma weak gofr_proto_batch_encode_log

static constexpr uint32_t kPrefix = 5;  // grpc-go's length-prefixed-message header: compressed flag, big-endian length

struct gofr_proto_frontend_batch {
    uint8_t* arena = nullptr;    // records back to back
    uint32_t* off = nullptr;     // max_batch + 1
    uint8_t* out = nullptr;      // grown by the dispatcher, never shrunk
    uint64_t out_cap = 0;
    uint32_t* out_off = nullptr; // max_batch + 1
    uint32_t* meta = nullptr;    // max_batch
    // log staging (gofr_proto_frontend_create_log)
    uint8_t* ids = nullptr;      // max_batch * 16
    gofr_log_desc* log_desc = nullptr;
    uint8_t* log_arena = nullptr;
    uint8_t* log_out = nullptr;
    uint32_t* log_off = nullptr;
    std::atomic<bool> logs{false};  // some caller of the filling batch asked for its line
};
using Staging = gofr_proto_frontend_batch;

struct gofr_proto_frontend {
    gofr_proto_frontend(uint32_t max_batch, uint32_t max_wait_us) : ring(max_batch, max_wait_us) {}
    gofr_engine* eng = nullptr;
    std::vector<gofr_proto_nmsg> msgs;
    std::vector<gofr_proto_nfield> fields;
    std::vector<uint8_t> presence;  // empty: none
    uint32_t root = 0, max_record_bytes = 0, per_byte = 0, per_record = 0;
    bool decode = false;
    bool log = false;
    uint32_t max_log_bytes = 0;           // log staging per call
    uint64_t log_cap = 0;                 // line bytes of a batch
    std::atomic<int64_t> log_clock{0};    // tests: the log time of every line (ns); 0 = wall clock
    Staging b[gofr_ring::kBatches];
    gofr_ring::Ring ring;
};
using ProtoFrontend = gofr_proto_frontend;

static void free_staging(Staging& x) {
    gofr_free_pinned(x.arena); gofr_free_pinned(x.off); gofr_free_pinned(x.out);
    gofr_free_pinned(x.out_off); gofr_free_pinned(x.meta);
    gofr_free_pinned(x.ids); gofr_free_pinned(x.log_desc); gofr_free_pinned(x.log_arena); gofr_free_pinned(x.log_out);
    gofr_free_pinned(x.log_off);
}

// the dispatcher's step: batch k's n records (arena_bytes in all) through the host-batch call of the front-end's direction
static int serve_batch(ProtoFrontend* f, int k, uint32_t n, uint32_t arena_bytes) {
    Staging& x = f->b[k];
    x.off[n] = arena_bytes;
    uint64_t need = 0;
    for (uint32_t i = 0; i < n; i++) need += (uint64_t)f->per_byte * (x.off[i + 1] - x.off[i]) + f->per_record;
    if (need > x.out_cap) {
        gofr_free_pinned(x.out);
        const uint64_t cap = (need + 0xFFFFu) & ~(uint64_t)0xFFFFu;
        x.out = (uint8_t*)gofr_alloc_pinned((size_t)cap);
        x.out_cap = x.out ? cap : 0;
        if (!x.out) {
            set_last_error("gofr_proto_frontend: no pinned output buffer of %llu bytes", (unsigned long long)cap);
            return GOFR_ERR_NOMEM;
        }
    }
    gofr_proto_batch in;
    memset(&in, 0, sizeof in);
    in.data = x.arena; in.data_bytes = arena_bytes; in.off = x.off; in.n = n;
    gofr_resp_batch out;
    memset(&out, 0, sizeof out);
    out.out = x.out; out.out_cap = x.out_cap; out.out_off = x.out_off; out.meta = x.meta;
    const uint8_t* pr = f->presence.empty() ? nullptr : f->presence.data();
    const uint32_t n_msgs = (uint32_t)f->msgs.size(), n_fields = (uint32_t)f->fields.size();
    gofr_ticket t = 0;
    int rc;
    if (x.logs.exchange(false, std::memory_order_acquire)) {  // the batch is closed: no caller sets it until it reopens
        gofr_batch_log log;
        memset(&log, 0, sizeof log);
        log.desc = x.log_desc; log.arena = x.log_arena; log.arena_bytes = (uint64_t)n * f->max_log_bytes;
        int64_t ns = f->log_clock.load(std::memory_order_relaxed);
        if (!ns) { struct timespec ts; clock_gettime(CLOCK_REALTIME, &ts); ns = (int64_t)ts.tv_sec * 1000000000ll + ts.tv_nsec; }
        log.log_unix_ns = ns;
        log.out = x.log_out; log.out_cap = f->log_cap; log.log_off = x.log_off;
        rc = gofr_proto_batch_encode_log(f->eng, f->msgs.data(), n_msgs, f->fields.data(), n_fields, f->root, pr, &in, x.ids, &out,
                                         &log, &t);
    } else {
        auto call = f->decode ? gofr_proto_batch_decode : gofr_proto_batch_encode;
        rc = call(f->eng, f->msgs.data(), n_msgs, f->fields.data(), n_fields, f->root, pr, &in, &out, &t);
    }
    if (rc == GOFR_OK) rc = gofr_batch_wait(f->eng, t);
    return rc;
}

static int proto_frontend_create(gofr_proto_frontend** out, gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs,
                                 const gofr_proto_nfield* fields, uint32_t n_fields, uint32_t root, const uint8_t* presence,
                                 int decode, uint32_t max_batch, uint32_t max_wait_us, uint32_t max_record_bytes, bool log,
                                 uint32_t max_log_bytes) {
    if (!out || !e || max_batch == 0 || max_batch > 0x7FFFFFFFu || (log && decode)) return GOFR_ERR_INVALID;
    uint32_t per_byte = 0, per_record = 0;  // validates the description as the batch calls do
    { int rc = gofr_proto_nested_bound(msgs, n_msgs, fields, n_fields, root, presence, decode, &per_byte, &per_record); if (rc) return rc; }
    // every record's arena bytes (a frame, or a row padded to 4) fit this; the arena's total stays a 32-bit claim
    const uint64_t per = ((uint64_t)max_record_bytes + kPrefix + 3u) & ~(uint64_t)3u;
    const uint64_t arena = (uint64_t)max_batch * per;
    // the batch call's output offsets are 32-bit: a full batch of the largest records must fit them
    const uint64_t bound = (uint64_t)max_batch * ((uint64_t)per_byte * ((uint64_t)max_record_bytes + kPrefix) + per_record);
    if (arena > 0xFFFFFFF0ull || bound > 0xFFFFFFFFull) {
        set_last_error("gofr_proto_frontend_create: %u records of %u bytes exceed the batch call's 32-bit offsets", max_batch,
                       max_record_bytes);
        return GOFR_ERR_CAPACITY;
    }
    // a batch's lines: gofr_batch_log_bound's rule for max_batch RPCLog records of max_log_bytes method bytes
    const uint64_t log_cap = log ? (uint64_t)max_batch * (320u + 7ull * max_log_bytes) : 0;
    if (log_cap > 0xFFFFFFF0ull || (uint64_t)max_batch * max_log_bytes > 0xFFFFFFF0ull) {
        set_last_error("gofr_proto_frontend_create_log: %u calls of %u method bytes exceed the lines' 32-bit offsets", max_batch,
                       max_log_bytes);
        return GOFR_ERR_CAPACITY;
    }
    ProtoFrontend* f = new ProtoFrontend(max_batch, max_wait_us);
    f->eng = e;
    f->msgs.assign(msgs, msgs + n_msgs);
    f->fields.assign(fields, fields + n_fields);
    if (presence) f->presence.assign(presence, presence + n_fields);
    f->root = root;
    f->decode = decode != 0;
    f->max_record_bytes = max_record_bytes;
    f->per_byte = per_byte;
    f->per_record = per_record;
    f->log = log;
    f->max_log_bytes = max_log_bytes;
    f->log_cap = log_cap;
    for (auto& x : f->b) {
        x.arena = (uint8_t*)gofr_alloc_pinned((size_t)arena + 16);
        x.off = (uint32_t*)gofr_alloc_pinned(((size_t)max_batch + 1) * 4);
        x.out_off = (uint32_t*)gofr_alloc_pinned(((size_t)max_batch + 1) * 4);
        x.meta = (uint32_t*)gofr_alloc_pinned((size_t)max_batch * 4);
        bool log_ok = true;
        if (log) {
            x.ids = (uint8_t*)gofr_alloc_pinned((size_t)max_batch * 16);
            x.log_desc = (gofr_log_desc*)gofr_alloc_pinned((size_t)max_batch * sizeof(gofr_log_desc));
            x.log_arena = (uint8_t*)gofr_alloc_pinned((size_t)max_batch * max_log_bytes + 64);
            x.log_out = (uint8_t*)gofr_alloc_pinned((size_t)log_cap + 64);
            x.log_off = (uint32_t*)gofr_alloc_pinned(((size_t)max_batch + 1) * 4);
            log_ok = x.ids && x.log_desc && x.log_arena && x.log_out && x.log_off;
        }
        if (!x.arena || !x.off || !x.out_off || !x.meta || !log_ok) {
            for (auto& y : f->b) free_staging(y);
            delete f;
            return GOFR_ERR_NOMEM;
        }
    }
    f->ring.start([f](int k, uint32_t n, uint32_t arena_bytes) { return serve_batch(f, k, n, arena_bytes); });
    *out = f;
    return GOFR_OK;
}

extern "C" {

int gofr_proto_frontend_create(gofr_proto_frontend** out, gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs,
                               const gofr_proto_nfield* fields, uint32_t n_fields, uint32_t root, const uint8_t* presence,
                               int decode, uint32_t max_batch, uint32_t max_wait_us, uint32_t max_record_bytes) {
    return proto_frontend_create(out, e, msgs, n_msgs, fields, n_fields, root, presence, decode, max_batch, max_wait_us,
                                 max_record_bytes, false, 0);
}

int gofr_proto_frontend_create_log(gofr_proto_frontend** out, gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs,
                                   const gofr_proto_nfield* fields, uint32_t n_fields, uint32_t root, const uint8_t* presence,
                                   int decode, uint32_t max_batch, uint32_t max_wait_us, uint32_t max_record_bytes,
                                   uint32_t max_log_bytes) {
    return proto_frontend_create(out, e, msgs, n_msgs, fields, n_fields, root, presence, decode, max_batch, max_wait_us,
                                 max_record_bytes, true, max_log_bytes);
}

void gofr_proto_frontend_destroy(gofr_proto_frontend* f) {
    if (!f) return;
    f->ring.stop();
    for (auto& x : f->b) free_staging(x);
    delete f;
}

int gofr_proto_frontend_stats(gofr_proto_frontend* f, uint64_t* batches, uint64_t* records) {
    if (!f) return GOFR_ERR_INVALID;
    if (batches) *batches = f->ring.batches.load(std::memory_order_relaxed);
    if (records) *records = f->ring.records.load(std::memory_order_relaxed);
    return GOFR_OK;
}

int gofr_proto_frontend_set_log_clock(gofr_proto_frontend* f, int64_t unix_ns) {
    if (!f) return GOFR_ERR_INVALID;
    f->log_clock.store(unix_ns, std::memory_order_relaxed);
    return GOFR_OK;
}

}  // extern "C"

// One caller's record, with its log record (log == NULL: a plain gofr_proto_frontend_call, GOFR_LOG_NONE on a log
// front-end).
static int proto_frontend_call(gofr_proto_frontend* f, const uint8_t* in, uint32_t in_len, const uint8_t* trace_id,
                               const gofr_log_desc* log, const uint8_t* method, uint8_t* out, uint32_t out_cap, uint32_t* out_len,
                               uint32_t* status, uint8_t* line, uint32_t line_cap, uint32_t* line_len) {
    if (!f || !out_len || !status || (in_len && !in) || (out_cap && !out)) return GOFR_ERR_INVALID;
    if (log) {
        if (!f->log || !trace_id || !line_len || (log->method_len && !method) || (line_cap && !line) ||
            (log->kind != GOFR_LOG_RPC && log->kind != GOFR_LOG_NONE)) {
            set_last_error(!f->log ? "the front-end was made without log staging (gofr_proto_frontend_create_log)" : "bad log record");
            return GOFR_ERR_INVALID;
        }
        if (log->method_len > f->max_log_bytes) {
            set_last_error("a method of %u bytes exceeds the front-end's max_log_bytes", (uint32_t)log->method_len);
            return GOFR_ERR_CAPACITY;
        }
        *line_len = 0;
    }
    if (in_len > f->max_record_bytes) {
        set_last_error("record of %u bytes exceeds the front-end's max_record_bytes", in_len);
        return GOFR_ERR_CAPACITY;
    }
    const uint32_t need = f->decode ? in_len + kPrefix : (in_len + 3u) & ~3u;
    gofr_ring::Seat s;
    if (!f->ring.claim(need, &s)) return GOFR_ERR_INVALID;
    Staging& x = f->b[s.k];
    uint8_t* p = x.arena + s.a;
    if (f->decode) {  // the frame the batch call takes: not compressed, big-endian length, the message
        p[0] = 0;
        p[1] = (uint8_t)(in_len >> 24); p[2] = (uint8_t)(in_len >> 16); p[3] = (uint8_t)(in_len >> 8); p[4] = (uint8_t)in_len;
        if (in_len) memcpy(p + kPrefix, in, in_len);
    } else {          // the row, zero padded to a multiple of 4
        if (in_len) memcpy(p, in, in_len);
        memset(p + in_len, 0, need - in_len);
    }
    x.off[s.i] = s.a;
    if (f->log) {
        gofr_log_desc r;
        memset(&r, 0, sizeof r);
        if (log) {
            r.start_unix_ns = log->start_unix_ns; r.elapsed_ns = log->elapsed_ns; r.tz_offset_s = log->tz_offset_s;
            r.method_len = log->method_len; r.kind = log->kind;
            if (r.method_len) memcpy(x.log_arena + (size_t)s.i * f->max_log_bytes, method, r.method_len);
        } else {
            r.kind = GOFR_LOG_NONE;
        }
        r.arena_off = s.i * f->max_log_bytes;
        x.log_desc[s.i] = r;
        if (log) memcpy(x.ids + (size_t)s.i * 16, trace_id, 16);
        else memset(x.ids + (size_t)s.i * 16, 0, 16);
        if (log) x.logs.store(true, std::memory_order_relaxed);
    }
    f->ring.filled(s);

    const uint32_t n = f->ring.wait(s);
    int rc = f->ring.b[s.k].rc;
    *out_len = 0;
    if (rc == GOFR_OK) {
        *status = x.meta[s.i];
        const uint32_t lo = x.out_off[s.i], hi = x.out_off[s.i + 1];
        // an encoded frame without its prefix: what Marshal returns (grpc-go writes the prefix itself); a failed record is empty
        const uint32_t skip = f->decode ? 0 : kPrefix;
        const uint32_t len = hi - lo > skip ? hi - lo - skip : 0;
        *out_len = len;
        if (len > out_cap) rc = GOFR_ERR_CAPACITY;
        else if (len) memcpy(out, x.out + lo + skip, len);
    }
    int line_rc = GOFR_OK;
    if (log && f->ring.b[s.k].rc == GOFR_OK) {
        const uint32_t l0 = x.log_off[s.i], ll = x.log_off[s.i + 1] - l0;
        *line_len = ll;
        if (ll > line_cap) line_rc = GOFR_ERR_CAPACITY;
        else if (ll) memcpy(line, x.log_out + l0, ll);
    }
    f->ring.leave(s, n);
    if (rc == GOFR_OK && line_rc != GOFR_OK) set_last_error("a log line of %u bytes does not fit line_cap %u", *line_len, line_cap);
    return rc != GOFR_OK ? rc : line_rc;
}

extern "C" {

int gofr_proto_frontend_call(gofr_proto_frontend* f, const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t out_cap,
                             uint32_t* out_len, uint32_t* status) {
    return proto_frontend_call(f, in, in_len, nullptr, nullptr, nullptr, out, out_cap, out_len, status, nullptr, 0, nullptr);
}

int gofr_proto_frontend_call_log(gofr_proto_frontend* f, const uint8_t* in, uint32_t in_len, const uint8_t trace_id[16],
                                 const gofr_log_desc* log, const uint8_t* method, uint8_t* out, uint32_t out_cap, uint32_t* out_len,
                                 uint32_t* status, uint8_t* line, uint32_t line_cap, uint32_t* line_len) {
    if (!log) return GOFR_ERR_INVALID;
    return proto_frontend_call(f, in, in_len, trace_id, log, method, out, out_cap, out_len, status, line, line_cap, line_len);
}

}  // extern "C"
