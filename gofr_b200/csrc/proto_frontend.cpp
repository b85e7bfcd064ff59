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
#include <cstring>
#include <vector>

#include "../../include/gofr_b200.h"
#include "engine_internal.h"
#include "frontend_ring.h"

static constexpr uint32_t kPrefix = 5;  // grpc-go's length-prefixed-message header: compressed flag, big-endian length

struct gofr_proto_frontend_batch {
    uint8_t* arena = nullptr;    // records back to back
    uint32_t* off = nullptr;     // max_batch + 1
    uint8_t* out = nullptr;      // grown by the dispatcher, never shrunk
    uint64_t out_cap = 0;
    uint32_t* out_off = nullptr; // max_batch + 1
    uint32_t* meta = nullptr;    // max_batch
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
    Staging b[gofr_ring::kBatches];
    gofr_ring::Ring ring;
};
using ProtoFrontend = gofr_proto_frontend;

static void free_staging(Staging& x) {
    gofr_free_pinned(x.arena); gofr_free_pinned(x.off); gofr_free_pinned(x.out);
    gofr_free_pinned(x.out_off); gofr_free_pinned(x.meta);
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
    auto call = f->decode ? gofr_proto_batch_decode : gofr_proto_batch_encode;
    gofr_ticket t = 0;
    int rc = call(f->eng, f->msgs.data(), (uint32_t)f->msgs.size(), f->fields.data(), (uint32_t)f->fields.size(), f->root, pr, &in,
                  &out, &t);
    if (rc == GOFR_OK) rc = gofr_batch_wait(f->eng, t);
    return rc;
}

extern "C" {

int gofr_proto_frontend_create(gofr_proto_frontend** out, gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs,
                               const gofr_proto_nfield* fields, uint32_t n_fields, uint32_t root, const uint8_t* presence,
                               int decode, uint32_t max_batch, uint32_t max_wait_us, uint32_t max_record_bytes) {
    if (!out || !e || max_batch == 0 || max_batch > 0x7FFFFFFFu) return GOFR_ERR_INVALID;
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
    for (auto& x : f->b) {
        x.arena = (uint8_t*)gofr_alloc_pinned((size_t)arena + 16);
        x.off = (uint32_t*)gofr_alloc_pinned(((size_t)max_batch + 1) * 4);
        x.out_off = (uint32_t*)gofr_alloc_pinned(((size_t)max_batch + 1) * 4);
        x.meta = (uint32_t*)gofr_alloc_pinned((size_t)max_batch * 4);
        if (!x.arena || !x.off || !x.out_off || !x.meta) {
            for (auto& y : f->b) free_staging(y);
            delete f;
            return GOFR_ERR_NOMEM;
        }
    }
    f->ring.start([f](int k, uint32_t n, uint32_t arena_bytes) { return serve_batch(f, k, n, arena_bytes); });
    *out = f;
    return GOFR_OK;
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

int gofr_proto_frontend_call(gofr_proto_frontend* f, const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t out_cap,
                             uint32_t* out_len, uint32_t* status) {
    if (!f || !out_len || !status || (in_len && !in) || (out_cap && !out)) return GOFR_ERR_INVALID;
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
    f->ring.leave(s, n);
    return rc;
}

}  // extern "C"
