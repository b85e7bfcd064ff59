// proto_nested_device.cuh — proto3 encoder for message types with nested and repeated fields
// (gofr_proto_encode_nested_device): proto.Marshal of the message a unary handler returns + grpc-go's 5-byte
// length-prefixed-message header (examples/grpc-server/grpc/hello_grpc.pb.go:73-89 hands the message to grpc-go's proto
// codec; protobuf-go v1.32.0, grpc-go v1.60.1) — the widening of grpc_device.cuh's flat encoder that SURVEY.md §8f rank 4
// leaves open.  Wire rules (protobuf-go impl/encode.go, codec_field.go, codec_gen.go):
//   * fields in ascending field-number order; a singular scalar holding its zero value is not written (proto3 implicit
//     presence); strings must be valid UTF-8;
//   * a singular message field is written when it is set, even when the message is empty (tag, length 0);
//   * repeated scalars of numeric type are PACKED: one tag (wire type 2), the payload length, the elements back to back —
//     nothing at all for zero elements; repeated strings / bytes / messages: one tag + length + payload PER ELEMENT,
//     empty elements included;
//   * map fields (codec_map.go) are repeated entry messages (1 key, 2 value) whose key and value are written even at their
//     zero value, a message value always (tag + length 0 when it is nil).  protobuf-go writes entries in Go's random map
//     order unless Deterministic is set, which sorts the keys; the row carries the entries in that order (checked: strictly
//     ascending keys, else BAD_ROW), so the bytes are the Deterministic ones;
//   * explicit presence (proto3 optional, oneof members; codec_field.go initOneofFieldCoders gives each member its own coder
//     in the field-number order): a set field is written even at its zero value or empty, an unset one not at all.
// Rows use the layout of the wider data model (include/gofr_b200.h "Row format"): fixed words of a message in field order
// (64-bit kinds two words, string / bytes their length, a singular message a presence word + its own fixed part inline, a
// repeated field its element count; an explicit-presence scalar / string a presence word before its usual words), then the
// variable part in field order (string bytes; a set message's variable part; repeated elements: scalars as their words,
// strings as u32 length + bytes, messages as fixed part + variable part).
// Device code does not recurse: the walk keeps an explicit stack of at most kPbnMaxDepth message levels (checked on the
// host when the call is made); the length prefix of a nested message comes from a sizing walk of that message.
// __host__ __device__ like the rest: tests/emu runs it on the CPU against the oracle and python google.protobuf.
#pragma once
#include "grpc_device.cuh"

namespace gofr {

struct PbnFrame {
    const uint8_t* fixed;  // fixed part of the message this frame walks
    uint32_t size;         // SIZE walk: bytes of the message's content so far
    uint32_t rep_left;     // elements still to come of the repeated message field the frame is in the middle of
    uint8_t mt, fi;        // message type, next field (index inside the type)
    uint8_t pend_tl;       // SIZE walk: tag length of the message field whose content the child frame is sizing
};
// SIZE walk, per frame with a map field in progress: the key of the entry seen last (kept apart from PbnFrame: the
// emitting walk, and message types without maps, never touch it)
struct PbnKey {
    uint64_t key;          // its order key (pbn_key_order), or for a string key:
    const uint8_t* s;      //     its bytes in the row
    uint32_t n;
    uint32_t have;         // an entry has been seen
};

GOFR_HD uint32_t pbn_ld32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

// map keys: the row words of an integer or bool key as a number whose unsigned order is the key order (bool false < true,
// signed kinds signed, unsigned kinds unsigned) — encoder and decoder compare through it
GOFR_HD uint64_t pbn_key_order(uint32_t flags, uint32_t cls, uint32_t w0, uint32_t w1) {
    if (cls & PC_BOOL) return w0 ? 1u : 0u;
    if (!(flags & PBN_SIGNED)) return (uint64_t)w0 | (uint64_t)((cls & PC_64) ? w1 : 0u) << 32;
    const uint64_t v = (cls & PC_64) ? ((uint64_t)w0 | (uint64_t)w1 << 32) : (uint64_t)(int64_t)(int32_t)w0;
    return v ^ 0x8000000000000000ull;
}
// string keys: Go's <, byte order with a shorter prefix first.  <0, 0, >0
GOFR_HD int pbn_bytes_cmp(const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn) {
    const uint32_t n = an < bn ? an : bn;
    for (uint32_t i = 0; i < n; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return an < bn ? -1 : an > bn ? 1 : 0;
}

// One walk over message type `mt` whose fixed part is at `fixed` and whose variable part starts at *var (end = end of the
// row).  EMIT == false: returns the size of the message's content, validates the row (*status: GOFR_GRPC_BAD_ROW /
// GOFR_GRPC_BAD_UTF8) and advances *var past the message's variable part.  EMIT == true: writes the content through w
// (the row has been validated by the sizing walk of the whole row).  MAPS == false: the instance for descriptions without
// map fields, with no map code in it.  PRES == true (with MAPS): the instance for descriptions with explicit-presence
// fields (PbnDesc::presence); the others contain no presence code.
template <bool EMIT, bool MAPS, bool PRES = false>
GOFR_HD_NOINLINE uint32_t pbn_walk(const PbnDesc& D, uint32_t mt, const uint8_t* fixed, const uint8_t** var_io, const uint8_t* end,
                                   Writer* w, uint32_t* status) {
    PbnFrame st[kPbnMaxDepth + 1];
    int depth = 0;
    const uint8_t* var = *var_io;
    uint32_t err = GOFR_GRPC_OK, result = 0;
    auto take = [&](uint32_t n) -> const uint8_t* {
        if ((uint32_t)(end - var) < n) { err = GOFR_GRPC_BAD_ROW; return nullptr; }
        const uint8_t* p = var;
        var += n;
        return p;
    };
    // SIZE walk, per frame: the oneof groups (bit k: group k) that have a present member so far (kept apart from PbnFrame,
    // like PbnKey: the instances without presence never touch it)
    uint8_t groups_set[kPbnMaxDepth + 1];
    auto push = [&](uint32_t m, const uint8_t* fx) {
        if (depth > kPbnMaxDepth) { err = GOFR_GRPC_BAD_ROW; return; }
        if constexpr (PRES) groups_set[depth] = 0;
        PbnFrame& f = st[depth++];
        f.fixed = fx; f.size = 0; f.rep_left = 0; f.mt = (uint8_t)m; f.fi = 0; f.pend_tl = 0;
    };
    PbnKey keys[kPbnMaxDepth + 1];
    // SIZE walk, the key of a map entry (frame fi; the map's frame is fi - 1): strictly above the previous entry's key
    auto key_in_order = [&](int fi, const PbnField& K, const uint8_t* p, const uint8_t* s) -> bool {
        PbnKey& M = keys[fi - 1];
        bool ok;
        if ((K.cls & PC_WIRE) == 2) {
            const uint32_t n = pbn_ld32(p);
            ok = !M.have || pbn_bytes_cmp(M.s, M.n, s, n) < 0;
            M.s = s; M.n = n;
        } else {
            const uint64_t k = pbn_key_order(K.flags, K.cls, pbn_ld32(p), (K.cls & PC_64) ? pbn_ld32(p + 4) : 0u);
            ok = !M.have || M.key < k;
            M.key = k;
        }
        M.have = 1;
        return ok;
    };
    auto put_varint = [&](uint64_t v) { w->reserve(3); proto_put_varint(*w, v); };
    // a scalar payload (what follows the tag) of class cls whose words are at p: its encoded length, written when EMIT
    auto scalar = [&](uint32_t cls, const uint8_t* p) -> uint32_t {
        const uint32_t w0 = pbn_ld32(p), w1 = (cls & PC_64) ? pbn_ld32(p + 4) : 0u;
        const uint32_t wire = cls & PC_WIRE;
        if (wire == 1) { if (EMIT) { w->reserve(3); w->put4(w0); w->put4(w1); } return 8; }
        if (wire == 5) { if (EMIT) { w->reserve(2); w->put4(w0); } return 4; }
        const uint64_t v = proto_varint_value(cls, w0, w1);
        if (EMIT) put_varint(v);
        return varint_len64(v);
    };
    // enters the message of field F (type F.msg) whose fixed part is at fx: the tag and length prefix now (EMIT) or when
    // the child frame is popped (SIZE)
    auto enter_message = [&](const PbnField& F, const uint8_t* fx, int parent) {
        if constexpr (EMIT) {  // (constexpr: the sizing instance must not contain a call to itself)
            const uint8_t* v2 = var;
            uint32_t st2 = GOFR_GRPC_OK;
            const uint32_t sub = pbn_walk<false, MAPS, PRES>(D, F.msg, fx, &v2, end, nullptr, &st2);
            put_varint(F.tag);
            put_varint(sub);
        } else st[parent].pend_tl = (uint8_t)varint_len(F.tag);
        push(F.msg, fx);
    };

    push(mt, fixed);
    while (depth > 0 && err == GOFR_GRPC_OK) {
        const int fi = depth - 1;
        const PbnField* fields = D.f + D.first[st[fi].mt];
        if (st[fi].rep_left) {  // next element of a repeated message field (the field before st[fi].fi)
            const PbnField& F = fields[st[fi].fi - 1];
            st[fi].rep_left--;
            const uint8_t* fx = take((uint32_t)D.fixed_words[F.msg] * 4u);
            if (fx) enter_message(F, fx, fi);
            continue;
        }
        if (st[fi].fi >= D.count[st[fi].mt]) {  // message done
            const uint32_t sub = st[fi].size;
            depth--;
            if (depth > 0) { if (!EMIT) st[depth - 1].size += st[depth - 1].pend_tl + varint_len(sub) + sub; }
            else result = sub;
            continue;
        }
        const PbnField& F = fields[st[fi].fi];
        // the field's fixed words: fields before it in the same message
        uint32_t wo = 0;
        for (uint32_t k = 0; k < st[fi].fi; k++) wo += fields[k].fixed_words;
        const uint8_t* p = st[fi].fixed + (size_t)wo * 4;
        st[fi].fi++;
        const uint32_t tl = varint_len(F.tag), cls = F.cls, wire = cls & PC_WIRE;
        if constexpr (PRES) {
            if (F.flags & (PBN_PRESENCE | PBN_ONEOF)) {  // explicit presence: the presence word, then the value words
                const uint32_t set = pbn_ld32(p), group = (uint32_t)F.flags >> PBN_ONEOF_SHIFT;
                if (!EMIT) {  // set is 0 / 1; an unset field's value words are zero; one set member per oneof group
                    bool bad = set > 1u;
                    if (!set) for (uint32_t k = 1; k < F.fixed_words; k++) bad |= pbn_ld32(p + 4u * k) != 0u;
                    if (set && group) { bad |= (groups_set[fi] >> group & 1u) != 0u; groups_set[fi] |= (uint8_t)(1u << group); }
                    if (bad) { err = GOFR_GRPC_BAD_ROW; break; }
                }
                if (!set) continue;
                const uint8_t* v = p + 4;
                if (F.msg != 0xFF) enter_message(F, v, fi);
                else if (wire == 2) {  // written even when empty
                    const uint32_t len = pbn_ld32(v);
                    const uint8_t* s = take(len);
                    if (!s) break;
                    if (!EMIT && (cls & PC_UTF8) && !proto_utf8_ok(s, len)) { err = GOFR_GRPC_BAD_UTF8; break; }
                    if (EMIT) { put_varint(F.tag); put_varint(len); if (len) w->copy<false>(s, len); }
                    st[fi].size += tl + varint_len(len) + len;
                } else {  // written even at its zero value
                    if (EMIT) put_varint(F.tag);
                    st[fi].size += tl + scalar(cls, v);
                }
                continue;
            }
        }
        // (a map-free description has no flag bits but PBN_REPEATED: its instance tests the byte, as before maps)
        if (!(MAPS ? (F.flags & PBN_REPEATED) : F.flags)) {
            // the key or value of a map entry: written at its zero value too; the key (field index 0) in order (SIZE walk of
            // the whole row: the entry's frame has its map's frame below it)
            const bool entry = MAPS && (F.flags & PBN_ENTRY), is_key = !EMIT && entry && st[fi].fi == 1 && fi > 0;
            if (F.msg != 0xFF) {  // singular message: presence word, then the fixed part inline
                if (pbn_ld32(p)) enter_message(F, p + 4, fi);
                else if (entry) {  // a nil map value is written as an empty message
                    if (EMIT) { put_varint(F.tag); put_varint(0); }
                    st[fi].size += tl + 1;
                }
            } else if (wire == 2) {  // string / bytes
                const uint32_t len = pbn_ld32(p);
                const uint8_t* s = take(len);
                if (!s) break;
                if (!EMIT && (cls & PC_UTF8) && !proto_utf8_ok(s, len)) { err = GOFR_GRPC_BAD_UTF8; break; }
                if (is_key && !key_in_order(fi, F, p, s)) { err = GOFR_GRPC_BAD_ROW; break; }
                if (len || entry) {
                    if (EMIT) { put_varint(F.tag); put_varint(len); if (len) w->copy<false>(s, len); }
                    st[fi].size += tl + varint_len(len) + len;
                }
            } else {
                const uint32_t w0 = pbn_ld32(p), w1 = (cls & PC_64) ? pbn_ld32(p + 4) : 0u;
                if (is_key && !key_in_order(fi, F, p, nullptr)) { err = GOFR_GRPC_BAD_ROW; break; }
                if ((w0 | w1) || entry) {
                    if (EMIT) put_varint(F.tag);
                    st[fi].size += tl + scalar(cls, p);
                }
            }
            continue;
        }
        const uint32_t n = pbn_ld32(p);
        if (F.msg != 0xFF) {  // repeated messages and map entries: one after the other through the frame's rep_left
            if ((uint32_t)(end - var) / 4u < n && D.fixed_words[F.msg]) { err = GOFR_GRPC_BAD_ROW; break; }
            if (n > 0x00FFFFFFu) { err = GOFR_GRPC_BAD_ROW; break; }
            st[fi].rep_left = n;
            if (!EMIT && MAPS && (F.flags & PBN_MAP)) keys[fi].have = 0;
        } else if (wire == 2) {  // repeated string / bytes: tag + length + payload per element
            if ((uint32_t)(end - var) / 4u < n) { err = GOFR_GRPC_BAD_ROW; break; }
            for (uint32_t i = 0; i < n; i++) {
                const uint8_t* lp = take(4);
                if (!lp) break;
                const uint32_t len = pbn_ld32(lp);
                const uint8_t* s = take(len);
                if (!s) break;
                if (!EMIT && (cls & PC_UTF8) && !proto_utf8_ok(s, len)) { err = GOFR_GRPC_BAD_UTF8; break; }
                if (EMIT) { put_varint(F.tag); put_varint(len); if (len) w->copy<false>(s, len); }
                st[fi].size += tl + varint_len(len) + len;
            }
        } else if (n) {  // packed repeated scalars: tag, payload length, the elements
            const uint32_t eb = (cls & PC_64) ? 8u : 4u;
            if ((uint32_t)(end - var) / eb < n) { err = GOFR_GRPC_BAD_ROW; break; }
            const uint8_t* e0 = take(n * eb);
            uint32_t payload = 0;
            if (wire == 1) payload = 8u * n;
            else if (wire == 5) payload = 4u * n;
            else for (uint32_t i = 0; i < n; i++) {
                const uint8_t* q = e0 + (size_t)i * eb;
                payload += varint_len64(proto_varint_value(cls, pbn_ld32(q), (cls & PC_64) ? pbn_ld32(q + 4) : 0u));
            }
            if (EMIT) {
                put_varint(F.tag);
                put_varint(payload);
                for (uint32_t i = 0; i < n; i++) scalar(cls, e0 + (size_t)i * eb);
            }
            st[fi].size += tl + varint_len(payload) + payload;
        }
    }
    *var_io = var;
    *status = err;
    return result;
}

struct PbnMsg {
    uint32_t status;   // GOFR_GRPC_OK / GOFR_GRPC_BAD_UTF8 / GOFR_GRPC_BAD_ROW
    uint32_t out_len;  // 5 + message bytes (0 on error)
};

// size pass of one row: validates it and returns the exact frame length.  The kernels instantiate it for MAPS == D.maps
// and PRES == D.presence (one kernel per choice, picked on the host: the map-free kernel contains no map code, only the
// presence kernels contain presence code — with maps, whether the description has any or not); pbn_size dispatches at
// run time.
template <bool MAPS, bool PRES = false>
GOFR_HD PbnMsg pbn_size_as(const PbnDesc& D, const uint8_t* row, uint32_t rn) {
    PbnMsg m = {GOFR_GRPC_OK, 0};
    const uint32_t fb = (uint32_t)D.fixed_words[D.root] * 4u;
    if (rn < fb) { m.status = GOFR_GRPC_BAD_ROW; return m; }
    const uint8_t* var = row + fb;
    uint32_t st = GOFR_GRPC_OK;
    const uint32_t len = pbn_walk<false, MAPS, PRES>(D, D.root, row, &var, row + rn, nullptr, &st);
    m.status = st;
    m.out_len = st == GOFR_GRPC_OK ? 5u + len : 0u;
    return m;
}

// emit pass: the frame at dst (arbitrary alignment inside the packed output)
template <bool MAPS, bool PRES = false>
GOFR_HD void pbn_emit_as(const PbnDesc& D, const uint8_t* row, uint32_t rn, const PbnMsg m, uint8_t* dst, uint32_t* stage_col) {
    if (!m.out_len) return;
    Writer w;
    w.init(dst, stage_col);
    const uint32_t plen = m.out_len - 5;
    w.put4(0u | (plen >> 24) << 8 | ((plen >> 16) & 0xFF) << 16 | ((plen >> 8) & 0xFF) << 24);  // 00, be32[0..2]
    w.putc(plen & 0xFF);
    const uint8_t* var = row + (size_t)D.fixed_words[D.root] * 4;
    uint32_t st = GOFR_GRPC_OK;
    pbn_walk<true, MAPS, PRES>(D, D.root, row, &var, row + rn, &w, &st);
    w.finish();
}

GOFR_HD PbnMsg pbn_size(const PbnDesc& D, const uint8_t* row, uint32_t rn) {
    if (D.presence) return pbn_size_as<true, true>(D, row, rn);
    return D.maps ? pbn_size_as<true>(D, row, rn) : pbn_size_as<false>(D, row, rn);
}
GOFR_HD void pbn_emit(const PbnDesc& D, const uint8_t* row, uint32_t rn, const PbnMsg m, uint8_t* dst, uint32_t* stage_col) {
    if (D.presence) pbn_emit_as<true, true>(D, row, rn, m, dst, stage_col);
    else if (D.maps) pbn_emit_as<true>(D, row, rn, m, dst, stage_col);
    else pbn_emit_as<false>(D, row, rn, m, dst, stage_col);
}

}  // namespace gofr
