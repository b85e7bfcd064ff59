// proto_nested_decode_device.cuh — proto3 decoder for message types with nested and repeated fields
// (gofr_proto_decode_nested_device): dec(in) of a unary handler (examples/grpc-server/grpc/hello_grpc.pb.go:73-89) — the
// 5-byte length-prefixed-message header checked, proto.Unmarshal into the message type, the values out as a row in the layout
// gofr_proto_encode_nested_device reads (include/gofr_b200.h "Row format").  protobuf-go v1.32.0 rules restated
// (impl/decode.go, codec_field.go, codec_gen.go), on top of the flat decoder's (grpc_device.cuh):
//   * a known field arriving with another wire type than its own is an unknown field — except that a repeated numeric
//     scalar is accepted BOTH packed (wire type 2, elements back to back) and unpacked (one element per tag), mixed freely,
//     elements in wire order;
//   * singular scalars / strings: the last occurrence wins; every occurrence of a string must be valid UTF-8;
//   * a singular message field occurring more than once is MERGED by protobuf-go; that is not done here: the frame comes
//     back with GOFR_GRPC_DEFER ("valid, but decode it on the host") — canonical encoders write the field once;
//   * repeated strings / bytes / messages: one element per occurrence, in wire order; unknown fields and balanced groups
//     are skipped at every level; nested messages are only parsed where the schema knows them;
//   * map fields (codec_map.go): each occurrence is an entry message, decoded like any message (last key and value win, a
//     value message sent twice is merged -> DEFER as above); across entries a later equal key replaces the earlier entry.
//     The row holds the map in the encoder's canonical form: keys ascending, each once.  The walks find it by SELECTION —
//     per output slot, the smallest key above the previous one among all entries, the last entry carrying it — no scratch,
//     quadratic, so more than kPbnMaxMapEntries entries of one map field in one message (duplicates counted) are DEFER
//     (the second pass, proto_nested_deferred_device.cuh, takes those frames with sorted lists instead: the MapStep policy);
//   * explicit presence: an optional field is set iff it occurs (with its own wire type), the last occurrence winning; of a
//     oneof group the member occurring last among all the group's members is the set one, with its last value.  A message
//     member sent twice (even with another member between) is DEFER, by the rule for singular message fields above.
// Three walks per frame, none recursive (explicit stacks, at most kPbnMaxDepth message levels):
//   validate   wire order: framing of every level that the schema knows, UTF-8, packed payloads, repeated singular messages
//   size       field order: the row's byte count
//   emit       field order again, this time storing — the fixed part of a message is written where its parent put it, the
//              variable part is appended; byte stores, no Writer: a row is not produced front to back.
// Status precedence when a frame has several problems: malformed > invalid UTF-8 > DEFER (protobuf-go reports whichever
// comes first in wire order; either way the RPC fails).  __host__ __device__: tests/emu runs it on the CPU.
#pragma once
#include "proto_nested_device.cuh"

namespace gofr {

struct PdnRow {
    uint32_t status;   // GOFR_GRPC_*
    uint32_t out_len;  // bytes of the row (multiple of 4; 0 unless GOFR_GRPC_OK)
};

// the scalar's row words from its wire value (the flat decoder's rules)
GOFR_HD void pdn_scalar_words(uint32_t cls, uint32_t wt, uint64_t v, uint32_t* w0, uint32_t* w1) {
    *w1 = 0;
    if (wt != 0 || ((cls & PC_64) && !(cls & PC_ZIGZAG))) { *w0 = (uint32_t)v; *w1 = (uint32_t)(v >> 32); }
    else if (cls & PC_ZIGZAG) {
        if (cls & PC_64) { const uint64_t z = (v >> 1) ^ (uint64_t)-(int64_t)(v & 1); *w0 = (uint32_t)z; *w1 = (uint32_t)(z >> 32); }
        else { const uint32_t x = (uint32_t)v; *w0 = (x >> 1) ^ (uint32_t)-(int32_t)(x & 1); }
    } else if (cls & PC_BOOL) *w0 = v != 0 ? 1u : 0u;
    else *w0 = (uint32_t)v;
    if (!(cls & PC_64)) *w1 = 0;
}

// One field of a message: tag and payload.  Returns false on malformed bytes.  wt 3 / 4 (groups) return with plen = 0.
struct PdnItem { uint32_t num, wt, poff, plen; uint64_t v; };
GOFR_HD bool pdn_next(const uint8_t* f, uint32_t* ip, uint32_t hi, PdnItem* it) {
    uint32_t i = *ip;
    uint64_t tag;
    int k = grpc_varint(f + i, hi - i, &tag);
    if (k < 0) return false;
    i += (uint32_t)k;
    const uint64_t num = tag >> 3;
    if (num == 0 || num > 0x1FFFFFFFull) return false;
    it->num = (uint32_t)num; it->wt = (uint32_t)(tag & 7); it->poff = 0; it->plen = 0; it->v = 0;
    uint64_t v = 0;
    if (it->wt == 0) {
        k = grpc_varint(f + i, hi - i, &v);
        if (k < 0) return false;
        i += (uint32_t)k;
    } else if (it->wt == 1) {
        if (hi - i < 8) return false;
        for (int q = 7; q >= 0; q--) v = v << 8 | f[i + (uint32_t)q];
        i += 8;
    } else if (it->wt == 5) {
        if (hi - i < 4) return false;
        for (int q = 3; q >= 0; q--) v = v << 8 | f[i + (uint32_t)q];
        i += 4;
    } else if (it->wt == 2) {
        k = grpc_varint(f + i, hi - i, &v);
        if (k < 0) return false;
        i += (uint32_t)k;
        if (v > hi - i) return false;
        it->poff = i;
        it->plen = (uint32_t)v;
        i += it->plen;
    } else if (it->wt != 3 && it->wt != 4) return false;
    it->v = v;
    *ip = i;
    return true;
}

// the field of message type mt that a (number, wire type) addresses, or -1: same number, and the field's own wire type or —
// for a repeated numeric scalar — either its element wire type or 2 (packed).  (MAPS == false: a map-free description,
// whose flag bytes hold PBN_REPEATED alone)
template <bool MAPS = true>
GOFR_HD int pdn_field_of(const PbnDesc& D, uint32_t mt, uint32_t num, uint32_t wt) {
    const PbnField* F = D.f + D.first[mt];
    for (uint32_t q = 0; q < D.count[mt]; q++) {
        if ((F[q].tag >> 3) != num) continue;
        const uint32_t own = F[q].msg != 0xFF ? 2u : (uint32_t)(F[q].cls & PC_WIRE);
        if (wt == own) return (int)q;
        if ((MAPS ? (F[q].flags & PBN_REPEATED) : F[q].flags) && F[q].msg == 0xFF && own != 2u && wt == 2u) return (int)q;  // packed
        return -1;
    }
    return -1;
}

// top-level items of [i, hi) (a message of type mt; unknown groups skipped whole) that address field q: how many — stops
// early at malformed bytes, which the validating walk reports anyway
GOFR_HD uint32_t pdn_count_after(const PbnDesc& D, const uint8_t* f, uint32_t i, uint32_t hi, uint32_t mt, uint32_t q) {
    uint32_t n = 0, g = 0;
    while (i < hi) {
        PdnItem it;
        if (!pdn_next(f, &i, hi, &it)) break;
        if (it.wt == 3) { g++; continue; }
        if (it.wt == 4) { if (!g) break; g--; continue; }
        if (!g && pdn_field_of(D, mt, it.num, it.wt) == (int)q) n++;
    }
    return n;
}

// A map's key in [lo, hi), the content of one entry (type E; its key is field index 0): the last occurrence, else the zero
// value.  Integer and bool keys as pbn_key_order numbers; string keys as (offset << 32 | length) of their bytes in f.
GOFR_HD uint64_t pdn_entry_key(const PbnDesc& D, const uint8_t* f, uint32_t lo, uint32_t hi, uint32_t E) {
    const PbnField& K = D.f[D.first[E]];
    const bool str = (K.cls & PC_WIRE) == 2;
    uint64_t key = str ? 0u : pbn_key_order(K.flags, K.cls, 0u, 0u);
    uint32_t i = lo, g = 0;
    while (i < hi) {
        PdnItem it;
        pdn_next(f, &i, hi, &it);
        if (it.wt == 3) { g++; continue; }
        if (it.wt == 4) { g--; continue; }
        if (g || pdn_field_of(D, E, it.num, it.wt) != 0) continue;
        if (str) key = (uint64_t)it.poff << 32 | it.plen;
        else {
            uint32_t w0, w1;
            pdn_scalar_words(K.cls, it.wt, it.v, &w0, &w1);
            key = pbn_key_order(K.flags, K.cls, w0, w1);
        }
    }
    return key;
}
GOFR_HD bool pdn_key_less(const uint8_t* f, bool str, uint64_t a, uint64_t b) {
    if (!str) return a < b;
    return pbn_bytes_cmp(f + (a >> 32), (uint32_t)a, f + (b >> 32), (uint32_t)b) < 0;
}

// The next entry of map field q (entry type E) of the message [lo, hi) of type mt in canonical order, by selection: the
// smallest key above *key (any key when !have_key), the last entry on the wire that carries it.  False when there is none.
GOFR_HD bool pdn_map_next(const PbnDesc& D, const uint8_t* f, uint32_t lo, uint32_t hi, uint32_t mt, uint32_t q, uint32_t E,
                          bool have_key, uint64_t* key, PdnItem* out) {
    const bool str = (D.f[D.first[E]].cls & PC_WIRE) == 2;
    bool found = false;
    uint64_t best = 0;
    uint32_t i = lo, g = 0;
    while (i < hi) {
        PdnItem it;
        pdn_next(f, &i, hi, &it);
        if (it.wt == 3) { g++; continue; }
        if (it.wt == 4) { g--; continue; }
        if (g || pdn_field_of(D, mt, it.num, it.wt) != (int)q) continue;
        const uint64_t k = pdn_entry_key(D, f, it.poff, it.poff + it.plen, E);
        if (have_key && !pdn_key_less(f, str, *key, k)) continue;  // not above the previous key
        if (found && pdn_key_less(f, str, best, k)) continue;      // above the best so far
        best = k;                                                  // smaller, or equal and later on the wire: this one
        *out = it;
        found = true;
    }
    if (found) *key = best;
    return found;
}

// The map step of the field-order walk (pdn_walk's MapStep), a policy of static functions:
//   begin(D, f, lo, hi, mt, q, E, level, it)  the number of distinct keys of map field q (entry type E) of the message
//                                          [lo, hi) of type mt; `level` counts the maps active around it (0 outermost);
//                                          *it is the walk's item, free to be used as scratch
//   next(..., level, have, cursor, out)    the next entry in canonical order after the one *cursor stands for (the first
//                                          when !have): its payload in out->poff / plen, *cursor moved on; false at the end
//   store()                                whether this thread makes the emitting walk's stores
//   kMaxEntries                            the most entries of one map field in one message it takes (more: DEFER)
// PdnSelect is the selection above: no scratch, quadratic, one thread per frame.  (proto_nested_deferred_device.cuh has the
// sorted-list policy, for one CTA per frame.)
struct PdnSelect {
    static constexpr uint32_t kMaxEntries = (uint32_t)kPbnMaxMapEntries;
    static GOFR_HD uint32_t begin(const PbnDesc& D, const uint8_t* f, uint32_t lo, uint32_t hi, uint32_t mt, uint32_t q, uint32_t E, int,
                                  PdnItem* it) {
        uint32_t n = 0;
        uint64_t key = 0;
        while (pdn_map_next(D, f, lo, hi, mt, q, E, n != 0, &key, it)) n++;
        return n;
    }
    static GOFR_HD bool next(const PbnDesc& D, const uint8_t* f, uint32_t lo, uint32_t hi, uint32_t mt, uint32_t q, uint32_t E, int,
                             bool have, uint64_t* cursor, PdnItem* out) {
        return pdn_map_next(D, f, lo, hi, mt, q, E, have, cursor, out);
    }
    static constexpr GOFR_HD bool store() { return true; }
};

// elements of a packed payload [lo, hi) of class cls: count them, or fail when the payload is not a whole number of elements
GOFR_HD bool pdn_packed_count(const uint8_t* f, uint32_t lo, uint32_t hi, uint32_t cls, uint32_t* n) {
    const uint32_t wire = cls & PC_WIRE;
    if (wire == 1) { if ((hi - lo) & 7u) return false; *n = (hi - lo) >> 3; return true; }
    if (wire == 5) { if ((hi - lo) & 3u) return false; *n = (hi - lo) >> 2; return true; }
    uint32_t c = 0;
    while (lo < hi) {
        uint64_t v;
        const int k = grpc_varint(f + lo, hi - lo, &v);
        if (k < 0) return false;
        lo += (uint32_t)k;
        c++;
    }
    *n = c;
    return true;
}

// ---- walk 1: validate, in wire order ----
// (MAPS == false: the instance for descriptions without map fields, as for the walks below.  MAXE: the most entries one map
// field may have in one message, duplicates counted; more are DEFER)
template <bool MAPS, uint32_t MAXE = (uint32_t)kPbnMaxMapEntries>
GOFR_HD_NOINLINE uint32_t pdn_validate(const PbnDesc& D, const uint8_t* f, uint32_t lo, uint32_t hi) {
    struct Lv { uint32_t end; uint64_t seen; uint8_t mt; uint8_t gbase; } lv[kPbnMaxDepth + 1];
    uint32_t groups[kMaxGroupDepth];
    int depth = 0;
    uint32_t gdepth = 0, i = lo;
    bool bad_utf8 = false, defer = false;
    lv[depth].end = hi; lv[depth].seen = 0; lv[depth].mt = (uint8_t)D.root; lv[depth].gbase = 0; depth++;
    for (;;) {
        Lv& L = lv[depth - 1];
        if (i == L.end) {
            if (gdepth != L.gbase) return GOFR_GRPC_BAD_PROTO;  // a group left open inside this message
            if (--depth == 0) break;
            continue;
        }
        PdnItem it;
        if (!pdn_next(f, &i, L.end, &it)) return GOFR_GRPC_BAD_PROTO;
        if (it.wt == 3) {
            if (gdepth == kMaxGroupDepth) return GOFR_GRPC_BAD_PROTO;
            groups[gdepth++] = it.num;
            continue;
        }
        if (it.wt == 4) {
            if (gdepth == L.gbase || groups[gdepth - 1] != it.num) return GOFR_GRPC_BAD_PROTO;
            gdepth--;
            continue;
        }
        if (gdepth != L.gbase) continue;  // inside an unknown group: nothing is known
        const int q = pdn_field_of<MAPS>(D, L.mt, it.num, it.wt);
        if (q < 0) continue;
        const PbnField& F = D.f[D.first[L.mt] + (uint32_t)q];
        if (F.msg != 0xFF) {
            if (!(MAPS ? (F.flags & PBN_REPEATED) : F.flags)) {
                if (L.seen >> q & 1u) defer = true;
                L.seen |= 1ull << q;
            } else if (MAPS && (F.flags & PBN_MAP) && !(L.seen >> q & 1u)) {  // first entry of a map field: count them all once
                L.seen |= 1ull << q;
                if (1u + pdn_count_after(D, f, i, L.end, L.mt, (uint32_t)q) > MAXE) defer = true;
            }
            if (depth > kPbnMaxDepth) return GOFR_GRPC_BAD_PROTO;  // cannot happen: the schema's depth was checked
            i = it.poff;  // descend: the payload is parsed as a message of type F.msg
            lv[depth].end = it.poff + it.plen; lv[depth].seen = 0; lv[depth].mt = F.msg; lv[depth].gbase = (uint8_t)gdepth; depth++;
            continue;
        }
        if (it.wt == 2) {
            if ((F.cls & PC_WIRE) == 2) { if ((F.cls & PC_UTF8) && !proto_utf8_ok(f + it.poff, it.plen)) bad_utf8 = true; }
            else { uint32_t n; if (!pdn_packed_count(f, it.poff, it.poff + it.plen, F.cls, &n)) return GOFR_GRPC_BAD_PROTO; }
        }
    }
    return bad_utf8 ? GOFR_GRPC_BAD_UTF8 : defer ? GOFR_GRPC_DEFER : GOFR_GRPC_OK;
}

GOFR_HD void pdn_st32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

// ---- walks 2 and 3: field order; EMIT stores into row[] ----
// Returns the row's byte count before padding.  The frame has been validated: no check can fail here.  PRES == true (with
// MAPS): the instance for descriptions with explicit-presence fields.  MapStep: how map entries are put in key order (see
// PdnSelect); only the threads whose MapStep::store() holds make the emitting walk's stores.
template <bool EMIT, bool MAPS, bool PRES = false, class MapStep = PdnSelect>
GOFR_HD_NOINLINE uint32_t pdn_walk(const PbnDesc& D, const uint8_t* f, uint32_t lo, uint32_t hi, uint8_t* row) {
    // in_rep: 1 elements of a repeated message field in wire order (scan: where to look on), 2 / 3 entries of a map field in
    // key order (3: keys[frame] = MapStep's cursor at the entry taken last)
    struct Fr { uint32_t lo, hi, fx, scan; uint8_t mt, fi, in_rep; } st[kPbnMaxDepth + 1];
    uint64_t keys[kPbnMaxDepth + 1];
    const bool stores = EMIT && MapStep::store();  // the emitting walk, and this thread makes its stores
    int maps = 0;  // map fields whose entries are being walked (the innermost one's level is maps - 1)
    int depth = 0;
    uint32_t vc = (uint32_t)D.fixed_words[D.root] * 4u;  // append position of the variable part
    st[0].lo = lo; st[0].hi = hi; st[0].fx = 0; st[0].scan = 0; st[0].mt = (uint8_t)D.root; st[0].fi = 0; st[0].in_rep = 0;
    depth = 1;
    // the next top-level item of [i, hi) that addresses field q of message type mt (unknown groups skipped whole)
    auto find = [&](uint32_t mt, uint32_t q, uint32_t* ip, uint32_t end, PdnItem* out) -> bool {
        uint32_t i = *ip, g = 0;
        while (i < end) {
            PdnItem it;
            pdn_next(f, &i, end, &it);
            if (it.wt == 3) { g++; continue; }
            if (it.wt == 4) { g--; continue; }
            if (g) continue;
            if (pdn_field_of<MAPS>(D, mt, it.num, it.wt) == (int)q) { *out = it; *ip = i; return true; }
        }
        *ip = i;
        return false;
    };
    while (depth > 0) {
        Fr& fr = st[depth - 1];
        const PbnField* fields = D.f + D.first[fr.mt];
        if (fr.in_rep) {  // repeated message field fr.fi - 1: the next occurrence (the next entry of a map) is the next element
            const PbnField& F = fields[fr.fi - 1];
            PdnItem it;
            bool more;
            if (!MAPS || fr.in_rep == 1) more = find(fr.mt, fr.fi - 1u, &fr.scan, fr.hi, &it);
            else {
                more = MapStep::next(D, f, fr.lo, fr.hi, fr.mt, fr.fi - 1u, F.msg, maps - 1, fr.in_rep == 3, &keys[depth - 1], &it);
                fr.in_rep = 3;
                if (!more) maps--;
            }
            if (more) {
                const uint32_t efx = vc;
                vc += (uint32_t)D.fixed_words[F.msg] * 4u;
                Fr& ch = st[depth++];
                ch.lo = it.poff; ch.hi = it.poff + it.plen; ch.fx = efx; ch.scan = 0; ch.mt = F.msg; ch.fi = 0; ch.in_rep = 0;
            } else fr.in_rep = 0;
            continue;
        }
        if (fr.fi >= D.count[fr.mt]) { depth--; continue; }
        const uint32_t q = fr.fi;
        const PbnField& F = fields[q];
        uint32_t wo = 0;
        for (uint32_t k = 0; k < q; k++) wo += fields[k].fixed_words;
        const uint32_t fxo = fr.fx + wo * 4u;  // where this field's fixed words go
        fr.fi++;
        const uint32_t cls = F.cls;
        PdnItem it;
        uint32_t i = fr.lo;
        if constexpr (PRES) {
            if (F.flags & (PBN_PRESENCE | PBN_ONEOF)) {
                // one pass over the message: the field's last occurrence, and whether a member of its oneof group came
                // after it (then that member is the set one)
                const uint32_t group = (uint32_t)F.flags >> PBN_ONEOF_SHIFT;
                bool set = false;
                uint32_t g = 0;
                while (i < fr.hi) {
                    PdnItem x;
                    pdn_next(f, &i, fr.hi, &x);
                    if (x.wt == 3) { g++; continue; }
                    if (x.wt == 4) { g--; continue; }
                    if (g) continue;
                    const int o = pdn_field_of<MAPS>(D, fr.mt, x.num, x.wt);
                    if (o == (int)q) { set = true; it = x; }
                    else if (group && o >= 0 && ((uint32_t)fields[o].flags >> PBN_ONEOF_SHIFT) == group) set = false;
                }
                if (stores) pdn_st32(row + fxo, set ? 1u : 0u);
                if (F.msg != 0xFF) {  // a oneof member of message type: its fixed part inline (zeros when unset)
                    if (set) {
                        Fr& ch = st[depth++];
                        ch.lo = it.poff; ch.hi = it.poff + it.plen; ch.fx = fxo + 4u; ch.scan = 0; ch.mt = F.msg; ch.fi = 0; ch.in_rep = 0;
                    } else if (stores) for (uint32_t k = 0; k < (uint32_t)D.fixed_words[F.msg] * 4u; k++) row[fxo + 4u + k] = 0;
                } else if ((cls & PC_WIRE) == 2) {
                    const uint32_t plen = set ? it.plen : 0u;
                    if (stores) {
                        pdn_st32(row + fxo + 4u, plen);
                        for (uint32_t k = 0; k < plen; k++) row[vc + k] = f[it.poff + k];
                    }
                    vc += plen;
                } else {
                    uint32_t w0 = 0, w1 = 0;
                    if (set) pdn_scalar_words(cls, it.wt, it.v, &w0, &w1);
                    if (stores) { pdn_st32(row + fxo + 4u, w0); if (cls & PC_64) pdn_st32(row + fxo + 8u, w1); }
                }
                continue;
            }
        }
        if (!(MAPS ? (F.flags & PBN_REPEATED) : F.flags)) {
            if (F.msg != 0xFF) {  // singular message: presence word + its fixed part inline (zeros when absent)
                // (a map value is always present: a missing one is an empty message)
                const bool present = find(fr.mt, q, &i, fr.hi, &it);
                if (stores) {
                    pdn_st32(row + fxo, present || (MAPS && (F.flags & PBN_ENTRY)) ? 1u : 0u);
                    if (!present) for (uint32_t k = 0; k < (uint32_t)D.fixed_words[F.msg] * 4u; k++) row[fxo + 4u + k] = 0;
                }
                if (present) {
                    Fr& ch = st[depth++];
                    ch.lo = it.poff; ch.hi = it.poff + it.plen; ch.fx = fxo + 4u; ch.scan = 0; ch.mt = F.msg; ch.fi = 0; ch.in_rep = 0;
                }
            } else if ((cls & PC_WIRE) == 2) {  // string / bytes: the last occurrence
                uint32_t poff = 0, plen = 0;
                while (find(fr.mt, q, &i, fr.hi, &it)) { poff = it.poff; plen = it.plen; }
                if (stores) {
                    pdn_st32(row + fxo, plen);
                    for (uint32_t k = 0; k < plen; k++) row[vc + k] = f[poff + k];
                }
                vc += plen;
            } else {
                uint32_t w0 = 0, w1 = 0;
                while (find(fr.mt, q, &i, fr.hi, &it)) pdn_scalar_words(cls, it.wt, it.v, &w0, &w1);
                if (stores) { pdn_st32(row + fxo, w0); if (cls & PC_64) pdn_st32(row + fxo + 4u, w1); }
            }
            continue;
        }
        // repeated: the count word, the elements appended
        if (MAPS && (F.flags & PBN_MAP)) {  // the distinct keys
            const uint32_t n = MapStep::begin(D, f, fr.lo, fr.hi, fr.mt, q, F.msg, maps, &it);
            if (stores) pdn_st32(row + fxo, n);
            if (n) { fr.in_rep = 2; maps++; }
        } else if (F.msg != 0xFF) {
            uint32_t n = 0;
            while (find(fr.mt, q, &i, fr.hi, &it)) n++;
            if (stores) pdn_st32(row + fxo, n);
            if (n) { fr.in_rep = 1; fr.scan = fr.lo; }
        } else if ((cls & PC_WIRE) == 2) {
            uint32_t n = 0;
            while (find(fr.mt, q, &i, fr.hi, &it)) {
                if (stores) {
                    pdn_st32(row + vc, it.plen);
                    for (uint32_t k = 0; k < it.plen; k++) row[vc + 4u + k] = f[it.poff + k];
                }
                vc += 4u + it.plen;
                n++;
            }
            if (stores) pdn_st32(row + fxo, n);
        } else {
            const uint32_t eb = (cls & PC_64) ? 8u : 4u, ewt = cls & PC_WIRE;
            uint32_t n = 0;
            while (find(fr.mt, q, &i, fr.hi, &it)) {
                if (it.wt == 2) {  // packed
                    uint32_t j = it.poff;
                    const uint32_t end = it.poff + it.plen;
                    while (j < end) {
                        uint64_t v = 0;
                        if (ewt == 0) { j += (uint32_t)grpc_varint(f + j, end - j, &v); }
                        else { for (int b = (int)eb - 1; b >= 0; b--) v = v << 8 | f[j + (uint32_t)b]; j += eb; }
                        if (stores) {
                            uint32_t w0, w1;
                            pdn_scalar_words(cls, ewt, v, &w0, &w1);
                            pdn_st32(row + vc, w0);
                            if (eb == 8) pdn_st32(row + vc + 4u, w1);
                        }
                        vc += eb;
                        n++;
                    }
                } else {
                    if (stores) {
                        uint32_t w0, w1;
                        pdn_scalar_words(cls, it.wt, it.v, &w0, &w1);
                        pdn_st32(row + vc, w0);
                        if (eb == 8) pdn_st32(row + vc + 4u, w1);
                    }
                    vc += eb;
                    n++;
                }
            }
            if (stores) pdn_st32(row + fxo, n);
        }
    }
    return vc;
}

// size pass of one frame.  The kernels instantiate it for MAPS == D.maps and PRES == D.presence (one kernel per choice,
// picked on the host: the map-free kernel contains no map code, only the presence kernels presence code); pdn_decode_size
// dispatches at run time.  Validation is the same for both values of PRES: a oneof member of message type is a singular
// message field (sent twice: DEFER), the other members and optional fields are checked like any singular field.  MapStep:
// the map step of the walks, whose entry limit validation applies.
template <bool MAPS, bool PRES = false, class MapStep = PdnSelect>
GOFR_HD PdnRow pdn_decode_size_as(const PbnDesc& D, const uint8_t* f, uint32_t fn) {
    PdnRow r = {GOFR_GRPC_OK, 0};
    if (fn < 5) { r.status = GOFR_GRPC_BAD_LENGTH; return r; }
    if (f[0] == 1) { r.status = GOFR_GRPC_COMPRESSED; return r; }
    if (f[0] != 0) { r.status = GOFR_GRPC_BAD_LENGTH; return r; }
    const uint32_t L = (uint32_t)f[1] << 24 | (uint32_t)f[2] << 16 | (uint32_t)f[3] << 8 | f[4];
    if (L != fn - 5) { r.status = GOFR_GRPC_BAD_LENGTH; return r; }
    r.status = pdn_validate<MAPS, MapStep::kMaxEntries>(D, f, 5, 5 + L);
    if (r.status != GOFR_GRPC_OK) return r;
    r.out_len = (pdn_walk<false, MAPS, PRES, MapStep>(D, f, 5, 5 + L, nullptr) + 3u) & ~3u;
    return r;
}

// emit pass: the row at dst (4-byte aligned: every row is a multiple of 4 bytes long)
template <bool MAPS, bool PRES = false, class MapStep = PdnSelect>
GOFR_HD void pdn_decode_emit_as(const PbnDesc& D, const uint8_t* f, uint32_t fn, const PdnRow r, uint8_t* dst) {
    if (!r.out_len) return;
    uint32_t end = pdn_walk<true, MAPS, PRES, MapStep>(D, f, 5, fn, dst);
    if (MapStep::store()) for (; end < r.out_len; end++) dst[end] = 0;
}

GOFR_HD PdnRow pdn_decode_size(const PbnDesc& D, const uint8_t* f, uint32_t fn) {
    if (D.presence) return pdn_decode_size_as<true, true>(D, f, fn);
    return D.maps ? pdn_decode_size_as<true>(D, f, fn) : pdn_decode_size_as<false>(D, f, fn);
}
GOFR_HD void pdn_decode_emit(const PbnDesc& D, const uint8_t* f, uint32_t fn, const PdnRow r, uint8_t* dst) {
    if (D.presence) pdn_decode_emit_as<true, true>(D, f, fn, r, dst);
    else if (D.maps) pdn_decode_emit_as<true>(D, f, fn, r, dst);
    else pdn_decode_emit_as<false>(D, f, fn, r, dst);
}

}  // namespace gofr
