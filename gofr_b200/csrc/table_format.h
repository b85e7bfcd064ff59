// table_format.h — binary layout of the sealed route/schema table ("image").
//
// The image is position independent (offsets from its base), so the same bytes are (a) broadcast from rank 0 to all
// ranks, (b) copied once to HBM, and (c) copied by every CTA into shared memory at kernel start (the "hot" part).
// It is the compiled form of what the reference keeps as a []*mux.Route plus closures
// (pkg/gofr/http/router.go:30-33, pkg/gofr/gofr.go:171-177): routes in registration order (= match priority), each
// pointing at a response *program* — a list of ops the serve kernel interprets to produce the exact bytes that
// handler + Responder.Respond + encoding/json + net/http framing produce in the reference.
#pragma once
#include <stdint.h>

namespace gofr {

constexpr uint32_t kMagic = 0x52464F47u;  // "GOFR"
constexpr uint32_t kImageVersion = 17;
constexpr uint32_t kMaxHotBytes = 40 * 1024;  // shared-memory budget for the table
constexpr int kMaxVars = 8;                   // variables per route template
constexpr int kMaxPieces = 16;                // literal + atom pieces per route template
constexpr int kMaxValueDepth = 8;            // struct nesting the generic value encoder walks (its frame stack)
constexpr int kMaxFields = 32;                // struct fields per schema

struct ImageHeader {  // 160 B
    uint32_t magic, version;
    uint32_t frame_mode;
    uint32_t n_routes, n_pieces, n_progs, n_ops, n_schemas;
    uint32_t routes_off, pieces_off, progs_off, ops_off, schemas_off, lits_off;
    uint32_t hot_bytes;    // [0, hot_bytes) is copied to shared memory
    uint32_t cold_off;     // file blobs: read from global memory only
    uint32_t total_bytes;
    uint16_t prog_301, prog_301_head, prog_404, prog_405, prog_405_head, prog_options, prog_panic, pad0;
    uint32_t max_fixed_len;  // largest fixed (literal) part of any program, for capacity estimates
    uint32_t has_catchall;
    // literal-route dispatch: hash(path) → first literal route of a chain (RouteRec.next_lit), in registration order
    uint32_t hash_off;       // uint16[1 << hash_bits], 0xFFFF = empty
    uint32_t hash_bits;
    uint32_t tmpl_off;       // uint16[n_tmpl]: live routes that are not plain literals (templates, prefixes), in order
    uint32_t n_tmpl;
    uint32_t last_method_off;  // uint16[16]: 1 + index of the last live route registered for that method, 0 = none
    uint32_t fixups_off;     // uint32[n_fixups]: literal-pool offsets of 29-byte Date placeholders
    uint32_t n_fixups;
    uint32_t bind_row_words;  // words of per-request Bind scratch (0: no GOFR_H_BIND_ECHO route)
    uint32_t tmplkey_off;    // uint32[4][n_tmpl]: {key0, key1, mask0, mask1} — the first <= 8 literal bytes of each template;
                             // a path whose first bytes differ cannot match it (checked inline before template_match)
    // keyed template dispatch: templates whose leading literal is >= 8 bytes are reached through a hash of those 8
    // bytes (chained through RouteRec.next_lit in registration order); tmpl_off lists only the others
    uint32_t thash_off;      // uint16[1 << thash_bits], 0xFFFF = empty
    uint32_t thash_bits;
    uint32_t checksum;       // FNV-1a over the whole image with this field zero: set at seal, checked by deserialize (the
                             // image travels between ranks); never read on the device
    uint32_t fast_off;       // FastRec[n_progs]: how the slot-layout kernel emits each program (templates + tail ops)
    uint32_t rawprog_off;    // uint16[n_routes][9]: GOFR_H_RESULT routes, programs of the response.Raw outcomes
                             // [(RAW_DATA, RAW_STRING, RAW_NIL) x (200, 500, 404)], 0xFFFF = none
    uint32_t schema_ids_off; // uint32[n_schemas]: the caller's schema ids in table order (gofr_bind_device looks one up)
    uint32_t data_expand;    // response bytes one byte of a request's data section can become, at most (engine_internal.h
                             // image_data_expand)
    uint32_t pad3;
};
static_assert(sizeof(ImageHeader) == 160, "ImageHeader layout");

enum RouteFlags : uint8_t {
    RF_PREFIX = 1,   // PathPrefix: regexp has no trailing '$'
    RF_DEAD = 2,     // mux route.err != nil: never matches
    RF_LITERAL = 4,  // no variables: one word-wise compare
    RF_DEFAULT = 8,  // appended by gofr_table_add_default_routes (health, favicon, catch-all): not the application's traffic
};

struct RouteRec {  // 32 B
    uint8_t method;  // GOFR_M_* or 255
    uint8_t flags;
    uint8_t n_pieces;
    uint8_t hkind;  // GOFR_H_*
    uint16_t first_piece;
    uint16_t schema;    // index into schemas
    uint16_t prog_ok;   // program of the normal outcome (0xFFFF: none — GOFR_H_HOST)
    uint16_t prog_err;  // GOFR_H_BIND_ECHO: the 500 program
    uint32_t lit_off;   // RF_LITERAL: the whole pattern, 4-byte aligned in the literal pool
    uint16_t lit_len;
    uint16_t key_len;   // GOFR_H_PARAM_FORMAT: query key
    uint32_t key_off;
    uint32_t def_off;   // default value, already JSON-escaped
    uint16_t def_len;
    uint16_t next_lit;  // next route in the same hash bucket (literal routes: hash of the path; keyed templates: hash of
                        // their first 8 literal bytes), registration order, 0xFFFF = end
};
static_assert(sizeof(RouteRec) == 32, "RouteRec layout");

enum PieceVarFlags : uint8_t { PV_FIRST = 1, PV_LAST = 2 };  // first / last atom of its variable
struct PieceRec {  // 48 B: literal, then (optionally) an atom of a variable = class repeated min_rep..max_rep times, greedy
    uint32_t lit_off;
    uint16_t lit_len;
    uint8_t has_var;
    uint8_t min_rep;
    uint32_t cls[8];  // 256-bit membership
    uint8_t max_rep;    // 0 = unbounded
    uint8_t var_idx;    // the variable (mux.Vars, template order) this atom is part of; a {name:regexp} may be several
                        // consecutive atoms ([a-z]+\.[a-z]{2,4}), all but the first with an empty literal
    uint8_t var_flags;  // PV_*
    uint8_t pad0;
    uint32_t pad;
};
static_assert(sizeof(PieceRec) == 48, "PieceRec layout");

enum OpCode : uint8_t {
    OP_LIT = 0,     // literal bytes lits[off .. off+len)
    OP_HEXID = 1,   // 32 lower-case hex chars of the request's trace id   (middleware/logger.go:46-47)
    OP_CLEN = 3,    // decimal length of the body                           (net/http Content-Length)
    OP_I64 = 4,     // strconv.AppendInt of a row field; off = word index in the row
    OP_I32 = 5,
    OP_BOOL = 6,    // true / false
    OP_STR = 7,     // encoding/json-escaped string contents (quotes live in the neighbouring literals);
                    // off = word index of its length, arg = ordinal among the string fields
    OP_PARAM = 8,   // escaped query value of the route's key, or the default  (request.go:28-30)
    OP_LOCATION = 9,  // url.String() of the cleaned URL                        (mux 301)
    OP_ERRMSG = 10,   // escaped err.Error() of a failed Bind                   (responder.go:43-57)
    OP_BLOB = 11,     // raw bytes from the cold section                        (response.File)
    OP_BSTR = 13,     // string field of a Bind span row: off = word index of (offset into the body, length | escaped<<31)
    OP_F64 = 14,      // float64 struct field: encoding/json floatEncoder text (float_device.cuh); off = word index of the bits
    OP_VALUE = 15,    // a field the generic encoder walks (pointer, slice, map, nested struct with omitempty members, bare
                      // schema): aux = schema index, arg = field index, off = word index of the field's fixed words;
                      // consumes the field's share of the row's variable part (serve_device.cuh value_encode)
    OP_KEY = 12,      // struct member key with dynamic comma / omitempty: emits [","] + lits[off..off+len) unless the
                      // field (arg) is empty and flagged; used only for schemas that have an omitempty field
};

// Value ops (everything except OP_LIT / OP_KEY / OP_BLOB) can carry a literal PREFIX: lits[aux .. aux+len) is emitted
// right before the op's own bytes (the builder folds `"name":"`-style literals into the field op that follows, which
// halves the interpreter's trip count).  The prefix is part of the program's fixed byte count.
enum OpFlags : uint8_t {
    OPF_BODY = 1,       // op belongs to the response body (counts toward Content-Length; dropped for HEAD)
    OPF_OMITEMPTY = 2,  // OP_KEY: skip key and value when the field is the zero value
    OPF_VALUE_OF_KEY = 4,  // value op governed by the preceding OP_KEY
};

struct Op {  // 16 B (one LDS.128)
    uint8_t code;
    uint8_t arg;
    uint8_t flags;
    uint8_t kind;  // OP_KEY: field kind (low 4 bits) and GOFR_C_* container (high 4) for the emptiness test
    uint32_t len;
    uint32_t off;
    uint32_t aux;
};
static_assert(sizeof(Op) == 16, "Op layout");

struct ProgRec {  // 32 B
    uint16_t first_op;
    uint16_t n_ops;
    uint16_t status;     // HTTP status code
    uint16_t flags;      // PF_*
    uint32_t hdr_fixed;  // sum of the fixed-length header bytes (literals, HEXID)
    uint32_t body_fixed; // sum of the fixed-length body bytes
    uint16_t first_dyn;  // the ops whose length depends on the request, in order: all the size pass has to visit
    uint16_t n_dyn;
    uint16_t n_hdr_ops;  // ops before the first body op (body ops come last): all a HEAD response emits
    uint16_t row_words;  // nonzero: the row's fixed part is this many words whatever the route's schema (GOFR_H_RESULT errors)
    uint8_t shape_class;  // 1..30: programs with the same op-code sequence (same control flow in run_prog) share a class;
                          // the kernel groups a tile's requests by class so that warps run few distinct programs
    uint8_t pad1[3];
    uint16_t encfail;     // program that answers when a float of this one turns out to be NaN / ±Inf (json.Encoder.Encode
                          // fails after Respond wrote the status: same headers, no body); 0xFFFF: cannot happen
    uint16_t pad2;
};
static_assert(sizeof(ProgRec) == 32, "ProgRec layout");

enum ProgFlags : uint16_t {
    PF_HAS_CLEN = 1,
    PF_DYNAMIC = 2,   // has at least one variable-length op besides CLEN
    PF_NEEDS_ROW = 4,
    PF_BIND = 8,      // the row is the Bind span row in scratch (bind_device.cuh), not the request's data section
    PF_FAST = 16,     // only literals, plain values and struct keys (LIT, HEXID, CLEN, I64, I32, BOOL, STR, BSTR, PARAM, KEY):
                      // eligible for the slot-layout fast path (FastRec) when the request has no escapes
    PF_VALUES = 32,   // has OP_F64 / OP_VALUE ops: runs through the VALUES instance of the interpreter (serve_device.cuh run_prog)
};

// Slot layout fast path (serve_device.cuh emit_fast).  A response owns a 16-byte aligned slot, so every byte of the
// response whose POSITION does not depend on the request — the status line and the sorted header block up to the first
// variable-length value, i.e. up to the Content-Length digits — can be prepared at seal time exactly as it will lie in the
// slot: a dst-aligned TEMPLATE in the literal pool (Date patched at kernel start like every literal, 32 placeholder bytes
// where the trace id goes).  The kernel copies it with aligned 16-byte loads and stores (no funnel shifts, no staging),
// patches the hex characters in, and interprets only the ops after it ("tail").  Programs without any variable-length
// value (static bodies, 404, OPTIONS ...) are template only: Content-Length is folded at seal time and the last window
// is zero padded like the slot layout wants it.
struct FastRec {  // 16 B
    uint32_t tmpl_off;     // literal-pool offset of the template, 16-byte aligned
    uint8_t tmpl_windows;  // template length in 16-byte windows; 0: no template (tail = whole program)
    uint8_t flags;         // FR_*
    uint16_t hex_pos;      // byte offset of the 32 hex characters inside the template; 0xFFFF: none
    uint16_t tail_op;      // absolute index of the first tail op (a private copy of the program's remaining ops: the first
                           // one has the bytes the template already covers cut off its literal)
    uint16_t n_tail_ops;
    uint32_t tmpl_bytes;   // response bytes the template covers (= 16 * tmpl_windows, less the zero padding of a
                           // template-only program)
};
static_assert(sizeof(FastRec) == 16, "FastRec layout");
enum FastFlags : uint8_t {
    FR_BIND = 1,       // PF_BIND
    FR_COMPLETE = 2,   // template only: nothing left to interpret
};

enum SchemaFlags : uint16_t {
    SF_FLAT = 1,  // int / bool / string fields by value only (what the op programs of round 1 take)
    SF_BARE = 2,  // one field standing for its own type (GOFR_FIELD_BARE)
    SF_BINDABLE = 4,  // scalar and string fields by value only, float64 included: what Bind takes (bind_device.cuh)
};
struct SchemaRec {  // 16 B + per-field table
    uint16_t n_fields;
    uint16_t n_strings;
    uint16_t fixed_words;  // words in the fixed part of a row
    uint16_t flags;        // SF_*
    uint32_t fields_off;  // FieldRec[n_fields]
    uint32_t type_off;    // reflect.Type.String(), for Bind error text
};

struct FieldRec {  // 32 B
    uint8_t kind;  // GOFR_F_*
    uint8_t omitempty;
    uint16_t word;      // word index in the fixed part of its struct
    uint16_t name_len;  // JSON key name (for Bind)
    uint16_t str_ord;   // ordinal among string fields
    uint32_t name_off;
    uint32_t fold_off;  // simple-folded (lower-cased) name
    uint16_t type_len;  // Go type name for error text ("int64", "string", ...)
    uint8_t container;  // GOFR_C_*
    uint8_t n_words;    // words the field owns in the fixed part (nested structs inline, pointers + 1)
    uint32_t type_off;
    uint32_t key_off;   // `"name":` as encoding/json writes it (escaped), for the generic encoder
    uint16_t key_len;
    uint16_t elem;      // GOFR_F_STRUCT: schema index of the struct type
};
static_assert(sizeof(FieldRec) == 32, "FieldRec layout");

// Hash of a path for the literal-route table: word-wise FNV-style over the 4-byte aligned, zero-padded path.
// The device computes it from the request bytes, the builder from the pattern; both use this function.
#if defined(__CUDACC__)
__host__ __device__
#endif
inline uint32_t path_hash_step(uint32_t h, uint32_t w) { return (h ^ w) * 0x9E3779B1u; }

}  // namespace gofr
