// engine_internal.h — declarations shared by the host-side translation units of libgofr_b200.
#pragma once
#include <stdint.h>

#include <vector>

struct gofr_table;

void set_last_error(const char* fmt, ...);
const std::vector<uint8_t>& gofr_table_image(const gofr_table* t);

namespace gofr {

// Launch parameters of the fused serve kernel (serve_kernel.cu).
struct ServeParams {
    const void* desc;        // gofr_req_desc[n]
    const void* ids;         // uint8[n][16]
    const uint8_t* arena;
    uint32_t n;
    uint32_t n_tiles;
    const uint8_t* image;    // sealed table in HBM
    uint32_t hot_bytes;
    uint32_t epoch;          // look-back generation (state words from older launches read as "not ready")
    uint8_t* out;
    uint64_t out_cap;
    uint32_t* out_off;       // n + 1
    uint32_t* meta;          // n
    unsigned long long* tile_state;  // n_tiles
    uint32_t* overflow;      // set to 1 if out_cap was too small
    uint32_t in_cap;         // shared-memory staging capacity for request bytes (multiple of 16)
    uint32_t date[8];        // 29-byte IMF-fixdate, zero padded
    uint32_t* bind_scratch;  // n * bind_row_words words (tables with GOFR_H_BIND_ECHO routes), else null
    uint32_t bind_row_words;
    const unsigned long long* chain_pos;  // host-batch path: packed position of the whole batch so far (else null)
    uint32_t slot_bytes;     // 0: packed output (out_off = offsets, n + 1 entries); else response i lives in the slot
                             // out + i * slot_bytes (multiple of 16) and out_off[i] receives its length
    uint32_t debug_flags;    // bit0: skip the look-back (tile_base = tile * tile_total; only valid for fixed-size responses)
};

constexpr int kEpochBits = 24;  // look-back generation field of a tile state word (tile_common.cuh)
constexpr uint32_t kEpochMask = (1u << kEpochBits) - 1;

constexpr int kServeThreads = 128;  // gRPC / request-log kernels: requests per tile = threads per CTA
#ifndef GOFR_SERVE_T
#define GOFR_SERVE_T 128
#endif
#ifndef GOFR_SERVE_CTAS
#define GOFR_SERVE_CTAS 5
#endif
constexpr int kServeT = GOFR_SERVE_T;        // serve kernel: requests per tile = threads per CTA
constexpr int kServeCtas = GOFR_SERVE_CTAS;  // serve kernel: CTAs per SM the register and shared-memory budgets aim at
#ifndef GOFR_SERVE_CTAS_WIDE
#define GOFR_SERVE_CTAS_WIDE 4
#endif
constexpr int kServeCtasWide = GOFR_SERVE_CTAS_WIDE;  // slot layout, "wide" instance: 128 registers per thread (serve_slots_kernel.cu)

// How many response bytes one byte of a request's data section can turn into, at most (ImageHeader::data_expand, set at
// seal): 6 for flat rows (a control character becomes \u00XX); more when the table has programs of the wider data model,
// where a 4-byte element of a slice of structs drags its key literals along (`{"a_long_key":true},`).
template <typename Header>
inline uint32_t image_data_expand(const Header& H) { return H.data_expand > 6u ? H.data_expand : 6u; }

// table_build.cpp: which slot-layout instance suits the sealed table (engine.cu choose_slot_residency)
bool image_wants_wide_slots(const uint8_t* image);

// egress of the host-batch path (egress_kernel.cu)
struct ChunkInfo {
    unsigned long long host_base;  // where this chunk starts in the caller's output buffer
    uint32_t base0;                // = host_base & 15: offset of the chunk inside its device buffer
    uint32_t total;
    uint32_t overflow;
    uint32_t pad;
};
int launch_advance(unsigned long long* chain_pos, const uint32_t* d_off, uint32_t n, uint32_t* d_overflow, ChunkInfo* info,
                   unsigned long long host_cap, void* stream);
int launch_egress(const ChunkInfo* info, const uint8_t* d_out, const uint32_t* d_off, const uint32_t* d_meta, uint32_t n,
                  uint8_t* h_out, uint32_t* h_off, uint32_t* h_meta, unsigned long long* h_status, int grid, void* stream);

struct GrpcParams {
    const uint8_t* in;
    const uint32_t* in_off;
    uint32_t n;
    uint32_t n_tiles;
    uint32_t epoch;
    uint8_t* out;
    uint64_t out_cap;
    uint32_t* out_off;
    uint32_t* meta;
    unsigned long long* tile_state;
    uint32_t* overflow;
};
// Launch parameters of the chunk pack kernel (pack_kernel.cu): the host-batch path of the proto calls packs each record's
// bytes from the codec's output buffer (source A) or, where the selector column says so, from a second buffer (source B)
// into the slot's output buffer, starting at *chain_pos & 15 as the serve kernel does.
struct PackParams {
    const uint8_t* a;        // source A: record i = a[a_off[i] .. a_off[i + 1]), a_cap bytes written at most
    const uint32_t* a_off;
    uint64_t a_cap;
    const uint8_t* b;        // source B (null: none), the same; record i comes from it when sel[i] == GOFR_GRPC_DEFER
    const uint32_t* b_off;
    uint64_t b_cap;
    const uint32_t* sel;
    uint32_t n;
    uint32_t n_tiles;
    uint32_t epoch;
    uint8_t* out;
    uint64_t out_cap;
    uint32_t* out_off;       // n + 1
    unsigned long long* tile_state;
    uint32_t* overflow;
    const unsigned long long* chain_pos;  // pinned-buffer path: packed position of the batch so far (else null)
};

// message types of gofr_proto_encode_nested_device (kernel parameter, by value): up to 8 message types with 48 fields in
// all; fields of a type are consecutive, in ascending field-number order.  Rows use the layout of the wider data model
// (include/gofr_b200.h "Row format"): a singular message field is a presence word + the message's fixed part inline, a
// repeated field a count word with its elements in the variable part.  A map field is laid out (and written) as a repeated
// message field of its entry type; the decoder takes at most kPbnMaxMapEntries entries of one map field in one message
// (selection of the canonical order is quadratic) and answers GOFR_GRPC_DEFER beyond that.
constexpr int kPbnMaxMsgs = 8, kPbnMaxFields = 48, kPbnMaxDepth = 4, kPbnMaxMapEntries = 64;
// The second pass (gofr_proto_decode_nested_deferred_device, proto_nested_deferred_kernel.cu) decodes the frames the first
// pass deferred, one per CTA, with up to kPdnMaxSortedEntries entries of one map field in one message: each active map level
// (at most kPdnMaxMapLevels under kPbnMaxDepth) has a sorted entry list of 16 bytes per entry in dynamic shared memory,
// behind a head of kPdnSortHeadBytes.
constexpr uint32_t kPdnMaxSortedEntries = 4096, kPdnMaxMapLevels = 2, kPdnSortHeadBytes = 144;
constexpr uint32_t pdn_sort_bytes(uint32_t levels) { return kPdnSortHeadBytes + levels * kPdnMaxSortedEntries * 16u; }
enum : uint8_t {
    PBN_REPEATED = 1u,  // a count word in the fixed part, the elements in the variable part (map fields too)
    PBN_MAP = 2u,       // a map field (GOFR_PB_MAP; always with PBN_REPEATED): entries in ascending key order
    PBN_ENTRY = 4u,     // the key or value of a map entry type: written even at its zero value, a value message always
    PBN_SIGNED = 8u,    // an entry's key of a signed integer type (key order)
    PBN_PRESENCE = 16u, // a singular scalar / string / bytes with explicit presence (proto3 optional, a oneof member): a
                        // presence word 0 / 1 before its value words; written when set, even at its zero value
    PBN_ONEOF = 0xE0u,  // the oneof group (1..7) of a member, << PBN_ONEOF_SHIFT; members of type message have this alone
};
constexpr int PBN_ONEOF_SHIFT = 5;
struct PbnField {
    uint32_t tag;        // number << 3 | wire type (2 for messages and for packed repeated scalars)
    uint8_t cls;         // PC_* bits of the scalar type; 0 for a message
    uint8_t flags;       // PBN_* bits
    uint8_t msg;         // message type index (type GOFR_PB_MESSAGE), the entry type of a map field, else 0xFF
    uint8_t fixed_words; // words the field owns in the fixed part of its message
};
struct PbnDesc {
    uint8_t n_msgs;
    uint8_t presence;  // some field has PBN_PRESENCE or PBN_ONEOF bits: the *_presence kernels run it (maps or not)
    uint16_t maps;  // the description has map fields: the *_maps kernels run it (map-free types keep the plain kernels)
    uint32_t root;
    uint16_t first[kPbnMaxMsgs], count[kPbnMaxMsgs], fixed_words[kPbnMaxMsgs];
    PbnField f[kPbnMaxFields];
};

// message type of gofr_proto_encode_device (kernel parameter, by value); 32 = GOFR_PROTO_MAX_FIELDS
struct ProtoSchema {
    uint32_t n_fields;
    uint32_t fixed_bytes;  // size of a row's fixed part
    uint32_t tag[32];      // number << 3 | wire type
    uint8_t cls[32];       // PC_* bits derived from the GOFR_PB_* type once, on the host (proto_class below)
};
#if defined(__CUDACC__)
#define GOFR_INTERNAL_HD __host__ __device__ inline
#else
#define GOFR_INTERNAL_HD inline
#endif
GOFR_INTERNAL_HD bool proto_is64(uint32_t t) {  // GOFR_PB_DOUBLE, INT64, UINT64, FIXED64, SFIXED64, SINT64
    return t == 1 || t == 3 || t == 4 || t == 6 || t == 16 || t == 18;
}
GOFR_INTERNAL_HD uint32_t proto_wire(uint32_t t) {
    if (t == 9 || t == 12) return 2;             // STRING, BYTES
    if (t == 1 || t == 6 || t == 16) return 1;   // DOUBLE, FIXED64, SFIXED64
    if (t == 2 || t == 7 || t == 15) return 5;   // FLOAT, FIXED32, SFIXED32
    return 0;
}
// What the per-message loops need to know about a field type, decided once per call on the host: the device tests bits
// instead of walking compare chains per field per message.
enum : uint32_t {
    PC_WIRE = 7u,       // wire type (0 varint, 1 fixed64, 2 length-delimited, 5 fixed32)
    PC_64 = 8u,         // two row words
    PC_ZIGZAG = 16u,    // sint32 / sint64
    PC_SIGNEXT = 32u,   // int32 / enum: negative values are sign-extended to 64 bits
    PC_UTF8 = 64u,      // string: must be valid UTF-8
    PC_BOOL = 128u,
};
GOFR_INTERNAL_HD uint32_t proto_class(uint32_t t) {
    uint32_t c = proto_wire(t);
    if (proto_is64(t)) c |= PC_64;
    if (t == 17 || t == 18) c |= PC_ZIGZAG;   // SINT32, SINT64
    if (t == 5 || t == 14) c |= PC_SIGNEXT;   // INT32, ENUM
    if (t == 9) c |= PC_UTF8;                 // STRING
    if (t == 8) c |= PC_BOOL;                 // BOOL
    return c;
}

constexpr int kRouteThreads = 256;  // route_kernel.cu: requests per CTA, one per thread
struct RouteParams {
    const void* desc;
    const uint8_t* arena;
    uint32_t n;
    const uint8_t* image;
    uint32_t hot_bytes;
    uint32_t* meta;   // n: status | route << 16
    uint32_t* vars;   // n * kMaxVars: off | len << 16
};

constexpr int kBindThreads = 128;   // bind_kernel.cu
struct BindParams {
    const void* desc;
    const uint8_t* arena;
    uint32_t n;
    const uint8_t* image;
    uint32_t hot_bytes;
    uint32_t schema_idx;
    uint8_t* out;          // n * slot_bytes
    uint32_t slot_bytes;
    uint32_t* len;         // n
    uint32_t* status;      // n
};

struct HttpParams {
    const uint8_t* raw;
    const uint32_t* raw_off;  // n + 1
    uint32_t n;
    uint32_t n_tiles;
    void* desc;               // gofr_req_desc[n]
    uint8_t* arena;           // as large as raw (+16)
    uint32_t* status;         // n
    unsigned long long* spans;  // n * GOFR_HTTP_SPANS
};

// http_frame_kernel.cu: a packed-output kernel whose output is the record column (words, not bytes)
struct HttpFrameParams {
    const uint8_t* buf;
    const uint32_t* buf_off;  // n + 1
    uint32_t n;               // connections
    uint32_t n_tiles;
    uint32_t epoch;
    uint8_t* out;             // d_rec_off: out_cap + 1 words
    uint64_t out_cap;         // records
    uint32_t* out_off;        // d_first: n + 1
    uint32_t* consumed;       // n
    uint32_t* status;         // n
    unsigned long long* tile_state;
    uint32_t* overflow;
};

// conn_kernel.cu: gofr_conn_batch_submit's compact step, a packed-output kernel over connections whose output is the
// compacted request columns (a connection's length is its number of whole requests)
struct ConnParams {
    const uint32_t* first;        // n + 1: the framer's record column of the chunk (d_first)
    const uint32_t* conn_status;  // n
    const uint32_t* rec_off;      // the framer's record starts (absolute buffer offsets)
    const void* desc_in;          // gofr_req_desc per record (the request-head kernel's output)
    uint64_t trace_seed;
    const uint64_t* trace_key;    // n: the connections' trace keys (gofr_conn_batch_respond_ex), or null: keys of (trace_seed, c)
    uint32_t conn0;               // the batch index of the chunk's first connection (trace ids)
    uint32_t req0;                // the batch index of the chunk's first request (req_first)
    uint32_t n;                   // connections
    uint32_t n_tiles;
    uint32_t epoch;
    uint8_t* out;                 // gofr_req_desc per request (out_cap requests)
    uint64_t out_cap;
    uint32_t* out_off;            // req_first: n + 1, rebased by req0
    uint32_t* req_at;             // per request
    uint8_t* ids;                 // 16 bytes per request
    unsigned long long* tile_state;
    uint32_t* overflow;
};

// conn_log_kernel.cu: gofr_conn_batch_submit_log's gather step, a packed-output kernel over connections whose output is the
// line column (a connection's length is its number of logged requests): per line a gofr_log_desc, its trace id and its
// batch request index, and the line's five strings in the log arena (conn_log_device.cuh)
struct ConnLogParams {
    const uint32_t* first;               // n + 1: the framer's record column of the chunk
    const uint32_t* conn_status;         // n
    const uint32_t* req_first;           // n + 1: the compact step's output (batch request indices)
    const uint32_t* rec_off;             // the framer's record starts (absolute buffer offsets)
    const unsigned long long* spans;     // per record: the request-head kernel's spans (absolute buffer offsets)
    const uint32_t* meta;                // per request of the chunk: the serve kernel's meta
    const uint8_t* ids;                  // per request of the chunk: 16 trace id bytes
    const uint8_t* buf;                  // the staged chunk, addressed by absolute buffer offsets
    const uint8_t* remote;               // the staged remote strings, addressed by absolute remote offsets
    const uint32_t* remote_off;          // n + 1
    const int64_t* start_ns;             // n
    int64_t log_ns;
    int32_t tz_offset_s;
    uint32_t alo;                        // the chunk's first staged buffer byte
    uint32_t remote_max;                 // R: the chunk's longest remote string
    uint32_t req0;                       // the batch index of the chunk's first request
    uint32_t n;                          // connections
    uint32_t n_tiles;
    uint32_t epoch;
    uint8_t* out;                        // gofr_log_desc per line (out_cap lines)
    uint64_t out_cap;
    uint32_t* out_off;                   // n + 1: the connection's first line in the chunk
    uint8_t* line_ids;                   // 16 bytes per line
    uint32_t* line_req;                  // per line
    uint8_t* arena;                      // the log arena
    unsigned long long* tile_state;
    uint32_t* overflow;
};

// conn_result_kernel.cu: gofr_conn_batch_respond's splice step, a packed-output kernel over the requests of a chunk whose
// output is the spliced arena (conn_result_device.cuh): request i's decoded path | query | pad4 | data section, its data
// section the closure's record rec[rec_off[i] .. rec_off[i + 1]) when that is not empty, else its own body
struct ConnResultParams {
    void* desc;                 // gofr_req_desc per request (parse-arena offsets), rewritten in place to spliced-arena ones
    const uint8_t* arena;       // the parse arena, addressed by absolute buffer offsets
    const uint8_t* rec;         // the chunk's records, addressed by the caller's record offsets
    const uint32_t* rec_off;    // n + 1: the caller's rec_off from the chunk's first request on
    uint32_t n;
    uint32_t n_tiles;
    uint32_t epoch;
    uint8_t* out;               // the spliced arena
    uint64_t out_cap;
    uint32_t* out_off;          // n + 1: request i's spliced form starts at out_off[i] (a multiple of 4)
    unsigned long long* tile_state;
    uint32_t* overflow;
};

struct LogParams {
    const void* desc;   // gofr_log_desc[n]
    const void* ids;    // n * 16 trace id bytes
    const uint8_t* arena;
    uint32_t n;
    uint32_t n_tiles;
    uint32_t epoch;
    uint8_t* out;
    uint64_t out_cap;
    uint32_t* out_off;
    unsigned long long* tile_state;
    uint32_t* overflow;
};

}  // namespace gofr
