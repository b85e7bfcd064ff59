/*
 * gofr_b200.h — C ABI of the H100-native GoFr request hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference (JigarJoshi04/gofr) has no FFI of its own: its seams
 * are in-process Go interfaces.  Each entry point below names the reference interface it stands in for, so a Go shim
 * (see INTEGRATION.md, go/gofrb200/) binds them one-to-one over cgo:
 *
 *   reference interface (file:line)                              replaced by
 *   ------------------------------------------------------------ ---------------------------------------------
 *   http.NewRouter                pkg/gofr/http/router.go:17-28    gofr_table_create
 *   Router.Add / App.add          pkg/gofr/http/router.go:30-33,   gofr_table_add_route
 *                                 pkg/gofr/gofr.go:171-177
 *   App.Run default routes        pkg/gofr/gofr.go:102-107         gofr_table_add_default_routes
 *   (route table frozen at Run)   pkg/gofr/gofr.go:90-126          gofr_table_seal / _serialize / _deserialize
 *   mux.Router.ServeHTTP → middleware chain → handler.ServeHTTP → Responder.Respond → net/http framing
 *                                 pkg/gofr/http/router.go:14,
 *                                 pkg/gofr/http/middleware/{tracer,logger,cors}.go,
 *                                 pkg/gofr/handler.go:32-36,
 *                                 pkg/gofr/http/responder.go:19-41 gofr_serve_device[_slots] / gofr_batch_submit+wait
 *   Request.Param / Bind          pkg/gofr/http/request.go:28-47   (fused into the serve kernel per handler kind)
 *   _Hello_SayHello_Handler       examples/grpc-server/grpc/
 *                                 hello_grpc.pb.go:73-89           gofr_grpc_hello_device
 *   dec(in) / proto.Marshal of any flat proto3 message type (the codec grpc-go calls around a unary handler)
 *                                 hello_grpc.pb.go:73-89           gofr_proto_decode_device / gofr_proto_encode_device
 *   encoding.Codec.Unmarshal / Marshal once per message on the RPC's goroutine
 *                                 hello_grpc.pb.go:73-89           gofr_proto_frontend_call (batches the concurrent callers)
 *   Router.Match + mux.Vars (routing only, closures on the host)
 *                                 pkg/gofr/http/router.go:14,30-33 gofr_route_device / gofr_batch_route
 *   router.ServeHTTP per request under net/http's conn goroutine
 *                                 pkg/gofr/httpServer.go:29-33     gofr_frontend_serve (batches the concurrent callers)
 *   net/http readRequest + url.ParseRequestURI (stdlib, reached from pkg/gofr/httpServer.go:29-33)
 *                                                                  gofr_http_parse_device
 *   middleware.Logging's RequestLog line → logger.Log
 *                                 pkg/gofr/http/middleware/logger.go:24-33,41-84,
 *                                 pkg/gofr/logging/logger.go:37-74 gofr_requestlog_device
 *
 * Conventions (mirroring the reference's "log and continue", responder.go:29,40): plain C types only, integer status
 * codes, never abort; per-request outcomes are reported in the response meta column; the table is immutable after
 * seal (the reference never mutates routes after Run()); no callbacks into the caller from CUDA threads (cgo-safe).
 * Values that are non-deterministic in the reference are INPUTS here: the 16-byte OTel trace id per request
 * (middleware/logger.go:46-47) and the IMF-fixdate `Date` string per batch (net/http).
 * Device-resident INPUT buffers of variable-length bytes (d_arena, d_in of frames, d_rows, d_raw, the strings of log
 * records): 16-byte aligned, and the allocation extends at least 16 bytes past the last byte an offset names — tiles are
 * staged in 16-byte units and the copy loops read whole aligned words; the bytes there are never looked at.  The host-buffer
 * entry points (gofr_batch_*) stage their inputs themselves and ask nothing of the kind.
 */
#ifndef GOFR_B200_H
#define GOFR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GOFR_ABI_VERSION 1

/* ---- status codes (returned by every entry point) ---- */
enum {
    GOFR_OK = 0,
    GOFR_ERR_INVALID = 1,      /* bad argument */
    GOFR_ERR_UNSUPPORTED = 2,  /* e.g. a {var:regexp} outside the supported class, a float field */
    GOFR_ERR_NOMEM = 3,
    GOFR_ERR_CUDA = 4,         /* a CUDA runtime call failed; gofr_last_error() has the text */
    GOFR_ERR_SEALED = 5,       /* mutation after seal */
    GOFR_ERR_NOT_SEALED = 6,
    GOFR_ERR_CAPACITY = 7,     /* batch / arena / output larger than the engine was created for */
    GOFR_ERR_NO_DEVICE = 8     /* no CUDA device: the product path has no CPU fallback, by design */
};

/* ---- request methods.  mux's methodMatcher compares exact upper-case strings; the shim maps the exact strings
 *      below and sends everything else (including lower-case spellings) as GOFR_M_OTHER, which matches no
 *      method-restricted route. ---- */
enum {
    GOFR_M_GET = 0, GOFR_M_HEAD = 1, GOFR_M_POST = 2, GOFR_M_PUT = 3, GOFR_M_PATCH = 4, GOFR_M_DELETE = 5,
    GOFR_M_CONNECT = 6, GOFR_M_OPTIONS = 7, GOFR_M_TRACE = 8, GOFR_M_OTHER = 15,
    GOFR_M_ANY = 255 /* registration only: no method matcher (PathPrefix("/") catch-all, gofr.go:104) */
};

/* ---- framing modes (SURVEY.md §8c Q1) ---- */
enum {
    GOFR_FRAME_WIRE = 0,     /* what net/http 1.21 puts on the socket: Responder sets Content-type AFTER WriteHeader
                                (responder.go:21 vs :39) so the type is sniffed: text/plain; charset=utf-8 */
    GOFR_FRAME_INTENDED = 1, /* what the reference's tests observe through the live recorder map
                                (responder_test.go:28, gofr_test.go:104): Content-Type: application/json */
    GOFR_FRAME_BODY = 2      /* response body only (unambiguous in both modes) */
};

/* ---- declarative handler kinds.  User handlers are arbitrary Go closures (handler.go:12) and cannot run on the
 *      GPU; the kinds below are the closures the reference's examples/tests use, expressed as data so the whole
 *      request can be served by one fused kernel.  GOFR_H_HOST is the general case: the GPU routes, the host runs
 *      the closure, the GPU encodes (two launches). ---- */
enum {
    GOFR_H_HOST = 0,          /* arbitrary closure on the host; serve emits nothing and reports route_id */
    GOFR_H_STATIC_STRING = 1, /* return s0, nil                       gofr_test.go:62-64 */
    GOFR_H_STATIC_ERROR = 2,  /* return nil, errors.New(s0)           examples/http-server/main.go:41-43 */
    GOFR_H_NIL = 3,           /* return nil, nil                      handler_test.go:29 */
    GOFR_H_PARAM_FORMAT = 4,  /* v := c.Param(s0); if v == "" { v = s1 }; return s2 + v + s3, nil
                                 examples/http-server/main.go:31-39, gofr_test.go:80-82 */
    GOFR_H_ROW = 5,           /* return <struct of schema>, nil; field values arrive in the request's data section */
    GOFR_H_BIND_ECHO = 6,     /* var v T; if err := c.Bind(&v); err != nil { return nil, err }; return v, nil
                                 T: a flat struct of int / int32 / int64 / float64 / bool / string fields.  A float64 member
                                 gets strconv.ParseFloat's correctly rounded value through ParseFloat's own fast steps (the
                                 exact cases, then Eisel-Lemire; sure overflows → the UnmarshalTypeError Go reports, sure
                                 underflows → 0); a request with a literal Go needs its big-decimal slow path for (an exact
                                 half-way case, a subnormal, 1e308-ish) comes back with status 0 ("run on the host"), like a
                                 body nested deeper than 64 levels */
    GOFR_H_HEALTH = 7,        /* healthHandler with no datasources: map{} handler.go:38-40, container.go:26-38 */
    GOFR_H_MISSING_FILE = 8,  /* catchAllHandler: return nil, http.ErrMissingFile      handler.go:51-53 */
    GOFR_H_FILE = 9,          /* return response.File{Content: blob, ContentType: s0}   handler.go:42-49 */
    GOFR_H_PANIC = 10,        /* handler panics; middleware.panicRecovery answers       middleware/logger.go:91-114 */
    GOFR_H_PATHPARAM_FORMAT = 11, /* v := c.PathParam(s0); return s2 + v + s3, nil         pkg/gofr/http/request.go:36-38 */
    GOFR_H_RESULT = 12        /* stage 2 of the split API: the closure already ran on the host (after gofr_route_device);
                                 its (data, err) arrives in the request's data section and Responder.Respond runs here
                                 (pkg/gofr/http/responder.go:19-62).  Data section: one LE u32 outcome word, then
                                   GOFR_RESULT_DATA     a row of the route's schema (as for GOFR_H_ROW)      → 200 {"data":{…}}
                                   GOFR_RESULT_ERROR    u32 length + err.Error() bytes                      → 500 {"error":{"message":…}}
                                   GOFR_RESULT_NIL      nothing                                             → 200 {}
                                   GOFR_RESULT_MISSING  u32 length + message; errors.Is(err, http.ErrMissingFile) → 404
                                   GOFR_RESULT_BOTH     (data, err) both non-nil: one row whose first field is the message
                                                        string followed by the schema's fields (length word + fixed
                                                        words, then message bytes + string bytes) → 500 {"error":…,"data":…}
                                   GOFR_RESULT_STRING   data is a Go string (what most of the reference's example handlers
                                                        return, examples/http-server/main.go:29-41): u32 length + bytes
                                                        → 200 {"data":"…"}  (the route needs no schema for this outcome)
                                 The closure returned a response.Raw (pkg/gofr/http/response/raw.go:3-5): Respond encodes
                                 Raw.Data bare, without the {"error":…,"data":…} envelope (responder.go:24-26); the error, if
                                 any, only picks the status code (written at responder.go:21 before the type switch):
                                   GOFR_RESULT_RAW_DATA    a row of the route's schema                      → {…}\n
                                   GOFR_RESULT_RAW_STRING  u32 length + bytes                               → "…"\n
                                   GOFR_RESULT_RAW_NIL     nothing (Raw{}: Data is a nil interface)         → null\n
                                 with the error in bits 8..15 of the outcome word: GOFR_RESULT_RAW_OK (err == nil, 200),
                                 GOFR_RESULT_RAW_ERR (500), GOFR_RESULT_RAW_MISSING (errors.Is(err, http.ErrMissingFile), 404);
                                 e.g. GOFR_RESULT_RAW_STRING | GOFR_RESULT_RAW_ERR << 8. */
};
enum { GOFR_RESULT_DATA = 0, GOFR_RESULT_ERROR = 1, GOFR_RESULT_NIL = 2, GOFR_RESULT_MISSING = 3, GOFR_RESULT_BOTH = 4,
       GOFR_RESULT_STRING = 5, GOFR_RESULT_RAW_DATA = 6, GOFR_RESULT_RAW_STRING = 7, GOFR_RESULT_RAW_NIL = 8 };
enum { GOFR_RESULT_RAW_OK = 0, GOFR_RESULT_RAW_ERR = 1, GOFR_RESULT_RAW_MISSING = 2 };

/* ---- struct field kinds for response / Bind schemas ---- */
enum {
    GOFR_F_INT64 = 1,
    GOFR_F_INT32 = 2,
    GOFR_F_BOOL = 3,
    GOFR_F_STRING = 4,
    GOFR_F_INT = 5,    /* Go int (64-bit); only the type name in Bind error text differs from INT64 */
    GOFR_F_FLOAT64 = 6, /* encoding/json floatEncoder: shortest digits that round-trip, 'e' form below 1e-6 and from 1e21,
                           "e-0X" written "e-X"; NaN / ±Inf make Encode fail: the response keeps its status and headers
                           and has no body (responder.go:40 drops the error).  Bind schemas: see GOFR_H_BIND_ECHO */
    GOFR_F_STRUCT = 7,  /* a struct value of the schema `elem_schema`                            response schemas only */
    GOFR_F_UINT64 = 8,  /* uint64 / uint / uintptr: two words, unsigned decimal (narrower unsigned types fit INT64, int8 /
                           int16 fit INT32: the text is the same)                               response schemas only */
    GOFR_F_BYTES = 9,   /* []byte: encoding/json writes base64.StdEncoding with padding in quotes, null when nil.  Row:
                           one fixed word = the byte length (GOFR_NIL_COUNT: nil), the bytes in the variable part;
                           as an element E([]byte) = u32 length (GOFR_NIL_COUNT: nil) + bytes     response schemas only */
    GOFR_F_FLOAT32 = 10, /* float32: one word (IEEE-754 bits), the shortest digits that identify the FLOAT32
                           (strconv.AppendFloat(…, -1, 32)), same format rules and NaN / Inf behaviour as FLOAT64
                                                                                                response schemas only */
    GOFR_F_TIME = 11    /* time.Time: Time.MarshalJSON = the quoted RFC 3339 text with nanoseconds, trailing zeros of the
                           fraction trimmed, "Z" for offset 0 else ±hh:mm ("2006-01-02T15:04:05.999999999Z07:00").  Four
                           words: Unix seconds (lo, hi; the zero Time is -62135596800), nanoseconds (0 .. 999999999), zone
                           offset in seconds east of UTC (int32).  A year outside [0, 9999] or a zone hour outside [0, 23]
                           makes MarshalJSON — and with it Encode — fail: the response keeps its status and headers and
                           has no body, as for NaN (a nanoseconds word >= 1e9, which no Time holds, is answered the same way).  Never "empty" for omitempty (a struct).     response schemas only */
};
/* What the field holds of its kind T (response schemas only; Bind schemas take GOFR_C_VALUE of kinds 1..6):
 *   GOFR_C_VALUE  T          GOFR_C_PTR  *T (nil → null)      GOFR_C_SLICE  []T (nil → null, empty → [])
 *   GOFR_C_MAP    map[string]T, T not a struct (nil → null; keys sorted bytewise like encoding/json does)
 * One container level per field; deeper types nest through GOFR_F_STRUCT (a struct field may again be a pointer, slice
 * or map).  interface{} values, [][]T (other than [][]byte) and maps of structs are not modelled: GOFR_ERR_UNSUPPORTED. */
enum { GOFR_C_VALUE = 0, GOFR_C_PTR = 1, GOFR_C_SLICE = 2, GOFR_C_MAP = 3,
       GOFR_C_SLICE_PTR = 4 /* []*T (what ORMs hand back): like []T, each element preceded by a presence word (0: nil → null) */ };
#define GOFR_FIELD_BARE 0x01u /* the schema has this ONE field and stands for the field's own type: the handler returns a
                                 []T, map[string]T, *T or float64 rather than a struct; no {"name":…} around the value */
#define GOFR_NIL_COUNT 0xFFFFFFFFu /* count word of a nil slice / map */

typedef struct gofr_field_desc {
    const char* go_name;   /* Go field name (case-insensitive Bind fallback, error text) */
    const char* json_name; /* `json:"..."` name; NULL/"" = go_name */
    uint8_t kind;          /* GOFR_F_* */
    uint8_t omitempty;     /* isEmptyValue: false, 0, 0.0 (either sign), "", nil pointer, nil or empty slice / map;
                              a struct value is never empty */
    uint8_t container;     /* GOFR_C_* */
    uint8_t flags;         /* GOFR_FIELD_* */
    uint16_t elem_schema;  /* GOFR_F_STRUCT: schema id of the struct type (added before this schema: no cycles) */
    uint8_t reserved[2];
} gofr_field_desc;

typedef struct gofr_handler_desc {
    uint32_t kind;        /* GOFR_H_* */
    uint32_t schema_id;   /* GOFR_H_ROW, GOFR_H_BIND_ECHO */
    const char* s0; uint32_t s0_len;
    const char* s1; uint32_t s1_len;
    const char* s2; uint32_t s2_len;
    const char* s3; uint32_t s3_len;
    const uint8_t* blob; uint32_t blob_len; /* GOFR_H_FILE */
} gofr_handler_desc;

/* ---- request batch (host or device memory, SoA): desc[n], trace_id[n][16], arena[arena_bytes] ----
 * A request's variable bytes are contiguous in the arena:
 *   [ URL.Path (decoded) | URL.RawQuery | pad to 4 | data section ]
 * arena_off must be a multiple of 4.  The data section is the request body for GOFR_H_BIND_ECHO routes and the
 * handler-result row for GOFR_H_ROW routes.  Row format of a struct S: its FIXED part, then its VARIABLE part.
 *   fixed part, little-endian 32-bit words, fields in schema order:
 *     INT64 / INT / UINT64 / FLOAT64  two words (lo, hi; FLOAT64: the IEEE-754 bits)   INT32 / FLOAT32  one   BOOL  one, 0/1
 *     BYTES                  one word, the byte length, GOFR_NIL_COUNT when nil
 *     TIME                   four words: seconds lo, hi, nanoseconds, zone offset
 *     STRING                 one word, the byte length                            STRUCT  the struct's fixed part, inline
 *     *T                     one word 0 (nil) / 1, then T's fixed words (ignored, and T's variable part ABSENT, when nil)
 *     []T, []*T, map[string]T  one word, the element count, GOFR_NIL_COUNT when nil
 *   variable part, bytes, fields in schema order, nothing aligned:
 *     STRING / BYTES  the bytes   STRUCT / *STRUCT  the struct's variable part   other scalars  nothing
 *     []T            count elements E(T)            map[string]T   count entries: u32 key length, key bytes, E(T)
 *     []*T           count elements: u32 presence (0 = nil, nothing follows; else 1), E(T)
 *     E(T): scalars — their fixed words; STRING / BYTES — u32 length + bytes; STRUCT — its fixed part + its variable part
 * A flat struct of scalars and strings therefore is: one word per field (INT64: two) followed by the string bytes of all
 * STRING fields concatenated in schema order. */
typedef struct gofr_req_desc {
    uint32_t arena_off;
    uint16_t path_len;
    uint16_t query_len;
    uint32_t data_len;
    uint8_t method; /* GOFR_M_* */
    uint8_t flags;  /* GOFR_REQ_* */
    uint16_t aux;
} gofr_req_desc;

#define GOFR_REQ_FORCE_QUERY 0x01u /* url.URL.ForceQuery: target ended in a bare '?' (only visible in a 301 Location) */

/* ---- response batch: out[out_off[i] .. out_off[i+1]) are request i's bytes, packed in request order;
 *      meta[i] = status (low 16 bits) | route_id << 16 (0xFFFF = no user route; status 0 = GOFR_H_HOST pending) ---- */
#define GOFR_META_STATUS(m) ((uint32_t)(m) & 0xFFFFu)
#define GOFR_META_ROUTE(m) ((uint32_t)(m) >> 16)
#define GOFR_ROUTE_NONE 0xFFFFu

typedef struct gofr_table gofr_table;
typedef struct gofr_engine gofr_engine;
typedef uint64_t gofr_ticket;

/* ================= route table (startup, single thread) ================= */
int gofr_table_create(gofr_table** out, uint32_t frame_mode);
void gofr_table_destroy(gofr_table*);
int gofr_table_add_schema(gofr_table*, uint32_t schema_id, const char* go_type_name, const gofr_field_desc* fields,
                          uint32_t n_fields);
/* Call order is match priority (mux scans routes in registration order).  Patterns: literals, {name} (= [^/]+) and
 * {name:regexp} where the regexp is a concatenation of quantified units: a unit is a bracket class, \d, \w, '.', an escaped
 * punctuation character or a literal character; a quantifier is + * ? {n} {n,} {n,m} (n, m <= 250) — e.g. [0-9]+,
 * \d{4}-\d{2}, v[0-9]+, [a-z]+\.[a-z]{2,4}.  Alternation, groups, anchors, lazy quantifiers, \s / \p{..} / POSIX classes and
 * counted repetition of classes with non-ASCII members ('.', negated classes: Go counts runes) → GOFR_ERR_UNSUPPORTED. */
int gofr_table_add_route(gofr_table*, uint32_t method, const char* pattern, uint32_t pattern_len,
                         const gofr_handler_desc* handler, uint32_t* route_id_out);
/* GET /.well-known/health, GET /favicon.ico, PathPrefix("/") catch-all — appended after the user routes, as
 * App.Run does.  Without this call the table behaves like the router before Run() (gofr_test.go:85-95): mux's own
 * plain-text 404 / empty 405 answer unmatched requests and no middleware runs for them. */
int gofr_table_add_default_routes(gofr_table*, const uint8_t* favicon, uint32_t favicon_len);
int gofr_table_seal(gofr_table*);
/* The sealed image is position independent: rank 0 seals and serializes, the bytes are broadcast (NCCL), every
 * other rank deserializes.  *len_inout: capacity in, size out (call with buf NULL to query). */
int gofr_table_serialize(const gofr_table*, uint8_t* buf, uint64_t* len_inout);
int gofr_table_deserialize(gofr_table** out, const uint8_t* buf, uint64_t len);
uint32_t gofr_table_route_count(const gofr_table*);
uint32_t gofr_table_max_response_bytes(const gofr_table*, uint32_t max_data_len);
/* Upper bound of ONE response given that request's sizes (what a host batcher sums up to size its output buffer). */
uint32_t gofr_table_response_bound(const gofr_table*, uint32_t path_len, uint32_t query_len, uint32_t data_len);

/* ================= engine (one per GPU / process) ================= */
int gofr_engine_create(gofr_engine** out, const gofr_table* sealed, int device);
void gofr_engine_destroy(gofr_engine*);

/* Device-resident batch: every pointer is device memory, `stream` is a cudaStream_t (NULL = default stream).
 * One fused launch: route match + middleware predicates + handler kind + JSON encode + HTTP framing.
 * date is the 29-byte IMF-fixdate for this batch (host memory).  out_off[n] receives the packed size.
 * d_arena must be 16-byte aligned and its allocation must extend at least 16 bytes past the last request byte; d_out must be
 * 16-byte aligned.  Launches on one engine must be stream-ordered with respect to each other (they share scratch). */
int gofr_serve_device(gofr_engine*, const gofr_req_desc* d_desc, const uint8_t* d_trace_ids, const uint8_t* d_arena,
                      uint32_t n, const char* date29, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                      uint32_t* d_meta, void* stream);

/* The same launch with a SLOT layout instead of packed offsets: response i is written at d_out + i * slot_bytes
 * (slot_bytes a multiple of 16, d_out 16-byte aligned) and d_out_len[i] receives its length; the bytes between the end
 * of a response and the next 16-byte boundary are zeroed, the rest of the slot is left untouched.  A response longer
 * than the slot is not written: d_out_len[i] > slot_bytes tells the caller to serve that request through the packed
 * call.  Slots remove the only dependence between requests (the running output offset): no scan, no look-back between
 * tiles, and every response starts aligned — this is the layout a ring of pinned response buffers wants anyway. */
int gofr_serve_device_slots(gofr_engine*, const gofr_req_desc* d_desc, const uint8_t* d_trace_ids, const uint8_t* d_arena,
                            uint32_t n, const char* date29, uint8_t* d_out, uint32_t slot_bytes, uint32_t* d_out_len,
                            uint32_t* d_meta, void* stream);

/* Host batch: pinned (gofr_alloc_pinned) or pageable caller-owned buffers; the engine pipelines
 * H2D → kernel → D2H in chunks over its own streams.  submit is thread-safe; wait blocks the caller. */
typedef struct gofr_req_batch {
    const gofr_req_desc* desc;
    const uint8_t* trace_ids;
    const uint8_t* arena;
    uint64_t arena_bytes;
    uint32_t n;
    char date[29];
    uint8_t pad[3];
} gofr_req_batch;

typedef struct gofr_resp_batch {
    uint8_t* out;       /* capacity out_cap */
    uint64_t out_cap;
    uint32_t* out_off;  /* n+1 */
    uint32_t* meta;     /* n */
    uint64_t out_bytes; /* filled by wait */
} gofr_resp_batch;

/* submit is thread-safe (submits are serialised inside the engine) and currently runs the batch to completion before it
 * returns; wait(ticket) reports that batch's status exactly once.  With pinned caller buffers egress is device driven
 * (no host stall per chunk); pageable buffers fall back to an exact-size cudaMemcpy pipeline. */
int gofr_batch_submit(gofr_engine*, const gofr_req_batch* in, gofr_resp_batch* out, gofr_ticket* ticket);
int gofr_batch_wait(gofr_engine*, gofr_ticket ticket);

/* Host batch with the slot layout: response i lands in out + i * slot_bytes (a ring of fixed-size response buffers),
 * its length in out_len[i] (> slot_bytes: not written, serve that request through the packed call).  Chunk sizes are
 * known on the host, so the results leave with plain asynchronous copies — no device-side packing, no egress kernel.
 * slot_bytes: a positive multiple of 16; out: 16-byte aligned, n * slot_bytes bytes.  Whole slots are copied back: the
 * bytes of a slot behind its (zero-padded) response are unspecified. */
typedef struct gofr_slot_batch {
    uint8_t* out;
    uint32_t slot_bytes;
    uint32_t reserved;
    uint32_t* out_len; /* n */
    uint32_t* meta;    /* n */
} gofr_slot_batch;
int gofr_batch_submit_slots(gofr_engine*, const gofr_req_batch* in, gofr_slot_batch* out, gofr_ticket* ticket);
int gofr_engine_set_chunk(gofr_engine*, uint32_t requests_per_chunk);
/* Tile geometry: shared-memory staging budget for request bytes, per request.  Tiles whose request bytes exceed the
 * budget are still served correctly, straight from HBM. */
int gofr_engine_set_tile(gofr_engine*, uint32_t in_bytes_per_req);
int gofr_engine_geometry(const gofr_engine*, uint32_t* grid, uint32_t* blocks_per_sm, uint32_t* smem_bytes,
                         uint32_t* sm_count);
/* Slot layout: which instance of the serve kernel answers — 4 CTAs/SM with 128 registers (the default for tables whose live
 * routes answer with one fast-path program shape) or 5 CTAs/SM with 96 registers (every other table).  ctas_per_sm 0 = query,
 * 4 or 5 = force; *in_effect (may be NULL)
 * receives the value in effect.  Tuning knob, no effect on results. */
int gofr_engine_slot_ctas(gofr_engine*, int ctas_per_sm, int* in_effect);
/* the engine's default for a sealed table (4 or 5), computable without a GPU */
int gofr_table_slot_ctas(const gofr_table*, int* ctas_per_sm);
/* The device calls with a packed output — gofr_serve_device, the frame codecs (gofr_grpc_hello_device, gofr_proto_encode_device,
 * gofr_proto_decode_device, gofr_proto_encode_nested_device, gofr_proto_decode_nested_device) and gofr_requestlog_device —
 * report an undersized d_out through this flag (the launch itself is asynchronous).  Output is written a tile of 128
 * records at a time: the first tile that does not fit and every tile after it are dropped whole, and nothing is written at
 * or past out_cap.  d_out_off and d_meta (where the call has one) are still written in full: the offsets every record would
 * have had with room enough (d_out_off[n] = the capacity needed) and every status. */
int gofr_engine_overflowed(gofr_engine*, int* flag_out, int reset);
int gofr_engine_set_timing(gofr_engine*, int on);

/* Binds the CALLING thread to the CPUs of the NUMA node the GPU hangs off (sysfs: /sys/bus/pci/devices/<bus id>/numa_node)
 * and makes that node the preferred one for the pages the thread touches from now on — call it before gofr_alloc_pinned
 * and before the threads that fill the batches are started.  With eight GPUs on two sockets, pinned buffers that all sit
 * on one socket make half of the H2D/D2H traffic cross the inter-socket link: the reference has nothing like it (its
 * goroutines are scheduled by the Go runtime, pkg/gofr/httpServer.go:29-33); a host that feeds GPUs needs it.
 * numa_node_out (may be NULL) receives the node, -1 if unknown.  GOFR_ERR_UNSUPPORTED when the topology cannot be read. */
int gofr_bind_host_thread(int device, int* numa_node_out);
void* gofr_alloc_pinned(size_t bytes);
void gofr_free_pinned(void*);

/* gRPC unary Hello (config 5): length-prefixed HelloRequest frames in, length-prefixed HelloResponse frames out,
 * packed; frame i of the input starts at in_off[i].  meta[i] = 0 ok, else a GOFR_GRPC_* error (frame emitted empty). */
enum { GOFR_GRPC_OK = 0, GOFR_GRPC_COMPRESSED = 1, GOFR_GRPC_BAD_LENGTH = 2, GOFR_GRPC_BAD_PROTO = 3, GOFR_GRPC_BAD_UTF8 = 4,
       GOFR_GRPC_BAD_ROW = 5,
       GOFR_GRPC_DEFER = 6 /* gofr_proto_decode_nested_device: a valid frame outside its subset (a singular message field sent
                              more than once, which protobuf-go merges; a map field with more than 64 entries).  Pass the
                              batch through gofr_proto_decode_nested_deferred_device, which decodes maps of up to 4096
                              entries; what is still DEFER after it, decode on the host */ };
int gofr_grpc_hello_device(gofr_engine*, const uint8_t* d_in, const uint32_t* d_in_off, uint32_t n, uint8_t* d_out,
                           uint64_t out_cap, uint32_t* d_out_off, uint32_t* d_meta, void* stream);

/* proto3 message encoder (SURVEY.md §8f rank 4): proto.Marshal of the message a unary gRPC handler returns + the
 * 5-byte length-prefixed-message header grpc-go puts in front (examples/grpc-server/grpc/hello_grpc.pb.go:73-89 hands
 * the response to grpc-go; protobuf-go v1.32.0, grpc-go v1.60.1), for a batch of flat messages with scalar fields.
 *   fields     the message type: (number, GOFR_PB_* type) in ascending field-number order — the order proto.Marshal
 *              emits them; at most GOFR_PROTO_MAX_FIELDS
 *   d_rows     row i = d_rows[d_row_off[i] .. d_row_off[i+1]), offsets multiples of 4, GOFR_H_ROW layout: per field
 *              (same order) 64-bit types two LE words (lo, hi), the others one (float / double: IEEE bits; string /
 *              bytes: byte length), then the string bytes in field order.  The buffer follows the rule for
 *              device input buffers at the top of this file: 16-byte aligned, 16 readable bytes past the last row.
 *   output     packed frames in row order, d_out_off[n+1]; d_meta[i] = GOFR_GRPC_OK, GOFR_GRPC_BAD_UTF8 (a string
 *              field is not valid UTF-8: proto.Marshal fails, the RPC fails — no frame), GOFR_GRPC_BAD_ROW (malformed
 *              row from the host shim — no frame).
 * Zero values are not emitted (proto3 implicit presence; -0.0 is not a zero value); negative int32 / enum values take
 * ten bytes; sint32 / sint64 are zigzag encoded. */
enum {
    GOFR_PB_DOUBLE = 1, GOFR_PB_FLOAT = 2, GOFR_PB_INT64 = 3, GOFR_PB_UINT64 = 4, GOFR_PB_INT32 = 5, GOFR_PB_FIXED64 = 6,
    GOFR_PB_FIXED32 = 7, GOFR_PB_BOOL = 8, GOFR_PB_STRING = 9, GOFR_PB_BYTES = 12, GOFR_PB_UINT32 = 13, GOFR_PB_ENUM = 14,
    GOFR_PB_SFIXED32 = 15, GOFR_PB_SFIXED64 = 16, GOFR_PB_SINT32 = 17, GOFR_PB_SINT64 = 18
}; /* google.protobuf.FieldDescriptorProto.Type */
#define GOFR_PROTO_MAX_FIELDS 32
typedef struct gofr_proto_field {
    uint32_t number; /* 1 .. 2^29-1 */
    uint32_t type;   /* GOFR_PB_* */
} gofr_proto_field;
int gofr_proto_encode_device(gofr_engine*, const gofr_proto_field* fields, uint32_t n_fields, const uint8_t* d_rows,
                             const uint32_t* d_row_off, uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                             uint32_t* d_meta, void* stream);
/* The other direction — dec(in) of the same handler: length-prefixed frames in (frame i = d_in[d_in_off[i] ..
 * d_in_off[i+1]), as for gofr_grpc_hello_device), proto.Unmarshal into the message type, the field values out as rows in
 * the layout above (row sizes are multiples of 4; absent fields hold their zero value), packed, d_row_off[n+1].
 * d_meta[i]: GOFR_GRPC_OK or COMPRESSED / BAD_LENGTH / BAD_PROTO / BAD_UTF8 as for the Hello call (a failed frame gives an
 * empty row).  Unknown fields — and known fields arriving with a foreign wire type — are skipped; the last occurrence of
 * a field wins; int32 / uint32 / enum keep the low 32 bits of the varint, bool is v != 0.  d_in follows the rule for
 * device input buffers at the top of this file: 16-byte aligned, 16 readable bytes past the last frame. */
int gofr_proto_decode_device(gofr_engine*, const gofr_proto_field* fields, uint32_t n_fields, const uint8_t* d_in,
                             const uint32_t* d_in_off, uint32_t n, uint8_t* d_rows, uint64_t rows_cap, uint32_t* d_row_off,
                             uint32_t* d_meta, void* stream);

/* The same encoder for message types with NESTED and REPEATED fields (proto.Marshal as protobuf-go v1.32.0 does it: fields
 * in field-number order, singular zero values skipped, a set message field written even when empty, repeated numeric
 * scalars packed, repeated strings / bytes / messages one tag per element).  msgs[m] names fields[first_field ..
 * first_field + n_fields) (ascending numbers); a field of type GOFR_PB_MESSAGE names its message type in `msg`; `root` is the
 * type of the rows.  At most 8 message types with 48 fields in all, nested at most 4 levels deep, no recursive types.
 * MAP FIELDS: a field of type GOFR_PB_MAP (repeated = 0) names its ENTRY TYPE in `msg`: a message type with exactly two
 * singular fields, number 1 the key (an integer kind, bool or string) and number 2 the value (any type but GOFR_PB_MAP).
 * An entry type may serve several map fields; it is not the root, not the type of a GOFR_PB_MESSAGE field, and its field
 * range is shared with no other message type (GOFR_ERR_INVALID otherwise); it counts
 * toward the limits (map<string, M> is two levels).  Every entry is written with its key and value, zero values included,
 * a message value always (tag, length 0 when its presence word is 0) — protobuf-go's Deterministic bytes: entries must be
 * in strictly ascending key order (bool false < true; signed kinds signed, unsigned kinds unsigned, strings by bytes with a
 * shorter prefix first, keys compared as the row words hold them), else the row is GOFR_GRPC_BAD_ROW (a Go map cannot hold
 * it).  Rows: the layout of "Row format" above — fixed words of a message in field order (64-bit kinds two words, string /
 * bytes their length, a singular message a presence word 0 / 1 followed by its own fixed part, a repeated field or a map
 * its element count), then the variable part in field order (string bytes; a set message's variable part; the elements of
 * a repeated field: scalars as their words, strings as u32 length + bytes, messages — and map entries — as fixed part +
 * variable part).  Output and d_meta as for gofr_proto_encode_device. */
#define GOFR_PB_MESSAGE 11u
#define GOFR_PB_MAP 32u
typedef struct gofr_proto_nfield {
    uint32_t number;
    uint8_t type;     /* GOFR_PB_*, GOFR_PB_MESSAGE or GOFR_PB_MAP */
    uint8_t repeated; /* 0 / 1 (0 for a map) */
    uint16_t msg;     /* GOFR_PB_MESSAGE: index into msgs; GOFR_PB_MAP: the entry type */
} gofr_proto_nfield;
typedef struct gofr_proto_nmsg {
    uint16_t first_field, n_fields;
} gofr_proto_nmsg;
int gofr_proto_encode_nested_device(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                    uint32_t n_fields, uint32_t root, const uint8_t* d_rows, const uint32_t* d_row_off, uint32_t n,
                                    uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off, uint32_t* d_meta, void* stream);
/* The other direction for the same message types: length-prefixed frames -> rows (proto.Unmarshal as protobuf-go does it:
 * unknown fields and balanced groups skipped at every level; a known number with a foreign wire type is unknown, except that
 * repeated numeric scalars are accepted packed and unpacked; singular scalars and strings: the last occurrence wins;
 * repeated strings / bytes / messages: one element per occurrence in wire order; strings must be valid UTF-8).  A map
 * field's row holds the resulting map in the encoder's canonical form: distinct keys in ascending order, the last entry on
 * the wire for each key winning (message values replaced, not merged); inside an entry the last key and value win, a
 * missing key or value is its zero value, a missing message value an empty message (presence 1: message values are always
 * present).  A value message sent twice inside one entry (merged by protobuf-go), and a map field with more than 64 entries
 * on the wire in one message (duplicates counted), give DEFER.  d_meta[i]:
 * GOFR_GRPC_OK or COMPRESSED / BAD_LENGTH / BAD_PROTO / BAD_UTF8 / DEFER (a failed frame gives an empty row); rows are
 * packed, 4-byte aligned, zero padded to a multiple of 4, d_row_off[n + 1]. */
int gofr_proto_decode_nested_device(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                    uint32_t n_fields, uint32_t root, const uint8_t* d_in, const uint32_t* d_in_off, uint32_t n,
                                    uint8_t* d_rows, uint64_t rows_cap, uint32_t* d_row_off, uint32_t* d_meta, void* stream);
/* validation of such a description without a GPU (map rules included: a description that breaks them is GOFR_ERR_INVALID);
 * desc_out (>= 512 bytes, may be NULL with desc_cap 0 to validate only... then GOFR_ERR_CAPACITY means "valid") receives
 * the kernel's internal descriptor (test infrastructure reads it) */
int gofr_proto_nested_describe(const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                               uint32_t root, void* desc_out, uint32_t desc_cap);

/* FIELD PRESENCE: the three calls above with `presence`, one byte per entry of `fields` (NULL: exactly the call above).
 *   0                  implicit presence, as above;
 *   GOFR_PB_OPTIONAL   a proto3 `optional` field (explicit presence; protoreflect: fd.HasOptionalKeyword());
 *   1 .. 7             a member of oneof group k of its message type (protoreflect: fd.ContainingOneof() when it is not
 *                      synthetic; at most 7 groups per message type).
 * A oneof member is singular (not repeated, not a map); the key and value of a map entry type carry no presence; optional
 * on a message field means what a singular message field means anyway.  Anything else is GOFR_ERR_INVALID.
 * Rows: an explicit-presence scalar, string or bytes field (optional, or a oneof member) owns a PRESENCE WORD 0 / 1
 * followed by its usual words in the fixed part; its string bytes are in the variable part only when it is set.  A
 * message-typed member keeps the layout of a singular message field (presence word + its fixed part inline).  Each oneof
 * member has its own slot, in field order.  The encoder refuses (GOFR_GRPC_BAD_ROW) a presence word other than 0 / 1 on
 * such a field, an unset one whose value words (a message member: its inline fixed part) are not all zero, and more than
 * one set member in one oneof group — so decode(encode(row)) == row for every row it accepts.
 * Encoder (proto.Marshal, protobuf-go v1.32.0): a set field is written even at its zero value or empty, an unset one not
 * at all; members go out at their own field numbers, in field-number order.  Decoder (proto.Unmarshal): an optional field
 * is set iff it occurs with its own wire type, the last occurrence winning; in a oneof group, the member whose occurrence is
 * last among all the group's members is the set one, with its last value, and the others are unset.  A member arriving
 * with a foreign wire type is an unknown field and does not change the case.  A message member that occurs twice at one
 * message level is GOFR_GRPC_DEFER, even with another member in between (protobuf-go merges A, A and replaces in A, B, A:
 * either way, decode it on the host).  UTF-8 is checked on every occurrence, the losing members' too; status precedence
 * malformed > invalid UTF-8 > DEFER as above.  The flat codec (gofr_proto_encode_device / _decode_device) has no presence:
 * a flat message type with it goes through these calls. */
#define GOFR_PB_OPTIONAL 0x80u
int gofr_proto_encode_nested_ex_device(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                       uint32_t n_fields, uint32_t root, const uint8_t* presence, const uint8_t* d_rows,
                                       const uint32_t* d_row_off, uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                                       uint32_t* d_meta, void* stream);
int gofr_proto_decode_nested_ex_device(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                       uint32_t n_fields, uint32_t root, const uint8_t* presence, const uint8_t* d_in,
                                       const uint32_t* d_in_off, uint32_t n, uint8_t* d_rows, uint64_t rows_cap, uint32_t* d_row_off,
                                       uint32_t* d_meta, void* stream);
int gofr_proto_nested_describe_ex(const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                                  uint32_t root, const uint8_t* presence, void* desc_out, uint32_t desc_cap);

/* LARGE MAPS: the second pass of the nested decoder.  Same description (presence may be NULL), frames and offsets as the
 * gofr_proto_decode_nested_ex_device call before it; d_meta_in is that call's status column.
 *   selection   frame i is decoded again when d_meta_in[i] == GOFR_GRPC_DEFER.  Any other frame gets an empty row and
 *               d_meta[i] = d_meta_in[i], so d_meta is the merged status column; d_meta may be d_meta_in itself.
 *   decoding    from scratch, by the rules of the _ex call, with one difference: a map field may have up to 4096 entries on
 *               the wire in one message (duplicates counted).  Still GOFR_GRPC_DEFER: a singular message (or a message
 *               member of a oneof, or a map's value message inside one entry) sent twice, and more than 4096 entries.
 *               Statuses and their precedence as for the _ex call.  Every selected frame is validated again, so a frame
 *               selected by mistake costs time but gets the answer of the _ex call: the same row, byte for byte.
 *   output      rows packed in frame order, d_row_off[n + 1], under the packed-output contract of the other frame calls
 *               (whole tiles of 128 frames dropped past rows_cap, the overflow flag set, offsets and statuses written in
 *               full).  d_in follows the rule for device input buffers at the top of this file.
 * A description without map fields is taken; its selected frames stay DEFER.  Each CTA decodes one selected frame at a
 * time, map entries put in key order by a sort in shared memory (64 KiB per level of maps inside map values).
 * Combining the two calls: row i is the first call's row unless d_meta_in[i] == GOFR_GRPC_DEFER and d_meta[i] ==
 * GOFR_GRPC_OK, in which case it is row i of this call; d_meta[i] is the final status either way. */
int gofr_proto_decode_nested_deferred_device(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                             uint32_t n_fields, uint32_t root, const uint8_t* presence, const uint8_t* d_in,
                                             const uint32_t* d_in_off, uint32_t n, const uint32_t* d_meta_in, uint8_t* d_rows,
                                             uint64_t rows_cap, uint32_t* d_row_off, uint32_t* d_meta, void* stream);

/* HOST BUFFERS for the nested codec: what a gRPC server holds (request frames, its handlers' responses) goes in and comes
 * back in host memory, through the chunk pipeline of gofr_batch_submit (three device slots, three streams).  Same
 * description arguments as the _ex calls (presence may be NULL).
 *   in     record i = data[off[i] .. off[i + 1]); off has n + 1 entries, non-decreasing, off[n] <= data_bytes; for encode
 *          the records are rows (the layout above) and every offset is a multiple of 4.  Offsets are checked on the host a
 *          chunk at a time: a bad batch returns GOFR_ERR_INVALID with nothing still writing into the caller's buffers.
 *   out    a gofr_resp_batch, collected with gofr_batch_wait: records packed in order, out_off[n + 1], meta[n], out_bytes.
 *          Pinned buffers (gofr_alloc_pinned) are streamed by the device; pageable ones are copied back at each chunk's
 *          exact size.
 * gofr_proto_batch_decode: frames → rows.  Row i and meta[i] are what gofr_proto_decode_nested_ex_device followed by
 * gofr_proto_decode_nested_deferred_device give, combined by the rule above; meta[i] is the final status.  A frame still
 * GOFR_GRPC_DEFER (a singular message sent twice, a map field with more than 4096 entries: decode it on the host) and a
 * failed frame get an empty row.  Rows are 4-byte aligned within out.
 * gofr_proto_batch_encode: rows → frames, byte for byte and status for status what gofr_proto_encode_nested_ex_device gives.
 * out_cap: gofr_proto_nested_bound sizes it.  When it is too small, gofr_batch_wait returns GOFR_ERR_CAPACITY, as for
 * gofr_batch_submit: nothing is written at or past out_cap, meta is complete, out_bytes = out_off[n] = the bytes written, and
 * out_off is meaningful only for the records of chunks that were written (a chunk that does not fit is dropped whole; the
 * offsets of its records are unspecified).  n == 0 takes no buffers. */
typedef struct gofr_proto_batch {
    const uint8_t* data;   /* frames (decode) or rows (encode) */
    uint64_t data_bytes;
    const uint32_t* off;   /* n + 1 */
    uint32_t n;
} gofr_proto_batch;
int gofr_proto_batch_decode(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                            uint32_t root, const uint8_t* presence, const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* ticket);
int gofr_proto_batch_encode(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                            uint32_t root, const uint8_t* presence, const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* ticket);
/* No GPU needed: (per_byte, per_record) such that no record of b bytes yields more than per_byte * b + per_record output
 * bytes — a row when decode != 0, a whole frame with its 5-byte prefix when encoding.  Sum it over a batch for out_cap. */
int gofr_proto_nested_bound(const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                            uint32_t root, const uint8_t* presence, int decode, uint32_t* per_byte, uint32_t* per_record);

/* Bind as a stage of the split API: Context.Bind(&v) for closures that stay on the host (pkg/gofr/context.go:52-54 ->
 * pkg/gofr/http/request.go:40-47 -> json.Unmarshal(body, &v), v a struct of a registered schema).  Body i is the data
 * section of request i (same descriptors / arena as the serve calls); result i lies in its own slot d_rows + i * slot_bytes
 * (slot_bytes a multiple of 16, d_rows 16-byte aligned), zero padded to the next 16-byte boundary:
 *   d_status[i] = GOFR_BIND_OK     the struct as a row in the GOFR_H_ROW layout (one LE u32 word per field in schema order,
 *                                  two for INT64 / INT / FLOAT64, STRING = byte length; then the DECODED string bytes in schema order:
 *                                  escapes resolved, invalid UTF-8 replaced by U+FFFD, as json.Unmarshal stores them).
 *                                  Keys are matched exactly, then case-insensitively; unknown keys are skipped; later
 *                                  duplicates win; null leaves the zero value.
 *   d_status[i] = GOFR_BIND_ERROR  err.Error() of json.Unmarshal: a syntax error ("invalid character 'x' after object key",
 *                                  "unexpected end of JSON input"), or the FIRST UnmarshalTypeError ("json: cannot unmarshal
 *                                  string into Go struct field T.f of type int64"); the partially filled struct Go also
 *                                  leaves behind in that case is not reported
 *   d_status[i] = GOFR_BIND_HOST   not decided on the device (nesting deeper than 64, or a number for a float64 member that
 *                                  is one of the rare literals left to Go's slow path — see GOFR_H_BIND_ECHO): run encoding/json on the host
 * d_len[i] = bytes of the result; a value above slot_bytes means it did not fit and nothing was written (bind it again in a
 * slot of at least d_len[i] bytes).
 * Pins: pkg/gofr/http/request_test.go:17-30, pkg/gofr/context_test.go:23-49. */
enum { GOFR_BIND_OK = 0, GOFR_BIND_ERROR = 1, GOFR_BIND_HOST = 2 };
/* The first row slot gofr::App and gofr_conn_app_frontend bind a body of data_len bytes in, for a schema of `fields`
 * fields: the fixed words (at most 8 bytes per field) plus the body, and 256 bytes for an error text; rounded up to 16 as
 * slot_bytes must be.  It holds the rows of ordinary bodies; those it does not hold are bound again in a wider slot.  64-bit. */
#define GOFR_BIND_ROW_SLOT(fields, data_len) ((8 * (uint64_t)(fields) + (uint64_t)(data_len) + 256 + 15) & ~(uint64_t)15)
/* What a row or error text of a body of data_len bytes can take at most, for a schema of `fields` fields whose Go type
 * name and longest JSON name take `names` bytes together.  A row is its fixed words (at most 8 bytes per field) and its
 * decoded strings: those come from disjoint pieces of the body, and no body byte yields more than 3 bytes (an invalid
 * UTF-8 byte becomes U+FFFD, EF BF BD; a valid sequence keeps its length; \uXXXX gives at most 3 bytes for 6, a surrogate
 * pair 4 for 12, the other escapes 1 for 2).  An error text takes at most 70 bytes besides a number literal (a piece of
 * the body) and the names: a syntax error ("invalid character '\u00XX' " and the longest scanner context) 69, "json:
 * cannot unmarshal number <literal> into Go struct field <T>.<name> of type float64" 69.  64-bit. */
#define GOFR_BIND_ROW_BOUND(fields, names, data_len) (8 * (uint64_t)(fields) + 3 * (uint64_t)(data_len) + 70 + (uint64_t)(names))
int gofr_bind_device(gofr_engine* e, uint32_t schema_id, const gofr_req_desc* d_desc, const uint8_t* d_arena, uint32_t n,
                     uint8_t* d_rows, uint32_t slot_bytes, uint32_t* d_len, uint32_t* d_status, void* stream);
/* The same stage with host buffers (what a host shim calls between gofr_batch_route and its closures); synchronous. */
int gofr_batch_bind(gofr_engine* e, uint32_t schema_id, const gofr_req_batch* in, uint8_t* rows, uint32_t slot_bytes,
                    uint32_t* len, uint32_t* status);

/* Stage 1 of the split API for routes whose closure stays on the host (GOFR_H_HOST): everything mux.Router.ServeHTTP
 * and the middleware chain decide before handler.ServeHTTP runs (pkg/gofr/http/router.go:14,30-33;
 * middleware/cors.go:10-13; pkg/gofr/handler.go:32-36), for a whole batch resident in HBM.
 *   d_meta[i] = status | route_id << 16, status: 301 cleanPath redirect, 404 / 405 mux's own handlers (route_id =
 *               GOFR_ROUTE_NONE), 200 OPTIONS answered by the CORS middleware, 0 = the handler of route_id runs;
 *   d_vars[i * GOFR_MAX_PATH_VARS + k] = offset | length << 16 of the k-th path variable inside the request's path
 *               (mux.Vars in template order — what Request.PathParam reads, pkg/gofr/http/request.go:36-38);
 *               0xFFFFFFFF for unused slots.
 * The host then runs the closures and hands their results to gofr_serve_device / gofr_batch_submit (same table: the
 * route is registered with the handler kind that describes its result, e.g. GOFR_H_ROW). */
#define GOFR_MAX_PATH_VARS 8
int gofr_route_device(gofr_engine*, const gofr_req_desc* d_desc, const uint8_t* d_arena, uint32_t n, uint32_t* d_meta,
                      uint32_t* d_vars, void* stream);
/* The same for a batch in host memory (synchronous: H2D of descriptors and paths, the route kernel, D2H of meta and vars
 * — n and n * GOFR_MAX_PATH_VARS words).  What the C++ stand-in of the app API (include/gofr_b200.hpp) calls before it
 * runs the closures. */
int gofr_batch_route(gofr_engine*, const gofr_req_batch* in, uint32_t* meta, uint32_t* vars);

/* The JSON line middleware.Logging hands to logger.Log after every request (SURVEY.md §8f rank 1; non-terminal writer:
 * json.NewEncoder(out).Encode(logEntry{Level: INFO, Time: time.Now(), Message: RequestLog{...}})):
 *   {"Level":"INFO","time":"<RFC 3339 nano>","message":{"id":"<32 hex>","start_time":"...","response_time":<µs>,
 *    "method":"..","user_agent":"..","ip":"..","uri":"..","response":<status>}}\n
 * with `omitempty` on every message field (logger.go:24-33).  What the reference reads from the clock and from the
 * request is an INPUT per record: the three clock readings, the local zone offset, and five byte strings laid back to
 * back in the arena in this order: req.Method | req.UserAgent() | first X-Forwarded-For header value | req.RemoteAddr |
 * req.RequestURI.  getIPAddress (first comma-separated element, else RemoteAddr, strings.TrimSpace) runs on the device.
 * Lines are packed: line i = d_out[d_out_off[i] .. d_out_off[i+1]).  The arena needs 32 readable bytes after the last
 * record byte.  trace ids: the same 16 bytes per request gofr_serve_device takes. */
/* kind GOFR_LOG_RPC is the gRPC LoggingInterceptor's line instead (pkg/gofr/grpc/log.go:15-50): logger.Infof("%s",
 * RPCLog{id, startTime, responseTime, method}) — the message is the STRING json.Marshal(RPCLog), escaped once more by
 * the outer encoder; `method` carries info.FullMethod, the other four strings are ignored. */
enum { GOFR_LOG_REQUEST = 0, GOFR_LOG_RPC = 1 };
typedef struct gofr_log_desc { /* 48 bytes */
    int64_t start_unix_ns;   /* start := time.Now()                        logger.go:44 */
    int64_t elapsed_ns;      /* time.Since(start)                          logger.go:53 */
    int64_t log_unix_ns;     /* time.Now() in logger.logf                  logging/logger.go:55 */
    uint32_t arena_off;
    uint16_t method_len, ua_len, xff_len, remote_len, uri_len;
    uint16_t status;         /* StatusResponseWriter.status (0: WriteHeader never ran → field omitted) */
    int32_t tz_offset_s;     /* offset of time.Local at that instant, seconds east of UTC */
    uint32_t kind;           /* GOFR_LOG_REQUEST or GOFR_LOG_RPC */
} gofr_log_desc;
int gofr_requestlog_device(gofr_engine*, const gofr_log_desc* d_desc, const uint8_t* d_trace_ids, const uint8_t* d_arena,
                           uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off, void* stream);

/* gofr_batch_submit / gofr_batch_submit_slots plus middleware.Logging's RequestLog line (gofr_requestlog_device's format)
 * for every request of the batch the middleware wraps, in the same call: the lines are a second output of the host-batch
 * chunk pipeline, written on the device from the statuses the serve kernel has just produced.  Responses, meta and the
 * packed / slot outputs are byte for byte and status for status what the call without a log gives.
 *   desc   one record per request of the batch (n = the gofr_req_batch's n).  Read: start_unix_ns, tz_offset_s, arena_off,
 *          the five lengths and kind, which is GOFR_LOG_REQUEST or GOFR_LOG_NONE (this request gets no line from the call:
 *          the caller logs it, or nobody does).  Filled by the call: status (the response's), log_unix_ns (the batch's)
 *          and elapsed_ns = log_unix_ns - start_unix_ns.
 *   arena  the five strings of each record, as gofr_requestlog_device takes them: method | User-Agent | first
 *          X-Forwarded-For value | RemoteAddr | RequestURI back to back from arena_off; arena_bytes long.
 * Which requests get a line: request i has one exactly when GOFR_META_ROUTE(meta[i]) != GOFR_ROUTE_NONE (gorilla/mux
 * wraps middleware around matched routes only, so the cleanPath 301 and mux's own 404 / 405 are not logged),
 * GOFR_META_STATUS(meta[i]) != 0 (a GOFR_H_HOST hole is logged by the call that serves its closure's result) and its kind
 * is GOFR_LOG_REQUEST.  The line's id is the request's trace id.  Every other request has an empty line.
 *   out    request i's line = out[log_off[i] .. log_off[i + 1]) (log_off has n + 1 entries), in request order; lines =
 *          the requests that have one, out_bytes = the bytes of all of them.
 * Capacity: a short out_cap makes gofr_batch_wait return GOFR_ERR_CAPACITY with lines and out_bytes set to what the batch
 * needed; nothing is written at or past out_cap, and the response columns are complete whenever their own capacities
 * suffice.  log_off holds 32-bit offsets: a batch whose lines pass 4 GiB is GOFR_ERR_CAPACITY too.  gofr_batch_log_bound
 * gives an out_cap that always suffices.  Pinned buffers (gofr_alloc_pinned) are streamed by the device, pageable ones are
 * copied back at each chunk's exact size.
 * GOFR_ERR_INVALID: the batch call's cases, a null log column (arena may be NULL when every string is empty), a record
 * whose strings pass arena_bytes, a kind other than GOFR_LOG_REQUEST / GOFR_LOG_NONE. */
enum { GOFR_LOG_NONE = 2 };
typedef struct gofr_batch_log {
    const gofr_log_desc* desc;     /* n */
    const uint8_t* arena;
    uint64_t arena_bytes;
    int64_t log_unix_ns;           /* the logger's time.Now() for every line of the batch */
    uint8_t* out;
    uint64_t out_cap;
    uint32_t* log_off;             /* n + 1 */
    uint32_t lines;                /* filled by submit, reported by wait */
    uint32_t reserved;
    uint64_t out_bytes;            /* filled by submit, reported by wait */
} gofr_batch_log;
int gofr_batch_submit_log(gofr_engine*, const gofr_req_batch* in, gofr_resp_batch* out, gofr_batch_log* log, gofr_ticket* ticket);
int gofr_batch_submit_slots_log(gofr_engine*, const gofr_req_batch* in, gofr_slot_batch* out, gofr_batch_log* log,
                                gofr_ticket* ticket);
/* No GPU needed: an out_cap that always suffices for the lines of these n records (gofr_batch_submit_log,
 * gofr_proto_batch_encode_log) — for each record whose kind is not GOFR_LOG_NONE, 320 bytes plus 6 per string byte, and
 * for a GOFR_LOG_RPC record one more per method byte (RPCLog's method is escaped twice: one byte may leave as 7). */
int gofr_batch_log_bound(const gofr_log_desc* desc, uint32_t n, uint64_t* out_cap);

/* gofr_proto_batch_encode plus the gRPC LoggingInterceptor's RPCLog line (gofr_requestlog_device's GOFR_LOG_RPC format)
 * for every call of the batch that asks for one, in the same call: the lines are a second output of the encode batch's
 * chunk pipeline, written on the device.  LoggingInterceptor (pkg/gofr/grpc/log.go:27-50) logs once the handler has
 * returned, which is when the call's response is handed to this call, and before grpc-go marshals it.  out, out_off, meta
 * and the frames are byte for byte and status for status what gofr_proto_batch_encode gives for the same batch; out_bytes
 * reports what the batch needed, as in the other _log calls.
 *   trace_ids  16 bytes per record: the trace id of the span the interceptor started, the line's id.
 *   log        one record per call (n = the gofr_proto_batch's n), in a gofr_batch_log as gofr_batch_submit_log takes it.
 *              Read: start_unix_ns, elapsed_ns (the interceptor's time.Since(start): the handler ran on the caller's
 *              thread), tz_offset_s, arena_off, method_len (info.FullMethod, at arena_off) and kind, which is GOFR_LOG_RPC
 *              or GOFR_LOG_NONE (no line from this call).  The other four lengths are checked against the arena and
 *              otherwise ignored.  Filled by the call: log_unix_ns (the batch's log->log_unix_ns).
 * Record i has a line exactly when its kind is GOFR_LOG_RPC, whatever meta[i] says; every other record has an empty line.
 * A call whose handler returned an error has no response for grpc-go to marshal: pass an empty row (off[i] == off[i + 1]).
 * It still gets its line, and its frame and status are to be ignored.
 * Lines, capacity, pinned and pageable buffers, the 4 GiB limit and n == 0 are as for gofr_batch_submit_log;
 * gofr_batch_log_bound sizes log->out_cap.
 * GOFR_ERR_INVALID: gofr_proto_batch_encode's cases, a null log column (arena may be NULL when every string is empty), a
 * null trace_ids when n > 0, a record whose strings pass arena_bytes, a kind other than GOFR_LOG_RPC / GOFR_LOG_NONE. */
int gofr_proto_batch_encode_log(gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                uint32_t n_fields, uint32_t root, const uint8_t* presence, const gofr_proto_batch* in,
                                const uint8_t* trace_ids, gofr_resp_batch* out, gofr_batch_log* log, gofr_ticket* ticket);

/* Batching front-end (SURVEY.md §8f rank 3): the reference serves one request per goroutine (net/http conn.serve →
 * router.ServeHTTP, pkg/gofr/httpServer.go:29-33); the GPU wants batches.  Any number of threads call
 * gofr_frontend_serve with ONE request each and block until its response is ready; a dispatcher thread closes a batch
 * when it holds max_batch requests or its oldest request has waited max_wait_us, serves it through
 * gofr_batch_submit_slots and wakes the callers.  A small ring of pinned batches rotates (one fills while another is in
 * flight; a batch whose callers are slow to pick up their responses is skipped).  The Date header of a batch is the
 * wall clock at dispatch (gofr_frontend_set_clock pins it for tests).
 * A response longer than slot_bytes is served again on its own through the packed call (same Date), into resp; serve
 * returns GOFR_ERR_CAPACITY (with *resp_len set) only when the response does not fit resp_cap.
 * destroy may only be called when no thread is inside gofr_frontend_serve. */
typedef struct gofr_frontend gofr_frontend;
int gofr_frontend_create(gofr_frontend** out, gofr_engine*, uint32_t max_batch, uint32_t max_wait_us, uint32_t slot_bytes,
                         uint32_t max_request_bytes);
void gofr_frontend_destroy(gofr_frontend*);
int gofr_frontend_set_clock(gofr_frontend*, int64_t unix_seconds);
int gofr_frontend_stats(gofr_frontend*, uint64_t* batches, uint64_t* requests);
int gofr_frontend_serve(gofr_frontend*, uint8_t method, const uint8_t* path, uint16_t path_len, const uint8_t* query,
                        uint16_t query_len, uint8_t flags, const uint8_t* data, uint32_t data_len, const uint8_t trace_id[16],
                        uint8_t* resp, uint32_t resp_cap, uint32_t* resp_len, uint32_t* meta);
/* A front-end whose callers may also ask for their request's RequestLog line: gofr_frontend_create plus log staging of
 * max_log_bytes string bytes per request.  Its batches run through gofr_batch_submit_slots_log when some caller of the
 * batch logs (callers of gofr_frontend_serve ride along as GOFR_LOG_NONE), else through gofr_batch_submit_slots. */
int gofr_frontend_create_log(gofr_frontend** out, gofr_engine*, uint32_t max_batch, uint32_t max_wait_us, uint32_t slot_bytes,
                             uint32_t max_request_bytes, uint32_t max_log_bytes);
/* The log time of every line (unix ns; 0 = the wall clock at dispatch).  gofr_frontend_set_clock keeps pinning the Date. */
int gofr_frontend_set_log_clock(gofr_frontend*, int64_t unix_ns);
/* gofr_frontend_serve plus the request's line by gofr_batch_submit_log's rule.  log: start_unix_ns, tz_offset_s, the five
 * lengths and kind (GOFR_LOG_REQUEST or GOFR_LOG_NONE) are read, arena_off is ignored; strings: the five strings back to
 * back (at most max_log_bytes).  The line goes to line[0 .. *line_len) (empty when the request has none); a line longer
 * than line_cap returns GOFR_ERR_CAPACITY with *line_len set, the response still delivered.  A response longer than its
 * slot is served again alone as gofr_frontend_serve does; its line is the batch's, written once.  GOFR_ERR_INVALID on a
 * front-end made by gofr_frontend_create. */
int gofr_frontend_serve_log(gofr_frontend*, uint8_t method, const uint8_t* path, uint16_t path_len, const uint8_t* query,
                            uint16_t query_len, uint8_t flags, const uint8_t* data, uint32_t data_len, const uint8_t trace_id[16],
                            const gofr_log_desc* log, const uint8_t* strings, uint8_t* resp, uint32_t resp_cap, uint32_t* resp_len,
                            uint32_t* meta, uint8_t* line, uint32_t line_cap, uint32_t* line_len);

/* Batching front-end of the nested proto3 codec: grpc-go calls its codec once per message (encoding.Codec.Unmarshal for a
 * request, Marshal for a response, on the RPC's goroutine; hello_grpc.pb.go:73-89 runs dec(in) between them); the GPU codec
 * wants batches.  Any number of threads call gofr_proto_frontend_call with ONE record each and block until its result is
 * ready; batches close and rotate as gofr_frontend_create's max_batch and max_wait_us say, and run through
 * gofr_proto_batch_decode when decode != 0, else gofr_proto_batch_encode.  One front-end serves one message type (the _ex description, presence may be
 * NULL) in one direction; several front-ends and a gofr_frontend may share an engine (their batches take turns on it).
 *   decode   in is the message as Unmarshal receives it: no 5-byte prefix, already decompressed; out receives the row.  Row
 *            and *status are what gofr_proto_batch_decode gives for the frame 00 | len_be32(m) | m, whatever else is in
 *            the batch: GOFR_GRPC_OK, BAD_PROTO, BAD_UTF8 or DEFER ("decode this one with protobuf-go").
 *   encode   in is a row, zero padded to a multiple of 4 by the front-end; out receives the marshalled message WITHOUT the
 *            prefix (what Marshal returns): gofr_proto_batch_encode's frame for that row minus its first 5 bytes, and its
 *            status: GOFR_GRPC_OK, BAD_UTF8 or BAD_ROW.
 * A failed record has *out_len = 0.  Returns GOFR_OK; GOFR_ERR_CAPACITY before anything is queued when in_len >
 * max_record_bytes (hand the message to protobuf-go); GOFR_ERR_CAPACITY with *out_len (and *status) set when the result does
 * not fit out_cap (the front-end keeps serving); the batch call's own error for every caller of that batch; GOFR_ERR_INVALID
 * for bad arguments and once destroy has started.
 * create checks the description as gofr_proto_nested_bound does (same codes) and refuses (GOFR_ERR_CAPACITY) a max_batch *
 * (per_byte * (max_record_bytes + 5) + per_record) beyond 32 bits (the batch call's output offsets), with per_byte and
 * per_record the bound of the direction.  A batch's pinned output grows to the sum of its records' bounds when that is
 * larger and never shrinks.  destroy may only be called when no thread is inside gofr_proto_frontend_call. */
typedef struct gofr_proto_frontend gofr_proto_frontend;
int gofr_proto_frontend_create(gofr_proto_frontend** out, gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs,
                               const gofr_proto_nfield* fields, uint32_t n_fields, uint32_t root, const uint8_t* presence,
                               int decode, uint32_t max_batch, uint32_t max_wait_us, uint32_t max_record_bytes);
void gofr_proto_frontend_destroy(gofr_proto_frontend*);
int gofr_proto_frontend_stats(gofr_proto_frontend*, uint64_t* batches, uint64_t* records);
int gofr_proto_frontend_call(gofr_proto_frontend*, const uint8_t* in, uint32_t in_len, uint8_t* out, uint32_t out_cap,
                             uint32_t* out_len, uint32_t* status);
/* An encode front-end whose callers may also ask for their call's RPCLog line: gofr_proto_frontend_create plus log
 * staging of max_log_bytes method bytes per call.  Its batches run through gofr_proto_batch_encode_log when some caller of
 * the batch logs (callers of gofr_proto_frontend_call ride along as GOFR_LOG_NONE), else through gofr_proto_batch_encode.
 * The line belongs to the encode direction: decode != 0 is GOFR_ERR_INVALID. */
int gofr_proto_frontend_create_log(gofr_proto_frontend** out, gofr_engine*, const gofr_proto_nmsg* msgs, uint32_t n_msgs,
                                   const gofr_proto_nfield* fields, uint32_t n_fields, uint32_t root, const uint8_t* presence,
                                   int decode, uint32_t max_batch, uint32_t max_wait_us, uint32_t max_record_bytes,
                                   uint32_t max_log_bytes);
/* The log time of every line (unix ns; 0 = the wall clock at dispatch). */
int gofr_proto_frontend_set_log_clock(gofr_proto_frontend*, int64_t unix_ns);
/* gofr_proto_frontend_call plus the call's line by gofr_proto_batch_encode_log's rule.  in: the row, empty for a call
 * whose handler failed (its message and status are then to be ignored; the line is still written).  log: start_unix_ns,
 * elapsed_ns, tz_offset_s, method_len and kind (GOFR_LOG_RPC or GOFR_LOG_NONE) are read, the rest is ignored; method:
 * info.FullMethod, method_len bytes (at most max_log_bytes).  The line goes to line[0 .. *line_len) (empty for
 * GOFR_LOG_NONE); a line longer than line_cap returns GOFR_ERR_CAPACITY with *line_len set, the message still delivered.
 * GOFR_ERR_INVALID on a front-end made by gofr_proto_frontend_create. */
int gofr_proto_frontend_call_log(gofr_proto_frontend*, const uint8_t* in, uint32_t in_len, const uint8_t trace_id[16],
                                 const gofr_log_desc* log, const uint8_t* method, uint8_t* out, uint32_t out_cap, uint32_t* out_len,
                                 uint32_t* status, uint8_t* line, uint32_t line_cap, uint32_t* line_len);

/* HTTP/1.1 request heads (SURVEY.md §8f rank 2): what net/http's readRequest + url.ParseRequestURI hand to
 * Router.ServeHTTP, for a batch of raw request messages resident in HBM, in the layout the serve calls consume.
 *   d_raw / d_raw_off: message i = d_raw[d_raw_off[i] .. d_raw_off[i+1]) — exactly one request (head + body) as framed
 *                      by the connection reader (gofr_http_frame_device below is one: its record column is a d_raw_off);
 *                      d_raw needs 16 readable bytes after the last message.
 *   d_status[i]      : GOFR_HTTP_OK, or GOFR_HTTP_DEFER = "not in the subset below: parse it on the host" (nothing is
 *                      claimed about such a message — it may be perfectly valid).  Never a different answer.
 *   d_desc[i], d_arena: for OK messages the gofr_req_desc and its bytes (decoded URL.Path | URL.RawQuery | pad4 | body) at
 *                      arena_off = d_raw_off[i] rounded up to 4 (the parsed form is never longer than the message, so
 *                      d_arena is a buffer as large as d_raw + 16 and no offsets have to be computed across requests).
 *   d_spans[i][k]    : offset into d_raw | length << 32 of METHOD, TARGET (= RequestURI), USER_AGENT, X_FORWARDED_FOR,
 *                      HOST, BODY — the strings a gofr_log_desc needs come straight from here.
 * The subset (anything else → DEFER): request line `METHOD SP target SP HTTP/1.1 CRLF`; METHOD one of GET HEAD POST PUT
 * PATCH DELETE OPTIONS; target in origin form (`/…`, not `//…`), bytes 0x21–0x7E, no '#', every '%' in the path part
 * followed by two hex digits; header lines `name: value CRLF` with RFC 7230 token names, no leading whitespace (no
 * obs-fold), value bytes HTAB / 0x20–0x7E / ≥ 0x80, CRLF line ends only, head ≤ 16 KiB; exactly one Host header with a
 * non-empty value of [A-Za-z0-9.:_-] and brackets; at most one Content-Length (1–9 digits) and then exactly that many body
 * bytes; or one `Transfer-Encoding: chunked` (no Content-Length beside it) and a chunk stream `hex-size CRLF data CRLF …
 * 0 CRLF CRLF` with sizes of 1–8 hex digits, no chunk extensions, no trailer fields and nothing after it — the arena then
 * holds the de-chunked body, as the handler's io.ReadAll(r.Body) would (BODY span: the chunk stream as received); otherwise
 * no bytes after the head; no Expect, Upgrade or Trailer header; a Connection header only with the value keep-alive.  For such a message URL.Path is the percent-decoded path, URL.RawQuery what follows
 * the first '?', ForceQuery a trailing '?' with nothing after it, header values are trimmed of spaces and tabs. */
enum { GOFR_HTTP_OK = 0, GOFR_HTTP_DEFER = 1 };
enum { GOFR_HTTP_SPAN_METHOD = 0, GOFR_HTTP_SPAN_TARGET = 1, GOFR_HTTP_SPAN_USER_AGENT = 2, GOFR_HTTP_SPAN_XFF = 3,
       GOFR_HTTP_SPAN_HOST = 4, GOFR_HTTP_SPAN_BODY = 5, GOFR_HTTP_SPANS = 6 };
int gofr_http_parse_device(gofr_engine*, const uint8_t* d_raw, const uint32_t* d_raw_off, uint32_t n, gofr_req_desc* d_desc,
                           uint8_t* d_arena, uint32_t* d_status, uint64_t* d_spans, void* stream);

/* Connection byte streams → request messages: the connection reader in front of gofr_http_parse_device (net/http's
 * conn.serve looping readRequest over one bufio.Reader).  A receive buffer holds zero, one or several requests (HTTP/1.1
 * pipelining, or two requests that arrived in one read), then nothing or the first part of the next request.
 *   d_buf / d_buf_off: connection c's received bytes = d_buf[d_buf_off[c] .. d_buf_off[c+1]), back to back; d_buf is 16-byte
 *                      aligned with 16 readable bytes after the last connection (the same buffer is then passed on as d_raw).
 *   d_rec_off        : a record column that TILES the buffer: d_rec_off[0 .. total], ascending, d_rec_off[0] = d_buf_off[0],
 *                      d_rec_off[total] = d_buf_off[n_conns].  A connection's records are its whole requests in order, then
 *                      — only when bytes are left over — one TAIL record with the rest of its buffer.  Records have no gaps,
 *                      so (d_buf, d_rec_off, total) is a valid (d_raw, d_raw_off, n) of gofr_http_parse_device.
 *   d_first          : n_conns + 1 entries; connection c owns records d_first[c] .. d_first[c+1]); d_first[n_conns] = total.
 *   d_consumed[c]    : bytes of the connection covered by whole requests (= the tail's offset in the connection, or the
 *                      connection's length when there is no tail).
 *   d_conn_status[c] : GOFR_HTTP_CONN_DONE  every byte belongs to a whole request; no tail (an empty buffer: no records);
 *                      GOFR_HTTP_CONN_MORE  the last record is a tail that can still become a request of the subset: keep
 *                                           those bytes and append the next read;
 *                      GOFR_HTTP_CONN_DEFER the last record is a tail the subset excludes already (HTTP/1.0, a control byte
 *                                           in a header value, Connection: close, ...): hand the connection's bytes from
 *                                           d_consumed[c] on to net/http.  The framer never resumes behind such a request:
 *                                           where the next one starts is only known when this one's framing is.
 *                      Bytes are judged as they arrive, header lines when they are complete (their CRLF is there).
 *   rec_cap          : d_rec_off has rec_cap + 1 entries.  One record per 16 buffer bytes plus one per connection always
 *                      suffices (the shortest request of the subset is longer).  When total > rec_cap the call behaves like
 *                      the packed-output calls: gofr_engine_overflowed reports it, d_first is still written in full
 *                      (d_first[n_conns] = the capacity needed), records are dropped by whole tiles of 128 connections and
 *                      no entry at or past rec_cap + 1 is written.
 * What makes the column safe to pass on: every non-tail record, given alone to gofr_http_parse_device, is GOFR_HTTP_OK, and
 * every tail record is GOFR_HTTP_DEFER (a zero descriptor) — the host skips the last record of a MORE / DEFER connection.
 * Conversely a message gofr_http_parse_device accepts, followed by anything, is cut at its own length.
 * n_conns == 0 touches no buffer.  GOFR_ERR_INVALID: a null argument, d_buf not 16-byte aligned, a column not 4-byte aligned. */
enum { GOFR_HTTP_CONN_DONE = 0, GOFR_HTTP_CONN_MORE = 1, GOFR_HTTP_CONN_DEFER = 2 };
int gofr_http_frame_device(gofr_engine*, const uint8_t* d_buf, const uint32_t* d_buf_off, uint32_t n_conns,
                           uint32_t* d_rec_off, uint32_t rec_cap, uint32_t* d_first, uint32_t* d_consumed,
                           uint32_t* d_conn_status, void* stream);

/* Connection receive buffers in HOST memory → the bytes to write back to every connection, in one call: frame
 * (gofr_http_frame_device), parse (gofr_http_parse_device), drop the tail records, serve every whole request (the packed
 * layout of gofr_batch_submit), all on the device, chunk after chunk over the engine's streams.  Collect with
 * gofr_batch_wait.
 *   in   buf / buf_off: connection c's received bytes = buf[buf_off[c] .. buf_off[c+1]); buf_off has n_conns + 1
 *        non-decreasing entries, buf_off[n_conns] <= buf_bytes.  date: the batch's IMF-fixdate.  trace_seed: see below.
 *   out  per request k (requests are numbered across the batch, connection after connection, in request order):
 *          out[out_off[k] .. out_off[k+1])  its response (out_off has req_cap + 1 entries);
 *          meta[k]                           as gofr_batch_submit's meta; status 0 = a GOFR_H_HOST route: a hole of no bytes;
 *          req_at[k]                         the request's first byte in buf;
 *          trace_ids[16k .. 16k+16)          its trace id (may be NULL);
 *        per connection c:
 *          req_first[c] .. req_first[c+1])   its requests (req_first has n_conns + 1 entries);
 *          consumed[c], conn_status[c]       as gofr_http_frame_device's d_consumed / d_conn_status;
 *        out_bytes: the response bytes of the batch (filled by submit, reported by wait).
 * Connection c's bytes to write are out[out_off[req_first[c]] .. out_off[req_first[c+1]]), its requests' responses in
 * request order.  A GOFR_H_HOST request is a hole: the caller runs that closure and splices its response in at the request's
 * place; the request's bytes are buf[req_at[k] .. end), end = req_at[k+1] within the connection, or buf_off[c] + consumed[c]
 * for its last request.  Tail records (the last record of a MORE / DEFER connection) are never served and never appear in a
 * per-request column.  A DEFER connection's requests before the deferred one are answered: write their responses, then hand
 * buf[buf_off[c] + consumed[c] ..] to net/http.
 * Trace ids: request j of connection c (j from 0 within the connection, c the connection's index in the batch) gets
 *   x = splitmix64(trace_seed ^ splitmix64(c)), bytes 0-7 = splitmix64(x + 2j), bytes 8-15 = splitmix64(x + 2j + 1),
 * little-endian; a pure function of (trace_seed, c, j), so chunking does not change it.  Pass a fresh seed per batch.
 * Capacity: when req_cap or out_cap is too small, wait returns GOFR_ERR_CAPACITY and nothing is written at or past either
 * capacity; the per-connection columns are still complete, and req_first[n_conns] and out_bytes are what the batch needed.
 * gofr_conn_batch_bound (host only) gives capacities that always suffice for the given offsets.
 * n_conns == 0 touches no buffer.  GOFR_ERR_INVALID: a null argument or column (trace_ids excepted), offsets that decrease
 * or pass buf_bytes.  Offsets are checked chunk by chunk as the batch is enqueued; when a later chunk is refused, the work
 * already enqueued is drained before the call returns and the engine stays usable. */
typedef struct gofr_conn_batch {
    const uint8_t* buf;
    const uint32_t* buf_off;  /* n_conns + 1 */
    uint64_t buf_bytes;
    uint32_t n_conns;
    char date[29];
    uint8_t pad[3];
    uint64_t trace_seed;
} gofr_conn_batch;

typedef struct gofr_conn_resp {
    uint8_t* out;
    uint64_t out_cap;
    uint32_t req_cap;
    uint32_t reserved;
    uint32_t* out_off;      /* req_cap + 1 */
    uint32_t* meta;         /* req_cap */
    uint32_t* req_at;       /* req_cap */
    uint8_t* trace_ids;     /* req_cap * 16, or NULL */
    uint32_t* req_first;    /* n_conns + 1 */
    uint32_t* consumed;     /* n_conns */
    uint32_t* conn_status;  /* n_conns: GOFR_HTTP_CONN_DONE / MORE / DEFER */
    uint64_t out_bytes;
} gofr_conn_resp;

int gofr_conn_batch_submit(gofr_engine*, const gofr_conn_batch* in, gofr_conn_resp* out, gofr_ticket* ticket);
/* Capacities that always suffice for connections with these offsets: one request per 16 buffer bytes plus one per
 * connection, and for the bytes gofr_table_response_bound summed over them (a request's path, query and body are never
 * longer than its record).  No GPU needed.  GOFR_ERR_INVALID: null arguments, offsets that decrease. */
int gofr_conn_batch_bound(const gofr_table*, const uint32_t* buf_off, uint32_t n_conns, uint32_t* req_cap, uint64_t* out_cap);

/* gofr_conn_batch_submit plus middleware.Logging's RequestLog line (gofr_requestlog_device's format) for every request it
 * answers on the device, in the same call.  With log == NULL it is gofr_conn_batch_submit.
 * Which requests get a line: request k has one exactly when GOFR_META_ROUTE(meta[k]) != GOFR_ROUTE_NONE,
 * GOFR_META_STATUS(meta[k]) != 0, and its method, User-Agent, first X-Forwarded-For value and target are each at most
 * 65535 bytes (gofr_log_desc's length fields; the caller logs a longer one, as it logs a hole).  gorilla/mux wraps
 * middleware around matched routes only, so the cleanPath 301 and mux's 404 / 405 are not logged; an OPTIONS request answered by CORS is (status 200: CORS runs inside Logging).  A hole
 * (status 0: a GOFR_H_HOST closure) has no line here: the caller writes it once its closure has set the status.
 * Each line's fields: method, user_agent and uri from the request head (its first User-Agent value, the request target);
 * ip = getIPAddress of the first X-Forwarded-For value, or of the connection's remote string when its first element is
 * empty; response = the status; start_time = start_unix_ns[c] of the request's connection; time = log_unix_ns; id = the
 * request's trace id (the bytes of its X-Correlation-Id header).
 *   in   remote / remote_off: connection c's req.RemoteAddr = remote[remote_off[c] .. remote_off[c+1]), n_conns + 1
 *        non-decreasing offsets, each string at most 255 bytes.  start_unix_ns: n_conns clock readings.
 *        log_unix_ns, tz_offset_s: the logger's clock and time.Local's offset at that instant, for every line.
 *   out  line m = out[log_off[m] .. log_off[m+1]) (log_off has line_cap + 1 entries), lines in request order;
 *        log_req[m] = the batch request index k of line m (ascending; line_cap entries);
 *        lines, out_bytes: the lines and bytes of the batch (filled by submit, reported by wait).
 * Capacity: when line_cap or out_cap is too small, wait returns GOFR_ERR_CAPACITY, nothing is written at or past either
 * capacity, and lines / out_bytes are what the batch needed.  The response columns are complete whenever their own
 * capacities suffice.  gofr_conn_log_bound gives capacities that always suffice.  log_off holds 32-bit offsets: a batch
 * whose lines pass 4 GiB gets GOFR_ERR_CAPACITY whatever out_cap is.
 * A chunk's log strings are placed in one buffer addressed with 32-bit offsets: a chunk whose staged bytes plus one remote
 * string per possible request (one per 16 bytes plus one per connection) would pass 4 GiB is refused with
 * GOFR_ERR_UNSUPPORTED (it takes a single connection of some hundred megabytes).
 * GOFR_ERR_INVALID: gofr_conn_batch_submit's cases, a null log column (remote may be NULL when every string is empty),
 * remote offsets that decrease or a string longer than 255 bytes. */
typedef struct gofr_conn_log {
    const uint8_t* remote;
    const uint32_t* remote_off;    /* n_conns + 1 */
    const int64_t* start_unix_ns;  /* n_conns: Logging's `start := time.Now()` for the connection's requests */
    int64_t log_unix_ns;           /* the logger's time.Now(): response_time = (log_unix_ns - start) / 1000 µs */
    int32_t tz_offset_s;           /* time.Local's offset at that instant, seconds east of UTC */
    uint32_t line_cap;
    uint8_t* out;
    uint64_t out_cap;
    uint32_t* log_off;             /* line_cap + 1 */
    uint32_t* log_req;             /* line_cap */
    uint32_t lines;
    uint32_t reserved;
    uint64_t out_bytes;
} gofr_conn_log;
int gofr_conn_batch_submit_log(gofr_engine*, const gofr_conn_batch* in, gofr_conn_resp* out, gofr_conn_log* log,
                               gofr_ticket* ticket);
/* Capacities that always suffice for gofr_conn_batch_submit_log's lines: one request per 16 buffer bytes plus one per
 * connection, each a line of at most 320 bytes plus 6 per byte of its head and of its connection's remote string.  No GPU
 * needed.  GOFR_ERR_INVALID: null arguments, offsets that decrease, a remote string longer than 255 bytes. */
int gofr_conn_log_bound(const uint32_t* buf_off, const uint32_t* remote_off, uint32_t n_conns, uint32_t* line_cap,
                        uint64_t* out_cap);

/* Connection buffers served with the app's handler closures, in two calls.  Stage 1 frames, parses and routes the buffers
 * on the device and hands back everything a closure needs; the caller runs the closures of the requests whose status is 0
 * and encodes their (data, err) as GOFR_H_RESULT records; stage 2 splices those records in on the device and answers every
 * request of every connection, as gofr_conn_batch_submit_log does.
 *
 * Stage 1 (synchronous): requests are numbered as gofr_conn_batch_submit numbers them, and their trace ids are the same
 * function of (trace_seed, c, j).
 *   out  per request k:
 *          meta[k], vars[k * GOFR_MAX_PATH_VARS ..]  as gofr_route_device gives them: status 301 / 404 / 405 / 200 (OPTIONS),
 *                                                   or 0 = the handler of route GOFR_META_ROUTE(meta[k]) runs;
 *          req_at[k], trace_ids[16k ..]              as gofr_conn_batch_submit's;
 *          desc[k]                                   the parsed request: arena[desc[k].arena_off ..] holds its decoded
 *                                                   URL.Path | URL.RawQuery | pad4 | body (de-chunked), the layout of
 *                                                   gofr_http_parse_device; so (desc, trace_ids, arena) is a valid
 *                                                   gofr_req_batch, which gofr_batch_bind takes for Context.Bind;
 *        per connection c: req_first, consumed, conn_status as gofr_conn_batch_submit's.
 *   arena has buf_bytes + 64 bytes.  A request's parsed form starts at its first byte in buf rounded up to 4 and ends
 *   inside its own message (a message of the subset is longer than its target plus its body plus 6 bytes), so each chunk
 *   copies back exactly the bytes [buf_off[lo], buf_off[hi]) of its connections, at their own offsets; arena bytes that
 *   belong to no request's parsed form are unspecified.
 * Capacity: req_cap as for gofr_conn_batch_submit (gofr_conn_batch_bound).  When it is too small the call returns
 * GOFR_ERR_CAPACITY, req_first[n_conns] is what the batch needed, the per-connection columns are complete and no
 * per-request entry at or past req_cap is written.  GOFR_ERR_INVALID: gofr_conn_batch_submit's cases, a null column.
 *
 * Stage 2 (collect with gofr_batch_wait): in must be the buffers, offsets and trace_seed stage 1 saw.  Record k (requests
 * numbered as in stage 1) is rec[rec_off[k] .. rec_off[k+1]); rec_off has n_req + 1 entries and n_req is stage 1's request
 * count.  A non-empty record replaces request k's data section: a GOFR_H_RESULT record (include/gofr_b200.h, handler kinds),
 * answered by Responder.Respond on the device.  An empty record leaves the request's own body in place, so fused kinds, the
 * router's own answers and GOFR_H_HOST holes are answered exactly as gofr_conn_batch_submit answers them.  out and log are
 * gofr_conn_batch_submit_log's; a request whose record produced a status gets its log line by that call's rule.  With
 * res == NULL the call is gofr_conn_batch_submit_log.
 * Nothing is kept between the stages: stage 2 uploads, frames and parses the buffers again.  It cannot tell buffers that
 * changed since stage 1 from the ones stage 1 saw, other than by their request count: res->n_req must equal it
 * (GOFR_ERR_INVALID otherwise, checked before the last chunk is served).
 * GOFR_ERR_INVALID also for gofr_conn_batch_submit_log's cases, a null rec_off (or a null rec with rec_bytes > 0), record
 * offsets that decrease or pass rec_bytes; these are checked chunk by chunk, and a refused batch leaves the engine usable.
 * GOFR_ERR_UNSUPPORTED: a chunk whose spliced requests (its buffer bytes plus its record bytes plus 8 per request) could
 * pass 4 GiB.  gofr_conn_respond_bound (host only) gives an out_cap that always suffices: the sum of
 * gofr_table_response_bound(path_len, query_len, len) over stage 1's descriptors, len the record's length when it is not
 * empty, else data_len. */
typedef struct gofr_conn_route {
    uint32_t req_cap;
    uint32_t reserved;
    gofr_req_desc* desc;    /* req_cap */
    uint8_t* arena;         /* buf_bytes + 64 */
    uint32_t* meta;         /* req_cap */
    uint32_t* vars;         /* req_cap * GOFR_MAX_PATH_VARS */
    uint32_t* req_at;       /* req_cap */
    uint8_t* trace_ids;     /* req_cap * 16 */
    uint32_t* req_first;    /* n_conns + 1 */
    uint32_t* consumed;     /* n_conns */
    uint32_t* conn_status;  /* n_conns */
} gofr_conn_route;
int gofr_conn_batch_route(gofr_engine*, const gofr_conn_batch* in, gofr_conn_route* out);

typedef struct gofr_conn_results {
    const uint8_t* rec;
    const uint32_t* rec_off;  /* n_req + 1 */
    uint64_t rec_bytes;
    uint32_t n_req;
    uint32_t reserved;
} gofr_conn_results;
int gofr_conn_batch_respond(gofr_engine*, const gofr_conn_batch* in, const gofr_conn_results* res, gofr_conn_resp* out,
                            gofr_conn_log* log, gofr_ticket* ticket);
int gofr_conn_respond_bound(const gofr_table*, const gofr_req_desc* desc, uint32_t n_req, const uint32_t* rec_off,
                            uint64_t* out_cap);
/* Stage 2 with the connections' trace keys given: trace_key[c] (n_conns entries) replaces x = splitmix64(trace_seed ^
 * splitmix64(c)) in gofr_conn_batch_submit's id function for connection c, so request j of connection c gets bytes 0-7 =
 * splitmix64(trace_key[c] + 2j), bytes 8-15 = splitmix64(trace_key[c] + 2j + 1).  That lets a stage 2 batch hold connections
 * from different stage 1 batches, or in another order, and still answer each with the ids its stage 1 handed out (the
 * closures' log lines and the X-Correlation-Id are the same bytes).  With trace_key == NULL it is gofr_conn_batch_respond;
 * everything else is that call's contract. */
int gofr_conn_batch_respond_ex(gofr_engine*, const gofr_conn_batch* in, const uint64_t* trace_key, const gofr_conn_results* res,
                               gofr_conn_resp* out, gofr_conn_log* log, gofr_ticket* ticket);

/* Batching front-end over gofr_conn_batch_submit_log: net/http runs one goroutine per connection (conn.serve looping
 * readRequest, pkg/gofr/httpServer.go:29-33), each holding only its own received bytes.  Any number of threads call
 * gofr_conn_frontend_serve with ONE read of one connection each (the kept tail plus the new bytes) and block until the batch
 * it joined has been served; batches close and rotate as gofr_frontend_create's max_batch and max_wait_us say.
 * What a call returns is what gofr_conn_batch_submit_log returns for that connection as a batch of one (n_conns = 1), except
 * for the trace ids:
 *   out  out[out_off[k] .. out_off[k+1]) is request k's response (offsets from the caller's out), meta[k], req_at[k] (the
 *        request's first byte in buf), trace_ids[16k ..] (may be NULL); req_first[0..1] = {0, requests}, consumed[0],
 *        conn_status[0] (GOFR_HTTP_CONN_DONE / MORE / DEFER) and out_bytes.  Holes (status 0) and DEFER mean what they mean
 *        for the batch call: serve a hole from buf[req_at[k] ..]; on DEFER write the responses, then hand buf[consumed[0] ..]
 *        to net/http; on MORE keep buf[consumed[0] ..] and append the next read to it.
 *   log  when log != NULL and the front-end was created with log != 0: the connection's lines in the output fields of
 *        gofr_conn_log, where log_req[m] indexes this call's requests; its input fields are ignored: remote (at most 255 bytes) and
 *        start_unix_ns (Logging's `start := time.Now()` for this read) are arguments, log time and zone the front-end's.
 *        Otherwise lines and out_bytes are 0.
 * Per batch: Date and log_unix_ns are the wall clock at dispatch (gofr_conn_frontend_set_clock pins them, in ns; 0 = wall
 * clock), and trace_seed = splitmix64(splitmix64(seed) + batch number), batches numbered from 0; the connection in slot c of
 * the batch gets gofr_conn_batch_submit's ids for (trace_seed, c, j).  Each id is the bytes of its response's X-Correlation-Id.
 * Returns GOFR_OK; at once, without joining a batch, for len == 0 (conn_status DONE, no requests); GOFR_ERR_CAPACITY before
 * anything is queued when len > max_conn_bytes (hand the connection to net/http); GOFR_ERR_CAPACITY with req_first[1],
 * out_bytes and the log's lines / out_bytes set to what the connection needed when the caller's req_cap, out_cap, line_cap
 * or log out_cap is short (columns whose capacities suffice are complete; the front-end keeps serving;
 * gofr_conn_batch_bound / gofr_conn_log_bound on {0, len} give capacities that always suffice); the batch call's own error
 * for every caller of that batch; GOFR_ERR_INVALID for bad arguments and once destroy has started.
 * One call per connection at a time.  A batch's response and log outputs grow when the batch call reports more than they
 * hold (the batch is then served again, counted in stats' reruns) and never shrink.  create refuses (GOFR_ERR_CAPACITY) a
 * max_batch * max_conn_bytes beyond 32 bits.  destroy may only be called when no thread is inside gofr_conn_frontend_serve. */
typedef struct gofr_conn_frontend gofr_conn_frontend;
int gofr_conn_frontend_create(gofr_conn_frontend** out, gofr_engine*, uint32_t max_batch, uint32_t max_wait_us,
                              uint32_t max_conn_bytes, int log, int32_t tz_offset_s, uint64_t seed);
void gofr_conn_frontend_destroy(gofr_conn_frontend*);
int gofr_conn_frontend_set_clock(gofr_conn_frontend*, int64_t unix_ns);
int gofr_conn_frontend_stats(gofr_conn_frontend*, uint64_t* batches, uint64_t* conns, uint64_t* reruns);
int gofr_conn_frontend_serve(gofr_conn_frontend*, const uint8_t* buf, uint32_t len, const uint8_t* remote, uint32_t remote_len,
                             int64_t start_unix_ns, gofr_conn_resp* out, gofr_conn_log* log);

/* Batching front-end over the closure path (gofr_conn_batch_route → closures → gofr_conn_batch_respond_ex), one read of one
 * connection per call, with the closures on the caller's thread: net/http's conn.serve runs the user's closure on the
 * connection's goroutine (pkg/gofr/httpServer.go:29-33, handler.go:32-36).  A read takes two calls, each a blocking call
 * that joins a batch of its own kind, batches closing and rotating as gofr_frontend_create's max_batch and max_wait_us say:
 *   route    the read → its requests routed, parsed and, for routes that declared a bind schema, bound; and its trace key;
 *   (the caller runs the closures of its status-0 requests and encodes their (data, err) as GOFR_H_RESULT records)
 *   respond  the same read, its trace key and its records → its responses and log lines.
 * Route batches and respond batches are independent: a respond batch holds connections from any route batches, and a
 * connection's response never waits for another connection's closure (a closure may call back into the front-end).  The
 * front-end holds nothing for a read between its two calls: a caller that routes and never responds costs nothing.
 *
 * route: what gofr_conn_batch_route returns for this connection as a batch of one, rebased to the caller's buffers:
 *   out  desc[k], meta[k], vars[k * GOFR_MAX_PATH_VARS ..], req_at[k] (the request's first byte in buf), trace_ids[16k ..];
 *        req_first[0..1] = {0, requests}, consumed[0], conn_status[0].  arena holds len + 80 bytes; desc[k].arena_off indexes
 *        it, and each parsed form keeps the alignment gofr_conn_batch_route gives it (the forms are moved by a multiple of 16),
 *        so (desc, trace_ids, arena) with arena_bytes = len + 80 is a valid gofr_req_batch.
 *   bind (may be NULL) Context.Bind of every status-0 request whose route route_schema maps to a schema (done for the whole
 *        batch with one gofr_batch_bind per schema): status[k] = GOFR_BIND_OK / ERROR / HOST, or 0xFFFFFFFF for a request
 *        that was not bound; its row (GOFR_BIND_OK) or error text (GOFR_BIND_ERROR) is rows[row_off[k] .. row_off[k+1]).
 *        A row longer than its first slot is bound again in a slot of the length reported for it (a row that would not fit
 *        even that one comes back GOFR_BIND_HOST with no bytes; gofr_batch_bind reports exact lengths, so it never does).
 *        rows_bytes is what the rows take; GOFR_BIND_ROW_BOUND summed over the requests always suffices, and so does
 *        req_cap * (8 * fields + 70 + names) + 3 * len, with fields and names those of the widest schema.
 *   *trace_key  splitmix64(trace_seed_b ^ splitmix64(slot)), the x of gofr_conn_batch_submit's id function for this read:
 *        trace_seed_b = splitmix64(splitmix64(seed) + route batch number), batches numbered from 0, slot the read's place in
 *        its route batch.  trace_ids are the ids of that key; hand it to respond.
 * respond: what gofr_conn_frontend_serve returns for this read (out and log as there), with the records res spliced in as
 *   gofr_conn_batch_respond splices them: res->n_req is the route call's request count and res->rec_off its n_req + 1 record
 *   offsets into res->rec.  The ids are trace_key's, so each X-Correlation-Id and log line carries the id the route call
 *   returned.  Date and log_unix_ns are the respond batch's (gofr_conn_app_frontend_set_clock pins them, in ns; 0 = wall
 *   clock); start_unix_ns is this read's.
 * Returns GOFR_OK; at once, without joining a batch, for len == 0 (conn_status DONE, no requests; respond wants n_req == 0);
 * GOFR_ERR_CAPACITY before anything is queued when len > max_conn_bytes (hand the connection to net/http); GOFR_ERR_CAPACITY
 * with req_first[1] (route), rows_bytes, out_bytes and the log's lines / out_bytes set to what the read needed when one of
 * the caller's capacities is short (gofr_conn_batch_bound / gofr_conn_log_bound on {0, len} give capacities that always
 * suffice); the batch call's own error for every caller of that batch; GOFR_ERR_INVALID for bad arguments and once destroy
 * has started.  respond also returns GOFR_ERR_INVALID, before queuing, for records whose offsets decrease or pass rec_bytes,
 * and, without failing its batch-mates, for records that do not match the read's requests (a wrong n_req, or bytes that
 * changed the request count since the route call): such a batch is served once more without records to count each read's
 * requests, and again without the offenders' records (stats: isolated).  A respond batch gathers its callers' records
 * behind 32-bit offsets: a caller whose records, with those of the callers before it in the batch, would bring the batch's
 * records plus its bytes plus 8 per possible request past 4 GiB gets GOFR_ERR_CAPACITY without failing the others (respond
 * again; records that pass that alone are never served).
 * One call per connection at a time.  Respond batches' outputs grow and are served again as gofr_conn_frontend's (stats:
 * reruns).  create: route_schema[r] (n_routes entries, may be NULL when n_routes is 0) is the schema route r binds, 0 for
 * none, and schema_fields[r] that schema's field count; refuses (GOFR_ERR_CAPACITY) a max_batch * max_conn_bytes beyond 32
 * bits.  destroy may only be called when no thread is inside a route or respond call. */
typedef struct gofr_conn_app_frontend gofr_conn_app_frontend;
typedef struct gofr_conn_app_bind {
    uint32_t* status;     /* req_cap */
    uint32_t* row_off;    /* req_cap + 1 */
    uint8_t* rows;
    uint64_t rows_cap;
    uint64_t rows_bytes;
} gofr_conn_app_bind;
typedef struct gofr_conn_app_stats {
    uint64_t route_batches, route_reads, respond_batches, respond_reads;
    uint64_t reruns;      /* respond batches served again after an output grew */
    uint64_t isolated;    /* respond batches served once more to count their reads' requests */
    uint64_t gather_ns;   /* the respond dispatcher's time gathering the callers' records */
} gofr_conn_app_stats;
int gofr_conn_app_frontend_create(gofr_conn_app_frontend** out, gofr_engine*, uint32_t max_batch, uint32_t max_wait_us,
                                  uint32_t max_conn_bytes, int log, int32_t tz_offset_s, uint64_t seed, const uint32_t* route_schema,
                                  uint32_t n_routes, const uint32_t* schema_fields);
void gofr_conn_app_frontend_destroy(gofr_conn_app_frontend*);
int gofr_conn_app_frontend_set_clock(gofr_conn_app_frontend*, int64_t unix_ns);
int gofr_conn_app_frontend_stats(gofr_conn_app_frontend*, gofr_conn_app_stats* stats);
int gofr_conn_app_frontend_route(gofr_conn_app_frontend*, const uint8_t* buf, uint32_t len, gofr_conn_route* out,
                                 gofr_conn_app_bind* bind, uint64_t* trace_key);
int gofr_conn_app_frontend_respond(gofr_conn_app_frontend*, const uint8_t* buf, uint32_t len, uint64_t trace_key,
                                   const gofr_conn_results* res, const uint8_t* remote, uint32_t remote_len, int64_t start_unix_ns,
                                   gofr_conn_resp* out, gofr_conn_log* log);

/* number of kernels launched by this engine so far (bench.py reports it as gpu_launches) */
uint64_t gofr_engine_launch_count(const gofr_engine*);
/* duration in ms of the kernels launched since the last reset, measured with CUDA events on the launch stream.  Every
 * kernel is timed except the two copy kernels of gofr_batch_submit's pinned-buffer path (chunk bookkeeping and egress
 * into the caller's buffers, on the engine's own streams).
 * Timing is OFF by default (each timed launch costs two event objects): gofr_engine_set_timing(e, 1) first. */
int gofr_engine_kernel_time_ms(gofr_engine*, double* total_ms, uint64_t* launches, int reset);

const char* gofr_last_error(void);
uint32_t gofr_abi_version(void);
void gofr_format_http_date(int64_t unix_seconds, char out29[29]);

#ifdef __cplusplus
}
#endif
#endif /* GOFR_B200_H */
