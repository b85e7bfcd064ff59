// engine.cu — per-GPU execution context behind the C ABI (include/gofr_b200.h).
//
// Stands where net/http's conn.serve → router.ServeHTTP sits in the reference (pkg/gofr/httpServer.go:29-33): the
// caller hands over a batch of parsed requests and gets the response bytes back.  Two entry styles:
//   gofr_serve_device   — everything already in HBM; one fused launch on the caller's stream;
//   gofr_batch_submit/_wait — host buffers; the batch is cut into chunks that flow through a 3-deep
//                         H2D → kernel → D2H pipeline on the engine's own streams (copy engines overlap the kernel).
// There is no CPU fallback: without a CUDA device engine creation fails with GOFR_ERR_NO_DEVICE.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <functional>
#include <initializer_list>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/gofr_b200.h"
#include "engine_internal.h"
#include "table_format.h"

static thread_local char g_err[512];

void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}

#define CUDA_TRY(expr)                                                                       \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return GOFR_ERR_CUDA;                                                            \
        }                                                                                    \
    } while (0)

using namespace gofr;

namespace gofr {
// The kernels (defined in the *_kernel.cu translation units; launched from here through launch()).
__global__ void serve_kernel(const ServeParams p);               // serve_kernel.cu: packed layout
__global__ void serve_kernel_values(const ServeParams p);        // serve_values_kernel.cu: packed, PF_VALUES programs
__global__ void serve_slots_kernel(const ServeParams p);         // serve_slots_kernel.cu: slot layout, 5 CTAs/SM
__global__ void serve_slots_kernel_wide(const ServeParams p);    // serve_slots_wide_kernel.cu: slot layout, 4 CTAs/SM
__global__ void serve_slots_kernel_values(const ServeParams p);  // serve_slots_values_kernel.cu: slot layout, PF_VALUES
__global__ void grpc_hello_kernel(const GrpcParams p);           // grpc_kernel.cu
__global__ void proto_encode_kernel(const GrpcParams p, const ProtoSchema S);
__global__ void proto_decode_kernel(const GrpcParams p, const ProtoSchema S);
__global__ void proto_encode_nested_kernel(const GrpcParams p, const PbnDesc D);  // proto_nested_kernel.cu
__global__ void proto_decode_nested_kernel(const GrpcParams p, const PbnDesc D);  // proto_nested_decode_kernel.cu
__global__ void proto_encode_nested_maps_kernel(const GrpcParams p, const PbnDesc D);  // proto_nested_maps_kernel.cu: the
__global__ void proto_decode_nested_maps_kernel(const GrpcParams p, const PbnDesc D);  // same for descriptions with maps
__global__ void proto_encode_nested_presence_kernel(const GrpcParams p, const PbnDesc D);  // proto_nested_presence_kernel.cu:
__global__ void proto_decode_nested_presence_kernel(const GrpcParams p, const PbnDesc D);  // with explicit presence (and maps)
__global__ void proto_decode_nested_deferred_kernel(const GrpcParams p, const uint32_t* meta_in, const PbnDesc D);  // proto_nested_deferred_kernel.cu
__global__ void reqlog_kernel(const LogParams p);                // reqlog_kernel.cu
__global__ void batch_log_kernel(const LogParams p, const uint32_t* meta, int64_t log_ns, unsigned long long* lines);  // batch_log_kernel.cu
__global__ void proto_log_kernel(const LogParams p, int64_t log_ns, unsigned long long* lines);  // proto_log_kernel.cu
__global__ void http_parse_kernel(const HttpParams p);           // http_kernel.cu
__global__ void http_frame_kernel(const HttpFrameParams p);      // http_frame_kernel.cu
__global__ void conn_compact_kernel(const ConnParams p);         // conn_kernel.cu
__global__ void conn_log_kernel(const ConnLogParams p);          // conn_log_kernel.cu
__global__ void conn_result_kernel(const ConnResultParams p);    // conn_result_kernel.cu
__global__ void route_kernel(const RouteParams p);               // route_kernel.cu
__global__ void bind_kernel(const BindParams p);                 // bind_kernel.cu
__global__ void chunk_pack_kernel(const PackParams p);           // pack_kernel.cu
}  // namespace gofr

namespace {

enum Kern {
    K_SERVE, K_SERVE_VALUES, K_SLOTS, K_SLOTS_WIDE, K_SLOTS_VALUES, K_HELLO, K_PROTO_ENC, K_PROTO_DEC, K_PBN_ENC, K_PBN_DEC,
    K_PBN_ENC_MAPS, K_PBN_DEC_MAPS, K_PBN_ENC_PRES, K_PBN_DEC_PRES, K_PBN_DEC_DEFERRED, K_REQLOG, K_HTTP, K_HTTP_FRAME, K_ROUTE, K_BIND, K_PACK,
    K_CONN, K_CONN_LOG, K_CONN_RESULT, K_BATCH_LOG, K_PROTO_LOG,
    K_COUNT
};
struct KernelRec {
    const void* fn;
    const char* what;  // in error messages: "<what> kernel launch failed"
    int threads;
};
const KernelRec kKernels[K_COUNT] = {
    {(const void*)serve_kernel, "serve", kServeT},
    {(const void*)serve_kernel_values, "serve", kServeT},
    {(const void*)serve_slots_kernel, "serve", kServeT},
    {(const void*)serve_slots_kernel_wide, "serve", kServeT},
    {(const void*)serve_slots_kernel_values, "serve", kServeT},
    {(const void*)grpc_hello_kernel, "grpc", kServeThreads},
    {(const void*)proto_encode_kernel, "proto", kServeThreads},
    {(const void*)proto_decode_kernel, "proto", kServeThreads},
    {(const void*)proto_encode_nested_kernel, "proto", kServeThreads},
    {(const void*)proto_decode_nested_kernel, "proto", kServeThreads},
    {(const void*)proto_encode_nested_maps_kernel, "proto", kServeThreads},
    {(const void*)proto_decode_nested_maps_kernel, "proto", kServeThreads},
    {(const void*)proto_encode_nested_presence_kernel, "proto", kServeThreads},
    {(const void*)proto_decode_nested_presence_kernel, "proto", kServeThreads},
    {(const void*)proto_decode_nested_deferred_kernel, "proto", kServeThreads},
    {(const void*)reqlog_kernel, "request-log", kServeThreads},
    {(const void*)http_parse_kernel, "http", kServeThreads},
    {(const void*)http_frame_kernel, "http-frame", kServeThreads},
    {(const void*)route_kernel, "route", kRouteThreads},
    {(const void*)bind_kernel, "bind", kBindThreads},
    {(const void*)chunk_pack_kernel, "pack", kServeThreads},
    {(const void*)conn_compact_kernel, "connection compact", kServeThreads},
    {(const void*)conn_log_kernel, "connection log", kServeThreads},
    {(const void*)conn_result_kernel, "connection result", kServeThreads},
    {(const void*)batch_log_kernel, "batch log", kServeThreads},
    {(const void*)proto_log_kernel, "proto log", kServeThreads},
};

constexpr int kSlots = 3;  // pipeline depth of the host-batch path

// Look-back scratch of the kernels that pack their output: one state word per tile of a launch (tile_common.cuh).
struct TileState {
    unsigned long long* words = nullptr;
    size_t tiles = 0;
};

struct Slot {
    cudaEvent_t done = nullptr;
    cudaEvent_t ev_h2d = nullptr, ev_served = nullptr, ev_egress = nullptr;  // the chunk pipeline
    bool egress_pending = false;
    // device buffers (grown on demand)
    void* d_desc = nullptr; void* d_ids = nullptr; uint8_t* d_arena = nullptr; uint8_t* d_out = nullptr;
    uint32_t* d_off = nullptr; uint32_t* d_meta = nullptr;
    uint32_t* d_flag = nullptr; uint32_t* d_bind = nullptr;
    TileState state;  // packed layout only
    size_t cap_n = 0, cap_arena = 0, cap_out = 0;
    // proto host path (grown on demand): the input offsets, the codec kernels' own outputs and offset columns (decode: [0]
    // the first pass, [1] the second) and the first pass's statuses
    uint32_t* d_in_off = nullptr; uint32_t* d_meta1 = nullptr;
    uint8_t* d_codec[2] = {nullptr, nullptr}; uint32_t* d_codec_off[2] = {nullptr, nullptr};
    size_t cap_codec_n = 0, cap_codec[2] = {0, 0};
    // connection host path (grown on demand): the staged receive buffers and their offsets, the framer's per-connection
    // columns and compacted req_first (per connection), its record column, and the request-head kernel's outputs and the
    // compacted req_at (per record)
    uint8_t* d_buf = nullptr; uint32_t* d_buf_off = nullptr;
    uint32_t* d_first = nullptr; uint32_t* d_cstatus = nullptr; uint32_t* d_consumed = nullptr; uint32_t* d_req_first = nullptr;
    uint32_t* d_rec = nullptr; void* d_pdesc = nullptr; uint32_t* d_pstatus = nullptr; unsigned long long* d_spans = nullptr;
    uint32_t* d_req_at = nullptr;
    uint64_t* d_tkey = nullptr;  // gofr_conn_batch_respond_ex: the chunk's per-connection trace keys
    size_t cap_buf = 0, cap_conns = 0, cap_recs = 0;
    // its request-log lines (grown on demand): the staged remote strings, their offsets and the start clocks (per
    // connection), the gather's per-connection line column, its descriptors, trace ids and request indices and the
    // reqlog and pack offset columns (per line), the log arena, the reqlog kernel's lines and the packed lines
    uint8_t* d_remote = nullptr; uint32_t* d_remote_off = nullptr; int64_t* d_start = nullptr; uint32_t* d_lfirst = nullptr;
    void* d_ldesc = nullptr; uint8_t* d_lids = nullptr; uint32_t* d_lreq = nullptr; uint32_t* d_lraw_off = nullptr; uint32_t* d_loff = nullptr;
    uint8_t* d_larena = nullptr; uint8_t* d_lraw = nullptr; uint8_t* d_lout = nullptr;
    size_t cap_remote = 0, cap_lconns = 0, cap_lrecs = 0, cap_larena = 0, cap_lraw = 0, cap_lout = 0;
    // the closures' results (gofr_conn_batch_respond, grown on demand): the chunk's record bytes, their offsets and the
    // spliced arena's offset column (per request), the spliced arena; gofr_conn_batch_route: the path variables
    uint8_t* d_rbytes = nullptr; uint32_t* d_roff = nullptr; uint32_t* d_soff = nullptr; uint8_t* d_sarena = nullptr;
    uint32_t* d_vars = nullptr;
    size_t cap_rbytes = 0, cap_rreqs = 0, cap_sarena = 0, cap_vars = 0;
    // pinned staging for the tiny per-chunk read-backs
    uint32_t* h_tail = nullptr;  // [2k] = a pageable output k's chunk size (connections: [0] records, [2] log lines); [2k + 1] = output k's overflow word

    int reserve(gofr_engine* e, uint32_t requests, size_t arena_bytes, size_t out_bytes);
    int reserve_codec(uint32_t records, size_t a_bytes, size_t b_bytes);
    int reserve_conn(uint32_t conns, uint32_t records, size_t buf_bytes);
    int reserve_log(uint32_t conns, uint32_t records, size_t remote_bytes);
    int reserve_lines(uint32_t lines);
    int reserve_line_bytes(size_t arena_bytes, uint64_t line_bytes);
};

}  // namespace

struct gofr_engine {
    int device = 0;
    int sm_count = 0;
    ImageHeader hdr;
    std::vector<uint32_t> schema_ids;  // the table's schema ids in table order
    std::vector<uint16_t> schema_flags;  // SchemaRec::flags, same order
    uint8_t* d_image = nullptr;
    uint32_t image_bytes = 0;
    // launch geometry
    uint32_t in_cap = 0, smem_bytes = 0;
    uint32_t w_in_cap = 0, w_smem_bytes = 0;  // the same for the wide slot-layout instance (4 CTAs/SM: a larger staging area fits)
    int wide_grid = 0, wide_blocks_per_sm = 0;
    bool slots_wide = false;  // choose_slot_residency
    bool has_values = false;  // some program has PF_VALUES: the packed layout runs serve_kernel_values (serve_values_kernel.cu)
    int grid = 0, blocks_per_sm = 0;
    int resident[K_COUNT] = {};  // resident grid of each kernel without dynamic shared memory, asked once (resident_grid)
    uint32_t epoch = 0;
    // resident path scratch
    TileState state;
    uint32_t* d_flag = nullptr;
    uint32_t* d_bind = nullptr;  // Bind scratch of the resident path
    size_t bind_cap = 0;
    // host path
    Slot slots[kSlots];
    cudaStream_t st_h2d = nullptr, st_compute = nullptr, st_egress = nullptr;
    cudaEvent_t ev_batch_done = nullptr;  // blocking-sync event: the caller's thread SLEEPS until its batch is back (a
                                          // spinning cudaStreamSynchronize per rank burns the CPU quota eight ranks share)
    unsigned long long* d_chain = nullptr;  // packed position of the batch in flight; [2] its log lines (gofr_batch_submit_log)
    ChunkInfo* d_info = nullptr;            // two per slot: [slot] the responses, [kSlots + slot] the request-log lines
    unsigned long long* h_status = nullptr; // pinned: [0] total bytes, [1] overflow; [2], [3] the same for the log lines;
                                            // [4] the log line count of gofr_batch_submit_log
    uint32_t* h_ends = nullptr;             // pinned, calls that report what they needed: per posted chunk its first and end
                                            // response offsets, then its first and end log line offsets (PackedOut::post)
    size_t ends_cap = 0;                    // (words)
    int egress_grid = 37;
    uint32_t chunk = 65536;
    std::mutex mu;
    uint64_t launches = 0;
    // kernel timing (events on the launch stream)
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timing;
    bool timing_on = false;  // off by default: each timed launch costs two event objects (gofr_engine_set_timing)
    uint32_t debug_flags = 0;  // GOFR_DEBUG_* environment switches, read once at creation
    double timed_ms = 0;
    uint64_t timed_launches = 0;
    // gofr_batch_route scratch (host-buffer stage 1 of the split API)
    uint8_t* d_rt_desc = nullptr; uint8_t* d_rt_arena = nullptr; uint8_t* d_rt_meta = nullptr; uint8_t* d_rt_vars = nullptr;
    size_t rt_desc_cap = 0, rt_arena_cap = 0, rt_meta_cap = 0, rt_vars_cap = 0;
    uint8_t* d_rt_rows = nullptr;  // gofr_batch_bind: result slots
    size_t rt_rows_cap = 0;
    // tickets
    // tickets of finished submits whose result has not been collected yet (submit completes the batch; wait reports)
    std::vector<std::pair<gofr_ticket, int>> done_tickets;
    gofr_ticket next_ticket = 1;
};

// Engines alive per device in this process.  The packed-layout kernels chain their tiles with a look-back that is only
// deadlock free when every CTA of the grid is resident at once (tile t waits for tiles < t, all owned by resident CTAs).
// A grid sized for the whole GPU is not co-resident with a second engine's grid on the same device, so every engine
// launches its look-back kernels with the device's capacity divided by the number of live engines on it.  Other processes
// on the same GPU (MPS) are not visible from here: INTEGRATION.md says one serving process per GPU.
static std::mutex g_reg_mu;
static int g_live_engines[64];
static int engines_on_device(int device) {
    std::lock_guard<std::mutex> g(g_reg_mu);
    const int k = device >= 0 && device < 64 ? g_live_engines[device] : 1;
    return k > 0 ? k : 1;
}
static void register_engine(int device, int delta) {
    std::lock_guard<std::mutex> g(g_reg_mu);
    if (device >= 0 && device < 64) g_live_engines[device] += delta;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to a kernel on a device, so it is shared by every engine there.  It
// is only ever raised: once a launch or an occupancy query has made sure it covers some size, it keeps covering it.
static std::mutex g_attr_mu;
static uint32_t g_smem_attr[K_COUNT][64];
static cudaError_t cover_smem(Kern k, int device, uint32_t smem) {
    std::lock_guard<std::mutex> g(g_attr_mu);
    const bool cached = device >= 0 && device < 64;
    if (cached && smem <= g_smem_attr[k][device]) return cudaSuccess;
    const cudaError_t er = cudaFuncSetAttribute(kKernels[k].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (er == cudaSuccess && cached) g_smem_attr[k][device] = smem;
    return er;
}

// CTAs of kernel k resident per SM with `smem` bytes of dynamic shared memory, asked from the runtime; -1 if it cannot say.
static int blocks_per_sm(Kern k, int device, uint32_t smem) {
    int nb = 0;
    if (cover_smem(k, device, smem) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kKernels[k].fn, kKernels[k].threads, smem) != cudaSuccess) return -1;
    return nb;
}

// The serve kernel's five instances: the layout (packed or slots), the programs the table has (PF_VALUES or not) and, for
// the slot layout, the register budget (the wide 4-CTA instance or the 5-CTA one) pick one.
static Kern serve_instance(bool slots, bool values, bool wide) {
    if (!slots) return values ? K_SERVE_VALUES : K_SERVE;
    return values ? K_SLOTS_VALUES : wide ? K_SLOTS_WIDE : K_SLOTS;
}

static uint32_t serve_smem_bytes(uint32_t hot_bytes, uint32_t in_cap) { return ((hot_bytes + 127u) & ~127u) + in_cap + 64; }

// CTAs per SM with which every instance of a residency group is resident for `smem` bytes of dynamic shared memory: the wide
// slot-layout instance alone, or all the others (packed / slots, with and without the wider data model).  Asked from the
// runtime (static shared memory, registers and the per-CTA reservation included) — a hand-kept formula fell behind the
// kernel once and the "5-CTA" instances silently ran 4 per SM.
static int serve_blocks_per_sm(int device, uint32_t smem, bool wide) {
    if (wide) return blocks_per_sm(K_SLOTS_WIDE, device, smem);
    int nb = 1 << 30;
    for (Kern k : {K_SERVE, K_SLOTS, K_SLOTS_VALUES, K_SERVE_VALUES}) {
        const int b = blocks_per_sm(k, device, smem);
        if (b < 0) return -1;
        nb = std::min(nb, b);
    }
    return nb;
}

// The largest request staging budget (bytes per request: a multiple of 16 from 16 to 256) with which `ctas` CTAs of the
// group stay resident per SM next to a table of hot_bytes; 0 when not even the smallest one fits.
static uint32_t serve_fit_in_per(int device, uint32_t hot_bytes, int ctas, bool wide) {
    for (uint32_t in_per = 256; in_per >= 16; in_per -= 16) {
        const uint32_t smem = serve_smem_bytes(hot_bytes, ((uint32_t)kServeT * in_per + 127u) & ~127u);
        if (smem > 227u * 1024u) continue;
        if (serve_blocks_per_sm(device, smem, wide) >= ctas) return in_per;
    }
    return 0;
}

// Which slot-layout instance serves this table (serve_slots_kernel.cu): the wide one (4 CTAs/SM, 128 registers) for tables
// whose live routes all answer through the template fast path with one program shape (image_wants_wide_slots,
// table_build.cpp), the 5-CTA one otherwise; GOFR_SLOT_CTAS=4 / 5 (or gofr_engine_slot_ctas) forces one.  On an H100 SXM
// (400 W power limit) the wide instance serves the 1 Mi config-2 batch in 0.821 ms against 0.854 ms for the 5-CTA one.
static bool choose_slot_residency(const std::vector<uint8_t>& img, const ImageHeader&) {
    if (const char* v = getenv("GOFR_SLOT_CTAS")) return atoi(v) == kServeCtasWide;
    return image_wants_wide_slots(img.data());
}

// in_per_req / w_in_per_req: bytes of request staging per request for the 5-CTA instances / the wide slot-layout instance
static int configure_geometry(gofr_engine* e, uint32_t in_per_req, uint32_t w_in_per_req) {
    // the slot layout keeps its deferred-request list (2 T words) in the staging area
    if (in_per_req < 16u) in_per_req = 16u;
    if (w_in_per_req < 16u) w_in_per_req = 16u;
    e->in_cap = (kServeT * in_per_req + 127u) & ~127u;
    e->smem_bytes = serve_smem_bytes(e->hdr.hot_bytes, e->in_cap);
    e->w_in_cap = (kServeT * w_in_per_req + 127u) & ~127u;
    e->w_smem_bytes = serve_smem_bytes(e->hdr.hot_bytes, e->w_in_cap);
    if (e->smem_bytes > 227 * 1024 || e->w_smem_bytes > 227 * 1024) { set_last_error("tile geometry needs %u bytes of shared memory", std::max(e->smem_bytes, e->w_smem_bytes)); return GOFR_ERR_CAPACITY; }
    e->blocks_per_sm = serve_blocks_per_sm(e->device, e->smem_bytes, false);
    if (e->blocks_per_sm <= 0) { set_last_error("serve kernel cannot be resident with %u bytes of shared memory", e->smem_bytes); return GOFR_ERR_CUDA; }
    e->grid = e->blocks_per_sm * e->sm_count;
    e->wide_blocks_per_sm = serve_blocks_per_sm(e->device, e->w_smem_bytes, true);
    e->wide_grid = std::max(0, e->wide_blocks_per_sm * e->sm_count);  // the wide instance is optional: the engine falls back to the others
    return GOFR_OK;
}

extern "C" {

static int engine_init(gofr_engine* e, const std::vector<uint8_t>& img, int device);

int gofr_engine_create(gofr_engine** out, const gofr_table* t, int device) {
    if (!out || !t) return GOFR_ERR_INVALID;
    const std::vector<uint8_t>& img = gofr_table_image(t);
    if (img.empty()) return GOFR_ERR_NOT_SEALED;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        set_last_error("no CUDA device: gofr_b200 has no CPU path");
        return GOFR_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= ndev) return GOFR_ERR_INVALID;
    CUDA_TRY(cudaSetDevice(device));
    gofr_engine* e = new gofr_engine();
    register_engine(device, +1);
    e->device = device;
    const int rc_create = engine_init(e, img, device);
    if (rc_create != GOFR_OK) { gofr_engine_destroy(e); return rc_create; }  // releases whatever the failed step left behind
    *out = e;
    return GOFR_OK;
}

static int engine_init(gofr_engine* e, const std::vector<uint8_t>& img, int device) {
    e->device = device;
    memcpy(&e->hdr, img.data(), sizeof(ImageHeader));
    e->schema_ids.resize(e->hdr.n_schemas);
    if (e->hdr.n_schemas) memcpy(e->schema_ids.data(), img.data() + e->hdr.schema_ids_off, (size_t)e->hdr.n_schemas * 4);
    e->schema_flags.resize(e->hdr.n_schemas);
    for (uint32_t k = 0; k < e->hdr.n_schemas; k++)
        e->schema_flags[k] = reinterpret_cast<const SchemaRec*>(img.data() + e->hdr.schemas_off)[k].flags;
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    e->sm_count = prop.multiProcessorCount;
    e->image_bytes = (uint32_t)img.size();
    CUDA_TRY(cudaMalloc(&e->d_image, img.size() + 64));
    CUDA_TRY(cudaMemcpy(e->d_image, img.data(), img.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&e->d_flag, 64));
    CUDA_TRY(cudaMemset(e->d_flag, 0, 64));
    // default tile geometry: as many request bytes per request staged in shared memory as still lets the instance keep
    // its CTAs per SM (5, or 4 for the wide slot-layout instance — the kernel is latency bound: residency matters more than
    // staging every tile; larger tiles are read from HBM directly).  The budget is found by asking the runtime's occupancy
    // calculator, not by a formula.
    uint32_t in_per = serve_fit_in_per(device, e->hdr.hot_bytes, kServeCtas, false);
    uint32_t w_in_per = serve_fit_in_per(device, e->hdr.hot_bytes, kServeCtasWide, true);
    if (in_per < 64u) in_per = 64u;    // a table this large: stage at least short requests, whatever residency is left
    if (w_in_per < in_per) w_in_per = in_per;
    int rc = configure_geometry(e, in_per, w_in_per);
    if (rc != GOFR_OK) return rc;
    e->slots_wide = choose_slot_residency(img, e->hdr);
    for (uint32_t k = 0; k < e->hdr.n_progs; k++)
        e->has_values |= (reinterpret_cast<const ProgRec*>(img.data() + e->hdr.progs_off)[k].flags & PF_VALUES) != 0;
    for (auto& s : e->slots) {
        CUDA_TRY(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
        CUDA_TRY(cudaMallocHost(&s.h_tail, 64));
        CUDA_TRY(cudaEventCreateWithFlags(&s.ev_h2d, cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&s.ev_served, cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&s.ev_egress, cudaEventDisableTiming));
    }
    CUDA_TRY(cudaStreamCreateWithFlags(&e->st_h2d, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&e->st_compute, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&e->st_egress, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&e->ev_batch_done, cudaEventBlockingSync | cudaEventDisableTiming));
    CUDA_TRY(cudaMalloc(&e->d_chain, 64));
    CUDA_TRY(cudaMalloc(&e->d_info, sizeof(ChunkInfo) * 2 * kSlots));
    CUDA_TRY(cudaMallocHost(&e->h_status, 64));
    if (const char* w = getenv("GOFR_DEBUG_EPOCH_START")) e->epoch = (uint32_t)strtoul(w, nullptr, 0) & kEpochMask;  // tests: start next to the wrap
    if (getenv("GOFR_DEBUG_NO_LOOKBACK")) e->debug_flags |= 1u;  // diagnostic only: offsets are wrong unless every response has the same size
    e->egress_grid = e->sm_count / 4 > 0 ? e->sm_count / 4 : 1;
    if (const char* g = getenv("GOFR_EGRESS_GRID")) { int v = atoi(g); if (v > 0) e->egress_grid = v; }
    return GOFR_OK;
}

void gofr_engine_destroy(gofr_engine* e) {
    if (!e) return;
    register_engine(e->device, -1);
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    for (auto& s : e->slots) {
        if (s.done) cudaEventDestroy(s.done);
        if (s.ev_h2d) cudaEventDestroy(s.ev_h2d);
        if (s.ev_served) cudaEventDestroy(s.ev_served);
        if (s.ev_egress) cudaEventDestroy(s.ev_egress);
        cudaFree(s.d_desc); cudaFree(s.d_ids); cudaFree(s.d_arena); cudaFree(s.d_out); cudaFree(s.d_off); cudaFree(s.d_meta);
        cudaFree(s.state.words); cudaFree(s.d_flag); cudaFree(s.d_bind);
        cudaFree(s.d_in_off); cudaFree(s.d_meta1);
        for (int k = 0; k < 2; k++) { cudaFree(s.d_codec[k]); cudaFree(s.d_codec_off[k]); }
        cudaFree(s.d_buf); cudaFree(s.d_buf_off); cudaFree(s.d_first); cudaFree(s.d_cstatus); cudaFree(s.d_consumed); cudaFree(s.d_tkey);
        cudaFree(s.d_req_first); cudaFree(s.d_rec); cudaFree(s.d_pdesc); cudaFree(s.d_pstatus); cudaFree(s.d_spans); cudaFree(s.d_req_at);
        cudaFree(s.d_remote); cudaFree(s.d_remote_off); cudaFree(s.d_start); cudaFree(s.d_lfirst); cudaFree(s.d_ldesc); cudaFree(s.d_lids);
        cudaFree(s.d_lreq); cudaFree(s.d_lraw_off); cudaFree(s.d_loff); cudaFree(s.d_larena); cudaFree(s.d_lraw); cudaFree(s.d_lout);
        cudaFree(s.d_rbytes); cudaFree(s.d_roff); cudaFree(s.d_soff); cudaFree(s.d_sarena); cudaFree(s.d_vars);
        if (s.h_tail) cudaFreeHost(s.h_tail);
    }
    for (auto& ev : e->timing) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
    if (e->st_h2d) cudaStreamDestroy(e->st_h2d);
    if (e->st_compute) cudaStreamDestroy(e->st_compute);
    if (e->st_egress) cudaStreamDestroy(e->st_egress);
    if (e->ev_batch_done) cudaEventDestroy(e->ev_batch_done);
    cudaFree(e->d_chain); cudaFree(e->d_info);
    if (e->h_status) cudaFreeHost(e->h_status);
    if (e->h_ends) cudaFreeHost(e->h_ends);
    cudaFree(e->d_image); cudaFree(e->state.words); cudaFree(e->d_flag); cudaFree(e->d_bind);
    cudaFree(e->d_rt_desc); cudaFree(e->d_rt_arena); cudaFree(e->d_rt_meta); cudaFree(e->d_rt_vars); cudaFree(e->d_rt_rows);
    delete e;
}

int gofr_engine_set_tile(gofr_engine* e, uint32_t in_bytes_per_req) {
    if (!e || !in_bytes_per_req) return GOFR_ERR_INVALID;
    std::lock_guard<std::mutex> g(e->mu);
    return configure_geometry(e, in_bytes_per_req, in_bytes_per_req);
}

int gofr_engine_set_chunk(gofr_engine* e, uint32_t requests_per_chunk) {
    if (!e || requests_per_chunk == 0) return GOFR_ERR_INVALID;
    std::lock_guard<std::mutex> g(e->mu);  // a batch in flight keeps the chunk size it started with
    e->chunk = requests_per_chunk;
    return GOFR_OK;
}

}  // extern "C"

// Called with the engine lock held before a timed launch: keeps the list of pending event pairs bounded when the
// caller never asks for the timings (finished pairs are folded into the totals; unfinished ones wait their turn).
static void fold_timing(gofr_engine* e) {
    if (e->timing.size() < 256) return;
    size_t k = 0;
    for (auto& ev : e->timing) {
        if (cudaEventQuery(ev.second) == cudaSuccess) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) { e->timed_ms += ms; e->timed_launches++; }
            cudaEventDestroy(ev.first);
            cudaEventDestroy(ev.second);
        } else e->timing[k++] = ev;
    }
    e->timing.resize(k);
    cudaGetLastError();  // cudaEventQuery reports cudaErrorNotReady through the sticky-free last-error slot
}


// Look-back generation for the next launch.  State words written by older launches carry an older epoch and read as
// "not ready"; the epoch field is kEpochBits wide, so it wraps.  Every state buffer the engine owns is cleared when it
// does (after the device has drained), otherwise a word left by launch k would read as ready in launch k + 2^kEpochBits
// for a tile index that no launch in between has overwritten.  Called with the engine lock held.
static int next_epoch(gofr_engine* e, uint32_t* out) {
    uint32_t ep = (e->epoch + 1) & gofr::kEpochMask;
    if (ep == 0) {  // wrapped (epoch 0 is what zero-initialised words carry: never handed out)
        if (cudaDeviceSynchronize() != cudaSuccess) { set_last_error("device synchronisation failed at the look-back epoch wrap"); return GOFR_ERR_CUDA; }
        if (e->state.words && cudaMemset(e->state.words, 0, e->state.tiles * 8) != cudaSuccess) return GOFR_ERR_CUDA;
        for (auto& s : e->slots)
            if (s.state.words && cudaMemset(s.state.words, 0, s.state.tiles * 8) != cudaSuccess) return GOFR_ERR_CUDA;
        ep = 1;
    }
    e->epoch = ep;
    *out = ep;
    return GOFR_OK;
}

// Grows look-back scratch to the tile count of a launch; new words are zero ("not ready" in every epoch).  A buffer in use
// by earlier launches is safe to replace: cudaFree synchronises the device.
static int grow_state(TileState& s, size_t tiles) {
    if (tiles <= s.tiles) return GOFR_OK;
    cudaFree(s.words);
    s.words = nullptr;
    s.tiles = 0;
    CUDA_TRY(cudaMalloc(&s.words, tiles * 8));
    CUDA_TRY(cudaMemset(s.words, 0, tiles * 8));
    s.tiles = tiles;
    return GOFR_OK;
}

// Every kernel launch goes through here, with the engine lock held: the dynamic shared memory the kernel may use on this
// device covers `smem`, the launch is timed with CUDA events on its stream when timing is on, and it is counted.
template <class... Args>
static int launch(gofr_engine* e, Kern k, int grid, uint32_t smem, cudaStream_t st, const Args&... args) {
    const KernelRec& K = kKernels[k];
    cudaError_t er = cover_smem(k, e->device, smem);
    if (er != cudaSuccess) { set_last_error("%s kernel cannot use %u bytes of shared memory: %s", K.what, smem, cudaGetErrorString(er)); return GOFR_ERR_CUDA; }
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (e->timing_on) {
        fold_timing(e);
        CUDA_TRY(cudaEventCreate(&ev0));
        CUDA_TRY(cudaEventCreate(&ev1));
        CUDA_TRY(cudaEventRecord(ev0, st));
    }
    void* argv[] = {const_cast<void*>(static_cast<const void*>(&args))...};
    cudaLaunchKernel(K.fn, dim3((unsigned)grid), dim3((unsigned)K.threads), argv, smem, st);
    er = cudaGetLastError();
    if (er != cudaSuccess) { set_last_error("%s kernel launch failed: %s", K.what, cudaGetErrorString(er)); return GOFR_ERR_CUDA; }
    if (e->timing_on) {
        CUDA_TRY(cudaEventRecord(ev1, st));
        e->timing.emplace_back(ev0, ev1);
    }
    e->launches++;
    return GOFR_OK;
}

// Resident grid (CTAs per SM x SMs) of a kernel without dynamic shared memory, asked once per engine; 0 with the error set.
static int resident_grid(gofr_engine* e, Kern k) {
    if (e->resident[k] <= 0) e->resident[k] = std::max(0, blocks_per_sm(k, e->device, 0)) * e->sm_count;
    if (e->resident[k] <= 0) set_last_error("%s kernel cannot be resident", kKernels[k].what);
    return e->resident[k];
}

// One fused serve launch.  The packed layout (slot_bytes == 0) chains its tiles through the look-back scratch `state`; the
// slot layout makes the tiles independent of each other and takes none.
static int launch_serve(gofr_engine* e, const void* d_desc, const void* d_ids, const uint8_t* d_arena, uint32_t n,
                        const char* date29, uint8_t* d_out, uint64_t out_cap, uint32_t* d_off, uint32_t* d_meta,
                        TileState* state, uint32_t* d_flag, uint32_t* d_bind, cudaStream_t stream,
                        const unsigned long long* chain_pos = nullptr, uint32_t slot_bytes = 0) {
    ServeParams p;
    memset(&p, 0, sizeof p);
    p.desc = d_desc; p.ids = d_ids; p.arena = d_arena; p.n = n;
    p.n_tiles = (n + kServeT - 1) / kServeT;
    if (!slot_bytes) {
        int rc = grow_state(*state, p.n_tiles);
        if (rc) return rc;
        p.tile_state = state->words;
    }
    p.image = e->d_image; p.hot_bytes = e->hdr.hot_bytes;
    { int erc = next_epoch(e, &p.epoch); if (erc) return erc; }
    p.out = d_out; p.out_cap = out_cap; p.out_off = d_off; p.meta = d_meta;
    p.overflow = d_flag;
    const bool wide = slot_bytes && e->slots_wide && !e->has_values && e->wide_grid > 0;
    p.in_cap = wide ? e->w_in_cap : e->in_cap;
    p.bind_scratch = d_bind; p.bind_row_words = e->hdr.bind_row_words;
    p.chain_pos = chain_pos;
    p.slot_bytes = slot_bytes;
    p.debug_flags = e->debug_flags;
    memcpy(p.date, date29, 29);
    int grid = (int)std::min<uint32_t>((uint32_t)(wide ? e->wide_grid : e->grid), p.n_tiles);
    if (!slot_bytes) grid = std::max(1, std::min(grid, e->grid / engines_on_device(e->device)));  // look-back: see engines_on_device
    return launch(e, serve_instance(slot_bytes != 0, e->has_values, wide), grid, wide ? e->w_smem_bytes : e->smem_bytes, stream, p);
}

// Bind scratch of the resident serve path (tables with GOFR_H_BIND_ECHO routes)
static int grow_bind_scratch(gofr_engine* e, uint32_t n) {
    if (!e->hdr.bind_row_words) return GOFR_OK;
    const size_t need = (size_t)n * e->hdr.bind_row_words * 4;
    if (need <= e->bind_cap) return GOFR_OK;
    cudaFree(e->d_bind);
    e->d_bind = nullptr;
    e->bind_cap = 0;
    CUDA_TRY(cudaMalloc(&e->d_bind, need + need / 4 + 256));
    e->bind_cap = need + need / 4;
    return GOFR_OK;
}

// The launch of the frame kernels (Hello, proto3 encode / decode, flat and nested, the request log, the chunk pack kernel):
// one thread per record, tiles of kServeThreads chained by the look-back over the scratch `state`, overflow reported in
// `d_flag`, `smem` bytes of dynamic shared memory per CTA and the resident grid asked for that size.  Called with the
// engine lock held.  The caller has validated its own arguments and filled the input fields of `p`; `extra` are the
// kernel's parameters after it (schema or descriptor).
template <class Params, class... Extra>
static int launch_frames_locked(gofr_engine* e, Kern k, uint32_t smem, Params p, uint32_t n, uint8_t* d_out, uint64_t out_cap,
                                uint32_t* d_out_off, TileState& state, uint32_t* d_flag, cudaStream_t st, const Extra&... extra) {
    if (n == 0) { if (d_out_off) CUDA_TRY(cudaMemsetAsync(d_out_off, 0, 4, st)); return GOFR_OK; }
    const uint32_t tiles = (n + kServeThreads - 1) / kServeThreads;
    { int rc = grow_state(state, tiles); if (rc) return rc; }
    int resident = 0;
    if (!smem) resident = resident_grid(e, k);
    else if ((resident = std::max(0, blocks_per_sm(k, e->device, smem)) * e->sm_count) <= 0)
        set_last_error("%s kernel cannot be resident with %u bytes of shared memory", kKernels[k].what, smem);
    if (!resident) return GOFR_ERR_CUDA;
    p.n = n; p.n_tiles = tiles;
    { int rc = next_epoch(e, &p.epoch); if (rc) return rc; }
    p.out = d_out; p.out_cap = out_cap; p.out_off = d_out_off;
    p.tile_state = state.words; p.overflow = d_flag;
    const int grid = (int)std::min<uint32_t>((uint32_t)std::max(1, resident / engines_on_device(e->device)), tiles);
    return launch(e, k, grid, smem, st, p, extra...);
}
// The device calls: the engine's resident scratch, on the caller's stream
template <class Params, class... Extra>
static int launch_frames_smem(gofr_engine* e, Kern k, uint32_t smem, Params p, uint32_t n, uint8_t* d_out, uint64_t out_cap,
                              uint32_t* d_out_off, void* stream, const Extra&... extra) {
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    return launch_frames_locked(e, k, smem, p, n, d_out, out_cap, d_out_off, e->state, e->d_flag, (cudaStream_t)stream, extra...);
}
template <class Params, class... Extra>
static int launch_frames(gofr_engine* e, Kern k, Params p, uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                         void* stream, const Extra&... extra) {
    return launch_frames_smem(e, k, 0, p, n, d_out, out_cap, d_out_off, stream, extra...);
}

// The schema index of a Bind target, or an error: not part of the engine's table, or not a struct Bind takes.
static int bind_schema(const gofr_engine* e, uint32_t schema_id, uint32_t* idx) {
    for (size_t k = 0; k < e->schema_ids.size(); k++) {
        if (e->schema_ids[k] != schema_id) continue;
        if (!(e->schema_flags[k] & SF_BINDABLE)) { set_last_error("schema %u: Bind takes flat structs of int / float64 / bool / string fields only", schema_id); return GOFR_ERR_UNSUPPORTED; }
        *idx = (uint32_t)k;
        return GOFR_OK;
    }
    set_last_error("schema %u is not part of the engine's table", schema_id);
    return GOFR_ERR_INVALID;
}

// The stages of the split API: one thread per request over the table's hot part in shared memory, no dependence between
// requests, so the grid is capped at a few CTAs per SM rather than sized for residency.
static int launch_route_kernel(gofr_engine* e, const void* d_desc, const uint8_t* d_arena, uint32_t n, uint32_t* d_meta,
                               uint32_t* d_vars, cudaStream_t st) {
    RouteParams p;
    memset(&p, 0, sizeof p);
    p.desc = d_desc; p.arena = d_arena; p.n = n; p.image = e->d_image; p.hot_bytes = e->hdr.hot_bytes;
    p.meta = d_meta; p.vars = d_vars;
    const uint32_t grid = std::min<uint32_t>((n + kRouteThreads - 1) / kRouteThreads, (uint32_t)e->sm_count * 4);
    return launch(e, K_ROUTE, (int)grid, (e->hdr.hot_bytes + 127u) & ~127u, st, p);
}

static int launch_bind_kernel(gofr_engine* e, uint32_t schema_idx, const void* d_desc, const uint8_t* d_arena, uint32_t n,
                              uint8_t* d_rows, uint32_t slot_bytes, uint32_t* d_len, uint32_t* d_status, cudaStream_t st) {
    BindParams p;
    memset(&p, 0, sizeof p);
    p.desc = d_desc; p.arena = d_arena; p.n = n; p.image = e->d_image; p.hot_bytes = e->hdr.hot_bytes; p.schema_idx = schema_idx;
    p.out = d_rows; p.slot_bytes = slot_bytes; p.len = d_len; p.status = d_status;
    const uint32_t grid = std::min<uint32_t>((n + kBindThreads - 1) / kBindThreads, (uint32_t)e->sm_count * 8);
    return launch(e, K_BIND, (int)grid, (e->hdr.hot_bytes + 127u) & ~127u, st, p);
}

extern "C" {

int gofr_serve_device(gofr_engine* e, const gofr_req_desc* d_desc, const uint8_t* d_trace_ids, const uint8_t* d_arena,
                      uint32_t n, const char* date29, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                      uint32_t* d_meta, void* stream) {
    if (!e || !date29 || (n && (!d_desc || !d_trace_ids || !d_out || !d_out_off || !d_meta))) return GOFR_ERR_INVALID;
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        if (d_out_off) CUDA_TRY(cudaMemsetAsync(d_out_off, 0, 4, st));
        return GOFR_OK;
    }
    { int rc = grow_bind_scratch(e, n); if (rc) return rc; }
    return launch_serve(e, d_desc, d_trace_ids, d_arena, n, date29, d_out, out_cap, d_out_off, d_meta, &e->state, e->d_flag,
                        e->d_bind, st);
}

int gofr_serve_device_slots(gofr_engine* e, const gofr_req_desc* d_desc, const uint8_t* d_trace_ids, const uint8_t* d_arena,
                            uint32_t n, const char* date29, uint8_t* d_out, uint32_t slot_bytes, uint32_t* d_out_len,
                            uint32_t* d_meta, void* stream) {
    if (!e || !date29 || (n && (!d_desc || !d_trace_ids || !d_out || !d_out_len || !d_meta))) return GOFR_ERR_INVALID;
    if (slot_bytes == 0 || (slot_bytes & 15u) || ((uintptr_t)d_out & 15u)) {
        set_last_error("slot_bytes must be a positive multiple of 16 and d_out 16-byte aligned");
        return GOFR_ERR_INVALID;
    }
    if (n == 0) return GOFR_OK;
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    { int rc = grow_bind_scratch(e, n); if (rc) return rc; }
    return launch_serve(e, d_desc, d_trace_ids, d_arena, n, date29, d_out, (uint64_t)n * slot_bytes, d_out_len, d_meta, nullptr,
                        e->d_flag, e->d_bind, (cudaStream_t)stream, nullptr, slot_bytes);
}

int gofr_engine_overflowed(gofr_engine* e, int* flag_out, int reset) {
    if (!e || !flag_out) return GOFR_ERR_INVALID;
    uint32_t f = 0;
    CUDA_TRY(cudaSetDevice(e->device));
    CUDA_TRY(cudaMemcpy(&f, e->d_flag, 4, cudaMemcpyDeviceToHost));
    if (reset && f) CUDA_TRY(cudaMemset(e->d_flag, 0, 4));
    *flag_out = (int)f;
    return GOFR_OK;
}

uint64_t gofr_engine_launch_count(const gofr_engine* e) { return e ? e->launches : 0; }

int gofr_engine_kernel_time_ms(gofr_engine* e, double* total_ms, uint64_t* launches, int reset) {
    if (!e) return GOFR_ERR_INVALID;
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    for (auto& ev : e->timing) {
        CUDA_TRY(cudaEventSynchronize(ev.second));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, ev.first, ev.second));
        e->timed_ms += ms;
        e->timed_launches++;
        cudaEventDestroy(ev.first);
        cudaEventDestroy(ev.second);
    }
    e->timing.clear();
    if (total_ms) *total_ms = e->timed_ms;
    if (launches) *launches = e->timed_launches;
    if (reset) { e->timed_ms = 0; e->timed_launches = 0; }
    return GOFR_OK;
}

int gofr_engine_set_timing(gofr_engine* e, int on) {
    if (!e) return GOFR_ERR_INVALID;
    std::lock_guard<std::mutex> g(e->mu);
    e->timing_on = on != 0;
    return GOFR_OK;
}

int gofr_engine_geometry(const gofr_engine* e, uint32_t* grid, uint32_t* blocks_per_sm, uint32_t* smem_bytes,
                         uint32_t* sm_count) {
    if (!e) return GOFR_ERR_INVALID;
    if (grid) *grid = (uint32_t)e->grid;
    if (blocks_per_sm) *blocks_per_sm = (uint32_t)e->blocks_per_sm;
    if (smem_bytes) *smem_bytes = e->smem_bytes;
    if (sm_count) *sm_count = (uint32_t)e->sm_count;
    return GOFR_OK;
}

int gofr_engine_slot_ctas(gofr_engine* e, int ctas_per_sm, int* in_effect) {
    if (!e) return GOFR_ERR_INVALID;
    std::lock_guard<std::mutex> g(e->mu);
    if (ctas_per_sm == kServeCtasWide) e->slots_wide = true;
    else if (ctas_per_sm == kServeCtas) e->slots_wide = false;
    else if (ctas_per_sm != 0) return GOFR_ERR_INVALID;
    if (in_effect) *in_effect = e->slots_wide && !e->has_values && e->wide_grid > 0 ? kServeCtasWide : kServeCtas;
    return GOFR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// host-batch path
// ---------------------------------------------------------------------------------------------------------------

static int grow(void** p, size_t* cap, size_t need, size_t slack) {
    if (need <= *cap) return GOFR_OK;
    cudaFree(*p);
    *p = nullptr;
    size_t c = need + need / 4 + slack;
    cudaError_t er = cudaMalloc(p, c);
    if (er != cudaSuccess) { set_last_error("cudaMalloc(%zu) failed: %s", c, cudaGetErrorString(er)); *cap = 0; return GOFR_ERR_NOMEM; }
    *cap = c;
    return GOFR_OK;
}

// One per-element device column of a group: per bytes per element plus extra bytes (none allocated when both are 0).
struct Col { void* p; size_t per, extra; };

// Grows a group of per-element columns (capacity *cap elements, `what` names the elements in the error) to hold n: all of
// them are freed and reallocated at n + n/4 + 256 elements.  Columns of n + 1 entries ask for one element extra; the
// kernels rely on every extra byte.
static int grow_cols(size_t* cap, size_t n, const char* what, std::initializer_list<Col> cols) {
    if (n <= *cap) return GOFR_OK;
    for (const Col& k : cols) { cudaFree(*(void**)k.p); *(void**)k.p = nullptr; }
    *cap = 0;
    const size_t c = n + n / 4 + 256;
    for (const Col& k : cols)
        if ((k.per || k.extra) && cudaMalloc((void**)k.p, c * k.per + k.extra) != cudaSuccess) {
            set_last_error("cudaMalloc failed for a chunk of %zu %s", c, what);
            return GOFR_ERR_NOMEM;
        }
    *cap = c;
    return GOFR_OK;
}

// The copy loops read their source in whole aligned words: up to 16 bytes past the last byte a request names may be touched
// (include/gofr_b200.h states the same for device-resident callers), so a staging arena is never sized to the byte.
static constexpr size_t kArenaSlack = 16;

// A chunk = contiguous record range [lo, hi), the input (arena) byte range it covers and a bound on its device output;
// with a log, the log-arena byte range its records' strings cover and a bound on its lines.
struct ChunkPlan { uint32_t lo, hi; uint32_t arena_lo, arena_hi; uint64_t out_bound; uint32_t log_lo, log_hi; uint64_t log_bound; };

// The arena byte range [*alo, *ahi) (16-byte granular) that requests [lo, hi) reference: their whole requests, or their paths
// only (what routing reads).  All arithmetic in 64 bits: a descriptor with a huge arena_off or data_len (say a data_len taken
// from a Content-Length header) must be refused, not wrap around and pass.  sizes (optional) receives the requests' total
// path + query bytes and total data bytes: what their responses are bounded by (chunk_out_bound).
static int chunk_arena_range(const gofr_req_batch* in, uint32_t lo, uint32_t hi, bool path_only, uint32_t* alo_out, uint32_t* ahi_out,
                             uint64_t* sizes = nullptr) {
    uint64_t alo = ~0ull, ahi = 0, pq = 0, data = 0;
    const gofr_req_desc* dd = in->desc;
    for (uint32_t i = lo; i < hi; i++) {
        const uint64_t a = dd[i].arena_off;
        const uint64_t dend = path_only ? a + dd[i].path_len : ((a + dd[i].path_len + dd[i].query_len + 3u) & ~3ull) + dd[i].data_len;
        alo = a < alo ? a : alo;
        ahi = dend > ahi ? dend : ahi;
        pq += (uint64_t)dd[i].path_len + dd[i].query_len;
        data += dd[i].data_len;
    }
    if (sizes) { sizes[0] = pq; sizes[1] = data; }
    if (hi <= lo) alo = 0;
    alo &= ~15ull;
    ahi = (ahi + 15ull) & ~15ull;
    if (ahi > (((uint64_t)in->arena_bytes + 15ull) & ~15ull) || ahi > 0xFFFFFFF0ull) {
        set_last_error("a descriptor of requests %u..%u points outside the arena", lo, hi);
        return GOFR_ERR_INVALID;
    }
    if (ahi > alo && !in->arena) { set_last_error("requests reference arena bytes but the batch has no arena"); return GOFR_ERR_INVALID; }
    *alo_out = (uint32_t)alo;
    *ahi_out = (uint32_t)(ahi > alo ? ahi : alo);
    return GOFR_OK;
}

// Device output bytes a packed chunk can need: the sum of gofr_table_response_bound over its requests (fixed part,
// Content-Length digits, six bytes per path and query byte, image_data_expand per data byte).  The arena span is no measure
// of it: requests may share arena bytes (many descriptors pointing at one cached row), and each of them answers in full.
static uint64_t chunk_out_bound(const gofr_engine* e, uint32_t cn, const uint64_t sizes[2]) {
    // (the sums are clamped to 2^32 first: the products cannot wrap, and the result is capped below that anyway)
    const uint64_t pq = std::min<uint64_t>(sizes[0], 1ull << 32), data = std::min<uint64_t>(sizes[1], 1ull << 32);
    const uint64_t b = (uint64_t)cn * (e->hdr.max_fixed_len + 16 + 2) + 6 * pq + (uint64_t)image_data_expand(e->hdr) * data;
    return std::min<uint64_t>(b, 0xFFFFFFF0ull);
}

// Enqueues the H2D copies of a chunk on `st`: descriptors and trace ids of requests [lo, lo + n) (no ids: d_ids null) and
// the arena bytes [alo, ahi) they reference, as far as the caller's arena has them.
static int upload_chunk(const gofr_req_batch* in, uint32_t lo, uint32_t n, uint32_t alo, uint32_t ahi, void* d_desc, void* d_ids,
                        uint8_t* d_arena, cudaStream_t st) {
    CUDA_TRY(cudaMemcpyAsync(d_desc, in->desc + lo, (size_t)n * 16, cudaMemcpyHostToDevice, st));
    if (d_ids) CUDA_TRY(cudaMemcpyAsync(d_ids, in->trace_ids + (size_t)lo * 16, (size_t)n * 16, cudaMemcpyHostToDevice, st));
    if (ahi > alo) {
        const size_t avail = in->arena_bytes > alo ? (size_t)in->arena_bytes - alo : 0;
        CUDA_TRY(cudaMemcpyAsync(d_arena, in->arena + alo, std::min<size_t>(ahi - alo, avail), cudaMemcpyHostToDevice, st));
    }
    return GOFR_OK;
}

// The slot's previous chunk must have left (egress) before its buffers are overwritten: a wait on the H2D stream, unless
// the buffers have to grow (cudaFree needs the host to be sure).
static int wait_egress(gofr_engine* e, Slot& s, bool grows) {
    if (!s.egress_pending) return GOFR_OK;
    if (grows) CUDA_TRY(cudaEventSynchronize(s.ev_egress));
    else CUDA_TRY(cudaStreamWaitEvent(e->st_h2d, s.ev_egress, 0));
    s.egress_pending = false;
    return GOFR_OK;
}

// Makes the slot's buffers ready for a chunk of `requests` requests, `arena_bytes` arena bytes and `out_bytes` of output.
int Slot::reserve(gofr_engine* e, uint32_t requests, size_t arena_bytes, size_t out_bytes) {
    { int rc = wait_egress(e, *this, requests > cap_n || arena_bytes + kArenaSlack > cap_arena || out_bytes > cap_out); if (rc) return rc; }
    const size_t bind = (size_t)e->hdr.bind_row_words * 4;
    { int rc = grow_cols(&cap_n, requests, "requests", {{&d_desc, 16, 0}, {&d_ids, 16, 0}, {&d_off, 4, 4}, {&d_meta, 4, 0},
                                                         {&d_bind, bind, bind ? 256u : 0u}}); if (rc) return rc; }
    if (!d_flag && (cudaMalloc(&d_flag, 64) != cudaSuccess || cudaMemset(d_flag, 0, 64) != cudaSuccess)) {
        set_last_error("cudaMalloc failed for a chunk's overflow flag");
        return GOFR_ERR_NOMEM;
    }
    int rc = grow((void**)&d_arena, &cap_arena, arena_bytes + kArenaSlack, 256);
    return rc ? rc : grow((void**)&d_out, &cap_out, out_bytes, 256);
}

// The proto host path's buffers for a chunk of `records` records whose codec outputs take a_bytes and b_bytes.  Only the
// chunk's own kernels use them, and a buffer that grows is freed by cudaFree, which waits for the device.  The copy of the
// pack kernel reads a source word past its last byte: grow's slack covers it.
int Slot::reserve_codec(uint32_t records, size_t a_bytes, size_t b_bytes) {
    int rc = grow_cols(&cap_codec_n, records, "records", {{&d_in_off, 4, 4}, {&d_meta1, 4, 0}, {&d_codec_off[0], 4, 4},
                                                          {&d_codec_off[1], 4, 4}});
    if (!rc) rc = grow((void**)&d_codec[0], &cap_codec[0], a_bytes, 256);
    return rc ? rc : grow((void**)&d_codec[1], &cap_codec[1], b_bytes, 256);
}

// Waits for everything enqueued on the egress stream.  A large batch takes milliseconds: the thread sleeps on a
// blocking-sync event.  A small one (the per-request front-end's batches) is back in tens of microseconds: spinning is
// the faster wake-up there.
static cudaError_t wait_batch(gofr_engine* e, uint32_t n) {
    if (n < 16384u) return cudaStreamSynchronize(e->st_egress);
    cudaError_t er = cudaEventRecord(e->ev_batch_done, e->st_egress);
    return er != cudaSuccess ? er : cudaEventSynchronize(e->ev_batch_done);
}

// Error exit of a host-batch call after work has been enqueued: earlier chunks' kernels and copies may still be
// writing into the caller's buffers, which the caller is free to release once we return.
static void drain_streams(gofr_engine* e) {
    cudaStreamSynchronize(e->st_h2d);
    cudaStreamSynchronize(e->st_compute);
    cudaStreamSynchronize(e->st_egress);
    for (auto& s : e->slots) s.egress_pending = false;
    cudaGetLastError();
}

// Runs a host-batch call under the engine lock.  Its input is validated chunk by chunk as the batch is enqueued (an
// up-front scan of 1 Mi records is milliseconds of pure latency), so an error can surface with earlier chunks in flight:
// nothing may still be writing into the caller's buffers when the error is returned.
static int host_batch(gofr_engine* e, const std::function<int()>& run) {
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    const int rc = run();
    if (rc != GOFR_OK) drain_streams(e);
    return rc;
}

// A finished submit: its result waits for gofr_batch_wait under a new ticket.
static void complete(gofr_engine* e, gofr_ticket* ticket, int rc) {
    *ticket = e->next_ticket++;
    e->done_tickets.emplace_back(*ticket, rc);
}

// Host memory the device can write (pinned or managed): the egress kernel stores into it directly
static bool device_visible(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

// The records of a batch counted against the caller's record capacity: a chunk's per-record columns are written only
// while every record so far fits.  From the first chunk that does not, none are (short: the batch fails), and the count
// goes on, so that the batch reports what it needed.
struct RecCount {
    uint64_t cap = 0, base = 0;  // the capacity; the records of the chunks before
    bool short_ = false;
    // Counts a chunk of n records, which start at the old base; whether its columns are written.
    bool add(uint32_t n) { short_ |= base + n > cap; base += n; return !short_; }
};

// A device→host copy to one of the caller's columns that goes with a chunk besides its offsets and per-record column:
// per record (made only when the chunk's records are written) or always (a per-connection column).  No dst: none.
struct ColCopy { void* dst; const void* src; size_t bytes; bool per_record; };

static int copy_cols(std::initializer_list<ColCopy> copies, bool records, cudaStream_t st) {
    for (const ColCopy& c : copies)
        if (c.dst && (records || !c.per_record)) CUDA_TRY(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost, st));
    return GOFR_OK;
}

// The slot's chunk has been handed to the egress stream: its buffers wait for this before they are written again
// (wait_egress).
static int fence_egress(gofr_engine* e, Slot& s) {
    CUDA_TRY(cudaEventRecord(s.ev_egress, e->st_egress));
    s.egress_pending = true;
    return GOFR_OK;
}

// A packed output of a host-batch call: the caller's bytes, their offsets and the one per-record column egress carries
// (meta, or log_req), and its record count.  Output k (0: responses or proto rows, 1: request-log lines) owns d_chain[k],
// h_status[2k..], d_info[k * kSlots ..], each slot's overflow word d_flag[k] and its read-back h_tail[2k + 1], and
// h_ends[4 j + 2k ..] for its j-th posted chunk.  A chunk is posted after the kernels that leave it on the device.
// Pinned buffers are filled by advance and egress without the host waiting (deliver); a pageable chunk is retired later:
// its exact bytes once the host has read its size.  Both skip a chunk's bytes when the device overflowed or when they
// would pass cap or 4 GiB (32-bit offsets): the batch then fails.
//
// `needed` decides what the batch reports at its end (report): what it needed, from each chunk's first and end offsets
// read back to h_ends (the log and connection calls), or what was written (gofr_batch_submit and the proto calls, whose
// columns are then complete whatever the capacity).
struct PackedOut {
    uint8_t* out = nullptr;
    uint64_t cap = 0;
    uint32_t* off = nullptr;
    uint32_t* col = nullptr;
    int k = 0;
    bool pinned = false, needed = false;
    RecCount recs;
    uint64_t written = 0, at = 0;  // bytes written (pinned: after finish); pageable: where the last retired chunk went
    bool overflow = false;         // some chunk's bytes were skipped (pinned: after finish)
    size_t shipped = 0;            // chunks posted with their ends read back (needed)

    PackedOut() = default;
    PackedOut(uint8_t* o, uint64_t c, uint32_t* f, uint32_t* m, uint64_t rec_cap, int k_, bool needed_)
        : out(o), cap(c), off(f), col(m), k(k_), pinned(device_visible(o) && device_visible(f) && device_visible(m)),
          needed(needed_), recs{rec_cap} {}
    unsigned long long* chain(gofr_engine* e) const { return pinned ? e->d_chain + k : nullptr; }
    uint32_t* h_flag(Slot& s) const { return s.h_tail + 2 * k + 1; }
    int start(gofr_engine* e) {
        if (!pinned) return GOFR_OK;
        CUDA_TRY(cudaMemsetAsync(e->d_chain + k, 0, 8, e->st_compute));
        e->h_status[2 * k] = e->h_status[2 * k + 1] = 0;
        return GOFR_OK;
    }
    // Chunk ci's n records, left in slot s's d_out / d_off (at *chain(e) & 15 when pinned, at 0 otherwise) and d_col by the
    // kernels on st_compute: the record-capacity test, and with `needed` the chunk's first and end offsets back to h_ends.
    // Pinned: deliver, then `copies` on st_egress behind the egress, then s.ev_egress.  Pageable: the chunk's size and
    // overflow word back to the host, then s.ev_served; retire(ci) takes it from there.
    int post(gofr_engine* e, Slot& s, size_t ci, const uint8_t* d_out, const uint32_t* d_off, const uint32_t* d_col, uint32_t n,
             std::initializer_list<ColCopy> copies = {}) {
        Posted& p = posted[ci % kSlots];
        p = {d_out, d_off, d_col, n, recs.base, s.h_tail + 2 * k, false, !pinned};
        p.put = recs.add(n) && n;
        const cudaStream_t st = e->st_compute;
        if (needed) {
            uint32_t* ends = e->h_ends + 4 * shipped++ + 2 * k;
            ends[0] = ends[1] = 0;
            if (n) {
                CUDA_TRY(cudaMemcpyAsync(&ends[0], d_off, 4, cudaMemcpyDeviceToHost, st));
                CUDA_TRY(cudaMemcpyAsync(&ends[1], d_off + n, 4, cudaMemcpyDeviceToHost, st));
            }
            p.size = &ends[1];
        }
        if (pinned) {
            int rc = deliver(e, s, ci, d_out, d_off, d_col, n, p.first, p.put);
            if (!rc) rc = copy_cols(copies, p.put, e->st_egress);
            return rc ? rc : fence_egress(e, s);
        }
        if (!needed) CUDA_TRY(cudaMemcpyAsync(p.size, d_off + n, 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(h_flag(s), s.d_flag + k, 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaEventRecord(s.ev_served, st));
        return GOFR_OK;
    }
    // The pageable chunk posted in slot ci % kSlots, if one is still there: the host waits for its read-backs and clears
    // the overflow word when set.  Unless the capacity test failed or the rule skips it, exactly its bytes go to
    // out + written.  Its offsets and column go with its bytes (needed) or always (written), then the `copies`.  Everything
    // goes on st_egress behind s.ev_egress; once it has landed the offsets are rebased.
    int retire(gofr_engine* e, size_t ci, std::initializer_list<ColCopy> copies = {}) {
        Posted& p = posted[ci % kSlots];
        if (!p.live) return GOFR_OK;
        p.live = false;
        Slot& s = e->slots[ci % kSlots];
        const cudaStream_t st = e->st_egress;
        CUDA_TRY(cudaEventSynchronize(s.ev_served));
        const uint32_t flag = *h_flag(s), total = *p.size;
        if (flag) CUDA_TRY(cudaMemsetAsync(s.d_flag + k, 0, 4, st));
        const bool wrote = p.put && !flag && written + total <= cap && written + total <= 0xFFFFFFFFull;
        overflow |= flag || (p.put && !wrote);
        if (wrote && total) CUDA_TRY(cudaMemcpyAsync(out + written, p.d_out, total, cudaMemcpyDeviceToHost, st));
        if (wrote || (p.put && !needed)) {
            CUDA_TRY(cudaMemcpyAsync(off + p.first, p.d_off, (size_t)p.n * 4, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(col + p.first, p.d_col, (size_t)p.n * 4, cudaMemcpyDeviceToHost, st));
        }
        int rc = copy_cols(copies, wrote, st);
        if (!rc) rc = fence_egress(e, s);
        if (rc) return rc;
        CUDA_TRY(cudaEventSynchronize(s.ev_egress));
        if (wrote) {
            at = written;
            written += total;
            if (at) for (uint64_t i = p.first; i < p.first + p.n; i++) off[i] += (uint32_t)at;
        }
        return GOFR_OK;
    }
    // post, then for a pageable chunk retire at once: the connection calls, whose loop waits on each chunk anyway.
    int ship(gofr_engine* e, Slot& s, size_t ci, const uint8_t* d_out, const uint32_t* d_off, const uint32_t* d_col, uint32_t n,
             std::initializer_list<ColCopy> copies) {
        int rc = post(e, s, ci, d_out, d_off, d_col, n, copies);
        return rc || pinned ? rc : retire(e, ci, copies);
    }
    // The end of a batch, after finish: *bytes receives the bytes its chunks needed (needed) or the bytes written.  The
    // closing offset off[recs.base] is stored when every chunk was written, and always when the output reports what was
    // written; otherwise the error is fmt with the records, the bytes, the record capacity and cap (all unsigned long
    // long), and the result GOFR_ERR_CAPACITY.
    int report(gofr_engine* e, uint64_t* bytes, const char* fmt) const {
        uint64_t b = written;
        if (needed) {
            b = 0;
            for (size_t j = 0; j < shipped; j++) b += e->h_ends[4 * j + 2 * k + 1] - e->h_ends[4 * j + 2 * k];
        }
        *bytes = b;
        const bool short_ = recs.short_ || overflow;
        if (!short_ || !needed) off[recs.base] = (uint32_t)written;
        if (!short_) return GOFR_OK;
        set_last_error(fmt, (unsigned long long)recs.base, (unsigned long long)b, (unsigned long long)recs.cap, (unsigned long long)cap);
        return GOFR_ERR_CAPACITY;
    }
    // Reads the pinned outputs' chain words back behind their egress and waits for it once (also when `wait`: other
    // columns left on the egress stream).
    static int finish(gofr_engine* e, uint32_t n, std::initializer_list<PackedOut*> outs, bool wait = false) {
        for (PackedOut* o : outs) {
            if (o->pinned) CUDA_TRY(cudaMemcpyAsync(&e->h_status[2 * o->k], e->d_chain + o->k, 8, cudaMemcpyDeviceToHost, e->st_egress));
            wait |= o->pinned;
        }
        if (!wait) return GOFR_OK;
        CUDA_TRY(wait_batch(e, n));
        for (auto& s : e->slots) s.egress_pending = false;
        for (PackedOut* o : outs)
            if (o->pinned) { o->written = e->h_status[2 * o->k]; o->overflow = e->h_status[2 * o->k + 1] != 0; }
        return GOFR_OK;
    }

private:
    // A posted chunk: its device buffers and records, where its size is read back to, whether its records fit the record
    // capacity (put) and whether it still waits for retire (live: pageable only).
    struct Posted {
        const uint8_t* d_out; const uint32_t* d_off; const uint32_t* d_col; uint32_t n; uint64_t first; uint32_t* size; bool put, live;
    };
    Posted posted[kSlots] = {};

    // Advance on st_compute, then egress of the n records to the caller's from `first` on st_egress.  Without put
    // neither runs and the overflow word is cleared.
    int deliver(gofr_engine* e, Slot& s, size_t ci, const uint8_t* d_out, const uint32_t* d_off, const uint32_t* d_col,
                uint32_t n, uint64_t first, bool put) {
        ChunkInfo* info = e->d_info + k * kSlots + ci % kSlots;
        if (put && launch_advance(e->d_chain + k, d_off, n, s.d_flag + k, info, cap, e->st_compute) != 0) {
            set_last_error("advance kernel launch failed"); return GOFR_ERR_CUDA;
        }
        if (!put) CUDA_TRY(cudaMemsetAsync(s.d_flag + k, 0, 4, e->st_compute));
        CUDA_TRY(cudaEventRecord(s.ev_served, e->st_compute));
        CUDA_TRY(cudaStreamWaitEvent(e->st_egress, s.ev_served, 0));
        if (put && launch_egress(info, d_out, d_off, d_col, n, out, off + first, col + first, e->h_status + 2 * k,
                                 e->egress_grid, e->st_egress) != 0) {
            set_last_error("egress kernel launch failed"); return GOFR_ERR_CUDA;
        }
        if (put) e->launches += 2;
        return GOFR_OK;
    }
};

// PackedOut's first and end offsets for a batch of up to max_chunks chunks
static int reserve_ends(gofr_engine* e, uint64_t max_chunks) {
    if (4 * max_chunks <= e->ends_cap) return GOFR_OK;
    if (e->h_ends) cudaFreeHost(e->h_ends);
    e->h_ends = nullptr;
    e->ends_cap = 0;
    CUDA_TRY(cudaMallocHost(&e->h_ends, 4 * max_chunks * 4));
    e->ends_cap = 4 * max_chunks;
    return GOFR_OK;
}

// What the calls on a request or proto batch do per chunk, where they differ:
//   plan     the chunk that starts at record lo: its end, its input byte range, a bound on its device output and, with a
//            log, its log-arena range and a bound on its lines; the records' input is validated here, chunk by chunk
//            (see host_batch);
//   upload   the H2D copies of the chunk's input into the slot (and any buffers of the caller's own it needs);
//   compute  the kernels that leave the chunk's responses in the slot's d_out / d_off / d_meta, a packed output placed at
//            *chain_pos & 15 when chain_pos is given (the serve kernel's convention), at 0 otherwise;
//   lines    with a log, after the responses have shipped: the kernels that leave the chunk's packed lines in the slot's
//            d_lout / d_loff, placed as compute places its output.
// max_chunks bounds the chunks plan cuts a batch into (0: chunks of e->chunk records); with a log, each chunk reads its
// offsets back to h_ends.
struct ChunkSteps {
    std::function<int(uint32_t lo, ChunkPlan* c)> plan;
    std::function<int(Slot& s, const ChunkPlan& c, cudaStream_t st)> upload;
    std::function<int(Slot& s, const ChunkPlan& c, cudaStream_t st, const unsigned long long* chain_pos)> compute, lines;
    uint64_t max_chunks = 0;
};

// The slot-layout responses of a chunk of n requests from lo: their size is known on the host (requests × slot bytes), so
// they leave with three plain copies on the egress stream behind the serve kernel.
static int ship_slots(gofr_engine* e, Slot& s, const gofr_slot_batch* out, uint32_t lo, uint32_t n) {
    CUDA_TRY(cudaEventRecord(s.ev_served, e->st_compute));
    CUDA_TRY(cudaStreamWaitEvent(e->st_egress, s.ev_served, 0));
    CUDA_TRY(cudaMemcpyAsync(out->out + (size_t)lo * out->slot_bytes, s.d_out, (size_t)n * out->slot_bytes, cudaMemcpyDeviceToHost, e->st_egress));
    CUDA_TRY(cudaMemcpyAsync(out->out_len + lo, s.d_off, (size_t)n * 4, cudaMemcpyDeviceToHost, e->st_egress));
    CUDA_TRY(cudaMemcpyAsync(out->meta + lo, s.d_meta, (size_t)n * 4, cudaMemcpyDeviceToHost, e->st_egress));
    return fence_egress(e, s);
}

// The chunk loop of the calls on a request or proto batch.  A call has one response output, packed (out) or in slots
// (slots), and with a log the request-log lines (output 1, their per-record column meta).  Per chunk: plan, the slot's
// buffers, upload on st_h2d, compute on st_compute, the responses shipped, then with a log the lines' kernels and the
// lines.  A pageable chunk is retired when its slot comes round again, so kSlots of them are in flight, and the rest at
// the end, oldest first.  The lines' kernel counts its lines into d_chain[2], read once at the end.
static int req_chunks(gofr_engine* e, uint32_t n, const ChunkSteps& steps, gofr_resp_batch* out, const gofr_slot_batch* slots,
                      gofr_batch_log* log, gofr_ticket* ticket) {
    if (out) out->out_bytes = 0;
    if (log) { log->lines = 0; log->out_bytes = 0; }
    if (n == 0) {  // nothing to do; the caller may have passed no buffers at all
        if (out && out->out_off) out->out_off[0] = 0;
        if (log && log->log_off) log->log_off[0] = 0;
        complete(e, ticket, GOFR_OK);
        return GOFR_OK;
    }
    // the calls with a log report what the batch needed, as the connection calls do; the others what was written
    PackedOut ro, lo;
    if (out) ro = PackedOut(out->out, out->out_cap, out->out_off, out->meta, n, 0, log != nullptr);
    if (log) {
        lo = PackedOut(log->out, log->out_cap, log->log_off, out ? out->meta : slots->meta, n, 1, true);
        int rc = reserve_ends(e, steps.max_chunks ? steps.max_chunks : (n + (uint64_t)e->chunk - 1) / e->chunk);
        if (rc) return rc;
    }
    { int rc = ro.start(e); if (!rc) rc = lo.start(e); if (rc) return rc; }
    if (log) CUDA_TRY(cudaMemsetAsync(e->d_chain + 2, 0, 8, e->st_compute));
    size_t ci = 0;
    for (uint32_t next = 0; next < n; ci++) {
        Slot& s = e->slots[ci % kSlots];
        ChunkPlan c;
        int rc = ro.retire(e, ci);
        if (!rc) rc = lo.retire(e, ci);
        if (!rc) rc = steps.plan(next, &c);
        if (rc) return rc;
        next = c.hi;
        const uint32_t cn = c.hi - c.lo;
        rc = s.reserve(e, cn, (size_t)c.arena_hi - c.arena_lo, c.out_bound);
        if (!rc && log) rc = s.reserve_lines(cn);
        if (!rc && log) rc = s.reserve_line_bytes((size_t)c.log_hi - c.log_lo, c.log_bound);
        if (!rc) rc = steps.upload(s, c, e->st_h2d);
        if (rc) return rc;
        CUDA_TRY(cudaEventRecord(s.ev_h2d, e->st_h2d));
        CUDA_TRY(cudaStreamWaitEvent(e->st_compute, s.ev_h2d, 0));
        rc = steps.compute(s, c, e->st_compute, ro.chain(e));
        if (!rc) rc = slots ? ship_slots(e, s, slots, c.lo, cn) : ro.post(e, s, ci, s.d_out, s.d_off, s.d_meta, cn);
        if (!rc && log) rc = steps.lines(s, c, e->st_compute, lo.chain(e));
        if (!rc && log) rc = lo.post(e, s, ci, s.d_lout, s.d_loff, s.d_meta, cn);
        if (rc) return rc;
    }
    for (size_t j = ci; j < ci + kSlots; j++) {
        int rc = ro.retire(e, j);
        if (!rc) rc = lo.retire(e, j);
        if (rc) return rc;
    }
    { int rc = PackedOut::finish(e, n, {&ro, &lo}, slots != nullptr); if (rc) return rc; }
    if (log) {
        CUDA_TRY(cudaMemcpyAsync(&e->h_status[4], e->d_chain + 2, 8, cudaMemcpyDeviceToHost, e->st_compute));
        CUDA_TRY(cudaStreamSynchronize(e->st_compute));
        log->lines = (uint32_t)e->h_status[4];
    }
    int rc = GOFR_OK;
    if (out)
        rc = ro.report(e, &out->out_bytes, log ? "the batch needs %llu requests and %llu response bytes: n %llu, out_cap %llu"
                                               : "output capacity too small (device chunk buffer or caller buffer)");
    if (log) {
        const int lrc = lo.report(e, &log->out_bytes, "the batch needs %llu log records and %llu log bytes: n %llu, out_cap %llu");
        if (lrc) rc = lrc;
    }
    complete(e, ticket, rc);
    return GOFR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// connection receive buffers in host memory (gofr_conn_batch_submit)
// ---------------------------------------------------------------------------------------------------------------

// Receive-buffer bytes one chunk stages at most; a connection larger than this gets a chunk of its own.
static constexpr uint32_t kConnChunkBudget = 8u << 20;

// The buffers of a chunk of `conns` connections, `records` records at most and `buf_bytes` staged buffer bytes (plus the
// 16 readable bytes the framer and the request-head kernel need, and 16 more for the bulk copies' rounding).
int Slot::reserve_conn(uint32_t conns, uint32_t records, size_t buf_bytes) {
    int rc = grow_cols(&cap_conns, conns, "connections", {{&d_buf_off, 4, 4}, {&d_first, 4, 4}, {&d_cstatus, 4, 0},
                                                          {&d_consumed, 4, 0}, {&d_req_first, 4, 4}, {&d_tkey, 8, 0}});
    if (!rc) rc = grow_cols(&cap_recs, records, "records", {{&d_rec, 4, 4}, {&d_pdesc, 16, 0}, {&d_pstatus, 4, 0},
                                                            {&d_spans, GOFR_HTTP_SPANS * 8, 0}, {&d_req_at, 4, 0}});
    return rc ? rc : grow((void**)&d_buf, &cap_buf, buf_bytes + 32, 256);
}

// The request-log buffers of a chunk of `conns` connections with `records` records at most and `remote_bytes` of remote
// strings: the inputs and every per-line column (a chunk has no more lines than records).  The byte buffers whose size is
// only known once the chunk is served grow in conn_log_chunk.
int Slot::reserve_log(uint32_t conns, uint32_t records, size_t remote_bytes) {
    int rc = grow_cols(&cap_lconns, conns, "logged connections", {{&d_remote_off, 4, 4}, {&d_start, 8, 0}, {&d_lfirst, 4, 4}});
    if (!rc) rc = reserve_lines(records);
    return rc ? rc : grow((void**)&d_remote, &cap_remote, remote_bytes + 16, 256);
}

// The per-line columns: descriptors, trace ids, request indices and the reqlog and pack offset columns.
int Slot::reserve_lines(uint32_t lines) {
    return grow_cols(&cap_lrecs, lines, "log lines", {{&d_ldesc, sizeof(gofr_log_desc), 0}, {&d_lids, 16, 0}, {&d_lreq, 4, 0},
                                                      {&d_lraw_off, 4, 4}, {&d_loff, 4, 4}});
}

// The log arena (plus the 32 readable bytes the reqlog kernel needs after the last string), and the reqlog kernel's lines
// and the packed lines for `line_bytes` of lines (plus the word the pack kernel's copy reads past a line, and the packed
// start at *chain_pos & 15).
int Slot::reserve_line_bytes(size_t arena_bytes, uint64_t line_bytes) {
    int rc = grow((void**)&d_larena, &cap_larena, arena_bytes + 64, 256);
    if (!rc) rc = grow((void**)&d_lraw, &cap_lraw, line_bytes + 16, 256);
    return rc ? rc : grow((void**)&d_lout, &cap_lout, line_bytes + 16, 256);
}

// A chunk: connections [lo, hi), staged from buffer byte alo (buf_off[lo] rounded down to 16, so that the absolute offsets
// address the staged copy through a rebased pointer), with room for rec_cap records.  With logging: its remote strings
// remote[rlo .. rhi), the longest of them remote_max bytes.
struct ConnChunk { uint32_t lo, hi, alo, rec_cap, rlo, rhi, remote_max; };

// The longest line of a request besides 6 bytes per byte of its strings (reqlog_device.cuh): the literals, two times of 35
// bytes, the id, a response_time of 20 characters and a status of 5 digits take 264 bytes.
static constexpr uint64_t kConnLogFrame = 320;

// The rule of the caller's offset columns: off[i + 1] is not below off[i] and not past limit, for i in [i0, i1).
static int check_offsets(const char* what, const uint32_t* off, uint64_t i0, uint64_t i1, uint64_t limit) {
    for (uint64_t i = i0; i < i1; i++)
        if (off[i + 1] < off[i] || off[i + 1] > limit) {
            set_last_error("%s[%llu] decreases or passes %llu", what, (unsigned long long)(i + 1), (unsigned long long)limit);
            return GOFR_ERR_INVALID;
        }
    return GOFR_OK;
}

// The rule of gofr_conn_log's remote offsets, checked at connection c: its remote string is at most 255 bytes long.
static int check_remote(const uint32_t* remote_off, uint32_t c) {
    return check_offsets("remote_off", remote_off, c, c + 1, (uint64_t)remote_off[c] + 255u);
}

// The chunk that starts at connection lo: at most e->chunk connections whose bytes fit kConnChunkBudget, at least one.  The
// offsets are validated here, chunk by chunk, and with logging the remote offsets too.
static int conn_plan(const gofr_engine* e, const gofr_conn_batch* in, const gofr_conn_log* log, uint32_t lo, ConnChunk* c) {
    const uint32_t* o = in->buf_off;
    const uint32_t* ro = log ? log->remote_off : nullptr;
    uint32_t hi = lo, rmax = 0;
    while (hi < in->n_conns && hi - lo < e->chunk) {
        if (int rc = check_offsets("buf_off", o, hi, hi + 1, in->buf_bytes)) return rc;
        if (hi > lo && o[hi + 1] - o[lo] > kConnChunkBudget) break;
        if (ro) {
            if (int rc = check_remote(ro, hi)) return rc;
            rmax = std::max(rmax, ro[hi + 1] - ro[hi]);
        }
        hi++;
    }
    c->lo = lo; c->hi = hi; c->alo = o[lo] & ~15u;
    c->rec_cap = (o[hi] - o[lo]) / 16 + (hi - lo);  // one record per 16 bytes plus one per connection (the framer's bound)
    c->rlo = ro ? ro[lo] : 0; c->rhi = ro ? ro[hi] : 0; c->remote_max = rmax;
    if (ro && c->rhi > c->rlo && !log->remote) { set_last_error("remote strings without a remote buffer"); return GOFR_ERR_INVALID; }
    // the log arena of the chunk is addressed with 32-bit offsets (conn_log_device.cuh): its bytes plus R per request
    if (ro && (uint64_t)(o[hi] - c->alo) + (uint64_t)c->rec_cap * rmax + 64 > 0xFFFFFFFFull) {
        set_last_error("the log strings of connections %u..%u could pass 4 GiB", lo, hi);
        return GOFR_ERR_UNSUPPORTED;
    }
    return GOFR_OK;
}

// First half of a chunk: stage its bytes, frame them, and bring back its record count (s.h_tail[0]) and its per-connection
// columns (the caller's consumed and conn_status).  s.done marks the moment the host may read them.
static int conn_frame(gofr_engine* e, const gofr_conn_batch* in, const uint64_t* trace_key, uint32_t* consumed, uint32_t* conn_status,
                      const gofr_conn_log* log, Slot& s, const ConnChunk& c) {
    const uint32_t cn = c.hi - c.lo, bytes = in->buf_off[c.hi] - c.alo;
    const uint64_t sizes[2] = {0, bytes};  // the chunk's paths, queries and bodies: never more than its bytes
    int rc = s.reserve(e, c.rec_cap, (size_t)bytes + 16, chunk_out_bound(e, c.rec_cap, sizes));
    if (!rc) rc = s.reserve_conn(cn, c.rec_cap, bytes);
    if (!rc && log) rc = s.reserve_log(cn, c.rec_cap, c.rhi - c.rlo);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(s.d_buf, in->buf + c.alo, bytes, cudaMemcpyHostToDevice, e->st_h2d));
    CUDA_TRY(cudaMemsetAsync(s.d_buf + bytes, 0, 32, e->st_h2d));
    CUDA_TRY(cudaMemcpyAsync(s.d_buf_off, in->buf_off + c.lo, (size_t)(cn + 1) * 4, cudaMemcpyHostToDevice, e->st_h2d));
    if (trace_key) CUDA_TRY(cudaMemcpyAsync(s.d_tkey, trace_key + c.lo, (size_t)cn * 8, cudaMemcpyHostToDevice, e->st_h2d));
    if (log) {
        if (c.rhi > c.rlo) CUDA_TRY(cudaMemcpyAsync(s.d_remote, log->remote + c.rlo, c.rhi - c.rlo, cudaMemcpyHostToDevice, e->st_h2d));
        CUDA_TRY(cudaMemcpyAsync(s.d_remote_off, log->remote_off + c.lo, (size_t)(cn + 1) * 4, cudaMemcpyHostToDevice, e->st_h2d));
        CUDA_TRY(cudaMemcpyAsync(s.d_start, log->start_unix_ns + c.lo, (size_t)cn * 8, cudaMemcpyHostToDevice, e->st_h2d));
    }
    CUDA_TRY(cudaEventRecord(s.ev_h2d, e->st_h2d));
    CUDA_TRY(cudaStreamWaitEvent(e->st_compute, s.ev_h2d, 0));
    HttpFrameParams p;
    memset(&p, 0, sizeof p);
    p.buf = s.d_buf - c.alo; p.buf_off = s.d_buf_off; p.consumed = s.d_consumed; p.status = s.d_cstatus;
    rc = launch_frames_locked(e, K_HTTP_FRAME, 0, p, cn, (uint8_t*)s.d_rec, c.rec_cap, s.d_first, s.state, s.d_flag, e->st_compute);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(&s.h_tail[0], s.d_first + cn, 4, cudaMemcpyDeviceToHost, e->st_compute));
    CUDA_TRY(cudaMemcpyAsync(conn_status + c.lo, s.d_cstatus, (size_t)cn * 4, cudaMemcpyDeviceToHost, e->st_compute));
    CUDA_TRY(cudaMemcpyAsync(consumed + c.lo, s.d_consumed, (size_t)cn * 4, cudaMemcpyDeviceToHost, e->st_compute));
    CUDA_TRY(cudaEventRecord(s.done, e->st_compute));
    return GOFR_OK;
}

// The request-log lines of chunk ci, after its serve kernel: the gather (conn_log_kernel.cu), then the existing reqlog_kernel
// and chunk_pack_kernel, then the lines' PackedOut (output 1).  The reqlog and pack kernels take the chunk's line count
// from the host: it is read back after the gather.  The log kernels report overflow in their own flag word, so that the
// responses' advance never sees it.  The chunk's requests are batch requests [req0, req0 + n_req).
static int conn_log_chunk(gofr_engine* e, const gofr_conn_batch* in, const gofr_conn_log* log, Slot& s, size_t ci,
                          const ConnChunk& c, PackedOut& lo, uint64_t req0, uint32_t n_req) {
    cudaStream_t st = e->st_compute;
    if (!n_req) return GOFR_OK;
    const uint32_t cn = c.hi - c.lo, bytes = in->buf_off[c.hi] - c.alo;
    uint32_t* flag = s.d_flag + 1;
    // the log arena: the chunk's bytes plus R per request (conn_plan has checked that this stays below 4 GiB), and the 32
    // readable bytes the reqlog kernel needs after the last string
    int rc = grow((void**)&s.d_larena, &s.cap_larena, (size_t)bytes + (size_t)n_req * c.remote_max + 64, 256);
    if (rc) return rc;
    ConnLogParams g;
    memset(&g, 0, sizeof g);
    g.first = s.d_first; g.conn_status = s.d_cstatus; g.req_first = s.d_req_first; g.rec_off = s.d_rec; g.spans = s.d_spans;
    g.meta = s.d_meta; g.ids = (const uint8_t*)s.d_ids; g.buf = s.d_buf - c.alo; g.remote = s.d_remote - c.rlo;
    g.remote_off = s.d_remote_off; g.start_ns = s.d_start; g.log_ns = log->log_unix_ns; g.tz_offset_s = log->tz_offset_s;
    g.alo = c.alo; g.remote_max = c.remote_max; g.req0 = (uint32_t)req0;
    g.line_ids = s.d_lids; g.line_req = s.d_lreq; g.arena = s.d_larena;
    rc = launch_frames_locked(e, K_CONN_LOG, 0, g, cn, (uint8_t*)s.d_ldesc, n_req, s.d_lfirst, s.state, flag, st);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(&s.h_tail[2], s.d_lfirst + cn, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(s.done, st));
    CUDA_TRY(cudaEventSynchronize(s.done));
    const uint32_t lines = s.h_tail[2];
    if (!lines) return GOFR_OK;
    // a line is at most kConnLogFrame bytes plus 6 per byte of its strings: its head's (disjoint spans of its record) and
    // its remote string
    const uint64_t bound = std::min<uint64_t>((uint64_t)lines * (kConnLogFrame + 6ull * c.remote_max) + 6ull * bytes, 0xFFFFFFF0ull);
    rc = grow((void**)&s.d_lraw, &s.cap_lraw, bound + 16, 256);  // + the word the pack kernel's copy reads past a line
    if (!rc) rc = grow((void**)&s.d_lout, &s.cap_lout, bound + 16, 256);  // + the packed start at *chain_pos & 15
    if (rc) return rc;
    LogParams lp;
    memset(&lp, 0, sizeof lp);
    lp.desc = s.d_ldesc; lp.ids = s.d_lids; lp.arena = s.d_larena;
    rc = launch_frames_locked(e, K_REQLOG, 0, lp, lines, s.d_lraw, s.cap_lraw - 16, s.d_lraw_off, s.state, flag, st);
    if (rc) return rc;
    PackParams q;
    memset(&q, 0, sizeof q);
    q.a = s.d_lraw; q.a_off = s.d_lraw_off; q.a_cap = s.cap_lraw - 16; q.chain_pos = lo.chain(e);
    rc = launch_frames_locked(e, K_PACK, 0, q, lines, s.d_lout, s.cap_lout, s.d_loff, s.state, flag, st);
    return rc ? rc : lo.ship(e, s, ci, s.d_lout, s.d_loff, s.d_lreq, lines, {});
}

// The chunk's framing is back: parse its records and compact its whole requests into s.d_desc, s.d_req_at, s.d_ids and
// s.d_req_first (batch request indices from req0).  The record count and the connection states (conn_status, on the host
// by now) size the launches; *n_req receives the chunk's request count.  With trace_key the ids come from the keys conn_frame
// staged, else from (trace_seed, c).
static int conn_parse(gofr_engine* e, const gofr_conn_batch* in, const uint64_t* trace_key, const uint32_t* conn_status, Slot& s,
                      const ConnChunk& c, uint32_t req0, uint32_t* n_req_out) {
    CUDA_TRY(cudaEventSynchronize(s.done));
    const uint32_t cn = c.hi - c.lo, n_rec = s.h_tail[0];
    uint32_t n_req = n_rec;
    for (uint32_t k = c.lo; k < c.hi; k++) n_req -= conn_status[k] != GOFR_HTTP_CONN_DONE ? 1u : 0u;
    *n_req_out = n_req;
    cudaStream_t st = e->st_compute;
    if (n_rec) {  // every record's result lands in the bytes it occupies: no look-back, the whole resident grid runs
        const int resident = resident_grid(e, K_HTTP);
        if (!resident) return GOFR_ERR_CUDA;
        HttpParams p;
        memset(&p, 0, sizeof p);
        p.raw = s.d_buf - c.alo; p.raw_off = s.d_rec; p.n = n_rec; p.n_tiles = (n_rec + kServeThreads - 1) / kServeThreads;
        p.desc = s.d_pdesc; p.arena = s.d_arena - c.alo; p.status = s.d_pstatus; p.spans = s.d_spans;
        int rc = launch(e, K_HTTP, (int)std::min<uint32_t>((uint32_t)resident, p.n_tiles), 0, st, p);
        if (rc) return rc;
    }
    ConnParams q;
    memset(&q, 0, sizeof q);
    q.first = s.d_first; q.conn_status = s.d_cstatus; q.rec_off = s.d_rec; q.desc_in = s.d_pdesc;
    q.trace_seed = in->trace_seed; q.trace_key = trace_key ? s.d_tkey : nullptr; q.conn0 = c.lo; q.req0 = req0; q.req_at = s.d_req_at; q.ids = (uint8_t*)s.d_ids;
    return launch_frames_locked(e, K_CONN, 0, q, cn, (uint8_t*)s.d_desc, n_rec, s.d_req_first, s.state, s.d_flag, st);
}

// The closures' results of chunk c (gofr_conn_batch_respond), after its compact step: the chunk's records, those of batch
// requests [req_base, req_base + n_req), go up, and the splice kernel writes every request of the chunk into the slot's
// spliced arena, in request order, rewriting the descriptors in place.  *d_arena receives the arena the serve kernel reads.
static int conn_splice_chunk(gofr_engine* e, const gofr_conn_batch* in, const gofr_conn_results* res, Slot& s, const ConnChunk& c,
                             uint64_t req_base, uint32_t n_req, const uint8_t** d_arena) {
    if (req_base + n_req > res->n_req || (c.hi == in->n_conns && req_base + n_req != res->n_req)) {
        set_last_error("the results are for %u requests, the connections hold %s%llu", res->n_req,
                       c.hi == in->n_conns ? "" : "at least ", (unsigned long long)(req_base + n_req));
        return GOFR_ERR_INVALID;
    }
    if (!n_req) return GOFR_OK;
    if (int rc = check_offsets("rec_off", res->rec_off, req_base, req_base + n_req, res->rec_bytes)) return rc;
    const uint32_t* ro = res->rec_off + req_base;
    // the spliced arena is addressed with 32-bit offsets: each request takes its path, query and data section plus two pads
    // of at most 3 bytes, and its path, query and body are never longer than its message
    const uint32_t rlo = ro[0] & ~15u, rhi = ro[n_req], bytes = in->buf_off[c.hi] - c.alo;
    const uint64_t spliced = (uint64_t)bytes + (rhi - ro[0]) + 8ull * n_req;
    if (spliced + 64 > 0xFFFFFFFFull) {
        set_last_error("the spliced requests of connections %u..%u could pass 4 GiB", c.lo, c.hi);
        return GOFR_ERR_UNSUPPORTED;
    }
    // the serve kernel's output bound: the data sections are the chunk's bytes and records now (a path byte is bounded by
    // a data byte's expansion)
    const uint64_t sizes[2] = {0, spliced};
    int rc = grow_cols(&s.cap_rreqs, n_req, "requests", {{&s.d_roff, 4, 4}, {&s.d_soff, 4, 4}});
    if (!rc) rc = grow((void**)&s.d_rbytes, &s.cap_rbytes, (size_t)(rhi - rlo) + 16, 256);
    if (!rc) rc = grow((void**)&s.d_sarena, &s.cap_sarena, (size_t)spliced + 16, 256);
    if (!rc) rc = grow((void**)&s.d_out, &s.cap_out, chunk_out_bound(e, n_req, sizes), 256);
    if (rc) return rc;
    cudaStream_t st = e->st_compute;
    if (rhi > rlo) CUDA_TRY(cudaMemcpyAsync(s.d_rbytes, res->rec + rlo, rhi - rlo, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(s.d_roff, ro, (size_t)(n_req + 1) * 4, cudaMemcpyHostToDevice, st));
    ConnResultParams p;
    memset(&p, 0, sizeof p);
    p.desc = s.d_desc; p.arena = s.d_arena - c.alo; p.rec = s.d_rbytes - rlo; p.rec_off = s.d_roff;
    rc = launch_frames_locked(e, K_CONN_RESULT, 0, p, n_req, s.d_sarena, s.cap_sarena, s.d_soff, s.state, s.d_flag, st);
    if (rc) return rc;
    *d_arena = s.d_sarena;
    return GOFR_OK;
}

// Second half of chunk ci: parse its records, compact the whole requests, splice the closures' results in (res not null),
// serve them, and send the results to the caller's columns.
static int conn_serve(gofr_engine* e, const gofr_conn_batch* in, const uint64_t* trace_key, const gofr_conn_results* res,
                      gofr_conn_resp* out, const gofr_conn_log* log, Slot& s, size_t ci, const ConnChunk& c, PackedOut& ro, PackedOut& lo) {
    const uint64_t req0 = ro.recs.base;
    uint32_t n_req = 0;
    int rc = conn_parse(e, in, trace_key, out->conn_status, s, c, (uint32_t)req0, &n_req);
    if (rc) return rc;
    const uint8_t* d_arena = s.d_arena - c.alo;
    if (res && (rc = conn_splice_chunk(e, in, res, s, c, req0, n_req, &d_arena)) != 0) return rc;
    if (n_req && (rc = launch_serve(e, s.d_desc, s.d_ids, d_arena, n_req, in->date, s.d_out, s.cap_out, s.d_off, s.d_meta,
                                    &s.state, s.d_flag, s.d_bind, e->st_compute, ro.chain(e))) != 0) return rc;
    rc = ro.ship(e, s, ci, s.d_out, s.d_off, s.d_meta, n_req,
                 {{out->req_at + req0, s.d_req_at, (size_t)n_req * 4, true},
                  {out->trace_ids ? out->trace_ids + req0 * 16 : nullptr, s.d_ids, (size_t)n_req * 16, true},
                  {out->req_first + c.lo, s.d_req_first, (size_t)(c.hi - c.lo) * 4, false}});
    if (!rc && log) rc = conn_log_chunk(e, in, log, s, ci, c, lo, req0, n_req);
    return rc;
}

// The chunks of a connection batch in order, one framed ahead of the one being stepped: the host learns a chunk's record
// count while the next chunk's bytes are on their way.  step(s, ci, c) finishes chunk ci, framed in slot s.
using ConnStep = std::function<int(Slot& s, size_t ci, const ConnChunk& c)>;
static int conn_chunks(gofr_engine* e, const gofr_conn_batch* in, const uint64_t* trace_key, uint32_t* consumed, uint32_t* conn_status,
                       const gofr_conn_log* log, const ConnStep& step) {
    const uint32_t n = in->n_conns;
    ConnChunk chunks[kSlots];
    size_t issued = 0, stepped = 0;
    for (uint32_t next = 0; next < n || stepped < issued;) {
        while (next < n && issued < stepped + 2) {
            ConnChunk& c = chunks[issued % kSlots];
            int rc = conn_plan(e, in, log, next, &c);
            if (!rc) rc = conn_frame(e, in, trace_key, consumed, conn_status, log, e->slots[issued % kSlots], c);
            if (rc) return rc;
            next = c.hi;
            issued++;
        }
        int rc = step(e->slots[stepped % kSlots], stepped, chunks[stepped % kSlots]);
        if (rc) return rc;
        stepped++;
    }
    return GOFR_OK;
}

static int conn_batch_locked(gofr_engine* e, const gofr_conn_batch* in, const uint64_t* trace_key, const gofr_conn_results* res,
                             gofr_conn_resp* out, gofr_conn_log* log, gofr_ticket* ticket) {
    const uint32_t n = in->n_conns;
    out->out_bytes = 0;
    if (log) { log->lines = 0; log->out_bytes = 0; }
    if (n == 0) {  // touches no buffer
        complete(e, ticket, GOFR_OK);
        return GOFR_OK;
    }
    // chunks end at e->chunk connections or at the byte budget, where two neighbours together pass it
    const uint64_t max_chunks = (n + (uint64_t)e->chunk - 1) / e->chunk + 2 * (std::min<uint64_t>(in->buf_bytes, 1ull << 32) / kConnChunkBudget) + 2;
    { int rc = reserve_ends(e, max_chunks); if (rc) return rc; }
    PackedOut ro(out->out, out->out_cap, out->out_off, out->meta, out->req_cap, 0, true), lo;
    { int rc = ro.start(e); if (rc) return rc; }
    if (log) {
        lo = PackedOut(log->out, log->out_cap, log->log_off, log->log_req, log->line_cap, 1, true);
        int rc = lo.start(e);
        if (rc) return rc;
    }
    int rc = conn_chunks(e, in, trace_key, out->consumed, out->conn_status, log, [&](Slot& s, size_t ci, const ConnChunk& c) {
        return conn_serve(e, in, trace_key, res, out, log, s, ci, c, ro, lo);
    });
    if (!rc) rc = PackedOut::finish(e, n, {&ro, &lo});
    if (rc) return rc;
    out->req_first[n] = (uint32_t)ro.recs.base;
    int final_rc = ro.report(e, &out->out_bytes, "the batch needs %llu requests and %llu response bytes: req_cap %llu, out_cap %llu");
    if (log) {
        log->lines = (uint32_t)lo.recs.base;
        rc = lo.report(e, &log->out_bytes, "the batch needs %llu log lines and %llu log bytes: line_cap %llu, out_cap %llu");
        if (rc) final_rc = rc;
    }
    complete(e, ticket, final_rc);
    return GOFR_OK;
}

int gofr_conn_batch_submit(gofr_engine* e, const gofr_conn_batch* in, gofr_conn_resp* out, gofr_ticket* ticket) {
    return gofr_conn_batch_submit_log(e, in, out, nullptr, ticket);
}

int gofr_conn_batch_submit_log(gofr_engine* e, const gofr_conn_batch* in, gofr_conn_resp* out, gofr_conn_log* log, gofr_ticket* ticket) {
    return gofr_conn_batch_respond(e, in, nullptr, out, log, ticket);
}

int gofr_conn_batch_respond(gofr_engine* e, const gofr_conn_batch* in, const gofr_conn_results* res, gofr_conn_resp* out,
                            gofr_conn_log* log, gofr_ticket* ticket) {
    return gofr_conn_batch_respond_ex(e, in, nullptr, res, out, log, ticket);
}

int gofr_conn_batch_respond_ex(gofr_engine* e, const gofr_conn_batch* in, const uint64_t* trace_key, const gofr_conn_results* res,
                               gofr_conn_resp* out, gofr_conn_log* log, gofr_ticket* ticket) {
    if (!e || !in || !out || !ticket) return GOFR_ERR_INVALID;
    if (in->n_conns && (!in->buf || !in->buf_off || !out->out || !out->out_off || !out->meta || !out->req_at || !out->req_first ||
                        !out->consumed || !out->conn_status)) return GOFR_ERR_INVALID;
    if (log && in->n_conns && (!log->remote_off || !log->start_unix_ns || !log->out || !log->log_off || !log->log_req)) return GOFR_ERR_INVALID;
    if (res && in->n_conns && (!res->rec_off || (res->rec_bytes && !res->rec))) return GOFR_ERR_INVALID;
    if (res && !in->n_conns && res->n_req) { set_last_error("the results are for %u requests, the batch has none", res->n_req); return GOFR_ERR_INVALID; }
    return host_batch(e, [&] { return conn_batch_locked(e, in, trace_key, res, out, log, ticket); });
}

// Stage 1 of the closure path (gofr_conn_batch_route), synchronous: the connection chunks of conn_chunks, each framed,
// parsed and compacted as the connection pipeline does, its requests routed, and its columns and parse-arena bytes
// brought back before the next one is stepped.  A request's parsed form lies inside its own message (include/gofr_b200.h),
// so a chunk's arena bytes are exactly its connections' byte range, copied to the same offsets of the caller's arena.
static int conn_route_locked(gofr_engine* e, const gofr_conn_batch* in, gofr_conn_route* out) {
    const cudaStream_t st = e->st_compute;
    RecCount r{out->req_cap};
    int rc = conn_chunks(e, in, nullptr, out->consumed, out->conn_status, nullptr, [&](Slot& s, size_t, const ConnChunk& c) -> int {
        const uint64_t req0 = r.base;
        uint32_t n_req = 0;
        int rc = conn_parse(e, in, nullptr, out->conn_status, s, c, (uint32_t)req0, &n_req);
        if (rc) return rc;
        if (r.add(n_req) && n_req) {
            const size_t vbytes = (size_t)n_req * 4 * GOFR_MAX_PATH_VARS;
            rc = grow((void**)&s.d_vars, &s.cap_vars, vbytes, 256);
            if (!rc) rc = launch_route_kernel(e, s.d_desc, s.d_arena - c.alo, n_req, s.d_meta, s.d_vars, st);
            if (rc) return rc;
            const uint32_t a0 = in->buf_off[c.lo], a1 = in->buf_off[c.hi];
            CUDA_TRY(cudaMemcpyAsync(out->desc + req0, s.d_desc, (size_t)n_req * 16, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(out->meta + req0, s.d_meta, (size_t)n_req * 4, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(out->vars + req0 * GOFR_MAX_PATH_VARS, s.d_vars, vbytes, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(out->req_at + req0, s.d_req_at, (size_t)n_req * 4, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(out->trace_ids + req0 * 16, s.d_ids, (size_t)n_req * 16, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaMemcpyAsync(out->arena + a0, s.d_arena + (a0 - c.alo), a1 - a0, cudaMemcpyDeviceToHost, st));
        }
        CUDA_TRY(cudaMemcpyAsync(out->req_first + c.lo, s.d_req_first, (size_t)(c.hi - c.lo) * 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        return GOFR_OK;
    });
    if (rc) return rc;
    out->req_first[in->n_conns] = (uint32_t)r.base;
    if (r.short_) {
        set_last_error("the batch needs %llu requests: req_cap %u", (unsigned long long)r.base, out->req_cap);
        return GOFR_ERR_CAPACITY;
    }
    return GOFR_OK;
}

int gofr_conn_batch_route(gofr_engine* e, const gofr_conn_batch* in, gofr_conn_route* out) {
    if (!e || !in || !out) return GOFR_ERR_INVALID;
    if (in->n_conns && (!in->buf || !in->buf_off || !out->desc || !out->arena || !out->meta || !out->vars || !out->req_at ||
                        !out->trace_ids || !out->req_first || !out->consumed || !out->conn_status)) return GOFR_ERR_INVALID;
    if (!in->n_conns) return GOFR_OK;
    return host_batch(e, [&] { return conn_route_locked(e, in, out); });
}

int gofr_conn_respond_bound(const gofr_table* t, const gofr_req_desc* desc, uint32_t n_req, const uint32_t* rec_off, uint64_t* out_cap) {
    if (!t || !out_cap || (n_req && (!desc || !rec_off))) return GOFR_ERR_INVALID;
    if (!gofr_table_response_bound(t, 0, 0, 0)) { set_last_error("the table is not sealed"); return GOFR_ERR_NOT_SEALED; }
    if (int rc = check_offsets("rec_off", rec_off, 0, n_req, 0xFFFFFFFFull)) return rc;
    uint64_t b = 0;
    for (uint32_t k = 0; k < n_req; k++) {
        const uint32_t len = rec_off[k + 1] > rec_off[k] ? rec_off[k + 1] - rec_off[k] : desc[k].data_len;
        b += gofr_table_response_bound(t, desc[k].path_len, desc[k].query_len, len);
    }
    *out_cap = b;
    return GOFR_OK;
}

int gofr_conn_batch_bound(const gofr_table* t, const uint32_t* buf_off, uint32_t n_conns, uint32_t* req_cap, uint64_t* out_cap) {
    if (!t || !req_cap || !out_cap || (n_conns && !buf_off)) return GOFR_ERR_INVALID;
    const uint64_t r0 = gofr_table_response_bound(t, 0, 0, 0);
    if (!r0) { set_last_error("the table is not sealed"); return GOFR_ERR_NOT_SEALED; }
    // a response grows by at most this much per path, query or body byte of its request
    const uint64_t per_byte = std::max(gofr_table_response_bound(t, 1, 0, 0), gofr_table_response_bound(t, 0, 0, 1)) - r0;
    if (int rc = check_offsets("buf_off", buf_off, 0, n_conns, 0xFFFFFFFFull)) return rc;
    const uint64_t bytes = n_conns ? buf_off[n_conns] - buf_off[0] : 0, reqs = bytes / 16 + n_conns;
    *req_cap = (uint32_t)std::min<uint64_t>(reqs, 0xFFFFFFFFull);
    *out_cap = reqs * r0 + per_byte * bytes;
    return GOFR_OK;
}

int gofr_conn_log_bound(const uint32_t* buf_off, const uint32_t* remote_off, uint32_t n_conns, uint32_t* line_cap, uint64_t* out_cap) {
    if (!line_cap || !out_cap || (n_conns && (!buf_off || !remote_off))) return GOFR_ERR_INVALID;
    if (int rc = check_offsets("buf_off", buf_off, 0, n_conns, 0xFFFFFFFFull)) return rc;
    uint64_t reqs = 0, remote = 0;
    for (uint32_t c = 0; c < n_conns; c++) {
        if (int rc = check_remote(remote_off, c)) return rc;
        const uint64_t r = (buf_off[c + 1] - buf_off[c]) / 16 + 1;  // the connection's requests at most
        reqs += r;
        remote += r * (remote_off[c + 1] - remote_off[c]);
    }
    const uint64_t bytes = n_conns ? buf_off[n_conns] - buf_off[0] : 0;
    *line_cap = (uint32_t)std::min<uint64_t>(reqs, 0xFFFFFFFFull);
    *out_cap = reqs * kConnLogFrame + 6 * (bytes + remote);
    return GOFR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// the serve calls on host batches: gofr_batch_submit / _slots, and with request-log lines _log
// ---------------------------------------------------------------------------------------------------------------

// The bytes a record's line may take (0 for GOFR_LOG_NONE): kConnLogFrame plus 6 per string byte, the most
// encoding/json's escaping makes of one byte (\u00XX); an RPCLog method byte is escaped twice and may take 7 (\\u00XX,
// rpc_method_slow in reqlog_device.cuh).
static uint64_t log_line_bound(const gofr_log_desc& d) {
    if (d.kind == GOFR_LOG_NONE) return 0;
    const uint64_t len = (uint64_t)d.method_len + d.ua_len + d.xff_len + d.remote_len + d.uri_len;
    return kConnLogFrame + 6 * len + (d.kind == GOFR_LOG_RPC ? d.method_len : 0);
}

// The log records of records [lo, hi): each is checked (its kind: `kind` or GOFR_LOG_NONE, its strings inside the arena),
// and *alo / *ahi receive the arena range of the records that may get a line (16-byte granular below), *bytes the bound of
// their lines.
static int batch_log_plan(const gofr_batch_log* log, uint32_t kind, uint32_t lo, uint32_t hi, uint32_t* alo_out, uint32_t* ahi_out,
                          uint64_t* bytes) {
    uint64_t alo = ~0ull, ahi = 0, b = 0;
    for (uint32_t i = lo; i < hi; i++) {
        const gofr_log_desc& d = log->desc[i];
        if (d.kind != kind && d.kind != GOFR_LOG_NONE) {
            set_last_error("log record %u: kind %u (%s or GOFR_LOG_NONE)", i, d.kind,
                           kind == GOFR_LOG_RPC ? "GOFR_LOG_RPC" : "GOFR_LOG_REQUEST");
            return GOFR_ERR_INVALID;
        }
        const uint64_t len = (uint64_t)d.method_len + d.ua_len + d.xff_len + d.remote_len + d.uri_len, end = d.arena_off + len;
        if (end > log->arena_bytes || (len && !log->arena)) {
            set_last_error("log record %u: its strings pass the log arena", i);
            return GOFR_ERR_INVALID;
        }
        if (d.kind == GOFR_LOG_NONE) continue;
        alo = std::min<uint64_t>(alo, d.arena_off);
        ahi = std::max(ahi, end);
        b += log_line_bound(d);
    }
    if (ahi == 0) alo = 0;
    *alo_out = (uint32_t)(alo & ~15ull);
    *ahi_out = (uint32_t)ahi;
    *bytes = b;
    if (b > 0xFFFFFFF0ull) {
        set_last_error("the log lines of records %u..%u could pass 4 GiB", lo, hi);
        return GOFR_ERR_UNSUPPORTED;
    }
    return GOFR_OK;
}

// The upload of a chunk's log records and the arena range of those that may get a line, on st; with ids, the chunk's
// trace ids too (to d_lids: the proto calls have no request ids of their own).
static int upload_log(Slot& s, const ChunkPlan& c, const gofr_batch_log* log, const uint8_t* ids, cudaStream_t st) {
    const uint32_t cn = c.hi - c.lo;
    CUDA_TRY(cudaMemcpyAsync(s.d_ldesc, log->desc + c.lo, (size_t)cn * sizeof(gofr_log_desc), cudaMemcpyHostToDevice, st));
    if (ids) CUDA_TRY(cudaMemcpyAsync(s.d_lids, ids + (size_t)c.lo * 16, (size_t)cn * 16, cudaMemcpyHostToDevice, st));
    if (c.log_hi > c.log_lo)
        CUDA_TRY(cudaMemcpyAsync(s.d_larena, log->arena + c.log_lo, std::min<uint64_t>(c.log_hi, log->arena_bytes) - c.log_lo,
                                 cudaMemcpyHostToDevice, st));
    return GOFR_OK;
}

// The lines step: request-log kernel k over the chunk's records (ids: their trace ids on the device; `extra` the
// instance's parameters after LogParams) writes every record's line in the lines' overflow word d_flag[1], then
// chunk_pack_kernel places them at *chain_pos & 15.
extern "C++" {
template <class... Extra>
static int chunk_lines(gofr_engine* e, Kern k, Slot& s, const ChunkPlan& c, const void* ids, cudaStream_t st,
                       const unsigned long long* chain_pos, const Extra&... extra) {
    const uint32_t cn = c.hi - c.lo;
    LogParams lp;
    memset(&lp, 0, sizeof lp);
    lp.desc = s.d_ldesc; lp.ids = ids; lp.arena = s.d_larena - c.log_lo;
    int rc = launch_frames_locked(e, k, 0, lp, cn, s.d_lraw, s.cap_lraw - 16, s.d_lraw_off, s.state, s.d_flag + 1, st, extra...);
    if (rc) return rc;
    PackParams q;
    memset(&q, 0, sizeof q);
    q.a = s.d_lraw; q.a_off = s.d_lraw_off; q.a_cap = s.cap_lraw - 16; q.chain_pos = chain_pos;
    return launch_frames_locked(e, K_PACK, 0, q, cn, s.d_lout, s.cap_lout, s.d_loff, s.state, s.d_flag + 1, st);
}
}  // extern "C++"

// The steps of the four serve calls: chunks of e->chunk requests, served into the packed layout (chained) or into slots
// of slot_bytes.  With a log, each chunk's log records and the arena range of those that may get a line go up with its
// requests; the serve-fed request-log kernel (batch_log_kernel.cu) reads each status from the chunk's meta and writes
// every request's line (empty for a request without one) in its own overflow word d_flag[1], and chunk_pack_kernel
// places the lines.  Line offsets are per request, so no count comes back mid-batch.
static ChunkSteps serve_steps(gofr_engine* e, const gofr_req_batch* in, uint32_t slot_bytes, const gofr_batch_log* log) {
    ChunkSteps steps;
    steps.plan = [=](uint32_t lo, ChunkPlan* c) -> int {
        const uint32_t hi = std::min<uint32_t>(in->n, lo + e->chunk);
        uint64_t sizes[2];
        *c = {lo, hi};
        int rc = chunk_arena_range(in, lo, hi, false, &c->arena_lo, &c->arena_hi, sizes);
        if (!rc && log) rc = batch_log_plan(log, GOFR_LOG_REQUEST, lo, hi, &c->log_lo, &c->log_hi, &c->log_bound);
        if (rc) return rc;
        c->out_bound = slot_bytes ? (uint64_t)(hi - lo) * slot_bytes : chunk_out_bound(e, hi - lo, sizes);
        return GOFR_OK;
    };
    steps.upload = [=](Slot& s, const ChunkPlan& c, cudaStream_t st) -> int {
        const uint32_t cn = c.hi - c.lo;
        int rc = upload_chunk(in, c.lo, cn, c.arena_lo, c.arena_hi, s.d_desc, s.d_ids, s.d_arena, st);
        return rc || !log ? rc : upload_log(s, c, log, nullptr, st);
    };
    // descriptors keep absolute arena offsets: pass a rebased arena pointer
    steps.compute = [=](Slot& s, const ChunkPlan& c, cudaStream_t st, const unsigned long long* chain_pos) -> int {
        return launch_serve(e, s.d_desc, s.d_ids, s.d_arena - c.arena_lo, c.hi - c.lo, in->date, s.d_out,
                            slot_bytes ? c.out_bound : s.cap_out, s.d_off, s.d_meta, &s.state, s.d_flag, s.d_bind, st, chain_pos,
                            slot_bytes);
    };
    if (log) steps.lines = [=](Slot& s, const ChunkPlan& c, cudaStream_t st, const unsigned long long* chain_pos) -> int {
        return chunk_lines(e, K_BATCH_LOG, s, c, s.d_ids, st, chain_pos, (const uint32_t*)s.d_meta, log->log_unix_ns, e->d_chain + 2);
    };
    return steps;
}

int gofr_batch_submit(gofr_engine* e, const gofr_req_batch* in, gofr_resp_batch* out, gofr_ticket* ticket) {
    if (!e || !in || !out || !ticket) return GOFR_ERR_INVALID;
    if (in->n && (!in->desc || !in->trace_ids || !out->out || !out->out_off || !out->meta)) return GOFR_ERR_INVALID;
    return host_batch(e, [&] { return req_chunks(e, in->n, serve_steps(e, in, 0, nullptr), out, nullptr, nullptr, ticket); });
}

int gofr_batch_submit_slots(gofr_engine* e, const gofr_req_batch* in, gofr_slot_batch* out, gofr_ticket* ticket) {
    if (!e || !in || !out || !ticket) return GOFR_ERR_INVALID;
    if (in->n && (!in->desc || !in->trace_ids || !out->out || !out->out_len || !out->meta)) return GOFR_ERR_INVALID;
    if (out->slot_bytes == 0 || (out->slot_bytes & 15u)) { set_last_error("slot_bytes must be a positive multiple of 16"); return GOFR_ERR_INVALID; }
    return host_batch(e, [&] { return req_chunks(e, in->n, serve_steps(e, in, out->slot_bytes, nullptr), nullptr, out, nullptr, ticket); });
}

static bool batch_log_valid(const gofr_req_batch* in, const gofr_batch_log* log) {
    return log && (!in->n || (log->desc && log->out && log->log_off));
}

int gofr_batch_submit_log(gofr_engine* e, const gofr_req_batch* in, gofr_resp_batch* out, gofr_batch_log* log, gofr_ticket* ticket) {
    if (!e || !in || !out || !ticket || !batch_log_valid(in, log)) return GOFR_ERR_INVALID;
    if (in->n && (!in->desc || !in->trace_ids || !out->out || !out->out_off || !out->meta)) return GOFR_ERR_INVALID;
    return host_batch(e, [&] { return req_chunks(e, in->n, serve_steps(e, in, 0, log), out, nullptr, log, ticket); });
}

int gofr_batch_submit_slots_log(gofr_engine* e, const gofr_req_batch* in, gofr_slot_batch* out, gofr_batch_log* log, gofr_ticket* ticket) {
    if (!e || !in || !out || !ticket || !batch_log_valid(in, log)) return GOFR_ERR_INVALID;
    if (in->n && (!in->desc || !in->trace_ids || !out->out || !out->out_len || !out->meta)) return GOFR_ERR_INVALID;
    if (out->slot_bytes == 0 || (out->slot_bytes & 15u)) { set_last_error("slot_bytes must be a positive multiple of 16"); return GOFR_ERR_INVALID; }
    return host_batch(e, [&] { return req_chunks(e, in->n, serve_steps(e, in, out->slot_bytes, log), nullptr, out, log, ticket); });
}

int gofr_batch_log_bound(const gofr_log_desc* desc, uint32_t n, uint64_t* out_cap) {
    if (!out_cap || (n && !desc)) return GOFR_ERR_INVALID;
    uint64_t b = 0;
    for (uint32_t i = 0; i < n; i++) b += log_line_bound(desc[i]);
    *out_cap = b;
    return GOFR_OK;
}

int gofr_batch_wait(gofr_engine* e, gofr_ticket ticket) {
    if (!e || ticket == 0) return GOFR_ERR_INVALID;
    std::lock_guard<std::mutex> g(e->mu);
    for (size_t k = 0; k < e->done_tickets.size(); k++) {
        if (e->done_tickets[k].first != ticket) continue;
        int rc = e->done_tickets[k].second;
        e->done_tickets.erase(e->done_tickets.begin() + (long)k);
        return rc;
    }
    return GOFR_ERR_INVALID;  // unknown ticket, or already waited for
}

// Parses a sysfs cpu list ("0-31,64-95") into a cpu_set_t; returns the number of CPUs.
static int parse_cpulist(const char* s, cpu_set_t* set) {
    CPU_ZERO(set);
    int count = 0;
    while (*s) {
        char* end = nullptr;
        long a = strtol(s, &end, 10);
        if (end == s) break;
        long b = a;
        if (*end == '-') { s = end + 1; b = strtol(s, &end, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) { CPU_SET((int)c, set); count++; }
        s = *end == ',' ? end + 1 : end;
        if (*end != ',') break;
    }
    return count;
}

int gofr_bind_host_thread(int device, int* numa_node_out) {
    if (numa_node_out) *numa_node_out = -1;
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, (int)sizeof bus, device) != cudaSuccess) { cudaGetLastError(); set_last_error("no PCI bus id for device %d", device); return GOFR_ERR_CUDA; }
    for (char* c = bus; *c; c++) if (*c >= 'A' && *c <= 'Z') *c = (char)(*c + 32);  // sysfs names are lower case
    auto read_line = [](const std::string& path, char* buf, size_t cap) -> bool {
        FILE* f = fopen(path.c_str(), "r");
        if (!f) return false;
        const bool ok = fgets(buf, (int)cap, f) != nullptr;
        fclose(f);
        return ok;
    };
    const std::string base = std::string("/sys/bus/pci/devices/") + bus + "/";
    char line[4096];
    int node = -1;
    if (read_line(base + "numa_node", line, sizeof line)) node = atoi(line);
    if (numa_node_out) *numa_node_out = node;
    cpu_set_t set;
    int ncpu = 0;
    if (node >= 0 && read_line("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist", line, sizeof line)) ncpu = parse_cpulist(line, &set);
    if (!ncpu && read_line(base + "local_cpulist", line, sizeof line)) ncpu = parse_cpulist(line, &set);
    if (!ncpu) { set_last_error("no NUMA information for device %d (%s)", device, bus); return GOFR_ERR_UNSUPPORTED; }
    // stay inside what the container allows
    cpu_set_t cur;
    if (sched_getaffinity(0, sizeof cur, &cur) == 0) {
        cpu_set_t both;
        CPU_AND(&both, &set, &cur);
        if (CPU_COUNT(&both) > 0) set = both;
    }
    if (sched_setaffinity(0, sizeof set, &set) != 0) { set_last_error("sched_setaffinity failed for device %d", device); return GOFR_ERR_UNSUPPORTED; }
#if defined(SYS_set_mempolicy)
    if (node >= 0 && node < 64) {  // MPOL_PREFERRED: pages this thread touches (pinned allocations included) come from the GPU's node
        unsigned long mask = 1ul << node;
        syscall(SYS_set_mempolicy, 1 /*MPOL_PREFERRED*/, &mask, 65ul);
    }
#endif
    return GOFR_OK;
}

void* gofr_alloc_pinned(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) { set_last_error("cudaMallocHost(%zu) failed", bytes); return nullptr; }
    return p;
}
void gofr_free_pinned(void* p) { if (p) cudaFreeHost(p); }

const char* gofr_last_error(void) { return g_err; }
uint32_t gofr_abi_version(void) { return GOFR_ABI_VERSION; }

void gofr_format_http_date(int64_t unix_seconds, char out29[29]) {
    static const char* days[] = {"Sun", "Mon", "Tue", "Wed", "Thu", "Fri", "Sat"};
    static const char* mons[] = {"Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"};
    time_t tt = (time_t)unix_seconds;
    struct tm g;
    gmtime_r(&tt, &g);
    char tmp[48];
    snprintf(tmp, sizeof tmp, "%s, %02d %s %04d %02d:%02d:%02d GMT", days[g.tm_wday], g.tm_mday, mons[g.tm_mon],
             g.tm_year + 1900, g.tm_hour, g.tm_min, g.tm_sec);
    memcpy(out29, tmp, 29);
}

int gofr_grpc_hello_device(gofr_engine* e, const uint8_t* d_in, const uint32_t* d_in_off, uint32_t n, uint8_t* d_out,
                           uint64_t out_cap, uint32_t* d_out_off, uint32_t* d_meta, void* stream) {
    if (!e || (n && (!d_in || !d_in_off || !d_out || !d_out_off || !d_meta))) return GOFR_ERR_INVALID;
    GrpcParams p;
    memset(&p, 0, sizeof p);
    p.in = d_in; p.in_off = d_in_off; p.meta = d_meta;
    return launch_frames(e, K_HELLO, p, n, d_out, out_cap, d_out_off, stream);
}

// rows → frames (decode == false) or frames → rows (decode == true): the same launch plumbing, two codecs
static int proto_run(gofr_engine* e, const gofr_proto_field* fields, uint32_t n_fields, const uint8_t* d_rows,
                     const uint32_t* d_row_off, uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                     uint32_t* d_meta, void* stream, bool decode) {
    if (!e || (n_fields && !fields) || (n && (!d_rows || !d_row_off || !d_out || !d_out_off || !d_meta))) return GOFR_ERR_INVALID;
    if (n_fields > GOFR_PROTO_MAX_FIELDS) { set_last_error("a message type may have at most %d fields", GOFR_PROTO_MAX_FIELDS); return GOFR_ERR_CAPACITY; }
    ProtoSchema S;
    memset(&S, 0, sizeof S);
    S.n_fields = n_fields;
    for (uint32_t k = 0; k < n_fields; k++) {
        const uint32_t num = fields[k].number, t = fields[k].type;
        const bool known = (t >= GOFR_PB_DOUBLE && t <= GOFR_PB_STRING) || (t >= GOFR_PB_BYTES && t <= GOFR_PB_SINT64);
        if (!known) { set_last_error("field %u: type %u is not a scalar proto3 type this encoder takes", num, t); return GOFR_ERR_UNSUPPORTED; }
        if (num == 0 || num > 0x1FFFFFFFu || (num >= 19000 && num <= 19999)) { set_last_error("field number %u is not valid", num); return GOFR_ERR_INVALID; }
        if (k && num <= fields[k - 1].number) { set_last_error("fields must be listed in ascending field-number order (%u after %u)", num, fields[k - 1].number); return GOFR_ERR_INVALID; }
        const bool is64 = t == GOFR_PB_DOUBLE || t == GOFR_PB_INT64 || t == GOFR_PB_UINT64 || t == GOFR_PB_FIXED64 || t == GOFR_PB_SFIXED64 || t == GOFR_PB_SINT64;
        const uint32_t wire = (t == GOFR_PB_STRING || t == GOFR_PB_BYTES) ? 2u : (t == GOFR_PB_DOUBLE || t == GOFR_PB_FIXED64 || t == GOFR_PB_SFIXED64) ? 1u
                            : (t == GOFR_PB_FLOAT || t == GOFR_PB_FIXED32 || t == GOFR_PB_SFIXED32) ? 5u : 0u;
        S.tag[k] = num << 3 | wire;
        S.cls[k] = (uint8_t)proto_class(t);
        S.fixed_bytes += is64 ? 8u : 4u;
    }
    GrpcParams p;
    memset(&p, 0, sizeof p);
    p.in = d_rows; p.in_off = d_row_off; p.meta = d_meta;
    return launch_frames(e, decode ? K_PROTO_DEC : K_PROTO_ENC, p, n, d_out, out_cap, d_out_off, stream, S);
}

// message types with nested / repeated fields -> the kernel's descriptor: validation, words of every fixed part, nesting depth.
// presence: one byte per field (0, GOFR_PB_OPTIONAL or a oneof group 1..7), or null
static int pbn_build(const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields, uint32_t root,
                     const uint8_t* presence, PbnDesc* D) {
    if (!msgs || !fields || n_msgs == 0 || n_msgs > (uint32_t)kPbnMaxMsgs || n_fields > (uint32_t)kPbnMaxFields || root >= n_msgs) {
        set_last_error("at most %d message types with %d fields in all", kPbnMaxMsgs, kPbnMaxFields);
        return GOFR_ERR_CAPACITY;
    }
    memset(D, 0, sizeof *D);
    D->n_msgs = (uint8_t)n_msgs;
    D->root = root;
    for (uint32_t m = 0; m < n_msgs; m++) {
        if (msgs[m].n_fields == 0 || (uint32_t)msgs[m].first_field + msgs[m].n_fields > n_fields) { set_last_error("message type %u: bad field range", m); return GOFR_ERR_INVALID; }
        D->first[m] = msgs[m].first_field;
        D->count[m] = msgs[m].n_fields;
        for (uint32_t k = 0; k < msgs[m].n_fields; k++) {
            const gofr_proto_nfield& f = fields[msgs[m].first_field + k];
            const uint32_t num = f.number, t = f.type;
            const bool scalar = (t >= GOFR_PB_DOUBLE && t <= GOFR_PB_STRING) || (t >= GOFR_PB_BYTES && t <= GOFR_PB_SINT64);
            const bool sub = t == GOFR_PB_MESSAGE || t == GOFR_PB_MAP;
            if (!scalar && !sub) { set_last_error("message type %u field %u: type %u is not taken", m, num, t); return GOFR_ERR_UNSUPPORTED; }
            if (sub && f.msg >= n_msgs) { set_last_error("message type %u field %u: unknown message type %u", m, num, f.msg); return GOFR_ERR_INVALID; }
            if (t == GOFR_PB_MAP && f.repeated) { set_last_error("message type %u field %u: a map field is not repeated", m, num); return GOFR_ERR_INVALID; }
            if (num == 0 || num > 0x1FFFFFFFu || (num >= 19000 && num <= 19999)) { set_last_error("field number %u is not valid", num); return GOFR_ERR_INVALID; }
            if (k && num <= fields[msgs[m].first_field + k - 1].number) { set_last_error("message type %u: fields must be in ascending field-number order", m); return GOFR_ERR_INVALID; }
            PbnField& F = D->f[msgs[m].first_field + k];
            F.flags = t == GOFR_PB_MAP ? (uint8_t)(PBN_REPEATED | PBN_MAP) : f.repeated ? (uint8_t)PBN_REPEATED : (uint8_t)0;
            F.msg = sub ? (uint8_t)f.msg : (uint8_t)0xFF;
            F.cls = sub ? 0 : (uint8_t)proto_class(t);
            // messages, map entries, strings, bytes and PACKED repeated scalars are length-delimited
            const uint32_t wire = (sub || (f.repeated && proto_wire(t) != 2)) ? 2u : proto_wire(t);
            F.tag = num << 3 | wire;
            // explicit presence: a oneof member is singular; optional on a message field is what a singular message field
            // is anyway (its presence word), so it marks nothing
            const uint32_t pr = presence ? presence[msgs[m].first_field + k] : 0u;
            if (pr > 7u && pr != GOFR_PB_OPTIONAL) { set_last_error("message type %u field %u: presence byte %u", m, num, pr); return GOFR_ERR_INVALID; }
            if (pr && (f.repeated || t == GOFR_PB_MAP)) {
                set_last_error("message type %u field %u: a repeated or map field has no presence", m, num);
                return GOFR_ERR_INVALID;
            }
            if (pr && pr != GOFR_PB_OPTIONAL) F.flags = (uint8_t)(pr << PBN_ONEOF_SHIFT | (sub ? 0u : (uint32_t)PBN_PRESENCE));
            else if (pr && !sub) F.flags = (uint8_t)PBN_PRESENCE;
            if (F.flags & (PBN_PRESENCE | PBN_ONEOF)) D->presence = 1;
        }
    }
    // map entry types: exactly (1 key, 2 value), singular; keys of integer, bool or string type; values anything but a map.
    // An entry type is neither the root nor the type of a message field.
    bool entry[kPbnMaxMsgs] = {false};
    for (uint32_t m = 0; m < n_msgs; m++)
        for (uint32_t k = 0; k < msgs[m].n_fields; k++)
            if (fields[msgs[m].first_field + k].type == GOFR_PB_MAP) entry[fields[msgs[m].first_field + k].msg] = true;
    for (uint32_t m = 0; m < n_msgs; m++) {
        for (uint32_t k = 0; k < msgs[m].n_fields; k++) {
            const gofr_proto_nfield& f = fields[msgs[m].first_field + k];
            if (f.type == GOFR_PB_MESSAGE && entry[f.msg]) { set_last_error("message type %u field %u: map entry type %u used as a message", m, f.number, f.msg); return GOFR_ERR_INVALID; }
        }
        if (!entry[m]) continue;
        D->maps = 1;
        if (m == root) { set_last_error("the root type %u is a map entry type", m); return GOFR_ERR_INVALID; }
        // the entry's key and value are marked in the shared field table: no other type may name them
        for (uint32_t o = 0; o < n_msgs; o++) {
            const uint32_t a0 = msgs[m].first_field, a1 = a0 + msgs[m].n_fields, b0 = msgs[o].first_field, b1 = b0 + msgs[o].n_fields;
            if (o != m && a0 < b1 && b0 < a1) { set_last_error("map entry type %u shares fields with message type %u", m, o); return GOFR_ERR_INVALID; }
        }
        const gofr_proto_nfield* kv = fields + msgs[m].first_field;
        if (msgs[m].n_fields != 2 || kv[0].number != 1 || kv[1].number != 2 || kv[0].repeated || kv[1].repeated) {
            set_last_error("map entry type %u: exactly the singular fields 1 (key) and 2 (value)", m);
            return GOFR_ERR_INVALID;
        }
        if (presence && (presence[msgs[m].first_field] || presence[msgs[m].first_field + 1])) {
            set_last_error("map entry type %u: its key and value carry no presence", m);
            return GOFR_ERR_INVALID;
        }
        const uint32_t kt = kv[0].type;
        const bool key_ok = kt == GOFR_PB_INT32 || kt == GOFR_PB_INT64 || kt == GOFR_PB_UINT32 || kt == GOFR_PB_UINT64 || kt == GOFR_PB_SINT32 ||
                            kt == GOFR_PB_SINT64 || kt == GOFR_PB_FIXED32 || kt == GOFR_PB_FIXED64 || kt == GOFR_PB_SFIXED32 ||
                            kt == GOFR_PB_SFIXED64 || kt == GOFR_PB_BOOL || kt == GOFR_PB_STRING;
        if (!key_ok) { set_last_error("map entry type %u: a key of type %u", m, kt); return GOFR_ERR_INVALID; }
        if (kv[1].type == GOFR_PB_MAP) { set_last_error("map entry type %u: a map-valued map", m); return GOFR_ERR_INVALID; }
        const bool signed_key = kt == GOFR_PB_INT32 || kt == GOFR_PB_INT64 || kt == GOFR_PB_SINT32 || kt == GOFR_PB_SINT64 ||
                                kt == GOFR_PB_SFIXED32 || kt == GOFR_PB_SFIXED64;
        D->f[D->first[m]].flags |= (uint8_t)(PBN_ENTRY | (signed_key ? PBN_SIGNED : 0));
        D->f[D->first[m] + 1].flags |= (uint8_t)PBN_ENTRY;
    }
    // fixed words and depth, depth first; a message type that reaches itself has no bound on its nesting
    int state[kPbnMaxMsgs] = {0}, depth[kPbnMaxMsgs] = {0};
    std::function<int(uint32_t)> visit = [&](uint32_t m) -> int {
        if (state[m] == 2) return GOFR_OK;
        if (state[m] == 1) { set_last_error("message type %u is recursive", m); return GOFR_ERR_UNSUPPORTED; }
        state[m] = 1;
        uint32_t words = 0;
        int d = 1;
        for (uint32_t k = 0; k < D->count[m]; k++) {
            PbnField& F = D->f[D->first[m] + k];
            uint32_t w = (F.flags & PBN_REPEATED) ? 1u : (F.cls & PC_64) ? 2u : 1u;
            if (F.flags & PBN_PRESENCE) w++;  // the presence word
            if (F.msg != 0xFF) {
                int rc = visit(F.msg);
                if (rc) return rc;
                d = std::max(d, 1 + depth[F.msg]);
                if (!(F.flags & PBN_REPEATED)) w = 1u + D->fixed_words[F.msg];
            }
            if (w > 255u) { set_last_error("message type %u: fixed part too wide", m); return GOFR_ERR_UNSUPPORTED; }
            F.fixed_words = (uint8_t)w;
            words += w;
        }
        if (words > 16383u) { set_last_error("message type %u: fixed part too wide", m); return GOFR_ERR_UNSUPPORTED; }
        D->fixed_words[m] = (uint16_t)words;
        depth[m] = d;
        state[m] = 2;
        return GOFR_OK;
    };
    for (uint32_t m = 0; m < n_msgs; m++) { int rc = visit(m); if (rc) return rc; }
    if (depth[root] > kPbnMaxDepth) { set_last_error("messages nest deeper than %d levels", kPbnMaxDepth); return GOFR_ERR_UNSUPPORTED; }
    return GOFR_OK;
}

// The nested codec's instance for a description: presence-free, no presence code; map-free too, no map code
static Kern pbn_kernel(const PbnDesc& D, bool decode) {
    return D.presence ? (decode ? K_PBN_DEC_PRES : K_PBN_ENC_PRES)
         : D.maps     ? (decode ? K_PBN_DEC_MAPS : K_PBN_ENC_MAPS) : (decode ? K_PBN_DEC : K_PBN_ENC);
}

static int proto_nested_run(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                            uint32_t root, const uint8_t* presence, const uint8_t* d_in, const uint32_t* d_in_off, uint32_t n,
                            uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off, uint32_t* d_meta, void* stream, bool decode) {
    if (!e || (n && (!d_in || !d_in_off || !d_out || !d_out_off || !d_meta))) return GOFR_ERR_INVALID;
    PbnDesc D;
    { int rc = pbn_build(msgs, n_msgs, fields, n_fields, root, presence, &D); if (rc) return rc; }
    GrpcParams p;
    memset(&p, 0, sizeof p);
    p.in = d_in; p.in_off = d_in_off; p.meta = d_meta;
    return launch_frames(e, pbn_kernel(D, decode), p, n, d_out, out_cap, d_out_off, stream, D);
}

int gofr_proto_encode_nested_device(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                    uint32_t n_fields, uint32_t root, const uint8_t* d_rows, const uint32_t* d_row_off, uint32_t n,
                                    uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off, uint32_t* d_meta, void* stream) {
    return proto_nested_run(e, msgs, n_msgs, fields, n_fields, root, nullptr, d_rows, d_row_off, n, d_out, out_cap, d_out_off, d_meta,
                            stream, false);
}

int gofr_proto_decode_nested_device(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                    uint32_t n_fields, uint32_t root, const uint8_t* d_in, const uint32_t* d_in_off, uint32_t n,
                                    uint8_t* d_rows, uint64_t rows_cap, uint32_t* d_row_off, uint32_t* d_meta, void* stream) {
    return proto_nested_run(e, msgs, n_msgs, fields, n_fields, root, nullptr, d_in, d_in_off, n, d_rows, rows_cap, d_row_off, d_meta,
                            stream, true);
}

int gofr_proto_encode_nested_ex_device(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                       uint32_t n_fields, uint32_t root, const uint8_t* presence, const uint8_t* d_rows,
                                       const uint32_t* d_row_off, uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                                       uint32_t* d_meta, void* stream) {
    return proto_nested_run(e, msgs, n_msgs, fields, n_fields, root, presence, d_rows, d_row_off, n, d_out, out_cap, d_out_off, d_meta,
                            stream, false);
}

int gofr_proto_decode_nested_ex_device(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                       uint32_t n_fields, uint32_t root, const uint8_t* presence, const uint8_t* d_in,
                                       const uint32_t* d_in_off, uint32_t n, uint8_t* d_rows, uint64_t rows_cap, uint32_t* d_row_off,
                                       uint32_t* d_meta, void* stream) {
    return proto_nested_run(e, msgs, n_msgs, fields, n_fields, root, presence, d_in, d_in_off, n, d_rows, rows_cap, d_row_off, d_meta,
                            stream, true);
}

// Map fields on the deepest path from message type m: how many sorted entry lists the second pass keeps at once
static uint32_t pbn_map_levels(const PbnDesc& D, uint32_t m) {
    uint32_t most = 0;
    for (uint32_t k = 0; k < D.count[m]; k++) {
        const PbnField& F = D.f[D.first[m] + k];
        if (F.msg != 0xFF) most = std::max(most, ((F.flags & PBN_MAP) ? 1u : 0u) + pbn_map_levels(D, F.msg));
    }
    return most;
}

int gofr_proto_decode_nested_deferred_device(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                             uint32_t n_fields, uint32_t root, const uint8_t* presence, const uint8_t* d_in,
                                             const uint32_t* d_in_off, uint32_t n, const uint32_t* d_meta_in, uint8_t* d_rows,
                                             uint64_t rows_cap, uint32_t* d_row_off, uint32_t* d_meta, void* stream) {
    if (!e || (n && (!d_in || !d_in_off || !d_meta_in || !d_rows || !d_row_off || !d_meta))) return GOFR_ERR_INVALID;
    PbnDesc D;
    { int rc = pbn_build(msgs, n_msgs, fields, n_fields, root, presence, &D); if (rc) return rc; }
    const uint32_t levels = pbn_map_levels(D, D.root);  // (the depth limit keeps it at kPdnMaxMapLevels or below)
    if (levels > kPdnMaxMapLevels) { set_last_error("map fields nest %u deep", levels); return GOFR_ERR_UNSUPPORTED; }
    GrpcParams p;
    memset(&p, 0, sizeof p);
    p.in = d_in; p.in_off = d_in_off; p.meta = d_meta;
    return launch_frames_smem(e, K_PBN_DEC_DEFERRED, pdn_sort_bytes(levels), p, n, d_rows, rows_cap, d_row_off, stream, d_meta_in, D);
}

// gofr_proto_nested_bound: (per_byte, per_record) such that no record of b bytes yields more than per_byte * b + per_record
// output bytes, from the description alone.
// Decode (frame → row; the rule of engine.row_growth_bound in Python, which calls this): every element of a repeated field
// or map takes at least two bytes on the wire (a tag, then a length or a value) and brings its fixed part (a message or map
// entry: its type's fixed words, absent singular messages inline as zeros) or at most 8 bytes; a packed element takes one
// byte and brings at most 8; string bytes are copied once; later equal keys of a map and repeated singular fields only
// replace.  So per_byte = max(8, ceil(fixed bytes of an element type / 2)), and an empty frame still gives the root's
// fixed part, rounded up to a word: per_record = its fixed bytes + 3.
// Encode (row → frame with its 5-byte prefix): each byte written is charged to a row word or to a string byte.  String and
// bytes contents are copied once (1 per byte).  A word is charged what its own field writes:
//   scalar                  tag (tl bytes) + at most 10 (a varint: a negative int32 takes ten), 8 or 4;
//   string / bytes length,  tag + a length of at most 5 (a frame's length fits 32 bits);
//   singular message presence word, packed repeated count word, repeated string element: the same, tl + 5;
//   packed element          at most 10 (a 64-bit kind spreads its ten over two words);
//   presence word of an explicit-presence scalar: nothing (its value word pays);
// plus, on the first word of an element of a repeated message field or a map (an entry: key, then value, both written
// even at zero values, each a scalar or message of its own above), that element's tag and length, tl + 5.  An element's
// fixed part is at least one word, because pbn_build refuses a message type with no fields, and a word is the first word
// of at most one element.  So with W the most a word pays for itself and H the largest element header, per_byte =
// ceil((W + H) / 4) (at least 1, for string bytes), per_record = 5.  tl is the varint length of the field's tag: 5 bytes
// for field numbers from 2^25 on.
static void pbn_bound(const PbnDesc& D, bool decode, uint32_t* per_byte, uint32_t* per_record) {
    auto vlen = [](uint32_t v) { return v < 0x80u ? 1u : v < 0x4000u ? 2u : v < 0x200000u ? 3u : v < 0x10000000u ? 4u : 5u; };
    uint32_t elem = 0, W = 0, H = 0;
    for (uint32_t m = 0; m < D.n_msgs; m++) {
        for (uint32_t k = 0; k < D.count[m]; k++) {
            const PbnField& F = D.f[D.first[m] + k];
            const bool sub = F.msg != 0xFF, rep = (F.flags & PBN_REPEATED) != 0;
            const uint32_t tl = vlen(F.tag), wire = F.cls & PC_WIRE;
            const uint32_t scalar = wire == 0 ? 10u : wire == 1 ? 8u : wire == 5 ? 4u : 5u;  // what follows the tag
            if (rep && sub) {  // a repeated message field or a map
                elem = std::max<uint32_t>(elem, 4u * D.fixed_words[F.msg]);
                H = std::max(H, tl + 5u);
            } else if (rep) {
                W = std::max(W, std::max(tl + 5u, wire == 2 ? tl + 5u : scalar));
            } else {
                W = std::max(W, sub ? tl + 5u : tl + scalar);
            }
        }
    }
    if (decode) {
        *per_byte = std::max(8u, (elem + 1u) / 2u);
        *per_record = 4u * D.fixed_words[D.root] + 3u;
    } else {
        *per_byte = std::max(1u, (W + H + 3u) / 4u);
        *per_record = 5u;
    }
}

int gofr_proto_nested_bound(const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                            uint32_t root, const uint8_t* presence, int decode, uint32_t* per_byte, uint32_t* per_record) {
    if (!per_byte || !per_record) return GOFR_ERR_INVALID;
    PbnDesc D;
    { int rc = pbn_build(msgs, n_msgs, fields, n_fields, root, presence, &D); if (rc) return rc; }
    pbn_bound(D, decode != 0, per_byte, per_record);
    return GOFR_OK;
}

// Device bytes a proto chunk's output bound may take per slot: a chunk holds at most e->chunk records and, unless it is a
// single record, records whose bounds sum to no more than this.  Decode grows by up to a few hundred bytes per wire byte
// in the worst case, so a record count alone could ask for gigabytes.  Each slot holds three buffers of this size when
// decoding (the two passes' rows and the packed chunk).
static constexpr uint64_t kProtoChunkBudget = 256ull << 20;

// The host-buffer calls of the nested codec: the chunk loop of the request batches (req_chunks) with the codec kernels,
// then the pack kernel.  With a log (encode only): each chunk's log records, their arena range and trace_ids go up with its
// rows, and after the frames have shipped the proto-fed request-log kernel (proto_log_kernel.cu) writes every record's
// line, which is empty unless its kind is GOFR_LOG_RPC; chunk_pack_kernel places the lines.
static int proto_batch_locked(gofr_engine* e, const PbnDesc& D, bool decode, const gofr_proto_batch* in, gofr_resp_batch* out,
                              gofr_batch_log* log, const uint8_t* trace_ids, gofr_ticket* ticket) {
    uint32_t per_byte = 0, per_record = 0;
    pbn_bound(D, decode, &per_byte, &per_record);
    const uint32_t levels = pbn_map_levels(D, D.root);
    if (decode && levels > kPdnMaxMapLevels) { set_last_error("map fields nest %u deep", levels); return GOFR_ERR_UNSUPPORTED; }
    const uint32_t* off = in->off;
    ChunkSteps steps;
    // Offsets come from the caller: validated here in 64 bits, a chunk at a time (non-decreasing, within data_bytes, rows
    // on 4-byte boundaries).  The chunk's output bound includes the 16 bytes the packed output may start into its buffer.
    steps.plan = [&](uint32_t lo, ChunkPlan* c) -> int {
        const uint32_t lim = lo + std::min<uint32_t>(e->chunk, in->n - lo);
        const uint64_t start = off[lo];
        if (start > in->data_bytes || (!decode && (start & 3u))) {
            set_last_error("record %u starts at %llu: outside the data or not a multiple of 4", lo, (unsigned long long)start);
            return GOFR_ERR_INVALID;
        }
        uint64_t bound = 0;
        uint32_t hi = lo;
        for (; hi < lim; hi++) {
            const uint64_t a = off[hi], b = off[hi + 1];
            if (b < a || b > in->data_bytes || (!decode && (b & 3u))) {
                set_last_error("record %u: offsets %llu .. %llu are decreasing, outside the data or not multiples of 4", hi,
                               (unsigned long long)a, (unsigned long long)b);
                return GOFR_ERR_INVALID;
            }
            const uint64_t rb = (uint64_t)per_byte * (b - a) + per_record;
            if (hi > lo && bound + rb > kProtoChunkBudget) break;
            bound += rb;
        }
        // a single record with a larger bound gets a chunk of its own; no output offset passes 32 bits, so neither does a
        // buffer (a record that would is reported as a capacity error by the kernels)
        *c = {lo, hi, (uint32_t)(start & ~15ull), off[hi], std::min<uint64_t>(bound, 1ull << 32) + 16};
        return log ? batch_log_plan(log, GOFR_LOG_RPC, lo, hi, &c->log_lo, &c->log_hi, &c->log_bound) : GOFR_OK;
    };
    // A chunk ends at e->chunk records, or where it and the next chunk's first record together pass the budget: two
    // neighbours' bounds, which sum to at most per_byte * data_bytes + per_record * n over the batch, take more than it.
    const uint64_t n = in->n, all = (uint64_t)per_byte * in->data_bytes + (uint64_t)per_record * n;
    steps.max_chunks = (n + e->chunk - 1) / e->chunk + 2 * (all / kProtoChunkBudget) + 2;
    steps.upload = [&](Slot& s, const ChunkPlan& c, cudaStream_t st) -> int {
        const uint32_t cn = c.hi - c.lo;
        { int rc = s.reserve_codec(cn, c.out_bound, decode ? c.out_bound : 0); if (rc) return rc; }
        CUDA_TRY(cudaMemcpyAsync(s.d_in_off, off + c.lo, (size_t)(cn + 1) * 4, cudaMemcpyHostToDevice, st));
        if (c.arena_hi > c.arena_lo) CUDA_TRY(cudaMemcpyAsync(s.d_arena, in->data + c.arena_lo, c.arena_hi - c.arena_lo, cudaMemcpyHostToDevice, st));
        return log ? upload_log(s, c, log, trace_ids, st) : GOFR_OK;
    };
    // records keep their absolute offsets: pass a rebased input pointer.  The codec kernels write from byte 0 of their own
    // buffers (16 bytes short of their end: the pack kernel's copy reads a word past a record's last byte).
    steps.compute = [&](Slot& s, const ChunkPlan& c, cudaStream_t st, const unsigned long long* chain_pos) -> int {
        const uint32_t cn = c.hi - c.lo;
        GrpcParams p;
        memset(&p, 0, sizeof p);
        p.in = s.d_arena - c.arena_lo; p.in_off = s.d_in_off;
        PackParams q;
        memset(&q, 0, sizeof q);
        q.a = s.d_codec[0]; q.a_off = s.d_codec_off[0]; q.a_cap = s.cap_codec[0] - 16; q.chain_pos = chain_pos;
        p.meta = decode ? s.d_meta1 : s.d_meta;
        int rc = launch_frames_locked(e, pbn_kernel(D, decode), 0, p, cn, s.d_codec[0], q.a_cap, s.d_codec_off[0], s.state, s.d_flag, st, D);
        if (!rc && decode) {  // the second pass over the first one's statuses, always: with nothing DEFER it is a scan
            p.meta = s.d_meta;
            q.b = s.d_codec[1]; q.b_off = s.d_codec_off[1]; q.b_cap = s.cap_codec[1] - 16; q.sel = s.d_meta1;
            rc = launch_frames_locked(e, K_PBN_DEC_DEFERRED, pdn_sort_bytes(levels), p, cn, s.d_codec[1], q.b_cap, s.d_codec_off[1],
                                      s.state, s.d_flag, st, (const uint32_t*)s.d_meta1, D);
        }
        if (!rc) rc = launch_frames_locked(e, K_PACK, 0, q, cn, s.d_out, s.cap_out, s.d_off, s.state, s.d_flag, st);
        return rc;
    };
    if (log) steps.lines = [&](Slot& s, const ChunkPlan& c, cudaStream_t st, const unsigned long long* chain_pos) -> int {
        return chunk_lines(e, K_PROTO_LOG, s, c, s.d_lids, st, chain_pos, log->log_unix_ns, e->d_chain + 2);
    };
    return req_chunks(e, in->n, steps, out, nullptr, log, ticket);
}

static int proto_batch(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                       uint32_t root, const uint8_t* presence, const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* ticket,
                       bool decode, gofr_batch_log* log = nullptr, const uint8_t* trace_ids = nullptr) {
    if (!e || !in || !out || !ticket) return GOFR_ERR_INVALID;
    if (in->n && (!in->off || !out->out || !out->out_off || !out->meta)) return GOFR_ERR_INVALID;
    if (in->data_bytes && !in->data) return GOFR_ERR_INVALID;
    PbnDesc D;
    { int rc = pbn_build(msgs, n_msgs, fields, n_fields, root, presence, &D); if (rc) return rc; }
    return host_batch(e, [&] { return proto_batch_locked(e, D, decode, in, out, log, trace_ids, ticket); });
}

int gofr_proto_batch_decode(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                            uint32_t root, const uint8_t* presence, const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* ticket) {
    return proto_batch(e, msgs, n_msgs, fields, n_fields, root, presence, in, out, ticket, true);
}

int gofr_proto_batch_encode(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                            uint32_t root, const uint8_t* presence, const gofr_proto_batch* in, gofr_resp_batch* out, gofr_ticket* ticket) {
    return proto_batch(e, msgs, n_msgs, fields, n_fields, root, presence, in, out, ticket, false);
}

int gofr_proto_batch_encode_log(gofr_engine* e, const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields,
                                uint32_t n_fields, uint32_t root, const uint8_t* presence, const gofr_proto_batch* in,
                                const uint8_t* trace_ids, gofr_resp_batch* out, gofr_batch_log* log, gofr_ticket* ticket) {
    if (!log || (in && in->n && (!log->desc || !log->out || !log->log_off || !trace_ids))) return GOFR_ERR_INVALID;
    return proto_batch(e, msgs, n_msgs, fields, n_fields, root, presence, in, out, ticket, false, log, trace_ids);
}

// the descriptor gofr_proto_encode_nested_device would hand to its kernel (tests/emu drives the device code with it)
int gofr_proto_nested_describe_ex(const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                                  uint32_t root, const uint8_t* presence, void* desc_out, uint32_t desc_cap) {
    PbnDesc D;
    int rc = pbn_build(msgs, n_msgs, fields, n_fields, root, presence, &D);
    if (rc) return rc;
    if (!desc_out || desc_cap < sizeof D) return GOFR_ERR_CAPACITY;
    memcpy(desc_out, &D, sizeof D);
    return GOFR_OK;
}

int gofr_proto_nested_describe(const gofr_proto_nmsg* msgs, uint32_t n_msgs, const gofr_proto_nfield* fields, uint32_t n_fields,
                               uint32_t root, void* desc_out, uint32_t desc_cap) {
    return gofr_proto_nested_describe_ex(msgs, n_msgs, fields, n_fields, root, nullptr, desc_out, desc_cap);
}

int gofr_proto_encode_device(gofr_engine* e, const gofr_proto_field* fields, uint32_t n_fields, const uint8_t* d_rows,
                             const uint32_t* d_row_off, uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off,
                             uint32_t* d_meta, void* stream) {
    return proto_run(e, fields, n_fields, d_rows, d_row_off, n, d_out, out_cap, d_out_off, d_meta, stream, false);
}

int gofr_proto_decode_device(gofr_engine* e, const gofr_proto_field* fields, uint32_t n_fields, const uint8_t* d_in,
                             const uint32_t* d_in_off, uint32_t n, uint8_t* d_rows, uint64_t rows_cap, uint32_t* d_row_off,
                             uint32_t* d_meta, void* stream) {
    return proto_run(e, fields, n_fields, d_in, d_in_off, n, d_rows, rows_cap, d_row_off, d_meta, stream, true);
}

int gofr_route_device(gofr_engine* e, const gofr_req_desc* d_desc, const uint8_t* d_arena, uint32_t n, uint32_t* d_meta,
                      uint32_t* d_vars, void* stream) {
    if (!e || (n && (!d_desc || !d_arena || !d_meta || !d_vars))) return GOFR_ERR_INVALID;
    if (n == 0) return GOFR_OK;
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    return launch_route_kernel(e, d_desc, d_arena, n, d_meta, d_vars, (cudaStream_t)stream);
}

int gofr_bind_device(gofr_engine* e, uint32_t schema_id, const gofr_req_desc* d_desc, const uint8_t* d_arena, uint32_t n,
                     uint8_t* d_rows, uint32_t slot_bytes, uint32_t* d_len, uint32_t* d_status, void* stream) {
    if (!e || (n && (!d_desc || !d_arena || !d_rows || !d_len || !d_status))) return GOFR_ERR_INVALID;
    if (slot_bytes == 0 || (slot_bytes & 15u) || ((uintptr_t)d_rows & 15u)) { set_last_error("slot_bytes must be a positive multiple of 16 and d_rows 16-byte aligned"); return GOFR_ERR_INVALID; }
    uint32_t sidx = 0;
    { int rc = bind_schema(e, schema_id, &sidx); if (rc) return rc; }
    if (n == 0) return GOFR_OK;
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    return launch_bind_kernel(e, sidx, d_desc, d_arena, n, d_rows, slot_bytes, d_len, d_status, (cudaStream_t)stream);
}

// The chunk loop of the split API's host stages (gofr_batch_route, gofr_batch_bind): a chunk's descriptors and the arena
// bytes it reads go up, `stage(lo, n, arena, stream)` launches its kernel on them and enqueues the copies of its result
// columns, and they are back before the next chunk goes up.
static int host_stage(gofr_engine* e, const gofr_req_batch* in, bool path_only,
                      const std::function<int(uint32_t, uint32_t, const uint8_t*, cudaStream_t)>& stage) {
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    const cudaStream_t st = e->st_compute;
    for (uint32_t lo = 0; lo < in->n; lo += e->chunk) {
        const uint32_t hi = std::min<uint32_t>(in->n, lo + e->chunk), cn = hi - lo;
        uint32_t alo = 0, ahi = 0;
        int rc = chunk_arena_range(in, lo, hi, path_only, &alo, &ahi);
        if (!rc) rc = grow((void**)&e->d_rt_desc, &e->rt_desc_cap, (size_t)cn * 16, 256);
        if (!rc) rc = grow((void**)&e->d_rt_arena, &e->rt_arena_cap, (size_t)ahi - alo + kArenaSlack, 256);
        if (!rc) rc = upload_chunk(in, lo, cn, alo, ahi, e->d_rt_desc, nullptr, e->d_rt_arena, st);
        if (!rc) rc = stage(lo, cn, e->d_rt_arena - alo, st);  // descriptors keep absolute arena offsets
        if (rc) return rc;
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    return GOFR_OK;
}

int gofr_batch_bind(gofr_engine* e, uint32_t schema_id, const gofr_req_batch* in, uint8_t* rows, uint32_t slot_bytes,
                    uint32_t* len, uint32_t* status) {
    if (!e || !in || (in->n && (!in->desc || !rows || !len || !status))) return GOFR_ERR_INVALID;
    if (slot_bytes == 0 || (slot_bytes & 15u)) { set_last_error("slot_bytes must be a positive multiple of 16"); return GOFR_ERR_INVALID; }
    uint32_t sidx = 0;
    { int rc = bind_schema(e, schema_id, &sidx); if (rc) return rc; }
    return host_stage(e, in, false, [&](uint32_t lo, uint32_t cn, const uint8_t* d_arena, cudaStream_t st) -> int {
        int rc = grow((void**)&e->d_rt_meta, &e->rt_meta_cap, (size_t)cn * 8, 256);
        if (!rc) rc = grow((void**)&e->d_rt_rows, &e->rt_rows_cap, (size_t)cn * slot_bytes, 256);
        uint32_t* d_len = (uint32_t*)e->d_rt_meta;
        if (!rc) rc = launch_bind_kernel(e, sidx, e->d_rt_desc, d_arena, cn, e->d_rt_rows, slot_bytes, d_len, d_len + cn, st);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(rows + (size_t)lo * slot_bytes, e->d_rt_rows, (size_t)cn * slot_bytes, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(len + lo, d_len, (size_t)cn * 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(status + lo, d_len + cn, (size_t)cn * 4, cudaMemcpyDeviceToHost, st));
        return GOFR_OK;
    });
}

int gofr_batch_route(gofr_engine* e, const gofr_req_batch* in, uint32_t* meta, uint32_t* vars) {
    if (!e || !in || (in->n && (!in->desc || !meta || !vars))) return GOFR_ERR_INVALID;
    return host_stage(e, in, true, [&](uint32_t lo, uint32_t cn, const uint8_t* d_arena, cudaStream_t st) -> int {
        const size_t vbytes = (size_t)cn * 4 * GOFR_MAX_PATH_VARS;
        int rc = grow((void**)&e->d_rt_meta, &e->rt_meta_cap, (size_t)cn * 4, 256);
        if (!rc) rc = grow((void**)&e->d_rt_vars, &e->rt_vars_cap, vbytes, 256);
        if (!rc) rc = launch_route_kernel(e, e->d_rt_desc, d_arena, cn, (uint32_t*)e->d_rt_meta, (uint32_t*)e->d_rt_vars, st);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(meta + lo, e->d_rt_meta, (size_t)cn * 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(vars + (size_t)lo * GOFR_MAX_PATH_VARS, e->d_rt_vars, vbytes, cudaMemcpyDeviceToHost, st));
        return GOFR_OK;
    });
}

int gofr_http_parse_device(gofr_engine* e, const uint8_t* d_raw, const uint32_t* d_raw_off, uint32_t n, gofr_req_desc* d_desc,
                           uint8_t* d_arena, uint32_t* d_status, uint64_t* d_spans, void* stream) {
    if (!e || (n && (!d_raw || !d_raw_off || !d_desc || !d_arena || !d_status || !d_spans))) return GOFR_ERR_INVALID;
    if (n == 0) return GOFR_OK;
    std::lock_guard<std::mutex> g(e->mu);
    CUDA_TRY(cudaSetDevice(e->device));
    const int resident = resident_grid(e, K_HTTP);
    if (!resident) return GOFR_ERR_CUDA;
    HttpParams p;
    memset(&p, 0, sizeof p);
    p.raw = d_raw; p.raw_off = d_raw_off; p.n = n; p.n_tiles = (n + kServeThreads - 1) / kServeThreads;
    p.desc = d_desc; p.arena = d_arena; p.status = d_status; p.spans = (unsigned long long*)d_spans;
    // no look-back: every message's result lands in the bytes it occupies, so the whole resident grid runs
    return launch(e, K_HTTP, (int)std::min<uint32_t>((uint32_t)resident, p.n_tiles), 0, (cudaStream_t)stream, p);
}

int gofr_http_frame_device(gofr_engine* e, const uint8_t* d_buf, const uint32_t* d_buf_off, uint32_t n_conns, uint32_t* d_rec_off,
                           uint32_t rec_cap, uint32_t* d_first, uint32_t* d_consumed, uint32_t* d_conn_status, void* stream) {
    if (!e) return GOFR_ERR_INVALID;
    if (n_conns == 0) return GOFR_OK;
    if (!d_buf || !d_buf_off || !d_rec_off || !d_first || !d_consumed || !d_conn_status) return GOFR_ERR_INVALID;
    if (((uintptr_t)d_buf & 15u) || (((uintptr_t)d_buf_off | (uintptr_t)d_rec_off | (uintptr_t)d_first | (uintptr_t)d_consumed |
                                      (uintptr_t)d_conn_status) & 3u)) {
        set_last_error("d_buf must be 16-byte aligned and the offset, record and per-connection columns 4-byte aligned");
        return GOFR_ERR_INVALID;
    }
    HttpFrameParams p;
    memset(&p, 0, sizeof p);
    p.buf = d_buf; p.buf_off = d_buf_off; p.consumed = d_consumed; p.status = d_conn_status;
    // the record column is the packed output (rec_cap records), d_first its offset column
    return launch_frames(e, K_HTTP_FRAME, p, n_conns, (uint8_t*)d_rec_off, rec_cap, d_first, stream);
}

int gofr_requestlog_device(gofr_engine* e, const gofr_log_desc* d_desc, const uint8_t* d_trace_ids, const uint8_t* d_arena,
                           uint32_t n, uint8_t* d_out, uint64_t out_cap, uint32_t* d_out_off, void* stream) {
    if (!e || (n && (!d_desc || !d_trace_ids || !d_arena || !d_out || !d_out_off))) return GOFR_ERR_INVALID;
    LogParams p;
    memset(&p, 0, sizeof p);
    p.desc = d_desc; p.ids = d_trace_ids; p.arena = d_arena;
    return launch_frames(e, K_REQLOG, p, n, d_out, out_cap, d_out_off, stream);
}

}  // extern "C"
