// reqlog_tiles.cuh — the tile loop of the request-log kernels (sm_90a), one thread per record on the tile skeleton of
// tile_common.cuh; lines are packed in record order through the staging Writer.  Per-record logic: reqlog_device.cuh.
//
// Three instances: reqlog_kernel.cu (gofr_requestlog_device, the connection path's lines) takes every record as it is;
// batch_log_kernel.cu (gofr_batch_submit_log) first lets the serve kernel's status decide, per record, whether it has a
// line at all, and proto_log_kernel.cu (gofr_proto_batch_encode_log) lets the record's kind decide (batch_log_device.cuh).
// The Feed does that: feed(i, d) may rewrite record i and returns whether it has a
// line; a record without one takes no staged bytes and gets an empty line.  Feed::kEvery says every record has one (the
// first instance: its code stays what it was before the loop was shared).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "engine_internal.h"
#include "reqlog_device.cuh"
#include "tile_common.cuh"

namespace gofr {

constexpr int LT = kServeThreads;
constexpr int LNW = LT / 32;
constexpr uint32_t kLogStage = 24 * 1024;  // bytes of record strings staged per tile (128 records × 192 B)

struct LogShared {
    uint64_t bar;
    uint32_t warp_sum[LNW];
    uint32_t warp_lo[LNW], warp_hi[LNW];
    unsigned long long tile_base;
    uint32_t in_lo, in_hi;
    uint32_t stage[GOFR_STAGE_WORDS * LT];
    __align__(16) uint8_t in[kLogStage + 32];
};

// A Feed's line count: each warp adds the lines of its records to *lines, the batch's count, so that it never has to come
// back mid-batch.  Returns `line`.
__device__ __forceinline__ bool count_line(bool line, unsigned long long* lines) {
    const uint32_t m = __activemask(), b = __ballot_sync(m, line);
    if (line && (threadIdx.x & 31u) == (uint32_t)(__ffs(b) - 1)) atomicAdd(lines, (unsigned long long)__popc(b));
    return line;
}

template <class Feed>
__device__ __forceinline__ void reqlog_tiles(const LogParams p, const Feed feed) {
    __shared__ __align__(16) LogShared sh;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) tile_barrier_init(&sh.bar);
    __syncthreads();
    uint32_t parity = 0;
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const uint32_t i = tile * LT + tid;
        const bool valid = i < p.n;
        LogDesc d;
        memset(&d, 0, sizeof d);
        bool fed = false;
        if (valid) {
            const uint4* q = (const uint4*)p.desc + (size_t)i * 3;
            uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2);
            uint4* dd = (uint4*)&d;
            dd[0] = a; dd[1] = b; dd[2] = c;
            fed = feed(i, d);
        }
        const bool line = Feed::kEvery ? valid : fed;
        const uint32_t rec_len = (uint32_t)d.method_len + d.ua_len + d.xff_len + d.remote_len + d.uri_len;

        // ---- the tile's arena byte range ----
        warp_range(line ? d.arena_off : 0xFFFFFFFFu, line ? d.arena_off + rec_len : 0u, sh.warp_lo, sh.warp_hi);
        __syncthreads();  // also: every thread is done reading the previous tile's staged bytes
        if (tid == 0) {
            // 4 bytes of tail: the Writer may read the aligned word after a source's last byte
            stage_start(&sh.bar, sh.in, p.arena, cta_range(sh.warp_lo, sh.warp_hi, 4u, sh.in_lo, sh.in_hi), kLogStage);
        }
        __syncthreads();
        const ByteRange in{sh.in_lo, sh.in_hi};
        const bool staged = stageable(in, kLogStage);
        const uint8_t* rec = stage_wait(&sh.bar, parity, sh.in, p.arena, in, kLogStage) + d.arena_off;

        LogCtx c;
        c.ip_off = c.ip_len = c.esc_mask = c.total_len = 0;
        if (line) reqlog_size(d, rec, staged, c);

        const TilePlace t = place_tile(p, tile, c.total_len, sh.warp_sum, sh.tile_base);
        if (valid) put_offsets(p.out_off, i, p.n, t, c.total_len);
        if (t.fits && line) {
            const uint4 idv = __ldg((const uint4*)p.ids + i);
            const uint32_t id[4] = {idv.x, idv.y, idv.z, idv.w};
            reqlog_emit(d, rec, staged, id, c, p.out + t.base + t.excl, &sh.stage[tid]);
        }
    }
}

}  // namespace gofr
