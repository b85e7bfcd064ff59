// conn_result_device.cuh — per-request logic of gofr_conn_batch_respond's splice step (conn_result_kernel.cu), compiled for
// the device and, through tests/emu/emu_conn_result.cpp, for the host.
//
// After the compact step, request i of a chunk has a descriptor into the parse kernel's arena: decoded path | query | pad4 |
// body at its raw offset rounded up to 4.  The caller's closures have produced GOFR_H_RESULT records for some requests.  The
// splice writes every request again, in request order, into a packed arena of its own: path | query | pad4 | data | pad4,
// where data is the request's record when that is not empty and its own body otherwise, and points the descriptor at it.
// The serve kernel then reads that arena as it reads any request batch.  Sources have any alignment (paths start at a
// multiple of 4, records anywhere), so the bytes go through the Writer's copy.
#pragma once
#include "engine_internal.h"
#include "serve_device.cuh"

namespace gofr {

struct ConnSplice {
    gofr_req_desc d;      // the request's descriptor in the parse arena
    const uint8_t* data;  // its data section: the record, or its body in the parse arena
    uint32_t data_len;
    uint32_t size;        // bytes of its spliced form: round4(path + query) + round4(data)
};

GOFR_HD uint32_t conn_round4(uint32_t x) { return (x + 3u) & ~3u; }

// Request i's data section and the size of its spliced form
GOFR_HD ConnSplice conn_splice(const ConnResultParams& p, uint32_t i) {
    ConnSplice s;
    s.d = ((const gofr_req_desc*)p.desc)[i];
    const uint32_t pq = (uint32_t)s.d.path_len + s.d.query_len;
    const uint32_t r0 = p.rec_off[i], r1 = p.rec_off[i + 1];
    if (r1 > r0) {
        s.data = p.rec + r0;
        s.data_len = r1 - r0;
    } else {
        s.data = p.arena + s.d.arena_off + conn_round4(pq);
        s.data_len = s.d.data_len;
    }
    s.size = conn_round4(pq) + conn_round4(s.data_len);
    return s;
}

// Request i's spliced form at p.out + at (a multiple of 4), its pads zero, and its descriptor rewritten to address it
GOFR_HD void conn_splice_emit(const ConnResultParams& p, uint32_t i, const ConnSplice& s, uint32_t at, uint32_t* stage_col) {
    const uint32_t pq = (uint32_t)s.d.path_len + s.d.query_len;
    Writer w;
    w.init(p.out + at, stage_col);
    w.copy<false>(p.arena + s.d.arena_off, pq);
    if (pq & 3u) {
        w.reserve(1);
        w.put(0u, 4u - (pq & 3u));
    }
    w.copy<false>(s.data, s.data_len);
    if (s.data_len & 3u) {
        w.reserve(1);
        w.put(0u, 4u - (s.data_len & 3u));
    }
    w.finish();
    gofr_req_desc d = s.d;
    d.arena_off = at;
    d.data_len = s.data_len;
    ((gofr_req_desc*)p.desc)[i] = d;
}

}  // namespace gofr
