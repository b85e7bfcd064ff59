// conn_log_device.cuh — per-connection logic of gofr_conn_batch_submit_log's gather step (conn_log_kernel.cu), compiled for
// the device and, through tests/emu/emu_conn_log.cpp, for the host.
//
// After the serve kernel, request k of a chunk (its compacted index) has its meta word, its trace id and, through its record,
// the request head's spans.  The gather turns every logged request into the input gofr_requestlog_device takes: a
// gofr_log_desc, the trace id, and the five strings method | User-Agent | first X-Forwarded-For value | remote address |
// request target back to back in a log arena.
//
// Placement without a second scan: the strings of request k (record r) start at (rec_off[r] - alo) + k * R, R the chunk's
// longest remote string.  The four head strings are disjoint spans of the record and the remote string is at most R bytes,
// so they end before (rec_off[r + 1] - alo) + (k + 1) * R, where the next request's strings start.
#pragma once
#include <stdint.h>
#include <string.h>

#include "conn_device.cuh"
#include "engine_internal.h"

namespace gofr {

GOFR_CONN_HD uint32_t conn_span_len(unsigned long long s) { return (uint32_t)(s >> 32); }

// Does request k (record r, spans sp) get a line on the device?  Logging wraps matched routes only (mux's 301 / 404 / 405
// carry GOFR_ROUTE_NONE); a hole (status 0) is logged by the host once its closure has run; and so is a request whose
// method, User-Agent, X-Forwarded-For value or target is longer than a gofr_log_desc length field holds (65535 bytes: the
// request-head subset limits where header lines start, not how long the last one is).
GOFR_CONN_HD bool conn_logged(uint32_t meta, const unsigned long long* sp) {
    return (meta >> 16) != GOFR_ROUTE_NONE && (meta & 0xFFFFu) != 0 && conn_span_len(sp[GOFR_HTTP_SPAN_METHOD]) <= 0xFFFFu &&
           conn_span_len(sp[GOFR_HTTP_SPAN_USER_AGENT]) <= 0xFFFFu && conn_span_len(sp[GOFR_HTTP_SPAN_XFF]) <= 0xFFFFu &&
           conn_span_len(sp[GOFR_HTTP_SPAN_TARGET]) <= 0xFFFFu;
}

// Logged requests among a connection's `count` requests, the first of which is request k0 and record rec0 of the chunk
GOFR_CONN_HD uint32_t conn_log_count(const ConnLogParams& p, uint32_t rec0, uint32_t k0, uint32_t count) {
    uint32_t lines = 0;
    for (uint32_t j = 0; j < count; j++) lines += conn_logged(p.meta[k0 + j], p.spans + (size_t)(rec0 + j) * GOFR_HTTP_SPANS) ? 1u : 0u;
    return lines;
}

GOFR_CONN_HD uint32_t conn_span_copy(uint8_t* dst, const uint8_t* buf, unsigned long long s) {
    const uint32_t n = conn_span_len(s);
    memcpy(dst, buf + (uint32_t)s, n);
    return n;
}

// Writes the lines of connection c, whose `count` requests start at request k0 and record rec0 of the chunk and whose
// logged requests become lines m0, m0 + 1, ...
GOFR_CONN_HD void conn_log_put(const ConnLogParams& p, uint32_t c, uint32_t rec0, uint32_t k0, uint32_t count, uint32_t m0) {
    const uint32_t ro = p.remote_off[c], rl = p.remote_off[c + 1] - ro;
    const int64_t start = p.start_ns[c];
    gofr_log_desc* out = (gofr_log_desc*)p.out;
    uint32_t m = m0;
    for (uint32_t j = 0; j < count; j++) {
        const uint32_t k = k0 + j, r = rec0 + j, meta = p.meta[k];
        const unsigned long long* sp = p.spans + (size_t)r * GOFR_HTTP_SPANS;
        if (!conn_logged(meta, sp)) continue;
        const uint32_t at = (p.rec_off[r] - p.alo) + k * p.remote_max;
        uint8_t* a = p.arena + at;
        gofr_log_desc d;
        d.start_unix_ns = start;
        d.elapsed_ns = p.log_ns - start;
        d.log_unix_ns = p.log_ns;
        d.arena_off = at;
        d.method_len = (uint16_t)conn_span_copy(a, p.buf, sp[GOFR_HTTP_SPAN_METHOD]);
        a += d.method_len;
        d.ua_len = (uint16_t)conn_span_copy(a, p.buf, sp[GOFR_HTTP_SPAN_USER_AGENT]);
        a += d.ua_len;
        d.xff_len = (uint16_t)conn_span_copy(a, p.buf, sp[GOFR_HTTP_SPAN_XFF]);
        a += d.xff_len;
        memcpy(a, p.remote + ro, rl);
        d.remote_len = (uint16_t)rl;
        a += rl;
        d.uri_len = (uint16_t)conn_span_copy(a, p.buf, sp[GOFR_HTTP_SPAN_TARGET]);
        d.status = (uint16_t)(meta & 0xFFFFu);
        d.tz_offset_s = p.tz_offset_s;
        d.kind = GOFR_LOG_REQUEST;
        out[m] = d;
        memcpy(p.line_ids + (size_t)m * 16, p.ids + (size_t)k * 16, 16);
        p.line_req[m] = p.req0 + k;
        m++;
    }
}

}  // namespace gofr
