// http_frame_device.cuh — where one HTTP/1.1 request ends in a connection's received bytes, one thread per connection
// (gofr_http_frame_device).
//
// Stands where net/http's conn.serve loops readRequest over one bufio.Reader (reached from pkg/gofr/httpServer.go:29-33):
// a receive buffer holds zero, one or several requests, then nothing or the first part of the next one.  http_frame_next
// answers, for the bytes left in a connection, "a whole request of length L", "need more bytes" or "defer"; the record
// column built from its answers is the offset column http_parse (http_device.cuh) takes.  The head walk restates
// http_parse's grammar instead of sharing it (http_parse_kernel is on a measured path and keeps its code); the two are held
// together by the contract below, which tests/test_http_frame.py checks.
//
// The contract:
//   1. Cut => accepted.  Every record the framer cuts as a whole request, given alone to http_parse, is GOFR_HTTP_OK.
//      (http_parse checks the framing exactly — body length == Content-Length, the chunk stream ends at the last byte — so
//      an accepted record is exactly one request.)
//   2. Tail => deferred.  Whatever is left of a connection after its whole requests (the tail record), given alone to
//      http_parse, is GOFR_HTTP_DEFER: no prefix of it is a request of the subset, so the serve step never answers it.
//   Conversely a message http_parse accepts, followed by anything, is cut at its own length.
//
// MORE or DEFER for a tail: bytes are judged as they arrive, header lines when they are complete.  A byte the grammar does
// not allow where it stands (a wrong version, a control byte in a value, a ninth hex digit of a chunk size), and a complete
// header line the subset excludes (a second Host, Connection: close, a Content-Length that is not 1-9 digits, Expect, ...)
// make the tail DEFER at once, request unfinished or not.  MORE means the walk ran out of bytes with none of that seen.
// The framer stops a connection at the first request it does not accept: where the next one starts is not known.
// __host__ __device__ like http_device.cuh: tests/emu runs it on the CPU against the oracle.
#pragma once
#include "http_device.cuh"

namespace gofr {

constexpr uint32_t kFrameWhole = 0;  // http_frame_next: a whole request; else GOFR_HTTP_CONN_MORE / GOFR_HTTP_CONN_DEFER

// is m[0..n) the beginning (or all) of `lit`?
GOFR_HD bool http_starts(const uint8_t* m, uint32_t n, const char* lit, uint32_t ln) {
    if (n > ln) return false;
    for (uint32_t k = 0; k < n; k++)
        if (m[k] != (uint8_t)lit[k]) return false;
    return true;
}

// The bytes m[0..n) left in a connection, n > 0: kFrameWhole with the request's length in *len, or why there is none.
GOFR_HD_NOINLINE uint32_t http_frame_next(const uint8_t* m, uint32_t n, uint32_t* len) {
    const uint32_t MORE = GOFR_HTTP_CONN_MORE, DEFER = GOFR_HTTP_CONN_DEFER;
    // ---- request line ----
    uint32_t ml = 0;
    while (ml < n && ml < 8 && m[ml] != ' ') ml++;
    {
        const bool sp = ml < n && m[ml] == ' ';
        // with the space the method is whole: one of the seven; without it, the beginning of one and nothing behind it
        const uint32_t k = sp ? ml + 1 : ml;
        const bool known = http_starts(m, k, "GET ", 4) || http_starts(m, k, "HEAD ", 5) || http_starts(m, k, "POST ", 5) ||
                           http_starts(m, k, "PUT ", 4) || http_starts(m, k, "PATCH ", 6) || http_starts(m, k, "DELETE ", 7) ||
                           http_starts(m, k, "OPTIONS ", 8);
        if (!known) return DEFER;
        if (!sp) return MORE;  // eight bytes without a space begin no method: ml == n here
    }
    const uint32_t t0 = ml + 1;
    uint32_t t1 = t0, qmark = 0xFFFFFFFFu;
    while (t1 < n && m[t1] != ' ') {
        const uint32_t c = m[t1];
        if (c < 0x21 || c > 0x7E || c == '#') return DEFER;
        if (c == '?' && qmark == 0xFFFFFFFFu) qmark = t1;
        t1++;
    }
    if (t1 > t0 && (m[t0] != '/' || (t1 - t0 >= 2 && m[t0 + 1] == '/'))) return DEFER;
    if (t1 - t0 > 8192) return DEFER;
    {
        // percent escapes of the path part; only a path that has ended (at '?' or the space) can have one cut short
        const uint32_t path_end = qmark == 0xFFFFFFFFu ? t1 : qmark;
        const bool ended = qmark != 0xFFFFFFFFu || t1 < n;
        for (uint32_t k = t0; k < path_end; k++) {
            if (m[k] != '%') continue;
            if (k + 1 < path_end && http_hex(m[k + 1]) < 0) return DEFER;
            if (k + 2 < path_end ? http_hex(m[k + 2]) < 0 : ended) return DEFER;
        }
    }
    if (t1 == n) return MORE;
    if (t1 == t0) return DEFER;
    {
        const char v[] = " HTTP/1.1\r\n";
        for (uint32_t k = 0; k < 11; k++) {
            if (t1 + k == n) return MORE;
            if (m[t1 + k] != (uint8_t)v[k]) return DEFER;
        }
    }
    // ---- header lines ----
    uint32_t pos = t1 + 11, hosts = 0, cls = 0, chunked = 0;
    uint64_t content_length = 0;
    for (;;) {
        if (pos == n) return MORE;
        if (m[pos] == '\r') {
            if (pos + 1 == n) return MORE;
            if (m[pos + 1] != '\n') return DEFER;
            pos += 2;
            break;
        }
        if (pos > 16384) return DEFER;
        const uint32_t n0 = pos;
        while (pos < n && http_tchar(m[pos])) pos++;
        if (pos == n) return MORE;
        if (pos == n0 || m[pos] != ':') return DEFER;
        const uint32_t nl = pos - n0;
        pos++;
        while (pos < n && (m[pos] == ' ' || m[pos] == '\t')) pos++;
        const uint32_t v0 = pos;
        for (; pos < n; pos++) {
            const uint32_t c = m[pos];
            if (c >= 0x20 && c != 0x7F) continue;
            if (c == '\t') continue;
            if (c == '\r') break;
            return DEFER;
        }
        if (pos + 1 >= n) return MORE;
        if (m[pos + 1] != '\n') return DEFER;
        uint32_t v1 = pos;
        while (v1 > v0 && (m[v1 - 1] == ' ' || m[v1 - 1] == '\t')) v1--;
        pos += 2;
        // ---- the line is complete: what it means ----
        const uint8_t* nm = m + n0;
        if (http_name_is(nm, nl, "host", 4)) {
            if (++hosts > 1 || v1 == v0) return DEFER;
            for (uint32_t k = v0; k < v1; k++) {
                const uint32_t c = m[k];
                if (!(c - '0' < 10u || (c | 0x20u) - 'a' < 26u || c == '.' || c == ':' || c == '-' || c == '_' || c == '[' || c == ']')) return DEFER;
            }
        } else if (http_name_is(nm, nl, "content-length", 14)) {
            if (++cls > 1 || chunked || v1 == v0 || v1 - v0 > 9) return DEFER;
            for (uint32_t k = v0; k < v1; k++) {
                if ((uint32_t)m[k] - (uint32_t)'0' >= 10u) return DEFER;
                content_length = content_length * 10 + (m[k] - '0');
            }
        } else if (http_name_is(nm, nl, "connection", 10)) {
            if (!http_name_is(m + v0, v1 - v0, "keep-alive", 10)) return DEFER;
        } else if (http_name_is(nm, nl, "transfer-encoding", 17)) {
            if (chunked || cls || !http_name_is(m + v0, v1 - v0, "chunked", 7)) return DEFER;
            chunked = 1;
        } else if (http_name_is(nm, nl, "expect", 6) || http_name_is(nm, nl, "upgrade", 7) || http_name_is(nm, nl, "trailer", 7)) return DEFER;
    }
    if (hosts != 1) return DEFER;
    // ---- the body: nothing, Content-Length bytes, or the chunk stream up to and including `0 CRLF CRLF` ----
    if (!chunked) {
        if (content_length > (uint64_t)(n - pos)) return MORE;
        *len = pos + (uint32_t)content_length;
        return kFrameWhole;
    }
    uint32_t q = pos;
    for (;;) {
        uint32_t size = 0, nd = 0;
        while (q < n && nd < 9 && http_hex(m[q]) >= 0) { size = size << 4 | (uint32_t)http_hex(m[q]); q++; nd++; }
        if (nd > 8) return DEFER;
        if (q == n) return MORE;
        if (nd == 0 || m[q] != '\r') return DEFER;
        if (q + 1 == n) return MORE;
        if (m[q + 1] != '\n') return DEFER;
        q += 2;
        // `size` data bytes (none after the last chunk's size line), then CRLF
        const uint32_t left = n - q;
        if (size >= left) return MORE;
        if (m[q + size] != '\r') return DEFER;
        if (size + 1 == left) return MORE;
        if (m[q + size + 1] != '\n') return DEFER;
        q += size + 2;
        if (size == 0) break;
    }
    *len = q;
    return kFrameWhole;
}

// One connection's framing as the kernel keeps it between its two walks: the number of records (whole requests, plus the
// tail record when bytes are left over), the bytes the whole requests cover, the connection status, and where the first
// few records after the first one start; records beyond those are found again by walking from the last kept start.
constexpr int kFrameKept = 3;
struct HttpFrameConn {
    uint32_t count, consumed, status;
    uint32_t start[kFrameKept];  // start[k] = offset in the connection of record k + 1
};

// First walk: counts the records of the connection b[0..n).
GOFR_HD void http_frame_count(const uint8_t* b, uint32_t n, HttpFrameConn& c) {
    uint32_t at = 0, k = 0, st = GOFR_HTTP_CONN_DONE;
#pragma unroll
    for (int j = 0; j < kFrameKept; j++) c.start[j] = 0;
    while (at < n) {
        uint32_t len = 0;
        st = http_frame_next(b + at, n - at, &len);
        if (st != kFrameWhole) break;
        at += len;
        // a select per slot instead of c.start[k] = at: the array stays in registers
#pragma unroll
        for (int j = 0; j < kFrameKept; j++)
            if ((uint32_t)j == k) c.start[j] = at;
        k++;
    }
    c.count = k + (at < n ? 1u : 0u);
    c.consumed = at;
    c.status = st;
}

// Second walk: the starts of the connection's c.count records, as offsets into the whole buffer (the connection starts at
// `origin` there), to rec[0 .. c.count).
GOFR_HD void http_frame_put(const uint8_t* b, uint32_t n, const HttpFrameConn& c, uint32_t origin, uint32_t* rec) {
    if (c.count == 0) return;
    rec[0] = origin;
    uint32_t at = 0;
#pragma unroll
    for (int j = 0; j < kFrameKept; j++)
        if ((uint32_t)j + 1 < c.count) { at = c.start[j]; rec[j + 1] = origin + at; }
    for (uint32_t k = kFrameKept + 1; k < c.count; k++) {
        uint32_t len = 0;
        http_frame_next(b + at, n - at, &len);  // whole: the first walk went past it
        at += len;
        rec[k] = origin + at;
    }
}

}  // namespace gofr
