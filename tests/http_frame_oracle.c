/* http_frame_oracle.c — TEST INFRASTRUCTURE ONLY: the CPU oracle of gofr_http_frame_device (parity unpinned like the rest of
 * the oracle: no Go toolchain in this image).  Built into its own library by tests/http_frame_oracle.py; nothing in the
 * product links or loads it.  The request-head oracle it stands in front of is oracle/orc_http.c (orc_http_parse); the
 * character classes below are restated from the RFC, not shared with it. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int is_tchar(uint8_t c) { /* RFC 7230 token character */
    if ((c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z')) return 1;
    return c != 0 && strchr("!#$%&'*+-.^_`|~", c) != NULL;
}
static int hexv(uint8_t c) {
    if (c >= '0' && c <= '9') return c - '0';
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return c - 'A' + 10;
    return -1;
}
static int ieq(const uint8_t* p, size_t n, const char* lit) { /* a name or value against a lower-case literal */
    if (n != strlen(lit)) return 0;
    for (size_t k = 0; k < n; k++) {
        uint8_t c = p[k];
        if (c >= 'A' && c <= 'Z') c = (uint8_t)(c + 32);
        if (c != (uint8_t)lit[k]) return 0;
    }
    return 1;
}

/* ---- the connection reader in front of the request-head oracle -------------------------------------------------------
 * net/http's conn.serve calls readRequest again and again over one bufio.Reader; this restates where each request of the
 * subset ends in a connection's received bytes, and what is to be done with the bytes behind the last whole request.
 * Line-first like the request-head oracle (the device code walks the bytes once).  The rule for what is left over: bytes are judged as
 * they arrive, a header line's meaning when its CRLF is there.  FR_MORE: nothing wrong yet; FR_DEFER: already outside. */
enum { FR_WHOLE = 0, FR_MORE = 1, FR_DEFER = 2 };
enum { T_FULL, T_CR, T_NONE, T_BAD }; /* how a line ends: CRLF; CR as the last byte present; no CR yet; CR + another byte */

static const char* const k_methods[] = {"GET", "HEAD", "POST", "PUT", "PATCH", "DELETE", "OPTIONS"};

/* the request target; whole = the space behind it is there */
static int target_ok(const uint8_t* t, size_t n, int whole) {
    if (n > 8192 || (whole && n == 0)) return 0;
    if (n >= 1 && t[0] != '/') return 0;
    if (n >= 2 && t[1] == '/') return 0;
    const uint8_t* q = NULL;
    for (size_t k = 0; k < n; k++) {
        if (t[k] < 0x21 || t[k] > 0x7E || t[k] == '#') return 0;
        if (t[k] == '?' && !q) q = t + k;
    }
    size_t plen = q ? (size_t)(q - t) : n;
    int path_whole = whole || q != NULL;
    for (size_t k = 0; k < plen; k++) {
        if (t[k] != '%') continue;
        size_t have = plen - k - 1; /* bytes of the path behind the '%' */
        if (have >= 1 && hexv(t[k + 1]) < 0) return 0;
        if (have >= 2 && hexv(t[k + 2]) < 0) return 0;
        if (have < 2 && path_whole) return 0;
    }
    return 1;
}

static int request_line(const uint8_t* L, size_t n, int term) {
    const uint8_t* s1 = memchr(L, ' ', n);
    if (!s1) { /* only (part of) a method */
        if (term != T_NONE) return FR_DEFER;
        for (int k = 0; k < 7; k++)
            if (n <= strlen(k_methods[k]) && memcmp(L, k_methods[k], n) == 0) return FR_MORE;
        return FR_DEFER;
    }
    size_t mlen = (size_t)(s1 - L);
    int known = 0;
    for (int k = 0; k < 7; k++) known |= mlen == strlen(k_methods[k]) && memcmp(L, k_methods[k], mlen) == 0;
    if (!known) return FR_DEFER;
    const uint8_t* rest = s1 + 1;
    size_t restn = n - mlen - 1;
    const uint8_t* s2 = memchr(rest, ' ', restn);
    if (!s2) {
        if (!target_ok(rest, restn, term != T_NONE)) return FR_DEFER;
        return term == T_NONE ? FR_MORE : FR_DEFER; /* a line end where the version should follow */
    }
    if (!target_ok(rest, (size_t)(s2 - rest), 1)) return FR_DEFER;
    const uint8_t* proto = s2 + 1;
    size_t pn = restn - (size_t)(s2 - rest) - 1;
    if (term == T_NONE) return pn <= 8 && memcmp(proto, "HTTP/1.1", pn) == 0 ? FR_MORE : FR_DEFER;
    if (pn != 8 || memcmp(proto, "HTTP/1.1", 8) != 0) return FR_DEFER;
    return term == T_CR ? FR_MORE : FR_WHOLE;
}

typedef struct { int hosts, cls, te; uint64_t cl; } head_state;

static int header_line(const uint8_t* L, size_t n, int term, head_state* h) {
    size_t c = 0;
    while (c < n && is_tchar(L[c])) c++;
    if (c == n && term == T_NONE) return FR_MORE; /* still inside the name */
    if (c == 0 || c == n || L[c] != ':') return FR_DEFER;
    for (size_t k = c + 1; k < n; k++)
        if ((L[k] < 0x20 && L[k] != '\t') || L[k] == 0x7F) return FR_DEFER;
    if (term != T_FULL) return FR_MORE;
    size_t v0 = c + 1, v1 = n;
    while (v0 < v1 && (L[v0] == ' ' || L[v0] == '\t')) v0++;
    while (v1 > v0 && (L[v1 - 1] == ' ' || L[v1 - 1] == '\t')) v1--;
    const uint8_t* v = L + v0;
    size_t vn = v1 - v0;
    if (ieq(L, c, "host")) {
        if (++h->hosts > 1 || vn == 0) return FR_DEFER;
        for (size_t k = 0; k < vn; k++)
            if (!((v[k] >= '0' && v[k] <= '9') || (v[k] >= 'a' && v[k] <= 'z') || (v[k] >= 'A' && v[k] <= 'Z') || strchr(".:-_[]", v[k]))) return FR_DEFER;
    } else if (ieq(L, c, "content-length")) {
        if (++h->cls > 1 || h->te || vn == 0 || vn > 9) return FR_DEFER;
        for (size_t k = 0; k < vn; k++) {
            if (v[k] < '0' || v[k] > '9') return FR_DEFER;
            h->cl = h->cl * 10 + (uint64_t)(v[k] - '0');
        }
    } else if (ieq(L, c, "connection")) {
        if (!ieq(v, vn, "keep-alive")) return FR_DEFER;
    } else if (ieq(L, c, "transfer-encoding")) {
        if (++h->te > 1 || h->cls || !ieq(v, vn, "chunked")) return FR_DEFER;
    } else if (ieq(L, c, "expect") || ieq(L, c, "upgrade") || ieq(L, c, "trailer")) return FR_DEFER;
    return FR_WHOLE;
}

/* the bytes m[0..n) left in a connection: FR_WHOLE and the request's length, or FR_MORE / FR_DEFER */
static int frame_one(const uint8_t* m, size_t n, size_t* len) {
    head_state h = {0, 0, 0, 0};
    size_t pos = 0;
    for (int li = 0;; li++) {
        size_t e = pos;
        while (e < n && m[e] != '\r') e++;
        int term = e == n ? T_NONE : e + 1 == n ? T_CR : m[e + 1] == '\n' ? T_FULL : T_BAD;
        if (term == T_BAD) return FR_DEFER; /* the head has no place for a CR that is not followed by LF */
        int r;
        if (li == 0) r = request_line(m, e, term);
        else if (e == pos) { /* the blank line, or the beginning of one */
            if (term != T_FULL) return FR_MORE;
            pos = e + 2;
            break;
        } else if (pos > 16384) return FR_DEFER; /* a header line may not start beyond 16 KiB */
        else r = header_line(m + pos, e - pos, term, &h);
        if (r != FR_WHOLE) return r;
        pos = e + 2;
    }
    if (h.hosts != 1) return FR_DEFER;
    if (!h.te) {
        if (h.cl > (uint64_t)(n - pos)) return FR_MORE;
        *len = pos + (size_t)h.cl;
        return FR_WHOLE;
    }
    for (;;) { /* chunk = size line, data, CRLF; the zero-size chunk ends the request */
        size_t e = pos;
        while (e < n && m[e] != '\r') e++;
        uint64_t size = 0;
        for (size_t k = pos; k < e; k++) {
            if (hexv(m[k]) < 0 || k - pos >= 8) return FR_DEFER;
            size = size * 16 + (uint64_t)hexv(m[k]);
        }
        if (e == n) return FR_MORE;
        if (e == pos) return FR_DEFER;
        if (e + 1 == n) return FR_MORE;
        if (m[e + 1] != '\n') return FR_DEFER;
        pos = e + 2;
        uint64_t left = n - pos;
        if (left <= size) return FR_MORE;
        if (m[pos + size] != '\r') return FR_DEFER;
        if (left == size + 1) return FR_MORE;
        if (m[pos + size + 1] != '\n') return FR_DEFER;
        pos += (size_t)size + 2;
        if (size == 0) break;
    }
    *len = pos;
    return FR_WHOLE;
}

/* Outputs as gofr_http_frame_device documents them; returns 1 when rec_cap records do not hold the column (first is still
 * complete). */
int orc_http_frame(const uint8_t* buf, const uint32_t* buf_off, uint32_t n_conns, uint32_t* rec_off, uint32_t rec_cap,
                   uint32_t* first, uint32_t* consumed, uint32_t* status) {
    uint64_t total = 0;
    for (uint32_t c = 0; c < n_conns; c++) {
        const uint8_t* b = buf + buf_off[c];
        size_t n = buf_off[c + 1] - buf_off[c], at = 0;
        int st = 0; /* GOFR_HTTP_CONN_DONE */
        first[c] = (uint32_t)total;
        while (at < n) { /* one record per whole request, then one for whatever is left */
            size_t len = 0;
            if (total < rec_cap) rec_off[total] = buf_off[c] + (uint32_t)at;
            total++;
            st = frame_one(b + at, n - at, &len);
            if (st != FR_WHOLE) break;
            at += len;
        }
        consumed[c] = (uint32_t)at;
        status[c] = (uint32_t)st;
    }
    if (n_conns) {
        first[n_conns] = (uint32_t)total;
        if (total <= rec_cap) rec_off[total] = buf_off[n_conns];
    }
    return total > rec_cap;
}
