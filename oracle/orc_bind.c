/*
 * orc_bind.c — TEST INFRASTRUCTURE ONLY (see gofr_oracle.h).
 *
 * Restatement of Request.Bind (pkg/gofr/http/request.go:40-47): io.ReadAll + json.Unmarshal(body, &i) where i holds
 * a *struct.  The arithmetic is Go 1.21 encoding/json, which is not in the reference checkout (stdlib):
 *   - checkValid: the byte-at-a-time scanner state machine and its SyntaxError texts        → scan_*()
 *   - decodeState.object/array/literalStore into a struct of string/int/bool fields          → dec_*()
 *   - UnmarshalTypeError texts with errorContext (Struct.Field path)                         → type_error()
 * Pins from the reference's own tests: pkg/gofr/http/request_test.go:17-30 ({"a": "b", "b": 5}) and
 * pkg/gofr/context_test.go:23-49 ({"ID":1,"Name":"Bob"}).
 */
#include "orc_internal.h"

#include <math.h>
#include <stdio.h>

/* ------------------------------------------------------------------------------------------------------------ */
/* scanner (validity pass)                                                                                      */
/* ------------------------------------------------------------------------------------------------------------ */

enum { PS_OBJECT_KEY, PS_OBJECT_VALUE, PS_ARRAY_VALUE };
enum {
    ST_BEGIN_VALUE_OR_EMPTY, ST_BEGIN_VALUE, ST_BEGIN_STRING_OR_EMPTY, ST_BEGIN_STRING, ST_END_VALUE, ST_END_TOP,
    ST_IN_STRING, ST_IN_STRING_ESC, ST_ESC_U, ST_ESC_U1, ST_ESC_U12, ST_ESC_U123, ST_NEG, ST_1, ST_0, ST_DOT, ST_DOT0,
    ST_E, ST_ESIGN, ST_E0, ST_T, ST_TR, ST_TRU, ST_F, ST_FA, ST_FAL, ST_FALS, ST_N, ST_NU, ST_NUL, ST_ERROR
};

typedef struct {
    int step;
    int end_top;
    uint8_t* ps;
    int nps, cap_ps;
    int has_err;
    obuf* err;
} scanner;

static int is_space(uint8_t c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n'; }

/* strconv.IsPrint restricted to U+0000..U+00FF */
static int latin1_is_print(unsigned c) {
    if (c < 0x20 || c == 0x7F) return 0;
    if (c < 0x7F) return 1;
    if (c < 0xA1) return 0; /* C1 controls and U+00A0 */
    return c != 0xAD;       /* soft hyphen */
}

/* json.quoteChar */
static void quote_char(obuf* b, uint8_t c) {
    if (c == '\'') { ob_puts(b, "'\\''"); return; }
    if (c == '"') { ob_puts(b, "'\"'"); return; }
    ob_putc(b, '\'');
    /* strconv.Quote(string(rune(c))) without the outer quotes */
    char tmp[8];
    if (c == '\\') ob_puts(b, "\\\\");
    else if (latin1_is_print(c)) {
        if (c < 0x80) ob_putc(b, c);
        else { ob_putc(b, (uint8_t)(0xC0 | (c >> 6))); ob_putc(b, (uint8_t)(0x80 | (c & 0x3F))); }
    } else {
        switch (c) {
            case '\a': ob_puts(b, "\\a"); break;
            case '\b': ob_puts(b, "\\b"); break;
            case '\f': ob_puts(b, "\\f"); break;
            case '\n': ob_puts(b, "\\n"); break;
            case '\r': ob_puts(b, "\\r"); break;
            case '\t': ob_puts(b, "\\t"); break;
            case '\v': ob_puts(b, "\\v"); break;
            default:
                if (c < 0x80) snprintf(tmp, sizeof tmp, "\\x%02x", c);
                else snprintf(tmp, sizeof tmp, "\\u%04x", c);
                ob_puts(b, tmp);
        }
    }
    ob_putc(b, '\'');
}

static int scan_error(scanner* s, uint8_t c, const char* context) {
    s->step = ST_ERROR;
    if (!s->has_err) {
        s->has_err = 1;
        ob_puts(s->err, "invalid character ");
        quote_char(s->err, c);
        ob_putc(s->err, ' ');
        ob_puts(s->err, context);
    }
    return -1;
}

static int push_ps(scanner* s, uint8_t c, int st) {
    if (s->nps == s->cap_ps) { s->cap_ps = s->cap_ps ? s->cap_ps * 2 : 32; s->ps = (uint8_t*)realloc(s->ps, (size_t)s->cap_ps); }
    s->ps[s->nps++] = (uint8_t)st;
    if (s->nps <= 10000) return 0;
    (void)c;
    s->step = ST_ERROR;
    if (!s->has_err) { s->has_err = 1; ob_puts(s->err, "exceeded max depth"); }
    return -1;
}

static void pop_ps(scanner* s) {
    s->nps--;
    if (s->nps == 0) { s->step = ST_END_TOP; s->end_top = 1; }
    else s->step = ST_END_VALUE;
}

static int scan_step(scanner* s, uint8_t c);

static int st_end_value(scanner* s, uint8_t c) {
    if (s->nps == 0) { s->step = ST_END_TOP; s->end_top = 1; return scan_step(s, c); }
    if (is_space(c)) { s->step = ST_END_VALUE; return 0; }
    switch (s->ps[s->nps - 1]) {
        case PS_OBJECT_KEY:
            if (c == ':') { s->ps[s->nps - 1] = PS_OBJECT_VALUE; s->step = ST_BEGIN_VALUE; return 0; }
            return scan_error(s, c, "after object key");
        case PS_OBJECT_VALUE:
            if (c == ',') { s->ps[s->nps - 1] = PS_OBJECT_KEY; s->step = ST_BEGIN_STRING; return 0; }
            if (c == '}') { pop_ps(s); return 0; }
            return scan_error(s, c, "after object key:value pair");
        default:
            if (c == ',') { s->step = ST_BEGIN_VALUE; return 0; }
            if (c == ']') { pop_ps(s); return 0; }
            return scan_error(s, c, "after array element");
    }
}

static int st_begin_value(scanner* s, uint8_t c) {
    if (is_space(c)) return 0;
    switch (c) {
        case '{': s->step = ST_BEGIN_STRING_OR_EMPTY; return push_ps(s, c, PS_OBJECT_KEY);
        case '[': s->step = ST_BEGIN_VALUE_OR_EMPTY; return push_ps(s, c, PS_ARRAY_VALUE);
        case '"': s->step = ST_IN_STRING; return 0;
        case '-': s->step = ST_NEG; return 0;
        case '0': s->step = ST_0; return 0;
        case 't': s->step = ST_T; return 0;
        case 'f': s->step = ST_F; return 0;
        case 'n': s->step = ST_N; return 0;
    }
    if (c >= '1' && c <= '9') { s->step = ST_1; return 0; }
    return scan_error(s, c, "looking for beginning of value");
}

static int is_hex(uint8_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'); }

static int lit_step(scanner* s, uint8_t c, uint8_t want, int next, const char* ctx) {
    if (c == want) { s->step = next; return 0; }
    return scan_error(s, c, ctx);
}

static int scan_step(scanner* s, uint8_t c) {
    switch (s->step) {
        case ST_BEGIN_VALUE_OR_EMPTY:
            if (is_space(c)) return 0;
            if (c == ']') return st_end_value(s, c);
            return st_begin_value(s, c);
        case ST_BEGIN_VALUE: return st_begin_value(s, c);
        case ST_BEGIN_STRING_OR_EMPTY:
            if (is_space(c)) return 0;
            if (c == '}') { s->ps[s->nps - 1] = PS_OBJECT_VALUE; return st_end_value(s, c); }
            /* fallthrough */
        case ST_BEGIN_STRING:
            if (is_space(c)) return 0;
            if (c == '"') { s->step = ST_IN_STRING; return 0; }
            return scan_error(s, c, "looking for beginning of object key string");
        case ST_END_VALUE: return st_end_value(s, c);
        case ST_END_TOP:
            if (!is_space(c)) return scan_error(s, c, "after top-level value");
            return 0;
        case ST_IN_STRING:
            if (c == '"') { s->step = ST_END_VALUE; return 0; }
            if (c == '\\') { s->step = ST_IN_STRING_ESC; return 0; }
            if (c < 0x20) return scan_error(s, c, "in string literal");
            return 0;
        case ST_IN_STRING_ESC:
            switch (c) {
                case 'b': case 'f': case 'n': case 'r': case 't': case '\\': case '/': case '"': s->step = ST_IN_STRING; return 0;
                case 'u': s->step = ST_ESC_U; return 0;
            }
            return scan_error(s, c, "in string escape code");
        case ST_ESC_U: case ST_ESC_U1: case ST_ESC_U12:
            if (is_hex(c)) { s->step++; return 0; }
            return scan_error(s, c, "in \\u hexadecimal character escape");
        case ST_ESC_U123:
            if (is_hex(c)) { s->step = ST_IN_STRING; return 0; }
            return scan_error(s, c, "in \\u hexadecimal character escape");
        case ST_NEG:
            if (c == '0') { s->step = ST_0; return 0; }
            if (c >= '1' && c <= '9') { s->step = ST_1; return 0; }
            return scan_error(s, c, "in numeric literal");
        case ST_1:
            if (c >= '0' && c <= '9') return 0;
            /* fallthrough */
        case ST_0:
            if (c == '.') { s->step = ST_DOT; return 0; }
            if (c == 'e' || c == 'E') { s->step = ST_E; return 0; }
            return st_end_value(s, c);
        case ST_DOT:
            if (c >= '0' && c <= '9') { s->step = ST_DOT0; return 0; }
            return scan_error(s, c, "after decimal point in numeric literal");
        case ST_DOT0:
            if (c >= '0' && c <= '9') return 0;
            if (c == 'e' || c == 'E') { s->step = ST_E; return 0; }
            return st_end_value(s, c);
        case ST_E:
            if (c == '+' || c == '-') { s->step = ST_ESIGN; return 0; }
            /* fallthrough */
        case ST_ESIGN:
            if (c >= '0' && c <= '9') { s->step = ST_E0; return 0; }
            return scan_error(s, c, "in exponent of numeric literal");
        case ST_E0:
            if (c >= '0' && c <= '9') return 0;
            return st_end_value(s, c);
        case ST_T: return lit_step(s, c, 'r', ST_TR, "in literal true (expecting 'r')");
        case ST_TR: return lit_step(s, c, 'u', ST_TRU, "in literal true (expecting 'u')");
        case ST_TRU: return lit_step(s, c, 'e', ST_END_VALUE, "in literal true (expecting 'e')");
        case ST_F: return lit_step(s, c, 'a', ST_FA, "in literal false (expecting 'a')");
        case ST_FA: return lit_step(s, c, 'l', ST_FAL, "in literal false (expecting 'l')");
        case ST_FAL: return lit_step(s, c, 's', ST_FALS, "in literal false (expecting 's')");
        case ST_FALS: return lit_step(s, c, 'e', ST_END_VALUE, "in literal false (expecting 'e')");
        case ST_N: return lit_step(s, c, 'u', ST_NU, "in literal null (expecting 'u')");
        case ST_NU: return lit_step(s, c, 'l', ST_NUL, "in literal null (expecting 'l')");
        case ST_NUL: return lit_step(s, c, 'l', ST_END_VALUE, "in literal null (expecting 'l')");
        default: return -1;
    }
}

/* json.checkValid: 0 ok, 1 error (message appended to err) */
static int check_valid(const uint8_t* data, size_t n, obuf* err) {
    scanner s;
    memset(&s, 0, sizeof s);
    s.step = ST_BEGIN_VALUE;
    s.err = err;
    int rc = 0;
    for (size_t i = 0; i < n; i++)
        if (scan_step(&s, data[i]) < 0) { rc = 1; break; }
    if (!rc) { /* scanner.eof() */
        if (!s.end_top) {
            scan_step(&s, ' ');
            if (s.has_err) rc = 1;
            else if (!s.end_top) { ob_puts(err, "unexpected end of JSON input"); rc = 1; }
        }
    }
    free(s.ps);
    return rc;
}

/* ------------------------------------------------------------------------------------------------------------ */
/* decode pass (input is known valid)                                                                           */
/* ------------------------------------------------------------------------------------------------------------ */

typedef struct {
    const uint8_t* p;
    size_t n, i;
    const orc_schema* sc;
    orc_value* vals;
    obuf* err;
    int saved;
} dec;

static void skip_ws(dec* d) { while (d->i < d->n && is_space(d->p[d->i])) d->i++; }

/* skip one value; returns [start,end) of it */
static void skip_value(dec* d, size_t* start, size_t* end) {
    skip_ws(d);
    *start = d->i;
    uint8_t c = d->p[d->i];
    if (c == '"') {
        d->i++;
        while (d->p[d->i] != '"') { if (d->p[d->i] == '\\') d->i++; d->i++; }
        d->i++;
    } else if (c == '{' || c == '[') {
        int depth = 0;
        for (;;) {
            uint8_t x = d->p[d->i];
            if (x == '"') { size_t a, b; skip_value(d, &a, &b); continue; }
            if (x == '{' || x == '[') depth++;
            if (x == '}' || x == ']') { depth--; if (depth == 0) { d->i++; break; } }
            d->i++;
        }
    } else {
        while (d->i < d->n) {
            uint8_t x = d->p[d->i];
            if (x == ',' || x == '}' || x == ']' || is_space(x)) break;
            d->i++;
        }
    }
    *end = d->i;
}

static int hex4(const uint8_t* s) {
    int v = 0;
    for (int i = 0; i < 4; i++) {
        uint8_t c = s[i];
        int h = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : c - 'A' + 10;
        v = v << 4 | h;
    }
    return v;
}

static void put_rune(obuf* b, uint32_t r) {
    if (r < 0x80) ob_putc(b, (uint8_t)r);
    else if (r < 0x800) { ob_putc(b, (uint8_t)(0xC0 | r >> 6)); ob_putc(b, (uint8_t)(0x80 | (r & 0x3F))); }
    else if (r < 0x10000) { ob_putc(b, (uint8_t)(0xE0 | r >> 12)); ob_putc(b, (uint8_t)(0x80 | ((r >> 6) & 0x3F))); ob_putc(b, (uint8_t)(0x80 | (r & 0x3F))); }
    else { ob_putc(b, (uint8_t)(0xF0 | r >> 18)); ob_putc(b, (uint8_t)(0x80 | ((r >> 12) & 0x3F))); ob_putc(b, (uint8_t)(0x80 | ((r >> 6) & 0x3F))); ob_putc(b, (uint8_t)(0x80 | (r & 0x3F))); }
}

/* utf8.DecodeRune on a byte range (same acceptance rules as the encoder's) */
static int dec_rune(const uint8_t* s, size_t n, uint32_t* r) {
    uint8_t b0 = s[0];
    if (b0 < 0x80) { *r = b0; return 1; }
    if (b0 < 0xC2 || b0 > 0xF4) { *r = 0xFFFD; return 1; }
    int need = b0 < 0xE0 ? 1 : b0 < 0xF0 ? 2 : 3;
    if (n < (size_t)need + 1) { *r = 0xFFFD; return 1; }
    uint8_t lo = 0x80, hi = 0xBF;
    if (b0 == 0xE0) lo = 0xA0;
    if (b0 == 0xED) hi = 0x9F;
    if (b0 == 0xF0) lo = 0x90;
    if (b0 == 0xF4) hi = 0x8F;
    if (s[1] < lo || s[1] > hi) { *r = 0xFFFD; return 1; }
    uint32_t v = need == 1 ? (b0 & 0x1F) : need == 2 ? (b0 & 0x0F) : (b0 & 0x07);
    v = v << 6 | (s[1] & 0x3F);
    for (int k = 2; k <= need; k++) {
        if ((s[k] & 0xC0) != 0x80) { *r = 0xFFFD; return 1; }
        v = v << 6 | (s[k] & 0x3F);
    }
    *r = v;
    return need + 1;
}

/* json.unquoteBytes on the quoted literal [s, s+n) including both quotes */
static void unquote(const uint8_t* s, size_t n, obuf* out) {
    size_t r = 1, e = n - 1;
    while (r < e) {
        uint8_t c = s[r];
        if (c == '\\') {
            r++;
            switch (s[r]) {
                case '"': case '\\': case '/': case '\'': ob_putc(out, s[r]); r++; break;
                case 'b': ob_putc(out, '\b'); r++; break;
                case 'f': ob_putc(out, '\f'); r++; break;
                case 'n': ob_putc(out, '\n'); r++; break;
                case 'r': ob_putc(out, '\r'); r++; break;
                case 't': ob_putc(out, '\t'); r++; break;
                case 'u': {
                    uint32_t rr = (uint32_t)hex4(s + r + 1);
                    r += 5;
                    if (rr >= 0xD800 && rr < 0xE000) { /* utf16.IsSurrogate */
                        if (r + 6 <= e && s[r] == '\\' && s[r + 1] == 'u') {
                            uint32_t rr1 = (uint32_t)hex4(s + r + 2);
                            if (rr < 0xDC00 && rr1 >= 0xDC00 && rr1 < 0xE000) { /* valid pair */
                                put_rune(out, ((rr - 0xD800) << 10 | (rr1 - 0xDC00)) + 0x10000);
                                r += 6;
                                break;
                            }
                        }
                        rr = 0xFFFD;
                    }
                    put_rune(out, rr);
                    break;
                }
            }
        } else if (c < 0x80) {
            ob_putc(out, c);
            r++;
        } else {
            uint32_t rr;
            int sz = dec_rune(s + r, e - r, &rr);
            put_rune(out, rr);
            r += (size_t)sz;
        }
    }
}

/* d.saveError(&UnmarshalTypeError{...}) with errorContext: first error wins */
static void type_error(dec* d, const char* value, size_t value_extra_n, const uint8_t* value_extra, const orc_field* f) {
    if (d->saved) return;
    d->saved = 1;
    ob_puts(d->err, "json: cannot unmarshal ");
    ob_puts(d->err, value);
    if (value_extra) ob_put(d->err, value_extra, value_extra_n);
    if (f) {
        /* Struct = reflect.Type.Name() (text after the last '.'), Field = JSON key name of the field */
        const char* name = strrchr(d->sc->go_type, '.');
        name = name ? name + 1 : d->sc->go_type;
        ob_puts(d->err, " into Go struct field ");
        ob_puts(d->err, name);
        ob_putc(d->err, '.');
        ob_puts(d->err, f->json_name);
        ob_puts(d->err, " of type ");
        ob_puts(d->err, orc_go_kind_name(f->kind));
    } else {
        ob_puts(d->err, " into Go value of type ");
        ob_puts(d->err, d->sc->go_type);
    }
}

/* strconv.ParseInt(s, 10, 64) on a valid JSON number literal; 0 ok */
static int parse_int64(const uint8_t* s, size_t n, int64_t* out) {
    size_t i = 0;
    int neg = 0;
    if (n && s[0] == '-') { neg = 1; i = 1; }
    if (i >= n) return -1;
    uint64_t v = 0;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return -1; /* '.', 'e', 'E' → syntax error in ParseInt */
        uint64_t d = (uint64_t)(s[i] - '0');
        if (v > (UINT64_MAX - d) / 10) return -1;
        v = v * 10 + d;
    }
    if (neg) { if (v > (uint64_t)1 << 63) return -1; *out = (int64_t)(0 - v); }
    else { if (v > (uint64_t)INT64_MAX) return -1; *out = (int64_t)v; }
    return 0;
}

/* simple-fold equality used for the case-insensitive key fallback: ASCII letters plus the two non-ASCII runes that
 * fold into ASCII (U+212A KELVIN SIGN ~ k, U+017F LATIN SMALL LETTER LONG S ~ s).  Other non-ASCII folding (e.g.
 * É ~ é) is not restated; DESIGN.md lists it as a limitation. */
static int fold_next(const uint8_t* s, size_t n, size_t* i, uint32_t* r) {
    uint32_t c;
    int sz = dec_rune(s + *i, n - *i, &c);
    *i += (size_t)sz;
    if (c >= 'A' && c <= 'Z') c += 32;
    else if (c == 0x212A) c = 'k';
    else if (c == 0x017F) c = 's';
    *r = c;
    return 1;
}
static int equal_fold(const uint8_t* a, size_t an, const uint8_t* b, size_t bn) {
    size_t i = 0, j = 0;
    while (i < an && j < bn) {
        uint32_t x, y;
        fold_next(a, an, &i, &x);
        fold_next(b, bn, &j, &y);
        if (x != y) return 0;
    }
    return i == an && j == bn;
}

static void store_value(dec* d, const orc_field* f, orc_value* v) {
    size_t a, b;
    skip_ws(d);
    uint8_t c = d->p[d->i];
    skip_value(d, &a, &b);
    const uint8_t* lit = d->p + a;
    size_t ln = b - a;
    if (c == '{') { type_error(d, "object", 0, NULL, f); return; }
    if (c == '[') { type_error(d, "array", 0, NULL, f); return; }
    if (c == 'n') return; /* null into string/int/bool: no-op */
    if (c == 't' || c == 'f') {
        if (f->kind == F_BOOL) v->i = (c == 't');
        else type_error(d, "bool", 0, NULL, f);
        return;
    }
    if (c == '"') {
        if (f->kind != F_STRING) { type_error(d, "string", 0, NULL, f); return; }
        obuf s;
        ob_init(&s);
        unquote(lit, ln, &s);
        free(v->owned);
        v->owned = s.p ? s.p : (uint8_t*)malloc(1);
        v->s = v->owned;
        v->sn = (int)s.n;
        return;
    }
    /* number */
    if (f->kind == F_STRING || f->kind == F_BOOL) { type_error(d, "number", 0, NULL, f); return; }
    if (f->kind == F_FLOAT64) {
        /* literalStore, reflect.Float64: strconv.ParseFloat(item, 64); err (only ErrRange is possible on a literal the
         * scanner accepted, and only overflow raises it: underflow yields 0, nil) or OverflowFloat → UnmarshalTypeError
         * "number <literal>".  ParseFloat rounds correctly (to nearest, ties to even) — so does glibc's strtod. */
        char tmp[64], *z = ln < sizeof tmp ? tmp : (char*)malloc(ln + 1);
        memcpy(z, lit, ln);
        z[ln] = 0;
        double x = strtod(z, NULL);
        if (z != tmp) free(z);
        if (isinf(x)) { type_error(d, "number ", ln, lit, f); return; }
        memcpy(&v->i, &x, 8); /* the value's bits */
        return;
    }
    int64_t x;
    int bad = parse_int64(lit, ln, &x) != 0;
    if (!bad && f->kind == F_INT32 && (x < INT32_MIN || x > INT32_MAX)) bad = 1; /* v.OverflowInt */
    if (bad) { type_error(d, "number ", ln, lit, f); return; }
    v->i = x;
}

static void dec_object(dec* d) {
    d->i++; /* '{' */
    skip_ws(d);
    if (d->p[d->i] == '}') { d->i++; return; }
    obuf key;
    ob_init(&key);
    for (;;) {
        size_t a, b;
        skip_value(d, &a, &b); /* key string */
        key.n = 0;
        unquote(d->p + a, b - a, &key);
        skip_ws(d);
        d->i++; /* ':' */
        /* exact name first, then case-insensitive fold, both in field declaration order */
        int fi = -1;
        for (int k = 0; k < d->sc->n_fields && fi < 0; k++) {
            const char* nm = d->sc->f[k].json_name;
            if (strlen(nm) == key.n && memcmp(nm, key.p ? key.p : (uint8_t*)"", key.n) == 0) fi = k;
        }
        for (int k = 0; k < d->sc->n_fields && fi < 0; k++) {
            const char* nm = d->sc->f[k].json_name;
            if (equal_fold((const uint8_t*)nm, strlen(nm), key.p, key.n)) fi = k;
        }
        if (fi >= 0) store_value(d, &d->sc->f[fi], &d->vals[fi]);
        else { size_t x, y; skip_value(d, &x, &y); }
        skip_ws(d);
        uint8_t c = d->p[d->i++];
        if (c == '}') break;
        /* ',' */
    }
    ob_free(&key);
}

int orc_unmarshal_struct(const orc_schema* sc, const uint8_t* body, size_t n, orc_value* vals, obuf* err) {
    for (int i = 0; i < sc->n_fields; i++) memset(&vals[i], 0, sizeof vals[i]);
    if (check_valid(body, n, err) != 0) return 1;
    dec d = {body, n, 0, sc, vals, err, 0};
    skip_ws(&d);
    uint8_t c = body[d.i];
    if (c == '{') dec_object(&d);
    else if (c == '[') type_error(&d, "array", 0, NULL, NULL);
    else if (c == '"') type_error(&d, "string", 0, NULL, NULL);
    else if (c == 't' || c == 'f') type_error(&d, "bool", 0, NULL, NULL);
    else if (c == 'n') { /* null: sets the local interface to nil; the caller's struct is untouched */ }
    else type_error(&d, "number", 0, NULL, NULL);
    return d.saved;
}
