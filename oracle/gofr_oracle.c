/*
 * gofr_oracle.c — TEST INFRASTRUCTURE ONLY (see gofr_oracle.h: "parity unpinned" status and who may call this).
 *
 * Scalar C restatement of one GoFr HTTP request, in the order the reference executes it
 * (SURVEY.md §3.4; all file:line below are relative to the reference, JigarJoshi04/gofr @ 17218229):
 *
 *   mux.Router.ServeHTTP            (gorilla/mux v1.8.1 via pkg/gofr/http/router.go:14)   → serve_one()
 *     cleanPath → 301               (mux, before any middleware)                           → mux_clean_path()
 *     Router.Match / Route.Match    (registration order, pkg/gofr/http/router.go:30-33)    → mux_match()
 *   middleware.Tracer/Logging/CORS  (pkg/gofr/http/router.go:19-23, middleware/{tracer,logger,cors}.go) → in serve_one()
 *   handler.ServeHTTP               (pkg/gofr/handler.go:32-36)                            → run_handler()
 *   Request.Param / Bind            (pkg/gofr/http/request.go:28-47)                       → query_get(), orc_bind.c
 *   Responder.Respond               (pkg/gofr/http/responder.go:19-57)                     → respond()
 *   net/http response framing       (Go 1.21 net/http server.go chunkWriter.writeHeader)   → rw_finish()
 *
 * The ResponseWriter is modelled literally (live header map, snapshot at WriteHeader) so that the reference's
 * WriteHeader-before-Header().Set order (responder.go:21 vs :39) produces what it produces on a real socket.
 */
#define _GNU_SOURCE
#include "gofr_oracle.h"
#include "orc_internal.h"

#include <pthread.h>
#include <stdio.h>
#include <time.h>

/* ------------------------------------------------------------------------------------------------------------ */
/* table                                                                                                        */
/* ------------------------------------------------------------------------------------------------------------ */

enum { M_ANY = 255 };
enum { FRAME_WIRE = 0, FRAME_INTENDED = 1, FRAME_BODY = 2 };
enum {
    H_HOST = 0, H_STATIC_STRING = 1, H_STATIC_ERROR = 2, H_NIL = 3, H_PARAM_FORMAT = 4, H_ROW = 5, H_BIND_ECHO = 6,
    H_HEALTH = 7, H_MISSING_FILE = 8, H_FILE = 9, H_PANIC = 10, H_PATHPARAM_FORMAT = 11, H_RESULT = 12
};

/* one piece of a mux path template: a literal followed (optionally) by a variable */
typedef struct {
    uint8_t* lit;
    int lit_len;
    int has_var;
    char* name;      /* variable name (mux.Vars key) */
    /* the variable's regexp as a concatenation of quantified character classes (mux default [^/]+ = one atom) */
    int n_atoms;
    struct tpl_atom {
        uint8_t cls[32]; /* 256-bit membership */
        int min_rep;     /* {min,max}; max < 0 = unbounded */
        int max_rep;
    } atoms[12];
} tpl_piece;

typedef struct {
    int method;  /* 0..15, or M_ANY */
    int prefix;  /* PathPrefix: no trailing '$' */
    int dead;    /* route.err != nil: never matches (e.g. pattern without leading slash) */
    int n_pieces;
    tpl_piece* pieces;
    int hkind, schema_id;
    uint8_t* s[4];
    int sl[4];
    uint8_t* blob;
    int blob_len;
} orc_route;

struct orc_table {
    int frame_mode;
    int n_routes, cap_routes;
    orc_route* routes;
    int n_schemas;
    orc_schema* schemas;
};

static char* dup_str(const char* s) {
    if (!s) s = "";
    size_t n = strlen(s);
    char* r = (char*)malloc(n + 1);
    memcpy(r, s, n + 1);
    return r;
}
static uint8_t* dup_bytes(const void* s, int n) {
    uint8_t* r = (uint8_t*)malloc((size_t)(n > 0 ? n : 1));
    if (n > 0) memcpy(r, s, (size_t)n);
    return r;
}

orc_table* orc_table_new(int frame_mode) {
    orc_table* t = (orc_table*)calloc(1, sizeof *t);
    t->frame_mode = frame_mode;
    return t;
}

void orc_table_free(orc_table* t) {
    if (!t) return;
    for (int i = 0; i < t->n_routes; i++) {
        orc_route* r = &t->routes[i];
        for (int k = 0; k < r->n_pieces; k++) { free(r->pieces[k].lit); free(r->pieces[k].name); }
        free(r->pieces);
        for (int k = 0; k < 4; k++) free(r->s[k]);
        free(r->blob);
    }
    free(t->routes);
    for (int i = 0; i < t->n_schemas; i++) {
        for (int k = 0; k < t->schemas[i].n_fields; k++) {
            free(t->schemas[i].f[k].go_name);
            free(t->schemas[i].f[k].json_name);
        }
        free(t->schemas[i].f);
        free(t->schemas[i].go_type);
    }
    free(t->schemas);
    free(t);
}

int orc_add_schema(orc_table* t, int schema_id, const char* go_type_name, int n_fields, const char* const* go_names,
                   const char* const* json_names, const int* kinds, const int* omitempty) {
    t->schemas = (orc_schema*)realloc(t->schemas, sizeof(orc_schema) * (size_t)(t->n_schemas + 1));
    orc_schema* s = &t->schemas[t->n_schemas++];
    s->id = schema_id;
    s->go_type = dup_str(go_type_name);
    s->n_fields = n_fields;
    s->f = (orc_field*)calloc((size_t)n_fields, sizeof(orc_field));
    for (int i = 0; i < n_fields; i++) {
        s->f[i].go_name = dup_str(go_names[i]);
        s->f[i].json_name = dup_str(json_names && json_names[i] && json_names[i][0] ? json_names[i] : go_names[i]);
        s->f[i].kind = kinds[i];
        s->f[i].omitempty = omitempty ? omitempty[i] : 0;
    }
    return 0;
}

/* the wider data model (include/gofr_b200.h gofr_field_desc: container, flags, elem_schema) for the last schema added */
int orc_schema_extend(orc_table* t, const int* containers, const int* flags, const int* elem_schemas) {
    if (!t->n_schemas) return -1;
    orc_schema* s = &t->schemas[t->n_schemas - 1];
    for (int i = 0; i < s->n_fields; i++) {
        s->f[i].container = containers ? containers[i] : 0;
        s->f[i].flags = flags ? flags[i] : 0;
        s->f[i].elem_schema = elem_schemas ? elem_schemas[i] : 0;
    }
    return 0;
}

const orc_schema* orc_find_schema(const orc_table* t, int id) {
    for (int i = 0; i < t->n_schemas; i++)
        if (t->schemas[i].id == id) return &t->schemas[i];
    return NULL;
}
static const orc_schema* find_schema(const orc_table* t, int id) { return orc_find_schema(t, id); }

static void cls_set(uint8_t* cls, int c) { cls[c >> 3] |= (uint8_t)(1u << (c & 7)); }
static int cls_has(const uint8_t* cls, int c) { return (cls[c >> 3] >> (c & 7)) & 1; }
static void cls_range(uint8_t* cls, int a, int b) { for (int c = a; c <= b; c++) cls_set(cls, c); }
static void cls_invert(uint8_t* cls) { for (int i = 0; i < 32; i++) cls[i] = (uint8_t)~cls[i]; }
static void cls_add_escape(uint8_t* cls, int e) {
    if (e == 'd') cls_range(cls, '0', '9');
    else if (e == 'w') { cls_range(cls, '0', '9'); cls_range(cls, 'a', 'z'); cls_range(cls, 'A', 'Z'); cls_set(cls, '_'); }
    else cls_set(cls, e);
}

/* Parse a variable's regexp into atoms.  Supported subset of RE2 syntax (regexp/syntax): a concatenation of units, each
 * optionally quantified —
 *     unit:   [...] bracket class (ranges, \d \w and escaped punctuation inside) | \d | \w | \<punct> | . | a literal char
 *     quant:  + * ? {n} {n,} {n,m}
 * without alternation, groups, anchors or lazy quantifiers.  Matching is done on bytes; Go matches runes, so whatever
 * would count non-ASCII runes ({n}, ?, a bare '.' or negated class) is outside the subset.  Returns 0 ok, -1 unsupported. */
static int is_alnum_c(int c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
static int parse_unit(const char* p, int n, int* ip, uint8_t* cls, int* has_high, int* is_set) {
    int i = *ip;
    memset(cls, 0, 32);
    *has_high = 0;
    *is_set = 0;
    int c = (uint8_t)p[i];
    if (c == '[') {
        *is_set = 1;
        int neg = 0, first = 1;
        i++;
        if (i < n && p[i] == '^') { neg = 1; i++; }
        for (; i < n && (p[i] != ']' || first); first = 0) {
            int a = (uint8_t)p[i];
            if (a == '[' && i + 1 < n && p[i + 1] == ':') return -1; /* POSIX classes */
            if (a == '\\') {
                if (i + 1 >= n) return -1;
                int e = (uint8_t)p[i + 1];
                if (e == 'd' || e == 'w') { cls_add_escape(cls, e); i += 2; continue; }
                if (is_alnum_c(e)) return -1; /* \s \p{..} \x.. \b ... */
                a = e;
                i++;
            }
            if (a >= 0x80) return -1;
            if (i + 2 < n && p[i + 1] == '-' && p[i + 2] != ']') {
                int b = (uint8_t)p[i + 2];
                if (b == '\\') { if (i + 3 >= n) return -1; b = (uint8_t)p[i + 3]; i++; }
                if (b >= 0x80 || b < a) return -1;
                cls_range(cls, a, b);
                i += 3;
            } else {
                cls_set(cls, a);
                i++;
            }
        }
        if (i >= n) return -1;
        i++; /* ']' */
        if (neg) { cls_invert(cls); *has_high = 1; } /* a negated class also matches every non-ASCII rune */
    } else if (c == '\\') {
        if (i + 1 >= n) return -1;
        int e = (uint8_t)p[i + 1];
        if (e == 'd' || e == 'w') cls_add_escape(cls, e);
        else if (is_alnum_c(e) || e >= 0x80) return -1;
        else cls_set(cls, e);
        i += 2;
    } else if (c == '.') {
        *is_set = 1;
        memset(cls, 0xFF, 32);
        cls[1] &= (uint8_t)~(1u << ('\n' & 7)); /* '.' does not match \n without (?s) */
        *has_high = 1;
        i++;
    } else if (strchr("()|^$+*?{}]", c)) {
        return -1;
    } else {
        cls_set(cls, c);
        if (c >= 0x80) *has_high = 1;
        i++;
    }
    *ip = i;
    return 0;
}

static int parse_var_pattern(const char* p, int n, tpl_piece* pc) {
    pc->n_atoms = 0;
    int i = 0;
    while (i < n) {
        if (pc->n_atoms == 12) return -1;
        struct tpl_atom* at = &pc->atoms[pc->n_atoms];
        int high = 0, is_set = 0, lead = (uint8_t)p[i];
        if (parse_unit(p, n, &i, at->cls, &high, &is_set) != 0) return -1;
        int lo = 1, hi = 1, quantified = 0;
        if (i < n && (p[i] == '+' || p[i] == '*' || p[i] == '?')) {
            lo = p[i] == '+';
            hi = p[i] == '?' ? 1 : -1;
            quantified = 1;
            i++;
        } else if (i < n && p[i] == '{') {
            int j = i + 1, d = 0;
            lo = 0;
            while (j < n && p[j] >= '0' && p[j] <= '9' && d < 4) { lo = lo * 10 + (p[j] - '0'); j++; d++; }
            if (d == 0 || lo > 250) return -1;
            if (j < n && p[j] == '}') hi = lo;
            else if (j + 1 < n && p[j] == ',' && p[j + 1] == '}') { hi = -1; j++; }
            else if (j < n && p[j] == ',') {
                j++;
                d = 0; hi = 0;
                while (j < n && p[j] >= '0' && p[j] <= '9' && d < 4) { hi = hi * 10 + (p[j] - '0'); j++; d++; }
                if (d == 0 || hi > 250 || hi < lo || hi == 0) return -1;
            } else return -1;
            if (j >= n || p[j] != '}') return -1;
            if (hi == 0) return -1; /* {0} */
            quantified = 1;
            i = j + 1;
        }
        if (i < n && (p[i] == '+' || p[i] == '*' || p[i] == '?' || p[i] == '{')) return -1; /* lazy, stacked */
        /* rune vs byte: only X+ / X* are the same thing on bytes when X can match non-ASCII */
        int open_ended = hi < 0 && lo <= 1;
        if (high && is_set && !open_ended) return -1;
        if (high && !is_set && quantified) return -1; /* a byte of a multi-byte literal cannot carry the quantifier */
        at->min_rep = lo;
        at->max_rep = hi;
        (void)lead;
        pc->n_atoms++;
    }
    return pc->n_atoms ? 0 : -1;
}

/* mux newRouteRegexp: split the template at top-level braces; {name} → [^/]+, {name:pattern} → pattern. */
static int parse_template(orc_route* r, const char* tpl, int n) {
    int cap = 4;
    r->pieces = (tpl_piece*)calloc((size_t)cap, sizeof(tpl_piece));
    r->n_pieces = 0;
    int i = 0, lit_start = 0;
    for (;;) {
        /* find next '{' */
        int j = i;
        while (j < n && tpl[j] != '{' && tpl[j] != '}') j++;
        if (j < n && tpl[j] == '}') return -2; /* unbalanced braces: mux error → dead route */
        if (r->n_pieces == cap) { cap *= 2; r->pieces = (tpl_piece*)realloc(r->pieces, sizeof(tpl_piece) * (size_t)cap); }
        tpl_piece* pc = &r->pieces[r->n_pieces++];
        memset(pc, 0, sizeof *pc);
        pc->lit = dup_bytes(tpl + lit_start, j - lit_start);
        pc->lit_len = j - lit_start;
        if (j >= n) break;
        /* matching '}' (braces may nest inside the regexp part) */
        int depth = 0, k = j;
        for (; k < n; k++) {
            if (tpl[k] == '{') depth++;
            else if (tpl[k] == '}') { depth--; if (depth == 0) break; }
        }
        if (k >= n) return -2;
        const char* body = tpl + j + 1;
        int bl = k - j - 1;
        int colon = -1;
        for (int q = 0; q < bl; q++) if (body[q] == ':') { colon = q; break; }
        int name_len = colon < 0 ? bl : colon;
        if (name_len == 0) return -2; /* mux: missing name → route error */
        pc->has_var = 1;
        pc->name = (char*)calloc((size_t)name_len + 1, 1);
        memcpy(pc->name, body, (size_t)name_len);
        for (int q = 0; q + 1 < r->n_pieces; q++) /* mux: "duplicated route variable" → route error */
            if (r->pieces[q].has_var && strcmp(r->pieces[q].name, pc->name) == 0) return -2;
        if (colon < 0) {
            pc->n_atoms = 1;
            memset(pc->atoms[0].cls, 0xFF, 32);
            pc->atoms[0].cls['/' >> 3] &= (uint8_t)~(1u << ('/' & 7));
            pc->atoms[0].min_rep = 1;
            pc->atoms[0].max_rep = -1;
        } else {
            if (bl - colon - 1 == 0) return -2; /* mux: missing pattern */
            if (parse_var_pattern(body + colon + 1, bl - colon - 1, pc) != 0) return -1;
        }
        i = k + 1;
        lit_start = i;
    }
    return 0;
}

int orc_add_route(orc_table* t, int method, const char* pattern, int pattern_len, int hkind, int schema_id,
                  const char* s0, int s0_len, const char* s1, int s1_len, const char* s2, int s2_len, const char* s3,
                  int s3_len, const uint8_t* blob, int blob_len) {
    if (t->n_routes == t->cap_routes) {
        t->cap_routes = t->cap_routes ? t->cap_routes * 2 : 16;
        t->routes = (orc_route*)realloc(t->routes, sizeof(orc_route) * (size_t)t->cap_routes);
    }
    orc_route* r = &t->routes[t->n_routes];
    memset(r, 0, sizeof *r);
    r->method = method;
    r->prefix = (method == M_ANY);
    r->hkind = hkind;
    r->schema_id = schema_id;
    const char* ss[4] = {s0, s1, s2, s3};
    int sl[4] = {s0_len, s1_len, s2_len, s3_len};
    for (int k = 0; k < 4; k++) { r->s[k] = dup_bytes(ss[k] ? ss[k] : "", sl[k]); r->sl[k] = ss[k] ? sl[k] : 0; }
    r->blob = dup_bytes(blob ? blob : (const uint8_t*)"", blob_len);
    r->blob_len = blob ? blob_len : 0;
    int rc = parse_template(r, pattern, pattern_len);
    if (rc == -1) return -1; /* unsupported regexp: refuse rather than mis-route */
    /* mux addRegexpMatcher: "path must start with a slash" → r.err set → Route.Match always false */
    if (rc == -2 || pattern_len == 0 || pattern[0] != '/') r->dead = 1;
    return t->n_routes++;
}

/* App.Run(): pkg/gofr/gofr.go:102-107 */
int orc_add_default_routes(orc_table* t, const uint8_t* favicon, int favicon_len) {
    orc_add_route(t, 0, "/.well-known/health", 19, H_HEALTH, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0);
    orc_add_route(t, 0, "/favicon.ico", 12, H_FILE, 0, "image/x-icon", 12, 0, 0, 0, 0, 0, 0, favicon, favicon_len);
    orc_add_route(t, M_ANY, "/", 1, H_MISSING_FILE, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0);
    return 0;
}

/* ------------------------------------------------------------------------------------------------------------ */
/* encoding/json (Go 1.21) — encoder                                                                            */
/* ------------------------------------------------------------------------------------------------------------ */

static const char HEXL[] = "0123456789abcdef";

/* utf8.DecodeRune: returns size (1..4) and *r; invalid → (0xFFFD, 1). */
static int go_decode_rune(const uint8_t* s, size_t n, uint32_t* r) {
    uint8_t b0 = s[0];
    if (b0 < 0x80) { *r = b0; return 1; }
    if (b0 < 0xC2 || b0 > 0xF4) { *r = 0xFFFD; return 1; }
    if (b0 < 0xE0) {
        if (n < 2 || (s[1] & 0xC0) != 0x80) { *r = 0xFFFD; return 1; }
        *r = ((uint32_t)(b0 & 0x1F) << 6) | (s[1] & 0x3F);
        return 2;
    }
    if (b0 < 0xF0) {
        uint8_t lo = 0x80, hi = 0xBF;
        if (b0 == 0xE0) lo = 0xA0;
        if (b0 == 0xED) hi = 0x9F;
        if (n < 3 || s[1] < lo || s[1] > hi || (s[2] & 0xC0) != 0x80) { *r = 0xFFFD; return 1; }
        *r = ((uint32_t)(b0 & 0x0F) << 12) | ((uint32_t)(s[1] & 0x3F) << 6) | (s[2] & 0x3F);
        return 3;
    }
    uint8_t lo = 0x80, hi = 0xBF;
    if (b0 == 0xF0) lo = 0x90;
    if (b0 == 0xF4) hi = 0x8F;
    if (n < 4 || s[1] < lo || s[1] > hi || (s[2] & 0xC0) != 0x80 || (s[3] & 0xC0) != 0x80) { *r = 0xFFFD; return 1; }
    *r = ((uint32_t)(b0 & 0x07) << 18) | ((uint32_t)(s[1] & 0x3F) << 12) | ((uint32_t)(s[2] & 0x3F) << 6) | (s[3] & 0x3F);
    return 4;
}

/* encodeState.string with escapeHTML=true (json.Encoder default). Go 1.21: \b and \f have no short form. */
void orc_enc_string(obuf* b, const uint8_t* s, size_t n) {
    ob_putc(b, '"');
    size_t i = 0;
    while (i < n) {
        uint8_t c = s[i];
        if (c < 0x80) {
            int safe = c >= 0x20 && c != '"' && c != '\\' && c != '<' && c != '>' && c != '&';
            if (safe) { ob_putc(b, c); i++; continue; }
            switch (c) {
                case '\\': case '"': ob_putc(b, '\\'); ob_putc(b, c); break;
                case '\n': ob_put(b, "\\n", 2); break;
                case '\r': ob_put(b, "\\r", 2); break;
                case '\t': ob_put(b, "\\t", 2); break;
                default:
                    ob_put(b, "\\u00", 4);
                    ob_putc(b, (uint8_t)HEXL[c >> 4]);
                    ob_putc(b, (uint8_t)HEXL[c & 0xF]);
            }
            i++;
            continue;
        }
        uint32_t r;
        int sz = go_decode_rune(s + i, n - i, &r);
        if (r == 0xFFFD && sz == 1) { ob_put(b, "\\ufffd", 6); i += 1; continue; }
        if (r == 0x2028 || r == 0x2029) { ob_put(b, "\\u202", 5); ob_putc(b, (uint8_t)HEXL[r & 0xF]); i += (size_t)sz; continue; }
        ob_put(b, s + i, (size_t)sz);
        i += (size_t)sz;
    }
    ob_putc(b, '"');
}

/* strconv.AppendInt(v, 10) */
void orc_enc_int(obuf* b, int64_t v) {
    char tmp[24];
    int k = 0;
    uint64_t u = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    do { tmp[k++] = (char)('0' + u % 10); u /= 10; } while (u);
    if (v < 0) ob_putc(b, '-');
    while (k) ob_putc(b, (uint8_t)tmp[--k]);
}

/* struct encoder: declaration order, `json:"name,omitempty"` (isEmptyValue: len==0 / ==0 / false) */
void orc_enc_struct(obuf* b, const orc_schema* sc, const orc_value* v) {
    ob_putc(b, '{');
    int first = 1;
    for (int i = 0; i < sc->n_fields; i++) {
        const orc_field* f = &sc->f[i];
        if (f->omitempty) {
            if (f->kind == F_STRING ? v[i].sn == 0 : f->kind == F_FLOAT64 ? ((uint64_t)v[i].i << 1) == 0 : v[i].i == 0) continue;
        }
        if (!first) ob_putc(b, ',');
        first = 0;
        /* field names are emitted through the same string encoder (HTML-safe) as `"name":` */
        orc_enc_string(b, (const uint8_t*)f->json_name, strlen(f->json_name));
        ob_putc(b, ':');
        switch (f->kind) {
            case F_STRING: orc_enc_string(b, v[i].s, (size_t)v[i].sn); break;
            case F_BOOL: ob_puts(b, v[i].i ? "true" : "false"); break;
            case F_FLOAT64: { /* Bind stores only finite values: the text always exists */
                double x;
                char tmp[40];
                memcpy(&x, &v[i].i, 8);
                ob_put(b, tmp, (size_t)orc_float_text(x, tmp));
                break;
            }
            default: orc_enc_int(b, v[i].i); break;
        }
    }
    ob_putc(b, '}');
}

/* ------------------------------------------------------------------------------------------------------------ */
/* path.Clean + mux cleanPath; net/url escaping                                                                 */
/* ------------------------------------------------------------------------------------------------------------ */

/* Go path.Clean for a rooted path (mux always prepends '/'). */
static void go_path_clean_rooted(const uint8_t* p, size_t n, obuf* out) {
    /* out acts as lazybuf; dotdot = 1 */
    size_t r = 1;
    ob_putc(out, '/');
    size_t base = out->n - 1; /* index of the leading '/' */
    while (r < n) {
        if (p[r] == '/') {
            r++;
        } else if (p[r] == '.' && (r + 1 == n || p[r + 1] == '/')) {
            r++;
        } else if (p[r] == '.' && p[r + 1] == '.' && (r + 2 == n || p[r + 2] == '/')) {
            r += 2;
            if (out->n - base > 1) { /* out.w > dotdot: back up to previous '/' */
                out->n--;
                while (out->n - base > 1 && out->p[out->n] != '/') out->n--;
            }
        } else {
            if (out->n - base != 1) ob_putc(out, '/');
            for (; r < n && p[r] != '/'; r++) ob_putc(out, p[r]);
        }
    }
}

/* mux.cleanPath (mux.go): "" → "/"; ensure leading '/'; path.Clean; restore a trailing slash. */
static void mux_clean_path(const uint8_t* p, size_t n, obuf* out) {
    if (n == 0) { ob_putc(out, '/'); return; }
    obuf tmp;
    ob_init(&tmp);
    if (p[0] != '/') ob_putc(&tmp, '/');
    ob_put(&tmp, p, n);
    size_t start = out->n;
    go_path_clean_rooted(tmp.p, tmp.n, out);
    size_t np_len = out->n - start;
    if (tmp.p[tmp.n - 1] == '/' && !(np_len == 1 && out->p[start] == '/')) ob_putc(out, '/');
    ob_free(&tmp);
}

/* url.escape(s, encodePath): unreserved and $&+,/:;=@ stay; everything else %XX (upper-case hex). */
static void url_escape_path(const uint8_t* s, size_t n, obuf* out) {
    static const char HEXU[] = "0123456789ABCDEF";
    for (size_t i = 0; i < n; i++) {
        uint8_t c = s[i];
        int keep = (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '-' || c == '_' ||
                   c == '.' || c == '~' || c == '$' || c == '&' || c == '+' || c == ',' || c == '/' || c == ':' ||
                   c == ';' || c == '=' || c == '@';
        if (keep) ob_putc(out, c);
        else { ob_putc(out, '%'); ob_putc(out, (uint8_t)HEXU[c >> 4]); ob_putc(out, (uint8_t)HEXU[c & 15]); }
    }
}

static int hexval(uint8_t c) {
    if (c >= '0' && c <= '9') return c - '0';
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return c - 'A' + 10;
    return -1;
}

/* url.QueryUnescape: returns 0 and appends to out, or -1 on a bad %-escape. */
static int query_unescape(const uint8_t* s, size_t n, obuf* out) {
    /* first pass (url.unescape): "if i+2 >= len(s) || !ishex(s[i+1]) || !ishex(s[i+2])" → EscapeError */
    for (size_t i = 0; i < n;) {
        if (s[i] == '%') {
            if (i + 2 >= n || hexval(s[i + 1]) < 0 || hexval(s[i + 2]) < 0) return -1;
            i += 3;
        } else {
            i++;
        }
    }
    for (size_t i = 0; i < n;) {
        if (s[i] == '%') { ob_putc(out, (uint8_t)(hexval(s[i + 1]) << 4 | hexval(s[i + 2]))); i += 3; }
        else if (s[i] == '+') { ob_putc(out, ' '); i++; }
        else { ob_putc(out, s[i]); i++; }
    }
    return 0;
}

/* req.URL.Query().Get(key): url.ParseQuery keeps going past bad pairs; first value wins.  request.go:28-30 */
static void query_get(const uint8_t* q, size_t qn, const uint8_t* key, size_t kn, obuf* out) {
    size_t i = 0;
    obuf k, v;
    ob_init(&k);
    ob_init(&v);
    while (i < qn) {
        size_t j = i;
        while (j < qn && q[j] != '&') j++;
        const uint8_t* pair = q + i;
        size_t pn = j - i;
        i = j < qn ? j + 1 : j;
        if (memchr(pair, ';', pn)) continue; /* "invalid semicolon separator in query" */
        if (pn == 0) continue;
        size_t e = 0;
        while (e < pn && pair[e] != '=') e++;
        k.n = 0;
        v.n = 0;
        if (query_unescape(pair, e, &k) != 0) continue;
        if (e < pn) { if (query_unescape(pair + e + 1, pn - e - 1, &v) != 0) continue; }
        if (k.n == kn && memcmp(k.p ? k.p : (uint8_t*)"", key, kn) == 0) {
            ob_put(out, v.p, v.n);
            break;
        }
    }
    ob_free(&k);
    ob_free(&v);
}

/* ------------------------------------------------------------------------------------------------------------ */
/* gorilla/mux v1.8.1 matching                                                                                  */
/* ------------------------------------------------------------------------------------------------------------ */

/* Anchored leftmost-first match of lit0 (var0 lit1 (var1 ...)) [$]: greedy variables with backtracking, which is
 * what Go's regexp reports for this shape. */
typedef struct { size_t off, len; } var_span;
static int tpl_match_from(const orc_route* r, int k, const uint8_t* p, size_t n, size_t pos, var_span* spans);
/* atoms a.. of piece k's variable, the variable having started at var_start */
static int tpl_match_atoms(const orc_route* r, int k, int a, const uint8_t* p, size_t n, size_t pos, size_t var_start, var_span* spans) {
    const tpl_piece* pc = &r->pieces[k];
    if (a == pc->n_atoms) {
        int ok = k + 1 < r->n_pieces ? tpl_match_from(r, k + 1, p, n, pos, spans) : (r->prefix || pos == n);
        if (ok && spans) { spans[k].off = var_start; spans[k].len = pos - var_start; }
        return ok;
    }
    const struct tpl_atom* at = &pc->atoms[a];
    size_t run = 0;
    while (pos + run < n && (at->max_rep < 0 || run < (size_t)at->max_rep) && cls_has(at->cls, p[pos + run])) run++;
    for (size_t take = run;; take--) { /* greedy, giving back one byte at a time */
        if (take >= (size_t)at->min_rep && tpl_match_atoms(r, k, a + 1, p, n, pos + take, var_start, spans)) return 1;
        if (take == 0) break;
    }
    return 0;
}
static int tpl_match_from(const orc_route* r, int k, const uint8_t* p, size_t n, size_t pos, var_span* spans) {
    const tpl_piece* pc = &r->pieces[k];
    if (n - pos < (size_t)pc->lit_len || memcmp(p + pos, pc->lit, (size_t)pc->lit_len) != 0) return 0;
    pos += (size_t)pc->lit_len;
    if (!pc->has_var) return r->prefix ? 1 : pos == n;
    return tpl_match_atoms(r, k, 0, p, n, pos, pos, spans);
}

static int path_matches(const orc_route* r, const uint8_t* p, size_t n) {
    if (r->n_pieces == 0) return 0;
    /* a template ending in a variable has a trailing empty literal piece; one ending in a literal has has_var=0 */
    return tpl_match_from(r, 0, p, n, 0, NULL);
}

enum { MATCH_404 = -1, MATCH_405 = -2, MATCH_301 = -3 };

/* Router.Match + Route.Match (mux v1.8.1 route.go): returns the route index or MATCH_404 / MATCH_405. */
static int mux_match(const orc_table* t, int method, const uint8_t* path, size_t n) {
    int match_err_mismatch = 0; /* match.MatchErr == ErrMethodMismatch */
    for (int i = 0; i < t->n_routes; i++) {
        const orc_route* r = &t->routes[i];
        if (r->dead) continue; /* r.err != nil → return false before touching match */
        int route_err = 0;     /* matchErr local to Route.Match */
        int failed = 0;
        /* matchers in the order Router.Add builds them: Methods(m) then Path(p)  (router.go:32) */
        if (r->method != M_ANY) {
            if (r->method != method || method == 15 /* OTHER never equals a registered method */) {
                route_err = 1; /* methodMatcher failed: remember, keep evaluating the remaining matchers */
            } else if (match_err_mismatch) {
                match_err_mismatch = 0; /* a matcher succeeded: clear a stale ErrMethodMismatch */
            }
        }
        if (!path_matches(r, path, n)) {
            failed = 1; /* non-method matcher failed: return false, MatchErr untouched */
        } else if (match_err_mismatch) {
            match_err_mismatch = 0;
        }
        if (failed) continue;
        if (route_err) { match_err_mismatch = 1; continue; }
        return i;
    }
    return match_err_mismatch ? MATCH_405 : MATCH_404;
}

int orc_match(const orc_table* t, int method, const uint8_t* path, int path_len) {
    obuf c;
    ob_init(&c);
    mux_clean_path(path, (size_t)path_len, &c);
    int changed = !(c.n == (size_t)path_len && memcmp(c.p, path, c.n) == 0);
    ob_free(&c);
    if (changed) return MATCH_301;
    return mux_match(t, method, path, (size_t)path_len);
}

/* Routing only: what Router.ServeHTTP and the middleware chain decide before the handler runs (router.go:14,30-33;
 * cors.go:10-13), plus the spans mux.Vars would hold.  meta = status | route << 16 with status 301 / 404 / 405 /
 * 200 (OPTIONS) / 0 (handler runs); vars[k] = off | len << 16 of the k-th variable, 0xFFFFFFFF unused. */
int orc_route_batch(const orc_table* t, const void* desc_v, const uint8_t* arena, uint32_t n, uint32_t* meta, uint32_t* vars,
              int max_vars) {
    const uint8_t* desc = (const uint8_t*)desc_v;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t d[4];
        memcpy(d, desc + (size_t)i * 16, 16);
        const uint8_t* path = arena + d[0];
        size_t pn = d[1] & 0xFFFFu;
        int method = (int)(d[3] & 0xFFu);
        for (int k = 0; k < max_vars; k++) vars[(size_t)i * (size_t)max_vars + (size_t)k] = 0xFFFFFFFFu;
        int m = orc_match(t, method, path, (int)pn);
        if (m < 0) {
            meta[i] = (uint32_t)(m == MATCH_301 ? 301 : m == MATCH_405 ? 405 : 404) | 0xFFFFu << 16;
            continue;
        }
        const orc_route* r = &t->routes[m];
        var_span spans[64];
        memset(spans, 0, sizeof spans);
        tpl_match_from(r, 0, path, pn, 0, spans);
        int nv = 0;
        for (int k = 0; k < r->n_pieces && nv < max_vars; k++)
            if (r->pieces[k].has_var)
                vars[(size_t)i * (size_t)max_vars + (size_t)nv++] = (uint32_t)spans[k].off | (uint32_t)spans[k].len << 16;
        meta[i] = (method == 7 /* OPTIONS */ ? 200u : 0u) | (uint32_t)m << 16;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------------------------ */
/* http.ResponseWriter model + net/http 1.21 framing                                                            */
/* ------------------------------------------------------------------------------------------------------------ */

typedef struct { const char* k; obuf v; } hdr;
typedef struct {
    hdr live[8];
    int n_live;
    hdr snap[8];
    int n_snap;
    int wrote_header;
    int status;
    obuf body;
    int frame_mode;
    int chunked; /* a Write larger than the 2 KiB bufio.Writer reached chunkWriter before the handler returned */
    int static_body; /* handler_result.static_body */
    int is_file; /* the body comes from resTypes.File */
} rw_t;

/* response.w is bufio.NewWriterSize(&w.cw, 2048): a Write of more than 2048 bytes into the empty buffer goes straight to
 * chunkWriter.Write, which writes the header block THEN — the handler has not returned, so no Content-Length is known and an
 * HTTP/1.1 response switches to "Transfer-Encoding: chunked" (server.go chunkWriter.writeHeader); the one Write becomes one
 * chunk.  Every body of this path is a single Write (json.Encoder.Encode, File).
 * For File bodies the product frames exactly like this.  For JSON bodies beyond 2 KiB it sends Content-Length instead — a
 * DEVIATION stated in DESIGN.md §8 — and the oracle follows the product unless orc_set_strict_chunking(1) is in effect, which
 * tests/test_result.py uses to pin what the difference is. */
static int g_strict_chunking = 0;
void orc_set_strict_chunking(int on) { g_strict_chunking = on; }

static void rw_init(rw_t* w, int frame_mode) { memset(w, 0, sizeof *w); w->frame_mode = frame_mode; ob_init(&w->body); }
static void rw_free(rw_t* w) {
    for (int i = 0; i < w->n_live; i++) ob_free(&w->live[i].v);
    for (int i = 0; i < w->n_snap; i++) ob_free(&w->snap[i].v);
    ob_free(&w->body);
}
/* Header().Set(k, v): k is given already canonicalised (textproto.CanonicalMIMEHeaderKey):
 * "X-Correlation-ID" → "X-Correlation-Id", "Content-type" → "Content-Type". */
static void rw_set(rw_t* w, const char* canon_key, const void* v, size_t vn) {
    for (int i = 0; i < w->n_live; i++)
        if (strcmp(w->live[i].k, canon_key) == 0) { w->live[i].v.n = 0; ob_put(&w->live[i].v, v, vn); return; }
    hdr* h = &w->live[w->n_live++];
    h->k = canon_key;
    ob_init(&h->v);
    ob_put(&h->v, v, vn);
}
static void rw_snapshot(rw_t* w) {
    for (int i = 0; i < w->n_snap; i++) ob_free(&w->snap[i].v);
    w->n_snap = w->n_live;
    for (int i = 0; i < w->n_live; i++) {
        w->snap[i].k = w->live[i].k;
        ob_init(&w->snap[i].v);
        ob_put(&w->snap[i].v, w->live[i].v.p, w->live[i].v.n);
    }
}
/* response.WriteHeader: first call wins; the header map is cloned here (server.go: cw.header = handlerHeader.Clone()). */
static void rw_write_header(rw_t* w, int code) {
    if (w->wrote_header) return;
    w->wrote_header = 1;
    w->status = code;
    rw_snapshot(w);
}
static void rw_write(rw_t* w, const void* p, size_t n) {
    if (!w->wrote_header) rw_write_header(w, 200);
    if (n > 2048 && w->body.n == 0 && w->frame_mode == FRAME_WIRE && (w->is_file || g_strict_chunking)) w->chunked = 1;
    ob_put(&w->body, p, n);
}

/* Encoder.Encode: enc.w.Write(e.Bytes()) — the body assembled in w->body above arrives as ONE Write (see rw_write) */
static void rw_encoded_in_one_write(rw_t* w) {
    if (w->body.n > 2048 && w->frame_mode == FRAME_WIRE && (g_strict_chunking || w->static_body)) w->chunked = 1;
}

static const char* status_text(int code) {
    switch (code) {
        case 200: return "OK";
        case 301: return "Moved Permanently";
        case 404: return "Not Found";
        case 405: return "Method Not Allowed";
        case 500: return "Internal Server Error";
        default: return "";
    }
}

/* http.DetectContentType (net/http sniff.go; the WHATWG MIME Sniffing tables), signatures in sniffSignatures' order: html
 * tags, xml, pdf / postscript, BOMs, images, audio / video incl. the mp4 box walk, fonts, archives, wasm, then text vs
 * binary.  (JSON text never contains a "binary" byte — all < 0x20 are \u-escaped — and never starts with a signature →
 * text/plain; charset=utf-8.) */
static int sig_at(const uint8_t* p, size_t n, size_t off, const char* pat, size_t len) {
    return n >= off + len && memcmp(p + off, pat, len) == 0;
}
/* allow_masked_font: the embedded-OpenType signature is 34 DON'T-CARE bytes followed by "LP" — the only signature JSON text
 * can hit (any body with "LP" at offset 34, e.g. inside a string, is sniffed as application/vnd.ms-fontobject by the
 * reference).  The product's programs assume JSON never sniffs as anything but text/plain — a DEVIATION stated in DESIGN.md
 * §8; the oracle follows the product for JSON bodies unless orc_set_strict_chunking(1) is in effect, and always applies the
 * signature to File bodies (as the product's seal-time sniffer does). */
static const char* detect_content_type(const uint8_t* p, size_t n, int allow_masked_font) {
    if (n > 512) n = 512;
    size_t ws = 0;
    while (ws < n && (p[ws] == '\t' || p[ws] == '\n' || p[ws] == '\x0c' || p[ws] == '\r' || p[ws] == ' ')) ws++;
    static const char* const html_sigs[] = {"<!DOCTYPE HTML", "<HTML", "<HEAD", "<SCRIPT", "<IFRAME", "<H1", "<DIV",
                                            "<FONT", "<TABLE", "<A", "<STYLE", "<TITLE", "<B", "<BODY", "<BR", "<P",
                                            "<!--"};
    for (size_t k = 0; k < sizeof html_sigs / sizeof *html_sigs; k++) {
        size_t L = strlen(html_sigs[k]);
        if (n - ws < L + 1) continue;
        size_t q = 0;
        for (; q < L; q++) {
            uint8_t c = p[ws + q], s = (uint8_t)html_sigs[k][q];
            if (s >= 'A' && s <= 'Z') c &= 0xDF;
            if (c != s) break;
        }
        if (q == L && (p[ws + L] == ' ' || p[ws + L] == '>')) return "text/html; charset=utf-8";
    }
    if (n - ws >= 5 && memcmp(p + ws, "<?xml", 5) == 0) return "text/xml; charset=utf-8";
    if (n >= 5 && memcmp(p, "%PDF-", 5) == 0) return "application/pdf";
    if (n >= 11 && memcmp(p, "%!PS-Adobe-", 11) == 0) return "application/postscript";
    if (n >= 4 && p[0] == 0xFE && p[1] == 0xFF) return "text/plain; charset=utf-16be";
    if (n >= 4 && p[0] == 0xFF && p[1] == 0xFE) return "text/plain; charset=utf-16le";
    if (n >= 4 && p[0] == 0xEF && p[1] == 0xBB && p[2] == 0xBF) return "text/plain; charset=utf-8";
    if (n >= 4 && memcmp(p, "\x00\x00\x01\x00", 4) == 0) return "image/x-icon";
    if (n >= 4 && memcmp(p, "\x00\x00\x02\x00", 4) == 0) return "image/x-icon";
    if (n >= 2 && memcmp(p, "BM", 2) == 0) return "image/bmp";
    if (n >= 6 && (memcmp(p, "GIF87a", 6) == 0 || memcmp(p, "GIF89a", 6) == 0)) return "image/gif";
    if (n >= 14 && memcmp(p, "RIFF", 4) == 0 && memcmp(p + 8, "WEBPVP", 6) == 0) return "image/webp";
    if (n >= 8 && memcmp(p, "\x89PNG\x0D\x0A\x1A\x0A", 8) == 0) return "image/png";
    if (n >= 3 && memcmp(p, "\xFF\xD8\xFF", 3) == 0) return "image/jpeg";
    /* audio and video */
    if (sig_at(p, n, 0, "FORM", 4) && sig_at(p, n, 8, "AIFF", 4)) return "audio/aiff";
    if (sig_at(p, n, 0, "ID3", 3)) return "audio/mpeg";
    if (sig_at(p, n, 0, "OggS\0", 5)) return "application/ogg";
    if (sig_at(p, n, 0, "MThd\0\0\0\x06", 8)) return "audio/midi";
    if (sig_at(p, n, 0, "RIFF", 4) && sig_at(p, n, 8, "AVI ", 4)) return "video/avi";
    if (sig_at(p, n, 0, "RIFF", 4) && sig_at(p, n, 8, "WAVE", 4)) return "audio/wave";
    if (n >= 12) { /* mp4Sig.match */
        size_t box = (size_t)p[0] << 24 | (size_t)p[1] << 16 | (size_t)p[2] << 8 | (size_t)p[3];
        if (n >= box && box % 4 == 0 && memcmp(p + 4, "ftyp", 4) == 0) {
            for (size_t st = 8; st < box; st += 4) {
                if (st == 12) continue; /* the version number of the major brand */
                if (memcmp(p + st, "mp4", 3) == 0) return "video/mp4";
            }
        }
    }
    if (sig_at(p, n, 0, "\x1A\x45\xDF\xA3", 4)) return "video/webm";
    /* fonts: 34 NUL bytes then "LP"; TrueType, OpenType, collections, WOFF */
    if (allow_masked_font && n >= 36 && p[34] == 'L' && p[35] == 'P') return "application/vnd.ms-fontobject"; /* the mask ignores bytes 0..33 */
    if (sig_at(p, n, 0, "\0\x01\0\0", 4)) return "font/ttf";
    if (sig_at(p, n, 0, "OTTO", 4)) return "font/otf";
    if (sig_at(p, n, 0, "ttcf", 4)) return "font/collection";
    if (sig_at(p, n, 0, "wOFF", 4)) return "font/woff";
    if (sig_at(p, n, 0, "wOF2", 4)) return "font/woff2";
    /* archives */
    if (n >= 3 && memcmp(p, "\x1F\x8B\x08", 3) == 0) return "application/x-gzip";
    if (n >= 4 && memcmp(p, "PK\x03\x04", 4) == 0) return "application/zip";
    if (sig_at(p, n, 0, "Rar!\x1A\x07\0", 7)) return "application/x-rar-compressed";
    if (sig_at(p, n, 0, "Rar!\x1A\x07\x01\0", 8)) return "application/x-rar-compressed";
    if (sig_at(p, n, 0, "\0\x61\x73\x6D", 4)) return "application/wasm";
    for (size_t i = ws; i < n; i++) { /* textSig: from the first non-whitespace byte */
        uint8_t c = p[i];
        if (c <= 0x08 || c == 0x0B || (c >= 0x0E && c <= 0x1A) || (c >= 0x1C && c <= 0x1F)) return "application/octet-stream";
    }
    return "text/plain; charset=utf-8";
}

static int hdr_cmp(const void* a, const void* b) { return strcmp(((const hdr*)a)->k, ((const hdr*)b)->k); }

/* finishRequest → chunkWriter.writeHeader + body (HTTP/1.1 keep-alive request, handler done, body < 2048 B or
 * any size: Content-Length is set because the handler has returned before the first flush for our bodies; bodies
 * beyond the 2 KiB bufio would be chunked in the reference — the File route notes this in DESIGN.md). */
static void rw_finish(rw_t* w, int is_head, const char* date29, obuf* out) {
    if (!w->wrote_header) rw_write_header(w, 200);
    if (w->frame_mode == FRAME_BODY) {
        if (!is_head) ob_put(out, w->body.p, w->body.n);
        return;
    }
    /* INTENDED mode models the httptest recorder's live map (what the reference's tests read) */
    hdr* H = w->frame_mode == FRAME_INTENDED ? w->live : w->snap;
    int nH = w->frame_mode == FRAME_INTENDED ? w->n_live : w->n_snap;
    char line[64];
    int L = snprintf(line, sizeof line, "HTTP/1.1 %d %s\r\n", w->status, status_text(w->status));
    ob_put(out, line, (size_t)L);
    hdr sorted[8];
    memcpy(sorted, H, sizeof(hdr) * (size_t)nH);
    qsort(sorted, (size_t)nH, sizeof(hdr), hdr_cmp); /* Header.WriteSubset → sortedKeyValues */
    int have_type = 0;
    for (int i = 0; i < nH; i++) {
        ob_puts(out, sorted[i].k);
        ob_put(out, ": ", 2);
        ob_put(out, sorted[i].v.p, sorted[i].v.n);
        ob_put(out, "\r\n", 2);
        if (strcmp(sorted[i].k, "Content-Type") == 0) have_type = 1;
    }
    /* extraHeader.Write order: Date, Content-Length, Content-Type, Connection, Transfer-Encoding */
    ob_put(out, "Date: ", 6);
    ob_put(out, date29, 29);
    ob_put(out, "\r\n", 2);
    size_t plen = w->body.n;
    if (!w->chunked && (!is_head || plen > 0)) { /* handlerDone && bodyAllowedForStatus && no Content-Length && (!isHEAD || len(p)>0) */
        L = snprintf(line, sizeof line, "Content-Length: %zu\r\n", plen);
        ob_put(out, line, (size_t)L);
    }
    if (!have_type && plen > 0) {
        ob_puts(out, "Content-Type: ");
        ob_puts(out, detect_content_type(w->body.p, w->body.n, w->is_file || g_strict_chunking));
        ob_put(out, "\r\n", 2);
    }
    if (w->chunked && !is_head) ob_puts(out, "Transfer-Encoding: chunked\r\n"); /* HEAD: "do nothing" — neither length nor encoding */
    ob_put(out, "\r\n", 2);
    if (is_head) return; /* chunkWriter.Write eats the body of a HEAD response */
    if (w->chunked) { /* one chunk, then chunkWriter.close's terminator */
        L = snprintf(line, sizeof line, "%zx\r\n", plen);
        ob_put(out, line, (size_t)L);
        ob_put(out, w->body.p, w->body.n);
        ob_puts(out, "\r\n0\r\n\r\n");
        return;
    }
    ob_put(out, w->body.p, w->body.n);
}

/* ------------------------------------------------------------------------------------------------------------ */
/* Responder.Respond  (pkg/gofr/http/responder.go:19-57)                                                         */
/* ------------------------------------------------------------------------------------------------------------ */

typedef struct {
    int data_kind; /* 0 nil, 1 string, 2 struct, 3 empty map (health), 4 File, 5 a value already encoded (orc_value.c) */
    const uint8_t* json; /* data_kind 5 */
    size_t json_len;
    int enc_failed;      /* data_kind 5: json.Encoder.Encode returned an UnsupportedValueError (NaN / Inf) */
    const uint8_t* str;
    size_t str_len;
    const orc_schema* sc;
    const orc_value* vals;
    const uint8_t* file;
    size_t file_len;
    const uint8_t* file_ct;
    size_t file_ct_len;
    int has_err;
    int err_is_missing_file; /* errors.Is(err, http.ErrMissingFile) */
    const uint8_t* err_msg;
    size_t err_len;
    int static_body; /* the handler returns a constant (GOFR_H_STATIC_*): the product knows the body length when the table is
                        sealed and frames bodies beyond 2 KiB as the reference does — see rw_write */
    int raw; /* data is a response.Raw{Data: ...}: Respond encodes v.Data bare (pkg/gofr/http/responder.go:24-26, response/raw.go:3-5) */
} handler_result;

static void respond(rw_t* w, const handler_result* r) {
    /* HTTPStatusFromError :43-57 */
    int status = 200;
    if (r->has_err) status = r->err_is_missing_file ? 404 : 500;
    rw_write_header(w, status); /* :21 — BEFORE the Content-type Set below */
    w->static_body = r->static_body;
    if (r->data_kind == 4) {    /* resTypes.File :27-31 */
        w->is_file = 1;
        rw_set(w, "Content-Type", r->file_ct, r->file_ct_len);
        rw_write(w, r->file, r->file_len);
        return;
    }
    rw_set(w, "Content-Type", "application/json", 16); /* :39 "Content-type" canonicalises to Content-Type */
    obuf* b = &w->body;
    if (!w->wrote_header) rw_write_header(w, 200);
    /* Encode marshals the whole value into its own buffer first and returns the error before touching w: nothing of the
     * body is written, and Respond drops the error (:40 `_ =`) */
    if (r->data_kind == 5 && r->enc_failed) return;
    if (r->raw) {
        /* case resTypes.Raw: resp = v.Data (:25-26) — no envelope, and the error object computed at :20 is not part of
         * the body (the status code it produced was already written at :21).  Raw{} holds a nil interface: "null". */
        if (r->data_kind == 0) ob_puts(b, "null");
        else if (r->data_kind == 1) orc_enc_string(b, r->str, r->str_len);
        else if (r->data_kind == 2) orc_enc_struct(b, r->sc, r->vals);
        else if (r->data_kind == 5) ob_put(b, r->json, r->json_len);
        else ob_puts(b, "{}");
        ob_putc(b, '\n');
        rw_encoded_in_one_write(w);
        return;
    }
    /* json.NewEncoder(w).Encode(response{Error, Data}) :40 ; struct order: error, data; both omitempty on interface */
    ob_putc(b, '{');
    int first = 1;
    if (r->has_err) {
        ob_puts(b, "\"error\":{\"message\":"); /* map[string]interface{}{"message": err.Error()} */
        orc_enc_string(b, r->err_msg, r->err_len);
        ob_putc(b, '}');
        first = 0;
    }
    if (r->data_kind != 0) {
        if (!first) ob_putc(b, ',');
        ob_puts(b, "\"data\":");
        if (r->data_kind == 1) orc_enc_string(b, r->str, r->str_len);
        else if (r->data_kind == 2) orc_enc_struct(b, r->sc, r->vals);
        else if (r->data_kind == 5) ob_put(b, r->json, r->json_len);
        else ob_puts(b, "{}");
    }
    ob_putc(b, '}');
    ob_putc(b, '\n'); /* Encoder.Encode appends a newline */
    rw_encoded_in_one_write(w);
}

/* ------------------------------------------------------------------------------------------------------------ */
/* one request                                                                                                  */
/* ------------------------------------------------------------------------------------------------------------ */

typedef struct {
    uint32_t arena_off;
    uint16_t path_len, query_len;
    uint32_t data_len;
    uint8_t method, flags;
    uint16_t aux;
} req_desc;

static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

/* decode a handler-result row (include/gofr_b200.h) into values; returns 0 or -1 if malformed */
static int decode_row(const orc_schema* sc, const uint8_t* row, size_t n, orc_value* v) {
    size_t fixed = 0;
    for (int i = 0; i < sc->n_fields; i++) fixed += (sc->f[i].kind == F_INT64 || sc->f[i].kind == F_INT) ? 8 : 4;
    if (n < fixed) return -1;
    size_t w = 0, s = fixed;
    for (int i = 0; i < sc->n_fields; i++) {
        memset(&v[i], 0, sizeof v[i]);
        switch (sc->f[i].kind) {
            case F_INT64: case F_INT:
                v[i].i = (int64_t)((uint64_t)rd32(row + w) | (uint64_t)rd32(row + w + 4) << 32);
                w += 8;
                break;
            case F_INT32: v[i].i = (int32_t)rd32(row + w); w += 4; break;
            case F_BOOL: v[i].i = rd32(row + w) != 0; w += 4; break;
            case F_STRING: {
                uint32_t L = rd32(row + w);
                w += 4;
                if (s + L > n) return -1;
                v[i].s = row + s;
                v[i].sn = (int)L;
                s += L;
                break;
            }
        }
    }
    return 0;
}

/* a row of any schema: flat ones go through decode_row + orc_enc_struct (the path the reference pins cover), the wider
 * data model through the row walker of orc_value.c.  fixed / var given separately (RESULT_BOTH interleaves a message). */
static void row_to_result(const orc_table* t, const orc_schema* sc, const uint8_t* fixed, size_t fixed_avail,
                          const uint8_t* var, const uint8_t* end, obuf* json, handler_result* hr) {
    int rc = orc_enc_row(json, t, sc, fixed, fixed_avail, var, end);
    if (rc == -1) { hr->data_kind = -1; return; }
    hr->data_kind = 5;
    hr->enc_failed = rc == -2;
    hr->json = json->p;
    hr->json_len = json->n;
}

static const char HTTP_ERR_MISSING_FILE[] = "http: no such file"; /* net/http.ErrMissingFile.Error() */

static void serve_one(const orc_table* t, const req_desc* d, const uint8_t* id16, const uint8_t* arena,
                      const char* date29, obuf* out, uint32_t* meta) {
    const uint8_t* path = arena + d->arena_off;
    size_t pn = d->path_len;
    const uint8_t* query = path + pn;
    size_t qn = d->query_len;
    const uint8_t* data = arena + ((d->arena_off + pn + qn + 3u) & ~3u);
    size_t dn = d->data_len;
    int method = d->method;
    int is_head = method == 1;

    rw_t w;
    rw_init(&w, t->frame_mode);
    int route_id = 0xFFFF;

    /* ---- mux.Router.ServeHTTP: cleanPath redirect happens before routing and before any middleware ---- */
    obuf cp;
    ob_init(&cp);
    mux_clean_path(path, pn, &cp);
    if (!(cp.n == pn && memcmp(cp.p, path, pn) == 0)) {
        /* url := *req.URL; url.Path = p; w.Header().Set("Location", url.String()); w.WriteHeader(301) */
        obuf loc;
        ob_init(&loc);
        url_escape_path(cp.p, cp.n, &loc);
        if (qn > 0 || (d->flags & 1)) { ob_putc(&loc, '?'); ob_put(&loc, query, qn); }
        rw_set(&w, "Location", loc.p, loc.n);
        rw_write_header(&w, 301);
        ob_free(&loc);
        ob_free(&cp);
        goto finish;
    }
    ob_free(&cp);

    {
        int m = mux_match(t, method, path, pn);
        if (m == MATCH_405) { /* mux methodNotAllowedHandler: w.WriteHeader(405), no middleware */
            rw_write_header(&w, 405);
            goto finish;
        }
        if (m == MATCH_404) { /* http.NotFoundHandler → http.Error(w, "404 page not found", 404) (Go 1.21) */
            rw_set(&w, "Content-Type", "text/plain; charset=utf-8", 25);
            rw_set(&w, "X-Content-Type-Options", "nosniff", 7);
            rw_write_header(&w, 404);
            rw_write(&w, "404 page not found\n", 19);
            goto finish;
        }
        route_id = m;
    }

    {
        const orc_route* r = &t->routes[route_id];
        /* ---- middleware.Tracer: span only.  middleware.Logging (logger.go:46-47): X-Correlation-ID = hex(trace id) */
        char hex[32];
        for (int i = 0; i < 16; i++) { hex[2 * i] = HEXL[id16[i] >> 4]; hex[2 * i + 1] = HEXL[id16[i] & 15]; }
        rw_set(&w, "X-Correlation-Id", hex, 32);
        /* ---- middleware.CORS (cors.go:8-14) ---- */
        rw_set(&w, "Access-Control-Allow-Origin", "*", 1);
        rw_set(&w, "Access-Control-Allow-Methods", "POST, GET, OPTIONS, PUT, DELETE", 31);
        if (method == 7) { /* OPTIONS */
            rw_write_header(&w, 200);
            goto finish;
        }
        /* ---- handler.ServeHTTP (handler.go:32-36): run the closure, Respond(data, err) ---- */
        handler_result hr;
        memset(&hr, 0, sizeof hr);
        obuf tmp, tmp2, json;
        ob_init(&tmp);
        ob_init(&tmp2);
        ob_init(&json);
        orc_value vals[64];
        memset(vals, 0, sizeof vals);
        int n_owned = 0;
        switch (r->hkind) {
            case H_HOST:
                /* closure runs on the host: nothing is emitted; status 0 marks "pending" */
                ob_free(&tmp); ob_free(&tmp2);
                rw_free(&w);
                *meta = 0u | (uint32_t)route_id << 16;
                return;
            case H_STATIC_STRING: hr.data_kind = 1; hr.str = r->s[0]; hr.str_len = (size_t)r->sl[0]; hr.static_body = 1; break;
            case H_STATIC_ERROR: hr.has_err = 1; hr.err_msg = r->s[0]; hr.err_len = (size_t)r->sl[0]; hr.static_body = 1; break;
            case H_NIL: break;
            case H_PARAM_FORMAT: {
                query_get(query, qn, r->s[0], (size_t)r->sl[0], &tmp);
                ob_put(&tmp2, r->s[2], (size_t)r->sl[2]);
                if (tmp.n == 0) ob_put(&tmp2, r->s[1], (size_t)r->sl[1]);
                else ob_put(&tmp2, tmp.p, tmp.n);
                ob_put(&tmp2, r->s[3], (size_t)r->sl[3]);
                hr.data_kind = 1; hr.str = tmp2.p; hr.str_len = tmp2.n;
                break;
            }
            case H_PATHPARAM_FORMAT: {
                /* v := c.PathParam(s0) — mux.Vars(r)[s0], "" when the route has no such variable (request.go:36-38) */
                var_span spans[64];
                memset(spans, 0, sizeof spans);
                tpl_match_from(r, 0, path, pn, 0, spans);
                ob_put(&tmp2, r->s[2], (size_t)r->sl[2]);
                for (int k = 0; k < r->n_pieces; k++)
                    if (r->pieces[k].has_var && strlen(r->pieces[k].name) == (size_t)r->sl[0] &&
                        memcmp(r->pieces[k].name, r->s[0], (size_t)r->sl[0]) == 0)
                        ob_put(&tmp2, path + spans[k].off, spans[k].len);
                ob_put(&tmp2, r->s[3], (size_t)r->sl[3]);
                hr.data_kind = 1; hr.str = tmp2.p; hr.str_len = tmp2.n;
                break;
            }
            case H_ROW: {
                const orc_schema* sc = find_schema(t, r->schema_id);
                if (sc && !orc_schema_is_flat(sc)) {
                    size_t fb = (size_t)orc_schema_fixed_words(t, sc) * 4;
                    row_to_result(t, sc, data, dn, data + (fb < dn ? fb : dn), data + dn, &json, &hr);
                } else if (!sc || decode_row(sc, data, dn, vals) != 0) {
                    /* malformed row from the host shim: not a reference behaviour; both sides answer as a panic */
                    hr.data_kind = -1;
                } else { hr.data_kind = 2; hr.sc = sc; hr.vals = vals; }
                break;
            }
            case H_RESULT: {
                /* stage 2 of the split API: the closure's (data, err) arrives in the data section and
                 * Responder.Respond runs on it (responder.go:19-62) */
                const orc_schema* sc = find_schema(t, r->schema_id);
                uint32_t outcome = 0xFFFFFFFFu;
                if (dn >= 4) memcpy(&outcome, data, 4);
                const uint8_t* rest = data + 4;
                size_t rn = dn >= 4 ? dn - 4 : 0;
                if ((outcome & 0xFFu) >= 6 && (outcome & 0xFFu) <= 8 && (outcome >> 8) <= 2) {
                    /* response.Raw{Data: struct | string | nil}; bits 8..: 0 = err == nil, 1 = some error (500),
                     * 2 = errors.Is(err, http.ErrMissingFile) (404).  The error only picks the status. */
                    const uint32_t kind = outcome & 0xFFu, es = outcome >> 8;
                    hr.raw = 1;
                    if (es) { hr.has_err = 1; hr.err_is_missing_file = es == 2; hr.err_msg = (const uint8_t*)""; hr.err_len = 0; }
                    if (kind == 6 && sc && !orc_schema_is_flat(sc)) {
                        size_t fb = (size_t)orc_schema_fixed_words(t, sc) * 4;
                        row_to_result(t, sc, rest, rn, rest + (fb < rn ? fb : rn), rest + rn, &json, &hr);
                    } else if (kind == 6) {
                        if (!sc || decode_row(sc, rest, rn, vals) != 0) hr.data_kind = -1;
                        else { hr.data_kind = 2; hr.sc = sc; hr.vals = vals; }
                    } else if (kind == 7) {
                        uint32_t len = 0;
                        if (rn >= 4) memcpy(&len, rest, 4);
                        if (rn < 4 || (uint64_t)len + 4 > rn) { hr.data_kind = -1; break; }
                        hr.data_kind = 1; hr.str = rest + 4; hr.str_len = len;
                    }
                    break;
                }
                if (outcome == 0 && sc && !orc_schema_is_flat(sc)) {
                    size_t fb = (size_t)orc_schema_fixed_words(t, sc) * 4;
                    row_to_result(t, sc, rest, rn, rest + (fb < rn ? fb : rn), rest + rn, &json, &hr);
                } else if (outcome == 0) {
                    if (!sc || decode_row(sc, rest, rn, vals) != 0) hr.data_kind = -1;
                    else { hr.data_kind = 2; hr.sc = sc; hr.vals = vals; }
                } else if (outcome == 1 || outcome == 3) {
                    uint32_t len = 0;
                    if (rn >= 4) memcpy(&len, rest, 4);
                    if (rn < 4 || (uint64_t)len + 4 > rn) { hr.data_kind = -1; break; }
                    hr.has_err = 1; hr.err_msg = rest + 4; hr.err_len = len;
                    hr.err_is_missing_file = outcome == 3;
                } else if (outcome == 4) {
                    /* (data, err): one row = [message length word][schema fixed words][message bytes][string bytes] */
                    size_t fixed = 4;
                    if (sc) fixed += (size_t)orc_schema_fixed_words(t, sc) * 4;
                    uint32_t mlen = 0;
                    if (rn >= 4) memcpy(&mlen, rest, 4);
                    if (!sc || rn < fixed || fixed + (uint64_t)mlen > rn) { hr.data_kind = -1; break; }
                    if (!orc_schema_is_flat(sc)) {
                        row_to_result(t, sc, rest + 4, fixed - 4, rest + fixed + mlen, rest + rn, &json, &hr);
                        if (hr.data_kind == 5) { hr.has_err = 1; hr.err_msg = rest + fixed; hr.err_len = mlen; }
                        break;
                    }
                    /* the struct's words follow the length word, its strings follow the message bytes: present them to
                     * decode_row as an ordinary row */
                    uint8_t* tmp_row = (uint8_t*)malloc(rn);
                    memcpy(tmp_row, rest + 4, fixed - 4);
                    memcpy(tmp_row + fixed - 4, rest + fixed + mlen, rn - fixed - mlen);
                    if (decode_row(sc, tmp_row, rn - 4 - mlen, vals) != 0) { free(tmp_row); hr.data_kind = -1; break; }
                    ob_put(&tmp2, tmp_row, rn - 4 - mlen);
                    free(tmp_row);
                    decode_row(sc, tmp2.p, tmp2.n, vals); /* vals must point into memory that outlives this block */
                    hr.has_err = 1; hr.err_msg = rest + fixed; hr.err_len = mlen;
                    hr.data_kind = 2; hr.sc = sc; hr.vals = vals;
                } else if (outcome == 5) {
                    /* data is a Go string: Respond marshals response{Data: "…"} (responder.go:59-62) */
                    uint32_t len = 0;
                    if (rn >= 4) memcpy(&len, rest, 4);
                    if (rn < 4 || (uint64_t)len + 4 > rn) { hr.data_kind = -1; break; }
                    hr.data_kind = 1; hr.str = rest + 4; hr.str_len = len;
                } else if (outcome != 2) hr.data_kind = -1;
                break;
            }
            case H_BIND_ECHO: {
                const orc_schema* sc = find_schema(t, r->schema_id);
                if (!sc) { hr.data_kind = -1; break; }
                if (orc_unmarshal_struct(sc, data, dn, vals, &tmp) != 0) {
                    hr.has_err = 1; hr.err_msg = tmp.p; hr.err_len = tmp.n;
                } else { hr.data_kind = 2; hr.sc = sc; hr.vals = vals; }
                n_owned = sc->n_fields;
                break;
            }
            case H_HEALTH: hr.data_kind = 3; break;
            case H_MISSING_FILE:
                hr.has_err = 1; hr.err_is_missing_file = 1;
                hr.err_msg = (const uint8_t*)HTTP_ERR_MISSING_FILE; hr.err_len = sizeof HTTP_ERR_MISSING_FILE - 1;
                break;
            case H_FILE:
                hr.data_kind = 4; hr.file = r->blob; hr.file_len = (size_t)r->blob_len;
                hr.file_ct = r->s[0]; hr.file_ct_len = (size_t)r->sl[0];
                break;
            case H_PANIC: hr.data_kind = -1; break;
        }
        if (hr.data_kind == -1) {
            /* middleware.panicRecovery (logger.go:91-114): 500 + map{code,message,status} (keys sorted) */
            rw_write_header(&w, 500);
            rw_write(&w, "{\"code\":500,\"message\":\"Some unexpected error has occurred\",\"status\":\"ERROR\"}\n", 77);
        } else {
            respond(&w, &hr);
        }
        for (int i = 0; i < n_owned; i++) free(vals[i].owned);
        ob_free(&tmp);
        ob_free(&tmp2);
        ob_free(&json);
    }

finish:
    rw_finish(&w, is_head, date29, out);
    *meta = (uint32_t)w.status | (uint32_t)route_id << 16;
    rw_free(&w);
}

typedef struct {
    const orc_table* t;
    const uint8_t* desc;
    const uint8_t* ids;
    const uint8_t* arena;
    const char* date29;
    uint32_t lo, hi;
    uint8_t* out;
    uint64_t out_base, out_cap;
    uint32_t* out_off;
    uint32_t* meta;
    int rc;
    uint64_t end;
} shard;

static void* shard_run(void* arg) {
    shard* s = (shard*)arg;
    obuf b;
    ob_init(&b);
    uint64_t pos = s->out_base;
    for (uint32_t i = s->lo; i < s->hi; i++) {
        req_desc d;
        memcpy(&d, s->desc + (size_t)i * 16, 16);
        b.n = 0;
        serve_one(s->t, &d, s->ids + (size_t)i * 16, s->arena, s->date29, &b, &s->meta[i]);
        if (pos + b.n > s->out_base + s->out_cap) { s->rc = -1; break; }
        memcpy(s->out + pos, b.p, b.n);
        s->out_off[i] = (uint32_t)pos;
        pos += b.n;
    }
    s->end = pos;
    ob_free(&b);
    return NULL;
}

int orc_serve(const orc_table* t, const void* desc, const uint8_t* ids, const uint8_t* arena, uint32_t n,
              const char* date29, uint8_t* out, uint64_t out_cap, uint32_t* out_off, uint32_t* meta, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > n && n > 0) nthreads = (int)n;
    shard* sh = (shard*)calloc((size_t)nthreads, sizeof(shard));
    pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
    uint64_t slice = out_cap / (uint64_t)nthreads;
    for (int k = 0; k < nthreads; k++) {
        sh[k] = (shard){t, (const uint8_t*)desc, ids, arena, date29, (uint32_t)((uint64_t)n * k / nthreads),
                        (uint32_t)((uint64_t)n * (k + 1) / nthreads), out, slice * (uint64_t)k, slice, out_off, meta, 0, 0};
        if (nthreads == 1) shard_run(&sh[k]);
        else pthread_create(&th[k], NULL, shard_run, &sh[k]);
    }
    int rc = 0;
    for (int k = 0; k < nthreads; k++) {
        if (nthreads > 1) pthread_join(th[k], NULL);
        if (sh[k].rc) rc = -1;
    }
    /* single thread: packed; out_off[n] = total.  multi thread: out_off[n] = end of the last slice's data */
    out_off[n] = (uint32_t)sh[nthreads - 1].end;
    free(sh);
    free(th);
    return rc;
}

/* ------------------------------------------------------------------------------------------------------------ */
/* unit-level entry points                                                                                      */
/* ------------------------------------------------------------------------------------------------------------ */

static int emit(obuf* b, uint8_t* out, int cap) {
    int n = (int)b->n;
    if (n > cap) { ob_free(b); return -1000000; }
    if (n) memcpy(out, b->p, (size_t)n);
    ob_free(b);
    return n;
}

int orc_json_string(const uint8_t* s, int n, uint8_t* out, int cap) {
    obuf b; ob_init(&b); orc_enc_string(&b, s, (size_t)n); return emit(&b, out, cap);
}
int orc_json_int(int64_t v, uint8_t* out, int cap) { obuf b; ob_init(&b); orc_enc_int(&b, v); return emit(&b, out, cap); }
int orc_clean_path(const uint8_t* p, int n, uint8_t* out, int cap) {
    obuf b; ob_init(&b); mux_clean_path(p, (size_t)n, &b); return emit(&b, out, cap);
}
int orc_query_get(const uint8_t* q, int qn, const uint8_t* key, int kn, uint8_t* out, int cap) {
    obuf b; ob_init(&b); query_get(q, (size_t)qn, key, (size_t)kn, &b); return emit(&b, out, cap);
}
int orc_escape_path(const uint8_t* p, int n, uint8_t* out, int cap) {
    obuf b; ob_init(&b); url_escape_path(p, (size_t)n, &b); return emit(&b, out, cap);
}

int orc_bind(const orc_table* t, int schema_id, const uint8_t* body, int n, uint8_t* row_out, int cap) {
    const orc_schema* sc = find_schema(t, schema_id);
    if (!sc) return -1000001;
    orc_value vals[64];
    memset(vals, 0, sizeof vals);
    obuf err, row;
    ob_init(&err);
    ob_init(&row);
    int rc = orc_unmarshal_struct(sc, body, (size_t)n, vals, &err);
    int ret;
    if (rc != 0) {
        ret = (int)err.n <= cap ? -(int)err.n : -1000000;
        if ((int)err.n <= cap) memcpy(row_out, err.p, err.n);
    } else {
        for (int i = 0; i < sc->n_fields; i++) {
            uint8_t w[8];
            uint64_t u = (uint64_t)vals[i].i;
            if (sc->f[i].kind == F_STRING) u = (uint64_t)vals[i].sn;
            for (int k = 0; k < 8; k++) w[k] = (uint8_t)(u >> (8 * k));
            ob_put(&row, w, (sc->f[i].kind == F_INT64 || sc->f[i].kind == F_INT || sc->f[i].kind == F_FLOAT64) ? 8 : 4);
        }
        for (int i = 0; i < sc->n_fields; i++)
            if (sc->f[i].kind == F_STRING) ob_put(&row, vals[i].s, (size_t)vals[i].sn);
        ret = (int)row.n <= cap ? (int)row.n : -1000000;
        if ((int)row.n <= cap) memcpy(row_out, row.p, row.n);
    }
    for (int i = 0; i < sc->n_fields; i++) free(vals[i].owned);
    ob_free(&err);
    ob_free(&row);
    return ret;
}

/* json.Marshal(RPCLog{...}) — pkg/gofr/grpc/log.go:15-25; golden at pkg/gofr/grpc/log_test.go:28 */
int orc_rpclog_string(const char* id, const char* start_time, int64_t response_time, const char* method, uint8_t* out,
                      int cap) {
    obuf b;
    ob_init(&b);
    ob_puts(&b, "{\"id\":");
    orc_enc_string(&b, (const uint8_t*)id, strlen(id));
    ob_puts(&b, ",\"startTime\":");
    orc_enc_string(&b, (const uint8_t*)start_time, strlen(start_time));
    ob_puts(&b, ",\"responseTime\":");
    orc_enc_int(&b, response_time);
    ob_puts(&b, ",\"method\":");
    orc_enc_string(&b, (const uint8_t*)method, strlen(method));
    ob_putc(&b, '}');
    return emit(&b, out, cap);
}

/* net/http appendTime: "Mon, 02 Jan 2006 15:04:05 GMT" */
void orc_format_http_date(int64_t unix_seconds, char out29[29]) {
    static const char days[] = "SunMonTueWedThuFriSat";
    static const char months[] = "JanFebMarAprMayJunJulAugSepOctNovDec";
    time_t tt = (time_t)unix_seconds;
    struct tm g;
    gmtime_r(&tt, &g);
    char tmp[40];
    snprintf(tmp, sizeof tmp, "%.3s, %02d %.3s %04d %02d:%02d:%02d GMT", days + 3 * g.tm_wday, g.tm_mday,
             months + 3 * g.tm_mon, g.tm_year + 1900, g.tm_hour, g.tm_min, g.tm_sec);
    memcpy(out29, tmp, 29);
}

const char* orc_go_kind_name(int kind) {
    switch (kind) {
        case F_INT64: return "int64";
        case F_INT32: return "int32";
        case F_BOOL: return "bool";
        case F_STRING: return "string";
        case F_INT: return "int";
        case F_FLOAT64: return "float64";
    }
    return "?";
}

/* ---- unit-level entry points for the wider data model (orc_value.c) ---- */
int orc_json_float64(double x, uint8_t* out, int cap) {
    char tmp[40];
    int n = orc_float_text(x, tmp);
    if (n > cap) return -1;
    memcpy(out, tmp, (size_t)n);
    return n;
}

int orc_json_float32(float x, uint8_t* out, int cap) {
    char tmp[40];
    int n = orc_float32_text(x, tmp);
    if (n > cap) return -1;
    memcpy(out, tmp, (size_t)n);
    return n;
}

/* the JSON text of one row: bytes written, -1 malformed / too small, -2 not encodable (NaN, Inf) */
int orc_encode_row_json(const orc_table* t, int schema_id, const uint8_t* row, int n, uint8_t* out, int cap) {
    const orc_schema* sc = orc_find_schema(t, schema_id);
    if (!sc) return -1;
    size_t fb = (size_t)orc_schema_fixed_words(t, sc) * 4;
    if (fb > (size_t)n) return -1;
    obuf b;
    ob_init(&b);
    int rc = orc_enc_row(&b, t, sc, row, (size_t)n, row + fb, row + n);
    int ret = rc < 0 ? rc : (b.n > (size_t)cap ? -1 : (int)b.n);
    if (ret > 0) memcpy(out, b.p, b.n);
    ob_free(&b);
    return ret;
}
