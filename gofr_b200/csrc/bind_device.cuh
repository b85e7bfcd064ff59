// bind_device.cuh — Request.Bind on the device (BASELINE config 3).
//
// Replaces Request.Bind / Request.body (pkg/gofr/http/request.go:40-47,58-67; Context.Bind pkg/gofr/context.go:52-54):
// io.ReadAll + json.Unmarshal(body, &i) with i holding a *struct of string / int / bool fields.  The arithmetic is Go
// 1.21 encoding/json (stdlib, go.mod:3), restated:
//   pass 1  bind_scan()    — checkValid: the byte-at-a-time scanner; a syntax error aborts before anything is stored
//                            and its text ("invalid character 'x' after object key", …) becomes the 500 body;
//   pass 2  bind_decode()  — object members in order; key matched exactly, then case-insensitively; unknown keys
//                            skipped; later duplicates win; null is a no-op; a value of the wrong kind or an integer
//                            that does not fit records the FIRST UnmarshalTypeError and decoding continues.
// Result: a "span row" in per-request scratch (HBM): 8 header words (error description) + the fields in bind layout
// (INT/INT64 two words, INT32 one, BOOL one, STRING two: offset into the body, length | escaped<<31).  The echo
// response program reads it with OP_BSTR; strings without escapes are copied straight from the request body.
// Pins: pkg/gofr/http/request_test.go:17-30, pkg/gofr/context_test.go:23-49 (tests/golden/reference_pins.json).
// Nesting deeper than 64 levels (Go allows 10000) is not decided on the device: the request comes back with status 0
// ("run this one on the host"), exactly like a GOFR_H_HOST route, so no response ever differs from encoding/json's.
#pragma once
#include "serve_device.cuh"

namespace gofr {

enum BindErr : uint32_t { BE_OK = 0, BE_EOF = 1, BE_CHAR = 2, BE_TYPE = 3, BE_DEPTH = 4, BE_DEFER = 5 };  // 4, 5: not decided here
enum BindCtx : uint32_t {
    BC_BEGIN_VALUE, BC_BEGIN_KEY, BC_AFTER_KEY, BC_AFTER_PAIR, BC_AFTER_ELEM, BC_AFTER_TOP, BC_IN_STRING, BC_IN_ESC,
    BC_IN_U, BC_IN_NUM, BC_AFTER_DOT, BC_IN_EXP, BC_TRUE_R, BC_TRUE_U, BC_TRUE_E, BC_FALSE_A, BC_FALSE_L, BC_FALSE_S,
    BC_FALSE_E, BC_NULL_U, BC_NULL_L, BC_COUNT
};
enum BindVal : uint32_t { BV_STRING, BV_NUMBER, BV_NUMBER_LIT, BV_BOOL, BV_OBJECT, BV_ARRAY };

// header words of a span row
enum { BR_ERR = 0, BR_CHAR = 1, BR_CTX = 2, BR_VALUE = 3, BR_FIELD = 4, BR_LIT_OFF = 5, BR_LIT_LEN = 6, BR_PAD = 7, BR_FIELDS = 8 };

GOFR_HD const char* bind_ctx_text(uint32_t ctx) {
    switch (ctx) {
        case BC_BEGIN_VALUE: return "looking for beginning of value";
        case BC_BEGIN_KEY: return "looking for beginning of object key string";
        case BC_AFTER_KEY: return "after object key";
        case BC_AFTER_PAIR: return "after object key:value pair";
        case BC_AFTER_ELEM: return "after array element";
        case BC_AFTER_TOP: return "after top-level value";
        case BC_IN_STRING: return "in string literal";
        case BC_IN_ESC: return "in string escape code";
        case BC_IN_U: return "in \\u hexadecimal character escape";
        case BC_IN_NUM: return "in numeric literal";
        case BC_AFTER_DOT: return "after decimal point in numeric literal";
        case BC_IN_EXP: return "in exponent of numeric literal";
        case BC_TRUE_R: return "in literal true (expecting 'r')";
        case BC_TRUE_U: return "in literal true (expecting 'u')";
        case BC_TRUE_E: return "in literal true (expecting 'e')";
        case BC_FALSE_A: return "in literal false (expecting 'a')";
        case BC_FALSE_L: return "in literal false (expecting 'l')";
        case BC_FALSE_S: return "in literal false (expecting 's')";
        case BC_FALSE_E: return "in literal false (expecting 'e')";
        case BC_NULL_U: return "in literal null (expecting 'u')";
        default: return "in literal null (expecting 'l')";
    }
}

GOFR_HD bool js_space(uint32_t c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n'; }
GOFR_HD bool js_hex(uint32_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'); }
GOFR_HD bool js_digit(uint32_t c) { return c >= '0' && c <= '9'; }

// scanner states
enum : uint32_t {
    SS_BEGIN_VALUE_OR_EMPTY, SS_BEGIN_VALUE, SS_BEGIN_STRING_OR_EMPTY, SS_BEGIN_STRING, SS_END_VALUE, SS_END_TOP,
    SS_IN_STRING, SS_ESC, SS_U0, SS_U1, SS_U2, SS_U3, SS_NEG, SS_1, SS_0, SS_DOT, SS_DOT0, SS_E, SS_ESIGN, SS_E0,
    SS_T, SS_TR, SS_TRU, SS_F, SS_FA, SS_FAL, SS_FALS, SS_N, SS_NU, SS_NUL
};

// json.checkValid.  Returns BE_OK, or the error kind with *e_char / *e_ctx filled.
GOFR_HD_NOINLINE uint32_t bind_scan(const uint8_t* s, uint32_t n, uint32_t* e_char, uint32_t* e_ctx) {
    uint32_t st = SS_BEGIN_VALUE;
    uint64_t stack = 0;  // bit = 1: array, 0: object; innermost at bit 0
    uint32_t depth = 0;
    bool key_pending = false;  // innermost object: the next string is a key (parseObjectKey)
    // The object state (key vs value) is tracked per level in a second bit stack.
    uint64_t kstack = 0;
    bool end_top = false;
    uint32_t i = 0;
    uint32_t c = 0;
    // one extra iteration with c = ' ' models scanner.eof()
    for (;;) {
        bool at_eof = i >= n;
        if (at_eof) {
            if (end_top) return BE_OK;
            c = ' ';
        } else c = s[i];
        bool again;  // re-dispatch the same byte in a new state (Go: "return stateX(s, c)")
        do {
            again = false;
            switch (st) {
                case SS_BEGIN_VALUE_OR_EMPTY:
                    if (js_space(c)) break;
                    if (c == ']') { st = SS_END_VALUE; again = true; break; }
                    st = SS_BEGIN_VALUE; again = true; break;
                case SS_BEGIN_VALUE:
                    if (js_space(c)) break;
                    if (c == '{' || c == '[') {
                        if (depth == 64) { return BE_DEPTH; }
                        stack = stack << 1 | (c == '[' ? 1u : 0u);
                        kstack = kstack << 1 | 1u;  // object: expecting a key
                        depth++;
                        st = c == '{' ? SS_BEGIN_STRING_OR_EMPTY : SS_BEGIN_VALUE_OR_EMPTY;
                        break;
                    }
                    if (c == '"') { st = SS_IN_STRING; break; }
                    if (c == '-') { st = SS_NEG; break; }
                    if (c == '0') { st = SS_0; break; }
                    if (c == 't') { st = SS_T; break; }
                    if (c == 'f') { st = SS_F; break; }
                    if (c == 'n') { st = SS_N; break; }
                    if (c >= '1' && c <= '9') { st = SS_1; break; }
                    *e_char = c; *e_ctx = BC_BEGIN_VALUE; return BE_CHAR;
                case SS_BEGIN_STRING_OR_EMPTY:
                    if (js_space(c)) break;
                    if (c == '}') { kstack &= ~1ull; st = SS_END_VALUE; again = true; break; }  // parseObjectValue
                    st = SS_BEGIN_STRING; again = true; break;
                case SS_BEGIN_STRING:
                    if (js_space(c)) break;
                    if (c == '"') { st = SS_IN_STRING; break; }
                    *e_char = c; *e_ctx = BC_BEGIN_KEY; return BE_CHAR;
                case SS_END_VALUE:
                    if (depth == 0) { st = SS_END_TOP; end_top = true; again = true; break; }
                    if (js_space(c)) break;
                    if (stack & 1) {  // array
                        if (c == ',') { st = SS_BEGIN_VALUE; break; }
                        if (c == ']') { stack >>= 1; kstack >>= 1; depth--; if (depth == 0) { st = SS_END_TOP; end_top = true; } break; }
                        *e_char = c; *e_ctx = BC_AFTER_ELEM; return BE_CHAR;
                    }
                    if (kstack & 1) {  // just read a key
                        if (c == ':') { kstack &= ~1ull; st = SS_BEGIN_VALUE; break; }
                        *e_char = c; *e_ctx = BC_AFTER_KEY; return BE_CHAR;
                    }
                    if (c == ',') { kstack |= 1ull; st = SS_BEGIN_STRING; break; }
                    if (c == '}') { stack >>= 1; kstack >>= 1; depth--; if (depth == 0) { st = SS_END_TOP; end_top = true; } break; }
                    *e_char = c; *e_ctx = BC_AFTER_PAIR; return BE_CHAR;
                case SS_END_TOP:
                    if (!js_space(c)) { *e_char = c; *e_ctx = BC_AFTER_TOP; return BE_CHAR; }
                    break;
                case SS_IN_STRING:
                    if (c == '"') { st = SS_END_VALUE; break; }
                    if (c == '\\') { st = SS_ESC; break; }
                    if (c < 0x20) { *e_char = c; *e_ctx = BC_IN_STRING; return BE_CHAR; }
                    break;
                case SS_ESC:
                    if (c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't' || c == '\\' || c == '/' || c == '"') { st = SS_IN_STRING; break; }
                    if (c == 'u') { st = SS_U0; break; }
                    *e_char = c; *e_ctx = BC_IN_ESC; return BE_CHAR;
                case SS_U0: case SS_U1: case SS_U2: case SS_U3:
                    if (js_hex(c)) { st = st == SS_U3 ? SS_IN_STRING : st + 1; break; }
                    *e_char = c; *e_ctx = BC_IN_U; return BE_CHAR;
                case SS_NEG:
                    if (c == '0') { st = SS_0; break; }
                    if (c >= '1' && c <= '9') { st = SS_1; break; }
                    *e_char = c; *e_ctx = BC_IN_NUM; return BE_CHAR;
                case SS_1:
                    if (js_digit(c)) break;
                    st = SS_0; again = true; break;
                case SS_0:
                    if (c == '.') { st = SS_DOT; break; }
                    if (c == 'e' || c == 'E') { st = SS_E; break; }
                    st = SS_END_VALUE; again = true; break;
                case SS_DOT:
                    if (js_digit(c)) { st = SS_DOT0; break; }
                    *e_char = c; *e_ctx = BC_AFTER_DOT; return BE_CHAR;
                case SS_DOT0:
                    if (js_digit(c)) break;
                    if (c == 'e' || c == 'E') { st = SS_E; break; }
                    st = SS_END_VALUE; again = true; break;
                case SS_E:
                    if (c == '+' || c == '-') { st = SS_ESIGN; break; }
                    st = SS_ESIGN; again = true; break;
                case SS_ESIGN:
                    if (js_digit(c)) { st = SS_E0; break; }
                    *e_char = c; *e_ctx = BC_IN_EXP; return BE_CHAR;
                case SS_E0:
                    if (js_digit(c)) break;
                    st = SS_END_VALUE; again = true; break;
#define GOFR_LIT_STEP(S, WANT, NEXT, CTX) \
                case S: if (c == WANT) { st = NEXT; break; } *e_char = c; *e_ctx = CTX; return BE_CHAR;
                GOFR_LIT_STEP(SS_T, 'r', SS_TR, BC_TRUE_R)
                GOFR_LIT_STEP(SS_TR, 'u', SS_TRU, BC_TRUE_U)
                GOFR_LIT_STEP(SS_TRU, 'e', SS_END_VALUE, BC_TRUE_E)
                GOFR_LIT_STEP(SS_F, 'a', SS_FA, BC_FALSE_A)
                GOFR_LIT_STEP(SS_FA, 'l', SS_FAL, BC_FALSE_L)
                GOFR_LIT_STEP(SS_FAL, 's', SS_FALS, BC_FALSE_S)
                GOFR_LIT_STEP(SS_FALS, 'e', SS_END_VALUE, BC_FALSE_E)
                GOFR_LIT_STEP(SS_N, 'u', SS_NU, BC_NULL_U)
                GOFR_LIT_STEP(SS_NU, 'l', SS_NUL, BC_NULL_L)
                GOFR_LIT_STEP(SS_NUL, 'l', SS_END_VALUE, BC_NULL_L)
#undef GOFR_LIT_STEP
                default: break;
            }
        } while (again);
        if (at_eof) return end_top ? BE_OK : BE_EOF;  // eof(): one ' ' was stepped; still not at the top → unexpected end
        i++;
    }
    (void)key_pending;
}

// ---- decode helpers (input known valid) ----
GOFR_HD uint32_t bd_skip_ws(const uint8_t* s, uint32_t n, uint32_t i) {
    while (i < n && js_space(s[i])) i++;
    return i;
}
#if GOFR_TU_VALUES
// end (exclusive) of the string starting at the quote s[i]
GOFR_HD uint32_t bd_skip_string(const uint8_t* s, uint32_t i) {
    i++;
    while (s[i] != '"') { if (s[i] == '\\') i++; i++; }
    return i + 1;
}
// end (exclusive) of the value starting at i.  Not recursive here: a recursive device function grows its stack at run
// time, beyond the per-thread size ptxas records for the kernel, and the VALUES instances' frames (1008 bytes packed,
// 1104 slot layout) leave less than one call's 48 bytes under the 1 KB default limit — an H100 reported an illegal
// memory access on the first Bind-echo request of a table with float64 members.  The default instances (frames of 480
// bytes) keep the recursive form below: the loop changed their register allocation and cost the packed kernel 2.4 %.
GOFR_HD_NOINLINE uint32_t bd_skip_value(const uint8_t* s, uint32_t n, uint32_t i) {
    uint32_t c = s[i];
    if (c == '"') return bd_skip_string(s, i);
    if (c == '{' || c == '[') {
        uint32_t depth = 0;
        for (;;) {
            uint32_t x = s[i];
            if (x == '"') { i = bd_skip_string(s, i); continue; }
            if (x == '{' || x == '[') depth++;
            if (x == '}' || x == ']') { depth--; if (depth == 0) return i + 1; }
            i++;
        }
    }
#else
// end (exclusive) of the value starting at i
GOFR_HD uint32_t bd_skip_value(const uint8_t* s, uint32_t n, uint32_t i) {
    uint32_t c = s[i];
    if (c == '"') {
        i++;
        while (s[i] != '"') { if (s[i] == '\\') i++; i++; }
        return i + 1;
    }
    if (c == '{' || c == '[') {
        uint32_t depth = 0;
        for (;;) {
            uint32_t x = s[i];
            if (x == '"') { i = bd_skip_value(s, n, i); continue; }
            if (x == '{' || x == '[') depth++;
            if (x == '}' || x == ']') { depth--; if (depth == 0) return i + 1; }
            i++;
        }
    }
#endif
    while (i < n) {
        uint32_t x = s[i];
        if (x == ',' || x == '}' || x == ']' || js_space(x)) break;
        i++;
    }
    return i;
}

GOFR_HD uint32_t bd_hex4(const uint8_t* s) {
    uint32_t v = 0;
    for (int k = 0; k < 4; k++) {
        uint32_t c = s[k];
        v = v << 4 | (c <= '9' ? c - '0' : (c | 0x20) - 'a' + 10);
    }
    return v;
}

// Decode the next rune of a JSON string's contents [i, e) as json.unquoteBytes does: escapes, surrogate pairs,
// invalid UTF-8 → U+FFFD.  Returns the rune, advances *i.
GOFR_HD uint32_t bd_next_rune(const uint8_t* s, uint32_t e, uint32_t* i) {
    uint32_t c = s[*i];
    if (c == '\\') {
        uint32_t x = s[*i + 1];
        *i += 2;
        switch (x) {
            case 'b': return '\b';
            case 'f': return '\f';
            case 'n': return '\n';
            case 'r': return '\r';
            case 't': return '\t';
            case 'u': {
                uint32_t r = bd_hex4(s + *i);
                *i += 4;
                if (r >= 0xD800 && r < 0xE000) {
                    if (*i + 6 <= e && s[*i] == '\\' && s[*i + 1] == 'u') {
                        uint32_t r2 = bd_hex4(s + *i + 2);
                        if (r < 0xDC00 && r2 >= 0xDC00 && r2 < 0xE000) { *i += 6; return ((r - 0xD800) << 10 | (r2 - 0xDC00)) + 0x10000; }
                    }
                    return 0xFFFD;
                }
                return r;
            }
            default: return x;  // " \ /
        }
    }
    if (c < 0x80) { *i += 1; return c; }
    uint32_t L = utf8_len_at(s + *i, e - *i);
    if (!L) { *i += 1; return 0xFFFD; }
    uint32_t r = L == 2 ? (c & 0x1F) : L == 3 ? (c & 0x0F) : (c & 0x07);
    for (uint32_t k = 1; k < L; k++) r = r << 6 | (s[*i + k] & 0x3F);
    *i += L;
    return r;
}

GOFR_HD uint32_t bd_fold(uint32_t r) {
    if (r >= 'A' && r <= 'Z') return r + 32;
    if (r == 0x212A) return 'k';
    if (r == 0x017F) return 's';
    return r;
}

// key (raw JSON string contents [ks, ke)) == name (plain UTF-8), exactly or under simple folding
GOFR_HD bool bd_key_matches(const uint8_t* s, uint32_t ks, uint32_t ke, const uint8_t* name, uint32_t nn, bool fold) {
    uint32_t i = ks, j = 0;
    while (i < ke && j < nn) {
        uint32_t a = bd_next_rune(s, ke, &i);
        uint32_t b;
        uint32_t c = name[j];
        if (c < 0x80) { b = c; j++; }
        else {
            uint32_t L = utf8_len_at(name + j, nn - j);
            if (!L) { b = 0xFFFD; j++; }
            else {
                b = L == 2 ? (c & 0x1F) : L == 3 ? (c & 0x0F) : (c & 0x07);
                for (uint32_t k = 1; k < L; k++) b = b << 6 | (name[j + k] & 0x3F);
                j += L;
            }
        }
        if (fold) { a = bd_fold(a); b = bd_fold(b); }
        if (a != b) return false;
    }
    return i == ke && j == nn;
}

// strconv.ParseInt(lit, 10, 64) on a valid JSON number literal
GOFR_HD bool bd_parse_int(const uint8_t* s, uint32_t n, int64_t* out) {
    uint32_t i = 0;
    bool neg = n && s[0] == '-';
    if (neg) i = 1;
    if (i >= n) return false;
    uint64_t v = 0;
    for (; i < n; i++) {
        uint32_t d = s[i] - '0';
        if (d > 9) return false;
        if (v > (0xFFFFFFFFFFFFFFFFull - d) / 10) return false;
        v = v * 10 + d;
    }
    if (neg) { if (v > (1ull << 63)) return false; *out = (int64_t)(0 - v); }
    else { if (v > 0x7FFFFFFFFFFFFFFFull) return false; *out = (int64_t)v; }
    return true;
}

// strconv.ParseFloat(lit, 64) on a valid JSON number literal, for float64 targets (literalStore, reflect.Float64).
// ParseFloat rounds correctly; what is decided here is the part of the input space where one IEEE operation does too
// (Clinger's exact cases, the same ones strconv's atof64exact takes first): at most 19 significant digits that fit 53
// bits, times or divided by an exactly representable power of ten (|exponent| <= 22, or up to 37 when the digits leave
// room).  Sure overflows (>= 1e310: UnmarshalTypeError "number <literal>", ErrRange) and sure underflows (< 1e-329:
// ±0, not an error in Go) are decided as well.  Everything else — long mantissas, large exponents, subnormals — is
// PF_DEFER: the request goes to the host like a body nested deeper than 64 levels, never to a differently rounded value.
// Between the two sits the Eisel-Lemire step (below), which settles nearly everything else: what is left for the host are
// exact half-way literals, subnormals, values within a decade of the overflow threshold, and literals with more than 19
// digits whose cut-off matters.
enum : uint32_t { PF_OK = 0, PF_OVERFLOW = 1, PF_DEFER = 2 };
GOFR_HD uint32_t bd_parse_float(const uint8_t* s, uint32_t n, uint64_t* bits);
#if GOFR_TU_VALUES  // defined (tables included) only where float64 members exist: the other translation units' modules keep their layout

// ---- the Eisel-Lemire step (strconv/eisel_lemire.go eiselLemire64; D. Lemire, "Number Parsing at a Gigabyte per
// Second"): what ParseFloat tries when the exact cases above do not apply.  man x 10^exp10 with a 128-bit (if need be 192-bit)
// product against a table of normalised powers of ten (el_tables.inc, generated with exact integers by
// scratch/gen/el_tables.py); it either yields the correctly rounded float64 or says it cannot tell (half-way cases, the
// subnormal and overflow ranges) — then Go falls back to its big-decimal slow path, and this code to the host. ----
#define EL_TABLE(name, n) static const uint64_t name##_host[n][2]
#include "el_tables.inc"
#undef EL_TABLE
#if defined(__CUDACC__)
#define EL_TABLE(name, n) static __device__ const uint64_t name##_dev[n][2]
#include "el_tables.inc"
#undef EL_TABLE
#endif
GOFR_HD const uint64_t* el_pow10(int32_t exp10) {  // -348 <= exp10 <= 347
#if defined(__CUDA_ARCH__)
    return EL_POW10_dev[exp10 + 348];
#else
    return EL_POW10_host[exp10 + 348];
#endif
}
GOFR_HD bool bd_eisel_lemire(uint64_t man, int64_t exp10, uint64_t* bits) {
    if (man == 0) { *bits = 0; return true; }
    if (exp10 < -348 || exp10 > 347) return false;
    const int clz = clz64(man);
    man <<= clz;
    uint64_t ret_exp2 = (uint64_t)(((217706 * exp10) >> 16) + 64 + 1023) - (uint64_t)clz;
    const uint64_t* pw = el_pow10((int32_t)exp10);
    uint64_t x_hi, x_lo = umul128(man, pw[1], &x_hi);
    if ((x_hi & 0x1FFu) == 0x1FFu && x_lo + man < man) {  // the 128-bit product may be one too low: add the next 64 bits
        uint64_t y_hi;
        const uint64_t y_lo = umul128(man, pw[0], &y_hi);
        uint64_t m_hi = x_hi;
        const uint64_t m_lo = x_lo + y_hi;
        if (m_lo < x_lo) m_hi++;
        if ((m_hi & 0x1FFu) == 0x1FFu && m_lo + 1 == 0 && y_lo + man < man) return false;
        x_hi = m_hi; x_lo = m_lo;
    }
    const uint64_t msb = x_hi >> 63;
    uint64_t ret_man = x_hi >> (msb + 9);  // 54 bits
    ret_exp2 -= 1 ^ msb;
    if (x_lo == 0 && (x_hi & 0x1FFu) == 0 && (ret_man & 3u) == 1) return false;  // exactly half-way: cannot tell
    ret_man += ret_man & 1;
    ret_man >>= 1;
    if (ret_man >> 53) { ret_man >>= 1; ret_exp2 += 1; }
    if (ret_exp2 - 1 >= 0x7FFull - 1) return false;  // subnormal or overflow: not decided here
    *bits = ret_exp2 << 52 | (ret_man & 0x000FFFFFFFFFFFFFull);
    return true;
}

GOFR_HD uint32_t bd_parse_float(const uint8_t* s, uint32_t n, uint64_t* bits) {
    uint32_t i = 0;
    const bool neg = n && s[0] == '-';
    if (neg) i = 1;
    uint64_t mant = 0;
    int32_t nd = 0;      // significant digits held in mant (<= 19)
    int64_t exp10 = 0;   // value = mant [+ dropped digits] x 10^exp10
    bool nonzero = false, trunc = false;
    for (; i < n && js_digit(s[i]); i++) {
        const uint32_t d = s[i] - '0';
        if (!nonzero && d == 0) continue;
        nonzero = true;
        if (nd < 19) { mant = mant * 10 + d; nd++; }
        else { trunc |= d != 0; exp10++; }
    }
    if (i < n && s[i] == '.') {
        for (i++; i < n && js_digit(s[i]); i++) {
            const uint32_t d = s[i] - '0';
            if (!nonzero && d == 0) { exp10--; continue; }
            nonzero = true;
            if (nd < 19) { mant = mant * 10 + d; nd++; exp10--; }
            else trunc |= d != 0;
        }
    }
    if (i < n && (s[i] | 0x20u) == 'e') {
        i++;
        bool eneg = false;
        if (i < n && (s[i] == '+' || s[i] == '-')) { eneg = s[i] == '-'; i++; }
        int64_t e = 0;
        for (; i < n && js_digit(s[i]); i++) if (e < 1000000) e = e * 10 + (s[i] - '0');
        exp10 += eneg ? -e : e;
    }
    const uint64_t sign = neg ? 0x8000000000000000ull : 0ull;
    if (mant == 0) { *bits = sign; return PF_OK; }
    // (with dropped digits the value lies in (mant, mant + 1) x 10^exp10 of the 19-digit mantissa: keep that scale)
    while (!trunc && mant % 10 == 0) { mant /= 10; exp10++; nd--; }
    const int64_t lead = exp10 + nd - 1;  // 10^lead <= |value| < 10^(lead + 1), dropped digits included
    if (lead >= 310) return PF_OVERFLOW;
    if (lead <= -330) { *bits = sign; return PF_OK; }
    // everything the exact cases below do not take: Eisel-Lemire; with dropped digits the value lies between mant and
    // mant + 1 — if both round to the same float64, that is the answer (strconv.atof64 does exactly this)
    auto approx = [&]() -> uint32_t {
        uint64_t f = 0, f_up = 0;
        if (!bd_eisel_lemire(mant, exp10, &f)) return PF_DEFER;
        if (trunc && (!bd_eisel_lemire(mant + 1, exp10, &f_up) || f_up != f)) return PF_DEFER;
        *bits = f | sign;
        return PF_OK;
    };
    if (trunc || (mant >> 53) != 0) return approx();
    double x = (double)(int64_t)mant;
    if (exp10 > 22) {
        if (exp10 > 22 + 15) return approx();
        uint64_t p = 1;
        for (int64_t k = 22; k < exp10; k++) p *= 10;
        if (mant > ((1ull << 53) - 1) / p) return approx();
        x = (double)(int64_t)(mant * p);
        exp10 = 22;
    } else if (exp10 < -22) return approx();
    double p10 = 1.0;  // 10^k is a double for k <= 22, so every partial product is exact
    for (int64_t k = exp10 < 0 ? -exp10 : exp10; k > 0; k--) p10 *= 10.0;
    x = exp10 < 0 ? x / p10 : x * p10;
#if defined(__CUDA_ARCH__)
    const uint64_t b = (uint64_t)__double_as_longlong(x);
#else
    uint64_t b;
    memcpy(&b, &x, 8);
#endif
    *bits = b | sign;
    return PF_OK;
}

#endif  // GOFR_TU_VALUES

// d.object / d.literalStore into the span row.  `row` has BR_FIELDS + bind-layout words, zero-initialised here.
// VO: whether this instance knows float64 members.  A Bind schema with one makes its echo program PF_VALUES (OP_F64), so
// such tables only ever run the VALUES instances of the serve kernels (serve_device.cuh GOFR_TU_VALUES) — the default
// instances keep exactly the code, registers and spills they had before float64 targets existed.
template <bool VO = (GOFR_TU_VALUES != 0)>
GOFR_HD_NOINLINE void bind_decode(const TableView tv, uint32_t schema_idx, const uint8_t* s, uint32_t n, uint32_t* row) {
    const SchemaRec S = tv.schemas()[schema_idx];
    const FieldRec* F = (const FieldRec*)(tv.base + S.fields_off);
    // bind layout: word offsets
    uint32_t nwords = 0;
    for (uint32_t k = 0; k < S.n_fields; k++) nwords += (F[k].kind == GOFR_F_INT32 || F[k].kind == GOFR_F_BOOL) ? 1 : 2;
    for (uint32_t k = 0; k < BR_FIELDS + nwords; k++) row[k] = 0;
    bool saved = false, deferred = false;
    auto type_error = [&](uint32_t value, uint32_t field, uint32_t lo, uint32_t ll) {
        if (saved) return;
        saved = true;
        row[BR_ERR] = BE_TYPE; row[BR_VALUE] = value; row[BR_FIELD] = field; row[BR_LIT_OFF] = lo; row[BR_LIT_LEN] = ll;
    };
    uint32_t i = bd_skip_ws(s, n, 0);
    uint32_t c = s[i];
    if (c != '{') {
        if (c == '[') type_error(BV_ARRAY, 0xFFFFFFFFu, 0, 0);
        else if (c == '"') type_error(BV_STRING, 0xFFFFFFFFu, 0, 0);
        else if (c == 't' || c == 'f') type_error(BV_BOOL, 0xFFFFFFFFu, 0, 0);
        else if (c != 'n') type_error(BV_NUMBER, 0xFFFFFFFFu, 0, 0);
        return;  // null: the local interface is set to nil, the caller's struct is untouched
    }
    i = bd_skip_ws(s, n, i + 1);
    if (s[i] == '}') return;
    for (;;) {
        i = bd_skip_ws(s, n, i);
        uint32_t ke = bd_skip_value(s, n, i);
        uint32_t ks = i + 1;
        uint32_t kend = ke - 1;  // contents are [ks, kend)
        i = bd_skip_ws(s, n, ke) + 1;  // ':'
        i = bd_skip_ws(s, n, i);
        // exact name first, then fold, both in declaration order
        uint32_t fi = 0xFFFFFFFFu;
        for (uint32_t k = 0; k < S.n_fields && fi == 0xFFFFFFFFu; k++)
            if (bd_key_matches(s, ks, kend, tv.lits() + F[k].name_off, F[k].name_len, false)) fi = k;
        for (uint32_t k = 0; k < S.n_fields && fi == 0xFFFFFFFFu; k++)
            if (bd_key_matches(s, ks, kend, tv.lits() + F[k].name_off, F[k].name_len, true)) fi = k;
        uint32_t vs = i, ve = bd_skip_value(s, n, i);
        i = ve;
        if (fi != 0xFFFFFFFFu) {
            uint32_t w = BR_FIELDS;
            for (uint32_t k = 0; k < fi; k++) w += (F[k].kind == GOFR_F_INT32 || F[k].kind == GOFR_F_BOOL) ? 1 : 2;
            const uint32_t kind = F[fi].kind;
            uint32_t vc = s[vs];
            if (vc == '{') type_error(BV_OBJECT, fi, 0, 0);
            else if (vc == '[') type_error(BV_ARRAY, fi, 0, 0);
            else if (vc == 'n') { /* null into string/int/bool: no-op */ }
            else if (vc == 't' || vc == 'f') {
                if (kind == GOFR_F_BOOL) row[w] = vc == 't';
                else type_error(BV_BOOL, fi, 0, 0);
            } else if (vc == '"') {
                if (kind != GOFR_F_STRING) type_error(BV_STRING, fi, 0, 0);
                else {
                    const uint8_t* p = s + vs + 1;
                    uint32_t len = ve - vs - 2;
                    // "escaped": anything encoding/json would not copy verbatim on the way out, or a backslash on the
                    // way in (0x5C is in the special set), or non-ASCII (needs UTF-8 validation)
                    bool esc = json_needs_escape<false>(p, len);
                    row[w] = vs + 1;
                    row[w + 1] = len | (esc ? 0x80000000u : 0u);
                }
            } else {  // number
                bool is_float = false;
                if constexpr (VO) is_float = kind == GOFR_F_FLOAT64;
                if (kind == GOFR_F_STRING || kind == GOFR_F_BOOL) type_error(BV_NUMBER, fi, 0, 0);
                else if (is_float) {
                    if constexpr (VO) {
                        uint64_t fb = 0;
                        const uint32_t pf = bd_parse_float(s + vs, ve - vs, &fb);
                        if (pf == PF_DEFER) deferred = true;
                        else if (pf == PF_OVERFLOW) type_error(BV_NUMBER_LIT, fi, vs, ve - vs);
                        else { row[w] = (uint32_t)fb; row[w + 1] = (uint32_t)(fb >> 32); }
                    }
                } else {
                    int64_t x;
                    bool ok = bd_parse_int(s + vs, ve - vs, &x);
                    if (ok && kind == GOFR_F_INT32 && (x < -2147483648ll || x > 2147483647ll)) ok = false;
                    if (!ok) type_error(BV_NUMBER_LIT, fi, vs, ve - vs);
                    else if (kind == GOFR_F_INT32) row[w] = (uint32_t)(int32_t)x;
                    else { row[w] = (uint32_t)x; row[w + 1] = (uint32_t)((uint64_t)x >> 32); }
                }
            }
        }
        i = bd_skip_ws(s, n, i);
        uint32_t d = s[i++];
        if (d == '}') break;
    }
    // a literal this code cannot round with certainty decides the whole request: whatever else was stored or recorded,
    // encoding/json on the host has the last word
    if (VO && deferred) row[BR_ERR] = BE_DEFER;
}

// Full Bind of one request body into `row`.  Returns true when the struct can be echoed.
template <bool VO>
GOFR_HD_NOINLINE bool bind_request(const TableView tv, uint32_t schema_idx, const uint8_t* body, uint32_t n, uint32_t* row) {
    uint32_t ech = 0, ectx = 0;
    uint32_t e = bind_scan(body, n, &ech, &ectx);
    if (e != BE_OK) {
        row[BR_ERR] = e; row[BR_CHAR] = ech; row[BR_CTX] = ectx;
        return false;
    }
    bind_decode<VO>(tv, schema_idx, body, n, row);
    return row[BR_ERR] == BE_OK;
}

// ---- string transcoder: JSON-escaped input → decoded runes → encoding/json-escaped output ----
template <bool EMIT>
GOFR_HD_NOINLINE uint32_t bind_string_slow(Writer* w, const uint8_t* s, uint32_t len) {
    uint32_t out = 0, i = 0;
    while (i < len) {
        uint32_t r = bd_next_rune(s, len, &i);
        uint8_t u[4];
        uint32_t L;
        if (r < 0x80) { u[0] = (uint8_t)r; L = 1; }
        else if (r < 0x800) { u[0] = (uint8_t)(0xC0 | r >> 6); u[1] = (uint8_t)(0x80 | (r & 0x3F)); L = 2; }
        else if (r < 0x10000) { u[0] = (uint8_t)(0xE0 | r >> 12); u[1] = (uint8_t)(0x80 | ((r >> 6) & 0x3F)); u[2] = (uint8_t)(0x80 | (r & 0x3F)); L = 3; }
        else { u[0] = (uint8_t)(0xF0 | r >> 18); u[1] = (uint8_t)(0x80 | ((r >> 12) & 0x3F)); u[2] = (uint8_t)(0x80 | ((r >> 6) & 0x3F)); u[3] = (uint8_t)(0x80 | (r & 0x3F)); L = 4; }
        // a \u escape may decode to a surrogate-free but otherwise arbitrary rune; lone surrogates became U+FFFD above,
        // so u[] is always valid UTF-8 and the encoder's rules apply to it directly
        out += json_escape_slow<EMIT>(w, u, L);
    }
    return out;
}

// ---- string decoder for the Bind stage of the split API (gofr_bind_device): JSON-escaped input → the Go string's bytes
//      (what json.Unmarshal stores: escapes resolved, invalid UTF-8 and lone surrogates replaced by U+FFFD) ----
template <bool EMIT>
GOFR_HD_NOINLINE uint32_t bind_string_raw(Writer* w, const uint8_t* s, uint32_t len) {
    uint32_t out = 0, i = 0;
    while (i < len) {
        const uint32_t r = bd_next_rune(s, len, &i);
        if (EMIT) w->reserve_out(2);
        if (r < 0x80) { if (EMIT) w->put1(r); out += 1; }
        else if (r < 0x800) { if (EMIT) w->putk((0xC0 | r >> 6) | (0x80 | (r & 0x3F)) << 8, 2); out += 2; }
        else if (r < 0x10000) { if (EMIT) w->putk((0xE0 | r >> 12) | (0x80 | ((r >> 6) & 0x3F)) << 8 | (0x80 | (r & 0x3F)) << 16, 3); out += 3; }
        else { if (EMIT) w->put4((0xF0 | r >> 18) | (0x80 | ((r >> 12) & 0x3F)) << 8 | (0x80 | ((r >> 6) & 0x3F)) << 16 | (0x80 | (r & 0x3F)) << 24); out += 4; }
    }
    return out;
}

// ---- err.Error() of a failed Bind; RAW == false: JSON-escaped (it is emitted inside {"error":{"message":"…"}}),
//      RAW == true: the text itself (gofr_bind_device hands it to the host closure) ----
template <bool EMIT, bool RAW = false>
GOFR_HD uint32_t be_put(Writer* w, const uint8_t* p, uint32_t n) {  // append a short plain piece
    if (!RAW) return json_escape_slow<EMIT>(w, p, n);
    if (EMIT) for (uint32_t i = 0; i < n; i++) w->put1(p[i]);
    return n;
}
template <bool EMIT, bool RAW = false>
GOFR_HD uint32_t be_puts(Writer* w, const char* z) {
    uint32_t n = 0;
    while (z[n]) n++;
    return be_put<EMIT, RAW>(w, (const uint8_t*)z, n);
}

template <bool EMIT, bool RAW>
GOFR_HD_NOINLINE uint32_t emit_bind_error(Writer* w, const TableView tv, uint32_t schema_idx, const uint8_t* body, const uint32_t* row) {
    uint32_t out = 0;
    const uint32_t err = row[BR_ERR];
    if (err == BE_EOF) return be_puts<EMIT, RAW>(w, "unexpected end of JSON input");
    if (err == BE_DEPTH) return be_puts<EMIT, RAW>(w, "exceeded max depth");
    if (err == BE_CHAR) {
        out += be_puts<EMIT, RAW>(w, "invalid character ");
        // json.quoteChar
        uint32_t c = row[BR_CHAR];
        uint8_t q[8];
        uint32_t k = 0;
        q[k++] = '\'';
        if (c == '\'') { q[k++] = '\\'; q[k++] = '\''; }
        else if (c == '"') { q[k++] = '"'; }
        else if (c == '\\') { q[k++] = '\\'; q[k++] = '\\'; }
        else if (c >= 0x20 && c < 0x7F) q[k++] = (uint8_t)c;
        else if (c >= 0xA1 && c != 0xAD) { q[k++] = (uint8_t)(0xC0 | c >> 6); q[k++] = (uint8_t)(0x80 | (c & 0x3F)); }  // printable Latin-1
        else {
            q[k++] = '\\';
            const char* sh = c == 7 ? "a" : c == 8 ? "b" : c == 12 ? "f" : c == 10 ? "n" : c == 13 ? "r" : c == 9 ? "t" : c == 11 ? "v" : nullptr;
            if (sh) q[k++] = (uint8_t)sh[0];
            else if (c < 0x80) { q[k++] = 'x'; q[k++] = (uint8_t)hex_lc(c >> 4); q[k++] = (uint8_t)hex_lc(c & 15); }
            else { q[k++] = 'u'; q[k++] = '0'; q[k++] = '0'; q[k++] = (uint8_t)hex_lc(c >> 4); q[k++] = (uint8_t)hex_lc(c & 15); }
        }
        out += be_put<EMIT, RAW>(w, q, k);
        out += be_puts<EMIT, RAW>(w, "' ");
        out += be_puts<EMIT, RAW>(w, bind_ctx_text(row[BR_CTX]));
        return out;
    }
    // UnmarshalTypeError
    const SchemaRec S = tv.schemas()[schema_idx];
    const FieldRec* F = (const FieldRec*)(tv.base + S.fields_off);
    out += be_puts<EMIT, RAW>(w, "json: cannot unmarshal ");
    const uint32_t v = row[BR_VALUE];
    out += be_puts<EMIT, RAW>(w, v == BV_STRING ? "string" : v == BV_BOOL ? "bool" : v == BV_OBJECT ? "object" : v == BV_ARRAY ? "array"
                                                       : v == BV_NUMBER ? "number" : "number ");
    if (v == BV_NUMBER_LIT) out += be_put<EMIT, RAW>(w, body + row[BR_LIT_OFF], row[BR_LIT_LEN]);
    const uint8_t* ty = tv.lits() + S.type_off;  // NUL-terminated reflect.Type.String()
    uint32_t tl = 0, dot = 0xFFFFFFFFu;
    while (ty[tl]) { if (ty[tl] == '.') dot = tl; tl++; }
    const uint32_t fi = row[BR_FIELD];
    if (fi == 0xFFFFFFFFu) {
        out += be_puts<EMIT, RAW>(w, " into Go value of type ");
        out += be_put<EMIT, RAW>(w, ty, tl);
    } else {
        out += be_puts<EMIT, RAW>(w, " into Go struct field ");
        uint32_t ns = dot == 0xFFFFFFFFu ? 0 : dot + 1;  // reflect.Type.Name()
        out += be_put<EMIT, RAW>(w, ty + ns, tl - ns);
        out += be_puts<EMIT, RAW>(w, ".");
        out += be_put<EMIT, RAW>(w, tv.lits() + F[fi].name_off, F[fi].name_len);
        out += be_puts<EMIT, RAW>(w, " of type ");
        out += be_put<EMIT, RAW>(w, tv.lits() + F[fi].type_off, F[fi].type_len);
    }
    return out;
}

// ---------------------------------------------------------------------------------------------------------------
// Bind as a stage of the split API (gofr_bind_device): Context.Bind(&v) for closures that stay on the host
// (pkg/gofr/context.go:52-54 -> pkg/gofr/http/request.go:40-47 -> json.Unmarshal).  One request: its body -> either the
// typed row the closure reads its struct from (GOFR_H_ROW layout: one word per field — two for INT64/INT — then the
// DECODED bytes of the string fields in schema order), or err.Error().  `row` is the span row bind_request filled.
// EMIT == false: only the size.
// ---------------------------------------------------------------------------------------------------------------
template <bool EMIT>
GOFR_HD uint32_t bind_row_out(Writer* w, const TableView tv, uint32_t schema_idx, const uint8_t* body, const uint32_t* row) {
    if (row[BR_ERR] != BE_OK) return emit_bind_error<EMIT, true>(w, tv, schema_idx, body, row);
    const SchemaRec S = tv.schemas()[schema_idx];
    const FieldRec* F = (const FieldRec*)(tv.base + S.fields_off);
    uint32_t out = 0, wi = BR_FIELDS;
    // fixed part
    for (uint32_t f = 0; f < S.n_fields; f++) {
        const uint32_t kind = F[f].kind;
        if (EMIT) w->reserve_out(2);
        if (kind == GOFR_F_INT64 || kind == GOFR_F_INT || kind == GOFR_F_FLOAT64) { if (EMIT) { w->put4(row[wi]); w->put4(row[wi + 1]); } out += 8; wi += 2; }
        else if (kind == GOFR_F_STRING) {
            const uint32_t lenw = row[wi + 1], len = lenw & 0x7FFFFFFFu;
            const uint32_t dl = (lenw >> 31) ? bind_string_raw<false>(nullptr, body + row[wi], len) : len;
            if (EMIT) w->put4(dl);
            out += 4; wi += 2;
        } else { if (EMIT) w->put4(row[wi]); out += 4; wi += 1; }  // INT32, BOOL
    }
    // string bytes
    wi = BR_FIELDS;
    for (uint32_t f = 0; f < S.n_fields; f++) {
        const uint32_t kind = F[f].kind;
        if (kind == GOFR_F_STRING) {
            const uint32_t lenw = row[wi + 1], len = lenw & 0x7FFFFFFFu;
            if (lenw >> 31) out += bind_string_raw<EMIT>(w, body + row[wi], len);
            else { if (EMIT && len) emit_bytes(*w, body + row[wi], len); out += len; }
            wi += 2;
        } else wi += (kind == GOFR_F_INT64 || kind == GOFR_F_INT || kind == GOFR_F_FLOAT64) ? 2 : 1;
    }
    return out;
}

// status words of gofr_bind_device (include/gofr_b200.h GOFR_BIND_*)
GOFR_HD uint32_t bind_row_status(const uint32_t* row) { return row[BR_ERR] == BE_OK ? 0u : (row[BR_ERR] == BE_DEPTH || row[BR_ERR] == BE_DEFER) ? 2u : 1u; }

}  // namespace gofr
