"""json.Unmarshal(body, &v) for v a flat struct (string, int64, int, int32, bool and float64 members), restated from Go
1.21's encoding/json (decode.go, scanner.go, fold.go) and unicode/utf8, unicode/utf16 — not from the project's decoder
(bind_device.cuh) or its C restatement (oracle/orc_bind.c).  The answer is what Context.Bind hands a closure, in the
row format of gofr_bind_device (include/gofr_b200.h):
  GOFR_BIND_OK     one little-endian word per field in schema order (INT64 and INT two, FLOAT64 two holding its bits,
                   INT32 and BOOL one, STRING one holding the byte length), then the string bytes in schema order;
  GOFR_BIND_ERROR  err.Error() of the first UnmarshalTypeError (a syntax error's text is not restated: only its verdict).
The rules, in the order decode.go applies them:
  * Top level.  checkValid runs over the whole document first: a syntax error wins and nothing is stored.  `null` leaves
    the struct zero.  An array, string, number or bool is "json: cannot unmarshal <kind> into Go value of type <pkg.T>".
  * Keys are unquoted like values.  The exact JSON name wins; otherwise the first field in declaration order whose name
    folds to the key's folding.  Folding here is ASCII case plus U+212A KELVIN SIGN ~ k and U+017F LONG S ~ s: Go 1.21's
    foldName maps every rune through unicode.ToUpper(unicode.ToLower(r)), which also folds non-ASCII names (É ~ é) and
    sends U+0130 and U+0131 to I; the project does not, a stated deviation (DESIGN.md) pinned by one known answer in
    tests/test_bind_unmarshal.py.  Unknown keys are skipped with their whole value.  Every occurrence of a key is
    assigned in order, so the last one wins.
  * Values.  null leaves the field as it is.  Int kinds take only integer literals in range (strconv.ParseInt, then
    OverflowInt): anything else is "number <literal>"; "-0" is 0.  A float64 takes strconv.ParseFloat's correctly rounded
    value (Python's float() rounds the same way); a literal past the largest double is "number <literal>" (ErrRange).  A
    kind mismatch names the JSON kind alone: string, number, bool, array or object.  The text is "json: cannot unmarshal
    <what> into Go struct field <T>.<json name> of type <go type>"; the first error is kept and decoding goes on.
  * Strings follow unquote: the escapes \\" \\\\ \\/ \\b \\f \\n \\r \\t \\uXXXX; a \\u surrogate is combined with the \\u
    escape right after it by utf16.DecodeRune, and when that fails it becomes U+FFFD and the next escape is read on its
    own; raw bytes go through utf8.DecodeRune, so an overlong form, a UTF-8-encoded surrogate, a code point past U+10FFFF
    or a truncated sequence gives one U+FFFD per byte it consumes (Python's errors="replace" gives one per maximal
    subpart instead), and a literal U+FFFD stays.
What the device may leave to the host (GOFR_BIND_HOST) is not Go's business, so it is a separate flag, `host_ok`: a body
nested deeper than 64 levels, or a number bound to a float64 member that tests/test_gpu_float_bind.py's Eisel-Lemire
model lets the device defer (defer_reason).  Nowhere else is HOST an answer."""
import json
import math
import struct
from dataclasses import dataclass
from typing import Optional

from gofr_b200 import spec as S

OK, ERROR, HOST = 0, 1, 2
MAX_DEVICE_DEPTH = 64
GO_TYPE = {S.F_INT64: "int64", S.F_INT: "int", S.F_INT32: "int32", S.F_BOOL: "bool", S.F_STRING: "string", S.F_FLOAT64: "float64"}
INT_RANGE = {S.F_INT64: 64, S.F_INT: 64, S.F_INT32: 32}
WS = b" \t\r\n"


@dataclass
class Answer:
    status: int                 # OK or ERROR: what Go answers
    row: Optional[bytes]        # the row or the error text; None for a syntax error (only its verdict is restated)
    host_ok: bool = False       # the device may answer GOFR_BIND_HOST instead


# ---- unicode/utf8.DecodeRune and encoding/json unquote ----
def decode_rune(b: bytes, i: int):
    """utf8.DecodeRune(b[i:]): (rune, size); (0xFFFD, 1) for every invalid or truncated sequence"""
    c = b[i]
    if c < 0x80:
        return c, 1
    if 0xC2 <= c <= 0xDF:
        n, lo, hi, r = 2, 0x80, 0xBF, c & 0x1F
    elif 0xE0 <= c <= 0xEF:
        n, r = 3, c & 0x0F
        lo, hi = (0xA0, 0xBF) if c == 0xE0 else (0x80, 0x9F) if c == 0xED else (0x80, 0xBF)   # no overlongs, no surrogates
    elif 0xF0 <= c <= 0xF4:
        n, r = 4, c & 0x07
        lo, hi = (0x90, 0xBF) if c == 0xF0 else (0x80, 0x8F) if c == 0xF4 else (0x80, 0xBF)   # no overlongs, <= U+10FFFF
    else:
        return 0xFFFD, 1        # 0x80..0xC1 (continuation bytes, overlong 2-byte leads) and 0xF5..0xFF
    if i + n > len(b) or not lo <= b[i + 1] <= hi:
        return 0xFFFD, 1
    r = r << 6 | (b[i + 1] & 0x3F)
    for k in range(2, n):
        if not 0x80 <= b[i + k] <= 0xBF:
            return 0xFFFD, 1
        r = r << 6 | (b[i + k] & 0x3F)
    return r, n


def encode_rune(r: int) -> bytes:
    """utf8.EncodeRune: surrogates and runes past U+10FFFF are written as U+FFFD (never produced below, kept for fidelity)"""
    if 0xD800 <= r < 0xE000 or r > 0x10FFFF:
        r = 0xFFFD
    return chr(r).encode("utf-8")


def _getu4(s: bytes, i: int) -> int:
    """getu4(s[i:]): the \\uXXXX escape at i, or -1"""
    if i + 6 > len(s) or s[i] != 0x5C or s[i + 1] != 0x75 or any(chr(x) not in "0123456789abcdefABCDEF" for x in s[i + 2:i + 6]):
        return -1
    return int(s[i + 2:i + 6].decode("ascii"), 16)


ESC = {0x22: b'"', 0x5C: b"\\", 0x2F: b"/", 0x62: b"\b", 0x66: b"\f", 0x6E: b"\n", 0x72: b"\r", 0x74: b"\t"}


def unquote(s: bytes) -> bytes:
    """unquoteBytes of a valid JSON string's contents (the bytes between its quotes): the Go string's bytes"""
    out = bytearray()
    i = 0
    while i < len(s):
        c = s[i]
        if c == 0x5C:
            e = s[i + 1]
            if e in ESC:
                out += ESC[e]
                i += 2
                continue
            r = _getu4(s, i)
            i += 6
            if 0xD800 <= r < 0xE000:   # utf16.IsSurrogate
                r2 = _getu4(s, i)
                if 0xD800 <= r < 0xDC00 and 0xDC00 <= r2 < 0xE000:   # utf16.DecodeRune succeeds: consume both
                    out += encode_rune(0x10000 + ((r - 0xD800) << 10 | (r2 - 0xDC00)))
                    i += 6
                    continue
                r = 0xFFFD
            out += encode_rune(r)
        elif c < 0x80:
            out.append(c)
            i += 1
        else:
            r, n = decode_rune(s, i)
            out += encode_rune(r)
            i += n
    return bytes(out)


def fold(name: bytes) -> bytes:
    """the key folding this project applies (see the module text): ASCII case, U+212A ~ k, U+017F ~ s"""
    out = bytearray()
    i = 0
    while i < len(name):
        r, n = decode_rune(name, i)
        i += n
        r = 0x6B if r == 0x212A else 0x73 if r == 0x017F else r + 32 if 0x41 <= r <= 0x5A else r
        out += encode_rune(r)
    return bytes(out)


# ---- the document: checkValid's verdict, then its structure with raw string bytes and number texts ----
class SyntaxErr(Exception):
    def __init__(self, pos):
        self.pos = pos


def _verdict(body: bytes):
    """None when the document is valid JSON, else the offset where checkValid stops.  Python's json module decides it on the
    body read as Latin-1 (one character per byte: bytes >= 0x80 are legal inside strings and illegal outside, as in Go's
    scanner); NaN and Infinity, Python extensions, are refused."""
    def refuse(c):
        raise ValueError(c)
    try:
        json.loads(body.decode("latin-1"), parse_constant=refuse)
        return None
    except json.JSONDecodeError as e:
        return e.pos
    except ValueError:   # NaN / Infinity / -Infinity: Go stops at their first letter; the offset only feeds the depth count
        return len(body)
    except RecursionError:
        return -1


def _depth_before(body: bytes, end: int) -> int:
    """the deepest nesting the scanner reaches before offset `end`"""
    depth = best = 0
    in_str = esc = False
    for c in body[:end]:
        if in_str:
            if esc:
                esc = False
            elif c == 0x5C:
                esc = True
            elif c == 0x22:
                in_str = False
        elif c == 0x22:
            in_str = True
        elif c in b"{[":
            depth += 1
            best = max(best, depth)
        elif c in b"}]":
            depth -= 1
    return best


def _skip_ws(b, i):
    while i < len(b) and b[i] in WS:
        i += 1
    return i


def _value(b: bytes, i: int):
    """one value of a valid document at i (no leading space): ((kind, payload), end).  Kinds: object (list of (raw key,
    value) in order, duplicates kept), array, string (raw contents), number (literal text), bool, null."""
    c = b[i]
    if c == 0x7B:
        members = []
        i = _skip_ws(b, i + 1)
        if b[i] == 0x7D:
            return ("object", members), i + 1
        while True:
            (_, key), i = _value(b, i)
            i = _skip_ws(b, i) + 1            # ':'
            v, i = _value(b, _skip_ws(b, i))
            members.append((key, v))
            i = _skip_ws(b, i)
            i += 1
            if b[i - 1] == 0x7D:
                return ("object", members), i
            i = _skip_ws(b, i)
    if c == 0x5B:
        elems = []
        i = _skip_ws(b, i + 1)
        if b[i] == 0x5D:
            return ("array", elems), i + 1
        while True:
            v, i = _value(b, i)
            elems.append(v)
            i = _skip_ws(b, i) + 1
            if b[i - 1] == 0x5D:
                return ("array", elems), i
            i = _skip_ws(b, i)
    if c == 0x22:
        j = i + 1
        while b[j] != 0x22:
            j += 2 if b[j] == 0x5C else 1
        return ("string", b[i + 1:j]), j + 1
    if c == 0x74:
        return ("bool", True), i + 4
    if c == 0x66:
        return ("bool", False), i + 5
    if c == 0x6E:
        return ("null", None), i + 4
    j = i
    while j < len(b) and b[j] in b"+-.0123456789eE":
        j += 1
    return ("number", b[i:j]), j


# ---- d.object / d.literalStore into the struct ----
def _parse_int(lit: bytes, bits: int):
    """strconv.ParseInt(lit, 10, 64) then OverflowInt for `bits`: the value, or None"""
    t = lit[1:] if lit[:1] == b"-" else lit
    if not t or not t.isdigit():
        return None
    v = int(lit)
    return v if -(1 << (bits - 1)) <= v < (1 << (bits - 1)) else None


def unmarshal(schema: S.Schema, body: bytes, float_defer=None) -> Answer:
    """json.Unmarshal(body, &v) with v a zero `schema` struct.  float_defer(lit) -> reason or None says which float64
    literals the device may leave to the host (tests/test_gpu_float_bind.py defer_reason by default)."""
    if float_defer is None:
        from tests.test_gpu_float_bind import defer_reason as float_defer
    stop = _verdict(body)
    if stop is not None:
        deep = stop < 0 or _depth_before(body, stop if stop >= 0 else len(body)) > MAX_DEVICE_DEPTH
        return Answer(ERROR, None, deep)
    doc, _ = _value(body, _skip_ws(body, 0))
    host_ok = _depth_before(body, len(body)) > MAX_DEVICE_DEPTH
    fields = schema.fields
    vals = [b"" if f.kind == S.F_STRING else 0.0 if f.kind == S.F_FLOAT64 else 0 for f in fields]
    err = None
    kind, payload = doc
    if kind != "object":
        if kind != "null":
            err = "json: cannot unmarshal %s into Go value of type %s" % (kind, schema.go_type)
        return _answer(schema, vals, err, host_ok)
    short = schema.go_type.rsplit(".", 1)[-1]
    exact = {}
    folded = {}
    for k, f in enumerate(fields):
        exact.setdefault(f.name.encode(), k)
        folded.setdefault(fold(f.name.encode()), k)
    for raw_key, (vk, v) in payload:
        key = unquote(raw_key)
        k = exact.get(key, folded.get(fold(key)))
        if k is None:
            continue
        f = fields[k]

        def type_error(what):
            return err or "json: cannot unmarshal %s into Go struct field %s.%s of type %s" % (what, short, f.name, GO_TYPE[f.kind])
        if vk == "null":
            continue
        if vk in ("object", "array"):
            err = type_error(vk)
        elif vk == "bool":
            if f.kind == S.F_BOOL:
                vals[k] = int(v)
            else:
                err = type_error("bool")
        elif vk == "string":
            if f.kind == S.F_STRING:
                vals[k] = unquote(v)
            else:
                err = type_error("string")
        elif f.kind in INT_RANGE:
            x = _parse_int(v, INT_RANGE[f.kind])
            if x is None:
                err = type_error("number " + v.decode())
            else:
                vals[k] = x
        elif f.kind == S.F_FLOAT64:
            host_ok = host_ok or float_defer(v) is not None
            x = float(v)
            if math.isinf(x):
                err = type_error("number " + v.decode())
            else:
                vals[k] = x
        else:
            err = type_error("number")
    return _answer(schema, vals, err, host_ok)


def _answer(schema, vals, err, host_ok) -> Answer:
    if err is not None:
        return Answer(ERROR, err.encode(), host_ok)
    return Answer(OK, encode_row(schema, vals), host_ok)


def encode_row(schema: S.Schema, vals) -> bytes:
    """the GOFR_H_ROW layout of a struct's values"""
    words, strs = b"", b""
    for f, v in zip(schema.fields, vals):
        if f.kind in (S.F_INT64, S.F_INT):
            words += struct.pack("<q", v)
        elif f.kind == S.F_FLOAT64:
            words += struct.pack("<d", v)
        elif f.kind == S.F_INT32:
            words += struct.pack("<i", v)
        elif f.kind == S.F_BOOL:
            words += struct.pack("<I", v)
        else:
            words += struct.pack("<I", len(v))
            strs += v
    return words + strs


def decode_row(schema: S.Schema, row: bytes):
    """the values of an OK row: ints, floats, bools, strings as bytes"""
    vals, at, lens = [], 0, []
    for f in schema.fields:
        if f.kind in (S.F_INT64, S.F_INT):
            vals.append(struct.unpack_from("<q", row, at)[0]); at += 8
        elif f.kind == S.F_FLOAT64:
            vals.append(struct.unpack_from("<d", row, at)[0]); at += 8
        elif f.kind == S.F_INT32:
            vals.append(struct.unpack_from("<i", row, at)[0]); at += 4
        elif f.kind == S.F_BOOL:
            vals.append(bool(struct.unpack_from("<I", row, at)[0])); at += 4
        else:
            lens.append((len(vals), struct.unpack_from("<I", row, at)[0])); vals.append(None); at += 4
    for k, n in lens:
        vals[k] = row[at:at + n]
        at += n
    return vals
