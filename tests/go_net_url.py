"""An independent model of the Go code that copies request bytes into a response or a log line: net/url's unescaping and
query parsing, path.Clean and mux's cleanPath, the Location of mux's 301, strings.TrimSpace and GoFr's getIPAddress, and
encoding/json's string encoder over arbitrary bytes — TEST INFRASTRUCTURE ONLY.

Written from Go 1.21's published sources (net/url/url.go, path/path.go, strings/strings.go, unicode/tables.go,
encoding/json/encode.go), gorilla/mux v1.8.1 (mux.go) and GoFr (pkg/gofr/http/request.go, middleware/logger.go).  It does
not read oracle/ or gofr_b200/csrc/, and it uses no Python URL, path or Unicode library for its answers: Python's
urllib, posixpath and str.isspace each differ from Go on inputs the tests send (tests/test_request_text.py plants them).
Everything works on bytes.
"""
from __future__ import annotations

from tests.go_unmarshal import decode_rune

ENCODE_PATH, ENCODE_QUERY_COMPONENT = "encodePath", "encodeQueryComponent"


# ---------------------------------------------------------------------------------------------------------------
# net/url: unescape, ParseQuery, Values.Get
# ---------------------------------------------------------------------------------------------------------------
def _ishex(c: int) -> bool:
    return 0x30 <= c <= 0x39 or 0x61 <= c <= 0x66 or 0x41 <= c <= 0x46


def _unhex(c: int) -> int:
    return c - 0x30 if c <= 0x39 else (c | 0x20) - 0x61 + 10


def unescape(s: bytes, mode: str):
    """url.unescape(s, mode) for encodePath and encodeQueryComponent: None on an EscapeError.  A '%' needs two hex digits
    after it ("i+2 >= len(s)" is an error, so "%4" and a trailing "%" fail); '+' is a space only in query components."""
    out = bytearray()
    i = 0
    while i < len(s):
        c = s[i]
        if c == 0x25:
            if i + 2 >= len(s) or not _ishex(s[i + 1]) or not _ishex(s[i + 2]):
                return None
            out.append(_unhex(s[i + 1]) << 4 | _unhex(s[i + 2]))
            i += 3
        elif c == 0x2B and mode == ENCODE_QUERY_COMPONENT:
            out.append(0x20)
            i += 1
        else:
            out.append(c)
            i += 1
    return bytes(out)


def query_unescape(s: bytes):
    """url.QueryUnescape"""
    return unescape(s, ENCODE_QUERY_COMPONENT)


def parse_query(q: bytes):
    """url.parseQuery: [(key, value)] in order.  strings.Cut on '&'; a pair containing ';' is skipped (an error is
    recorded, parsing goes on); an empty pair is skipped; strings.Cut on the first '='; a key or value whose
    QueryUnescape fails skips that pair."""
    pairs = []
    rest = q
    while rest:
        key, sep, rest = rest.partition(b"&")
        if b";" in key or key == b"":
            continue
        k, _, v = key.partition(b"=")
        k, v = query_unescape(k), query_unescape(v)
        if k is None or v is None:
            continue
        pairs.append((k, v))
    return pairs


def values_get(pairs, key: bytes) -> bytes:
    """url.Values.Get: the FIRST value stored for key, "" when there is none"""
    for k, v in pairs:
        if k == key:
            return v
    return b""


def query_param(raw_query: bytes, key: bytes) -> bytes:
    """ctx.Param(key) = req.URL.Query().Get(key) (pkg/gofr/http/request.go): Query() ignores ParseQuery's error"""
    return values_get(parse_query(raw_query), key)


# ---------------------------------------------------------------------------------------------------------------
# path.Clean, mux cleanPath, the 301's Location
# ---------------------------------------------------------------------------------------------------------------
def path_clean(p: bytes) -> bytes:
    """path.Clean with its lazybuf: the write index w over a copy, `dotdot` the index a ".." may not back up past"""
    if p == b"":
        return b"."
    rooted = p[0] == 0x2F
    n = len(p)
    out = bytearray()
    r, dotdot = 0, 0
    if rooted:
        out.append(0x2F)
        r, dotdot = 1, 1
    while r < n:
        if p[r] == 0x2F:                                                   # empty path element
            r += 1
        elif p[r] == 0x2E and (r + 1 == n or p[r + 1] == 0x2F):           # . element
            r += 1
        elif p[r] == 0x2E and p[r + 1] == 0x2E and (r + 2 == n or p[r + 2] == 0x2F):   # .. element: remove to last /
            r += 2
            if len(out) > dotdot:                 # out.w--; back up while out.index(out.w) != '/'
                w = len(out) - 1
                while w > dotdot and out[w] != 0x2F:
                    w -= 1
                del out[w:]
            elif not rooted:                                               # cannot backtrack, but not rooted: append ..
                if out:
                    out.append(0x2F)
                out += b".."
                dotdot = len(out)
        else:                                                              # real path element: add slash if needed
            if (rooted and len(out) != 1) or (not rooted and len(out) != 0):
                out.append(0x2F)
            while r < n and p[r] != 0x2F:
                out.append(p[r])
                r += 1
    return bytes(out) if out else b"."


def clean_path(p: bytes) -> bytes:
    """mux cleanPath: "" → "/"; a leading "/" is added; path.Clean; the trailing slash is put back unless the result is "/" """
    if p == b"":
        return b"/"
    if p[0] != 0x2F:
        p = b"/" + p
    np_ = path_clean(p)
    if p[-1] == 0x2F and np_ != b"/":
        np_ += b"/"
    return np_


def redirects(path: bytes) -> bool:
    """Router.ServeHTTP: `if p := cleanPath(path); p != path` → 301 (skipClean and useEncodedPath are off in GoFr)"""
    return clean_path(path) != path


_UNRESERVED = frozenset(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789-_.~")
_RESERVED = frozenset(b"$&+,/:;=?@")


def should_escape_path(c: int) -> bool:
    """shouldEscape(c, encodePath): alphanumerics and -_.~ stay; of the reserved $&+,/:;=?@ only '?' is escaped in a
    path; everything else (control bytes, space, !"#%'()*<>[\\]^`{|}, DEL, bytes >= 0x80) is escaped"""
    if c in _UNRESERVED:
        return False
    if c in _RESERVED:
        return c == 0x3F
    return True


def escape_path(p: bytes) -> bytes:
    """url.escape(p, encodePath): %XX with upper-case hex for every byte shouldEscape names"""
    return b"".join(b"%%%02X" % c if should_escape_path(c) else bytes([c]) for c in p)


def escaped_location(path: bytes, raw_query: bytes, force_query: bool) -> bytes:
    """The Location mux sets: `url := *req.URL; url.Path = cleanPath(path); url.String()` for an origin-form request (no
    scheme, host or user; url.String writes EscapedPath, then "?" + RawQuery when RawQuery != "" or ForceQuery).

    EscapedPath would return RawPath only if unescape(RawPath, encodePath) == Path.  RawPath is kept from the request, and
    setPath stored it only when unescape(RawPath) equalled the request's Path; the redirect happens exactly when the
    cleaned path differs from that Path, so the test fails and EscapedPath is escape(cleanPath(path), encodePath) — never
    the request's own spelling, whatever escapes the client used.  The cleaned path starts with "/", so url.String's "./"
    prefix for a first segment holding ':' never applies."""
    loc = escape_path(clean_path(path))
    if raw_query or force_query:
        loc += b"?" + raw_query
    return loc


def location_has_expectation(raw_query: bytes) -> bool:
    """net/http never hands mux a RawQuery with an ASCII control byte, DEL or space (url.Parse refuses CTLs; the request
    line is cut at spaces), and its header writer would rewrite CR / LF to spaces and trim the value.  For such a query
    the model states no Location: the oracle alone judges those lines."""
    return not any(c < 0x21 or c == 0x7F for c in raw_query)


# ---------------------------------------------------------------------------------------------------------------
# strings.TrimSpace (unicode.IsSpace) and getIPAddress
# ---------------------------------------------------------------------------------------------------------------
# unicode.IsSpace: '\t', '\n', '\v', '\f', '\r', ' ', U+0085 (NEL), U+00A0 (NBSP) in Latin-1; beyond it the White_Space
# property: U+1680, U+2000..U+200A, U+2028, U+2029, U+202F, U+205F, U+3000.  Not U+001C..U+001F, not U+180E, not U+200B.
WHITE_SPACE = frozenset([0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0, 0x1680] + list(range(0x2000, 0x200B)) +
                        [0x2028, 0x2029, 0x202F, 0x205F, 0x3000])


def is_space(r: int) -> bool:
    return r in WHITE_SPACE


def decode_last_rune(b: bytes):
    """utf8.DecodeLastRune: back up to UTFMax bytes to a byte that can start a rune, decode from there; (0xFFFD, 1) when
    that rune does not end exactly at len(b)"""
    end = len(b)
    if b[end - 1] < 0x80:
        return b[end - 1], 1
    lim = max(end - 4, 0)
    start = end - 1
    while start >= lim:
        if b[start] & 0xC0 != 0x80:      # utf8.RuneStart
            break
        start -= 1
    if start < 0:
        start = 0
    r, size = decode_rune(b, start)
    if start + size != end:
        return 0xFFFD, 1
    return r, size


def trim_space(s: bytes) -> bytes:
    """strings.TrimSpace: TrimLeftFunc with DecodeRune, TrimRightFunc with DecodeLastRune, both on unicode.IsSpace (the
    ASCII fast path gives the same answer).  An invalid byte decodes as U+FFFD, which is not space."""
    i = 0
    while i < len(s):
        r, size = decode_rune(s, i)
        if not is_space(r):
            break
        i += size
    s = s[i:]
    while s:
        r, size = decode_last_rune(s)
        if not is_space(r):
            break
        s = s[:-size]
    return s


def get_ip_address(xff: bytes, remote_addr: bytes) -> bytes:
    """middleware/logger.go getIPAddress: strings.Split(X-Forwarded-For, ",")[0], RemoteAddr when that is "", then
    strings.TrimSpace.  A value that is only spaces is not "" before the trim, so it does not fall back."""
    ip = xff.split(b",")[0]
    if ip == b"":
        ip = remote_addr
    return trim_space(ip)


# ---------------------------------------------------------------------------------------------------------------
# encoding/json string encoder (escapeHTML on), over arbitrary bytes
# ---------------------------------------------------------------------------------------------------------------
_SHORT = {0x22: b'\\"', 0x5C: b"\\\\", 0x0A: b"\\n", 0x0D: b"\\r", 0x09: b"\\t"}
_HEX = b"0123456789abcdef"


def json_string(s: bytes) -> bytes:
    """encodeState.string / appendString with escapeHTML: ASCII outside htmlSafeSet is written as a short escape
    (only \\" \\\\ \\n \\r \\t in Go 1.21, so \\b and \\f are \\u0008 and \\u000c) or \\u00XX with lower-case hex;
    every byte utf8.DecodeRune rejects (size 1, RuneError) becomes one \\ufffd; U+2028 and U+2029 are escaped;
    every other rune, including a well-formed U+FFFD, is copied."""
    out = bytearray(b'"')
    i = 0
    while i < len(s):
        c = s[i]
        if c < 0x80:
            if c in _SHORT:
                out += _SHORT[c]
            elif c < 0x20 or c in (0x3C, 0x3E, 0x26):
                out += b"\\u00" + bytes([_HEX[c >> 4], _HEX[c & 15]])
            else:
                out.append(c)
            i += 1
            continue
        r, size = decode_rune(s, i)
        if r == 0xFFFD and size == 1:
            out += b"\\ufffd"
        elif r in (0x2028, 0x2029):
            out += b"\\u202" + bytes([_HEX[r & 15]])
        else:
            out += s[i:i + size]
        i += size
    out += b'"'
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------
# handler bodies
# ---------------------------------------------------------------------------------------------------------------
def data_body(text: bytes) -> bytes:
    """Respond(string, nil) → json.NewEncoder(w).Encode(response{Data: text}): {"data":"…"} and Encode's newline"""
    return b'{"data":' + json_string(text) + b"}\n"


def param_format_body(raw_query: bytes, key: bytes, default: bytes, prefix: bytes, suffix: bytes) -> bytes:
    """H_PARAM_FORMAT: v := ctx.Param(key); if v == "" { v = default }; fmt.Sprintf(prefix + "%s" + suffix, v)"""
    v = query_param(raw_query, key)
    return data_body(prefix + (v if v else default) + suffix)


def path_param_format_body(value: bytes, prefix: bytes, suffix: bytes) -> bytes:
    """H_PATHPARAM_FORMAT: fmt.Sprintf(prefix + "%s" + suffix, ctx.PathParam(key)) with mux's variable from URL.Path"""
    return data_body(prefix + value + suffix)
