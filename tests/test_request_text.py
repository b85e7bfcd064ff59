"""Request bytes that reach a response or a log line, checked three ways on the CPU: the independent model
(tests/go_net_url.py), the oracle, and the device code run by tests/emu at all four output misalignments.

Most bytes the serve kernels write come from the table.  These do not: ctx.Param's query value (url.ParseQuery, Values.Get,
QueryUnescape, then encoding/json), ctx.PathParam's span of the decoded URL.Path, the Location of mux's 301 (cleanPath, then
escape(·, encodePath) and "?" + RawQuery), and the RequestLog's uri, user_agent and ip (strings.Split, strings.TrimSpace).
The corpus below is hostile on purpose — every byte value escaped and raw, broken escapes, UTF-8 split across escapes,
overlongs and surrogates, every White_Space rune, every escape class, string lengths 0-64 at every offset mod 16 and the
worst-case growth of each text — and tests/test_gpu_request_text.py sends the same corpus through the kernels.

The corpus has two shapes.  Host-batch descriptors carry URL.Path and RawQuery directly and may hold any byte, as
gofr_batch_submit accepts them.  Raw HTTP/1.1 messages go through the request-head parser first, so %2E and %2F in a path
are decoded before mux sees it.  For a redirect whose RawQuery holds a control byte, DEL or space — which net/http never
hands mux — the model states no Location (go_net_url.location_has_expectation) and the oracle alone judges that line.
"""
import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200.table import Table
from tests import go_net_url as G
from tests import oracle as O
from tests import test_values as TV
from tests.emu import emu as E

DATE = S.http_date(1_700_000_000)
DATE_TEXT = "Tue, 14 Nov 2023 22:13:20 GMT"
KEY, DEFAULT, PREFIX, SUFFIX = b"name", b"World", b"Hello ", b"!"


# ---------------------------------------------------------------------------------------------------------------
# tables
# ---------------------------------------------------------------------------------------------------------------
def _text_routes():
    return [S.Route(S.M_GET, "/hello", S.H_PARAM_FORMAT, s0=KEY, s1=DEFAULT, s2=PREFIX, s3=SUFFIX),
            S.Route(S.M_GET, "/users/{id}", S.H_PATHPARAM_FORMAT, s0=b"id", s2=b"user ", s3=b"!"),
            S.Route(S.M_GET, "/w/{rest:.*}", S.H_PATHPARAM_FORMAT, s0=b"rest", s2=b"[", s3=b"]")]


def text_spec(mode=S.FRAME_WIRE):
    """ctx.Param and ctx.PathParam handlers, without App.Run's default routes: anything else is mux's 404"""
    return S.TableSpec(frame_mode=mode, default_routes=False, routes=_text_routes())


def wide_spec():
    """only H_PARAM_FORMAT routes of one program shape: the table image_wants_wide_slots accepts"""
    return S.TableSpec(default_routes=False, routes=[
        S.Route(S.M_GET, "/hello", S.H_PARAM_FORMAT, s0=KEY, s1=DEFAULT, s2=PREFIX, s3=SUFFIX),
        S.Route(S.M_GET, "/hi", S.H_PARAM_FORMAT, s0=b"who", s1=b"you", s2=b"Hi ", s3=b".")])


def values_spec():
    """the text routes plus one route of the wider data model: the serve kernels' _values instances run this table"""
    vs = TV._spec(S.FRAME_WIRE, S.H_ROW, [TV.USER])
    return S.TableSpec(default_routes=False, schemas=vs.schemas, routes=_text_routes() + vs.routes)


# ---------------------------------------------------------------------------------------------------------------
# what Go answers (from the model)
# ---------------------------------------------------------------------------------------------------------------
def route_model(path: bytes):
    """mux's regexps for the text routes, on URL.Path: ^/hello$, ^/users/(?P<v0>[^/]+)$ and ^/w/(?P<v0>.*)$ — Go's '.'
    does not match '\\n'; '[^/]' does; both match any invalid byte as U+FFFD"""
    if path == b"/hello":
        return ("param",)
    if path.startswith(b"/users/") and len(path) > 7 and b"/" not in path[7:]:
        return ("path", path[7:], b"user ", b"!")
    if path.startswith(b"/w/") and b"\n" not in path[3:]:
        return ("path", path[3:], b"[", b"]")
    return None


def expect(path: bytes, query: bytes, force: bool, routes=route_model, key=KEY, default=DEFAULT, prefix=PREFIX, suffix=SUFFIX):
    """(status, Location or None, body or None) for a GET of URL.Path `path` with RawQuery `query`"""
    if G.redirects(path):
        return 301, G.escaped_location(path, query, force) if G.location_has_expectation(query) else None, None
    r = routes(path)
    if r is None:
        return 404, None, None
    if r[0] == "param":
        return 200, None, G.param_format_body(query, key, default, prefix, suffix)
    return 200, None, G.path_param_format_body(r[1], r[2], r[3])


def parse_wire(wire: bytes):
    """one HTTP/1.1 response through h11: (status, headers (lower-case names → bytes), body)"""
    import h11
    c = h11.Connection(h11.CLIENT)
    c.send(h11.Request(method="GET", target="/", headers=[("Host", "h")]))
    c.send(h11.EndOfMessage())
    c.receive_data(wire)
    ev = c.next_event()
    assert isinstance(ev, h11.Response), ev
    body = b""
    while True:
        e = c.next_event()
        if isinstance(e, h11.Data):
            body += bytes(e.data)
        elif isinstance(e, h11.EndOfMessage):
            break
        else:
            raise AssertionError(e)
    return ev.status_code, {k.decode().lower(): bytes(v) for k, v in ev.headers}, body


def wire_problem(wire: bytes, want):
    """None when the response is what the model expects: status, Location, Content-Length == body length, body bytes"""
    status, loc, body = want
    try:
        st, hdr, got = parse_wire(wire)
    except Exception as e:                       # noqa: BLE001 — an unparseable response is a finding
        if loc is None and status == 301:
            return None                          # the oracle alone judges a Location the model states nothing about
        return "h11: %r" % e
    if st != status:
        return "status %d, model %d" % (st, status)
    if hdr.get("date") != DATE_TEXT.encode():
        return "date %r" % hdr.get("date")
    if "content-length" in hdr and int(hdr["content-length"]) != len(got):
        return "Content-Length %s, body %d" % (hdr["content-length"], len(got))
    if loc is not None and hdr.get("location") != loc:
        return "Location %r, model %r" % (hdr.get("location", b"")[:200], loc[:200])
    if body is not None and got != body:
        return "body %r, model %r" % (got[:200], body[:200])
    return None


# ---------------------------------------------------------------------------------------------------------------
# the corpus
# ---------------------------------------------------------------------------------------------------------------
# UTF-8 split across escapes, across escaped and raw bytes; overlongs, surrogates, beyond U+10FFFF, lone continuations
UTF8_EDGES = [b"%e2%82%ac", b"%E2%82%AC", b"%e2\x82%ac", b"\xe2%82\xac", b"%e2%82", b"%e2%82x", b"%e2", b"%e2%82%ac%e2%82",
              b"%f0%9f%98%80", b"%f0%9f%98", b"\xf0%9f%98%80", b"%c0%af", b"%c1%bf", b"%e0%80%af", b"%e0%9f%bf", b"%f0%80%80%af",
              b"%f0%8f%bf%bf", b"%ED%A0%80", b"%ed%bf%bf", b"%ed%9f%bf", b"%F4%90%80%80", b"%f4%8f%bf%bf", b"%f5%80%80%80",
              b"%80", b"%bf%80", b"a%80b", b"%fe%ff", b"%c2", b"%c2%20", b"%c2%c2%a0", b"%ef%bf%bd", b"%ef%bf%be",
              b"%e2%80%a8", b"%e2%80%a9", b"%e2%80%a8%e2%80%a9x", b"\xe2\x80\xa8", b"%c2%85", b"%22%3C%3E%26%5C", b'"<>&\\',
              b"%08%0c%0a%0d%09%00%1f%7f", b"\xff", b"\xc3\xa9", b"%c3%a9", b"%C3\xa9"]
# query pairs: + against %2B, ';' inside a pair, empty pairs, a key that needs unescaping, first value invalid or empty
QUERY_EDGES = [b"", b"name", b"name=", b"name=+", b"name=%2B", b"name=a+b%20c", b"name=a;b", b"x=1;name=2&name=3", b"name=a;b&name=c",
               b"&&name=x&", b"=&name=v", b"name&name=v", b"name=&name=ok", b"name=%zz&name=ok", b"name=%&name=ok",
               b"name=%4&name=ok", b"name=ok%", b"name=ok%4", b"name=%", b"nam%=x&name=y", b"name%6=x&name=ok", b"na%6De=v",
               b"na%6de=v&name=w", b"na+me=v&name=w", b"%6e%61%6d%65=enc", b"name=a=b=c", b"Name=x", b"name=x&Name=y",
               b"name=%3B&x", b"name%3D=v&name=w", b"name=1&name=2", b"a=1&b=2&c=3&name=" + b"z" * 300,
               b"name=" + b"%41" * 700, b"name=" + b"\xe2\x82\xac" * 300]
# paths: dot segments, trailing slashes, every escape class of shouldEscape (in redirected paths)
PATH_EDGES = [b"", b"/", b"hello", b"/hello/", b"//hello", b"/hello/.", b"/./hello", b"/hello/..", b"/a/../hello", b"/hello/x/..",
              b"/users/../users/x", b"/users/./x", b"/users/x/../y/", b"/a//b/", b"/a/b/../../..", b"/../../..", b"/..a/..",
              b"/a/.../..//", b"/.", b"/..", b"/a/./././b", b"/users/x/", b"/users/", b"/users//x", b"/w/", b"/w/a/b/c",
              b"/w/a/../b", b"/w/a\nb", b"/w/\n", b"/users/a\nb", b"/users/a b", b"/users/\xff", b"/users/%2F", b"/users/a%2Fb",
              b"//a/b?c", b"/a b//c", b"/\xc3\xa9//", b"/%41//", b"/x/./y/", b"//", b"/hello//"]
WHITE = [b"\t", b"\n", b"\x0b", b"\x0c", b"\r", b" ", b"\xc2\x85", b"\xc2\xa0", b"\xe1\x9a\x80"] + \
    [chr(0x2000 + k).encode() for k in range(11)] + \
    [c.encode() for c in "\u2028\u2029\u202f\u205f\u3000"]
NOT_WHITE = [b"\x1c", b"\x1d", b"\x1e", b"\x1f", b"\x00", b"\xe1\xa0\x8e", b"\xe2\x80\x8b", b"\xef\xbb\xbf", b"\xc2", b"\xe2\x80",
             b"\x85", b"\xa0", b"\xe3\x80", b"\xc2\xc2\xa0"]


def _special(k):
    return [b'"', b"\x01", b"\x80", b"<", b"\\", b"\xe2\x80\xa8", b"\xc3\xa9", b"%22"][k % 8]


def host_corpus():
    """[(label, Req)] in the host-batch shape: URL.Path and RawQuery may hold any byte"""
    out = []
    add = lambda label, p, q=b"", f=0: out.append((label, S.Req(S.M_GET, p, q, flags=f)))
    for b in range(256):
        add("query %%%02X" % b, b"/hello", b"name=%%%02X" % b)
        add("query a%%%02Xb" % b, b"/hello", b"name=a%%%02xb" % b)
        add("query raw %02x" % b, b"/hello", b"name=" + bytes([b]) + b"z")
        add("key raw %02x" % b, b"/hello", bytes([b]) + b"=1&name=" + bytes([b]))
        add("pathvar raw %02x" % b, b"/users/a" + bytes([b]) + b"b")
        add("rest raw %02x" % b, b"/w/" + bytes([b]))
        add("redirect raw %02x" % b, b"//x" + bytes([b]) + b"/", b"q=" + bytes([b]) if b >= 0x21 and b != 0x7F else b"q=1")
    add("redirect every byte", b"/./" + bytes(range(256)), b"k=v")
    add("redirect control query", b"//hello", b"a=\x01\r\n b\x7f")        # the model states no Location
    for e in UTF8_EDGES:
        add("utf8 " + repr(e), b"/hello", b"name=" + e)
        add("utf8 tail " + repr(e), b"/hello", b"name=" + e + b"&name=second")
    for t in (b"%", b"%4", b"%e2%8", b"%e2%82%a"):
        add("truncated value " + repr(t), b"/hello", b"name=ab" + t)
        add("truncated key " + repr(t), b"/hello", b"name" + t + b"=x&name=y")
    for q in QUERY_EDGES:
        add("pairs " + repr(q[:40]), b"/hello", q)
    for p in PATH_EDGES:
        for q, f in ((b"", 0), (b"x=1&y=%41", 0), (b"", S.REQ_FORCE_QUERY), (b"a=\xc3\xa9", 0)):
            add("path " + repr(p), p, q, f)
    for c in range(256):                          # every class of shouldEscape, in a redirected path
        add("escape class %02x" % c, b"/a/./" + bytes([c]) + b"z")
    # lengths 0..64 at every offset mod 16 (the lead and keep masks of json_needs_escape): the value starts k bytes later
    for L in range(65):
        for k in range(16):
            clean = b"".join(bytes([0x61 + (i * 7 + L) % 26]) for i in range(L))
            add("len %d off %d" % (L, k), b"/hello", b"&" * k + b"name=" + clean)
            if L:
                at = (L * 5 + k) % L
                s = clean[:at] + _special(L + k) + clean[at + 1:]
                add("len %d off %d special" % (L, k), b"/hello", b"&" * k + b"name=" + s)
                add("pathvar len %d off %d" % (L, k), b"/users/" + b"x" * k + s.replace(b"/", b"_"))
    # worst-case growth of each text
    add("growth <", b"/hello", b"name=" + b"<" * 7995)
    add("growth %00", b"/hello", b"name=" + b"%00" * 2665)
    add("growth invalid", b"/hello", b"name=" + b"%ff" * 2665)
    add("growth redirect", b"//" + b"\xff" * 8000, b"")
    add("growth redirect query", b"/./" + b"\x01" * 6000, b"q=" + b"y" * 2000)
    add("growth pathvar", b"/users/" + b"\x01" * 8000)
    return out


def host_batch(spec_corpus=None):
    c = host_corpus() if spec_corpus is None else spec_corpus
    return S.RequestBatch.pack([r for _, r in c], seed=0x7E57), [lab for lab, _ in c]


def host_expect(req: S.Req):
    return expect(req.path, req.query, bool(req.flags & S.REQ_FORCE_QUERY))


# ---- raw HTTP/1.1 messages (the connection path) ----
def raw_corpus():
    """[(label, target, user_agent, x_forwarded_for)]: targets in the parser's subset (no '//' start, printable ASCII)"""
    out = []
    for b in range(256):
        out.append(("query %%%02X" % b, b"/hello?name=%%%02X" % b))
        out.append(("pathvar %%%02X" % b, b"/users/a%%%02Xb" % b))
    for e in UTF8_EDGES:
        if all(0x21 <= c <= 0x7E and c != 0x23 for c in e):
            out.append(("utf8 " + repr(e), b"/hello?name=" + e))
            out.append(("pathvar utf8 " + repr(e), b"/users/" + e))
    for t in (b"/a/%2E%2E/hello", b"/a/%2e%2e/hello/", b"/%2E/hello", b"/hello/%2E", b"/hello%2F..", b"/users/a%2Fb", b"/users/%2F",
              b"/w/a%2Fb", b"/w/%0A", b"/users/%0A", b"/a/..%2Fhello", b"/./hello?", b"/./hello?x=%zz", b"/a/../hello?name=1&name=2",
              b"/x/%3F/../y", b"/x/%23/..", b"/%E2%82%AC/./", b"/%ff/./", b"/a%20b/../c", b"/hello?", b"/hello?name=%e2%82%ac"):
        out.append(("path " + repr(t), t))
    uas, xffs = log_strings()
    msgs = []
    for k, (lab, t) in enumerate(out):
        ua, xff = uas[k % len(uas)], xffs[k % len(xffs)]
        msgs.append((lab, t, ua, xff))
    return msgs


def raw_message(target, ua, xff):
    m = b"GET " + target + b" HTTP/1.1\r\nHost: h\r\n"
    if ua is not None:
        m += b"User-Agent: " + ua + b"\r\n"
    if xff is not None:
        m += b"X-Forwarded-For: " + xff + b"\r\n"
    return m + b"\r\n"


def raw_expect(target: bytes):
    path, q, query = target.partition(b"?")
    return expect(G.unescape(path, G.ENCODE_PATH), query, bool(q) and not query)


def raw_buffers(msgs):
    """one connection per message: (buf, buf_off)"""
    parts = [raw_message(t, ua, xff) for _, t, ua, xff in msgs]
    off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint32)
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), off


# ---- log records ----
def log_strings():
    """User-Agent and X-Forwarded-For values that a request head can carry (no control byte but HTAB): every White_Space
    rune that is not ASCII at both ends, a leading comma, obs-text and invalid UTF-8"""
    uas, xffs = [None, b"Go-http-client/1.1"], [None, b"1.2.3.4", b",1.2.3.4", b" , 5.6.7.8", b"9.9.9.9 , 1.1.1.1"]
    for w in WHITE + NOT_WHITE:
        if all(c >= 0x20 or c == 9 for c in w):
            xffs.append(w + b"10.0.0.1" + w)
            xffs.append(w + w + b"10.0.0.2" + w + b"," + w)
            uas.append(w + b"agent <&> \"\\" + w)
    xffs += [b"\xff1.2.3.4\xfe", b"\xe2\x80\x80\xe2\x80", b"\xc2\xa0\xc2", b"\t\t", b"\xe3\x80\x80", b","]
    uas += [bytes(range(0x80, 0x100)), b"\xe2\x80\xa8\xe2\x80\xa9", b"a\tb"]
    return uas, xffs


def log_corpus():
    """[LogRec] for the request-log kernel and gofr_batch_submit_log: every byte in the strings, every White_Space rune
    (ASCII control ones included: a host batch may carry them) at both ends of X-Forwarded-For and RemoteAddr"""
    recs = []
    t0 = 1_700_000_000_000_000_000
    add = lambda ua, xff, remote, uri: recs.append(S.LogRec(t0, 1234567, t0 + 1234567, b"GET", ua, xff, remote, uri, 200))
    for w in WHITE + NOT_WHITE:
        add(w + b"ua" + w, w + b"10.0.0.1" + w, b"r", b"/u?" + w)
        add(b"", w + b"," + w, w + b"192.0.2.1:5" + w, w)
        add(w, w + w, w + b"x" + w + w, b"/")
        add(b"", b"", w + w, b"/")
    for b in range(256):
        add(bytes([b]), bytes([b]) + b"1.1.1.1" + bytes([b]), bytes([b]), b"/" + bytes([b]))
    add(b"", b",1.2.3.4", b" 203.0.113.9 ", b"/")
    add(bytes(range(256)), bytes(range(256)), bytes(range(256)), bytes(range(256)))
    add(b"<" * 3000, b"\xff" * 3000, b"", b"%00" * 1000)
    return recs


def log_segment(rec: S.LogRec) -> bytes:
    """the part of a RequestLog line from "method" to "response": method, user_agent, ip and uri in encoding/json's
    escaping, each left out when empty (omitempty)"""
    seg = b'"method":' + G.json_string(rec.method)
    for key, v in ((b"user_agent", rec.user_agent), (b"ip", G.get_ip_address(rec.xff, rec.remote_addr)), (b"uri", rec.uri)):
        if v:
            seg += b',"' + key + b'":' + G.json_string(v)
    return seg + b',"response":'


# ---------------------------------------------------------------------------------------------------------------
# the checks
# ---------------------------------------------------------------------------------------------------------------
def model_problems(resps, meta, expects):
    """[(index, problem)] of the responses against the model"""
    bad = []
    for i, (wire, want) in enumerate(zip(resps, expects)):
        if (int(meta[i]) & 0xFFFF) != want[0]:
            bad.append((i, "meta status %d, model %d" % (int(meta[i]) & 0xFFFF, want[0])))
            continue
        p = wire_problem(wire, want)
        if p:
            bad.append((i, p))
    return bad


def _serve_three_ways(spec, batch, expects, labels):
    img = Table(spec).serialize()
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    r1 = O.responses(o1, f1)
    bad = model_problems(r1, m1, expects)
    assert not bad, [(labels[i], p) for i, p in bad[:8]]
    for mis in range(4):
        o2, f2, m2 = E.serve(img, batch, DATE, misalign=mis)
        assert np.array_equal(m1, m2) and np.array_equal(f1 + np.uint32(mis), f2), mis   # offsets start at the misalignment
        r2 = O.responses(o2, f2)
        diff = [i for i in range(batch.n) if r1[i] != r2[i]]
        assert not diff, (mis, [(labels[i], r1[i][-120:], r2[i][-120:]) for i in diff[:4]])
    return r1, m1


def test_known_answers():
    """hand-derived answers, each with the Go rule it comes from"""
    # unescape: '%' needs two hex digits ("i+2 >= len" fails); '+' is a space only in query components
    assert G.unescape(b"a%41+", G.ENCODE_QUERY_COMPONENT) == b"aA " and G.unescape(b"a%41+", G.ENCODE_PATH) == b"aA+"
    assert G.unescape(b"%4", G.ENCODE_PATH) is None and G.unescape(b"x%", G.ENCODE_PATH) is None
    assert G.unescape(b"%zz", G.ENCODE_PATH) is None and G.unescape(b"%2e%2E", G.ENCODE_PATH) == b".."
    # parseQuery: ';' skips the pair, empty pairs skip, a bad escape skips the pair, the first value wins
    assert G.query_param(b"name=a;b&name=c", b"name") == b"c"
    assert G.query_param(b"name=%zz&name=ok", b"name") == b"ok" and G.query_param(b"name=&name=ok", b"name") == b""
    assert G.query_param(b"na%6De=v", b"name") == b"v" and G.query_param(b"name", b"name") == b""
    assert G.query_param(b"name=a+b%2B", b"name") == b"a b+" and G.query_param(b"name=a=b", b"name") == b"a=b"
    # H_PARAM_FORMAT: "" → the default; the value is json-escaped after decoding
    assert G.param_format_body(b"name=", KEY, DEFAULT, PREFIX, SUFFIX) == b'{"data":"Hello World!"}\n'
    assert G.param_format_body(b"name=%3C", KEY, DEFAULT, PREFIX, SUFFIX) == b'{"data":"Hello \\u003c!"}\n'
    # encoding/json over bytes: one \ufffd per byte DecodeRune rejects (Python's "replace" gives one for e2 82)
    assert G.json_string(b"\xe2\x82") == b'"\\ufffd\\ufffd"' and G.json_string(b"\xe2\x82\xac") == b'"\xe2\x82\xac"'
    assert G.json_string(b"\xed\xa0\x80") == b'"\\ufffd\\ufffd\\ufffd"' and G.json_string(b"\xf4\x90\x80\x80") == b'"' + b"\\ufffd" * 4 + b'"'
    assert G.json_string(b"\xc0\xaf") == b'"\\ufffd\\ufffd"' and G.json_string(b"\xef\xbf\xbd") == b'"\xef\xbf\xbd"'
    assert G.json_string(b"\x08\x0c\n\r\t\"\\<>&\x7f") == b'"\\u0008\\u000c\\n\\r\\t\\"\\\\\\u003c\\u003e\\u0026\x7f"'
    assert G.json_string("\u2028\u2029".encode()) == b'"\\u2028\\u2029"'
    # path.Clean drops every extra leading slash (posixpath.normpath keeps "//"); cleanPath keeps one trailing slash
    assert G.path_clean(b"//a") == b"/a" and G.path_clean(b"/../a/./b/..") == b"/a" and G.path_clean(b"a/../..") == b".."
    assert G.clean_path(b"") == b"/" and G.clean_path(b"a//") == b"/a/" and G.clean_path(b"/./") == b"/" and G.clean_path(b"//") == b"/"
    assert not G.redirects(b"/a/") and G.redirects(b"/a//") and G.redirects(b"a")
    # shouldEscape(·, encodePath): $&+,/:;=@ stay, ? and !*'() are escaped, upper-case hex
    assert G.escape_path(b"/$&+,/:;=@-_.~az09") == b"/$&+,/:;=@-_.~az09"
    assert G.escape_path(b"?!*'() \x00\xff%") == b"%3F%21%2A%27%28%29%20%00%FF%25"
    assert G.escaped_location(b"//a b", b"", False) == b"/a%20b" and G.escaped_location(b"//a", b"", True) == b"/a?"
    assert G.escaped_location(b"/x/%2E%2E/y/", b"q=%41", False) == b"/x/%252E%252E/y/?q=%41"
    assert G.escaped_location(G.unescape(b"/a/%2E%2E/b", G.ENCODE_PATH), b"", False) == b"/b"
    # TrimSpace: unicode.IsSpace, not str.isspace (U+001C..U+001F are not space); DecodeLastRune on the right
    assert G.trim_space(b"\x1c1.2.3.4\x1f") == b"\x1c1.2.3.4\x1f" and G.trim_space(b"\xc2\xa0x\xe3\x80\x80") == b"x"
    assert G.trim_space(b"\xe2\x80x\xe2\x80") == b"\xe2\x80x\xe2\x80" and G.trim_space(b"\x85x\xa0") == b"\x85x\xa0"
    assert G.trim_space(b"\xc2\xc2\xa0") == b"\xc2" and G.trim_space(b"\xe1\xa0\x8ex") == b"\xe1\xa0\x8ex"   # U+180E: not space
    # getIPAddress: the first comma-separated element, RemoteAddr only when it is "" before the trim
    assert G.get_ip_address(b",1.2.3.4", b" r ") == b"r" and G.get_ip_address(b" , 1.2.3.4", b"r") == b""
    assert G.get_ip_address(b"\t5.6.7.8 ,x", b"r") == b"5.6.7.8"


def test_oracle_building_blocks_against_the_model():
    """O.query_get, O.clean_path, O.escape_path and O.json_string equal the model on every piece of the corpus"""
    texts = set()
    for _, r in host_corpus():
        assert O.query_get(r.query, KEY) == G.query_param(r.query, KEY), r.query[:80]
        assert O.clean_path(r.path) == G.clean_path(r.path), r.path[:80]
        assert O.escape_path(r.path) == G.escape_path(r.path), r.path[:80]
        texts.add(r.path)
        texts.add(G.query_param(r.query, KEY))
    for rec in log_corpus():
        texts.update([rec.user_agent, rec.xff, rec.remote_addr, rec.uri])
    for t in texts:
        assert O.json_string(t) == G.json_string(t), t[:80]


def test_host_batch_three_ways():
    """the host-batch corpus: model == oracle == device code at all four output misalignments"""
    corpus = host_corpus()
    batch, labels = host_batch(corpus)
    _serve_three_ways(text_spec(), batch, [host_expect(r) for _, r in corpus], labels)


@pytest.mark.parametrize("mode", [S.FRAME_INTENDED, S.FRAME_BODY])
def test_host_batch_other_frame_modes(mode):
    """the same corpus in the other framings: the oracle and the device code agree, and the bodies are the model's"""
    corpus = host_corpus()
    batch, labels = host_batch(corpus)
    spec = text_spec(mode)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    o2, f2, m2 = E.serve(Table(spec).serialize(), batch, DATE, misalign=1)
    assert np.array_equal(m1, m2) and np.array_equal(f1 + np.uint32(1), f2) and o1[:int(f1[-1])].tobytes() == o2[1:int(f2[-1])].tobytes()
    for i, (wire, (_, r)) in enumerate(zip(O.responses(o1, f1), corpus)):
        body = host_expect(r)[2]
        if body is not None:
            got = wire if mode == S.FRAME_BODY else wire.partition(b"\r\n\r\n")[2]
            assert got == body, (labels[i], got[:100], body[:100])


def test_wide_and_values_tables_three_ways():
    """the query corpus on the table the wide slot instance serves and on the text table plus a wider-data-model route"""
    corpus = [(lab, r) for lab, r in host_corpus() if r.path == b"/hello"]
    corpus += [(lab + " /hi", S.Req(S.M_GET, b"/hi", r.query.replace(b"name", b"who"))) for lab, r in corpus[:400]]
    batch, labels = host_batch(corpus)

    def wide_routes(p):
        return ("param",) if p == b"/hello" else ("hi",) if p == b"/hi" else None

    def want(r):
        if r.path == b"/hi" and not G.redirects(r.path):
            return 200, None, G.param_format_body(r.query, b"who", b"you", b"Hi ", b".")
        return expect(r.path, r.query, False, routes=wide_routes)
    _serve_three_ways(wide_spec(), batch, [want(r) for _, r in corpus], labels)
    full = host_corpus()
    batch, labels = host_batch(full)
    _serve_three_ways(values_spec(), batch, [host_expect(r) for _, r in full], labels)


def test_slot_layout_three_ways():
    """the slot layout of the device code: every response that fits is the packed one, a longer one leaves its slot alone"""
    corpus = host_corpus()
    batch, labels = host_batch(corpus)
    spec = text_spec()
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    for slot in (512, 4096):
        out, ln, meta = E.serve_slots(Table(spec).serialize(), batch, DATE, slot)
        assert np.array_equal(meta, m1) and np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32))
        ob = o1.tobytes()
        for i in range(batch.n):
            L = int(ln[i])
            if L <= slot:
                assert out[i, :L].tobytes() == ob[int(f1[i]):int(f1[i]) + L], labels[i]
            else:
                assert (out[i] == 0xEE).all(), labels[i]
        assert (ln > slot).any()


def test_raw_messages_three_ways():
    """raw HTTP/1.1 messages: the request-head parser of the oracle and of the device code agree (URL.Path decoded), and
    the responses equal the model, which decodes the target with url.unescape(·, encodePath) itself"""
    msgs = raw_corpus()
    buf, off = raw_buffers(msgs)
    d1, a1, s1, sp1 = O.http_parse(buf, off)
    d2, a2, s2, sp2 = E.http_parse(buf, off)
    assert (s1 == 0).all(), [msgs[i][0] for i in np.flatnonzero(s1)[:5]]
    assert np.array_equal(s1, s2) and np.array_equal(sp1, sp2) and d1.tobytes() == d2.tobytes()[:d1.nbytes]
    batch = S.RequestBatch(d1, np.zeros((len(msgs), 16), np.uint8), a1)
    _serve_three_ways(text_spec(), batch, [raw_expect(t) for _, t, _, _ in msgs], [m[0] for m in msgs])


def test_request_log_three_ways():
    """RequestLog lines: the oracle and the device code agree at all four misalignments, and each line's method,
    user_agent, ip and uri are the model's encoding/json bytes (compared as bytes, not after json.loads)"""
    recs = log_corpus()
    lb = S.LogBatch.pack(recs)
    lo, lf = O.request_log(lb)
    lines = O.responses(lo, lf)
    for i, rec in enumerate(recs):
        assert log_segment(rec) in lines[i], (i, rec, lines[i][:300])
    for mis in range(4):
        eo, ef = E.request_log(lb, misalign=mis)
        assert np.array_equal(ef, lf + np.uint32(mis)) and eo[mis:int(ef[-1])].tobytes() == lo[:int(lf[-1])].tobytes(), mis


def _all_checks():
    """every model comparison of this file, as a list of failures (empty when the model agrees with the oracle)"""
    bad = []
    corpus = host_corpus()
    batch, labels = host_batch(corpus)
    spec = text_spec()
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    bad += model_problems(O.responses(o1, f1), m1, [host_expect(r) for _, r in corpus])
    lb = S.LogBatch.pack(log_corpus())
    lines = O.responses(*O.request_log(lb))
    bad += [i for i, rec in enumerate(log_corpus()) if log_segment(rec) not in lines[i]]
    return bad


def test_model_catches_planted_mistakes(monkeypatch):
    """each plausible misreading of Go, planted in the model, disagrees with the oracle on the corpus"""
    assert _all_checks() == []
    real_json, real_unescape, real_clean = G.json_string, G.unescape, G.path_clean

    def python_replace(s):       # one U+FFFD per maximal subpart of an invalid sequence
        return real_json(s.decode("utf-8", "replace").encode("utf-8"))

    def plus_kept(s, mode):
        return real_unescape(s, G.ENCODE_PATH)

    def last_wins(pairs, key):
        vs = [v for k, v in pairs if k == key]
        return vs[-1] if vs else b""

    def posix(p):
        import posixpath
        return posixpath.normpath(p.decode("latin-1")).encode("latin-1") if p else b"."

    def urllib_quote(p):
        import urllib.parse
        return urllib.parse.quote(p, safe="/").encode()

    def isspace_trim(s):
        return s.decode("latin-1").strip().encode("latin-1") if s.isascii() else s.strip()

    def python_isspace(r):
        return chr(r).isspace()

    plants = [("json_string", python_replace), ("unescape", plus_kept), ("values_get", last_wins), ("path_clean", posix),
              ("escape_path", urllib_quote), ("is_space", python_isspace)]
    for name, fn in plants:
        with monkeypatch.context() as m:
            m.setattr(G, name, fn)
            assert _all_checks(), name + ": the planted mistake went unnoticed"
    with monkeypatch.context() as m:
        m.setattr(G, "trim_space", isspace_trim)
        assert _all_checks(), "str.strip trimming went unnoticed"


def slow_path_counts():
    """from the model: corpus entries whose query value needs decoding or escaping, whose path variable needs escaping,
    that redirect, and whose ip needs trimming"""
    q = v = r = ip = 0
    for _, req in host_corpus():
        if G.redirects(req.path):
            r += 1
            continue
        route = route_model(req.path)
        if route and route[0] == "param":
            raw = next((val for k, val in ((p.partition(b"=")[0], p.partition(b"=")[2]) for p in req.query.split(b"&"))
                        if G.query_unescape(k) == KEY), b"")
            val = G.query_param(req.query, KEY)
            q += bool(val) and (raw != val or G.json_string(val) != b'"' + val + b'"')
        elif route:
            v += G.json_string(route[1]) != b'"' + route[1] + b'"'
    for rec in log_corpus():
        ip0 = rec.xff.split(b",")[0] or rec.remote_addr
        ip += G.get_ip_address(rec.xff, rec.remote_addr) != ip0
    return {"query value decoded or escaped": q, "path variable escaped": v, "redirect": r, "ip trimmed": ip}


def test_slow_path_counts():
    counts = slow_path_counts()
    print("corpus entries per slow path:", counts)
    assert all(counts.values()), counts


def test_bound_covers_the_worst_cases():
    """every response of the corpus (its worst-case generators included) fits gofr_table_response_bound"""
    L = _abi.lib()
    for spec in (text_spec(), values_spec()):
        t = Table(spec)
        corpus = host_corpus()
        batch, labels = host_batch(corpus)
        _, f1, _ = O.OracleTable(spec).serve(batch, DATE)
        ln = np.diff(f1.astype(np.int64))
        for i, (_, r) in enumerate(corpus):
            bound = int(L.gofr_table_response_bound(t.handle, len(r.path), len(r.query), len(r.data)))
            assert ln[i] <= bound, (labels[i], int(ln[i]), bound)
