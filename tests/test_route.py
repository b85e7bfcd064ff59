"""Routing only (gofr_route_device): Router.Match + mux.Vars + the middleware decisions taken before a handler runs
(pkg/gofr/http/router.go:14,30-33; middleware/cors.go:10-13; pkg/gofr/http/request.go:36-38) — stage 1 of the split
API for closures that stay on the host (DESIGN.md §1, SURVEY.md §8 a6/a8)."""
import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O
from tests.emu import emu


def _multi_var_spec() -> S.TableSpec:
    host = lambda m, p: S.Route(m, p, S.H_HOST)
    return S.TableSpec(default_routes=False, routes=[
        host(S.M_GET, "/users/{id}"),
        host(S.M_GET, "/users/{id}/posts/{post:[0-9]+}"),
        host(S.M_POST, "/users/{id}"),
        host(S.M_GET, "/files/{dir}/{name}.{ext}"),
        host(S.M_GET, "/v{major:[0-9]+}.{minor:[0-9]+}/ping"),
        host(S.M_GET, "/static"),
        host(S.M_GET, "/a/{x}{y:[0-9]+}"),          # adjacent variables: leftmost-first with backtracking
        host(S.M_DELETE, "/users/{id}"),
    ])


def _multi_var_batch() -> S.RequestBatch:
    R = S.Req
    reqs = [R(S.M_GET, b"/users/42"), R(S.M_GET, b"/users/42/posts/7"), R(S.M_GET, b"/users/42/posts/x7"),
            R(S.M_POST, b"/users/abc"), R(S.M_PUT, b"/users/abc"), R(S.M_GET, b"/files/etc/passwd.txt"),
            R(S.M_GET, b"/files/a/b.c.d"), R(S.M_GET, b"/v12.345/ping"), R(S.M_GET, b"/v.1/ping"), R(S.M_GET, b"/static"),
            R(S.M_OPTIONS, b"/static"), R(S.M_OPTIONS, b"/users/9"), R(S.M_GET, b"/a/bc123"), R(S.M_GET, b"/a/123"),
            R(S.M_GET, b"/a/1"), R(S.M_GET, b"//users/1"), R(S.M_GET, b"/users/"), R(S.M_GET, b"/nope"),
            R(S.M_DELETE, b"/users/%C3%A9"), R(S.M_HEAD, b"/users/1"), R(S.M_OTHER, b"/static"), R(S.M_GET, b"/users/../x")]
    return S.RequestBatch.pack(reqs)


def test_oracle_spans_by_hand():
    spec, b = _multi_var_spec(), _multi_var_batch()
    meta, vars_ = O.route(O.OracleTable(spec), b)
    span = lambda i, k: (int(vars_[i, k]) & 0xFFFF, int(vars_[i, k]) >> 16)
    path = lambda i: bytes(b.arena[int(b.desc[i]["arena_off"]):][:int(b.desc[i]["path_len"])])
    get = lambda i, k: path(i)[span(i, k)[0]:][:span(i, k)[1]]
    assert meta[0] == 0 | 0 << 16 and get(0, 0) == b"42" and vars_[0, 1] == 0xFFFFFFFF
    assert meta[1] == 0 | 1 << 16 and (get(1, 0), get(1, 1)) == (b"42", b"7")
    assert meta[2] & 0xFFFF == 404
    assert meta[3] == 0 | 2 << 16 and get(3, 0) == b"abc"
    assert meta[4] & 0xFFFF == 405                       # PUT: no Run() catch-all here → mux's own 405
    assert (get(5, 0), get(5, 1), get(5, 2)) == (b"etc", b"passwd", b"txt")
    assert (get(6, 0), get(6, 1), get(6, 2)) == (b"a", b"b.c", b"d")   # greedy {name}, shortest {ext}
    assert (get(7, 0), get(7, 1)) == (b"12", b"345")
    assert meta[8] & 0xFFFF == 404
    # OPTIONS only matches routes registered for it (app.GET → Methods("GET")): without Run()'s catch-all mux answers
    # 405 before any middleware; with it the catch-all matches and CORS answers 200 (test_options_with_catch_all)
    assert meta[10] & 0xFFFF == 405 and meta[11] & 0xFFFF == 405
    assert (get(12, 0), get(12, 1)) == (b"bc12", b"3")   # {x} greedy, gives back one byte for {y:[0-9]+}
    assert (get(13, 0), get(13, 1)) == (b"12", b"3")
    assert meta[14] & 0xFFFF == 404                      # "1" cannot feed both variables
    assert meta[15] & 0xFFFF == 301 and meta[21] & 0xFFFF == 301
    assert meta[19] & 0xFFFF == 405 and meta[20] & 0xFFFF == 405


def test_keyed_templates_same_prefix_keep_registration_order():
    host = lambda m, p: S.Route(m, p, S.H_HOST)
    spec = S.TableSpec(default_routes=False, routes=[
        host(S.M_GET, "/apiserver/{a}"),            # 0: leading literal "/apiserver/" (>= 8 bytes → keyed)
        host(S.M_GET, "/apiserver/fixed"),          # 1: literal, shadowed by 0 for GET
        host(S.M_POST, "/apiserver/fixed"),         # 2
        host(S.M_GET, "/apiservice/{b}/x"),         # 3: same first 8 bytes as 0 → same bucket
        host(S.M_GET, "/apiserv{c}"),               # 4: leading literal exactly 8 bytes
        host(S.M_GET, "/api/{d}"),                  # 5: short leading literal → linear list
    ])
    R = S.Req
    b = S.RequestBatch.pack([R(S.M_GET, b"/apiserver/fixed"), R(S.M_POST, b"/apiserver/fixed"), R(S.M_GET, b"/apiservice/q/x"),
                             R(S.M_GET, b"/apiservX"), R(S.M_GET, b"/apiserv"), R(S.M_GET, b"/api/z"), R(S.M_GET, b"/apiserver/"),
                             R(S.M_DELETE, b"/apiserver/1"), R(S.M_GET, b"/apiservice/q/y"), R(S.M_GET, b"/apiserverX")])
    m1, v1 = O.route(O.OracleTable(spec), b)
    assert [int(x) >> 16 for x in m1[:6]] == [0, 2, 3, 4, 0xFFFF, 5]
    assert m1[6] & 0xFFFF == 404          # {a} must not be empty, {c} = [^/]+ cannot swallow the slash
    assert m1[7] & 0xFFFF == 405 and m1[8] & 0xFFFF == 404 and m1[9] >> 16 == 4
    m2, v2 = emu.route(Table(spec).serialize(), b)
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2)


def test_options_with_catch_all():
    spec = _multi_var_spec()
    spec.default_routes = True
    b = S.RequestBatch.pack([S.Req(S.M_OPTIONS, b"/static"), S.Req(S.M_OPTIONS, b"/users/9"), S.Req(S.M_PUT, b"/static")])
    meta, vars_ = O.route(O.OracleTable(spec), b)
    catch_all = len(spec.routes) + 2  # health, favicon, then PathPrefix("/") (gofr.go:102-107)
    assert meta[0] == 200 | catch_all << 16 and meta[1] == 200 | catch_all << 16
    assert meta[2] == 0 | catch_all << 16          # the catch-all's handler answers 404 itself
    assert (vars_ == 0xFFFFFFFF).all()


@pytest.mark.parametrize("which", ["multi", "config4", "config1"])
def test_emu_matches_oracle(which):
    if which == "multi":
        spec, b = _multi_var_spec(), _multi_var_batch()
    elif which == "config4":
        spec, b = synth.config4_spec(), synth.config4_batch(6000)
    else:
        spec, b = synth.config1_spec(), synth.config1_batch(300)
    m1, v1 = O.route(O.OracleTable(spec), b)
    t = Table(spec)
    m2, v2 = emu.route(t.serialize(), b)
    assert np.array_equal(m1, m2)
    assert np.array_equal(v1, v2)


def test_route_agrees_with_serve_meta():
    # the serve path's meta column carries the same route ids; statuses agree wherever the router itself answers
    spec, b = synth.config4_spec(), synth.config4_batch(4000)
    ot = O.OracleTable(spec)
    m1, _ = O.route(ot, b)
    _, _, meta = ot.serve(b, S.http_date(1_700_000_000))
    router_answers = (m1 & 0xFFFF) != 0
    assert np.array_equal(m1[router_answers], meta[router_answers])
    assert np.array_equal(m1 >> 16, meta >> 16)


@pytest.mark.gpu
@pytest.mark.parametrize("which,n", [("multi", 0), ("config4", 262144), ("config2", 100000)])
def test_gpu_matches_oracle(which, n):
    from gofr_b200.engine import Engine
    if which == "multi":
        spec, b = _multi_var_spec(), _multi_var_batch()
    elif which == "config4":
        spec, b = synth.config4_spec(), synth.config4_batch(n)
    else:
        spec, b = synth.config2_spec(), synth.config2_batch(n)
    m1, v1 = O.route(O.OracleTable(spec), b)
    eng = Engine(Table(spec), 0)
    meta, vars_ = eng.route_device(eng.upload(b))
    assert np.array_equal(m1, meta.cpu().numpy().view(np.uint32))
    assert np.array_equal(v1, vars_.cpu().numpy().view(np.uint32))
    eng.set_chunk(30000)                     # several chunks through the host-buffer variant
    m2, v2 = eng.route_host(b)
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2)
    eng.close()


# ---- random route tables × random paths: the device matcher (hash dispatch + iterative backtracking) against the
# oracle's literal restatement of mux (recursive leftmost-first), including variable spans ----
from hypothesis import given, settings, strategies as st  # noqa: E402

# the long segments give templates a leading literal of >= 8 bytes (keyed dispatch), two of them with the same first 8 bytes
SEGMENTS = ["a", "b", "ab", "users", "v1", "x.y", "1", "22", "a-b", "_", "apiservice", "apiserver", "api"]
VARIABLES = ["{id}", "{n:[0-9]+}", "{w:[a-z]+}", "{s:[a-z0-9.]*}", "{id}.{ext}", "{a}{b:[0-9]+}", "p{q}", "{d:\\d+}x",
             "{y:[0-9]{2}}", "{v:v[0-9]+}", "{f:[a-z]+\\.[a-z]{1,3}}", "{o:[a-z]?[0-9]{1,2}}", "{r:\\d{1,}-?\\w*}", "{m:a{2,}b?}",
             "{h:[a-z]+-[a-z0-9]+}", "{t:.*x}"]
ROUTE_METHODS = [S.M_GET, S.M_GET, S.M_POST, S.M_DELETE, S.M_ANY]
REQ_METHODS = [S.M_GET, S.M_POST, S.M_DELETE, S.M_OPTIONS, S.M_HEAD, S.M_OTHER]
PATH_SEGMENTS = ["a", "b", "ab", "users", "v1", "x.y", "1", "22", "a-b", "_", "42", "abc9", "apiservice", "apiserver", "api", "apiserv",
                 "p7", "3x", "q.tar.gz", "", ".", ".."]
_seg = st.sampled_from(SEGMENTS)
_var = st.sampled_from(VARIABLES)
_piece = st.one_of(_seg, _var)
_pattern = st.lists(_piece, min_size=0, max_size=4).map(lambda ps: "/" + "/".join(ps))
_method = st.sampled_from(ROUTE_METHODS)


def _rename_vars(pattern: str, k: int) -> str:
    # mux refuses duplicate variable names inside one route; keep names unique per route
    out, i, c = "", 0, 0
    while i < len(pattern):
        if pattern[i] == "{":
            j = pattern.index("}", i)
            body = pattern[i + 1:j]
            name, sep, rest = body.partition(":")
            out += "{%s%d_%d%s%s}" % (name, k, c, sep, rest)
            c += 1
            i = j + 1
        else:
            out += pattern[i]
            i += 1
    return out


@settings(max_examples=250, deadline=None)
@given(st.lists(st.tuples(_method, _pattern), min_size=1, max_size=10), st.booleans(),
       st.lists(st.tuples(st.sampled_from(REQ_METHODS), st.lists(st.sampled_from(PATH_SEGMENTS), min_size=0, max_size=4)),
                min_size=1, max_size=24))
def test_random_tables_property(routes, defaults, reqs):
    spec = S.TableSpec(default_routes=defaults,
                       routes=[S.Route(m, _rename_vars(p, k), S.H_HOST) for k, (m, p) in enumerate(routes)])
    batch = S.RequestBatch.pack([S.Req(m, ("/" + "/".join(segs)).encode()) for m, segs in reqs])
    m1, v1 = O.route(O.OracleTable(spec), batch)
    m2, v2 = emu.route(Table(spec).serialize(), batch)
    assert np.array_equal(m1, m2), (spec.routes, reqs)
    assert np.array_equal(v1, v2), (spec.routes, reqs)
    # and the full serve path reports the same route ids (H_HOST routes come back with status 0)
    _, _, m3 = emu.serve(Table(spec).serialize(), batch, S.http_date(1_700_000_000))
    assert np.array_equal(m1 >> 16, m3 >> 16)


# ---------------------------------------------------------------------------------------------------------------
# variable regexps beyond one class: concatenations of quantified classes, cross-checked with Python's re
# ---------------------------------------------------------------------------------------------------------------
QUANT_ROUTES = ["/d/{date:[0-9]{4}-[0-9]{2}-[0-9]{2}}", "/api/{ver:v[0-9]+}/items/{id:[0-9]{1,3}}", "/f/{name:[a-z]+\\.[a-z]{2,4}}",
                "/o/{x:[a-z]?[0-9]{2,}}/{y:\\w+-\\w+}", "/m/{a:a{2,}b?}c", "/t/{pre:.*}-{n:\\d+}", "/z/{k:[a-c]*}{l:[b-d]{2}}e",
                "/s/{slug:[a-z0-9]+(?:-[a-z0-9]+)*}", "/q/{e:x{0,2}}y", "/u/{w:[^/]+}.{ext:[a-z]{3}}", "/c/{n:\\d\\d:\\d\\d}"]


def _mux_regex(pattern: str):
    """the regexp mux builds from a template (newRouteRegexp): ^ + QuoteMeta(literal) + (?P<v0>pattern) ... + $"""
    import re
    out, i, names = "^", 0, []
    while i < len(pattern):
        if pattern[i] == "{":
            depth, j = 0, i
            while True:
                depth += pattern[j] == "{"
                depth -= pattern[j] == "}"
                if depth == 0:
                    break
                j += 1
            name, _, pat = pattern[i + 1:j].partition(":")
            out += "(%s)" % (pat or "[^/]+")
            names.append(name)
            i = j + 1
        else:
            j = pattern.find("{", i)
            j = len(pattern) if j < 0 else j
            out += re.escape(pattern[i:j])
            i = j
    return re.compile((out + "$").encode()), names


def test_quantified_variable_patterns_against_python_re():
    """oracle == device code == Python's re (leftmost-first backtracking, like RE2 reports for these patterns) on which
    route matches and what every variable captures; patterns outside the subset are refused when the route is added"""
    import random
    ok_routes = []
    for r in QUANT_ROUTES:
        try:
            Table(S.TableSpec(default_routes=False, routes=[S.Route(S.M_GET, r, S.H_HOST)]))
            ok_routes.append(r)
        except Exception:
            assert "(?:" in r, r          # the only pattern of the list outside the subset: a group
    assert len(ok_routes) == len(QUANT_ROUTES) - 1
    spec = S.TableSpec(default_routes=False, routes=[S.Route(S.M_GET, r, S.H_HOST) for r in ok_routes])
    rnd = random.Random(11)
    frag = ["2024", "-", "01", "1", "v", "12", "abc", ".", "tar", "gz", "a", "aa", "aaa", "b", "c", "x", "y", "_", "ab-cd", "7", "e", "bb", "cd", "12:30", ":", "0"]
    heads = ["/d/", "/api/", "/f/", "/o/", "/m/", "/t/", "/z/", "/q/", "/u/", "/c/", "/items/", "/"]
    paths = [b"/d/2024-01-31", b"/d/2024-1-31", b"/api/v12/items/7", b"/api/v12/items/1234", b"/api/v/items/1", b"/f/archive.tar", b"/f/a.b",
             b"/f/x.abcde", b"/o/a12/b-c", b"/o/123/x_1-y", b"/o/ab12/b-c", b"/m/aac", b"/m/aabc", b"/m/abc", b"/m/aaabbc", b"/t/a-b-12",
             b"/t/-1", b"/t/x-", b"/z/abcbce", b"/z/bce", b"/z/ce", b"/q/y", b"/q/xxy", b"/q/xxxy", b"/u/a.b.txt", b"/u/.txt", b"/c/12:30", b"/c/1:30"]
    for _ in range(1500):
        paths.append((rnd.choice(heads) + "".join(rnd.choice(frag) + rnd.choice(["", "", "/"]) for _ in range(rnd.randint(1, 5)))).encode())
    # near misses and hits built from each template: every variable filled from a pool of plausible values
    pool = ["2024", "01", "31", "1", "12", "123", "1234", "v1", "v12", "v", "abc", "a", "aa", "aaa", "aab", "b", "tar", "gz", "abcde", "x", "xx", "xxx",
            "", "a1", "ab12", "12a", "b-c", "x_1-y", "1-", "7-ab", "-", "a-b", "ab", "bc", "cd", "abcbc", "12:30", "1:30", "a.b", ".", "é", "2024-01-31", "ab.txt"]
    import re
    for r in ok_routes:
        parts = re.split(r"\{(?:[^{}]|\{[^{}]*\})*\}", r)
        for _ in range(250):
            paths.append("".join(part + (rnd.choice(pool) if k + 1 < len(parts) else "") for k, part in enumerate(parts)).encode())
    paths = [p for p in paths if b"//" not in p and not p.endswith(b"/.")]
    batch = S.RequestBatch.pack([S.Req(S.M_GET, p) for p in paths])
    m1, v1 = O.route(O.OracleTable(spec), batch)
    m2, v2 = emu.route(Table(spec).serialize(), batch)
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2)
    regs = [_mux_regex(r) for r in ok_routes]
    hits = 0
    for i, p in enumerate(paths):
        want = None
        for ri, (rx, names) in enumerate(regs):
            m = rx.match(p)
            if m:
                want = (ri, [m.span(k + 1) for k in range(len(names))])
                break
        if (int(m1[i]) & 0xFFFF) == 301:
            continue                       # cleanPath redirect decided before matching
        if want is None:
            assert int(m1[i]) & 0xFFFF == 404, (p, hex(int(m1[i])))
            continue
        hits += 1
        assert int(m1[i]) >> 16 == want[0] and int(m1[i]) & 0xFFFF == 0, (p, want, hex(int(m1[i])))
        for k, (a, b) in enumerate(want[1]):
            assert (int(v1[i, k]) & 0xFFFF, int(v1[i, k]) >> 16) == (a, b - a), (p, k, want)
    assert hits > 100


def test_patterns_outside_the_subset_are_refused():
    for pat in ["{a:(x|y)}", "{a:x|y}", "{a:[a-z]+?}", "{a:.{3}}", "{a:[^/]{2}}", "{a:\\s+}", "{a:[[:alpha:]]+}", "{a:^x}", "{a:x$}", "{a:é+}", "{a:.}",
                "{a:[a-z]{0}}", "{a:[a-z]{3,2}}", "{a:[a-z]{300}}", "{a:\\pL+}", "{a:*}", "{a:a**}"]:
        with pytest.raises(Exception):
            Table(S.TableSpec(default_routes=False, routes=[S.Route(S.M_GET, "/p/" + pat, S.H_HOST)]))
    for pat in ["{a:é}", "{a:[a-z]{0,}}", "{a:\\.}", "{a:.+}", "{a:[^/]*}", "{a:a{1}}"]:
        Table(S.TableSpec(default_routes=False, routes=[S.Route(S.M_GET, "/p/" + pat, S.H_HOST)]))


def test_fuzzed_variable_regexps_three_ways():
    """random variable regexps: the product and the oracle accept exactly the same ones, and on the accepted ones the
    oracle, the device code and Python's re agree on the match and on every capture"""
    import random
    import re
    rnd = random.Random(7)
    units = ["[0-9]", "[a-z]", "[a-c0-2_]", "\\d", "\\w", ".", "[^/]", "[^a-c]", "a", "b", "-", "\\.", "\\-", "x", "é", "(", ")", "|", "^", "$",
             "[", "]", "\\s", "[[:alpha:]]"]
    quants = ["", "", "+", "*", "?", "{2}", "{1,3}", "{2,}", "{0,1}", "{0}", "+?", "**", "{3,2}", "{300}"]
    pool = ["a", "b", "ab", "abc", "12", "1", "a1", "a-b", "x.y", "aa", "aab", "bbb", "012", "_", "ab-12", "a.b", "", "aaa", "0", "a/b"]
    accepted = 0
    for k in range(700):
        body = "".join(rnd.choice(units) + rnd.choice(quants) for _ in range(rnd.randint(1, 4)))
        pat = "/r/{v:%s}%s" % (body, rnd.choice(["", "/t", "-{w}", ".{e:[a-z]+}"]))
        spec = S.TableSpec(default_routes=False, routes=[S.Route(S.M_GET, pat, S.H_HOST), S.Route(S.M_GET, "/r/{any}", S.H_HOST)])
        try:
            t, okp = Table(spec), True
        except Exception:
            t, okp = None, False
        try:
            ot, oko = O.OracleTable(spec), True
        except ValueError:          # "oracle refused route": outside the subset
            ot, oko = None, False
        assert okp == oko, pat
        if not okp:
            continue
        accepted += 1
        reqs = [S.Req(S.M_GET, ("/r/" + rnd.choice(pool) + rnd.choice(["", "", "/t", "-q", ".txt", rnd.choice(pool)])).encode()) for _ in range(30)]
        b = S.RequestBatch.pack(reqs)
        m1, v1 = O.route(ot, b)
        m2, v2 = emu.route(t.serialize(), b)
        assert np.array_equal(m1, m2) and np.array_equal(v1, v2), pat
        try:
            rx, names = _mux_regex(pat)
        except re.error:
            continue
        for i, rq in enumerate(reqs):
            if (int(m1[i]) & 0xFFFF) == 301:
                continue
            mm = rx.match(rq.path)
            assert bool(mm) == ((int(m1[i]) >> 16) == 0 and (int(m1[i]) & 0xFFFF) == 0), (pat, rq.path)
            if mm:
                for kk in range(len(names)):
                    a, e = mm.span(kk + 1)
                    assert (int(v1[i, kk]) & 0xFFFF, int(v1[i, kk]) >> 16) == (a, e - a), (pat, rq.path, kk)
    assert accepted > 50
