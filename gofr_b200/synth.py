"""Synthetic request streams for the BASELINE.json configs (SURVEY.md §8d).

Request i is a pure function of (seed, i) through a counter-based generator (splitmix64 of seed ^ counter), so a rank
can generate exactly its shard and the CPU oracle and the GPU see identical bytes.
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np

from . import spec as S

SEED = 0x60F2B200
_ALNUM = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789", dtype=np.uint8)


def splitmix64(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = (x + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def rand_u64(seed: int, idx: np.ndarray, stream: int) -> np.ndarray:
    """One 64-bit draw per (request index, stream)."""
    with np.errstate(over="ignore"):
        ctr = idx.astype(np.uint64) * np.uint64(0x100000001B3) + np.uint64(stream) * np.uint64(0xD6E8FEB86659FD93)
        return splitmix64(ctr ^ np.uint64(seed))


def rand_bytes(seed: int, idx: np.ndarray, stream: int, width: int) -> np.ndarray:
    """(len(idx), width) random bytes."""
    words = (width + 7) // 8
    cols = [rand_u64(seed, idx, stream * 64 + k) for k in range(words)]
    m = np.stack(cols, axis=1).view(np.uint8).reshape(len(idx), words * 8)
    return m[:, :width]


def trace_ids(seed: int, idx: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(rand_bytes(seed, idx, 1000, 16))


# ---------------------------------------------------------------------------------------------------------------
# config 1: examples/http-server (reference examples/http-server/main.go:14-29) + defaults
# ---------------------------------------------------------------------------------------------------------------
def config1_spec(frame_mode: int = S.FRAME_WIRE) -> S.TableSpec:
    return S.TableSpec(frame_mode=frame_mode, routes=[
        S.Route(S.M_GET, "/hello", S.H_PARAM_FORMAT, s0=b"name", s1=b"World", s2=b"Hello ", s3=b"!"),
        S.Route(S.M_GET, "/error", S.H_STATIC_ERROR, s0=b"some error occurred"),
        S.Route(S.M_GET, "/redis", S.H_HOST),
        S.Route(S.M_GET, "/trace", S.H_HOST),
        S.Route(S.M_GET, "/mysql", S.H_HOST),
    ])


def config1_batch(n: int = 1000, seed: int = SEED) -> S.RequestBatch:
    """`GET /hello` × n, with every 10th request one of the 404 / 500 / health / query variants."""
    variants = [(b"/", b""), (b"/error", b""), (b"/.well-known/health", b""), (b"/hello", b"name=gofr")]
    reqs = []
    for i in range(n):
        if i % 10 == 9:
            p, q = variants[(i // 10) % len(variants)]
        else:
            p, q = b"/hello", b""
        reqs.append(S.Req(S.M_GET, p, q))
    b = S.RequestBatch.pack(reqs)
    b.trace_ids[:] = trace_ids(seed, np.arange(n))
    return b


# ---------------------------------------------------------------------------------------------------------------
# config 2: 16-route GET table, 256-byte JSON struct response
# ---------------------------------------------------------------------------------------------------------------
C2_SCHEMA = S.Schema(1, "main.Profile", [
    S.Field("ID", S.F_INT64, "id"), S.Field("Name", S.F_STRING, "name"), S.Field("Email", S.F_STRING, "email"),
    S.Field("Active", S.F_BOOL, "active"), S.Field("Count", S.F_INT32, "count")])
C2_NAME_LEN = 64
C2_EMAIL_LEN_TRUE = 110   # active=true is 4 bytes, false 5: the email absorbs the difference so the body stays 256 B
C2_REQ_STRIDE = 212       # 11-byte path + pad + 24-byte fixed row + 174/173 string bytes, padded to 4


def config2_spec(frame_mode: int = S.FRAME_WIRE, n_routes: int = 16) -> S.TableSpec:
    routes = [S.Route(S.M_GET, "/api/v1/r%02d" % k, S.H_ROW, schema_id=1) for k in range(n_routes)]
    return S.TableSpec(frame_mode=frame_mode, schemas=[C2_SCHEMA], routes=routes)


def config2_batch(n: int, start: int = 0, seed: int = SEED, n_routes: int = 16, escape_every: int = 0) -> S.RequestBatch:
    """Requests [start, start+n) of the config-2 stream.  Every body is exactly 256 bytes (`{"data":{...}}\\n`).
    escape_every=k replaces one name byte of every k-th request by a byte that needs escaping (body grows)."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    r = rand_u64(seed, idx, 1)
    route = (r % np.uint64(n_routes)).astype(np.int64)
    active = ((r >> np.uint64(8)) & np.uint64(1)).astype(np.uint32)
    count = (np.uint64(10000) + (r >> np.uint64(16)) % np.uint64(90000)).astype(np.uint32)
    ident = (np.uint64(10 ** 15) + rand_u64(seed, idx, 2) % np.uint64(9 * 10 ** 15)).astype(np.uint64)
    strings = _ALNUM[rand_bytes(seed, idx, 3, C2_NAME_LEN + C2_EMAIL_LEN_TRUE) % 62]
    email_len = np.where(active == 1, C2_EMAIL_LEN_TRUE, C2_EMAIL_LEN_TRUE - 1).astype(np.uint32)
    if escape_every:
        specials = np.frombuffer(b'"\\<>&\n\t\x01\x7f\xff', dtype=np.uint8)
        sel = np.nonzero((idx % np.uint64(escape_every)) == 0)[0]
        pos = (rand_u64(seed, idx[sel], 4) % np.uint64(C2_NAME_LEN)).astype(np.int64)
        strings[sel, pos] = specials[(rand_u64(seed, idx[sel], 5) % np.uint64(len(specials))).astype(np.int64)]

    rows = np.zeros((n, C2_REQ_STRIDE), dtype=np.uint8)
    path = np.frombuffer(b"/api/v1/r", dtype=np.uint8)
    rows[:, :9] = path
    rows[:, 9] = 48 + route // 10
    rows[:, 10] = 48 + route % 10
    fixed = np.zeros((n, 6), dtype=np.uint32)
    fixed[:, 0] = (ident & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    fixed[:, 1] = (ident >> np.uint64(32)).astype(np.uint32)
    fixed[:, 2] = C2_NAME_LEN
    fixed[:, 3] = email_len
    fixed[:, 4] = active
    fixed[:, 5] = count
    rows[:, 12:36] = fixed.view(np.uint8).reshape(n, 24)
    rows[:, 36:36 + C2_NAME_LEN + C2_EMAIL_LEN_TRUE] = strings
    # the unused last email byte of active=false rows is padding
    rows[active == 0, 36 + C2_NAME_LEN + C2_EMAIL_LEN_TRUE - 1] = 0

    desc = np.zeros(n, dtype=S.DESC_DTYPE)
    desc["arena_off"] = np.arange(n, dtype=np.uint32) * C2_REQ_STRIDE
    desc["path_len"] = 11
    desc["query_len"] = 0
    desc["data_len"] = 24 + C2_NAME_LEN + email_len
    desc["method"] = S.M_GET
    arena = rows.reshape(-1)
    pad = (-arena.size) % 16
    if pad:
        arena = np.concatenate([arena, np.zeros(pad, dtype=np.uint8)])
    return S.RequestBatch(desc, trace_ids(seed, idx), np.ascontiguousarray(arena))


C2_BODY_BYTES = 256
C2_WIRE_BYTES = 521  # 265-byte header block + 256-byte body (SURVEY.md §8 a11)


# ---------------------------------------------------------------------------------------------------------------
# config 4: 64 mixed routes, the reference's three middlewares, OPTIONS / 404 / 301 traffic
# ---------------------------------------------------------------------------------------------------------------
C4_SCHEMA = S.Schema(2, "main.Item", [
    S.Field("SKU", S.F_STRING, "sku"), S.Field("Qty", S.F_INT32, "qty"), S.Field("Price", S.F_INT64, "price_cents"),
    S.Field("InStock", S.F_BOOL, "in_stock"), S.Field("Note", S.F_STRING, "note", omitempty=True)])


def config4_spec(frame_mode: int = S.FRAME_WIRE) -> S.TableSpec:
    routes: List[S.Route] = []
    for k in range(48):
        if k % 6 == 0:
            routes.append(S.Route(S.M_GET, "/svc/%02d/items/{id}" % k, S.H_ROW, schema_id=2))
        elif k % 6 == 1:
            routes.append(S.Route(S.M_GET, "/svc/%02d/greet" % k, S.H_PARAM_FORMAT, s0=b"name", s1=b"World", s2=b"Hello ", s3=b"!"))
        elif k % 6 == 2:
            routes.append(S.Route(S.M_GET, "/svc/%02d/ping" % k, S.H_STATIC_STRING, s0=b"pong %02d" % k))
        elif k % 6 == 3:
            routes.append(S.Route(S.M_GET, "/svc/%02d/users/{uid:[0-9]+}/profile" % k, S.H_ROW, schema_id=1))
        elif k % 6 == 4:
            routes.append(S.Route(S.M_GET, "/svc/%02d/fail" % k, S.H_STATIC_ERROR, s0=b"backend %02d unavailable" % k))
        else:
            routes.append(S.Route(S.M_GET, "/svc/%02d/list" % k, S.H_ROW, schema_id=2))
    for k in range(16):
        routes.append(S.Route(S.M_POST, "/svc/%02d/items" % k, S.H_ROW, schema_id=2))
    return S.TableSpec(frame_mode=frame_mode, schemas=[C2_SCHEMA, C4_SCHEMA], routes=routes)


def config4_batch(n: int, start: int = 0, seed: int = SEED) -> S.RequestBatch:
    """~75/25 GET/POST over the 64 routes, 2 % OPTIONS, 2 % unmatched, 1 % '//' paths that mux redirects."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    r = rand_u64(seed, idx, 11)
    r2 = rand_u64(seed, idx, 12)
    strs = _ALNUM[rand_bytes(seed, idx, 13, 48) % 62]
    reqs: List[S.Req] = []
    item = C4_SCHEMA
    prof = C2_SCHEMA
    for i in range(n):
        x = int(r[i])
        y = int(r2[i])
        kind = x % 100
        s = strs[i].tobytes()
        item_row = item.encode_row([s[:8 + y % 8], y % 1000, (y >> 12) % 10 ** 7, (y >> 40) & 1,
                                    b"" if (y >> 41) & 1 else s[16:16 + (y >> 44) % 24]])
        is_post = (x >> 8) % 4 == 0
        if is_post:
            k = (x >> 16) % 16
            method, path, query, data = S.M_POST, b"/svc/%02d/items" % k, b"", item_row
        else:
            k = (x >> 16) % 48
            method, query, data = S.M_GET, b"", b""
            if k % 6 == 0:
                path, data = b"/svc/%02d/items/%s" % (k, s[24:24 + 1 + y % 12]), item_row
            elif k % 6 == 1:
                path = b"/svc/%02d/greet" % k
                query = [b"", b"name=" + s[:6], b"x=1&name=" + s[:9] + b"&name=zz", b"name=a%20b+c", b"name=%zz&name=ok"][y % 5]
            elif k % 6 == 2:
                path = b"/svc/%02d/ping" % k
            elif k % 6 == 3:
                path = b"/svc/%02d/users/%d/profile" % (k, y % 100000)
                data = prof.encode_row([y % 10 ** 12, s[:20], s[20:44], y & 1, y % 77777])
            elif k % 6 == 4:
                path = b"/svc/%02d/fail" % k
            else:
                path, data = b"/svc/%02d/list" % k, item_row
        if kind < 2:
            method = S.M_OPTIONS
        elif kind < 4:
            path = path + b"/nope"
        elif kind < 5:
            path = b"/" + path  # "//svc/.." → 301
        elif kind < 6:
            method = S.M_HEAD
        elif kind < 7:
            method = S.M_DELETE  # registered path, wrong method → catch-all 404
        reqs.append(S.Req(method, path, query, data))
    b = S.RequestBatch.pack(reqs)
    b.trace_ids[:] = trace_ids(seed, idx)
    return b


# ---------------------------------------------------------------------------------------------------------------
# config 5: gRPC unary Hello frames (examples/grpc-server)
# ---------------------------------------------------------------------------------------------------------------
def config5_frames(n: int, start: int = 0, seed: int = SEED) -> Tuple[np.ndarray, np.ndarray]:
    """Length-prefixed HelloRequest frames; 10 % empty names, the rest ASCII 1–16 bytes.  Returns (bytes, in_off[n+1])."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    r = rand_u64(seed, idx, 21)
    name_len = np.where(r % np.uint64(10) == 0, 0, 1 + (r >> np.uint64(8)) % np.uint64(16)).astype(np.int64)
    names = _ALNUM[rand_bytes(seed, idx, 22, 16) % 62]
    # frame = 00 | be32(len(msg)) | msg ; msg = (0a | len | name) or empty
    msg_len = np.where(name_len > 0, name_len + 2, 0)
    flen = 5 + msg_len
    off = np.zeros(n + 1, dtype=np.uint32)
    np.cumsum(flen, out=off[1:])
    buf = np.zeros(int(off[n]) + 16, dtype=np.uint8)
    base = off[:-1].astype(np.int64)
    buf[base + 4] = msg_len.astype(np.uint8)
    nz = name_len > 0
    buf[base[nz] + 5] = 0x0A
    buf[base[nz] + 6] = name_len[nz].astype(np.uint8)
    for k in range(16):
        m = name_len > k
        buf[base[m] + 7 + k] = names[m, k]
    return buf, off


# ---------------------------------------------------------------------------------------------------------------
# config 3: POST /echo — ctx.Bind() into a 5-field struct, echoed back
# ---------------------------------------------------------------------------------------------------------------
C3_SCHEMA = S.Schema(3, "main.Person", [
    S.Field("ID", S.F_INT64, "id"), S.Field("Name", S.F_STRING, "name"), S.Field("Email", S.F_STRING, "email"),
    S.Field("Active", S.F_BOOL, "active"), S.Field("Age", S.F_INT32, "age")])


def config3_spec(frame_mode: int = S.FRAME_WIRE) -> S.TableSpec:
    return S.TableSpec(frame_mode=frame_mode, schemas=[C3_SCHEMA],
                       routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=3)])


def config3_batch(n: int = 65536, start: int = 0, seed: int = SEED, variant_every: int = 100) -> S.RequestBatch:
    """Compact JSON bodies with the keys in declaration order; every `variant_every`-th request is a variant:
    reordered / case-folded / unknown keys, whitespace, escapes, or an invalid body (→ 500 with Go's error text)."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    r = rand_u64(seed, idx, 31)
    strs = _ALNUM[rand_bytes(seed, idx, 32, 40) % 62]
    variants = [
        lambda i, nm, em: b'{ "name" : "%s" , "ID" : %d , "zzz" : {"a":[1,2,{"b":null}]} , "EMAIL":"%s","active":true }' % (nm, i, em),
        lambda i, nm, em: b'{"id":%d,"name":"a\\"b\\\\c\\u00e9\\ud83d\\ude00\\n<%s>","email":"\xc3\xa9%s","active":false,"age":-7}' % (i, nm, em),
        lambda i, nm, em: b'{"id":"%d","name":"%s"}' % (i, nm),
        lambda i, nm, em: b'{"id":%d,"name":"%s","age":3000000000}' % (i, nm),
        lambda i, nm, em: b'{"id":%d,"name":"%s"' % (i, nm),
        lambda i, nm, em: b'{"id":%d,,"name":"%s"}' % (i, nm),
        lambda i, nm, em: b'[%d]' % i,
        lambda i, nm, em: b'null',
        lambda i, nm, em: b'{"id":1.5e3,"name":"%s","active":"yes"}' % nm,
        lambda i, nm, em: b'',
    ]
    reqs: List[S.Req] = []
    for k in range(n):
        x = int(r[k])
        ident = x % 10 ** 12
        nm = strs[k, :8 + x % 12].tobytes()
        em = strs[k, 20:20 + 10 + (x >> 8) % 10].tobytes()
        if variant_every and (start + k) % variant_every == variant_every - 1:
            body = variants[((start + k) // variant_every) % len(variants)](ident, nm, em)
        else:
            body = b'{"id":%d,"name":"%s","email":"%s@example.com","active":%s,"age":%d}' % (
                ident, nm, em, b"true" if (x >> 20) & 1 else b"false", (x >> 24) % 120)
        reqs.append(S.Req(S.M_POST, b"/echo", b"", body))
    b = S.RequestBatch.pack(reqs)
    b.trace_ids[:] = trace_ids(seed, idx)
    return b


# ---------------------------------------------------------------------------------------------------------------
# RequestLog lines (SURVEY.md §8f rank 1): what middleware.Logging would log for the config-2 stream
# ---------------------------------------------------------------------------------------------------------------
_UAS = [b"Go-http-client/1.1", b"curl/8.4.0", b"Mozilla/5.0 (X11; Linux x86_64) AppleWebKit/537.36 (KHTML, like Gecko)",
        b"k6/0.47.0 (https://k6.io/)", b""]


def reqlog_batch(n: int, start: int = 0, seed: int = SEED, n_routes: int = 16, hostile_every: int = 0,
                 tz_offset_s: int = 0, rpc_every: int = 0) -> S.LogBatch:
    """Log records of requests [start, start+n) of the config-2 stream.  hostile_every=k makes every k-th record carry
    strings that need JSON escaping, Unicode spaces around the forwarded address, zero fields (omitempty), odd clocks."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    r = rand_u64(seed, idx, 11)
    r2 = rand_u64(seed, idx, 12)
    t0 = 1_700_000_000_000_000_000
    recs = []
    for k in range(n):
        i = int(idx[k])
        a, b = int(r[k]), int(r2[k])
        start_ns = t0 + i * 977 + (a % 1000) * 1000  # µs resolution is common; some records get full ns below
        if a % 7 == 0:
            start_ns += b % 1000
        if a % 31 == 0:
            start_ns -= start_ns % 1_000_000_000  # whole second: no fraction at all
        elapsed = 20_000 + (b >> 8) % 3_000_000
        route = a % n_routes
        rec = S.LogRec(start_ns, elapsed, start_ns + elapsed + 1500, b"GET", _UAS[(a >> 8) % len(_UAS)],
                       b"" if (a >> 16) % 3 else b"10.%d.%d.%d, 35.191.0.%d" % ((a >> 20) % 256, (a >> 28) % 256, (a >> 36) % 256, b % 256),
                       b"192.168.%d.%d:%d" % ((b >> 16) % 256, (b >> 24) % 256, 1024 + (b >> 32) % 60000),
                       b"/api/v1/r%02d" % route, 200, tz_offset_s)
        if hostile_every and i % hostile_every == 0:
            v = (i // hostile_every) % 8
            if v == 0:
                rec.user_agent = b'agent "quoted" <b>&amp;\\ \x01\x7f \xe2\x80\xa8 \xff\xfe'
            elif v == 1:
                rec.xff = b" \t\xc2\xa0 203.0.113.9\xe2\x80\x83\xe3\x80\x80 , 10.0.0.1"
            elif v == 2:
                rec.xff, rec.remote_addr = b",10.0.0.1", b"\xc2\x85[::1]:8080\xe1\x9a\x80\r\n"
            elif v == 3:
                rec.elapsed_ns, rec.status, rec.user_agent, rec.method = 999, 0, b"", b""
            elif v == 4:
                rec.uri = b"/search?q=<script>&x=\xc3\xa9%20\"y\""
                rec.method = b"M-SEARCH"
            elif v == 5:
                rec.start_unix_ns, rec.tz_offset_s, rec.status = -1, -(3 * 3600 + 30 * 60), 404
                rec.log_unix_ns = 1
            elif v == 6:
                rec.xff, rec.remote_addr = b"  \xe2\x80\x8a ", b""
                rec.tz_offset_s = 5 * 3600 + 45 * 60 + 30
            else:
                rec.start_unix_ns = 4_102_444_799_999_999_990  # 2099-12-31T23:59:59.99999999
                rec.log_unix_ns = rec.start_unix_ns + 10
                rec.elapsed_ns = -2_000_500
                rec.tz_offset_s = 14 * 3600
        if rpc_every and i % rpc_every == 0:  # the gRPC interceptor's RPCLog line for the same clock readings
            rec.kind = S.LOG_RPC
            if not (hostile_every and i % hostile_every == 0):
                rec.method = b"/Hello/SayHello"
            elif rec.method == b"GET":
                rec.method = b'/pkg.Svc/Do"it"\\<now>&\xe2\x80\xa9\n\x02\xff\xc3\xa9'
        recs.append(rec)
    b = S.LogBatch.pack(recs)
    b.trace_ids[:] = trace_ids(seed, idx)
    return b


# ---------------------------------------------------------------------------------------------------------------
# raw HTTP/1.1 request messages (SURVEY.md §8f rank 2): the config-2 stream as a client would send it
# ---------------------------------------------------------------------------------------------------------------
def http_messages(n: int, start: int = 0, seed: int = SEED, n_routes: int = 16, seed_msgs=None):
    """n request messages back to back: (raw uint8, raw_off uint32[n+1]).  seed_msgs (directed cases, valid or not) are
    interleaved every 50 messages when given."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    r = rand_u64(seed, idx, 21)
    msgs = []
    for k in range(n):
        a = int(r[k])
        if seed_msgs and k % 50 == 7:
            msgs.append(seed_msgs[(k // 50) % len(seed_msgs)])
            continue
        route = a % n_routes
        ua = _UAS[(a >> 8) % len(_UAS)]
        head = b"GET /api/v1/r%02d HTTP/1.1\r\nHost: api.example.com:8000\r\n" % route
        if ua:
            head += b"User-Agent: " + ua + b"\r\n"
        if (a >> 16) % 3 == 0:
            head += b"X-Forwarded-For: 10.%d.%d.%d, 35.191.0.1\r\n" % ((a >> 20) % 256, (a >> 28) % 256, (a >> 36) % 256)
        head += b"Accept: application/json\r\nAccept-Encoding: gzip\r\n\r\n"
        msgs.append(head)
    raw = np.frombuffer(b"".join(msgs), dtype=np.uint8).copy()
    off = np.cumsum([0] + [len(m) for m in msgs]).astype(np.uint32)
    return raw, off


def http_streams(n_conns: int, seed: int = SEED, reqs=(0, 5), tail_every: int = 0, defer_every: int = 0, seed_msgs=None):
    """n_conns connection receive buffers back to back: (buf uint8, buf_off uint32[n_conns+1]).  The http_messages stream cut
    into connections of reqs[0]..reqs[1] requests each (seeded).  tail_every: every such connection ends with the first part
    of one more request, cut at a seeded byte; defer_every: every such connection gets a request outside the subset at a
    seeded place among its own.  seed_msgs: as in http_messages."""
    r = rand_u64(seed, np.arange(n_conns, dtype=np.uint64), 22)
    counts = (reqs[0] + r % np.uint64(reqs[1] - reqs[0] + 1)).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(counts)])
    total = int(starts[-1])
    raw, off = http_messages(total + 1, seed=seed, seed_msgs=seed_msgs)
    rawb = raw.tobytes()
    if not tail_every and not defer_every:   # whole messages only: the connections are slices of the stream as it is
        return raw[:int(off[total])].copy(), off[starts].astype(np.uint32)
    old = b"GET /legacy HTTP/1.0\r\nHost: api.example.com\r\n\r\n"
    conns = []
    for c in range(n_conns):
        a = int(r[c]) >> 8
        lo, hi = int(starts[c]), int(starts[c + 1])
        parts = [rawb[int(off[k]):int(off[k + 1])] for k in range(lo, hi)]
        if defer_every and c % defer_every == defer_every // 2:
            parts.insert(a % (len(parts) + 1), old)
        if tail_every and c % tail_every == tail_every - 1:
            nxt = rawb[int(off[hi]):int(off[hi + 1])]
            parts.append(nxt[:1 + (a >> 8) % (len(nxt) - 1)])
        conns.append(b"".join(parts))
    buf = np.frombuffer(b"".join(conns), dtype=np.uint8).copy()
    return buf, np.cumsum([0] + [len(x) for x in conns]).astype(np.uint32)


def conn_clients(n_conns: int, seed: int = SEED, t0: int = 1_700_000_000_000_000_000):
    """What gofr_conn_batch_submit_log takes per connection besides its bytes, seeded: the remote addresses (IPv4 host:port
    and bracketed IPv6, as net/http's req.RemoteAddr) back to back, their offsets uint32[n_conns + 1], and each
    connection's start clock (int64 unix ns, some on whole seconds, some with a nanosecond fraction)."""
    idx = np.arange(n_conns, dtype=np.uint64)
    r, r2 = rand_u64(seed, idx, 31), rand_u64(seed, idx, 32)
    addrs = []
    for a, b in zip(r.tolist(), r2.tolist()):
        port = 1024 + (b >> 40) % 64000
        if a % 5 == 0:
            addrs.append(b"[2001:db8:%x::%x]:%d" % ((a >> 8) % 65536, (a >> 24) % 65536, port))
        else:
            addrs.append(b"%d.%d.%d.%d:%d" % ((a >> 8) % 256, (a >> 16) % 256, (a >> 24) % 256, (a >> 32) % 256, port))
    remote = np.frombuffer(b"".join(addrs), dtype=np.uint8).copy()
    remote_off = np.cumsum([0] + [len(x) for x in addrs]).astype(np.uint32)
    start = (np.int64(t0) + idx.astype(np.int64) * 1_000_003 + (r2 % np.uint64(1_000_000)).astype(np.int64) * 1000
             + np.where(r % np.uint64(7) == 0, (r2 >> np.uint64(20)) % np.uint64(1000), 0).astype(np.int64))
    start = np.where(r % np.uint64(31) == 0, start - start % 1_000_000_000, start)
    return remote, remote_off, start.astype(np.int64)
