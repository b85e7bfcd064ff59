"""Connection byte streams cut into HTTP/1.1 request records (gofr_http_frame_device): pipelined requests, partial tails and
bytes consumed per connection, in front of gofr_http_parse_device.

CPU: the oracle (tests/http_frame_oracle.c) against the device code (http_frame_device.cuh through tests/emu) everywhere;
known answers; every truncation point of the accepted corpus; a second statement of the cut points that uses only the
request-head oracle; the two invariants (cut => accepted, tail => deferred) on mutated streams; deferred records through the
serve path.  GPU: the kernel against the oracle, and the resident path streams → frame → parse → serve slots."""
import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O
from tests import http_frame_oracle as FO
from tests.emu import emu, emu_http_frame
from tests.test_http_parse import DEFERRED, GOOD

OK, DEFER = 0, 1
DONE, MORE, CDEFER = 0, 1, 2

GET = b"GET /a HTTP/1.1\r\nHost: h\r\n\r\n"
GET2 = b"GET /hello?name=x HTTP/1.1\r\nHost: localhost:8000\r\nUser-Agent: curl/8.4.0\r\n\r\n"
POST = b"POST /echo HTTP/1.1\r\nHost: h\r\nContent-Length: 9\r\n\r\n{\"id\":12}"
CHUNKED = b"POST /echo HTTP/1.1\r\nHost: h\r\nTransfer-Encoding: chunked\r\n\r\n5\r\n{\"id\"\r\n4\r\n:12}\r\n0\r\n\r\n"
OLD = b"GET /old HTTP/1.0\r\nHost: h\r\n\r\n"


def _pack(conns):
    buf = np.frombuffer(b"".join(conns), dtype=np.uint8).copy()
    off = np.cumsum([0] + [len(c) for c in conns]).astype(np.uint32)
    return buf, off


def _both(conns):
    """the oracle's framing of the connections, after checking that the device code says the same"""
    buf, off = _pack(conns)
    a, e = FO.http_frame(buf, off), emu_http_frame.http_frame(buf, off)
    for x, y, what in zip(a, e, ("rec_off", "first", "consumed", "status")):
        assert np.array_equal(x, y), what
    return a


def _cuts(conns):
    """per connection: (record lengths, consumed, status)"""
    rec, first, consumed, status = _both(conns)
    _, off = _pack(conns)
    assert rec[0] == off[0] and rec[-1] == off[-1] and (np.diff(rec.astype(np.int64)) > 0).all()
    out = []
    for c in range(len(conns)):
        r = rec[int(first[c]):int(first[c + 1]) + 1].astype(np.int64)
        assert r[0] == off[c] and (first[c] == first[c + 1] or r[-1] == off[c + 1])
        out.append((np.diff(r).tolist(), int(consumed[c]), int(status[c])))
    return out


def _long_head(blank: bool) -> bytes:
    """a head whose last header line starts beyond 16 KiB"""
    h = b"GET /a HTTP/1.1\r\nHost: h\r\n"
    while len(h) <= 16384:
        h += b"X-Pad: " + b"p" * 500 + b"\r\n"
    return h + b"X-Last: v\r\n" + (b"\r\n" if blank else b"")


def test_known_answers():
    n0, n2, np_, nc = len(GET), len(GET2), len(POST), len(CHUNKED)
    cases = [
        (b"", ([], 0, DONE)),
        (GET, ([n0], n0, DONE)),
        (GET + GET2 + GET, ([n0, n2, n0], 2 * n0 + n2, DONE)),
        (POST + GET, ([np_, n0], np_ + n0, DONE)),
        (CHUNKED + GET, ([nc, n0], nc + n0, DONE)),
        (GET + GET2[:30], ([n0, 30], n0, MORE)),                      # half a head
        (GET + POST[:-4], ([n0, np_ - 4], n0, MORE)),                 # a head and part of its body
        (GET + CHUNKED[:-9], ([n0, nc - 9], n0, MORE)),               # a partial chunk stream
        (GET + CHUNKED[:-1], ([n0, nc - 1], n0, MORE)),
        (GET + b"GET / HTTP/1.0\r\n", ([n0, 16], n0, CDEFER)),        # outside the subset before its blank line is there
        (GET + b"GET / HTTP/1.0", ([n0, 14], n0, CDEFER)),
        (GET + b"GET / HTT", ([n0, 9], n0, MORE)),
        (GET + b"BREW", ([n0, 4], n0, CDEFER)),
        (GET + b"PA", ([n0, 2], n0, MORE)),
        (GET + OLD + GET + GET, ([n0, len(OLD) + 2 * n0], n0, CDEFER)),   # valid requests behind a deferred one stay in the tail
        (OLD, ([len(OLD)], 0, CDEFER)),
        (GET + b"GET /a HTTP/1.1\r\nHost: h\r\nConnection: close\r\n", ([n0, 45], n0, CDEFER)),   # a complete line is judged
        (GET + b"GET /a HTTP/1.1\r\nHost: h\r\nConnection: close", ([n0, 43], n0, MORE)),         # an incomplete one is not
        (GET + b"GET /a HTTP/1.1\r\nHost: h\r\nHost: h\r\n", ([n0, 35], n0, CDEFER)),
        (GET + b"GET /a HTTP/1.1\r\nHost: h\r\nX: a\x01", ([n0, 31], n0, CDEFER)),                # a byte is judged as it arrives
        (GET + b"POST /a HTTP/1.1\r\nHost: h\r\nTransfer-Encoding: chunked\r\n\r\n1;", ([n0, 59], n0, CDEFER)),
        (_long_head(False), ([len(_long_head(False))], 0, CDEFER)),   # 16 KiB + of head and still no blank line
        (_long_head(True), ([len(_long_head(True))], 0, CDEFER)),
        (b"GET /a HTTP/1.1\r\nHost: h\r\nX-Pad: " + b"p" * 20000, ([20033], 0, MORE)),   # one long line that began in time
    ]
    got = _cuts([c for c, _ in cases])
    for (conn, want), g in zip(cases, got):
        assert g == want, conn[:80]


def test_every_truncation_point_of_the_accepted_corpus():
    for m, _ in GOOD:
        conns = [m[:k] for k in range(1, len(m))] + [m] + [m + bytes([b]) for b in range(256)]
        got = _cuts(conns)
        for k in range(1, len(m)):
            assert got[k - 1] == ([k], 0, MORE), (m, k)
        assert got[len(m) - 1] == ([len(m)], len(m), DONE), m
        for b in range(256):
            lens, consumed, status = got[len(m) + b]
            assert lens == [len(m), 1] and consumed == len(m) and status in (MORE, CDEFER), (m, b)


def test_every_deferred_message_stays_uncut():
    """nothing the request-head parser defers is cut as a request, alone or behind a good one"""
    for m in DEFERRED:
        if not m:
            continue
        accepted_prefix = _first_accepted(m)
        (lens, consumed, status), (lens2, consumed2, _) = _cuts([m, GET + m])
        if accepted_prefix is None:
            assert lens == [len(m)] and consumed == 0 and status in (MORE, CDEFER), m
            assert lens2 == [len(GET), len(m)] and consumed2 == len(GET), m
        else:   # deferred only because bytes follow the message: the framer's case
            assert lens[0] == accepted_prefix and lens2[:2] == [len(GET), accepted_prefix], m


def _first_accepted(rem: bytes):
    """the prefix lengths of rem that orc_http_parse accepts, by brute force: one batched call over all of them"""
    raw, off = _pack([rem[:k] for k in range(1, len(rem) + 1)])
    status = O.http_parse(raw, off)[2]
    hits = np.flatnonzero(status == OK)
    assert len(hits) <= 1, rem          # a request of the subset ends in one place only
    return int(hits[0]) + 1 if len(hits) else None


def test_cut_points_are_the_unique_prefixes_the_parser_accepts():
    """the second statement, independent of the framer's code: request k of a connection is the one prefix of the remaining
    bytes that the request-head oracle accepts; framing stops where there is none"""
    rng = np.random.default_rng(20240611)
    pool = [GET, GET2, POST, CHUNKED, b"PUT /p HTTP/1.1\r\nHost: h\r\nContent-Length: 0\r\n\r\n",
            b"GET /a%20b? HTTP/1.1\r\nhOsT: [::1]:80\r\n\r\n", b"GET /a HTTP/1.1\r\nHost: h\r\nTransfer-Encoding: chunked\r\n\r\n0\r\n\r\n"]
    bad = [OLD, b"GET /a HTTP/1.1\r\nHost: h\r\nConnection: close\r\n\r\n", b"GET /a HTTP/1.1\r\n\r\n", b"\r\n",
           b"POST /a HTTP/1.1\r\nHost: h\r\nTransfer-Encoding: chunked\r\n\r\n1;x\r\na\r\n0\r\n\r\n", b"get / HTTP/1.1\r\nHost: h\r\n\r\n"]
    conns = []
    for _ in range(60):
        parts = [pool[int(rng.integers(len(pool)))] for _ in range(int(rng.integers(0, 4)))]
        kind = int(rng.integers(4))
        if kind == 1:
            nxt = pool[int(rng.integers(len(pool)))]
            parts.append(nxt[:int(rng.integers(1, len(nxt)))])
        elif kind == 2:
            parts.insert(int(rng.integers(len(parts) + 1)), bad[int(rng.integers(len(bad)))])
        elif kind == 3 and parts:
            b = bytearray(b"".join(parts))
            b[int(rng.integers(len(b)))] = int(rng.integers(256))
            parts = [bytes(b)]
        conns.append(b"".join(parts))
    got = _cuts(conns)
    for conn, (lens, consumed, status) in zip(conns, got):
        at, want = 0, []
        while at < len(conn):
            k = _first_accepted(conn[at:])
            if k is None:
                break
            want.append(k)
            at += k
        assert consumed == at and lens[:len(want)] == want and len(lens) == len(want) + (at < len(conn)), conn
        assert (status == DONE) == (at == len(conn)), conn


def _mutate(rng, m: bytes, other: bytes) -> bytes:
    op = int(rng.integers(6))
    b = bytearray(m)
    if op == 0 and b:                                       # a byte flipped
        b[int(rng.integers(len(b)))] ^= 1 << int(rng.integers(8))
    elif op == 1 and b"\r" in m:                            # a CR dropped
        ks = [k for k, c in enumerate(m) if c == 13]
        del b[ks[int(rng.integers(len(ks)))]]
    elif op == 2:                                           # a header line duplicated
        lines = m.split(b"\r\n")
        k = int(rng.integers(1, max(2, len(lines) - 2)))
        b = bytearray(b"\r\n".join(lines[:k + 1] + lines[k:]))
    elif op == 3 and b"Content-Length: " in m:              # a Content-Length digit changed
        k = m.index(b"Content-Length: ") + 16
        b[k] = 48 + int(rng.integers(10))
    elif op == 4 and b:                                     # spliced into another stream
        k = int(rng.integers(len(b)))
        b = bytearray(m[:k] + other + m[k:])
    elif b:                                                 # cut short
        b = b[:int(rng.integers(len(b)))]
    return bytes(b)


def _mutated_streams(n: int, seed: int):
    rng = np.random.default_rng(seed)
    pool = [m for m, _ in GOOD] + [GET, GET2, POST, CHUNKED, OLD]
    conns = []
    for _ in range(n):
        parts = [pool[int(rng.integers(len(pool)))] for _ in range(int(rng.integers(1, 5)))]
        for _ in range(int(rng.integers(0, 3))):
            k = int(rng.integers(len(parts)))
            parts[k] = _mutate(rng, parts[k], pool[int(rng.integers(len(pool)))])
        conns.append(b"".join(parts))
    return conns


def test_invariants_on_mutated_streams():
    """cut => accepted, tail => deferred, under the request-head device code itself; the records tile the buffer"""
    conns = _mutated_streams(2000, 7)
    buf, off = _pack(conns)
    rec, first, consumed, status = _both(conns)
    total = int(first[-1])
    assert (np.diff(first.astype(np.int64)) >= 0).all() and first[0] == 0
    assert rec[0] == 0 and rec[-1] == off[-1] and (np.diff(rec.astype(np.int64)) > 0).all() and len(rec) == total + 1
    parsed = emu.http_parse(buf, rec)[2]
    assert np.array_equal(parsed, O.http_parse(buf, rec)[2])
    seen = np.zeros(3, dtype=np.int64)
    for c in range(len(conns)):
        lo, hi = int(first[c]), int(first[c + 1])
        length = int(off[c + 1] - off[c])
        has_tail = status[c] != DONE
        seen[status[c]] += 1
        assert rec[lo] == off[c] if hi > lo else length == 0
        assert (parsed[lo:hi - 1 if has_tail else hi] == OK).all(), conns[c]
        if has_tail:
            assert hi > lo and parsed[hi - 1] == DEFER, conns[c]
            assert int(consumed[c]) + int(rec[hi] - rec[hi - 1]) == length
        else:
            assert int(consumed[c]) == length
    assert (seen > 100).all(), seen     # the campaign reaches all three outcomes


def test_deferred_records_through_the_serve_path():
    """what the parse step leaves for a tail is a zero descriptor; both serve layouts answer it like the oracle does, reading
    nothing outside the arena (scratch/emu_asan.sh runs this file under AddressSanitizer)"""
    spec = synth.config2_spec()
    buf, off = synth.http_streams(300, tail_every=3, defer_every=5)
    rec, first, consumed, status = _both_arrays(buf, off)
    desc, arena, parsed, _ = emu.http_parse(buf, rec)
    desc = np.asarray(desc).view(S.DESC_DTYPE).copy()
    n = len(rec) - 1
    tails = np.flatnonzero(parsed == DEFER)
    assert len(tails) > 50 and not desc[tails].view(np.uint8).any()
    batch = S.RequestBatch(desc, synth.trace_ids(synth.SEED, np.arange(n, dtype=np.uint64)), arena[:buf.size].copy())
    date = S.http_date(1_700_000_000)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, date)
    image = Table(spec).serialize()
    o2, f2, m2 = emu.serve(image, batch, date)
    assert np.array_equal(f1, f2) and np.array_equal(m1, m2) and o1[:f1[-1]].tobytes() == o2[:f2[-1]].tobytes()
    slots, ln, m3 = emu.serve_slots(image, batch, date, 512)
    assert np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32)) and np.array_equal(m3, m1)
    ob = o1.tobytes()
    for i in range(n):
        assert slots[i, :int(ln[i])].tobytes() == ob[int(f1[i]):int(f1[i + 1])], i


def _both_arrays(buf, off):
    a, e = FO.http_frame(buf, off), emu_http_frame.http_frame(buf, off)
    assert all(np.array_equal(x, y) for x, y in zip(a, e))
    return a


def test_synthetic_streams_oracle_equals_device_code():
    for kw in ({}, {"tail_every": 4, "defer_every": 9}, {"reqs": (1, 1)},
               {"tail_every": 2, "seed_msgs": [m for m, _ in GOOD] + DEFERRED}):
        buf, off = synth.http_streams(1500, **kw)
        rec, first, consumed, status = _both_arrays(buf, off)
        if not kw:
            assert (status == DONE).all() and np.array_equal(consumed, np.diff(off.astype(np.int64)))
        if kw.get("reqs") == (1, 1):
            assert np.array_equal(rec, off) and np.array_equal(first, np.arange(1501))   # one record per connection


def test_record_capacity_and_arguments():
    buf, off = synth.http_streams(50, tail_every=3)
    rec, first, _, _ = FO.http_frame(buf, off)
    total = int(first[-1])
    assert len(emu_http_frame.http_frame(buf, off, rec_cap=total)[0]) == total + 1     # exactly enough
    for frame in (FO.http_frame, emu_http_frame.http_frame):
        with pytest.raises(RuntimeError):
            frame(buf, off, rec_cap=total - 1)
    # the C ABI: no engine is an invalid argument, with or without connections
    L = _abi.lib()
    assert L.gofr_http_frame_device(None, None, None, 0, None, 0, None, None, None, None) == 1
    assert L.gofr_http_frame_device(None, None, None, 4, None, 0, None, None, None, None) == 1


# ---- GPU ----
def _gpu_frame(eng, buf, off, rec_cap=None):
    d_buf, rec, first, consumed, status = eng.http_frame_device(buf, off, rec_cap)
    first = first.cpu().numpy().view(np.uint32)
    return (d_buf, rec, rec.cpu().numpy().view(np.uint32)[:int(first[-1]) + 1], first, consumed.cpu().numpy().view(np.uint32),
            status.cpu().numpy().view(np.uint32))


@pytest.mark.gpu
def test_gpu_matches_oracle():
    from gofr_b200.engine import Engine
    eng = Engine(Table(synth.config1_spec()), 0)
    big = [b"GET /big HTTP/1.1\r\nHost: h\r\nX-Pad: " + b"p" * 9000 + b"\r\n\r\n",      # tiles beyond the staging budget
           b"POST /big HTTP/1.1\r\nHost: h\r\nContent-Length: 30000\r\n\r\n" + b"b" * 30000]
    buf, off = synth.http_streams(40000, tail_every=6, defer_every=17, seed_msgs=[m for m, _ in GOOD] + DEFERRED + big)
    # tiles made only of empty connections, in the middle and at the end
    off = np.concatenate([off[:20001], np.full(300, off[20000], dtype=np.uint32), off[20001:], np.full(200, off[-1], dtype=np.uint32)])
    cases = [(buf, off)]
    for n in (1, 127, 128, 129):
        cases.append(synth.http_streams(n, tail_every=5, defer_every=7, seed=n))
    cases.append(synth.http_streams(400000, reqs=(0, 2), tail_every=50))   # several tiles for every CTA of the resident grid
    for b, o in cases:
        want = FO.http_frame(b, o)
        got = _gpu_frame(eng, b, o)[2:]
        for w, g, what in zip(want, got, ("rec_off", "first", "consumed", "status")):
            assert np.array_equal(w, g), (len(o) - 1, what)
        assert not eng.overflowed()
    eng.close()


@pytest.mark.gpu
def test_gpu_record_capacity_and_arguments():
    import torch
    from gofr_b200.engine import Engine
    eng = Engine(Table(synth.config1_spec()), 0)
    buf, off = synth.http_streams(1000, tail_every=3)
    want_rec, want_first, _, _ = FO.http_frame(buf, off)
    total = int(want_first[-1])
    _, rec, _, first, _, _ = _gpu_frame(eng, buf, off, total)                # exactly enough
    assert not eng.overflowed() and np.array_equal(rec.cpu().numpy().view(np.uint32), want_rec)
    d_buf, rec, first, consumed, status = eng.http_frame_device(buf, off, total - 1)   # one short
    assert eng.overflowed() and not eng.overflowed()
    assert np.array_equal(first.cpu().numpy().view(np.uint32), want_first)   # still complete: first[n] is the capacity needed
    assert rec.numel() == total                                              # the call had rec_cap + 1 entries to write
    L = _abi.lib()
    p = [d_buf.data_ptr(), torch.zeros(4, dtype=torch.int32, device="cuda").data_ptr()]
    cols = [rec.data_ptr(), first.data_ptr(), consumed.data_ptr(), status.data_ptr()]
    call = lambda b, o, n, r, f, c, s: L.gofr_http_frame_device(eng._e, b, o, n, r, 8, f, c, s, None)
    assert call(p[0], p[1], 0, *cols) == 0 and call(None, None, 0, None, None, None, None) == 0   # no connections: nothing touched
    assert call(None, p[1], 1, *cols) == 1 and call(p[0], None, 1, *cols) == 1
    assert call(p[0] + 4, p[1], 1, *cols) == 1 and call(p[0], p[1] + 2, 1, *cols) == 1
    for k in range(4):
        assert call(p[0], p[1], 1, *[None if j == k else x for j, x in enumerate(cols)]) == 1
    eng.close()


@pytest.mark.gpu
def test_gpu_streams_to_wire_bytes_resident():
    """connection streams → gofr_http_frame_device → gofr_http_parse_device on the record column → gofr_serve_device_slots,
    nothing leaving HBM in between but the record count; against the oracle framing, parsing and serving the same bytes."""
    import torch
    from gofr_b200.engine import DeviceBatch, Engine
    spec = synth.config2_spec()
    eng = Engine(Table(spec), 0)
    buf, off = synth.http_streams(12000, tail_every=5, defer_every=13)
    n_conns = len(off) - 1
    d_buf, d_rec, rec, first, consumed, status = _gpu_frame(eng, buf, off)
    total = int(first[-1])
    desc, arena, parsed, _ = eng.http_parse_resident(d_buf, d_rec, total)
    ids_np = synth.trace_ids(synth.SEED, np.arange(total, dtype=np.uint64))
    ids = torch.from_numpy(ids_np.reshape(-1).copy()).cuda()
    date = S.http_date(1_700_000_000)
    out, out_len, meta = eng.serve_device_slots(DeviceBatch(desc, ids, arena, total, 0), date, 512)
    # the oracle's side
    rec1, first1, consumed1, status1 = FO.http_frame(buf, off)
    assert np.array_equal(rec, rec1) and np.array_equal(first, first1) and np.array_equal(consumed, consumed1) and np.array_equal(status, status1)
    d1, a1, s1, _ = O.http_parse(buf, rec1)
    assert np.array_equal(parsed.cpu().numpy().view(np.uint32), s1)
    o1, f1, m1 = O.OracleTable(spec).serve(S.RequestBatch(d1, ids_np, a1), date)
    ln = out_len.cpu().numpy().view(np.uint32)
    o = out.cpu().numpy().reshape(total, 512)
    ob, mt = o1.tobytes(), meta.cpu().numpy().view(np.uint32)
    answered = 0
    for c in range(n_conns):
        lo, hi = int(first[c]), int(first[c + 1]) - (1 if status[c] != DONE else 0)   # the connection's whole requests
        assert (s1[lo:hi] == OK).all() and (status[c] == DONE or s1[hi] == DEFER)
        got = b"".join(o[i, :int(ln[i])].tobytes() for i in range(lo, hi))
        assert got == ob[int(f1[lo]):int(f1[hi])] and np.array_equal(mt[lo:hi], m1[lo:hi]), c
        answered += hi - lo
    assert answered > 2 * n_conns
    eng.close()
