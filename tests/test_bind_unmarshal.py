"""Context.Bind against an independent json.Unmarshal (tests/go_unmarshal.py, restated from Go 1.21's encoding/json), on a
corpus aimed at where a decoder goes wrong: every raw byte 0x80-0xFF in a string, truncated UTF-8 at the closing quote
and before an escape, every surrogate combination, escaped / folded / invalid-UTF-8 keys, duplicates with null between,
int32 and int64 bounds, every pair of JSON kind and field kind, two errors in one body, whitespace, and rows placed
around the first bind slot (GOFR_BIND_ROW_SLOT).  Two schemas: the known-answer one (INT64, STRING, BOOL, INT32) and one
with float64 members whose Go type name and a JSON name take most of what a sealed table's shared memory holds.

CPU: the device code (tests/emu: gofr_bind_device's rows, and the fused GOFR_H_BIND_ECHO programs at every output
misalignment) and the oracle (oracle/orc_bind.c) against the model; the model against three planted mistakes.
GPU (-m gpu): gofr_bind_device at batch sizes 1, 31, 32, 33 and 65 536, slots at and below the row lengths, sentinel fill
beyond the zero pad; the fused serve kernels (packed and slot layout) against the model's struct encoded as encoding/json
writes it; and the C++ App's three serve entries, which must hand every closure the model's row."""
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from gofr_b200 import spec as S
from gofr_b200.table import Table
from tests import go_unmarshal as G
from tests import oracle as O
from tests.emu import emu
from tests.test_oracle_golden import BIND_SCHEMA
from tests.test_values import go_json

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATE = S.http_date(1789974595)

KAT_SPEC = S.TableSpec(frame_mode=S.FRAME_BODY, schemas=[BIND_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=7)])
# 8000-byte Go type and JSON names: the sealed table's hot part (the literal pool holds each name several times) then
# takes about 37 KB of the 40 KB of shared memory a table may use.  "kask" carries the two non-ASCII folds (U+212A, U+017F).
LONG = 8000
LONG_SCHEMA = S.Schema(12, "pkg." + "T" * LONG, [
    S.Field("Name", S.F_STRING, "n" * LONG), S.Field("Value", S.F_FLOAT64, "value"), S.Field("Kask", S.F_INT, "kask"),
    S.Field("Delta", S.F_FLOAT64, "delta", True), S.Field("Flag", S.F_BOOL, "flag"), S.Field("Small", S.F_INT32, "small"),
    S.Field("Note", S.F_STRING, "note")])
LONG_SPEC = S.TableSpec(frame_mode=S.FRAME_BODY, schemas=[LONG_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=12)])
SPECS = {"kat": KAT_SPEC, "long": LONG_SPEC}


def row_slot(schema, data_len):
    """GOFR_BIND_ROW_SLOT (include/gofr_b200.h)"""
    return (8 * len(schema.fields) + data_len + 256 + 15) & ~15


def row_bound(schema, data_len):
    """GOFR_BIND_ROW_BOUND (include/gofr_b200.h)"""
    names = len(schema.go_type) + max(len(f.name.encode()) for f in schema.fields)
    return 8 * len(schema.fields) + 3 * data_len + 70 + names


# ---------------------------------------------------------------------------------------------------------------
# the corpus
# ---------------------------------------------------------------------------------------------------------------
TRUNCATED = [b"\xc3", b"\xe2", b"\xe2\x82", b"\xe0\xa0", b"\xed\x9f", b"\xf0", b"\xf0\x9f", b"\xf0\x9f\x98", b"\xf4\x8f\xbf"]
INVALID = [b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\xaf", b"\xe0\x9f\xbf", b"\xf0\x80\x80\xaf", b"\xf0\x8f\xbf\xbf", b"\xed\xa0\x80",
           b"\xed\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf8\x88\x80\x80\x80", b"\xfe", b"\xff", b"\x80", b"\xbf\xbf",
           b"\xe2\x28\xa1", b"\xc3\x28", b"\xe2\x82\x28"]
VALID = [b"\xc2\x80", b"\xdf\xbf", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xef\xbf\xbd", b"\xef\xbf\xbf", b"\xf0\x90\x80\x80",
         b"\xf4\x8f\xbf\xbf", b"\xe2\x80\xa8", b"caf\xc3\xa9"]
SURR = [b"\\ud800", b"\\udbff", b"\\udc00", b"\\udfff", b"\\uD83D", b"\\uDE00", b"\\u0041", b"\\ufffd"]
INTS64 = [b"0", b"-0", b"1", b"-1", b"9223372036854775807", b"-9223372036854775808", b"9223372036854775808", b"-9223372036854775809",
          b"18446744073709551615", b"18446744073709551616", b"99999999999999999999", b"-99999999999999999999", b"12345678901234567890",
          b"1e0", b"1E2", b"-0.0", b"0.0", b"1.0", b"1.5", b"0e0", b"-1e-0", b"123456789012345678901234567890"]
INTS32 = [b"2147483647", b"-2147483648", b"2147483648", b"-2147483649", b"4294967295", b"4294967296", b"-0", b"1e0", b"-0.0"]
KINDS = [b'"s"', b'""', b'"\\u00e9"', b"7", b"-7", b"2.5", b"1e400", b"true", b"false", b"null", b"{}", b'{"id":1}', b"[]", b"[1,2]"]
WS = [b" ", b"\t", b"\r", b"\n", b" \t\r\n "]


def _kat_corpus():
    bodies = []
    s = lambda v: b'{"name":"' + v + b'"}'
    bodies += [s(b"a" + bytes([c]) + b"z") for c in range(0x80, 0x100)]
    bodies += [s(bytes([c])) for c in range(0x80, 0x100)]
    for t in TRUNCATED + INVALID + VALID:
        bodies += [s(t), s(b"x" + t), s(t + b"\\n"), s(t + b"\\u0041"), s(t + b"\\ud83d\\ude00"), s(t + t), s(t + b"a" + t)]
    for a in SURR:
        bodies += [s(a), s(b"x" + a + b"y")]
        for b in SURR:
            bodies += [s(a + b), s(a + b + b"z"), s(a + b"\\n" + b)]
            for c in SURR[:4]:
                bodies.append(s(a + b + c))
    bodies += [s(b"\\ud83d\\ud83d\\ude00"), s(b"\\ud83d\xf0\x9f\x98\x80"), s(b"\\ud83d\\u0041"), s(b"\\ud83d\\"), s(b"\\ud83d\\/"),
               s(b"\\ud83d\\u"), s(b"\\ud83d\\ude0"), s(b"\\\"\\\\\\/\\b\\f\\n\\r\\t"), s(b"\\u0000\\u001f\\u007f"), s(b"<&>\\u2028")]
    # keys: escaped, folded (ASCII, U+212A in "ok", U+017F nowhere in these names), invalid UTF-8, unknown
    for k in (b"\\u006eame", b"n\\u0061me", b"NAME", b"nAmE", b"Name", b"NAME ", b"na\xffme", b"\xffname", b"name\xff", b"na\\u00ffme",
              b"\\u004eAME", b"\\u0000name", b"nam", b"names", b"\xe2\x84\xaaname"):
        bodies.append(b'{"' + k + b'":"v"}')
    for k in (b"o\xe2\x84\xaa", b"O\xe2\x84\xaa", b"o\\u212a", b"o\\u212A", b"\xe2\x84\xaaok", b"OK", b"oK", b"o\xc5\xbf", b"\\u006fk"):
        bodies.append(b'{"' + k + b'":true}')
    bodies += [b'{"\\u0130D":5}', b'{"\xc4\xb1d":5}', b'{"I\\u0044":5}', b'{"i\\u0064":5}', b'{"\xef\xbc\xa9D":5}']
    # duplicates, exact and folded, with null between
    bodies += [b'{"name":"a","name":null,"name":"b"}', b'{"name":"a","name":null}', b'{"name":"a","NAME":null}', b'{"NAME":"x","name":"y"}',
               b'{"name":"y","NAME":"x"}', b'{"NAME":"a","name":"b","Name":"c"}', b'{"id":1,"ID":null,"Id":3}', b'{"id":1,"id":"x","id":2}',
               b'{"id":"x","id":2}', b'{"ok":true,"OK":null}', b'{"ok":true,"o\xe2\x84\xaa":false}', b'{"n":1,"n":null,"N":2,"n":null}',
               b'{"name":"' + b"\xff" * 40 + b'","name":"short"}', b'{"name":"short","name":"' + b"\xff" * 40 + b'"}']
    # integer bounds, 20-digit literals, spellings an int refuses
    bodies += [b'{"id":' + v + b"}" for v in INTS64] + [b'{"n":' + v + b"}" for v in INTS32 + INTS64[:8]]
    bodies += [b'{"id":' + v + b',"n":1}' for v in (b"1e0", b"-0.0")]
    # every pair of JSON kind and field kind, and two errors in one body (the first one is reported)
    for f in (b"id", b"name", b"ok", b"n", b"zz"):
        bodies += [b'{"' + f + b'":' + v + b"}" for v in KINDS]
    bodies += [b'{"id":"x","name":5}', b'{"name":5,"id":"x"}', b'{"ok":1,"n":1e0,"name":"kept"}', b'{"n":[1],"ok":{}}',
               b'{"id":99999999999999999999,"n":2147483648}', b'{"id":"x","id":"y"}', b'{"name":true,"name":"after"}']
    # top level: null, other kinds, syntax errors, nesting at and past 64
    bodies += [b"null", b" null ", b"[1]", b"[]", b'"s"', b"12", b"-0", b"1e400", b"true", b"false", b"{}", b" {} ", b"", b" ", b"{",
               b'{"id":1', b'{"id":1,}', b"{'id':1}", b'{"id":01}', b'{"id":1}x', b'{"name":"\x01"}', b'{"name":"\\x"}', b'{"name":"\\u12"}',
               b'{"id":NaN}', b'{"id":-}', b'{"id":1.}', b'{"id":1e}', b"nul", b"tru", b"\xef\xbb\xbf{}", b'{"\xff":1,}',
               b'{"x":' + b"[" * 63 + b"]" * 63 + b"}", b'{"x":' + b"[" * 64 + b"]" * 64 + b"}", b'{"x":' + b"[" * 70 + b"]" * 70 + b',"name":"d"}',
               b'{"x":' + b"[" * 70 + b"]" * 69 + b"}"]
    # whitespace everywhere it is allowed
    for w in WS:
        bodies += [w + b'{' + w + b'"id"' + w + b":" + w + b"1" + w + b"," + w + b'"name"' + w + b":" + w + b'"a"' + w + b"}" + w,
                   b'{"ok"' + w + b":" + w + b"true" + w + b"}", w + b"null" + w, b'{"x":[' + w + b"1" + w + b"," + w + b"{}" + w + b"]}"]
    bodies += [b'{"id":1}\x0b', b'\x0c{"id":1}', b'{"id":1}\xc2\xa0']
    return bodies


def _long_corpus():
    name = b"n" * LONG
    bodies = [b'{"' + name + b'":"' + v + b'","note":"' + w + b'"}' for v, w in ((b"x", b"y"), (b"\xff", b"\xe2\x82"), (b"\\ud800", b"\\udc00z"))]
    bodies += [b'{"' + name.upper() + b'":"folded"}', b'{"' + name[:-1] + b'":"short key"}', b'{"' + name + b'n":"long key"}']
    for f in (b"value", b"delta", b"kask", b"flag", b"small", b"note", name):
        bodies += [b'{"' + f + b'":' + v + b"}" for v in KINDS + [b"1e0", b"-0.0", b"-0", b"1.7976931348623157e308", b"1e309", b"9007199254740993",
                                                                     b"4.9e-324", b"2.5e-5", b"123456789012345678901234567890"]]
    bodies += [b'{"' + k + b'":3}' for k in (b"KASK", b"\xe2\x84\xaaask", b"ka\xc5\xbfk", b"\\u212aa\\u017fk", b"K\xe2\x84\xaaSK", b"kas")]
    bodies += [b'{"small":2147483648,"value":1e400}', b'{"value":1e400,"small":2147483648}', b'{"kask":9223372036854775808,"flag":1}',
               b'{"value":1.5,"value":null,"delta":-0.0,"flag":true,"small":-2147483648,"kask":-9223372036854775808,"note":"n"}',
               b'{"value":9007199254740993,"small":"x"}', b'{"delta":0,"note":""}', b"[1]", b"null", b"{}"]
    return bodies


def _aimed(schema, family, params):
    """bodies of a family whose model row length lands at slot - 16, slot - 1, slot and slot + 1 of its own first slot"""
    found = {}
    for p in params:
        body = family(p)
        d = len(G.unmarshal(schema, body).row) - row_slot(schema, len(body))
        if d in (-16, -1, 0, 1) and d not in found:
            found[d] = body
    assert sorted(found) == [-16, -1, 0, 1], (schema.go_type[:8], sorted(found))
    return [found[d] for d in (-16, -1, 0, 1)]


def _aimed_bodies(schema):
    pairs = [(a, b) for a in range(100, 200) for b in range(16)]
    if schema is BIND_SCHEMA:   # invalid UTF-8 triples the string
        return _aimed(schema, lambda p: b'{"name":"' + b"\xff" * p[0] + b"x" * p[1] + b'"}', pairs)
    # the long type name and a literal in an error text, the body lengthened by an ignored string; invalid UTF-8 in "note"
    return (_aimed(schema, lambda p: b'{"zz":"' + b"s" * (LONG - 1600 + 16 * (p[0] - 100)) + b'","small":' + b"1" * (11 + p[1]) + b"}", pairs) +
            _aimed(schema, lambda p: b'{"note":"' + b"\xfe" * p[0] + b"x" * p[1] + b'"}', pairs))


def _random_bodies(schema, seed, n):
    """seeded members drawn from the corpus's atoms"""
    rnd = random.Random(seed)
    keys = [f.name.encode() for f in schema.fields if len(f.name) < 100] + [b"NAME", b"Id", b"o\xe2\x84\xaa", b"zz", b"na\xffme", b"\\u006e"]
    vals = KINDS + INTS32 + INTS64[:12] + [b'"' + t + b'"' for t in TRUNCATED + INVALID + VALID + SURR]
    out = []
    for _ in range(n):
        members = [b'"' + rnd.choice(keys) + b'"' + rnd.choice([b"", b" "]) + b":" + rnd.choice(vals) for _ in range(rnd.randint(0, 6))]
        out.append(b"{" + b",".join(members) + b"}")
    return out


_CORPUS = {}


def corpus(which):
    """the bodies of one schema's corpus (fixed lists, aimed slot edges, seeded members) and the model's answers"""
    if which not in _CORPUS:
        schema = SPECS[which].schemas[0]
        bodies = (_kat_corpus() if which == "kat" else _long_corpus()) + _aimed_bodies(schema) + _random_bodies(schema, 3, 300)
        _CORPUS[which] = (bodies, [G.unmarshal(schema, b) for b in bodies])
    return _CORPUS[which]


def batch_of(bodies):
    return S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])


# ---------------------------------------------------------------------------------------------------------------
# the verdict
# ---------------------------------------------------------------------------------------------------------------
def row_problems(bodies, answers, status, ln, rows, slot, syntax_rows=None):
    """gofr_bind_device's (status, len, rows[n, slot], pre-filled with 0xEE) against the model: status and len equal the
    model's (HOST only where host_ok), bytes equal where len <= slot, zeros to the next 16-byte boundary, 0xEE beyond.
    syntax_rows[i]: the text to hold a syntax error's row to (the model restates only the verdict).  Returns (index, why)."""
    bad = []
    for i, (b, a) in enumerate(zip(bodies, answers)):
        s, n = int(status[i]), int(ln[i])
        if s == G.HOST:
            if not a.host_ok or n:
                bad.append((i, "host"))
            continue
        want = a.row if a.row is not None else (syntax_rows[i] if syntax_rows is not None else None)
        if s != a.status or (want is not None and n != len(want)):
            bad.append((i, "status/len"))
            continue
        r = rows[i]
        if n > slot:
            if not (r == 0xEE).all():
                bad.append((i, "wrote past slot"))
            continue
        pad = min(slot, (n + 15) & ~15)
        if (want is not None and r[:n].tobytes() != want) or r[n:pad].any() or not (r[pad:] == 0xEE).all():
            bad.append((i, "bytes"))
    return bad


def echo_problems(schema, spec, bodies, answers, resp, meta):
    """the fused GOFR_H_BIND_ECHO responses (FRAME_BODY) against the model: {"data":<the struct as encoding/json writes it>}
    or the error envelope (a syntax error: its verdict); meta status 0 exactly where HOST is allowed"""
    bad = []
    for i, (a, r, m) in enumerate(zip(answers, resp, meta)):
        code = int(m) & 0xFFFF
        if code == 0:
            if not a.host_ok or r:
                bad.append((i, "host"))
        elif a.status == G.OK:
            want = b'{"data":' + go_json(spec, schema, G.decode_row(schema, a.row)).encode() + b"}\n"
            if code != 200 or r != want:
                bad.append((i, "data"))
        elif code != 500 or not r.startswith(b'{"error":{"message":"') or (a.row is not None and r != b'{"error":{"message":' + O.json_string(a.row) + b"}}\n"):
            bad.append((i, "error"))
    return bad


def _emu_rows(which, bodies, slot):
    rows, ln, status = emu.bind_rows(Table(SPECS[which]).serialize(), 0, batch_of(bodies), slot)
    return rows, ln, status


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
def test_model_known_answers():
    """what Go 1.21 answers, written out by hand"""
    T = BIND_SCHEMA
    row = lambda i=0, name=b"", ok=0, n=0: struct.pack("<qIIi", i, len(name), ok, n) + name
    fffd = b"\xef\xbf\xbd"
    cases = [(b'{"name":"\xe2\x82a"}', row(name=fffd * 2 + b"a")),                  # one U+FFFD per byte, not per maximal subpart
             (b'{"name":"\xed\xa0\x80"}', row(name=fffd * 3)), (b'{"name":"\xf0\x9f\x98"}', row(name=fffd * 3)),
             (b'{"name":"\xef\xbf\xbd"}', row(name=fffd)),
             (b'{"name":"\\ud83d\\ude00"}', row(name="\U0001F600".encode())),
             (b'{"name":"\\ud83d\\ud83d\\ude00"}', row(name=fffd + "\U0001F600".encode())),
             (b'{"name":"\\udc00\\ud800"}', row(name=fffd * 2)), (b'{"name":"\\ud800x"}', row(name=fffd + b"x")),
             (b'{"name":"a","NAME":"b","Name":null}', row(name=b"b")), (b'{"o\xe2\x84\xaa":true}', row(ok=1)),
             (b'{"\\u0130D":5}', row()),                                              # Go folds it to "ID"; the stated deviation
             (b'{"id":-0}', row()), (b"null", row()), (b'{"n":-2147483648}', row(n=-2 ** 31)),
             (b'{"id":1e0}', b"json: cannot unmarshal number 1e0 into Go struct field T.id of type int64"),
             (b'{"n":2147483648}', b"json: cannot unmarshal number 2147483648 into Go struct field T.n of type int32"),
             (b'{"id":"x","name":5}', b"json: cannot unmarshal string into Go struct field T.id of type int64"),
             (b'{"ok":{}}', b"json: cannot unmarshal object into Go struct field T.ok of type bool"),
             (b'{"name":7}', b"json: cannot unmarshal number into Go struct field T.name of type string"),
             (b"[1]", b"json: cannot unmarshal array into Go value of type main.T"),
             (b'"s"', b"json: cannot unmarshal string into Go value of type main.T")]
    for body, want in cases:
        a = G.unmarshal(T, body)
        assert a.row == want and a.status == (G.OK if not want.startswith(b"json:") else G.ERROR) and not a.host_ok, body
    assert G.unmarshal(T, b'{"id":1,}').status == G.ERROR and G.unmarshal(T, b'{"id":1,}').row is None
    assert G.unmarshal(T, b'{"x":' + b"[" * 65 + b"]" * 65 + b"}").host_ok
    assert not G.unmarshal(T, b'{"x":' + b"[" * 63 + b"]" * 63 + b"}").host_ok


def test_corpus_reaches_its_targets():
    for which in SPECS:
        bodies, answers = corpus(which)
        schema = SPECS[which].schemas[0]
        over = [len(a.row) - row_slot(schema, len(b)) for b, a in zip(bodies, answers) if a.row is not None]
        assert {-16, -1, 0, 1} <= set(over)
        assert {a.status for a in answers} == {G.OK, G.ERROR} and any(a.host_ok for a in answers)
    assert any(a.row is None for a in corpus("kat")[1])   # syntax errors


@pytest.mark.parametrize("which", list(SPECS))
def test_emu_rows_against_model(which):
    """gofr_bind_device's device code on the CPU: every row, at a slot that holds them all and at one below them"""
    bodies, answers = corpus(which)
    ot = O.OracleTable(SPECS[which])
    schema_id = SPECS[which].schemas[0].id
    syntax = {i: ot.bind(schema_id, b)[1] for i, (b, a) in enumerate(zip(bodies, answers)) if a.row is None}
    rows, ln, status = _emu_rows(which, bodies, 16)
    full = (int(ln.max()) + 15) & ~15
    for slot in (full, (sorted(int(x) for x in ln)[len(ln) // 2] + 15) & ~15):
        rows, ln, status = _emu_rows(which, bodies, slot)
        assert row_problems(bodies, answers, status, ln, rows, slot, [syntax.get(i) for i in range(len(bodies))]) == []
        assert any(int(x) > slot for x in ln) == (slot < full)


@pytest.mark.parametrize("which", list(SPECS))
def test_oracle_against_model(which):
    bodies, answers = corpus(which)
    ot = O.OracleTable(SPECS[which])
    sid = SPECS[which].schemas[0].id
    for b, a in zip(bodies, answers):
        ok, got = ot.bind(sid, b)
        assert ok == (a.status == G.OK), b[:80]
        if a.row is not None:
            assert got == a.row, b[:80]


@pytest.mark.parametrize("mis", [0, 1, 2, 3])
@pytest.mark.parametrize("which", list(SPECS))
def test_emu_echo_against_model(which, mis):
    """the fused GOFR_H_BIND_ECHO programs (packed layout at every output misalignment)"""
    bodies, answers = corpus(which)
    spec = SPECS[which]
    out, off, meta = emu.serve(Table(spec).serialize(), batch_of(bodies), DATE, misalign=mis)
    assert echo_problems(spec.schemas[0], spec, bodies, answers, O.responses(out, off), meta) == []


_atoms = st.sampled_from([b'"id"', b'"name"', b'"ok"', b'"n"', b'"NAME"', b'"o\xe2\x84\xaa"', b'"na\xffme"', b'"\\u006eame"', b'"zz"'])
_vals = st.sampled_from(KINDS + INTS32 + INTS64 + [b'"' + t + b'"' for t in TRUNCATED + INVALID + VALID + SURR] + [b'"\\ud83d' + s[1:] for s in SURR])


@settings(max_examples=300, deadline=None)
@given(st.lists(st.lists(st.tuples(_atoms, st.sampled_from([b"", b" "]), _vals), max_size=6), min_size=1, max_size=8))
def test_emu_random_members_against_model(objs):
    bodies = [b"{" + b",".join(k + w + b":" + w + v for k, w, v in o) + b"}" for o in objs]
    answers = [G.unmarshal(BIND_SCHEMA, b) for b in bodies]
    rows, ln, status = _emu_rows("kat", bodies, 1024)
    assert row_problems(bodies, answers, status, ln, rows, 1024) == []


def test_model_catches_planted_mistakes(monkeypatch):
    """each of three plausible misreadings of Go, planted in the model, disagrees with the device on the corpus"""
    bodies, answers = corpus("kat")
    rows, ln, status = _emu_rows("kat", bodies, 1024)
    ot = O.OracleTable(KAT_SPEC)
    syntax = [ot.bind(7, b)[1] if a.row is None else None for b, a in zip(bodies, answers)]

    def problems():
        return row_problems(bodies, [G.unmarshal(BIND_SCHEMA, b) for b in bodies], status, ln, rows, 1024, syntax)
    assert problems() == []
    # Python's decoder: one U+FFFD per maximal subpart of an invalid sequence
    real_unquote = G.unquote
    with monkeypatch.context() as m:
        m.setattr(G, "unquote", lambda s: real_unquote(s.decode("utf-8", "replace").encode("utf-8")))
        assert problems()
    # the first of several equal (or folded) keys wins
    real_value = G._value

    def first_wins(b, i):
        (kind, payload), end = real_value(b, i)
        if kind == "object":
            seen, kept = set(), []
            for k, v in payload:
                if G.fold(real_unquote(k)) not in seen:
                    seen.add(G.fold(real_unquote(k)))
                    kept.append((k, v))
            payload = kept
        return (kind, payload), end
    with monkeypatch.context() as m:
        m.setattr(G, "_value", first_wins)
        assert problems()
    # the old slot rule: a row longer than its body's first slot is not bound (HOST)
    real = G.unmarshal

    def dropping(schema, body, float_defer=None):
        a = real(schema, body, float_defer)
        if a.row is not None and len(a.row) > row_slot(schema, len(body)):
            return G.Answer(G.HOST, None, True)
        return a
    assert row_problems(bodies, [dropping(BIND_SCHEMA, b) for b in bodies], status, ln, rows, 1024, syntax)


def test_row_bound_at_its_worst_case():
    """GOFR_BIND_ROW_BOUND holds for the corpus, and at the two worst cases it is derived from: a string of invalid bytes
    only, and the longest number literal in an error text naming the longest Go type and JSON name"""
    for which in SPECS:
        schema = SPECS[which].schemas[0]
        for b, a in zip(*corpus(which)):
            assert a.row is None or len(a.row) <= row_bound(schema, len(b))
    worst = [(BIND_SCHEMA, b'{"name":"' + b"\xff" * 5000 + b'"}'), (LONG_SCHEMA, b'{"note":"' + b"\x80" * 5000 + b'"}'),
             (LONG_SCHEMA, b'{"' + b"n" * LONG + b'":' + b"9" * 3000 + b"}"), (LONG_SCHEMA, b'{"small":' + b"9" * 3000 + b".5e-7}")]
    rows = []
    for schema, body in worst:
        spec = KAT_SPEC if schema is BIND_SCHEMA else LONG_SPEC
        a = G.unmarshal(schema, body)
        r, ln, st_ = emu.bind_rows(Table(spec).serialize(), 0, batch_of([body]), 32768)
        assert int(st_[0]) == a.status and r[0, :int(ln[0])].tobytes() == a.row
        rows.append((len(a.row), row_bound(schema, len(body)), len(body)))
    assert all(n <= bound for n, bound, _ in rows)
    # the invalid-byte strings use 3 bytes per body byte: the bound is tight but for the JSON around the string
    assert rows[0][1] - rows[0][0] <= 3 * 12 + 70 + len(BIND_SCHEMA.go_type) + 4 + 8 * 4
    # the syntax error texts and the longest scanner context fit the 70 bytes stated for them
    assert len(b"invalid character '\\u00ff' looking for beginning of object key string") <= 70


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
def _run_child(fn):
    r = subprocess.run([sys.executable, "-c", "import tests.test_bind_unmarshal as t; t.%s()" % fn], cwd=ROOT,
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-4000:]
    return r.stdout


def _gpu_bind_check():
    """gofr_bind_device over each corpus at batch sizes 1, 31, 32, 33 and 65 536 (the corpus repeated), slots at the longest
    row and below the row lengths; rows pre-filled with 0xEE"""
    import torch
    from gofr_b200.engine import Engine
    for which, spec in SPECS.items():
        bodies, answers = corpus(which)
        ot = O.OracleTable(spec)
        sid = spec.schemas[0].id
        syntax = [ot.bind(sid, b)[1] if a.row is None else None for b, a in zip(bodies, answers)]
        lens = sorted(len(a.row if a.row is not None else s) for a, s in zip(answers, syntax))
        full = (lens[-1] + 15) & ~15
        eng = Engine(Table(spec), 0)
        for n in (1, 31, 32, 33, 65536):
            idx = [(k * 7 + n) % len(bodies) for k in range(n)]   # n = 1 .. 33 take different bodies; 65 536 repeats them
            b = [bodies[i] for i in idx]
            db = eng.upload(batch_of(b))
            for slot in (full, (lens[len(lens) // 2] + 15) & ~15):
                pre = torch.full((n * slot,), 0xEE, dtype=torch.uint8, device="cuda")
                rows, ln, status = eng.bind_device(db, sid, slot, rows=pre)
                torch.cuda.synchronize()
                rows = rows.cpu().numpy().reshape(n, slot)
                ln, status = ln.cpu().numpy().view(np.uint32), status.cpu().numpy().view(np.uint32)
                bad = _grouped_row_problems(idx, bodies, answers, syntax, status, ln, rows, slot)
                assert bad == [], (which, n, slot, bad[:5], [bodies[idx[i]][:60] for i, _ in bad[:5]])
                print(which, n, slot, "rows ok", int((ln > slot).sum()), "past the slot", int((status == 2).sum()), "host")
        eng.close()


def _grouped_row_problems(idx, bodies, answers, syntax, status, ln, rows, slot):
    """row_problems for a batch whose request k is corpus body idx[k], one comparison per distinct body"""
    by = {}
    for k, i in enumerate(idx):
        by.setdefault(i, []).append(k)
    bad = []
    for i, ks in by.items():
        ks = np.array(ks)
        st_, n_ = status[ks], ln[ks]
        if (st_ != st_[0]).any() or (n_ != n_[0]).any() or (rows[ks] != rows[ks[0]]).any():
            bad.append((int(ks[0]), "requests with the same body differ"))
            continue
        for _, why in row_problems([bodies[i]], [answers[i]], st_[:1], n_[:1], rows[ks[:1]], slot, [syntax[i]]):
            bad.append((int(ks[0]), why))
    return bad


def _gpu_echo_check():
    """the fused GOFR_H_BIND_ECHO serve kernels, packed and slot layout, over each corpus repeated to 65 536 requests"""
    import torch
    from gofr_b200.engine import Engine
    for which, spec in SPECS.items():
        schema = spec.schemas[0]
        bodies, answers = corpus(which)
        n = 65536
        idx = [k % len(bodies) for k in range(n)]
        batch = batch_of([bodies[i] for i in idx])
        eng = Engine(Table(spec), 0)
        o1, f1, _ = O.OracleTable(spec).serve(batch_of(bodies), DATE, out_cap=sum(6 * len(b) + 4 * LONG + 4096 for b in bodies))
        lens = np.diff(f1.astype(np.int64))
        longest = int(lens.max())
        db = eng.upload(batch)
        resp = eng.alloc_responses(n, int(lens[idx].sum()) + 1024)
        eng.serve_device(db, DATE, resp)
        torch.cuda.synchronize()
        assert not eng.overflowed()
        out, off, meta = resp.to_host()
        packed = O.responses(out, off)
        slot = (longest + 15) & ~15
        s_out, s_len, s_meta = eng.serve_device_slots(db, DATE, slot)
        torch.cuda.synchronize()
        s_out = s_out.cpu().numpy().reshape(n, slot)
        s_len, s_meta = s_len.cpu().numpy().view(np.uint32), s_meta.cpu().numpy().view(np.uint32)
        sloted = [s_out[k, :int(s_len[k])].tobytes() for k in range(n)]
        for got, m in ((packed, meta), (sloted, s_meta)):
            first = {}
            for k, i in enumerate(idx):
                if i in first:
                    assert got[k] == got[first[i]] and m[k] == m[first[i]], (which, k)
                else:
                    first[i] = k
            ks = [first[i] for i in range(len(bodies))]
            bad = echo_problems(schema, spec, bodies, answers, [got[k] for k in ks], [m[k] for k in ks])
            assert bad == [], (which, bad[:5], [bodies[i][:60] for i, _ in bad[:5]])
        print(which, "echo ok", sum(1 for m in meta if (int(m) & 0xFFFF) == 0), "host")
        eng.close()


@pytest.mark.gpu
def test_gpu_bind_device_against_model():
    out = _run_child("_gpu_bind_check")
    assert out.count("rows ok") == 2 * 5 * 2


@pytest.mark.gpu
def test_gpu_bind_echo_against_model():
    out = _run_child("_gpu_echo_check")
    assert out.count("echo ok") == 2


@pytest.mark.gpu
def test_gpu_cpp_app_entries_bind_alike(tmp_path):
    """Serve, ServeConnections and ServeRead of the C++ App: every closure's c.Bind gives the model's row (or its error),
    and all three entries answer with the same bytes.  A 300-byte body of invalid UTF-8 (a 920-byte row, its first slot
    608 bytes) alone in its batch and next to a longer batch-mate."""
    from gofr_b200 import _abi
    from tests.test_cpp_app import _compile
    _abi.lib()
    exe = str(tmp_path / "app_bind_entries")
    _compile(os.path.join(ROOT, "tests", "emu", "app_bind_entries.cpp"), exe)
    bodies, answers = corpus("kat")
    ff = b'{"name":"' + b"\xff" * 300 + b'"}'
    mate = b'{"name":"' + b"m" * 700 + b'"}'
    assert len(G.unmarshal(BIND_SCHEMA, ff).row) > row_slot(BIND_SCHEMA, len(ff))
    groups = [bodies, [ff], [ff, mate], [mate, ff, b'{"id":1}']]
    lines = "".join(",".join(b.hex() or "-" for b in g) + "\n" for g in groups)
    r = subprocess.run([exe], input=lines, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = {}
    for line in r.stdout.splitlines():
        entry, g, k, bind, body = line.split(" ")
        got[(entry, int(g), int(k))] = (bytes.fromhex(bind) if bind != "-" else b"", bytes.fromhex(body) if body != "-" else b"")
    for g, group in enumerate(groups):
        for k, body in enumerate(group):
            a = G.unmarshal(BIND_SCHEMA, body)
            seen = {e: got[(e, g, k)] for e in ("serve", "conns", "read")}
            assert seen["serve"] == seen["conns"] == seen["read"], (g, k, body[:60])
            bind, _ = seen["serve"]
            if a.host_ok:
                continue
            if a.row is None:
                assert bind[:1] == b"E", body[:60]
            else:
                assert bind == (b"O" if a.status == G.OK else b"E") + a.row, (g, k, body[:60], bind[:80])
