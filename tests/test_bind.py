"""Config 3 — Request.Bind + echo.  CPU: the kernel's device code (tests/emu) vs the oracle on the known-answer lists of
test_oracle_golden.py, the synthetic config-3 stream and random JSON-ish bodies.  GPU (-m gpu): the CUDA kernel."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import oracle as O
from tests.emu import emu
from tests.test_oracle_golden import BIND_ERR_KAT, BIND_OK_KAT, BIND_SCHEMA

DATE = S.http_date(1789974595)
KAT_SPEC = S.TableSpec(schemas=[BIND_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=7)])
OE_SCHEMA = S.Schema(8, "pkg.Opt", [S.Field("A", S.F_STRING, "a", True), S.Field("B", S.F_INT, "b", True),
                                    S.Field("C", S.F_BOOL, "c", True), S.Field("D", S.F_STRING, "d")])


def _cmp(spec, bodies, mis=1, frame=S.FRAME_WIRE):
    spec.frame_mode = frame
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    o2, f2, m2 = emu.serve(Table(spec).serialize(), batch, DATE, misalign=mis)
    for i, (a, b) in enumerate(zip(O.responses(o1, f1), O.responses(o2, f2))):
        assert a == b, (bodies[i], a, b)
    assert (m1 == m2).all()
    return O.responses(o1, f1), m1


@pytest.mark.parametrize("mis", [0, 1, 2, 3])
def test_emu_known_answer_bodies(mis):
    bodies = [b for b, _ in BIND_ERR_KAT] + [b for b, _ in BIND_OK_KAT]
    res, meta = _cmp(KAT_SPEC, bodies, mis, S.FRAME_BODY)
    for (body, want), r, m in zip(BIND_ERR_KAT, res, meta):
        assert (m & 0xFFFF) == 500
        assert r == b'{"error":{"message":' + O.json_string(want) + b"}}\n"
    for r, m in zip(res[len(BIND_ERR_KAT):], meta[len(BIND_ERR_KAT):]):
        assert (m & 0xFFFF) == 200 and r.startswith(b'{"data":{"id":')


def test_emu_error_characters():
    """quoteChar over every byte value, in the contexts where the scanner reports it."""
    bodies = [bytes([c]) for c in range(256)] + [b'{"name":"' + bytes([c]) + b'"}' for c in range(0x20)] + \
             [b'{"name":"\\' + bytes([c]) + b'"}' for c in range(0x20, 0x80)] + [b'{"id":1' + bytes([c]) + b"}" for c in range(256)]
    _cmp(KAT_SPEC, bodies, 2)


def test_emu_omitempty_and_nesting():
    spec = S.TableSpec(schemas=[OE_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=8)])
    bodies = [b"{}", b'{"a":"","b":0,"c":false,"d":""}', b'{"a":"x","b":-5,"c":true,"d":"y"}', b'{"A":"\\u0041","D":"<&>"}',
              b'{"x":' + b"[" * 63 + b"]" * 63 + b"}", b'{"d":{"a":{"a":{"a":1}}},"a":"q"}',
              b'{"b":9223372036854775807}', b'{"b":9223372036854775808}', b'{"b":-9223372036854775808}', b'{"b":-9223372036854775809}',
              b'{"b":1e2}', b'{"b":12.0}', b'{"b":-0}', b' \t\r\n{ "d" : "v" } \n', b'{"d":"v"} x', b'{"\\u0064":"esc-key"}']
    for mis in range(4):
        _cmp(spec, bodies, mis)


def test_deep_nesting_is_deferred_to_the_host():
    """> 64 levels: the device does not decide (status 0, nothing emitted); the oracle shows what Go answers."""
    spec = S.TableSpec(schemas=[OE_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=8)])
    deep = b'{"x":' + b"[" * 70 + b"]" * 70 + b',"d":"ok"}'
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", deep), S.Req(S.M_POST, b"/echo", b"", b'{"d":"ok"}')])
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    o2, f2, m2 = emu.serve(Table(spec).serialize(), batch, DATE)
    r1, r2 = O.responses(o1, f1), O.responses(o2, f2)
    assert (m1[0] & 0xFFFF) == 200 and (m2[0] & 0xFFFF) == 0 and r2[0] == b"" and (m2[0] >> 16) == 0
    assert r1[1] == r2[1] and m1[1] == m2[1]


@pytest.mark.parametrize("mode", [S.FRAME_WIRE, S.FRAME_BODY])
def test_emu_config3_stream(mode):
    _cmp_batch = synth.config3_batch(6000, variant_every=7)
    spec = synth.config3_spec(mode)
    o1, f1, m1 = O.OracleTable(spec).serve(_cmp_batch, DATE)
    o2, f2, m2 = emu.serve(Table(spec).serialize(), _cmp_batch, DATE, misalign=3)
    assert O.responses(o1, f1) == O.responses(o2, f2) and (m1 == m2).all()
    assert {int(m) & 0xFFFF for m in m1} == {200, 500}


_json_atoms = st.sampled_from([b'{', b'}', b'[', b']', b':', b',', b'"', b'\\', b'u', b'00e9', b'd83d', b'"id"', b'"name"', b'"ok"',
                               b'"n"', b'1', b'-', b'0', b'.5', b'e9', b'true', b'false', b'null', b' ', b'\n', b'x', b'\xc3\xa9',
                               b'\xff', b'<', b'"a\\nb"', b'123456789012345678901', b'"\\ud800"', b'NaMe', b'\\u212a'])


@settings(max_examples=300, deadline=None)
@given(st.lists(st.lists(_json_atoms, min_size=0, max_size=14).map(b"".join), min_size=1, max_size=8), st.integers(0, 3))
def test_emu_random_bodies(bodies, mis):
    _cmp(KAT_SPEC, bodies, mis)


@settings(max_examples=150, deadline=None)
@given(st.lists(st.tuples(st.integers(-2 ** 63, 2 ** 63 - 1), st.text(max_size=12), st.booleans(), st.integers(-2 ** 31, 2 ** 31 - 1)),
                min_size=1, max_size=6), st.integers(0, 3))
def test_emu_valid_json_roundtrip(rows, mis):
    """Bodies produced by a real JSON encoder (python json): bind + echo must reproduce the values."""
    import json
    bodies = [json.dumps({"id": i, "name": s, "ok": b, "n": n}).encode() for i, s, b, n in rows]
    res, meta = _cmp(KAT_SPEC, bodies, mis, S.FRAME_BODY)
    for (i, s, b, n), r in zip(rows, res):
        assert json.loads(r)["data"] == {"id": i, "name": s, "ok": b, "n": n}


@pytest.mark.gpu
def test_gpu_config3_full_size():
    from tests.test_gpu_parity import _check
    _check(synth.config3_spec(), synth.config3_batch(65536))


@pytest.mark.gpu
def test_gpu_bind_edge_cases_and_host_path():
    from tests.test_gpu_parity import _check
    bodies = ([b for b, _ in BIND_ERR_KAT] + [b for b, _ in BIND_OK_KAT]) * 30
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    _check(KAT_SPEC, batch)
    _check(synth.config3_spec(), synth.config3_batch(20000, variant_every=5), host=True, chunk=3000)


@settings(max_examples=400, deadline=None)
@given(st.lists(st.lists(_json_atoms, min_size=0, max_size=14).map(b"".join), min_size=1, max_size=8))
def test_syntax_verdict_agrees_with_python_json(bodies):
    """Independent check of the scanner: a body Python's json module rejects as malformed must not bind (Go's decoder
    checks the whole document before it stores anything), and a body that binds is something Python can load.  The
    two parsers disagree only on things this generator avoids or that are filtered below: NaN / Infinity literals
    (Python extension) and raw bytes that are not UTF-8 (Python refuses to decode the document, Go replaces them)."""
    import json
    spec = KAT_SPEC
    spec.frame_mode = S.FRAME_BODY
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    out, off, meta = O.OracleTable(spec).serve(batch, DATE)
    for b, r, m in zip(bodies, O.responses(out, off), meta):
        try:
            text = b.decode("utf-8")
        except UnicodeDecodeError:
            continue
        try:
            doc = json.loads(text, parse_constant=lambda c: (_ for _ in ()).throw(ValueError(c)))
            py_ok = True
        except ValueError:
            py_ok = False
        bound = (int(m) & 0xFFFF) == 200
        if not py_ok:
            assert not bound, (b, r)
            assert b"invalid character" in r or b"unexpected end of JSON input" in r or b"invalid" in r or b"cannot unmarshal" in r, (b, r)
        elif bound:
            assert isinstance(doc, dict) or doc is None, (b, r)   # only an object (or null) binds into a struct


# ---- Bind as a stage of the split API (gofr_bind_device): body -> typed row | err.Error(), for closures on the host ----

def _bind_stage_bodies():
    bodies = [b for b, _ in BIND_ERR_KAT] + [b for b, _ in BIND_OK_KAT]
    bodies += [b'{"id":1,"name":"caf\\u00e9 \\ud83d\\ude00 \\ud800 x","email":"a\\"b\\\\c\\/d\\n","active":true,"count":-7}',
               b'{"name":"\xff\xfe raw bytes \xc3\xa9"}', b'{"NAME":"folded key","Id":12}', b'{"id":null,"name":null}',
               b'{"name":"' + b"x" * 900 + b'"}', b"{}", b"null", b"[1,2]", b'"str"', b"12", b"",
               b'{"x":' + b"[" * 70 + b"]" * 70 + b"}"]
    return bodies


def _check_bind_stage(rows, ln, status, bodies, slot, ot, schema_id):
    for i, body in enumerate(bodies):
        ok, want = ot.bind(schema_id, body)
        deep = body.count(b"[") > 64
        if deep:
            assert status[i] == 2 and ln[i] == 0, i          # the device does not decide; Go (the oracle) does
            continue
        assert status[i] == (0 if ok else 1), (i, body, status[i])
        assert ln[i] == len(want), (i, body, ln[i], len(want))
        if ln[i] <= slot:
            assert rows[i, :ln[i]].tobytes() == want, (i, body, rows[i, :ln[i]].tobytes(), want)
            pad = (-int(ln[i])) % 16
            assert (rows[i, ln[i]:ln[i] + pad] == 0).all()


def test_emu_bind_stage_known_answers():
    """the device code of gofr_bind_device on the CPU against the oracle's json.Unmarshal restatement (orc_bind): the
    reference's pins (request_test.go:17-30, context_test.go:23-49 are in BIND_OK_KAT), every error text, escapes,
    invalid UTF-8, case-folded keys, oversize strings, non-object documents, deep nesting"""
    bodies = _bind_stage_bodies()
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    slot = 512
    rows, ln, status = emu.bind_rows(Table(KAT_SPEC).serialize(), 0, batch, slot)
    _check_bind_stage(rows, ln, status, bodies, slot, O.OracleTable(KAT_SPEC), 7)
    assert any(l > slot for l in ln)                         # the 900-byte string did not fit: reported, not written


def test_emu_bind_stage_config3_stream():
    batch = synth.config3_batch(3000, variant_every=5)
    spec = synth.config3_spec()
    bodies = []
    ar = batch.arena.tobytes()
    for d in batch.desc:
        a = (int(d["arena_off"]) + int(d["path_len"]) + int(d["query_len"]) + 3) & ~3
        bodies.append(ar[a:a + int(d["data_len"])])
    rows, ln, status = emu.bind_rows(Table(spec).serialize(), 0, batch, 1024)
    _check_bind_stage(rows, ln, status, bodies, 1024, O.OracleTable(spec), spec.schemas[0].id)
    assert set(int(s) for s in status) == {0, 1}


@pytest.mark.gpu
def test_gpu_bind_stage():
    import torch
    from gofr_b200.engine import Engine
    bodies = _bind_stage_bodies()
    eng = Engine(Table(KAT_SPEC), 0)
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    rows, ln, status = eng.bind_device(eng.upload(batch), 7, 512)
    torch.cuda.synchronize()
    _check_bind_stage(rows.cpu().numpy().reshape(batch.n, 512), ln.cpu().numpy().view(np.uint32), status.cpu().numpy().view(np.uint32),
                      bodies, 512, O.OracleTable(KAT_SPEC), 7)
    eng.close()
    spec = synth.config3_spec()
    eng = Engine(Table(spec), 0)
    batch = synth.config3_batch(65536, variant_every=9)
    ar = batch.arena.tobytes()
    bodies = []
    for d in batch.desc:
        a = (int(d["arena_off"]) + int(d["path_len"]) + int(d["query_len"]) + 3) & ~3
        bodies.append(ar[a:a + int(d["data_len"])])
    rows, ln, status = eng.bind_device(eng.upload(batch), spec.schemas[0].id, 1024)
    torch.cuda.synchronize()
    r, l, s = rows.cpu().numpy().reshape(batch.n, 1024), ln.cpu().numpy().view(np.uint32), status.cpu().numpy().view(np.uint32)
    idx = list(range(0, batch.n, 13))
    _check_bind_stage(r[idx], l[idx], s[idx], [bodies[i] for i in idx], 1024, O.OracleTable(spec), spec.schemas[0].id)
    eng.close()


# ---- float64 targets (round 2): strconv.ParseFloat's correctly rounded value where ONE IEEE operation gives it, the
#      host otherwise — checked against Python's float(), which rounds correctly too ----
FL_SCHEMA = S.Schema(9, "pkg.Reading", [S.Field("Name", S.F_STRING, "name"), S.Field("Value", S.F_FLOAT64, "value"),
                                        S.Field("Delta", S.F_FLOAT64, "delta", True), S.Field("N", S.F_INT, "n")])
FL_SPEC = S.TableSpec(schemas=[FL_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=9)])


def _float_cmp(bodies, mis=1):
    """device code vs oracle on every body the device decides; returns the indices it left to the host"""
    FL_SPEC.frame_mode = S.FRAME_BODY
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    o1, f1, m1 = O.OracleTable(FL_SPEC).serve(batch, DATE)
    o2, f2, m2 = emu.serve(Table(FL_SPEC).serialize(), batch, DATE, misalign=mis)
    r1, r2 = O.responses(o1, f1), O.responses(o2, f2)
    # the same requests through the slot layout of the device code (what gofr_serve_device_slots runs)
    s_out, s_len, s_meta = emu.serve_slots(Table(FL_SPEC).serialize(), batch, DATE, 1024)
    s_out = np.asarray(s_out).reshape(batch.n, 1024)
    deferred = []
    for i, b in enumerate(bodies):
        if (m2[i] & 0xFFFF) == 0:
            assert r2[i] == b"" and s_len[i] == 0 and (s_meta[i] & 0xFFFF) == 0, b
            deferred.append(i)
        else:
            assert r1[i] == r2[i] and m1[i] == m2[i], (b, r1[i], r2[i])
            assert s_meta[i] == m1[i] and s_out[i, :int(s_len[i])].tobytes() == r1[i], b
    return r1, deferred


def test_emu_bind_float_known_answers():
    import json
    lits = [b"0", b"-0", b"0.0", b"-0.0e5", b"1", b"-1", b"1.5", b"3.14159", b"1e2", b"1E+2", b"1e-2", b"100", b"1e21", b"1e20", b"1e-6", b"1e-7",
            b"123456789012345", b"9007199254740991", b"0.1", b"0.2", b"0.30000000000000004", b"2.5e-5", b"1e22", b"1e23", b"123e35", b"1.7976931348623157e308",
            b"1e400", b"-1e400", b"1e-400", b"-1e-400", b"1e309", b"1e310", b"4.9e-324", b"2.2250738585072014e-308", b"9007199254740993",
            b"0.000000000000000000000000000001", b"1" + b"0" * 30, b"1" + b"0" * 400, b"0." + b"0" * 400 + b"1", b"12345678901234567890123",
            b"1.00000000000000000000000000000000001", b"1e0000000000000000000002", b"1e-0000000000000000000002", b"5e-1", b"625e-4",
            b"123456789012345678", b"8.5e-310", b"1.7976931348623158e308", b"1.7976931348623159e308", b"9007199254740992.5",
            b"9007199254740993.0000000000000000000001", b"0.1234567890123456789012345", b"7.2057594037927933e16", b"1e-320"]
    bodies = [b'{"name":"s","value":' + x + b',"n":3}' for x in lits]
    r1, deferred = _float_cmp(bodies)
    decided = 0
    for i, x in enumerate(lits):
        v = float(x)
        if v in (float("inf"), float("-inf")):  # ErrRange -> UnmarshalTypeError naming the literal
            assert json.loads(r1[i])["error"]["message"] == "json: cannot unmarshal number " + x.decode() + " into Go struct field Reading.value of type float64"
        else:
            assert float(json.loads(r1[i])["data"]["value"]) == v, x  # the oracle's strtod against Python's float() (an integral
            # float is written without a point: json.loads makes it an int)
        decided += i not in deferred
    # nearly everything is decided on the device (exact cases, then Eisel-Lemire); what is left for the host: exact half-way
    # literals, subnormals, the last decade before the overflow threshold
    for x in (b"0", b"-0", b"1.5", b"3.14159", b"1e22", b"1e23", b"123e35", b"0.1", b"1e400", b"-1e400", b"1e-400", b"1e310", b"9007199254740991",
              b"1" + b"0" * 30, b"1" + b"0" * 400, b"0." + b"0" * 400 + b"1", b"625e-4", b"1e0000000000000000000002",
              b"1.7976931348623157e308", b"12345678901234567890123", b"1.00000000000000000000000000000000001", b"0.30000000000000004",
              b"2.2250738585072014e-308"):
        assert lits.index(x) not in deferred, x
    for x in (b"9007199254740993", b"4.9e-324", b"1e309"):
        assert lits.index(x) in deferred, x
    assert decided >= 40


def test_emu_bind_float_type_errors_and_omitempty():
    bodies = [b'{"value":"1.5"}', b'{"value":true}', b'{"value":[1]}', b'{"value":{}}', b'{"value":null,"n":2}', b'{"n":1.5}', b'{"n":1e2}',
              b'{"value":1,"delta":0}', b'{"value":1,"delta":-0.0}', b'{"value":1,"delta":0.5}', b'{"VALUE":2.5,"Delta":1e-7}',
              b'{"value":1e400,"n":"x"}', b'{"n":"x","value":1e400}', b'{"value":1e400,"value":2}', b'{"name":3.5}', b'3.5', b'{"value":1.5,"value":"s"}',
              # a literal the device cannot round decides the whole request, whatever else is wrong with it
              b'{"n":"x","value":9007199254740993}']
    for mis in range(4):
        r1, deferred = _float_cmp(bodies, mis)
        assert deferred == [len(bodies) - 1]
    assert r1[7] == b'{"data":{"name":"","value":1,"n":0}}\n' and r1[8] == r1[7] and r1[9] == b'{"data":{"name":"","value":1,"delta":0.5,"n":0}}\n'
    assert r1[10] == b'{"data":{"name":"","value":2.5,"delta":1e-7,"n":0}}\n'
    assert b"cannot unmarshal number 1e400 into Go struct field Reading.value of type float64" in r1[11]
    assert b"cannot unmarshal string into Go struct field Reading.n of type int" in r1[12]


def test_emu_bind_float_bulk_against_strtod():
    """bd_parse_float on 2 million generated literals against glibc's correctly rounded strtod (scratch/parse_float_campaign.py
    runs 420 million: profiles/r02/parse_float_campaign.txt): no decided literal may differ; encoder output (the 15 .. 17 digit
    texts of random doubles) is decided on the device practically always"""
    import ctypes as C
    L = emu.lib()
    L.emu_parse_float_check.argtypes = [C.c_uint64, C.c_uint64, C.c_int, C.POINTER(C.c_uint64), C.c_char_p, C.c_uint32]
    for mode in range(4):
        out = (C.c_uint64 * 4)()
        bad = C.create_string_buffer(600)
        L.emu_parse_float_check(99 + mode, 500_000, mode, out, bad, 600)
        assert out[2] == 0, (mode, bad.value)
        assert out[0] + out[1] == 500_000
        if mode == 1:
            assert out[1] < 2000   # ~0.1 %: subnormals and the like
        if mode == 2:
            assert out[1] > 10000  # the exact half-way integers must NOT be decided


@settings(max_examples=200, deadline=None)
@given(st.lists(st.one_of(
    st.floats(allow_nan=False, allow_infinity=False).map(lambda v: repr(v).encode()),
    st.tuples(st.integers(0, 10 ** 17), st.integers(-30, 30)).map(lambda t: b"%de%d" % t),
    st.tuples(st.integers(0, 10 ** 9), st.integers(0, 10 ** 9), st.integers(-12, 12)).map(lambda t: b"-%d.%09dE%+d" % t),
    st.decimals(allow_nan=False, allow_infinity=False, places=6, min_value=-10 ** 8, max_value=10 ** 8).map(lambda d: format(d, "f").encode())),
    min_size=1, max_size=12), st.integers(0, 3))
def test_emu_bind_float_against_python_float(lits, mis):
    """every literal the device decides carries exactly the double Python's float() — correctly rounded, like
    strconv.ParseFloat — gives; literals with at most 15 digits and a small exponent are always decided"""
    import json, struct
    lits = [x if x[:1] != b"-" or x[1:2].isdigit() else x[1:] for x in lits]
    bodies = [b'{"value":' + x + b"}" for x in lits]
    r1, deferred = _float_cmp(bodies, mis)
    for i, x in enumerate(lits):
        if i in deferred:   # only what Eisel-Lemire cannot settle: half-way literals (17+ digits), subnormals, the top decade
            digits = x.split(b"e")[0].split(b"E")[0].replace(b"-", b"").replace(b".", b"").lstrip(b"0").rstrip(b"0")
            assert len(digits) > 15 or abs(float(x)) > 1e307 or (float(x) != 0 and abs(float(x)) < 2.3e-308), x
        else:
            got = float(json.loads(r1[i])["data"]["value"])
            assert struct.pack("<d", got) == struct.pack("<d", float(x)) or (got == 0 and float(x) == 0), (x, got)


def test_emu_bind_stage_float_fields():
    """gofr_bind_device with float64 members: the value's bits as two row words (like INT64), ErrRange as the error text,
    GOFR_BIND_HOST for literals the device does not round itself"""
    import struct
    bodies = [b'{"name":"a","value":1.5,"delta":-2.5e-3,"n":7}', b'{"value":1e400}', b'{"value":0.1,"delta":1e23}', b'{"value":"x"}',
              b'{"value":9007199254740993}', b'{"value":-0}', b'{"value":123456789.125,"name":"caf\\u00e9"}']
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    rows, ln, status = emu.bind_rows(Table(FL_SPEC).serialize(), 0, batch, 256)
    ot = O.OracleTable(FL_SPEC)
    for i, body in enumerate(bodies):
        ok, want = ot.bind(9, body)
        if i == 4:
            assert status[i] == 2 and ln[i] == 0
            continue
        assert status[i] == (0 if ok else 1) and rows[i, :ln[i]].tobytes() == want, (body, rows[i, :ln[i]].tobytes(), want)
    # layout: name length, value bits, delta bits, n (two words), then the string bytes
    assert rows[0, :ln[0]].tobytes() == struct.pack("<IddqB", 1, 1.5, -2.5e-3, 7, ord("a"))
    assert rows[5, 4:12].tobytes() == struct.pack("<d", -0.0)


def _gpu_float_check():
    import torch
    from gofr_b200.engine import Engine
    rng = np.random.default_rng(5)
    bodies = []
    for i in range(20000):
        v = float(rng.integers(-10 ** 9, 10 ** 9)) / 10 ** int(rng.integers(0, 9))
        d = [b"0", b"1e-7", b"2.5e21", b"-0.0", b"1e400", b'"s"', b"9007199254740993"][i % 7]   # the last one: exactly half-way, left to the host
        bodies.append(b'{"name":"r%d","value":%s,"delta":%s,"n":%d}' % (i, repr(v).encode(), d, i))
    FL_SPEC.frame_mode = S.FRAME_WIRE
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    # packed and slot layouts against the oracle; requests the device leaves to the host (status 0) are skipped there
    eng = Engine(Table(FL_SPEC), 0)
    o1, f1, m1 = O.OracleTable(FL_SPEC).serve(batch, DATE)
    s_out, s_len, s_meta = eng.serve_device_slots(eng.upload(batch), DATE, 1024)
    torch.cuda.synchronize()
    s_out = s_out.cpu().numpy().reshape(batch.n, 1024)
    s_len, s_meta = s_len.cpu().numpy().view(np.uint32), s_meta.cpu().numpy().view(np.uint32)
    host = 0
    for i in range(batch.n):
        if (s_meta[i] & 0xFFFF) == 0:
            assert s_len[i] == 0 and i % 7 == 6, i
            host += 1
            continue
        L = int(f1[i + 1]) - int(f1[i])
        assert s_meta[i] == m1[i] and s_len[i] == L and s_out[i, :L].tobytes() == o1[int(f1[i]):int(f1[i + 1])].tobytes(), (i, bodies[i])
    assert host == len(range(6, batch.n, 7))
    rows, ln, status = eng.bind_device(eng.upload(batch), 9, 256)
    torch.cuda.synchronize()
    rows, ln, status = rows.cpu().numpy().reshape(batch.n, 256), ln.cpu().numpy().view(np.uint32), status.cpu().numpy().view(np.uint32)
    ot = O.OracleTable(FL_SPEC)
    for i in range(0, batch.n, 3):
        ok, want = ot.bind(9, bodies[i])
        if i % 7 == 6:
            assert status[i] == 2
        else:
            assert status[i] == (0 if ok else 1) and rows[i, :ln[i]].tobytes() == want, (i, bodies[i])
    eng.close()


@pytest.mark.gpu
def test_gpu_bind_float_fields():
    """the serve kernels (VALUES instance, PF_BIND program with OP_F64) and gofr_bind_device on 20 000 bodies with float64
    members — in a child process, so that a fault cannot leave a sticky CUDA error behind for the other GPU tests"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import tests.test_bind as t; t._gpu_float_check()"], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
