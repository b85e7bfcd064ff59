"""Respond's wider data model (VERDICT r01 item 6): float64, nested structs, pointers, slices, map[string]T and bare
(non-struct) values, encoded as encoding/json does (pkg/gofr/http/responder.go:32-40).

Three independent statements of the same rules are compared:
  * `go_json` below — Python: dict / list walking, sorted(keys), float text derived from repr() (shortest round-trip
    digits, like strconv's) re-formatted the way encoding/json's floatEncoder does;
  * the oracle (oracle/orc_value.c) — C, walks the row, finds shortest digits by printf / strtod search;
  * the device code (value_device.cuh, float_device.cuh: Ryu) — on the CPU through tests/emu, on the GPU with -m gpu."""
import math
import random
import struct
from decimal import Decimal

import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200.table import Table
from tests import go_net_url as G
from tests import oracle as O
from tests.emu import emu as E

DATE = S.http_date(1_700_000_000)


# ---------------------------------------------------------------------------------------------------------------
# Python model
# ---------------------------------------------------------------------------------------------------------------
def go_json_float(x: float) -> str:
    """encoding/json floatEncoder: strconv.AppendFloat(b, f, 'f' or 'e', -1, 64), 'e' when abs < 1e-6 or abs >= 1e21, and
    "e-0X" cleaned to "e-X".  "" for NaN / Inf (UnsupportedValueError)."""
    if x != x or x in (math.inf, -math.inf):
        return ""
    if x == 0:
        return "-0" if math.copysign(1, x) < 0 else "0"
    sign = "-" if x < 0 else ""
    t = Decimal(repr(abs(x))).as_tuple()
    raw = "".join(map(str, t.digits))
    digs = raw.lstrip("0")
    exp = t.exponent + len(raw) - 1 - (len(raw) - len(digs))   # decimal exponent of the first significant digit
    digs = digs.rstrip("0") or "0"
    if abs(x) < 1e-6 or abs(x) >= 1e21:
        s = digs[0] + ("." + digs[1:] if len(digs) > 1 else "") + "e" + ("-" if exp < 0 else "+") + "%02d" % abs(exp)
        if s[-4:-1] == "e-0":
            s = s[:-2] + s[-1]
        return sign + s
    if exp < 0:
        return sign + "0." + "0" * (-exp - 1) + digs
    ip = (digs + "0" * (exp + 1))[:exp + 1]
    fp = digs[exp + 1:]
    return sign + ip + ("." + fp if fp else "")


HTML = {"<": "\\u003c", ">": "\\u003e", "&": "\\u0026", " ": "\\u2028", " ": "\\u2029"}


def go_json_float32(x) -> str:
    """floatEncoder with bits == 32: strconv.AppendFloat(b, float64(f), fmt, -1, 32) — the shortest digits that identify the
    FLOAT32 (numpy's Dragon4 in unique mode finds the same digits), 'e' when float32(abs) < 1e-6 or >= 1e21."""
    x = np.float32(x)
    if not np.isfinite(x):
        return ""
    if x == 0:
        return "-0" if np.signbit(x) else "0"
    sign = "-" if x < 0 else ""
    s = np.format_float_scientific(abs(x), unique=True, trim="-", exp_digits=1)   # d[.ddd]e[+-]X
    mant, _, e = s.partition("e")
    exp = int(e)
    digs = mant.replace(".", "")
    if abs(x) < np.float32(1e-6) or abs(x) >= np.float32(1e21):
        return sign + digs[0] + ("." + digs[1:] if len(digs) > 1 else "") + "e" + ("-" if exp < 0 else "+") + ("%02d" % abs(exp) if exp >= 0 else str(abs(exp)) if abs(exp) >= 10 else str(abs(exp)))
    if exp < 0:
        return sign + "0." + "0" * (-exp - 1) + digs
    ip = (digs + "0" * (exp + 1))[:exp + 1]
    fp = digs[exp + 1:]
    return sign + ip + ("." + fp if fp else "")


def go_json_time(v) -> str:
    """Time.MarshalJSON (Go 1.21) of (unix seconds, nanoseconds, zone offset seconds): quoted RFC 3339 with nanoseconds, trailing
    zeros trimmed, Z for offset 0; "" when it fails (year outside [0, 9999], zone hour >= 24).  Python's datetime does the calendar."""
    import datetime
    sec, nsec, off = v
    if nsec >= 10 ** 9:     # not a Time: answered like one that cannot be marshalled
        return ""
    local = sec + off
    zone = abs(off) // 60 if off >= 0 else (-off) // 60
    if zone // 60 >= 24:
        return ""
    if -62167219200 <= local < -62135596800:      # year 0 (datetime starts at year 1): 0000 is a leap year of 366 days
        d = datetime.datetime(4, 1, 1) + datetime.timedelta(seconds=local + 62167219200)   # year 4 has the same calendar
        ymd = "0000-%02d-%02d" % (d.month, d.day)
    elif -62135596800 <= local < 253402300800:
        d = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=local)
        ymd = "%04d-%02d-%02d" % (d.year, d.month, d.day)
    else:
        return ""
    s = ymd + "T%02d:%02d:%02d" % (d.hour, d.minute, d.second)
    if nsec:
        s += "." + ("%09d" % nsec).rstrip("0")
    # zone := offset / 60 (truncated); the sign is the sign of THAT: an offset of -30 s prints as +00:00
    s += "Z" if off == 0 else "%s%02d:%02d" % ("-" if off < 0 and zone else "+", zone // 60, zone % 60)
    return '"' + s + '"'


def go_json_string(v) -> str:
    """encoding/json string with escapeHTML, over any bytes (tests/go_net_url.py: one \\ufffd per invalid byte)"""
    return G.json_string(v.encode("utf-8") if isinstance(v, str) else bytes(v)).decode("utf-8")


# RESULT_STRING payloads: invalid UTF-8 (truncated, overlong, surrogate, beyond U+10FFFF, lone continuation), U+2028/9
STRING_PAYLOADS = [b"ok", b"\xe2\x82", b"\xe2\x82\xac", b"\xc0\xaf", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\x80\xbf", b"\xff<\xfe>",
                   b"\xe2\x80\xa8\xe2\x80\xa9", b"\x08\x0c\x00", b"\xf0\x9f\x98", b"\xef\xbf\xbd", b""]


class Unencodable(Exception):
    pass


def go_json(spec: S.TableSpec, schema: S.Schema, values) -> str:
    def scalar(kind, v):
        if kind in (S.F_INT64, S.F_INT, S.F_INT32):
            return str(int(v))
        if kind == S.F_BOOL:
            return "true" if v else "false"
        if kind == S.F_FLOAT64:
            t = go_json_float(v)
            if not t:
                raise Unencodable()
            return t
        if kind == S.F_STRING:
            return go_json_string(v)
        if kind == S.F_UINT64:
            return str(int(v))
        if kind == S.F_FLOAT32:
            t = go_json_float32(v)
            if not t:
                raise Unencodable()
            return t
        if kind == S.F_BYTES:
            import base64
            return "null" if v is None else '"' + base64.b64encode(bytes(v)).decode() + '"'
        if kind == S.F_TIME:
            t = go_json_time(v)
            if not t:
                raise Unencodable()
            return t
        raise AssertionError(kind)

    def t_value(f, v):
        return go_json(spec, spec.schema(f.elem_schema), v) if f.kind == S.F_STRUCT else scalar(f.kind, v)

    def empty(f, v):
        if f.container == S.C_PTR:
            return v is None
        if f.container in (S.C_SLICE, S.C_MAP, S.C_SLICE_PTR):
            return v is None or len(v) == 0
        if f.kind == S.F_STRUCT:
            return False
        if f.kind == S.F_STRING:
            return len(v) == 0
        if f.kind == S.F_BYTES:
            return v is None or len(v) == 0
        if f.kind == S.F_TIME:
            return False
        return v == 0   # False == 0, -0.0 == 0

    def field_value(f, v):
        if f.container == S.C_VALUE:
            return t_value(f, v)
        if v is None:
            return "null"
        if f.container == S.C_PTR:
            return t_value(f, v)
        if f.container == S.C_SLICE:
            return "[" + ",".join(t_value(f, e) for e in v) + "]"
        if f.container == S.C_SLICE_PTR:   # []*T: ptrEncoder per element
            return "[" + ",".join("null" if e is None else t_value(f, e) for e in v) + "]"
        keys = sorted(v, key=lambda k: k.encode("utf-8") if isinstance(k, str) else bytes(k))
        return "{" + ",".join(go_json_string(k) + ":" + t_value(f, v[k]) for k in keys) + "}"

    if len(schema.fields) == 1 and schema.fields[0].flags & S.FIELD_BARE:
        return field_value(schema.fields[0], values[0])
    parts = []
    for f, v in zip(schema.fields, values):
        if f.omitempty and empty(f, v):
            continue
        parts.append(go_json_string(f.name) + ":" + field_value(f, v))
    return "{" + ",".join(parts) + "}"


# ---------------------------------------------------------------------------------------------------------------
# floats
# ---------------------------------------------------------------------------------------------------------------
def _float_corpus(n, seed):
    rnd = random.Random(seed)
    vals = [0.0, -0.0, 1.0, -1.0, 0.1, 0.5, 1e21, 1e20, 9.999999999999999e20, 1e-6, 9.999999999999999e-7, 1e-7, 123456789.125,
            5e-324, 1.7976931348623157e308, 2.2250738585072014e-308, 2.225073858507201e-308, 100.0, 1e22, 1e23, 3.0e-5,
            9.5367431640625e-07, float(2 ** 53), float(2 ** 53 + 2), 0.3, 2 / 3, 1 / 3, 4.35, 0.000001, 1234567.0, 1e15, 1e16, 1e17,
            123456789012345680000.0, 5e-7, 1.5e300, -2.5e-300, 8.41e21, 4.9406564584124654e-324]
    vals += [2.0 ** k for k in range(-1074, 1024)]
    vals += [10.0 ** k for k in range(-323, 309)]
    for _ in range(n):
        vals.append(struct.unpack("<d", struct.pack("<Q", rnd.getrandbits(64)))[0])
        vals.append(rnd.uniform(-1e6, 1e6))
        vals.append(round(rnd.uniform(0, 1000), rnd.randint(0, 6)))
        vals.append(rnd.uniform(0, 1) * 10.0 ** rnd.randint(-30, 30))
        vals.append(float(rnd.randint(-10 ** 6, 10 ** 6)))
    return vals


def test_float_text_three_ways():
    """oracle (printf/strtod search), device code (Ryu) and the Python model (repr digits) write the same text"""
    vals = _float_corpus(40000, 11)
    bits = np.array([struct.unpack("<Q", struct.pack("<d", v))[0] for v in vals], dtype=np.uint64)
    out, off = E.float_text_many(bits)
    L = O.lib()
    import ctypes as C
    buf = C.create_string_buffer(64)
    for i, v in enumerate(vals):
        want = go_json_float(v).encode()
        dev = out[off[i]:off[i + 1]].tobytes()
        n = L.orc_json_float64(v, buf, 64)
        assert dev == want, (v, dev, want)
        assert buf.raw[:n] == want, (v, buf.raw[:n], want)


def test_float_text_known_answers():
    """strconv / encoding/json documented behaviour: the format switch at 1e-6 and 1e21, the e-0X clean-up, shortest digits"""
    known = {1e21: "1e+21", 1e20: "100000000000000000000", 1e-6: "0.000001", 1e-7: "1e-7", 1.5e-10: "1.5e-10", 0.1: "0.1",
             100.0: "100", -0.0: "-0", 3.14: "3.14", 1e100: "1e+100", 5e-324: "5e-324", 123456789.0: "123456789",
             1.7976931348623157e308: "1.7976931348623157e+308", 0.000001234: "0.000001234", 2.5e-7: "2.5e-7"}
    for v, want in known.items():
        assert go_json_float(v) == want
        assert E.float_text(struct.unpack("<Q", struct.pack("<d", v))[0]) == want.encode()
    for v in (math.nan, math.inf, -math.inf):
        assert E.float_text(struct.unpack("<Q", struct.pack("<d", v))[0]) == b""


def test_float32_text_three_ways_and_against_libc():
    """float32 members (floatEncoder with bits == 32): device code (Ryu with float32 parameters), oracle (printf / strtof
    search) and numpy's Dragon4 agree; a stride through ALL float32 bit patterns and every power of two against the C
    library (round trip, shortest, nearest) — scratch/float32_exhaustive.py runs the same check over all 2^31 of them."""
    known = {1.0: "1", 0.1: "0.1", 3.14: "3.14", 1e-6: "0.000001", 9.9999994e-7: "9.999999e-7", 1e21: "1e+21", 9.999999e20: "999999900000000000000",
             1e-7: "1e-7", 16777216.0: "16777216", 3.4028235e38: "3.4028235e+38", 1e-45: "1e-45", 0.3: "0.3", 100.0: "100", -0.0: "-0",
             1.5474251e26: "1.5474251e+26",   # 2^87: the nearest 8-digit decimal (1.5474250e26) lies outside the rounding interval
             123456.79: "123456.79", 1.17549435e-38: "1.1754944e-38"}
    L = O.lib()
    import ctypes as C
    buf = C.create_string_buffer(64)
    for v, want in known.items():
        bits = struct.unpack("<I", struct.pack("<f", v))[0]
        assert E.float32_text(bits) == want.encode(), (v, E.float32_text(bits))
        assert go_json_float32(v) == want, (v, go_json_float32(v))
        n = L.orc_json_float32(C.c_float(v), buf, 64)
        assert buf.raw[:n] == want.encode(), (v, buf.raw[:n])
    for b in (0x7F800000, 0xFF800000, 0x7FC00000):
        assert E.float32_text(b) == b""
    rnd = random.Random(7)
    for _ in range(20000):
        b = rnd.getrandbits(32)
        if (b >> 23) & 0xFF == 0xFF:
            continue
        x = struct.unpack("<f", struct.pack("<I", b))[0]
        dev = E.float32_text(b)
        n = L.orc_json_float32(C.c_float(x), buf, 64)
        assert dev == buf.raw[:n] == go_json_float32(x).encode(), (hex(b), dev, buf.raw[:n], go_json_float32(x))
    assert E.float32_check(1, 4099, (1 << 31) // 4099) == (0, 0)
    assert E.float32_check(1 << 23, 1 << 23, 254) == (0, 0)          # every power of two: the asymmetric intervals
    assert E.float32_check(1, 1, 1 << 16) == (0, 0)                  # subnormals


# ---------------------------------------------------------------------------------------------------------------
# schemas and values
# ---------------------------------------------------------------------------------------------------------------
ADDR = S.Schema(10, "main.Addr", [S.Field("City", S.F_STRING, "city"), S.Field("Zip", S.F_INT32, "zip", True),
                                  S.Field("Geo", S.F_FLOAT64, "geo", container=S.C_SLICE)])
POINT = S.Schema(13, "main.Point", [S.Field("X", S.F_FLOAT64, "x"), S.Field("Y", S.F_FLOAT64, "y"), S.Field("Label", S.F_STRING, "label")])
USER = S.Schema(11, "main.User", [
    S.Field("Name", S.F_STRING, "name"), S.Field("Score", S.F_FLOAT64, "score"), S.Field("Home", S.F_STRUCT, "home", elem_schema=10),
    S.Field("Work", S.F_STRUCT, "work", True, S.C_PTR, 10), S.Field("Tags", S.F_STRING, "tags", False, S.C_SLICE),
    S.Field("Attrs", S.F_STRING, "attrs", True, S.C_MAP), S.Field("Hist", S.F_STRUCT, "hist", False, S.C_SLICE, 10),
    S.Field("N", S.F_INT64, "n", True, S.C_PTR), S.Field("Counts", S.F_INT64, "counts", False, S.C_MAP),
    S.Field("At", S.F_STRUCT, "at", elem_schema=13), S.Field("Ok", S.F_BOOL, "ok")])
# no omitempty anywhere, plain nested structs only: flattened into one straight-line program at seal time
SHAPE = S.Schema(14, "main.Shape", [S.Field("ID", S.F_INT64, "id"), S.Field("Centre", S.F_STRUCT, "centre", elem_schema=13),
                                    S.Field("Area", S.F_FLOAT64, "area"), S.Field("Name", S.F_STRING, "name<>"),
                                    S.Field("Corner", S.F_STRUCT, "corner", elem_schema=13), S.Field("Closed", S.F_BOOL, "closed")])
BARE_LIST = S.Schema(12, "[]main.Addr", [S.Field("", S.F_STRUCT, "", container=S.C_SLICE, elem_schema=10, flags=S.FIELD_BARE)])
BARE_MAP = S.Schema(15, "map[string]string", [S.Field("", S.F_STRING, "", container=S.C_MAP, flags=S.FIELD_BARE)])
BARE_FLOATS = S.Schema(16, "[]float64", [S.Field("", S.F_FLOAT64, "", container=S.C_SLICE, flags=S.FIELD_BARE)])
BARE_PTR = S.Schema(17, "*main.Point", [S.Field("", S.F_STRUCT, "", container=S.C_PTR, elem_schema=13, flags=S.FIELD_BARE)])
DEEP1 = S.Schema(20, "main.D1", [S.Field("V", S.F_FLOAT64, "v", True), S.Field("S", S.F_STRING, "s", True, S.C_SLICE)])
DEEP2 = S.Schema(21, "main.D2", [S.Field("In", S.F_STRUCT, "in", container=S.C_SLICE, elem_schema=20), S.Field("P", S.F_STRUCT, "p", True, S.C_PTR, 20)])
DEEP3 = S.Schema(22, "main.D3", [S.Field("A", S.F_STRUCT, "a", elem_schema=21), S.Field("B", S.F_STRUCT, "b", container=S.C_SLICE, elem_schema=21),
                                  S.Field("M", S.F_FLOAT64, "m", True, S.C_MAP), S.Field("F", S.F_BOOL, "f", True, S.C_PTR),
                                  S.Field("I32", S.F_INT32, "i32s", False, S.C_SLICE), S.Field("BM", S.F_BOOL, "bm", False, S.C_MAP)])
# uint64 / uint, []byte (base64) and float32 members, by value and inside pointers, slices and maps
BLOB = S.Schema(23, "main.Blob", [S.Field("ID", S.F_UINT64, "id"), S.Field("Data", S.F_BYTES, "data"), S.Field("Sum", S.F_BYTES, "sum", True),
                                  S.Field("Ratio", S.F_FLOAT32, "ratio"), S.Field("W", S.F_FLOAT32, "w", True),
                                  S.Field("Big", S.F_UINT64, "big", True), S.Field("Name", S.F_STRING, "name")])
MIXED = S.Schema(24, "main.Mixed", [S.Field("Parts", S.F_BYTES, "parts", False, S.C_SLICE), S.Field("Keys", S.F_BYTES, "keys", True, S.C_MAP),
                                    S.Field("U", S.F_UINT64, "u", False, S.C_SLICE), S.Field("UM", S.F_UINT64, "um", False, S.C_MAP),
                                    S.Field("F", S.F_FLOAT32, "f", False, S.C_SLICE), S.Field("FM", S.F_FLOAT32, "fm", True, S.C_MAP),
                                    S.Field("PB", S.F_BYTES, "pb", False, S.C_PTR), S.Field("PU", S.F_UINT64, "pu", True, S.C_PTR),
                                    S.Field("PF", S.F_FLOAT32, "pf", False, S.C_PTR), S.Field("Blobs", S.F_STRUCT, "blobs", False, S.C_SLICE, 23),
                                    S.Field("Kids", S.F_STRUCT, "kids", False, S.C_SLICE_PTR, 23), S.Field("PS", S.F_STRING, "ps", True, S.C_SLICE_PTR),
                                    S.Field("PI", S.F_INT64, "pi", False, S.C_SLICE_PTR), S.Field("Tail", S.F_STRING, "tail")])
BARE_BYTES = S.Schema(25, "[]uint8", [S.Field("", S.F_BYTES, "", flags=S.FIELD_BARE)])
EVENT = S.Schema(26, "main.Event", [S.Field("ID", S.F_INT64, "id"), S.Field("CreatedAt", S.F_TIME, "created_at"), S.Field("UpdatedAt", S.F_TIME, "updated_at", True),
                                    S.Field("DeletedAt", S.F_TIME, "deleted_at", False, S.C_PTR), S.Field("Seen", S.F_TIME, "seen", True, S.C_SLICE),
                                    S.Field("Marks", S.F_TIME, "marks", False, S.C_MAP), S.Field("Note", S.F_STRING, "note")])
SCHEMAS = [ADDR, POINT, USER, SHAPE, BARE_LIST, BARE_MAP, BARE_FLOATS, BARE_PTR, DEEP1, DEEP2, DEEP3, BLOB, MIXED, BARE_BYTES, EVENT]
ROUTED = [USER, SHAPE, BARE_LIST, BARE_MAP, BARE_FLOATS, BARE_PTR, DEEP3, ADDR, BLOB, MIXED, BARE_BYTES]   # (one table: the shared-memory budget of the hot part)
# the schema set the GPU ran (and matched) in this round's last GPU test run; the kinds added afterwards have their own,
# separately reported GPU test (test_gpu_late_kinds)
ROUTED_GPU_VALIDATED = ROUTED[:8]
LATE = [BLOB, MIXED, BARE_BYTES, EVENT]


def _spec(mode=S.FRAME_WIRE, kind=S.H_ROW, routed=None):
    routed = ROUTED if routed is None else routed
    routes = [S.Route(S.M_GET, "/v/%d" % sc.id, kind, schema_id=sc.id) for sc in routed]
    schemas = [sc for sc in SCHEMAS if sc not in LATE or any(r in LATE for r in routed)]
    return S.TableSpec(frame_mode=mode, schemas=schemas, routes=routes)


WORDS = ["", "a", "Paris", "x<y>&z", "tab\there", 'q"uote', "naïve", "日本語", " sep", "long" * 23, "back\\slash", "\x01ctl", "ok"]


def _rand_value(rnd, spec, schema, nan_rate=0.0):
    def fl():
        if nan_rate and rnd.random() < nan_rate:
            return rnd.choice([math.nan, math.inf, -math.inf])
        r = rnd.random()
        if r < 0.2:
            return float(rnd.randint(-1000, 1000))
        if r < 0.4:
            return round(rnd.uniform(-500, 500), rnd.randint(0, 4))
        if r < 0.5:
            return rnd.choice([0.0, -0.0, 1e21, 1e-7, 5e-324, 1e-6])
        return rnd.uniform(-1, 1) * 10.0 ** rnd.randint(-25, 25)

    def t(f):
        if f.kind == S.F_STRUCT:
            return _rand_value(rnd, spec, spec.schema(f.elem_schema), nan_rate)
        if f.kind == S.F_STRING:
            return rnd.choice(WORDS)
        if f.kind == S.F_BOOL:
            return rnd.random() < 0.5
        if f.kind == S.F_FLOAT64:
            return fl()
        if f.kind == S.F_INT32:
            return rnd.choice([0, 1, -1, 2 ** 31 - 1, -2 ** 31, rnd.randint(-10 ** 6, 10 ** 6)])
        if f.kind == S.F_TIME:
            r = rnd.random()
            if r < 0.1:
                sec = rnd.choice([-62135596800, 0, -62167219200, -62167219201, 253402300799, 253402300800, -62135596801, 951782400, 1709164800])
            elif r < 0.2 and nan_rate:
                sec = rnd.choice([-10 ** 12, 10 ** 12, 2 ** 62, -2 ** 62])   # far outside [0, 9999]: MarshalJSON fails
            else:
                sec = rnd.randint(-62135596800, 253402300799) if r < 0.5 else rnd.randint(0, 2 * 10 ** 9)
            nsec = rnd.choice([0, 0, 1, 10, 500000000, 999999999, 123456000, rnd.randint(0, 999999999)])
            off = rnd.choice([0, 0, 3600, -3600, 19800, -34200, 30, -30, 86399, -86399, 50400, 86400 if nan_rate else 0, rnd.randint(-50000, 50000)])
            return (sec, nsec, off)
        if f.kind == S.F_UINT64:
            return rnd.choice([0, 1, 2 ** 64 - 1, 2 ** 63, 10 ** 19, rnd.randint(0, 10 ** 15), rnd.getrandbits(64)])
        if f.kind == S.F_BYTES:
            r = rnd.random()
            return None if r < 0.15 else b"" if r < 0.3 else bytes(rnd.getrandbits(8) for _ in range(rnd.choice([1, 2, 3, 4, 5, 16, 31, 100])))
        if f.kind == S.F_FLOAT32:
            if nan_rate and rnd.random() < nan_rate:
                return rnd.choice([math.nan, math.inf, -math.inf])
            r = rnd.random()
            if r < 0.3:
                return float(np.float32(round(rnd.uniform(-500, 500), rnd.randint(0, 3))))
            if r < 0.4:
                return rnd.choice([0.0, -0.0, float(np.float32(1e21)), float(np.float32(1e-6)), float(np.float32(1e-7)), 1.401298464324817e-45, 3.4028234663852886e+38, 16777216.0])
            return float(np.float32(struct.unpack("<f", struct.pack("<I", rnd.getrandbits(32) & 0x7F7FFFFF | rnd.getrandbits(1) << 31))[0]))
        return rnd.choice([0, 7, -7, 2 ** 63 - 1, -2 ** 63, rnd.randint(-10 ** 12, 10 ** 12)])

    vals = []
    for f in schema.fields:
        if f.container == S.C_VALUE:
            vals.append(t(f))
        elif f.container == S.C_PTR:
            vals.append(None if rnd.random() < 0.35 else t(f))
        elif f.container == S.C_SLICE:
            r = rnd.random()
            vals.append(None if r < 0.2 else [t(f) for _ in range(0 if r < 0.35 else rnd.randint(1, 5))])
        elif f.container == S.C_SLICE_PTR:
            r = rnd.random()
            vals.append(None if r < 0.2 else [None if rnd.random() < 0.3 else t(f) for _ in range(0 if r < 0.35 else rnd.randint(1, 5))])
        else:
            r = rnd.random()
            if r < 0.2:
                vals.append(None)
            else:
                keys = rnd.sample(["z", "a", "aa", "b<", "é", "Z", "", "a\x00", "k1", "k10", "k2", "日"], 0 if r < 0.35 else rnd.randint(1, 7))
                vals.append({k: t(f) for k in keys})
    return vals


def _batch(spec, n, seed, nan_rate=0.0, result=False, routed=None):
    routed = ROUTED if routed is None else routed
    rnd = random.Random(seed)
    reqs, want = [], []
    for i in range(n):
        sc = routed[rnd.randrange(len(routed))]
        vals = _rand_value(rnd, spec, sc, nan_rate)
        row = sc.encode_row(vals, spec.schema)
        try:
            body = go_json(spec, sc, vals)
        except Unencodable:
            body = None
        if result:
            which = rnd.randrange(4)
            if which == 0:
                data, body = S.result_record(S.RESULT_DATA, row), None if body is None else '{"data":%s}\n' % body
            elif which == 1:
                es = rnd.randrange(3)
                data, body = S.result_record(S.RESULT_RAW_DATA, row, es), None if body is None else body + "\n"
            elif which == 2:
                msg = rnd.choice(["boom", "bad <thing>", ""])
                data = S.result_both(sc, vals, msg.encode(), spec.schema)
                body = None if body is None else '{"error":{"message":%s},"data":%s}\n' % (go_json_string(msg), body)
            else:                                      # a string result of arbitrary bytes: invalid UTF-8 included
                text = rnd.choice(STRING_PAYLOADS) + bytes(rnd.getrandbits(8) for _ in range(rnd.randrange(6)))
                data, body = S.result_record(S.RESULT_STRING, text), '{"data":%s}\n' % go_json_string(text)
        else:
            data, body = row, None if body is None else '{"data":%s}\n' % body
        reqs.append(S.Req(S.M_GET, b"/v/%d" % sc.id, b"", data))
        want.append(body)
    return S.RequestBatch.pack(reqs, seed=seed), want


def _bodies(out, off):
    ob = out.tobytes()
    res = []
    for i in range(len(off) - 1):
        r = ob[int(off[i]):int(off[i + 1])]
        head, _, body = r.partition(b"\r\n\r\n")
        res.append((head, body))
    return res


@pytest.mark.parametrize("mode", [S.FRAME_WIRE, S.FRAME_INTENDED, S.FRAME_BODY])
@pytest.mark.parametrize("result", [False, True])
@pytest.mark.parametrize("late", [False, True])
def test_emu_values_match_oracle_and_model(mode, result, late):
    routed = LATE + [USER] if late else None   # late: the kinds added last (uint64, []byte, float32, time.Time) in a table of their own
    spec = _spec(mode, S.H_RESULT if result else S.H_ROW, routed)
    batch, want = _batch(spec, 700, 5 + mode, nan_rate=0.01, result=result, routed=routed)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    image = Table(spec).serialize()
    for flush in (0, 2):
        E.set_flush_mode(flush)
        try:
            o2, f2, m2 = E.serve(image, batch, DATE)
        finally:
            E.set_flush_mode(0)
        assert np.array_equal(m1, m2)
        assert np.array_equal(f1, f2)
        assert o1[:int(f1[-1])].tobytes() == o2[:int(f1[-1])].tobytes()
    # the Python model: bodies of the oracle's responses
    failed = 0
    for i, (head, body) in enumerate(_bodies(o1, f1)) if mode != S.FRAME_BODY else []:
        is_head = batch.desc["method"][i] == S.M_HEAD
        if want[i] is None:      # NaN / Inf: Encode failed — status and headers stand, the body is empty
            failed += 1
            assert body == b"" and b"Content-Length: 0" in head, (i, head, body)
            assert (b"Content-Type: application/json" in head) == (mode == S.FRAME_INTENDED)
        elif not is_head:
            assert body.decode("utf-8") == want[i], (i, body, want[i])
            assert b"Content-Length: %d\r\n" % len(body) in head + b"\r\n"
    if mode == S.FRAME_BODY:
        ob = o1.tobytes()
        for i in range(batch.n):
            got = ob[int(f1[i]):int(f1[i + 1])]
            if batch.desc["method"][i] != S.M_HEAD:
                assert got.decode("utf-8") == (want[i] or ""), i
    else:
        assert failed > 0


@pytest.mark.parametrize("slot", [512, 4096])
def test_emu_values_in_slots(slot):
    spec = _spec()
    batch, _ = _batch(spec, 500, 77, nan_rate=0.01)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    out, ln, meta = E.serve_slots(Table(spec).serialize(), batch, DATE, slot)
    assert np.array_equal(meta, m1)
    want_len = np.diff(f1.astype(np.int64)).astype(np.uint32)
    assert np.array_equal(ln, want_len)
    ob = o1.tobytes()
    for i in range(batch.n):
        L = int(ln[i])
        if L <= slot:
            assert out[i, :L].tobytes() == ob[int(f1[i]):int(f1[i]) + L], i
    assert (ln > slot).any() == (slot == 512)


def test_reference_pin_map_response():
    """pkg/gofr/http/responder_test.go:23 "map response type": Respond(map[string]string{}, nil) → Content-Type
    application/json; the body encoding/json writes for an empty map inside the envelope is {"data":{}}"""
    spec = S.TableSpec(frame_mode=S.FRAME_INTENDED, schemas=[BARE_MAP], routes=[S.Route(S.M_GET, "/m", S.H_ROW, schema_id=15)])
    rows = [{}, None, {"b": "2", "a": "1"}]
    batch = S.RequestBatch.pack([S.Req(S.M_GET, b"/m", b"", BARE_MAP.encode_row([r])) for r in rows], seed=1)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    o2, f2, m2 = E.serve(Table(spec).serialize(), batch, DATE)
    assert np.array_equal(f1, f2) and o1[:int(f1[-1])].tobytes() == o2[:int(f1[-1])].tobytes()
    got = _bodies(o1, f1)
    assert [b for _, b in got] == [b'{"data":{}}\n', b'{"data":null}\n', b'{"data":{"a":"1","b":"2"}}\n']
    assert all(b"Content-Type: application/json\r\n" in h + b"\r\n" for h, _ in got)


def test_malformed_rows_answer_like_a_panic():
    """rows that end before the walk does (a truncated slice, a map entry running off the data section) are not a
    reference behaviour: both sides answer 500 like middleware.panicRecovery, as for flat rows"""
    spec = _spec()
    rnd = random.Random(3)
    reqs = []
    for i in range(300):
        sc = ROUTED[i % len(ROUTED)]
        row = sc.encode_row(_rand_value(rnd, spec, sc), spec.schema)
        cut = rnd.randrange(0, len(row) + 1)
        reqs.append(S.Req(S.M_GET, b"/v/%d" % sc.id, b"", row[:cut]))
    # counts that promise more than the row holds
    reqs.append(S.Req(S.M_GET, b"/v/16", b"", (1 << 30).to_bytes(4, "little") + b"\0" * 64))
    reqs.append(S.Req(S.M_GET, b"/v/15", b"", (0xFFFFFFFE).to_bytes(4, "little") + b"\0" * 64))
    reqs.append(S.Req(S.M_GET, b"/v/12", b"", (5).to_bytes(4, "little") + b"\0" * 10))
    batch = S.RequestBatch.pack(reqs, seed=9)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    o2, f2, m2 = E.serve(Table(spec).serialize(), batch, DATE)
    assert np.array_equal(m1, m2) and np.array_equal(f1, f2) and o1[:int(f1[-1])].tobytes() == o2[:int(f1[-1])].tobytes()
    assert ((m1 & 0xFFFF) == 500).sum() > 50 and ((m1 & 0xFFFF) == 200).sum() > 5


def test_flat_schemas_agree_between_the_two_oracle_encoders():
    """the row walker (orc_value.c) and the pinned flat-struct encoder (orc_enc_struct) are two code paths of the oracle"""
    from gofr_b200 import synth
    spec = synth.config2_spec()
    t = O.OracleTable(spec)
    batch = synth.config2_batch(300, escape_every=5)
    o1, f1, _ = t.serve(batch, DATE)
    for i, (_, body) in enumerate(_bodies(o1, f1)):
        off, dl = int(batch.desc["arena_off"][i]), int(batch.desc["data_len"][i])
        pl, ql = int(batch.desc["path_len"][i]), int(batch.desc["query_len"][i])
        start = (off + pl + ql + 3) & ~3
        row = batch.arena[start:start + dl].tobytes()
        assert body == b'{"data":' + t.encode_row_json(1, row) + b"}\n"


def test_schema_validation():
    def seal(schemas, routes=()):
        return Table(S.TableSpec(schemas=schemas, routes=list(routes)))
    with pytest.raises(Exception):   # struct type not added yet (also what a recursive type would need)
        seal([S.Schema(1, "T", [S.Field("A", S.F_STRUCT, "a", elem_schema=2)])])
    with pytest.raises(Exception):   # maps of structs
        seal([POINT, S.Schema(1, "T", [S.Field("A", S.F_STRUCT, "a", container=S.C_MAP, elem_schema=13)])])
    with pytest.raises(Exception):   # a bare field must be alone
        seal([S.Schema(1, "T", [S.Field("A", S.F_INT64, "a", flags=S.FIELD_BARE), S.Field("B", S.F_INT64, "b")])])
    with pytest.raises(Exception):   # Bind takes flat structs only (nested structs, pointers, slices, maps: not yet)
        seal([POINT, SHAPE], [S.Route(S.M_POST, "/p", S.H_BIND_ECHO, schema_id=14)])
    seal([POINT], [S.Route(S.M_POST, "/p", S.H_BIND_ECHO, schema_id=13)])   # float64 members are taken (tests/test_bind.py)
    chain = [S.Schema(100, "L0", [S.Field("V", S.F_INT64, "v")])]
    for k in range(1, 9):
        chain.append(S.Schema(100 + k, "L%d" % k, [S.Field("C", S.F_STRUCT, "c", container=S.C_PTR, elem_schema=99 + k)]))
    seal(chain[:8])                  # 8 levels: the walker's frame stack
    with pytest.raises(Exception):
        seal(chain)


def test_time_known_answers():
    """Time.MarshalJSON as documented (time.RFC3339Nano with strict checks): known texts, three ways"""
    bare = S.Schema(30, "time.Time", [S.Field("", S.F_TIME, "", flags=S.FIELD_BARE)])
    spec = S.TableSpec(frame_mode=S.FRAME_BODY, schemas=[bare], routes=[S.Route(S.M_GET, "/t", S.H_ROW, schema_id=30)])
    known = [((-62135596800, 0, 0), '"0001-01-01T00:00:00Z"'),                       # the zero Time
             ((0, 0, 0), '"1970-01-01T00:00:00Z"'),
             ((1709210096, 123456789, 19800), '"2024-02-29T18:04:56.123456789+05:30"'),
             ((1709210096, 500000000, -28800), '"2024-02-29T04:34:56.5-08:00"'),
             ((1709210096, 120000, 0), '"2024-02-29T12:34:56.00012Z"'),
             ((951782400, 0, 0), '"2000-02-29T00:00:00Z"'),
             ((4107542400, 1, 3600), '"2100-03-01T01:00:00.000000001+01:00"'),       # 2100 is not a leap year
             ((253402300799, 999999999, 0), '"9999-12-31T23:59:59.999999999Z"'),
             ((-62167219200, 0, 0), '"0000-01-01T00:00:00Z"'),
             ((0, 0, -30), '"1969-12-31T23:59:30+00:00"'),                            # zone minutes truncate to 0: "+00:00", not "Z"
             ((0, 0, 86340), '"1970-01-01T23:59:00+23:59"'),
             ((253402300800, 0, 0), None), ((-62167219201, 0, 0), None),              # years 10000 and -1: MarshalJSON fails
             ((0, 0, 86400), None), ((0, 0, -90000), None),                           # zone hour outside [0, 23]
             ((253402300799, 0, 1), None),                                            # the wall clock is what counts
             ((0, 10 ** 9, 0), None), ((0, 2 ** 32 - 1, 0), None),                    # nanoseconds no Time holds
             ((2 ** 63 - 1, 0, 86399), None), ((-2 ** 63, 0, -86399), None), ((2 ** 63 - 1, 999999999, 0), None)]   # no overflow on the way
    reqs = [S.Req(S.M_GET, b"/t", b"", bare.encode_row([v])) for v, _ in known]
    batch = S.RequestBatch.pack(reqs)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    o2, f2, m2 = E.serve(Table(spec).serialize(), batch, DATE)
    r1, r2 = O.responses(o1, f1), O.responses(o2, f2)
    for (v, want), a, b in zip(known, r1, r2):
        w = b"" if want is None else ('{"data":%s}\n' % want).encode()
        assert a == b == w, (v, a, b, w)
        assert go_json_time(v) == (want or ""), v


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("result", [False, True])
def test_gpu_values_match_oracle(result, routed=None):
    import torch
    from gofr_b200.engine import Engine
    assert torch.cuda.is_available()
    routed = ROUTED_GPU_VALIDATED if routed is None else routed
    spec = _spec(S.FRAME_WIRE, S.H_RESULT if result else S.H_ROW, routed)
    batch, _ = _batch(spec, 6000, 21, nan_rate=0.01, result=result, routed=routed)
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE)
    eng = Engine(Table(spec), 0)
    resp = eng.alloc_responses(batch.n, int(f1[-1]) + 4096)
    eng.serve_device(eng.upload(batch), DATE, resp)
    torch.cuda.synchronize()
    out, off, meta = resp.to_host()
    assert np.array_equal(meta, m1)
    assert np.array_equal(off, f1)
    assert out[:int(f1[-1])].tobytes() == o1[:int(f1[-1])].tobytes()
    slot = 2048
    canary = torch.full((batch.n * slot,), 0xEE, dtype=torch.uint8, device="cuda")
    so, sl, sm = eng.serve_device_slots(eng.upload(batch), DATE, slot, out=canary)
    so = so.cpu().numpy().reshape(batch.n, slot)
    ln = sl.cpu().numpy().view(np.uint32)
    assert np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32))
    ob = o1.tobytes()
    for i in range(batch.n):
        L = int(ln[i])
        if L <= slot:
            assert so[i, :L].tobytes() == ob[int(f1[i]):int(f1[i]) + L], i
            assert (so[i, L + (-L) % 16:] == 0xEE).all(), i
    eng.close()


def _gpu_late_kinds_check():
    test_gpu_values_match_oracle(False, LATE + [USER])
    test_gpu_values_match_oracle(True, LATE + [USER])


@pytest.mark.gpu
def test_gpu_late_kinds():
    """6 000 rows of the kinds added late (uint64, []byte as base64, float32; by value, behind pointers, in slices and maps),
    packed and slot layouts, GOFR_H_ROW and GOFR_H_RESULT — in a child process (a fault cannot reach the other GPU tests)"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import tests.test_values as t; t._gpu_late_kinds_check()"], cwd=root,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.gpu
def test_gpu_float_text_matches_python_repr():
    """the Ryu digits as the GPU computes them (__umul64hi, device tables): a bare []float64 route carries the corpus"""
    import torch
    from gofr_b200.engine import Engine
    spec = S.TableSpec(frame_mode=S.FRAME_BODY, schemas=[BARE_FLOATS], routes=[S.Route(S.M_GET, "/f", S.H_ROW, schema_id=16)])
    vals = [v for v in _float_corpus(20000, 23)]
    per = 50
    reqs, want = [], []
    for k in range(0, len(vals), per):
        chunk = vals[k:k + per]
        reqs.append(S.Req(S.M_GET, b"/f", b"", BARE_FLOATS.encode_row([chunk])))
        texts = [go_json_float(v) for v in chunk]
        # a NaN / Inf among the random bit patterns makes Encode fail for the whole value: no body at all
        want.append(('{"data":[' + ",".join(texts) + "]}\n").encode() if all(texts) else b"")
    batch = S.RequestBatch.pack(reqs, seed=4)
    eng = Engine(Table(spec), 0)
    resp = eng.alloc_responses(batch.n, sum(len(w) for w in want) + 4096)
    eng.serve_device(eng.upload(batch), DATE, resp)
    torch.cuda.synchronize()
    out, f, meta = resp.to_host()
    ob = out.tobytes()
    for i, w in enumerate(want):
        assert ob[int(f[i]):int(f[i + 1])] == w, i
    eng.close()


def test_response_bound_holds_for_the_wider_data_model():
    """gofr_table_response_bound sizes the host path's output buffers.  Six response bytes per data byte is the worst case of
    flat rows (a control character becomes \\u00XX); an element of a slice of structs drags its key literals along, so tables
    with such programs carry their own factor (engine_internal.h image_data_expand)."""
    from gofr_b200 import _abi
    L = _abi.lib()
    inner = S.Schema(1, "main.I", [S.Field("F", S.F_BOOL, "a_rather_long_key_name_for_one_bit_of_information")])
    mid = S.Schema(2, "main.M", [S.Field("In", S.F_STRUCT, "another_quite_long_key_name", elem_schema=1)])
    outer = S.Schema(3, "[]main.M", [S.Field("", S.F_STRUCT, "", container=S.C_SLICE, elem_schema=2, flags=S.FIELD_BARE)])
    spec = S.TableSpec(schemas=[inner, mid, outer], routes=[S.Route(S.M_GET, "/p", S.H_ROW, schema_id=3)])
    t = Table(spec)
    row = outer.encode_row([[[[True]]] * 200], spec.schema)
    b = S.RequestBatch.pack([S.Req(S.M_GET, b"/p", b"", row)])
    o, f, m = O.OracleTable(spec).serve(b, DATE, out_cap=1 << 20)
    o2, f2, m2 = E.serve(t.serialize(), b, DATE, out_cap=1 << 20)
    assert np.array_equal(f, f2) and o[:int(f[1])].tobytes() == o2[:int(f[1])].tobytes()
    assert int(f[1]) > 6 * len(row)                                   # the old bound would have been too small
    assert L.gofr_table_response_bound(t.handle, 2, 0, len(row)) >= int(f[1])
    spec = _spec()
    t = Table(spec)
    batch, _ = _batch(spec, 2000, 5)
    o, f, m = O.OracleTable(spec).serve(batch, DATE)
    ln = np.diff(f.astype(np.int64))
    for i in range(batch.n):
        d = batch.desc[i]
        assert L.gofr_table_response_bound(t.handle, int(d["path_len"]), int(d["query_len"]), int(d["data_len"])) >= ln[i], i
    # tables without such programs keep the six-fold bound
    from gofr_b200 import synth
    t2 = Table(synth.config2_spec())
    assert L.gofr_table_response_bound(t2.handle, 0, 0, 1000) - L.gofr_table_response_bound(t2.handle, 0, 0, 0) == 6000


# ---------------------------------------------------------------------------------------------------------------
# random SCHEMAS (not only random values): struct trees with every kind, container and omitempty combination
# ---------------------------------------------------------------------------------------------------------------
def _rand_schemas(rnd, n_types, late=False):
    """n_types struct types, each free to use the ones before it, plus bare types on top of them (late: uint64, []byte and
    float32 members as well)"""
    extra = [S.F_UINT64, S.F_BYTES, S.F_FLOAT32, S.F_TIME] * 2 if late else []
    schemas = []
    names = ["a", "id", "Name", "x<y", "long_key_name_%d", "k", "é", "v1", "data", "0"]
    for t in range(n_types):
        fields = []
        for k in range(rnd.randint(1, 5)):
            kind = rnd.choice([S.F_INT64, S.F_INT32, S.F_BOOL, S.F_STRING, S.F_INT, S.F_FLOAT64] + extra + ([S.F_STRUCT] * 2 if schemas else []))
            cont = rnd.choice([S.C_VALUE, S.C_VALUE, S.C_PTR, S.C_SLICE, S.C_MAP] + ([S.C_SLICE_PTR] if late else []))
            elem = 0
            if kind == S.F_STRUCT:
                elem = rnd.choice(schemas).id
                if cont == S.C_MAP:
                    cont = S.C_SLICE
            jn = rnd.choice(names)
            jn = (jn % k if "%" in jn else jn) + str(k)
            fields.append(S.Field("F%d" % k, kind, jn, rnd.random() < 0.4, cont, elem))
        schemas.append(S.Schema(100 + t, "main.T%d" % t, fields))
    bare = []
    for t in range(3):
        kind = rnd.choice([S.F_INT64, S.F_BOOL, S.F_STRING, S.F_FLOAT64, S.F_STRUCT] + extra)
        cont = rnd.choice([S.C_PTR, S.C_SLICE, S.C_MAP]) if kind not in (S.F_FLOAT64, S.F_BYTES, S.F_FLOAT32, S.F_TIME) else rnd.choice([S.C_VALUE, S.C_SLICE])
        elem = rnd.choice(schemas).id if kind == S.F_STRUCT else 0
        if kind == S.F_STRUCT and cont == S.C_MAP:
            cont = S.C_SLICE
        bare.append(S.Schema(200 + t, "bare%d" % t, [S.Field("", kind, "", container=cont, elem_schema=elem, flags=S.FIELD_BARE)]))
    return schemas, bare


def _random_schema_case(seed, n=400):
    """A table of random schemas and n requests of random values for them: (spec, routed schemas, batch, want) where
    want[i] is the body the Python model writes (None: encoding/json cannot encode the value)."""
    rnd = random.Random(1000 + seed)
    structs, bare = _rand_schemas(rnd, rnd.randint(2, 5), late=seed >= 12)
    routed = structs + bare
    mode = [S.FRAME_WIRE, S.FRAME_BODY, S.FRAME_INTENDED][seed % 3]
    spec = S.TableSpec(frame_mode=mode, schemas=structs + bare,
                       routes=[S.Route(S.M_GET, "/t/%d" % sc.id, S.H_RESULT if seed % 2 else S.H_ROW, schema_id=sc.id) for sc in routed])
    reqs, want = [], []
    for i in range(n):
        sc = routed[rnd.randrange(len(routed))]
        vals = _rand_value(rnd, spec, sc, nan_rate=0.005)
        row = sc.encode_row(vals, spec.schema)
        try:
            body = go_json(spec, sc, vals)
        except Unencodable:
            body = None
        if seed % 2:
            raw = rnd.random() < 0.5
            data = S.result_record(S.RESULT_RAW_DATA if raw else S.RESULT_DATA, row)
            body = None if body is None else (body + "\n" if raw else '{"data":%s}\n' % body)
        else:
            data = row
            body = None if body is None else '{"data":%s}\n' % body
        reqs.append(S.Req(S.M_GET, b"/t/%d" % sc.id, b"", data))
        want.append(body)
    return spec, routed, S.RequestBatch.pack(reqs, seed=seed), want


@pytest.mark.parametrize("seed", range(24))
def test_random_schemas_three_ways(seed):
    spec, routed, batch, want = _random_schema_case(seed)
    mode = spec.frame_mode
    try:
        table = Table(spec)
    except Exception as e:      # deeper than 8 levels cannot happen with <= 5 types; anything else is a bug
        raise AssertionError((e, routed))
    o1, f1, m1 = O.OracleTable(spec).serve(batch, DATE, out_cap=1 << 22)
    image = table.serialize()
    E.set_flush_mode(seed % 3)
    try:
        o2, f2, m2 = E.serve(image, batch, DATE, out_cap=1 << 22)
    finally:
        E.set_flush_mode(0)
    assert np.array_equal(m1, m2) and np.array_equal(f1, f2)
    assert o1[:int(f1[-1])].tobytes() == o2[:int(f1[-1])].tobytes()
    ob = o1.tobytes()
    for i in range(batch.n):
        r = ob[int(f1[i]):int(f1[i + 1])]
        body = r if mode == S.FRAME_BODY else r.partition(b"\r\n\r\n")[2]
        assert body.decode("utf-8") == (want[i] or ""), (i, routed, want[i])
    # the same batch through the slot layout of the device code
    out, ln, meta = E.serve_slots(image, batch, DATE, 8192)
    assert np.array_equal(ln, np.diff(f1.astype(np.int64)).astype(np.uint32))
    for i in range(0, batch.n, 3):
        L = int(ln[i])
        if L <= 8192:
            assert out[i, :L].tobytes() == ob[int(f1[i]):int(f1[i]) + L], i


def _mutated_rows(rnd, spec, routed, kind, n):
    """n requests for the /t/<id> routes of `routed` whose rows (or result records) have bytes flipped, count words
    overwritten, tails cut off or garbage appended"""
    reqs = []
    for i in range(n):
        sc = routed[rnd.randrange(len(routed))]
        row = sc.encode_row(_rand_value(rnd, spec, sc), spec.schema)
        data = bytearray(S.result_record(rnd.choice([S.RESULT_DATA, S.RESULT_RAW_DATA]), row) if kind == S.H_RESULT else row)
        for _k in range(rnd.randint(0, 3)):
            if not data:
                break
            r, p = rnd.random(), rnd.randrange(len(data))
            if r < 0.4:
                data[p] ^= 1 << rnd.randrange(8)
            elif r < 0.6:
                data[p & ~3:(p & ~3) + 4] = rnd.choice([0xFFFFFFFF, 0xFFFFFFFE, 0x7FFFFFFF, 1 << 20, 3]).to_bytes(4, "little")
            elif r < 0.8:
                del data[p:]
            else:
                data += bytes(rnd.randrange(256) for _ in range(rnd.randint(1, 9)))
        reqs.append(S.Req(S.M_GET, b"/t/%d" % sc.id, b"", bytes(data)))
    return reqs


@pytest.mark.parametrize("seed", list(range(6)) + list(range(10, 18)))
def test_mutated_rows_device_code_equals_oracle(seed):
    """rows of random schemas with bytes flipped, count words overwritten, tails cut off or garbage appended: whatever the
    walk meets first — a float encoding/json cannot write, or the end of the row — decides, on both sides alike"""
    rnd = random.Random(4000 + seed)
    for _ in range(3):
        structs, bare = _rand_schemas(rnd, rnd.randint(2, 5), late=seed >= 10)   # late: uint64, []byte, float32, time.Time, []*T too
        routed = structs + bare
        kind = S.H_RESULT if seed % 2 else S.H_ROW
        spec = S.TableSpec(schemas=routed, routes=[S.Route(S.M_GET, "/t/%d" % sc.id, kind, schema_id=sc.id) for sc in routed])
        b = S.RequestBatch.pack(_mutated_rows(rnd, spec, routed, kind, 250), seed=seed)
        o1, f1, m1 = O.OracleTable(spec).serve(b, DATE, out_cap=1 << 24)
        o2, f2, m2 = E.serve(Table(spec).serialize(), b, DATE, out_cap=1 << 24)
        assert np.array_equal(m1, m2) and np.array_equal(f1, f2)
        assert o1[:int(f1[-1])].tobytes() == o2[:int(f1[-1])].tobytes()
        st = m1 & 0xFFFF
        assert (st == 500).any() and (st == 200).any()
