"""Context.Bind into float64 members (bind_device.cuh bd_parse_float / bd_eisel_lemire) against exact rounding.

strconv.ParseFloat rounds correctly, so every literal the device decides must carry exactly the double Python's float()
gives; the device may instead leave a literal to the host (status 2), but only where the stated may-defer rules below
allow it.  The corpus is a seeded generator of JSON number literals in families (exact-case edges, every Eisel-Lemire
table row, half-way points, range ends, encoder output, spellings).  A Python restatement of the parser's branch
selection (exact integers, no device code) says which path each literal takes and which table row it reads; it is used
for coverage, not for values.  CPU: the device code through tests/emu.  GPU (-m gpu): gofr_bind_device on an H100, per
literal against the emulation and against float() separately."""
import math
import os
import re
import struct
from fractions import Fraction

import numpy as np
import pytest

from gofr_b200 import spec as S
from gofr_b200.table import Table
from tests.emu import emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1

# A schema with several float64 members: `a` sits at an odd word of the span row (an int32 before it), `c` is omitempty.
# Bind row (bind_row_out): i int32 @0, a float64 @4, f bool @12, c float64 @16, s string length @24, d float64 @28.
FB_SCHEMA = S.Schema(21, "pkg.Reading", [S.Field("I", S.F_INT32, "i"), S.Field("A", S.F_FLOAT64, "a"), S.Field("F", S.F_BOOL, "f"),
                                         S.Field("C", S.F_FLOAT64, "c", True), S.Field("S", S.F_STRING, "s"),
                                         S.Field("D", S.F_FLOAT64, "d")])
FB_SPEC = S.TableSpec(frame_mode=S.FRAME_BODY, schemas=[FB_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=21)])
FIELDS = (("a", 4), ("c", 16), ("d", 28))
SLOT = 1024

# ---- the Eisel-Lemire power table, restated with exact integers (the rule scratch/gen/el_tables.py generates it by) ----
EL_MIN, EL_MAX = -348, 347


def el_row(q):
    if q >= 0:
        c = 5 ** q
        c = c << max(0, 128 - c.bit_length()) if c.bit_length() < 128 else c >> (c.bit_length() - 128)
        return c
    p = 5 ** -q
    z = (p - 1).bit_length()
    c = (1 << (z + 127)) // p + 1 if q >= -27 else (1 << (2 * z + 128)) // p + 1
    return c >> max(0, c.bit_length() - 128)


EL = [el_row(q) for q in range(EL_MIN, EL_MAX + 1)]


def eisel_lemire(man, exp10):
    """strconv eiselLemire64 on exact integers: (ok, bits without sign, wider product taken)"""
    if man == 0:
        return True, 0, False
    if exp10 < EL_MIN or exp10 > EL_MAX:
        return False, 0, False
    clz = 64 - man.bit_length()
    man <<= clz
    ret_exp2 = (((217706 * exp10) >> 16) + 64 + 1023 - clz) & M64
    pw = EL[exp10 - EL_MIN]
    x = man * (pw >> 64)
    x_hi, x_lo = x >> 64, x & M64
    wide = (x_hi & 0x1FF) == 0x1FF and ((x_lo + man) & M64) < man
    if wide:
        y = man * (pw & M64)
        y_hi, y_lo = y >> 64, y & M64
        m_lo = (x_lo + y_hi) & M64
        m_hi = x_hi + (1 if m_lo < x_lo else 0)
        if (m_hi & 0x1FF) == 0x1FF and m_lo == M64 and ((y_lo + man) & M64) < man:
            return False, 0, True
        x_hi, x_lo = m_hi & M64, m_lo
    msb = x_hi >> 63
    ret_man = x_hi >> (msb + 9)
    ret_exp2 = (ret_exp2 - (1 ^ msb)) & M64
    if x_lo == 0 and (x_hi & 0x1FF) == 0 and (ret_man & 3) == 1:
        return False, 0, wide
    ret_man += ret_man & 1
    ret_man >>= 1
    if ret_man >> 53:
        ret_man >>= 1
        ret_exp2 += 1
    if ((ret_exp2 - 1) & M64) >= 0x7FF - 1:
        return False, 0, wide
    return True, ret_exp2 << 52 | (ret_man & ((1 << 52) - 1)), wide


def parse(lit: bytes):
    """bd_parse_float's scan: (mant, nd, exp10, trunc) with value = mant [+ dropped digits] x 10^exp10"""
    n, i = len(lit), 0
    if lit[:1] == b"-":
        i = 1
    mant = nd = exp10 = 0
    nonzero = trunc = False
    while i < n and 48 <= lit[i] <= 57:
        d = lit[i] - 48
        i += 1
        if not nonzero and d == 0:
            continue
        nonzero = True
        if nd < 19:
            mant, nd = mant * 10 + d, nd + 1
        else:
            trunc |= d != 0
            exp10 += 1
    if i < n and lit[i] == 46:
        i += 1
        while i < n and 48 <= lit[i] <= 57:
            d = lit[i] - 48
            i += 1
            if not nonzero and d == 0:
                exp10 -= 1
                continue
            nonzero = True
            if nd < 19:
                mant, nd, exp10 = mant * 10 + d, nd + 1, exp10 - 1
            else:
                trunc |= d != 0
    if i < n and lit[i] in b"eE":
        i += 1
        neg = False
        if i < n and lit[i] in b"+-":
            neg = lit[i] == 45
            i += 1
        e = 0
        while i < n and 48 <= lit[i] <= 57:
            if e < 1000000:
                e = e * 10 + lit[i] - 48
            i += 1
        exp10 += -e if neg else e
    if mant:
        while not trunc and mant % 10 == 0:
            mant, exp10, nd = mant // 10, exp10 + 1, nd - 1
    return mant, nd, exp10, trunc


def branch(lit: bytes):
    """Which path bd_parse_float takes: (path, table rows read, wider-product hits).  Paths: zero, underflow, overflow,
    exact, el128, el192, trunc."""
    mant, nd, exp10, trunc = parse(lit)
    if mant == 0:
        return "zero", (), 0
    lead = exp10 + nd - 1
    if lead >= 310:
        return "overflow", (), 0
    if lead <= -330:
        return "underflow", (), 0
    exact = not trunc and mant >> 53 == 0 and -22 <= exp10 <= 22 + 15 and \
        (exp10 <= 22 or mant <= ((1 << 53) - 1) // 10 ** (exp10 - 22))
    if exact:
        return "exact", (), 0
    rows = (exp10,) if EL_MIN <= exp10 <= EL_MAX else ()
    ok, _, wide = eisel_lemire(mant, exp10)
    hits = int(wide)
    if trunc and ok:
        hits += int(eisel_lemire(mant + 1, exp10)[2])
    return ("trunc" if trunc else "el192" if hits else "el128"), rows, hits


# ---- the reference: float() for the value, Fraction for which literals the device may leave to the host ----
# The rules read the literal's decimal digits themselves (sig_digits), not the parser's scan.  A literal with at most 19
# significant digits may be deferred only when it IS a half-way point between two doubles: the 128-bit product with the
# 192-bit correction settles every other one in the corpus.  HALF_ULP_BOUND is that tightest bound, distance 0 (the
# corpus runs below assert that it is enough); literals with more digits are judged by the two ends of their 19-digit cut.
HALF_ULP_BOUND = Fraction(0)
DBL_MIN = 2.2250738585072014e-308


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _round(x: Fraction) -> float:
    """correctly rounded, inf past DBL_MAX"""
    try:
        return float(x)
    except OverflowError:
        return math.inf


def sig_digits(lit: bytes):
    """(significant digits without leading / trailing zeros, lead) with |value| = 0.DIGITS x 10^(lead + 1); ("", 0) for 0"""
    t = lit.decode().lstrip("-").lower()
    m, _, e = t.partition("e")
    ip, _, fp = m.partition(".")
    digits = ip + fp
    point = len(ip) + (int(e) if e else 0)     # the decimal point sits after this many digits
    stripped = digits.lstrip("0")
    point -= len(digits) - len(stripped)
    stripped = stripped.rstrip("0")
    return stripped, point - 1


def defer_reason(lit: bytes):
    """None when the device must decide the literal, else why it may leave it to the host"""
    d, lead = sig_digits(lit)
    if not d or lead >= 310 or lead <= -330:   # 0, sure ErrRange, sure underflow to 0: always decided
        return None
    if lead >= 309:
        return "top"
    f = float(lit)
    if math.isinf(f):   # rounds past DBL_MAX: ErrRange, from the lead digit at 308 on
        return "top"
    if abs(f) < DBL_MIN:
        return "subnormal"
    if len(d) > 19:
        # the device rounds both ends of the 19-digit cut: they must agree, and each must not be a half-way point
        scale = Fraction(10) ** (lead - 18)
        ends = (int(d[:19]) * scale, (int(d[:19]) + 1) * scale)
        if _round(ends[0]) != _round(ends[1]) or _near_half(ends[0]) or _near_half(ends[1]):
            return "cut"
        return None
    return "half" if _near_half(int(d) * Fraction(10) ** (lead + 1 - len(d))) else None


def _near_half(v: Fraction) -> bool:
    """v (> 0, normal range) lies within HALF_ULP_BOUND ulp of a half-way point between two doubles"""
    f = _round(v)
    if math.isinf(f):
        return True
    a = Fraction(f)
    # the two doubles around the exact value (above DBL_MAX: where the next one would be, 2^1024)
    lo, hi = (Fraction(math.nextafter(f, 0.0)), a) if v < a else (a, a + Fraction(math.ulp(f)))
    return abs(v - (lo + hi) / 2) <= (hi - lo) * HALF_ULP_BOUND


def overflow_text(lit: bytes, field: str) -> bytes:
    return b"json: cannot unmarshal number " + lit + b" into Go struct field Reading." + field.encode() + b" of type float64"


def check(lits, status, got, fields):
    """Per literal: status (0 decided, 1 error, 2 deferred) and what the row says (bits for 0, error text for 1).
    Returns the problems: (kind, index)."""
    bad = []
    for k, lit in enumerate(lits):
        st = int(status[k])
        want = float(lit)
        if st == 2:
            if defer_reason(lit) is None:
                bad.append(("deferred", k))
        elif math.isinf(want):
            if st != 1 or got[k] != overflow_text(lit, fields[k]):
                bad.append(("overflow", k))
        elif st != 0 or got[k] != f64_bits(want):
            bad.append(("value", k))
    return bad


# ---- the corpus ----
def _exact_edges(rng):
    mans = [1, 2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 10 ** 15 - 1, 10 ** 19 - 1] + [int(x) for x in rng.integers(1, 2 ** 53, 40)]
    return [b"%de%d" % (m, e) for m in mans for e in range(-25, 41)]


def _rows(rng, per_row):
    out = []
    for q in range(EL_MIN, EL_MAX + 1):
        for k in range(per_row):
            nd = 1 + k % 19
            m = int(rng.integers(10 ** (nd - 1), 10 ** nd, dtype=np.uint64)) if nd < 20 else 0
            if k % 5 == 4:
                m = int(rng.integers(2 ** 53, 10 ** 19, dtype=np.uint64))   # >= 2^53: the approximation even inside +-22
            m = m * 10 + int(rng.integers(1, 10)) if m % 10 == 0 else m
            m = m // 10 if m >= 10 ** 19 else m
            # place the literal so that the parser's normalised exponent is q: value = m x 10^q
            out.append(b"%de%d" % (m, q) if k % 2 else b"%s.%se%d" % (str(m)[:1].encode(), str(m)[1:].encode() or b"0",
                                                                       q + len(str(m)) - 1))
    return out


def _halfway(rng, count):
    out = []
    for _ in range(count):
        b = int(rng.integers(0x0010000000000000, 0x7FE0000000000000, dtype=np.uint64))
        lo = struct.unpack("<d", struct.pack("<Q", b))[0]
        hi = math.nextafter(lo, math.inf)
        mid = (Fraction(lo) + Fraction(hi)) / 2
        # mid = n / 2^k exactly: its decimal expansion terminates
        den = mid.denominator
        k = den.bit_length() - 1
        digits = mid.numerator * 5 ** k if k else mid.numerator
        s = str(digits)
        e = len(s) - 1 - k
        one = lambda t, ee: b"%s.%se%d" % (t[:1].encode(), (t[1:] or "0").encode(), ee)
        out.append(one(s, e))
        last = int(s[-1])
        out.append(one(str(digits + 1), e if len(str(digits + 1)) == len(s) else e + 1))
        if last or digits > 1:
            out.append(one(str(digits - 1), e if len(str(digits - 1)) == len(s) else e - 1))
        for t in (17, 19, 20, 25):
            if len(s) > t:
                out.append(one(s[:t], e))
    return out


def _range_ends():
    lits = [b"1.7976931348623157e308", b"1.7976931348623158e308", b"1.7976931348623159e308", b"1.797693134862315708145274237317043567981e308",
            b"1.797693134862315807937289714053034150799e308", b"-1.7976931348623157e308", b"8.98846567431158e307",
            b"2.2250738585072014e-308", b"2.2250738585072011e-308", b"2.225073858507201e-308", b"4.9e-324", b"5e-324", b"2.4703282292062328e-324",
            b"2.4703282292062327e-324", b"1e-320", b"1e-329", b"1e-330", b"-1e-330", b"1e-400", b"0e999999999", b"1e-99999999999",
            b"1e99999999999", b"-1e99999999999", b"1e0000000000000000000000000000000000000000007", b"1e-00000000000000000000000000000000000010",
            b"1e1000000", b"1e-1000000", b"1e10000000", b"1e+0001000000", b"123456789e-1000005", b"0.000e-99999999999"]
    lits += [b"%de%d" % (m, e) for e in range(300, 312) for m in (1, 9, 17976931348623157, 99999999999999999)]
    lits += [b"1e%d" % e for e in range(-345, -320)]
    return lits


def _encoder(rng, count):
    out = []
    for b in rng.integers(0, 2 ** 63, count, dtype=np.uint64):
        b = int(b)
        if (b >> 52) & 0x7FF == 0x7FF:
            b &= ~(1 << 62)
        x = struct.unpack("<d", struct.pack("<Q", b))[0]
        out += [repr(x).encode(), b"%.17e" % x, b"%.16e" % x]
    return out


def _spellings():
    lits = [b"-0", b"0", b"-0.0", b"0.0e+5", b"1E5", b"1e+5", b"1e-5", b"1E-5", b"-1.5E+10", b"0." + b"0" * 300 + b"15",
            b"-0." + b"0" * 330 + b"1", b"1" + b"0" * 400, b"1" + b"0" * 308, b"1" + b"0" * 309, b"12345" + b"0" * 300 + b"e-300",
            b"0." + b"0" * 20 + b"9007199254740993", b"9007199254740993" + b"0" * 40 + b"e-40", b"1.0000000000000000000000000000001",
            b"0.30000000000000004", b"100000000000000000000000e-23", b"-2.5000000000000000000000000000000000000001e-1"]
    return lits


def corpus(seed=11, scale=1):
    """(family, literal) pairs, deterministic for (seed, scale)"""
    rng = np.random.default_rng(seed)
    fams = [("exact", _exact_edges(rng)), ("rows", _rows(rng, 38 * scale)), ("halfway", _halfway(rng, 4000 * scale)),
            ("range", _range_ends()), ("encoder", _encoder(rng, 20000 * scale)), ("spelling", _spellings())]
    return [(f, x) for f, lits in fams for x in lits]


def bodies_of(lits):
    """one literal per body, in field a / c / d by turn; the other members carry plain values"""
    bodies, fields = [], []
    for k, lit in enumerate(lits):
        f = FIELDS[k % 3][0]
        bodies.append(b'{"i":%d,"f":true,"%s":%s,"s":"x"}' % (k & 0x7FFF, f.encode(), lit))
        fields.append(f)
    return bodies, fields


def read_rows(rows, ln, status, n):
    """per literal: bits (status 0) or error text (status 1), from the Bind rows"""
    got = []
    for k in range(n):
        off = FIELDS[k % 3][1]
        if status[k] == 0:
            got.append(struct.unpack_from("<Q", rows[k].tobytes(), off)[0])
        elif status[k] == 1:
            got.append(rows[k, :int(ln[k])].tobytes())
        else:
            got.append(None)
    return got


def _bind(lits):
    bodies, fields = bodies_of(lits)
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    rows, ln, st = emu.bind_rows(Table(FB_SPEC).serialize(), 0, batch, SLOT)
    return batch, fields, st, read_rows(rows, ln, st, len(lits))


_CACHE = {}


def _cpu_run():
    if "run" not in _CACHE:
        pairs = corpus()
        lits = [x for _, x in pairs]
        _, fields, st, got = _bind(lits)
        _CACHE["run"] = (pairs, lits, fields, st, got)
    return _CACHE["run"]


def test_el_table_matches_exact_powers():
    """every one of the 696 rows of el_tables.inc (the host and the device copy are both built from it) against 10^q
    normalised with exact integers"""
    text = open(os.path.join(ROOT, "gofr_b200", "csrc", "el_tables.inc")).read()
    rows = [(int(lo, 16), int(hi, 16)) for lo, hi in re.findall(r"\{0x([0-9a-f]{16})ull, 0x([0-9a-f]{16})ull\}", text)]
    assert len(rows) == 696
    for q, (lo, hi) in zip(range(EL_MIN, EL_MAX + 1), rows):
        assert hi << 64 | lo == EL[q - EL_MIN], q
        # the table entry is 10^q's mantissa rounded so that the 128-bit product never overestimates by more than the
        # wider step can correct: within one unit of the true value
        exact = Fraction(10) ** q
        e2 = (10 ** q).bit_length() - 1 if q >= 0 else -((10 ** -q - 1).bit_length())   # floor(log2(10^q))
        assert (217706 * q) >> 16 == e2, q                                                 # the exponent the parser implies
        assert abs(Fraction(EL[q - EL_MIN]) - exact * Fraction(2) ** (127 - e2)) <= 1, q


def test_python_eisel_lemire_agrees_with_float():
    """the branch restatement's Eisel-Lemire gives float()'s bits whenever it decides"""
    rng = np.random.default_rng(3)
    for _ in range(20000):
        m = int(rng.integers(1, 10 ** 19, dtype=np.uint64))
        q = int(rng.integers(-340, 300))
        ok, bits, _ = eisel_lemire(m, q)
        if ok:
            assert bits == f64_bits(float(Fraction(m) * Fraction(10) ** q)), (m, q)


def test_emu_corpus_against_exact_rounding():
    """the whole corpus through the device code on the CPU: no decided literal differs from float(), only may-defer
    literals are deferred, overflow gives Go's error text; per-family deferral limits"""
    pairs, lits, fields, st, got = _cpu_run()
    bad = check(lits, st, got, fields)
    assert not bad, [(k, lits[i]) for k, i in bad[:10]]
    fam = {}
    for (f, _), s in zip(pairs, st):
        tot, dfr = fam.get(f, (0, 0))
        fam[f] = (tot + 1, dfr + (s == 2))
    assert fam["encoder"][1] <= fam["encoder"][0] // 1000          # <= 0.1 %: what clients actually send is decided
    assert fam["rows"][1] <= fam["rows"][0] // 20                 # the subnormal rows and the top decade
    assert fam["exact"][1] <= 4 * 66                                # only 2^53+1 x 10^e (exactly half-way) and its like


def test_emu_corpus_coverage():
    """every path is taken; every table row bd_parse_float can reach is read; the 192-bit correction runs"""
    pairs, lits, fields, st, got = _cpu_run()
    paths, rows, hits = {}, set(), 0
    for lit in lits:
        p, r, h = branch(lit)
        paths[p] = paths.get(p, 0) + 1
        rows.update(r)
        hits += h
    assert set(paths) == {"zero", "underflow", "overflow", "exact", "el128", "el192", "trunc"}, paths
    # rows below -347 and above 309 are never read: the parser answers 0 / ErrRange before (lead digit <= -330 / >= 310),
    # and a mantissa has at most 19 digits; their contents are checked by test_el_table_matches_exact_powers
    assert rows == set(range(-347, 310)), sorted(set(range(-347, 310)) - rows)[:10]
    assert hits >= 200, hits


def test_checker_catches_subtle_errors():
    """the checker fails on one ulp, on a deferral it does not allow and on a wrong overflow text"""
    lits = [b"0.1", b"1e23", b"123456789012345678", b"1e400", b"9007199254740993", repr(2.0 ** -1000 * 3).encode()]
    fields = ["a", "c", "d", "a", "c", "d"]
    st = np.array([0, 0, 0, 1, 2, 0])
    got = [f64_bits(0.1), f64_bits(1e23), f64_bits(123456789012345678.0), overflow_text(b"1e400", "a"), None, f64_bits(2.0 ** -1000 * 3)]
    assert check(lits, st, got, fields) == []
    g = list(got); g[1] ^= 1
    assert check(lits, st, g, fields) == [("value", 1)]                        # one ulp off
    s = st.copy(); s[0] = 2
    assert check(lits, s, got, fields) == [("deferred", 0)]                    # an exact-case literal deferred
    s = st.copy(); s[5] = 2
    assert check(lits, s, got, fields) == [("deferred", 5)]                    # encoder output deferred
    g = list(got); g[3] = overflow_text(b"1e400", "c")
    assert check(lits, st, g, fields) == [("overflow", 3)]                     # the error names the wrong field
    s = st.copy(); s[3] = 2
    assert check(lits, s, got, fields) == [("deferred", 3)]                    # a sure overflow is not the host's


def _gpu_check():
    import torch
    from gofr_b200.engine import Engine
    pairs = corpus(seed=12, scale=4)
    lits = [x for _, x in pairs]
    bodies, fields = bodies_of(lits)
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    eng = Engine(Table(FB_SPEC), 0)
    rows, ln, st = eng.bind_device(eng.upload(batch), 21, SLOT)
    torch.cuda.synchronize()
    rows, ln, st = rows.cpu().numpy().reshape(batch.n, SLOT), ln.cpu().numpy().view(np.uint32), st.cpu().numpy().view(np.uint32)
    eng.close()
    got = read_rows(rows, ln, st, len(lits))
    e_rows, e_ln, e_st = emu.bind_rows(Table(FB_SPEC).serialize(), 0, batch, SLOT)
    e_got = read_rows(e_rows, e_ln, e_st, len(lits))
    gpu_vs_emu = [k for k in range(len(lits)) if st[k] != e_st[k] or got[k] != e_got[k]]   # a device-only cause
    emu_vs_float = check(lits, e_st, e_got, fields)                                          # a cause shared with the CPU
    gpu_vs_float = check(lits, st, got, fields)
    fam = {}
    for (f, _), s in zip(pairs, st):
        tot, dfr = fam.get(f, (0, 0))
        fam[f] = (tot + 1, dfr + int(s == 2))
    paths, rws, hits = {}, set(), 0
    for lit in lits:
        p, r, h = branch(lit)
        paths[p] = paths.get(p, 0) + 1
        rws.update(r)
        hits += h
    print("float64 Bind on the GPU: %d literals, %d decided, deferred per family %s, paths %s, table rows covered %d, "
          "EL-192 hits %d, mismatches GPU/emu %d, emu/float %d, GPU/float %d"
          % (len(lits), int((st != 2).sum()), {f: d for f, (_, d) in fam.items()}, paths, len(rws), hits, len(gpu_vs_emu),
             len(emu_vs_float), len(gpu_vs_float)))
    assert not gpu_vs_emu, [(lits[k], int(st[k]), got[k], int(e_st[k]), e_got[k]) for k in gpu_vs_emu[:5]]
    assert not emu_vs_float, [(kind, lits[k]) for kind, k in emu_vs_float[:5]]
    assert not gpu_vs_float
    _gpu_serve_sample(bodies[::7][:65536], st[::7][:65536])


def _gpu_serve_sample(bodies, bind_status):
    """the same bodies through the fused serve kernels (the VALUES instances: packed and slot layout) against the oracle;
    what they leave to the host (status 0) must be exactly what the Bind stage left to it"""
    import torch
    from gofr_b200.engine import Engine
    from tests import oracle as O
    date = S.http_date(1789974595)
    batch = S.RequestBatch.pack([S.Req(S.M_POST, b"/echo", b"", b) for b in bodies])
    o1, f1, m1 = O.OracleTable(FB_SPEC).serve(batch, date)
    want = O.responses(o1, f1)
    host = bind_status == 2
    eng = Engine(Table(FB_SPEC), 0)
    resp = eng.alloc_responses(batch.n, int(f1[-1]) + 4096)
    eng.serve_device(eng.upload(batch), date, resp)
    torch.cuda.synchronize()
    out, off, meta = resp.to_host()
    slot = 2048
    s_out, s_len, s_meta = eng.serve_device_slots(eng.upload(batch), date, slot)
    torch.cuda.synchronize()
    s_out, s_len = s_out.cpu().numpy().reshape(batch.n, slot), s_len.cpu().numpy().view(np.uint32)
    s_meta = s_meta.cpu().numpy().view(np.uint32)
    eng.close()
    ob = out.tobytes()
    for i in range(batch.n):
        if host[i]:
            assert (meta[i] & 0xFFFF) == 0 and off[i + 1] == off[i], (i, bodies[i])
            assert (s_meta[i] & 0xFFFF) == 0 and s_len[i] == 0, (i, bodies[i])
            continue
        assert meta[i] == m1[i] and ob[int(off[i]):int(off[i + 1])] == want[i], (i, bodies[i], ob[int(off[i]):int(off[i + 1])], want[i])
        assert s_meta[i] == m1[i] and s_len[i] == len(want[i]) and s_out[i, :len(want[i])].tobytes() == want[i], (i, bodies[i])
    print("serve sample: %d bodies, packed and slot layouts identical to the oracle, %d left to the host as by the Bind stage"
          % (batch.n, int(host.sum())))


@pytest.mark.gpu
def test_gpu_bind_float_corpus():
    """gofr_bind_device over ~460 000 literals of every family, per literal against the emulation and against float(); a
    64 Ki sample of the bodies through the packed and slot-layout serve kernels against the oracle —
    in a child process, so that a fault cannot leave a sticky CUDA error behind for the other GPU tests"""
    import subprocess
    import sys
    r = subprocess.run([sys.executable, "-c", "import tests.test_gpu_float_bind as t; t._gpu_check()"], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
