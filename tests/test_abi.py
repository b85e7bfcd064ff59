"""Host-side checks that need no GPU: the C-ABI library builds, loads and exports every declared symbol; tables seal,
serialize and deserialize; errors are reported as codes."""
import ctypes as C
import re
import os

import numpy as np
import pytest

from gofr_b200 import _abi
from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests.conftest import has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    L = _abi.lib()
    header = open(os.path.join(ROOT, "include", "gofr_b200.h")).read()
    declared = set(re.findall(r"\b(gofr_[a-z0-9_]+)\s*\(", header))
    declared -= {"gofr_table", "gofr_engine"}
    assert declared, "no declarations found"
    assert declared == set(_abi.DECLARED_SYMBOLS)
    for name in sorted(declared):
        assert hasattr(L, name), f"{name} declared in include/gofr_b200.h but not exported"
    assert L.gofr_abi_version() == 1


def test_no_torch_types_in_header():
    header = open(os.path.join(ROOT, "include", "gofr_b200.h")).read()
    assert "torch" not in header and "at::" not in header


def test_table_seal_serialize_roundtrip():
    t = Table(synth.config4_spec())
    img = t.serialize()
    assert t.route_count() == 64 + 3
    t2 = Table(image=img)
    assert t2.serialize() == img and t2.route_count() == 67


def test_table_errors_are_codes():
    L = _abi.lib()
    with pytest.raises(_abi.GofrError) as e:
        Table(S.TableSpec(routes=[S.Route(S.M_GET, "/x/{id:(a|b)}", S.H_NIL)]))
    assert e.value.code == 2  # GOFR_ERR_UNSUPPORTED
    with pytest.raises(_abi.GofrError) as e:
        Table(S.TableSpec(routes=[S.Route(S.M_GET, "/x", S.H_ROW, schema_id=99)]))
    assert e.value.code == 1
    t = Table(synth.config1_spec())
    h = _abi.HandlerDesc(kind=S.H_NIL)
    assert L.gofr_table_add_route(t.handle, 0, b"/late", 5, C.byref(h), None) == 5  # GOFR_ERR_SEALED
    with pytest.raises(_abi.GofrError):
        Table(image=b"\x00" * 200)
    # seal-time rejections: the code and the text gofr_last_error() gives
    not_bindable = S.Schema(4, "main.Tags", [S.Field("Tags", S.F_STRING, "tags", container=S.C_SLICE)])
    for routes, schemas, code, text in (
            ([S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=4)], [not_bindable], 2, "Bind takes flat structs"),
            ([S.Route(S.M_GET, "/q", S.H_PARAM_FORMAT, s0=b"k", s2=b"\xff")], [], 2, "must be valid UTF-8"),
            ([S.Route(S.M_GET, "/x", 13)], [], 1, "unknown handler kind 13")):
        with pytest.raises(_abi.GofrError) as e:
            Table(S.TableSpec(schemas=schemas, routes=routes))
        assert e.value.code == code and text in L.gofr_last_error().decode(), (code, text)
    # a table whose hot part exceeds the 40 KB shared-memory budget is refused, and the failed seal leaves it unsealed
    big = C.c_void_p()
    assert L.gofr_table_create(C.byref(big), S.FRAME_WIRE) == 0
    for i in range(200):
        p = ("/" + ("r%03d" % i) * 60).encode()
        assert L.gofr_table_add_route(big, S.M_GET, p, len(p), C.byref(h), None) == 0
    favicon = S.TableSpec().favicon
    assert L.gofr_table_add_default_routes(big, favicon, len(favicon)) == 0
    assert L.gofr_table_seal(big) == 7  # GOFR_ERR_CAPACITY
    assert b"needs 76400 bytes of shared memory" in L.gofr_last_error()
    assert L.gofr_table_max_response_bytes(big, 100) == 0 and L.gofr_table_response_bound(big, 10, 0, 10) == 0
    n = C.c_uint64(0)
    assert L.gofr_table_serialize(big, None, C.byref(n)) == 6  # GOFR_ERR_NOT_SEALED
    L.gofr_table_destroy(big)


def test_http_date_helper():
    out = C.create_string_buffer(29)
    _abi.lib().gofr_format_http_date(1789974595, out)
    assert out.raw == b"Mon, 21 Sep 2026 07:09:55 GMT"


@pytest.mark.skipif(has_gpu(), reason="checks the no-device behaviour")
def test_engine_fails_loudly_without_a_gpu():
    """There is no CPU fallback: creating an engine without a CUDA device is an error, not a slow path."""
    t = Table(synth.config1_spec())
    e = C.c_void_p()
    rc = _abi.lib().gofr_engine_create(C.byref(e), t.handle, 0)
    assert rc == 8  # GOFR_ERR_NO_DEVICE
    assert b"no CPU path" in _abi.lib().gofr_last_error()


def test_sealed_image_integrity():
    """the sealed image travels between ranks (NCCL broadcast): deserialize refuses anything that is not byte for byte what
    seal produced — flipped bits, truncation, trailing bytes, a foreign version"""
    import ctypes as C
    import numpy as np
    from gofr_b200 import _abi, synth
    from gofr_b200.table import Table
    L = _abi.lib()
    image = Table(synth.config4_spec()).serialize()
    rng = np.random.default_rng(1)

    def load(b: bytes) -> int:
        t = C.c_void_p()
        buf = np.frombuffer(b, dtype=np.uint8).copy()
        rc = L.gofr_table_deserialize(C.byref(t), buf.ctypes.data, len(b))
        if rc == 0:
            L.gofr_table_destroy(t)
        return rc

    assert load(image) == 0
    for _ in range(200):
        b = bytearray(image)
        pos = int(rng.integers(0, len(b)))
        b[pos] ^= 1 << int(rng.integers(0, 8))
        assert load(bytes(b)) != 0, pos
    assert load(image[:-16]) != 0 and load(image + b"\0" * 16) != 0 and load(image[:100]) != 0


def test_response_bound_covers_every_response():
    """gofr_table_response_bound is what a host batcher sums up to size its output buffer (include/gofr_b200.hpp does):
    it must never be below the response the oracle produces for that request"""
    import numpy as np
    from gofr_b200 import _abi, spec as S, synth
    from gofr_b200.table import Table
    from tests import oracle as O
    L = _abi.lib()
    date = S.http_date(1_700_000_000)
    hostile = S.TableSpec(routes=[S.Route(S.M_GET, "/hello", S.H_RESULT), S.Route(S.M_GET, "/p/{v}", S.H_PATHPARAM_FORMAT, s0=b"v", s2=b"<", s3=b">"),
                                  S.Route(S.M_GET, "/q", S.H_PARAM_FORMAT, s0=b"k", s1=b"d", s2=b"[", s3=b"]")])
    hb = S.RequestBatch.pack(
        [S.Req(S.M_GET, b"/hello", data=S.result_record(S.RESULT_STRING, bytes([1]) * 300)),     # every byte grows six-fold
         S.Req(S.M_GET, b"/hello", data=S.result_record(S.RESULT_ERROR, b"<&>" * 100)),
         S.Req(S.M_GET, b"/p/" + bytes([2]) * 200), S.Req(S.M_GET, b"/q", b"k=" + b"%01" * 150),
         S.Req(S.M_GET, b"//a/../" + b"x" * 500, b"y=" + b"z" * 400),                            # 301 with a long Location
         S.Req(S.M_GET, b"/" + b"%".join([b"a"] * 200))])
    cases = [(synth.config1_spec(), synth.config1_batch(300)), (synth.config2_spec(), synth.config2_batch(300, escape_every=3)),
             (synth.config3_spec(), synth.config3_batch(300)), (synth.config4_spec(), synth.config4_batch(600)), (hostile, hb)]
    for spec, batch in cases:
        for frame in (S.FRAME_WIRE, S.FRAME_INTENDED, S.FRAME_BODY):
            spec.frame_mode = frame
            t = Table(spec)
            out, off, meta = O.OracleTable(spec).serve(batch, date)
            lens = np.diff(off.astype(np.int64))
            for i in range(batch.n):
                d = batch.desc[i]
                bound = L.gofr_table_response_bound(t.handle, int(d["path_len"]), int(d["query_len"]), int(d["data_len"]))
                assert bound >= lens[i], (frame, i, bound, int(lens[i]))
