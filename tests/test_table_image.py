"""The sealed image (table_format.h) of a fixed corpus of tables, pinned by length and SHA-256.

Every kernel reads the image, rank 0 broadcasts it and gofr_table_deserialize checks it, so the table compiler must turn
the same registrations into the same bytes.  A deliberate format change re-pins: `python -m tests.test_table_image`
prints the current values."""
import hashlib

import pytest

from gofr_b200 import spec as S
from gofr_b200 import synth
from gofr_b200.table import Table
from tests import test_bind as TB
from tests import test_result as TR
from tests import test_values as TV


def _every_kind() -> S.TableSpec:
    """one route of every handler kind; GOFR_H_RESULT with a schema and without"""
    return S.TableSpec(schemas=[synth.C2_SCHEMA, synth.C3_SCHEMA], routes=[
        S.Route(S.M_GET, "/host", S.H_HOST),
        S.Route(S.M_GET, "/string", S.H_STATIC_STRING, s0=b"pong <&>"),
        S.Route(S.M_GET, "/error", S.H_STATIC_ERROR, s0=b"some error occurred"),
        S.Route(S.M_GET, "/nil", S.H_NIL),
        S.Route(S.M_GET, "/health", S.H_HEALTH),
        S.Route(S.M_GET, "/missing", S.H_MISSING_FILE),
        S.Route(S.M_GET, "/panic", S.H_PANIC),
        S.Route(S.M_GET, "/hello", S.H_PARAM_FORMAT, s0=b"name", s1=b"World", s2=b"Hello ", s3=b"!"),
        S.Route(S.M_GET, "/p/{v}", S.H_PATHPARAM_FORMAT, s0=b"v", s2=b"<", s3=b">"),
        S.Route(S.M_GET, "/row", S.H_ROW, schema_id=1),
        S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=3),
        S.Route(S.M_GET, "/result", S.H_RESULT, schema_id=1),
        S.Route(S.M_GET, "/result/strings", S.H_RESULT),
    ])


def _files(frame_mode: int) -> S.TableSpec:
    """response.File: an empty blob, a small one and one past net/http's 2 KiB buffer (chunked on the wire)"""
    return S.TableSpec(frame_mode=frame_mode, routes=[
        S.Route(S.M_GET, "/empty", S.H_FILE, s0=b"text/plain"),
        S.Route(S.M_GET, "/small", S.H_FILE, s0=b"text/html", blob=b"<html><body>hi</body></html>"),
        S.Route(S.M_GET, "/large", S.H_FILE, s0=b"application/json", blob=bytes(range(256)) * 9),
    ])


def _patterns() -> S.TableSpec:
    """{name:regexp} variables of several atoms, dead routes, templates keyed by a long leading literal, a prefix route"""
    return S.TableSpec(routes=[
        S.Route(S.M_GET, "/date/{day:\\d{4}-\\d{2}}", S.H_HOST),
        S.Route(S.M_GET, "/host/{name:[a-z]+\\.[a-z]{2,4}}/v{n:[0-9]+}", S.H_PATHPARAM_FORMAT, s0=b"name", s2=b"[", s3=b"]"),
        S.Route(S.M_GET, "no-leading-slash", S.H_NIL),
        S.Route(S.M_GET, "/x/{a}}", S.H_NIL),
        S.Route(S.M_GET, "/a/long/leading/literal/{id}", S.H_NIL),
        S.Route(S.M_GET, "/a/long/leading/other/{id}", S.H_STATIC_STRING, s0=b"other"),
        S.Route(S.M_ANY, "/static/", S.H_HOST),
    ])


CORPUS = {
    "config1_spec": lambda: synth.config1_spec(),
    "config2_spec": lambda: synth.config2_spec(),
    "config2_spec_64": lambda: synth.config2_spec(n_routes=64),
    "config3_spec": lambda: synth.config3_spec(),
    "config4_spec": lambda: synth.config4_spec(),
    "config2_spec_intended": lambda: synth.config2_spec(S.FRAME_INTENDED),
    "config2_spec_body": lambda: synth.config2_spec(S.FRAME_BODY),
    "every_kind": _every_kind,
    "files": lambda: _files(S.FRAME_WIRE),
    "files_intended": lambda: _files(S.FRAME_INTENDED),
    "patterns": _patterns,
    # flat (C2), omitempty (C4, ITEM), flattenable nested structs (SHAPE), bare schemas and the values model (float64,
    # pointers, slices, maps)
    "result_omitempty": lambda: TR._spec(),
    "values_row": lambda: TV._spec(),
    "values_result": lambda: TV._spec(S.FRAME_WIRE, S.H_RESULT),
    "bind_float64": lambda: S.TableSpec(schemas=[TB.FL_SCHEMA], routes=[S.Route(S.M_POST, "/echo", S.H_BIND_ECHO, schema_id=9)]),
}

PINS = {
    'bind_float64': (5856, '815ee9b54f3f9dd21b3b81f4bc9caceecb2da22e2586e7d69aea72e74125f6e6'),
    'config1_spec': (6448, '0fe719eff6399514d6a41e0e275e26496ecb6c1ea3914e29ebe85e193be449dc'),
    'config2_spec': (7936, 'db229518286917e29749131b366c43189a719f5b5e2354739755cf320a01a8db'),
    'config2_spec_64': (14176, '99aa4f02e1872112a94d3e5e7c92fe784dd04130ae4dbb8b6111a41c7bf2a551'),
    'config2_spec_body': (4272, '16534c52bfcc38ce608afa9913cb8ba61513472f70086b91003780e236ffc614'),
    'config2_spec_intended': (8144, '20978c79e7eddde3820e34018d191ae79ceaf0b0940483599439951bf825ad5a'),
    'config3_spec': (6144, 'c2888343aedaba45381bc99594bb67975c4894b7967c9e3cb85cce189570b07b'),
    'config4_spec': (23984, '009cab696bdb19b2efe3781debfbd0b22acfcfafad984389ccd2ae8635a61810'),
    'every_kind': (17568, '3a21d13e9bd8ed64783dc810d57504f1a0d7dcd39dfb8b4f16d0b8a9c334681b'),
    'files': (7888, '0eb1f446cb623a11ccb893ee3a950b95ceee8e1138fc016b5af17ae3ddcbe5cb'),
    'files_intended': (8592, 'aa91cbbe3c45e0522e288b573bb4d11ae918a139380629f37df67beceaae7fad'),
    'patterns': (7520, 'e79fc3cb6e08e9db52162e04c565bda193f51ef055e512beeb2f9ebf6632a245'),
    'result_omitempty': (17648, 'cdc86ec6546acf462885bfcfa46e9f60910b1b6675ca17328c16c7b49fc648f3'),
    'values_result': (38976, '73281d848023bc018cf52a3e01c04a50968c938d33beba18f866599c5f2d2344'),
    'values_row': (14992, 'd6008ce3a52f328d3cbd143e0234ef23bdb7fb262e16d51e0042087a246e47d1'),
}


def _image(name: str) -> bytes:
    return Table(CORPUS[name]()).serialize()


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_sealed_image_is_pinned(name):
    img = _image(name)
    assert (len(img), hashlib.sha256(img).hexdigest()) == PINS[name], f"the sealed image of {name} changed"
    assert Table(image=img).serialize() == img, f"{name}: deserialize(serialize(t)) differs"


if __name__ == "__main__":
    for name in sorted(CORPUS):
        img = _image(name)
        print(f"    {name!r}: ({len(img)}, {hashlib.sha256(img).hexdigest()!r}),")
