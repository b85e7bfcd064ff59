"""Map fields in the nested proto3 codec: how a description picks its kernels, and descriptions whose field ranges overlap.

gofr_proto_nested_describe hands out the kernels' descriptor; its `maps` half-word (bytes 2..3) selects, on the host, the
kernels compiled with map code.  Map-free descriptions keep the kernels without it."""
import numpy as np

from gofr_b200 import spec as S
from gofr_b200 import _abi
from tests import proto_nested_harness as H

F = S.ProtoNField
INVALID, CAP = 1, 7   # GOFR_ERR_INVALID; GOFR_ERR_CAPACITY = "valid, but no room to write the descriptor"


def _describe(nm, n_msgs, nf, k):
    """the ABI call on hand-edited tables (spec.proto_nested_tables cannot make them)"""
    return _abi.lib().gofr_proto_nested_describe(nm.ctypes.data, n_msgs, nf.ctypes.data, k, 0, None, 0)


def _maps_word(msgs):
    desc = np.zeros(512, np.uint8)
    assert H.describe(msgs, 0, desc) == 0
    return int(desc[2]) | int(desc[3]) << 8


def test_descriptor_marks_descriptions_with_maps():
    assert _maps_word(H.MSGS) == 0
    assert _maps_word([[F(1, S.PB_INT32), F(2, S.PB_MESSAGE, True, 1)], [F(1, S.PB_STRING)]]) == 0
    assert _maps_word([[F(1, S.PB_MAP, False, 1)], [F(1, S.PB_STRING), F(2, S.PB_INT32)]]) == 1
    # a map two levels down marks the whole description
    assert _maps_word([[F(1, S.PB_MESSAGE, False, 1)], [F(3, S.PB_MAP, False, 2)], [F(1, S.PB_BOOL), F(2, S.PB_BYTES)]]) == 1


def test_entry_type_sharing_fields_is_refused():
    # M0 { map<int32, int32> m = 1; }  E = fields 1..2; M2 names the same two fields as a plain message type
    nm, nf, k = S.proto_nested_tables([[F(1, S.PB_MAP, False, 1), F(2, S.PB_MESSAGE, False, 2)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]])
    assert _describe(nm, 2, nf, k) == INVALID                      # type 2 does not exist yet: unknown message type
    nm3 = np.concatenate([nm, nm[1:2]])                            # type 2 = the entry type's field range
    assert _describe(nm3, 3, nf, k) == INVALID
    nm3[2] = (int(nm[1][0]) + 1, 1)                                # ... or a part of it (the value field alone)
    assert _describe(nm3, 3, nf, k) == INVALID
    # the same shapes without the sharing are valid
    ok = [[F(1, S.PB_MAP, False, 1), F(2, S.PB_MESSAGE, False, 2)], [F(1, S.PB_INT32), F(2, S.PB_INT32)], [F(1, S.PB_INT32), F(2, S.PB_INT32)]]
    nm, nf, k = S.proto_nested_tables(ok)
    assert _describe(nm, 3, nf, k) == CAP
