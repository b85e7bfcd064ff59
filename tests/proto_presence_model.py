"""A second statement of the nested proto3 codec WITH FIELD PRESENCE (proto3 optional, oneof), for
tests/test_proto_presence.py.

It is the model of tests/proto_maps_model.py (maps included) with presence added, and reuses that module's wire helpers.
protobuf-go v1.32.0 (impl/codec_field.go initOneofFieldCoders, encode.go, decode.go) restated, independently of the device
code:
  encode   a set explicit-presence field (ProtoNField.presence: PB_OPTIONAL, or a oneof group 1..7) is written even at its
           zero value or empty, an unset one not at all; every oneof member at its own number, in field-number order.  The
           row: a scalar / string / bytes field with presence has a presence word 0 / 1 before its usual words; a message
           member keeps the singular-message layout.  BAD_ROW for a presence word other than 0 / 1, an unset field whose
           value words are not zero, and two set members of one group.
  decode   list-first, as the maps model: every occurrence of every field is collected with its wire position.  An optional
           field is set iff it occurs; of a oneof group, the member holding the group's last position is set, with its last
           value (the device code finds it in the member's own pass).  A message member occurring twice is DEFER, as every
           singular message field is.
On descriptions without presence it answers as tests/proto_maps_model.py does (checked by the tests)."""
from gofr_b200 import spec as S
from tests import proto_maps_model as PM
from tests.proto_maps_model import (BAD_LENGTH, BAD_ROW, BAD_UTF8, COMPRESSED, DEFER, MAX_MAP_ENTRIES, OK, _Fail, _is64, _items,
                                    _key_of, _packed, _Row, _scalar_payload, _utf8_ok, _varint, _wire, _words)

__all__ = ["OK", "COMPRESSED", "BAD_LENGTH", "BAD_ROW", "BAD_UTF8", "DEFER", "encode", "decode", "fixed_bytes"]


def explicit(f):
    """a singular scalar / string / bytes field with explicit presence: a presence word before its value words"""
    return bool(f.presence) and not f.repeated and f.type not in (S.PB_MESSAGE, S.PB_MAP)


def group(f):
    """the oneof group (1..7) of a member, else 0"""
    return f.presence if 1 <= f.presence <= 7 else 0


def _has_presence(f):
    return explicit(f) or (f.type == S.PB_MESSAGE and group(f) != 0)


def fixed_bytes(msgs, m):
    n = 0
    for f in msgs[m]:
        if f.repeated or f.type == S.PB_MAP:
            n += 4
        elif f.type == S.PB_MESSAGE:
            n += 4 + fixed_bytes(msgs, f.msg)
        else:
            n += (8 if _is64(f.type) else 4) + (4 if explicit(f) else 0)
    return n


# ------------------------------------------------------------------------------------------------------------------
# encode
# ------------------------------------------------------------------------------------------------------------------
def _marshal(msgs, m, fixed: bytes, R: _Row, entry=False, prev=None):
    """the content of one message; entry: m is a map entry type (zero values written; prev[0] the previous key or None)"""
    out = bytearray()
    p = 0
    groups = set()                      # oneof groups with a set member so far
    for k, f in enumerate(msgs[m]):
        tag = f.number << 3
        if _has_presence(f):
            w = fixed_bytes(msgs, f.msg) if f.type == S.PB_MESSAGE else 8 if _is64(f.type) else 4
            present = int.from_bytes(fixed[p:p + 4], "little")
            val = fixed[p + 4:p + 4 + w]
            p += 4 + w
            if present > 1 or (not present and any(val)) or (present and group(f) in groups):
                raise _Fail(BAD_ROW)
            if not present:
                continue
            if group(f):
                groups.add(group(f))
            if f.type == S.PB_MESSAGE:
                sub = _marshal(msgs, f.msg, val, R)
                out += _varint(tag | 2) + _varint(len(sub)) + sub
            elif f.type in (S.PB_STRING, S.PB_BYTES):
                ln = int.from_bytes(val, "little")
                s = R.take(ln)
                if f.type == S.PB_STRING and not _utf8_ok(s):
                    raise _Fail(BAD_UTF8)
                out += _varint(tag | 2) + _varint(ln) + s
            else:
                out += _varint(tag | _wire(f.type)) + _scalar_payload(f.type, val)
            continue
        if f.repeated or f.type == S.PB_MAP:
            n = int.from_bytes(fixed[p:p + 4], "little")
            p += 4
            if (len(R.row) - R.var) // 4 < n:
                raise _Fail(BAD_ROW)
            if f.type in (S.PB_MESSAGE, S.PB_MAP):
                fb = fixed_bytes(msgs, f.msg)
                last = [None]
                for _ in range(n):
                    fx = R.take(fb)
                    sub = _marshal(msgs, f.msg, fx, R, f.type == S.PB_MAP, last)
                    out += _varint(tag | 2) + _varint(len(sub)) + sub
            elif f.type in (S.PB_STRING, S.PB_BYTES):
                for _ in range(n):
                    ln = int.from_bytes(R.take(4), "little")
                    s = R.take(ln)
                    if f.type == S.PB_STRING and not _utf8_ok(s):
                        raise _Fail(BAD_UTF8)
                    out += _varint(tag | 2) + _varint(ln) + s
            elif n:
                eb = 8 if _is64(f.type) else 4
                pk = b"".join(_scalar_payload(f.type, R.take(eb)) for _ in range(n))
                out += _varint(tag | 2) + _varint(len(pk)) + pk
            continue
        is_key = entry and k == 0
        if f.type == S.PB_MESSAGE:
            present = int.from_bytes(fixed[p:p + 4], "little")
            fb = fixed_bytes(msgs, f.msg)
            if present:
                sub = _marshal(msgs, f.msg, fixed[p + 4:p + 4 + fb], R)
                out += _varint(tag | 2) + _varint(len(sub)) + sub
            elif entry:
                out += _varint(tag | 2) + b"\x00"
            p += 4 + fb
        elif f.type in (S.PB_STRING, S.PB_BYTES):
            ln = int.from_bytes(fixed[p:p + 4], "little")
            p += 4
            s = R.take(ln)
            if f.type == S.PB_STRING and not _utf8_ok(s):
                raise _Fail(BAD_UTF8)
            if is_key:
                if prev[0] is not None and not prev[0] < bytes(s):
                    raise _Fail(BAD_ROW)
                prev[0] = bytes(s)
            if ln or entry:
                out += _varint(tag | 2) + _varint(ln) + s
        else:
            eb = 8 if _is64(f.type) else 4
            w = fixed[p:p + eb]
            p += eb
            if is_key:
                key = _key_of(f.type, w)
                if prev[0] is not None and not prev[0] < key:
                    raise _Fail(BAD_ROW)
                prev[0] = key
            if any(w) or entry:
                out += _varint(tag | _wire(f.type)) + _scalar_payload(f.type, w)
    return bytes(out)


def encode(msgs, root, rows, row_off):
    """rows -> (list of frames (b"" on failure), statuses)"""
    frames, meta = [], []
    fb = fixed_bytes(msgs, root)
    for i in range(len(row_off) - 1):
        row = bytes(rows[int(row_off[i]):int(row_off[i + 1])])
        try:
            if len(row) < fb:
                raise _Fail(BAD_ROW)
            body = _marshal(msgs, root, row[:fb], _Row(row, fb))
            frames.append(b"\x00" + len(body).to_bytes(4, "big") + body)
            meta.append(OK)
        except _Fail as e:
            frames.append(b"")
            meta.append(e.status)
    return frames, meta


# ------------------------------------------------------------------------------------------------------------------
# decode
# ------------------------------------------------------------------------------------------------------------------
class _Dec(PM._Dec):
    """the maps model's decoder (its string and map-entry handling) with this module's message layout"""

    def message(self, m, lo, hi, entry=False):
        """(fixed, var) of one message of type m in b[lo:hi]; entry: a map entry (a missing message value is empty)"""
        fields = self.msgs[m]
        occ = [[] for _ in fields]
        last = [-1] * len(fields)       # wire position of each field's last occurrence
        for j, (num, wt, v) in enumerate(_items(self.b, lo, hi)):
            for q, f in enumerate(fields):
                if f.number != num:
                    continue
                if wt == _wire(f.type) or (f.repeated and _wire(f.type) != 2 and wt == 2):
                    occ[q].append((wt, v))
                    last[q] = j
                break
        group_last = {}                 # a oneof member is set iff it holds its group's last position
        for q, f in enumerate(fields):
            if group(f):
                group_last[group(f)] = max(group_last.get(group(f), -1), last[q])
        fixed, var = bytearray(), bytearray()
        for q, (f, L) in enumerate(zip(fields, occ)):
            utf8 = f.type == S.PB_STRING
            if _has_presence(f):
                is_set = bool(L) and (not group(f) or last[q] == group_last[group(f)])
                fixed += (1 if is_set else 0).to_bytes(4, "little")
                if f.type == S.PB_MESSAGE:
                    if len(L) > 1:
                        self.defer = True                          # as for any singular message field
                    parsed = [self.message(f.msg, v[0], v[1]) for _, v in L]
                    fixed += parsed[-1][0] if is_set else bytes(fixed_bytes(self.msgs, f.msg))
                    var += parsed[-1][1] if is_set else b""
                elif f.type in (S.PB_STRING, S.PB_BYTES):
                    ss = [self.string(v[0], v[1], utf8) for _, v in L]   # every occurrence checked, the losing ones too
                    s = ss[-1] if is_set else b""
                    fixed += len(s).to_bytes(4, "little")
                    var += s
                else:
                    fixed += _words(f.type, *L[-1]) if is_set else bytes(8 if _is64(f.type) else 4)
                continue
            if f.type == S.PB_MAP:
                if len(L) > MAX_MAP_ENTRIES:
                    self.defer = True
                ents = [self.entry(f.msg, v[0], v[1]) for _, v in L]
                ents.sort(key=lambda e: e[0])                      # stable: equal keys keep wire order
                keep = [e for j, e in enumerate(ents) if j + 1 == len(ents) or ents[j + 1][0] != e[0]]
                fixed += len(keep).to_bytes(4, "little")
                for _, fx, vr in keep:
                    var += fx + vr
            elif f.repeated and f.type == S.PB_MESSAGE:
                fixed += len(L).to_bytes(4, "little")
                for _, v in L:
                    fx, vr = self.message(f.msg, v[0], v[1])
                    var += fx + vr
            elif f.repeated and f.type in (S.PB_STRING, S.PB_BYTES):
                fixed += len(L).to_bytes(4, "little")
                for _, v in L:
                    s = self.string(v[0], v[1], utf8)
                    var += len(s).to_bytes(4, "little") + s
            elif f.repeated:
                els = []
                for wt, v in L:
                    els += _packed(f.type, self.b, v[0], v[1]) if wt == 2 else [_words(f.type, wt, v)]
                fixed += len(els).to_bytes(4, "little")
                var += b"".join(els)
            elif f.type == S.PB_MESSAGE:
                if len(L) > 1:
                    self.defer = True                              # protobuf-go merges: decode it on the host
                parsed = [self.message(f.msg, v[0], v[1]) for _, v in L]
                if parsed:
                    fixed += (1).to_bytes(4, "little") + parsed[0][0]
                    var += parsed[0][1]
                else:
                    fixed += (1 if entry else 0).to_bytes(4, "little") + bytes(fixed_bytes(self.msgs, f.msg))
            elif f.type in (S.PB_STRING, S.PB_BYTES):
                ss = [self.string(v[0], v[1], utf8) for _, v in L]
                s = ss[-1] if ss else b""
                fixed += len(s).to_bytes(4, "little")
                var += s
            else:
                fixed += _words(f.type, *L[-1]) if L else bytes(8 if _is64(f.type) else 4)
        return bytes(fixed), bytes(var)


def decode(msgs, root, frames):
    """frames -> (rows (b"" unless OK; zero padded to a multiple of 4), statuses)"""
    rows, meta = [], []
    for fr in frames:
        fr = bytes(fr)
        st = OK
        if len(fr) < 5:
            st = BAD_LENGTH
        elif fr[0] == 1:
            st = COMPRESSED
        elif fr[0] != 0 or int.from_bytes(fr[1:5], "big") != len(fr) - 5:
            st = BAD_LENGTH
        row = b""
        if st == OK:
            d = _Dec(msgs, fr)
            try:
                fx, vr = d.message(root, 5, len(fr))
                st = BAD_UTF8 if d.bad_utf8 else DEFER if d.defer else OK
                row = fx + vr
                row += bytes(-len(row) % 4)
            except _Fail as e:
                st = e.status
        rows.append(row if st == OK else b"")
        meta.append(st)
    return rows, meta
