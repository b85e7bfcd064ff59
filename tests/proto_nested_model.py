"""A second statement of the nested proto3 codec — nested, repeated, map and explicit-presence fields — written
independently of the device code.  protobuf-go v1.32.0 (impl/codec_field.go, codec_map.go, initOneofFieldCoders,
encode.go, decode.go) restated:

  nested / repeated
    encode   proto.MarshalOptions{Deterministic: true} + grpc-go's 5-byte prefix.  Recursive: a message is marshalled into
             its own buffer, then copied behind its length.  A field at its zero value is not written; a set singular
             message is, even empty; repeated scalars are packed.
    decode   proto.Unmarshal into the same types, the row in canonical form.  List-first: every occurrence of every field of
             a message is collected in wire order, then the row is laid out field by field.  A singular scalar or string
             keeps its last value; a singular message occurring twice is DEFER (protobuf-go merges: the host decodes it).
  maps
    encode   A map entry writes key and value at their zero values too and a message value always (empty when nil); the row
             must hold the entries in strictly ascending key order, else BAD_ROW.
    decode   A map field's entries are all parsed, STABLE-SORTED by key, and only the last of each run of equal keys is kept
             (the device code selects the next key by rescanning instead).  More than MAX_MAP_ENTRIES entries is DEFER.
  presence (proto3 optional, oneof)
    encode   A set explicit-presence field (ProtoNField.presence: PB_OPTIONAL, or a oneof group 1..7) is written even at its
             zero value or empty, an unset one not at all; every oneof member at its own number, in field-number order.  The
             row: a scalar / string / bytes field with presence has a presence word 0 / 1 before its usual words; a message
             member keeps the singular-message layout.  BAD_ROW for a presence word other than 0 / 1, an unset field whose
             value words are not zero, and two set members of one group.
    decode   An optional field is set iff it occurs; of a oneof group, the member holding the group's last wire position is
             set, with its last value (the device code finds it in the member's own pass).  A message member occurring twice
             is DEFER, as every singular message field is.
The description is spec.ProtoNField lists; rows follow include/gofr_b200.h "Row format".  Statuses as GOFR_GRPC_*."""
from gofr_b200 import spec as S

OK, COMPRESSED, BAD_LENGTH, BAD_PROTO, BAD_UTF8, BAD_ROW, DEFER = 0, 1, 2, 3, 4, 5, 6
MAX_MAP_ENTRIES = 64
_SIGNED = (S.PB_INT32, S.PB_INT64, S.PB_SINT32, S.PB_SINT64, S.PB_SFIXED32, S.PB_SFIXED64)
_FIX64 = (S.PB_DOUBLE, S.PB_FIXED64, S.PB_SFIXED64)
_FIX32 = (S.PB_FLOAT, S.PB_FIXED32, S.PB_SFIXED32)


class _Fail(Exception):
    def __init__(self, status):
        self.status = status


def _is64(t):
    return t in S.PB_64BIT or t == S.PB_DOUBLE


def _wire(t):
    if t in (S.PB_STRING, S.PB_BYTES, S.PB_MESSAGE, S.PB_MAP):
        return 2
    return 1 if t in _FIX64 else 5 if t in _FIX32 else 0


def _varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _utf8_ok(b):
    try:
        bytes(b).decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


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


def _key_of(t, words: bytes):
    """the order of an integer / bool key from its row words"""
    v = int.from_bytes(words[:8] if _is64(t) else words[:4], "little")
    if t == S.PB_BOOL:
        return 1 if v else 0
    bits = 64 if _is64(t) else 32
    if t in _SIGNED and v >> (bits - 1):
        v -= 1 << bits
    return v


# ------------------------------------------------------------------------------------------------------------------
# encode
# ------------------------------------------------------------------------------------------------------------------
class _Row:
    def __init__(self, row: bytes, var: int):
        self.row, self.var = row, var

    def take(self, n):
        if len(self.row) - self.var < n:
            raise _Fail(BAD_ROW)
        p = self.var
        self.var += n
        return self.row[p:p + n]


def _scalar_payload(t, w: bytes):
    w0 = int.from_bytes(w[:4], "little")
    v64 = int.from_bytes(w[:8], "little") if _is64(t) else w0
    if t in (S.PB_INT64, S.PB_UINT64):
        return _varint(v64)
    if t == S.PB_SINT64:
        s = v64 - (1 << 64) if v64 >> 63 else v64
        return _varint(((s << 1) ^ (s >> 63)) & (2 ** 64 - 1))
    if t in (S.PB_INT32, S.PB_ENUM):
        return _varint((w0 - (1 << 32) if w0 >> 31 else w0) & (2 ** 64 - 1))
    if t == S.PB_UINT32:
        return _varint(w0)
    if t == S.PB_SINT32:
        s = w0 - (1 << 32) if w0 >> 31 else w0
        return _varint(((s << 1) ^ (s >> 31)) & 0xFFFFFFFF)
    if t == S.PB_BOOL:
        return b"\x01" if w0 else b"\x00"
    return bytes(w[:8]) if t in _FIX64 else bytes(w[:4])


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
def _get_varint(b, i, end):
    x = 0
    for k in range(10):
        if i + k >= end:
            raise _Fail(BAD_PROTO)
        c = b[i + k]
        if k == 9 and c > 1:
            raise _Fail(BAD_PROTO)
        x |= (c & 0x7F) << (7 * k)
        if c < 0x80:
            return x, i + k + 1
    raise _Fail(BAD_PROTO)


def _items(b, lo, hi):
    """(number, wire type, value or payload slice) of the top-level fields of [lo, hi), unknown groups dropped"""
    out, groups, i = [], [], lo
    while i < hi:
        tag, i = _get_varint(b, i, hi)
        num, wt = tag >> 3, tag & 7
        if num == 0 or num > 0x1FFFFFFF:
            raise _Fail(BAD_PROTO)
        if wt == 0:
            v, i = _get_varint(b, i, hi)
        elif wt == 1:
            if hi - i < 8:
                raise _Fail(BAD_PROTO)
            v, i = int.from_bytes(b[i:i + 8], "little"), i + 8
        elif wt == 5:
            if hi - i < 4:
                raise _Fail(BAD_PROTO)
            v, i = int.from_bytes(b[i:i + 4], "little"), i + 4
        elif wt == 2:
            n, i = _get_varint(b, i, hi)
            if n > hi - i:
                raise _Fail(BAD_PROTO)
            v, i = (i, i + n), i + n
        elif wt == 3:
            if len(groups) == 16:
                raise _Fail(BAD_PROTO)
            groups.append(num)
            continue
        elif wt == 4:
            if not groups or groups[-1] != num:
                raise _Fail(BAD_PROTO)
            groups.pop()
            continue
        else:
            raise _Fail(BAD_PROTO)
        if not groups:
            out.append((num, wt, v))
    if groups:
        raise _Fail(BAD_PROTO)
    return out


def _words(t, wt, v):
    """the row words of a scalar from its wire value"""
    if wt == 0:
        if t == S.PB_SINT64:
            v = (v >> 1) ^ -(v & 1)
        elif t == S.PB_SINT32:
            x = v & 0xFFFFFFFF
            v = (x >> 1) ^ -(x & 1)
        elif t == S.PB_BOOL:
            v = 1 if v else 0
    return (v & (2 ** 64 - 1)).to_bytes(8, "little") if _is64(t) else (v & 0xFFFFFFFF).to_bytes(4, "little")


def _packed(t, b, lo, hi):
    w, out, i = _wire(t), [], lo
    while i < hi:
        if w == 0:
            v, i = _get_varint(b, i, hi)
        else:
            eb = 8 if w == 1 else 4
            if hi - i < eb:
                raise _Fail(BAD_PROTO)
            v, i = int.from_bytes(b[i:i + eb], "little"), i + eb
        out.append(_words(t, w, v))
    return out


class _Dec:
    def __init__(self, msgs, b):
        self.msgs, self.b, self.bad_utf8, self.defer = msgs, b, False, False

    def string(self, lo, hi, utf8):
        s = bytes(self.b[lo:hi])
        if utf8 and not _utf8_ok(s):
            self.bad_utf8 = True
        return s

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

    def entry(self, e, lo, hi):
        """(key order, fixed, var) of one map entry of entry type e"""
        fx, vr = self.message(e, lo, hi, entry=True)
        kt = self.msgs[e][0].type
        if kt == S.PB_STRING:
            n = int.from_bytes(fx[:4], "little")
            return bytes(vr[:n]), fx, vr
        return _key_of(kt, fx), fx, vr


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
