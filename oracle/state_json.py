"""Restatement of the JSON state writer (surge_b200/csrc/state_writer.h): a state row's program bytes -> the model's JSON state
value, as play-json's Json.toJson(state) writes a case class of flat members. The tests compare the device and the host build of
state_writer.h with this module byte for byte.

    {"name":value,...}   members in table order, no whitespace (Json.format of a case class)

Members (name, kind, program byte offset, slot bytes), kinds as include/sgr.h SGR_JSON_*:
    I32 / I64  plain decimal, '-' for negatives
    UUID       36 lowercase hex characters 8-4-4-4-12, most significant byte first (java.util.UUID.toString)
    PSTR       a string of the slot's first length-byte bytes (padding ignored); refused when the length byte exceeds len - 1 or
               the bytes are not well-formed UTF-8
    F64        see format_f64; NaN and infinities are refused (BigDecimal cannot hold them)
    ID         the row's aggregate id as a string; refused when it is not well-formed UTF-8, or when the row has no id

Strings: '"' -> \\", '\\' -> \\\\, \\b \\t \\n \\f \\r short, other characters below U+0020 as \\u00XX with UPPERCASE hex (Jackson),
everything else, U+007F and non-ASCII included, as its own UTF-8 bytes. json.dumps is not used: it writes lowercase hex.

Doubles. The digits are the shortest decimal that rounds back to the double, closest to it (Python's repr; Double.toString from
JDK 19 on). play-json 2.9.2 writes a JsNumber(BigDecimal(d)), which starts from those digits. The layout below is what we
understand its JsValueSerializer to do; the play-json source is NOT available here, so it is a restatement, not a pin:
    trailing zeros stripped; plain notation when 1e-10 <= |v| <= 1e20, else BigDecimal.toString's scientific form
    0.0, -0.0 -> 0;  1100.0 -> 1100;  -2.5e-7 -> -0.00000025;  1e20 -> 100000000000000000000;  1.5e21 -> 1.5E+21;
    1e21 -> 1E+21;  1.5e-11 -> 1.5E-11;  5e-324 -> 5E-324
Known doubts, to be settled by GenVectors.scala's stateValues on a JVM:
  - JDKs before 19 print a few doubles with longer digits (4.9E-324 for 5e-324). Those parse back to the same double.
  - play-json may pass a stripped value with no '.' through BigInteger, which would refuse 1E+21.
"""
from __future__ import annotations

import math
import struct
from typing import Optional, Sequence, Tuple

I32, I64, F64, UUID, PSTR, ID = 0, 1, 2, 3, 4, 5

# the refusal texts of state_writer.h (reason_text)
F64_NOT_FINITE = "a Double member holds NaN or an infinity, which a JSON number cannot hold"
PSTR_LENGTH = "a string member's length byte is larger than its slot"
PSTR_UTF8 = "a string member is not well-formed UTF-8"
ID_UTF8 = "the aggregate id is not well-formed UTF-8"
NO_ID = "the row has no aggregate id in the key table"


class Refused(ValueError):
    def __init__(self, member: int, reason: str):
        super().__init__(f"member {member}: {reason}")
        self.member, self.reason = member, reason


_SHORT = {0x22: b'\\"', 0x5C: b"\\\\", 0x08: b"\\b", 0x09: b"\\t", 0x0A: b"\\n", 0x0C: b"\\f", 0x0D: b"\\r"}


def utf8_ok(b: bytes) -> bool:
    try:
        b.decode("utf-8", "strict")   # (Python's codec refuses overlongs, surrogates and code points above U+10FFFF)
        return True
    except UnicodeDecodeError:
        return False


def quote(b: bytes) -> bytes:
    out = bytearray(b'"')
    for c in b:
        if c in _SHORT:
            out += _SHORT[c]
        elif c < 0x20:
            out += b"\\u00%02X" % c
        else:
            out.append(c)
    out += b'"'
    return bytes(out)


def shortest_digits(x: float) -> Tuple[str, int]:
    """(digits without leading or trailing zeros, e) with |x| = int(digits) * 10^e, from repr: x finite and non-zero."""
    s = repr(abs(x))
    mant, _, ex = s.partition("e")
    whole, _, frac = mant.partition(".")
    digits = (whole + frac).lstrip("0")
    e = (int(ex) if ex else 0) - len(frac)
    stripped = digits.rstrip("0")
    return stripped, e + len(digits) - len(stripped)


def format_f64(x: float) -> bytes:
    if math.isnan(x) or math.isinf(x):
        raise ValueError("not finite")
    if x == 0.0:
        return b"0"
    d, e = shortest_digits(x)
    nd = len(d)
    E = nd - 1 + e
    sign = "-" if x < 0 else ""
    if E < -10 or E > 20 or (E == 20 and d != "1"):
        body = d[0] + ("." + d[1:] if nd > 1 else "")
        return f"{sign}{body}E{'+' if E >= 0 else '-'}{abs(E)}".encode()
    if e >= 0:
        return f"{sign}{d}{'0' * e}".encode()
    if E >= 0:
        return f"{sign}{d[:E + 1]}.{d[E + 1:]}".encode()
    return f"{sign}0.{'0' * (-E - 1)}{d}".encode()


def format_uuid(b: bytes) -> bytes:
    h = b[:16].hex()
    return f'"{h[:8]}-{h[8:12]}-{h[12:16]}-{h[16:20]}-{h[20:]}"'.encode()


Member = Tuple  # (name, kind, off, len) or (name, ID)


def member_size(m: Member) -> int:
    kind = m[1]
    return {I32: 4, I64: 8, F64: 8, UUID: 16}.get(kind, m[3] if kind == PSTR else 0)


def write_value(members: Sequence[Member], row: bytes, agg_id: Optional[bytes]) -> bytes:
    """The JSON value of a row (its program bytes) with aggregate id agg_id (None: the row has no id). Raises Refused."""
    out = bytearray(b"{")
    for i, m in enumerate(members):
        name, kind = m[0], m[1]
        if i:
            out += b","
        out += quote(name.encode("utf-8") if isinstance(name, str) else name) + b":"
        if kind == ID:
            if agg_id is None:
                raise Refused(i, NO_ID)
            if not utf8_ok(agg_id):
                raise Refused(i, ID_UTF8)
            out += quote(agg_id)
            continue
        off = m[2]
        if kind == I32:
            out += str(struct.unpack_from("<i", row, off)[0]).encode()
        elif kind == I64:
            out += str(struct.unpack_from("<q", row, off)[0]).encode()
        elif kind == F64:
            x = struct.unpack_from("<d", row, off)[0]
            if math.isnan(x) or math.isinf(x):
                raise Refused(i, F64_NOT_FINITE)
            out += format_f64(x)
        elif kind == UUID:
            out += format_uuid(row[off:off + 16])
        elif kind == PSTR:
            n = row[off]
            if n > m[3] - 1:
                raise Refused(i, PSTR_LENGTH)
            s = bytes(row[off + 1:off + 1 + n])
            if not utf8_ok(s):
                raise Refused(i, PSTR_UTF8)
            out += quote(s)
        else:
            raise ValueError(f"member {i}: unknown kind {kind}")
    out += b"}"
    return bytes(out)


def parse_value(members: Sequence[Member], value: bytes, user: int) -> Tuple[bytes, Optional[str]]:
    """A written value back to (program bytes, id) through Python's json and float: the parse-back check. Members the table
    does not cover stay zero; a PSTR slot is zero padded, as the restore writes it."""
    import json

    obj = json.loads(value.decode("utf-8"), parse_float=float)
    row = bytearray(user)
    agg_id = None
    for m in members:
        name, kind = m[0], m[1]
        v = obj[name if isinstance(name, str) else name.decode("utf-8")]
        if kind == ID:
            agg_id = v
        elif kind == I32:
            struct.pack_into("<i", row, m[2], int(v))
        elif kind == I64:
            struct.pack_into("<q", row, m[2], int(v))
        elif kind == F64:
            struct.pack_into("<d", row, m[2], float(v))
        elif kind == UUID:
            row[m[2]:m[2] + 16] = bytes.fromhex(v.replace("-", ""))
        elif kind == PSTR:
            b = v.encode("utf-8")
            row[m[2]] = len(b)
            row[m[2] + 1:m[2] + 1 + len(b)] = b
    return bytes(row), agg_id


def same_row(members: Sequence[Member], a: bytes, b: bytes) -> bool:
    """Two rows agree on every member the table covers: doubles by == (so -0.0 equals 0.0), PSTR by length byte and content."""
    for m in members:
        kind = m[1]
        if kind == ID:
            continue
        off = m[2]
        if kind == F64:
            if struct.unpack_from("<d", a, off)[0] != struct.unpack_from("<d", b, off)[0]:
                return False
        elif kind == PSTR:
            if a[off:off + 1 + a[off]] != b[off:off + 1 + b[off]]:
                return False
        elif a[off:off + member_size(m)] != b[off:off + member_size(m)]:
            return False
    return True
