"""TEST INFRASTRUCTURE — corpora of record values for the value framings (surge_b200/csrc/value_framing.h).

Only tests/ import this module. The same values go through the host build of value_framing.h next to the host decoder
(tests/test_value_framing_cpu.py, under ASan + UBSan) and through the device parse kernel next to the host decoder
(tests/test_gpu_value_framing_corpus.py); Python's float() and int() are the independent references for numbers.

  * member tables: COUNTER, BANK, UPD, STATE as (class name, event type, [(member, kind, record offset, slot bytes)]), the
    layout Ingest.set_json_packer takes;
  * play-json values: counter_values, bank_values, UPD_VALUES, STATE_VALUES, and mutants of any of them;
  * protobuf Event values: protobuf_good, PROTOBUF_HAND;
  * number texts: f64_corpus (shortest and 17-digit reprs, truncated and perturbed midpoints, fast-path edges, subnormal and
    overflow edges).

Every generator draws from the numpy Generator it is given, in a fixed order: the same seed gives the same bytes.
"""
from __future__ import annotations

import decimal
import json
import math
import struct
import uuid

import numpy as np

I32, I64, F64, UUID, PSTR = 0, 1, 2, 3, 4          # = surge_b200.native.JSON_*

COUNTER = [("surge.core.TestBoundedContext.CountIncremented", 0, [("incrementBy", I32, 16, 0), ("sequenceNumber", I32, 4, 0)]),
           ("surge.core.TestBoundedContext.CountDecremented", 1, [("decrementBy", I32, 16, 0), ("sequenceNumber", I32, 4, 0)]),
           ("surge.core.TestBoundedContext.NoOpEvent", 2, [("sequenceNumber", I32, 4, 0)])]
BANK = [("docs.command.BankAccountCreated", 0, [("accountNumber", UUID, 16, 0), ("balance", F64, 32, 0), ("accountOwner", PSTR, 40, 16),
                                                 ("securityCode", PSTR, 56, 8)]),
        ("docs.command.BankAccountUpdated", 1, [("accountNumber", UUID, 16, 0), ("newBalance", F64, 32, 0)])]
UPD = [("Updé", 1, [("newBalance", F64, 32, 0), ("big", I64, 40, 0)])]
STATE = [("State", 0, [("count", I32, 16, 0), ("version", I32, 20, 0)])]
T_INC = "surge.core.TestBoundedContext.CountIncremented"


def mutants(rng, good, n):
    out = []
    while len(out) < n:
        b = bytearray(good[int(rng.integers(0, len(good)))])
        style = rng.random()
        if style < 0.5 and b:
            for _ in range(int(rng.integers(1, 3))):
                pos = int(rng.integers(0, len(b)))
                b[pos] = int(rng.choice(list(b'{}[]",:\\ 0123456789-+.eEu\x00\x1f\x7f\xff'))) if rng.random() < 0.6 else int(rng.integers(0, 256))
        elif style < 0.7:
            b = b[:int(rng.integers(0, len(b) + 1))]
        elif style < 0.85 and b:
            pos = int(rng.integers(0, len(b)))
            del b[pos:pos + int(rng.integers(1, 4))]
        else:
            pos = int(rng.integers(0, len(b) + 1))
            b[pos:pos] = bytes(rng.choice(list(b'{}[]",:\\ \t\n\r0123456789-.eE'), int(rng.integers(1, 4))).tolist())
        out.append(bytes(b))
    return out


def escape_some(rng, s):
    """JSON string content for s with some characters written as \\uXXXX (surrogate pairs above the BMP) or short escapes."""
    out = []
    for ch in s:
        r = rng.random()
        cp = ord(ch)
        if r < 0.25:
            if cp >= 0x10000:
                hi, lo = 0xD800 + ((cp - 0x10000) >> 10), 0xDC00 + ((cp - 0x10000) & 0x3FF)
                out.append("\\u%04x\\u%04X" % (hi, lo))
            else:
                out.append(("\\u%04x" if rng.random() < 0.5 else "\\u%04X") % cp)
        elif r < 0.3 and ch == "/":
            out.append("\\/")
        else:
            out.append(json.dumps(ch)[1:-1] if ch in '"\\' or cp < 0x20 else ch)
    return "".join(out)


def _ws(rng):
    return "".join(rng.choice([" ", "\t", "\n", "\r"], int(rng.integers(0, 3)))) if rng.random() < 0.5 else ""


def obj_text(rng, items):
    """items: [(raw key content, raw JSON value text)] -> an object with random whitespace"""
    parts = [f'{_ws(rng)}"{k}"{_ws(rng)}:{_ws(rng)}{v}{_ws(rng)}' for k, v in items]
    return "{" + ",".join(parts) + "}" if parts else "{" + _ws(rng) + "}"


def nested(depth, leaf="1"):
    t = leaf
    for d in range(depth):
        t = ('{"x":' + t + "}") if d % 2 else ("[" + t + "]")
    return t


def counter_values(rng):
    vals = []
    T = T_INC.encode()
    vals += [b'{"_type":"%s","incrementBy":1.5,"sequenceNumber":1}' % T, b'{"_type":"%s","incrementBy":2147483648,"sequenceNumber":1}' % T,
             b'{"_type":"%s","incrementBy":-2147483648,"sequenceNumber":1}' % T, b'{"_type":"%s","incrementBy":-2147483649,"sequenceNumber":1}' % T,
             b'{"_type":"%s","incrementBy":"1","sequenceNumber":1}' % T, b'{"_type":"%s","sequenceNumber":1}' % T,
             b'{"_type":"nope","sequenceNumber":1}', b'{"sequenceNumber":1}', b'[1,2]', b'', b' ', b'{', b'}', b'{}', b'{"_type":5}',
             b'{"_type":"%s","incrementBy":1,"sequenceNumber":1} x' % T, b'{"_type":"%s","incrementBy":01,"sequenceNumber":1}' % T,
             b'{"_type":"%s","incrementBy":1,"sequenceNumber":1' % T, b'{"_type":"%s" "incrementBy":1}' % T, b'{"a":"unterminated',
             b'{"x":{"_type":"nope","incrementBy":9},"_type":"nope","_type":"%s","incrementBy":7,"incrementBy":8,"sequenceNumber":2}' % T,
             b'{"_type":"%s","incrementBy":-0,"sequenceNumber":0}' % T, b'{"_type":"%s","incrementBy":1e2,"sequenceNumber":0}' % T,
             b'{"_type":"%s","incrementBy":99999999999999999999,"sequenceNumber":0}' % T,
             b'{"_type":"%s","incrementBy":' % T + b"1" * 63 + b',"sequenceNumber":0}', b'{"_type":"%s","incrementBy":' % T + b"1" * 64 + b',"sequenceNumber":0}',
             b'{"_type":"%s","incrementBy":1,"sequenceNumber":1,}' % T, b'{"a":[1,]}', b'{"a":[1 2]}', b'{"a":{"b" 1}}', b'{"a":{"b":1,}}',
             b'{"a":tru}', b'{"a":nul}', b'{"a":-}', b'{"a":1.}', b'{"a":1e}', b'{"a":1e+}', b'{"a":.5}', b'{"a":"\x01"}', b'{"a":"\\\x01"}',
             b'{"a\\u00":1}', b'{"_type":"\\u0073urge.core.TestBoundedContext.NoOpEvent","sequenceNumber":3}', b'{"\\u005ftype":"%s","incrementBy":4,"sequenceNumber":5}' % T,
             b'{"_type":"%s","incre\\mentBy":4,"incrementBy":6,"sequenceNumber":5}' % T, b'{"_type":"%s\\x","incrementBy":4,"sequenceNumber":5}' % T,
             b'{"a":' + nested(31).encode() + b',"_type":"%s","incrementBy":1,"sequenceNumber":1}' % T, b'{"a":' + nested(32).encode() + b'}',
             b'{"a":' + nested(33).encode() + b'}', b'{"a":' + nested(40, '"x"').encode() + b'}', b'{"a":[[[[]]]],"b":{}}', b'\xef\xbb\xbf{}']
    # 48 and 49 members
    for n in (47, 48, 49, 50):
        items = [(f"m{k}", str(k)) for k in range(n - 2)] + [("_type", json.dumps(T_INC)), ("sequenceNumber", "7")]
        vals.append(obj_text(rng, items).encode())
    names = ["CountIncremented", "CountDecremented", "NoOpEvent", "SomethingElse"]
    for d in range(1500):
        t = int(rng.integers(0, 4))
        by = int(rng.choice([int(rng.integers(-2**31, 2**31)), 2**31 - 1, -2**31, 0, int(rng.integers(-1000, 1000))]))
        seq = int(rng.integers(0, 2**31))
        cls = f"surge.core.TestBoundedContext.{names[t]}"
        items = [("_type", json.dumps(cls, ensure_ascii=bool(d % 2))), ("aggregateId", json.dumps(f"agg-{d}")), ("sequenceNumber", str(seq))]
        if t == 0:
            items.append(("incrementBy", str(by)))
        if t == 1:
            items.append(("decrementBy", str(by)))
        if d % 3 == 0:
            items.append(("extra", json.dumps({"nested": [1, "two", {"_type": "x", "incrementBy": 5}], "s": 'a"b\\é\U0001F600'}, ensure_ascii=bool(d % 2))))
        if d % 5 == 0:
            items.append(("flag", rng.choice(["true", "false", "null", "-1.5e-3", "[]", "{}"])))
        if d % 7 == 0:                                         # a duplicate that the later one overrides
            items.insert(0, ("sequenceNumber", str(int(rng.integers(0, 100)))))
        if d % 4 == 0:                                         # escaped member names and class names
            items = [(escape_some(rng, k), '"' + escape_some(rng, json.loads(v)) + '"' if v.startswith('"') else v) for k, v in items]
        rng.shuffle(items)
        vals.append(obj_text(rng, items).encode("utf-8"))
    # lone and paired surrogates in a class name
    vals += [b'{"_type":"\\ud800","sequenceNumber":1}', b'{"_type":"\\udc00x","sequenceNumber":1}', b'{"_type":"\\ud83d\\ude00","sequenceNumber":1}',
             b'{"_type":"\\ud83d\\u0041","sequenceNumber":1}', b'{"_type":"\\ud83d\\","sequenceNumber":1}', b'{"_type":"\\ud83d\\u12","sequenceNumber":1}']
    return vals


def _uuid_text(rng):
    u = str(uuid.UUID(int=int(rng.integers(0, 2**63)) << 65 | int(rng.integers(0, 2**63))))
    return u.upper() if rng.random() < 0.2 else u


def bank_values(rng):
    vals = []
    for d in range(900):
        if d % 3:
            owner = rng.choice(["Jane Doe", "Zoë", "", "x" * 15, "x" * 16, "\U0001F600abc", 'q"\\'])
            code = rng.choice(["1234", "", "abcdefg", "abcdefgh"])
            bal = rng.choice([float(rng.integers(0, 10**6)) / 100, float(np.frombuffer(rng.bytes(8), "<f8")[0]), -0.0, 1e-310])
            if not math.isfinite(bal):
                bal = 1.0
            items = [("_type", '"docs.command.BankAccountCreated"'), ("accountNumber", json.dumps(_uuid_text(rng))), ("accountOwner", json.dumps(owner, ensure_ascii=bool(d % 2))),
                     ("securityCode", json.dumps(code)), ("balance", repr(bal))]
        else:
            bal = float(np.frombuffer(rng.bytes(8), "<f8")[0]) if d % 2 else round(float(rng.normal(0, 1e5)), 2)
            if not math.isfinite(bal):
                bal = 0.5
            items = [("_type", '"docs.command.BankAccountUpdated"'), ("accountNumber", json.dumps(_uuid_text(rng))), ("newBalance", repr(bal))]
        if d % 4 == 0:
            items = [(k, '"' + escape_some(rng, json.loads(v)) + '"' if v.startswith('"') else v) for k, v in items]
        rng.shuffle(items)
        vals.append(obj_text(rng, items).encode("utf-8"))
    U = str(uuid.UUID(int=1))
    for acct in ["not-a-uuid", "0000000g-0000-0000-0000-000000000000", U.replace("-", "_"), U + "0", U[:-1], "\\u0030" + U[1:], "0000000\\u0067" + U[8:], U.replace("-", "\\u002d")]:
        vals.append(b'{"_type":"docs.command.BankAccountUpdated","accountNumber":"%s","newBalance":1.0}' % acct.encode())
    vals.append(b'{"_type":"docs.command.BankAccountUpdated","accountNumber":5,"newBalance":1.0}')
    vals.append(b'{"_type":"docs.command.BankAccountUpdated","accountNumber":"%s","newBalance":"1.0"}' % U.encode())
    vals.append(b'{"_type":"docs.command.BankAccountCreated","accountNumber":"%s","accountOwner":"\\q","securityCode":"","balance":1}' % U.encode())
    vals.append(b'{"_type":"docs.command.BankAccountCreated","accountNumber":"%s","accountOwner":5,"securityCode":"","balance":1}' % U.encode())
    return vals


# UPD: a non-ASCII class name behind the discriminator "t", an I64 member at its edges
UPD_VALUES = [json.dumps({"t": "Updé", "newBalance": v, "big": b}, ensure_ascii=bool(d % 2)).encode("utf-8")
              for d, (v, b) in enumerate([(0.1, -2**63), (-0.0, 2**63 - 1), (1e300, 0), (5e-324, -1), (2.2250738585072014e-308, 5), (123456789.12345679, 7), (1.0, 8)])]
UPD_VALUES += [b'{"t":"Upd\\u00e9","newBalance":1,"big":9223372036854775808}', b'{"t":"Upd\\u00e9","newBalance":1,"big":-9223372036854775809}',
               b'{"t":"Upd\\u00E9","newBalance":1e400,"big":-0}', b'{"t":"Upd\xc3\xa9","newBalance":-1e-400,"big":1}']
# STATE: no discriminator, one class
STATE_VALUES = [b'{"aggregateId":"a","count":4,"version":4}', b'{"aggregateId":"b","count":-7,"version":2}', b'{"version":9,"count":1,"aggregateId":"a"}',
                b'{"count":1}', b'{}', b'{"count":1,"version":2,"_type":"whatever"}']


def pb_varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def protobuf_good(rng):
    """600 protobuf Events {aggregateId = 1, payload = 2} with unknown fields of every skippable wire type and repeated payloads"""
    ev = lambda n: struct.pack("<IIi", int(rng.integers(0, 3)), int(rng.integers(0, 2**31)), int(rng.integers(-2**31, 2**31))) + bytes(n)  # noqa: E731
    good = []
    for d in range(600):
        payload = ev(int(rng.integers(0, 45)))
        fields = [b"\x0a" + pb_varint(len(f"agg-{d}")) + f"agg-{d}".encode(), b"\x12" + pb_varint(len(payload)) + payload]
        if d % 3 == 0:                                          # unknown fields of every skippable wire type
            fields.append(pb_varint((int(rng.integers(3, 1000)) << 3) | 0) + pb_varint(int(rng.integers(0, 2**63))))
            fields.append(pb_varint((5 << 3) | 1) + bytes(8))
            fields.append(pb_varint((6 << 3) | 5) + bytes(4))
            fields.append(pb_varint((7 << 3) | 2) + b"\x03abc")
        if d % 4 == 0:                                          # a repeated payload: the last one wins
            other = ev(int(rng.integers(0, 60)))
            fields.insert(0, b"\x12" + pb_varint(len(other)) + other)
        rng.shuffle(fields)
        good.append(b"".join(fields))
    return good


PROTOBUF_HAND = [b"\x12\x7f" + bytes(5), b"\x0a\x01a", b"\x13", b"\x14", b"\x16", b"\x17", b"", b"\x12", b"\x12\x08" + bytes(8), b"\x12\x07" + bytes(7),
                 b"\x12\x38" + bytes(56), b"\x12\x39" + bytes(57), b"\x80" * 10 + b"\x00", b"\x80" * 11, b"\x92\x00\x08" + bytes(8),
                 b"\x09" + bytes(7), b"\x0d" + bytes(3), b"\x08" + b"\xff" * 9 + b"\x01", b"\x08" + b"\xff" * 10, b"\x12\x08" + bytes(8) + b"\x0a"]


def f64_corpus(rng):
    D = decimal.Decimal
    decimal.getcontext().prec = 1200
    texts = []

    def add(t):
        if len(t) < 64:
            texts.append(t)

    def sci(d, k):
        """d (a positive Decimal) with k significant digits, truncated, as d.ddddE+x"""
        s, exp = f"{d:.{k + 5}e}".split("e")
        digits = s.replace(".", "")[:k]
        return digits[0] + ("." + digits[1:] if k > 1 else "") + "e" + str(int(exp))

    doubles = np.frombuffer(rng.bytes(8 * 60000), "<f8")
    for x in doubles:
        if not math.isfinite(x):
            continue
        add(repr(float(x)))
        add("%.17g" % x)
    for x in np.frombuffer(rng.bytes(8 * 20000), "<f8"):
        x = float(x)
        if not math.isfinite(x) or x == 0:
            continue
        x = abs(x)
        mid = (D(x) + D(math.nextafter(x, math.inf))) / 2
        k = int(rng.integers(17, 63))
        t = sci(mid, k)
        add(t)
        mant, ex = t.split("e")
        last = int(mant[-1])
        for delta in (-1, 1):                                     # perturbed in the last digit
            if 0 <= last + delta <= 9:
                add(mant[:-1] + str(last + delta) + "e" + ex)
        add(sci(mid, 40) + "")
    # short decimals of every size class (the fast path and its edges)
    for _ in range(40000):
        nd = int(rng.integers(1, 20))
        digits = "".join(str(int(c)) for c in rng.integers(0, 10, nd))
        digits = str(int(rng.integers(1, 10))) + digits[1:]
        e = int(rng.integers(-30, 30))
        add(f"{digits}e{e}")
        add(f"-{digits[:1]}.{digits[1:] or '0'}E+{abs(e)}")
    # subnormal and overflow edges
    for t in ["4.9e-324", "5e-324", "4.9406564584124654e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "2.4703282292062326e-324",
              "2.47032822920623272e-324", "2.2250738585072011e-308", "2.2250738585072012e-308", "2.2250738585072014e-308", "2.225073858507201e-308",
              "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1.79769313486231580793e308", "1.797693134862315807937e308",
              "1.7976931348623157e+308", "1e308", "1e309", "1e-323", "1e-324", "1e-325", "0.1e-323", "10e307", "0.00001e313",
              "1e999999999999", "-1e999999999999", "1e-999999999999", "0e999999", "0.0e-999", "-0", "-0.0", "-0e5", "0", "0.0",
              "1" + "0" * 50 + "e-50", "0." + "0" * 50 + "1e50", "0." + "0" * 58 + "1", "1" + "0" * 60, "9" * 62, "9" * 62 + "e-400",
              "9007199254740993", "9007199254740992.5", "9007199254740993.0000000000000000000000000001", "1e23", "8.98846567431158e307",
              "3.0517578125e-05", "123456789012345678901234567890e-300", "1e-" + "0" * 55 + "7", "1e+" + "0" * 55 + "7"]:
        add(t)
        add("-" + t if not t.startswith("-") else t[1:])
    half = D(2) ** -1075
    for k in range(17, 60):
        add(sci(half, k))
        t = sci(half, k)
        add(t.replace("e", "1e", 1) if "." in t else t)
    top = (D(2) - D(2) ** -52) * D(2) ** 1023 + D(2) ** 970                 # DBL_MAX + half an ulp: the overflow threshold
    for k in range(17, 60):
        add(sci(top, k))
    return texts
