"""The JSON state writer (surge_b200/csrc/state_writer.h) on the CPU, against its restatement oracle/state_json.py.

tests/fuzz/state_writer_main.cpp builds the header for the host under ASan + UBSan. Doubles: the value corpus's numbers, two
million random bit patterns, every subnormal and normal boundary and the powers of ten around the plain / scientific switch
(1e-10 and 1e20) must give the restatement's bytes, whose digits are Python's repr (the shortest that round-trips) and which
float() reads back to the same double. Rows: integers at their extremes, UUIDs, strings with every escape class and multi-byte
UTF-8, ill-formed UTF-8 and NaN / infinity (refused with the reason and the member), ids with and without a key-table entry. Every
written value must also parse back to its row through the device restore's parser (json_pack<STATE>, host build) and Python's
json. The power tables are regenerated from exact integers and must equal the committed header.
"""
import math
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from oracle import state_json as S
from oracle import value_corpus as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_build")
BIN = os.path.join(OUT, "state_writer_asan")
CSRC = os.path.join(ROOT, "surge_b200", "csrc")


def _build():
    os.makedirs(OUT, exist_ok=True)
    src = os.path.join(ROOT, "tests", "fuzz", "state_writer_main.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in ("state_writer.h", "f64_tables.h", "value_framing.h")]
    if os.path.exists(BIN) and os.path.getmtime(BIN) >= max(os.path.getmtime(s) for s in deps):
        return
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
           "-fno-omit-frame-pointer", src, "-o", BIN]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        if "sanitize" in r.stderr or "asan" in r.stderr.lower():
            pytest.skip("sanitizer build unavailable: " + r.stderr[-300:])
        raise AssertionError(r.stderr[-3000:])


def _run(tmp_path, mode, body):
    src, dst = tmp_path / f"{mode}.in", tmp_path / f"{mode}.out"
    src.write_bytes(body)
    r = subprocess.run([BIN, mode, str(src), str(dst)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return r.stdout, dst.read_bytes()


def _f64_texts(tmp_path, bits):
    bits = np.ascontiguousarray(bits, dtype="<u8")
    _, out = _run(tmp_path, "f64", struct.pack("<Q", len(bits)) + bits.tobytes())
    res, p = [], 0
    for _ in range(len(bits)):
        (n,) = struct.unpack_from("<I", out, p)
        p += 4
        if n == 0xFFFFFFFF:
            res.append(None)
        else:
            res.append(out[p:p + n])
            p += n
    assert p == len(out)
    return res


def _boundary_doubles():
    xs = [0.0, -0.0, 5e-324, 1e-323, 2.2250738585072009e-308, 2.2250738585072014e-308, 1.7976931348623157e308, 1.0, 0.5, 2.0,
          0.1, 0.2, 0.3, 1 / 3, 2 / 3, 9007199254740992.0, 9007199254740993.0, 1e15, 1e16, 1e17, 1e21, 1e22, 1e23, 1.5e21, 1.5e-11,
          1100.0, 0.25, -2.5e-7, 123456789.0, 4.35, 100.0]
    for e in range(-1074, 1024):   # every power of two: the interval's lower end is closer except for the subnormals
        xs.append(math.ldexp(1.0, e))
        xs.append(math.nextafter(math.ldexp(1.0, e), math.inf))
        xs.append(math.nextafter(math.ldexp(1.0, e), 0.0))
    for k in range(-30, 31):       # around the plain / scientific switch and beyond
        for base in (1e-10, 1e20):
            p = base * 10.0 ** k if abs(k) < 20 else float(f"1e{int(math.log10(base)) + k}")
            xs += [p, math.nextafter(p, math.inf), math.nextafter(p, 0.0), 1.5 * p, 9.999 * p]
    for e in range(-325, 309):     # every power of ten and its neighbours
        p = float(f"1e{e}")
        xs += [p, math.nextafter(p, math.inf), math.nextafter(p, 0.0)]
    xs += [-x for x in xs]
    return np.array(xs, dtype="<f8").view("<u8")


def _check_f64(tmp_path, bits):
    texts = _f64_texts(tmp_path, bits)
    bad = []
    for b, got in zip(bits.tolist(), texts):
        x = struct.unpack("<d", struct.pack("<Q", b))[0]
        if not math.isfinite(x):
            if got is not None:
                bad.append((hex(b), got))
            continue
        want = S.format_f64(x)
        if got != want or float(got) != x:
            bad.append((hex(b), repr(x), got, want))
    assert not bad, bad[:10]
    return len(texts)


def test_doubles_match_the_restatement_on_boundaries_and_the_corpus(tmp_path):
    _build()
    rng = np.random.default_rng(20261016)
    corpus = np.array([float(t) for t in V.f64_corpus(rng)], dtype="<f8").view("<u8")
    specials = np.array([0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF], dtype="<u8")
    assert _check_f64(tmp_path, np.concatenate([_boundary_doubles(), corpus, specials])) > 100000


def test_doubles_match_repr_on_random_bit_patterns(tmp_path):
    _build()
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 1 << 64, size=2_000_000, dtype=np.uint64)
    assert _check_f64(tmp_path, bits) == 2_000_000


def test_documented_double_layouts():
    cases = {0.0: b"0", -0.0: b"0", 1100.0: b"1100", 0.25: b"0.25", -2.5e-7: b"-0.00000025", 1e20: b"100000000000000000000",
             1.5e21: b"1.5E+21", 1e21: b"1E+21", 1.5e-11: b"1.5E-11", 5e-324: b"5E-324", 1e-10: b"0.0000000001", 1.5e20: b"1.5E+20"}
    for x, want in cases.items():
        assert S.format_f64(x) == want, (x, S.format_f64(x))


# ------------------------------------------------------------------------------------------------------------------------- rows
def _values_body(members, user, rows):
    body = bytearray(struct.pack("<II", user, len(members)))
    for m in members:
        name = m[0].encode("utf-8") if isinstance(m[0], str) else m[0]
        off, ln = (m[2], m[3] if len(m) > 3 else 0) if m[1] != S.ID else (0, 0)
        body += struct.pack("<I", len(name)) + name + struct.pack("<III", m[1], off, ln)
    body += struct.pack("<I", len(rows))
    for row, agg_id in rows:
        assert len(row) == user
        body += struct.pack("<II", agg_id is not None, len(agg_id or b"")) + (agg_id or b"") + row
    return bytes(body)


def _check_rows(tmp_path, members, user, rows):
    stdout, out = _run(tmp_path, "values", _values_body(members, user, rows))
    last = stdout.strip().splitlines()[-1]
    assert "parse_back_mismatches 0" in last, stdout[-2000:]
    p, n_written, n_refused = 0, 0, 0
    for i, (row, agg_id) in enumerate(rows):
        status, n = struct.unpack_from("<II", out, p)
        p += 8
        got = out[p:p + n]
        p += n
        try:
            want = S.write_value(members, row, agg_id)
        except S.Refused as r:
            assert status, (i, row, agg_id, got)
            assert status >> 8 == r.member, (i, status, r.member)
            assert _REASONS[status & 0xFF] == r.reason, (i, status, r.reason)
            n_refused += 1
            continue
        assert status == 0 and got == want, (i, status, got, want)
        back, back_id = S.parse_value(members, got, user)
        assert S.same_row(members, row, back), (i, got)
        if any(m[1] == S.ID for m in members):
            assert back_id.encode("utf-8") == agg_id
        n_written += 1
    assert p == len(out)
    return n_written, n_refused


_REASONS = {1: S.F64_NOT_FINITE, 2: S.PSTR_LENGTH, 3: S.PSTR_UTF8, 4: S.ID_UTF8, 5: S.NO_ID}

# every escape class, multi-byte UTF-8 of each length, U+007F, and strings ill-formed in each way the validator knows
GOOD_STRINGS = [b"", b"a", b'"', b"\\", b"/", b"\b\t\n\f\r", bytes(range(0x20)), b"\x7f", "é".encode(), "€".encode(), "😀".encode(),
                "aé€😀\"\\\x00\x1f".encode(), "ࠀ￿\U00010000\U0010ffff".encode(), b"plain ascii id 42"]
BAD_STRINGS = [b"\x80", b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xed\xa0\x80", b"\xf0\x80\x80\x80", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80",
               b"\xff", b"\xc3", b"\xe2\x82", b"\xf0\x9f\x98", b"a\xc3(", b"\xe2\x28\xa1"]


def test_counter_rows_with_ids_of_every_escape_class(tmp_path):
    _build()
    members = [("aggregateId", S.ID), ("count", S.I32, 0, 4), ("version", S.I32, 4, 4)]
    rows = []
    ints = [0, 1, -1, 7, -7, 2**31 - 1, -2**31, 10, 99, 100, 123456789]
    for k, s in enumerate(GOOD_STRINGS + BAD_STRINGS):
        rows.append((struct.pack("<ii", ints[k % len(ints)], ints[(k * 3 + 1) % len(ints)]) + bytes(8), s))
    rows.append((bytes(16), None))   # a row past the key table
    rng = np.random.default_rng(3)
    for _ in range(3000):
        s = bytes(rng.integers(0, 256, int(rng.integers(0, 12)), dtype=np.uint8))
        rows.append((rng.bytes(8) + bytes(8), s))
    w, r = _check_rows(tmp_path, members, 16, rows)
    assert w > 100 and r > len(BAD_STRINGS)


def test_bank_account_rows(tmp_path):
    _build()
    members = [("accountNumber", S.UUID, 0, 16), ("accountOwner", S.PSTR, 16, 16), ("securityCode", S.PSTR, 32, 8), ("balance", S.F64, 40, 8)]
    rng = np.random.default_rng(11)
    rows = []

    def pstr(b, slot):
        return bytes([len(b)]) + b + bytes(slot - 1 - len(b))

    owners = [s for s in GOOD_STRINGS if len(s) <= 15] + [s for s in BAD_STRINGS if len(s) <= 15]
    balances = [0.0, -0.0, 1100.0, 0.25, -2.5e-7, 1e20, 1.5e21, 1e21, 1.5e-11, 5e-324, 1.7976931348623157e308, math.nan, math.inf, -math.inf,
                12.34, -99.99, 1e-10, 9.999999999999999e-11]
    for k in range(4000):
        owner = owners[k % len(owners)]
        code = [b"", b"1234", b"\x00\x01", b"abcdefg"][k % 4]
        bal = balances[k % len(balances)] if k < 200 else struct.unpack("<d", rng.bytes(8))[0]
        row = rng.bytes(16) + pstr(owner, 16) + pstr(code, 8) + struct.pack("<d", bal) + rng.bytes(8)
        rows.append((row, None))
    # an overlong length byte, and padding bytes behind the string (ignored)
    rows.append((bytes(16) + bytes([16]) + bytes(15) + pstr(b"", 8) + bytes(16), None))
    rows.append((bytes(16) + bytes([15]) + b"x" * 15 + bytes([8]) + bytes(7) + bytes(16), None))
    rows.append((bytes(16) + bytes([2]) + b"ab" + b"\xff" * 13 + pstr(b"", 8) + bytes(16), None))
    w, r = _check_rows(tmp_path, members, 56, rows)
    assert w > 1500 and r > 100


def test_mixed_120_byte_rows(tmp_path):
    _build()
    members = [("id", S.ID), ("a", S.I64, 0, 8), ("é\"\\\n\x01", S.F64, 8, 8), ("u", S.UUID, 16, 16), ("s", S.PSTR, 32, 64),
               ("i", S.I32, 96, 4), ("t", S.PSTR, 100, 4), ("z", S.F64, 104, 8), ("last", S.I64, 112, 8)]
    rng = np.random.default_rng(5)
    rows = []
    for k in range(2000):
        row = bytearray(rng.bytes(120))
        s = GOOD_STRINGS[k % len(GOOD_STRINGS)][:63]
        row[32] = len(s)
        row[33:33 + len(s)] = s
        row[100] = k % 4            # 3 fits a 4-byte slot; never refused by length
        row[101:104] = b"abc"
        struct.pack_into("<q", row, 112, [-2**63, 2**63 - 1, 0, -1][k % 4])
        if k % 3:
            struct.pack_into("<d", row, 8, float(rng.normal() * 10 ** int(rng.integers(-15, 25))))
            struct.pack_into("<d", row, 104, float(rng.normal()))
        rows.append((bytes(row), GOOD_STRINGS[k % len(GOOD_STRINGS)] if k % 50 else None))
    w, r = _check_rows(tmp_path, members, 120, rows)
    assert w > 1000 and r > 0


def test_power_tables_regenerate(tmp_path):
    out = tmp_path / "f64_tables.h"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gen_f64_tables.py"), str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with open(os.path.join(CSRC, "f64_tables.h")) as f:
        assert out.read_text() == f.read()
