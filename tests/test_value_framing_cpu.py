"""The device ingest's value conversion (surge_b200/csrc/value_framing.h) against the host decoder of ingest.cpp, on the CPU.

The header compiles for the host too; tests/fuzz/value_framing_main.cpp runs it under ASan + UBSan next to the host decoder:
every value goes through both (the host as one single-record batch through sgr_ingest_record_batches) and both must refuse with
the same text or accept with the same 56 bytes. The corpus holds the host tests' JSON and protobuf cases, generated objects
(member order, whitespace, escapes, duplicates, nesting to 32 and 33 levels, 48 and 49 members) and thousands of byte mutations
of valid values. Doubles are checked apart, on a few hundred thousand number texts, against Python's float() (correctly
rounded, and independent of both decoders) and a sample against the host's strtod. The corpora live in oracle/value_corpus.py,
shared with the device run of the same values (tests/test_gpu_value_framing_corpus.py).
"""
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import value_corpus as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_build")
BIN = os.path.join(OUT, "value_framing_asan")


def _build():
    os.makedirs(OUT, exist_ok=True)
    srcs = [os.path.join(ROOT, "surge_b200", "csrc", "ingest.cpp"), os.path.join(ROOT, "tests", "fuzz", "value_framing_main.cpp")]
    deps = srcs + [os.path.join(ROOT, "surge_b200", "csrc", "value_framing.h")]
    if os.path.exists(BIN) and os.path.getmtime(BIN) >= max(os.path.getmtime(s) for s in deps):
        return
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer",
           *srcs, "-o", BIN, "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        if "sanitize" in r.stderr or "asan" in r.stderr.lower():
            pytest.skip("sanitizer build unavailable: " + r.stderr[-300:])
        raise AssertionError(r.stderr[-3000:])


def _u32(v):
    return struct.pack("<I", v & 0xFFFFFFFF)


def _s(b):
    b = b.encode("utf-8") if isinstance(b, str) else b
    return _u32(len(b)) + b


def _run_values(tmp_path, framing, values, disc="", events=(), unknown_type=-1):
    body = bytearray(_u32(framing) + _s(disc) + _u32(unknown_type) + _u32(len(events)))
    for name, ty, fields in events:
        body += _s(name) + _u32(ty) + _u32(len(fields))
        for fname, kind, off, ln in fields:
            body += _s(fname) + _u32(kind) + _u32(off) + _u32(ln)
    body += _u32(len(values))
    for v in values:
        body += _s(v)
    path = tmp_path / f"values_{framing}_{len(values)}.bin"
    path.write_bytes(bytes(body))
    r = subprocess.run([BIN, "values", str(path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    last = r.stdout.strip().splitlines()[-1]
    assert "mismatches 0" in last, r.stdout[-4000:]
    return int(last.split("accepted")[1].split()[0]), int(last.split("refused")[1].split()[0])


def test_json_values_agree_with_the_host_decoder(tmp_path):
    _build()
    rng = np.random.default_rng(20261015)
    counter = V.counter_values(rng)
    for unknown in (3, -1):
        acc, ref = _run_values(tmp_path, 2, counter + V.mutants(rng, counter, 3000), "_type", V.COUNTER, unknown)
        assert acc > 1000 and ref > 1000
    bank = V.bank_values(rng)
    acc, ref = _run_values(tmp_path, 2, bank + V.mutants(rng, bank, 3000), "_type", V.BANK)
    assert acc > 300 and ref > 1000
    upd = V.UPD_VALUES
    _run_values(tmp_path, 2, upd + V.mutants(rng, upd, 500), "t", V.UPD)
    state = V.STATE_VALUES
    acc, _ = _run_values(tmp_path, 2, state + V.mutants(rng, state, 500), "", V.STATE)
    assert acc >= 3


def test_protobuf_values_agree_with_the_host_decoder(tmp_path):
    _build()
    rng = np.random.default_rng(7)
    good = V.protobuf_good(rng)
    hand = V.PROTOBUF_HAND
    acc, ref = _run_values(tmp_path, 1, good + hand + V.mutants(rng, good, 3000))
    assert acc > 600 and ref > 100


# ----------------------------------------------------------------------------------------------------------------- doubles
def test_doubles_are_correctly_rounded(tmp_path):
    _build()
    rng = np.random.default_rng(1234)
    texts = V.f64_corpus(rng)
    assert len(texts) > 200000
    body = bytearray(_u32(len(texts)))
    for t in texts:
        body += _s(t) + struct.pack("<d", float(t))
    path = tmp_path / "f64.bin"
    path.write_bytes(bytes(body))
    r = subprocess.run([BIN, "f64", str(path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    last = r.stdout.strip().splitlines()[-1]
    assert "mismatches 0" in last, r.stdout[-4000:]
