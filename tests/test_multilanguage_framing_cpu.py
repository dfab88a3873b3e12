"""Multilanguage JSON topics on the CPU: SGR_VALUE_PROTOBUF_JSON (a protobuf Event / State whose payload is a flat JSON object)
and the state writer's protobuf wrapping.

  * value_framing.h against the host decoder under ASan + UBSan (tests/fuzz/pbjson_framing_main.cpp, shaped like the harness
    of tests/test_value_framing_cpu.py): the JSON corpus of oracle/value_corpus.py wrapped by the protobuf runtime, and byte
    mutations of both layers. Both must refuse with the same text or accept with the same 56 bytes.
  * the three reference models' values, packed by the host decoder, against the records their restatements expect;
  * framing-3 set-up refusals of sgr_ingest_*;
  * the writer's wrapping (state_writer.h, built for the host under ASan by tests/fuzz/state_wrap_main.cpp) against
    State(aggregateId, payload).SerializeToString() of the protobuf runtime.
The protobuf messages are built at run time from their descriptor (modules/multilanguage-protocol/.../multilanguage-protocol.proto:
Event and State are both {string aggregateId = 1; bytes payload = 2;}), an implementation of the wire format independent of both
decoders."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import multilanguage as ML
from oracle import value_corpus as V
from surge_b200 import native as N
from surge_b200.ingest import Ingest, IngestError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_build")
VF_BIN = os.path.join(OUT, "value_framing_pbjson_asan")
WRAP_BIN = os.path.join(OUT, "state_wrap_asan")


def _pb_class(name):
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

    fdp = descriptor_pb2.FileDescriptorProto(name=f"{name}.proto", package="surge.multilanguage", syntax="proto3")
    m = fdp.message_type.add(name=name)
    m.field.add(name="aggregateId", number=1, type=descriptor_pb2.FieldDescriptorProto.TYPE_STRING, label=descriptor_pb2.FieldDescriptorProto.LABEL_OPTIONAL)
    m.field.add(name="payload", number=2, type=descriptor_pb2.FieldDescriptorProto.TYPE_BYTES, label=descriptor_pb2.FieldDescriptorProto.LABEL_OPTIONAL)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName(f"surge.multilanguage.{name}"))


def _sanitized_build(srcs, deps, binary):
    os.makedirs(OUT, exist_ok=True)
    if os.path.exists(binary) and os.path.getmtime(binary) >= max(os.path.getmtime(s) for s in deps):
        return
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer",
           *srcs, "-o", binary, "-lpthread"]
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


def _run_values(tmp_path, values, disc, events, unknown_type=-1):
    csrc = os.path.join(ROOT, "surge_b200", "csrc")
    srcs = [os.path.join(csrc, "ingest.cpp"), os.path.join(ROOT, "tests", "fuzz", "pbjson_framing_main.cpp")]
    _sanitized_build(srcs, srcs + [os.path.join(csrc, "value_framing.h")], VF_BIN)
    body = bytearray(_s(disc) + _u32(unknown_type) + _u32(len(events)))
    for name, ty, fields in events:
        body += _s(name) + _u32(ty) + _u32(len(fields))
        for fname, kind, off, ln in fields:
            body += _s(fname) + _u32(kind) + _u32(off) + _u32(ln)
    body += _u32(len(values))
    for v in values:
        body += _s(v)
    path = tmp_path / f"pbjson_{len(values)}.bin"
    path.write_bytes(bytes(body))
    r = subprocess.run([VF_BIN, str(path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    last = r.stdout.strip().splitlines()[-1]
    assert "mismatches 0" in last, r.stdout[-4000:]
    return int(last.split("accepted")[1].split()[0]), int(last.split("refused")[1].split()[0])


# ------------------------------------------------------------------------------------------------- value corpus
def test_protobuf_json_values_agree_with_the_host_decoder(tmp_path):
    Event = _pb_class("Event")
    rng = np.random.default_rng(20261019)
    counter = V.counter_values(rng)
    for unknown in (3, -1):
        acc, ref = _run_values(tmp_path, ML.pbjson_corpus(rng, counter, Event), "_type", V.COUNTER, unknown)
        assert acc > 1000 and ref > 3000
    bank = V.bank_values(rng)
    acc, ref = _run_values(tmp_path, ML.pbjson_corpus(rng, bank, Event), "_type", V.BANK)
    assert acc > 300 and ref > 2000
    upd = V.UPD_VALUES
    _run_values(tmp_path, ML.pbjson_corpus(rng, upd, Event), "t", V.UPD)
    acc, _ = _run_values(tmp_path, ML.pbjson_corpus(rng, V.STATE_VALUES, Event), "", V.STATE)
    assert acc >= 3


# ------------------------------------------------------------------------------------ the three reference models
def _host_pack(packer, unknown_type, values):
    ing = Ingest()
    try:
        ing.set_json_packer(*packer, unknown_type=unknown_type)
        ing.set_value_framing(N.VALUE_PROTOBUF_JSON)
        ing.record_batches(0, K.encode_record_batch(0, [(d, b"k%d" % d, v) for d, v in enumerate(values)], compression="lz4"))
        return ing.pending().copy()
    finally:
        ing.close()


def _record(etype, seq, payload_words):
    rec = bytearray(64)
    rec[0:8] = struct.pack("<Ii", etype, seq)
    for off, x in payload_words:
        rec[off:off + 4] = struct.pack("<i", x)
    return bytes(rec)


def test_reference_models_pack_as_their_restatements_expect():
    Event = _pb_class("Event")
    rng = np.random.default_rng(5)
    # multilanguage test model: play-json with the sealed trait's "_type" (TestBoundedContext.scala:92-109)
    cls = {0: ML.ML_COUNTER_EVENTS[1][0][0], 1: ML.ML_COUNTER_EVENTS[1][1][0]}
    vals, want = [], []
    for d in range(500):
        t, by, seq = int(rng.integers(0, 2)), int(rng.integers(-2**31, 2**31)), int(rng.integers(0, 2**31))
        obj = {"_type": cls[t], "aggregateId": "a%d" % d, ("incrementBy" if t == 0 else "decrementBy"): by, "sequenceNumber": seq}
        vals.append(Event(aggregateId="a%d" % d, payload=json.dumps(obj, separators=(",", ":")).encode()).SerializeToString())
        want.append(_record(t, seq, [(16, by)]))
    got = _host_pack(ML.ML_COUNTER_EVENTS, -1, vals)
    assert [r[:8].tobytes() + bytes(8) + r[16:].tobytes() for r in got] == want
    # Scala SDK sample: json4s, one event class, no discriminator (Main.scala:19-57)
    vals, want = [], []
    for d in range(300):
        a = int(rng.integers(-2**31, 2**31))
        vals.append(Event(aggregateId="b", payload=json.dumps({"amount": a}).encode()).SerializeToString())
        want.append(_record(0, 0, [(16, a)]))
    got = _host_pack(ML.INT_BALANCE_EVENTS, -1, vals)
    assert [r[:8].tobytes() + bytes(8) + r[16:].tobytes() for r in got] == want
    # C# SDK sample: Newtonsoft with the "Type" discriminator; any other Type is the handler's `_ => None` arm
    vals, want, events = [], [], []
    for d in range(300):
        ty = str(rng.choice(["MoneyWithdrawn", "MoneyDeposited", "BankEvent", "MoneyTransferred"]))
        a = int(rng.integers(-2**31, 2**31))
        obj = {"Type": ty, "Amount": a}
        vals.append(Event(aggregateId="c", payload=json.dumps(obj).encode()).SerializeToString())
        ev = ML.csharp_bank_event(obj)
        events.append(ev)
        etype = {ML.MoneyWithdrawn: 0, ML.MoneyDeposited: 1}.get(type(ev), ML.CSHARP_BANK_UNKNOWN_TYPE)
        want.append(_record(etype, 0, [(16, a)] if etype < 2 else []))
    got = _host_pack(ML.CSHARP_BANK_EVENTS, ML.CSHARP_BANK_UNKNOWN_TYPE, vals)
    assert [r[:8].tobytes() + bytes(8) + r[16:].tobytes() for r in got] == want
    # the handler's own arms, as the program table states them (MATERIALISE + SUB / ADD, TOMBSTONE)
    assert ML.csharp_bank_event_handler(None, ML.MoneyWithdrawn(5)) == ML.Account(-5)
    assert ML.csharp_bank_event_handler(ML.Account(2**31 - 1), ML.MoneyDeposited(1)) == ML.Account(-2**31)
    assert ML.csharp_bank_event_handler(ML.Account(7), ML.OtherBankEvent("BankEvent")) is None


# ------------------------------------------------------------------------------------------ set-up refusals
def test_framing_3_setup_refusals_on_the_host_decoder():
    ing = Ingest()
    try:
        with pytest.raises(IngestError) as ei:
            ing.set_value_framing(N.VALUE_PROTOBUF_JSON)
        assert ei.value.code == N.SGR_ERR_INVALID and "JSON packer" in str(ei.value)
        for bad in (4, -1, 99):
            with pytest.raises(IngestError) as ei:
                ing.set_value_framing(bad)
            assert ei.value.code == N.SGR_ERR_INVALID
        ing.set_json_packer(*ML.INT_BALANCE_EVENTS)
        ing.set_value_framing(N.VALUE_PROTOBUF_JSON)
        # a refused value names the layer: the message, then the payload
        for value, why in [(b"\x12\x05{}", "value is not a protobuf Event"), (b"\x0a\x01a", "JSON event: the value is not a JSON object"),
                           (b"\x12\x02{}", "JSON event: a numeric member of the event is missing or not a number")]:
            with pytest.raises(IngestError) as ei:
                ing.record_batches(0, K.encode_record_batch(0, [(0, b"k", value)]))
            assert ei.value.code == N.SGR_ERR_INVALID and str(ei.value).endswith(why), str(ei.value)
    finally:
        ing.close()


# --------------------------------------------------------------------------------------- the writer's wrapping
def test_writer_wrapping_matches_the_protobuf_runtime(tmp_path):
    State = _pb_class("State")
    csrc = os.path.join(ROOT, "surge_b200", "csrc")
    src = os.path.join(ROOT, "tests", "fuzz", "state_wrap_main.cpp")
    _sanitized_build([src], [src, os.path.join(csrc, "state_writer.h"), os.path.join(csrc, "f64_tables.h")], WRAP_BIN)
    cases = []
    for n_id in (0, 1, 127, 128, 16383, 16384):
        for n_json in (2, 127, 128, 16383, 16384):
            aid = ("é" * (n_id // 2) + "x" * (n_id % 2)).encode()   # n_id bytes of well-formed UTF-8, as the writer requires of an id
            cases.append((aid, ML.padded(b'{"count":1}', n_json) if n_json > 2 else b"{}"))
    body = bytearray(_u32(len(cases)))
    for aid, js in cases:
        body += _s(aid) + _s(js)
    inp, outp = tmp_path / "wrap.in", tmp_path / "wrap.out"
    inp.write_bytes(bytes(body))
    r = subprocess.run([WRAP_BIN, str(inp), str(outp)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "mismatches 0" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    data, at = outp.read_bytes(), 0
    for aid, js in cases:
        (n,) = struct.unpack_from("<I", data, at)
        got = data[at + 4:at + 4 + n]
        at += 4 + n
        assert got == State(aggregateId=aid.decode(), payload=js).SerializeToString(), (len(aid), len(js))
        back = State.FromString(got)
        assert back.aggregateId.encode() == aid and back.payload == js
    assert at == len(data)
