"""-m gpu: protobuf-wrapped and play-json record values decoded on the device (value_framing.h inside the parse kernel) against
the host decoder on identical fetches: the same state rows per id, the same ids, offsets and poll statistics, and the same
refusal texts. On an H100 the whole file takes well under a minute (its largest poll is 8 200 batches, 4.2 M records)."""
import json
import math
import struct
import uuid

import numpy as np
import pytest

from oracle import kafka_batch as K
from surge_b200 import ReplayEngine
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest, IngestError

pytestmark = pytest.mark.gpu

CLS = "surge.core.TestBoundedContext."
COUNTER = [(CLS + "CountIncremented", 0, [("incrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)]),
           (CLS + "CountDecremented", 1, [("decrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)]),
           (CLS + "NoOpEvent", 2, [("sequenceNumber", N.JSON_I32, 4)])]
BANK = [("docs.command.BankAccountCreated", 0, [("accountNumber", N.JSON_UUID, 16), ("balance", N.JSON_F64, 32),
                                                 ("accountOwner", N.JSON_PSTR, 40, 16), ("securityCode", N.JSON_PSTR, 56, 8)]),
        ("docs.command.BankAccountUpdated", 1, [("accountNumber", N.JSON_UUID, 16), ("newBalance", N.JSON_F64, 32)])]


class _Pair:
    """One device ingest and one host ingest with the same program and framing, polled with the same bytes."""

    def __init__(self, prog, framing, packer=None, null_type=None, max_keys=1 << 16):
        self.dev, self.host = ReplayEngine(0), ReplayEngine(0)
        self.dev.register_program(prog)
        self.host.register_program(prog)
        self.dg, self.ing = DeviceIngest(self.dev, max_keys), Ingest()
        for g in (self.dg, self.ing):
            if packer is not None:
                g.set_json_packer(*packer)
            g.set_value_framing(framing)
            if null_type is not None:
                g.set_null_value_type(null_type)
        self.parts = set()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.dg.close()
        self.ing.close()
        self.dev.close()
        self.host.close()

    def poll(self, fetches, skip_stats=()):
        host_st = {}
        for p, d in fetches:
            self.dg.submit(p, d)
            for k, v in self.ing.record_batches(p, d).items():
                host_st[k] = host_st.get(k, 0) + v
            self.parts.add(p)
        dev_st = self.dg.fold()
        self.host.fold_ingested(self.ing)
        drop = {"n_trailing_bytes", *skip_stats}
        assert {k: v for k, v in dev_st.items() if k not in drop} == {k: v for k, v in host_st.items() if k not in drop}
        self.check()
        return dev_st

    def refused(self, fetches, same_text=True):
        """both ingests refuse the poll (with the same reason unless same_text is False); returns the device's reason"""
        with pytest.raises(IngestError) as hi:
            for p, d in fetches:
                self.ing.record_batches(p, d)
        with pytest.raises(IngestError) as di:
            for p, d in fetches:
                self.dg.submit(p, d)
            self.dg.fold()
        assert hi.value.code == di.value.code == N.SGR_ERR_INVALID
        host_why, dev_why = str(hi.value).split(": ", 2)[-1], str(di.value).split(": ", 2)[-1]
        assert host_why == dev_why or not same_text, (str(hi.value), str(di.value))
        return dev_why

    def check(self):
        keys = self.ing.keys()
        table, ref = self.dev.export_states(), self.host.export_states()
        _, _, idx = self.dev.get_many(keys, arrays=True)
        assert (idx >= 0).all() and len(set(idx.tolist())) == len(keys)
        assert all(table[i].tobytes() == ref[j].tobytes() for j, i in enumerate(idx.tolist()))
        assert {p: self.dg.offsets(p) for p in self.parts} == {p: self.ing.offsets(p) for p in self.parts}


def _batch(off, recs, **kw):
    return K.encode_record_batch(off, [(d, k, v) for d, (k, v) in enumerate(recs)], **kw)


def _counter_ev(name, agg, seq, **kw):
    return (f"{agg}:{seq}".encode(), json.dumps({"_type": CLS + name, "aggregateId": agg, **kw, "sequenceNumber": seq}, separators=(",", ":")).encode())


def test_reference_counter_json_events_fold_to_their_golden_states():
    events = [_counter_ev("CountIncremented", "a", s, incrementBy=1) for s in (1, 2, 3, 4, 5)]
    events += [_counter_ev("CountIncremented", "ml", 1, incrementBy=1), _counter_ev("CountIncremented", "ml", 2, incrementBy=1),
               _counter_ev("CountDecremented", "ml", 3, decrementBy=1)]
    events += [_counter_ev("NoOpEvent", "n", 9), _counter_ev("ExceptionThrowingEvent", "x", 1, errorMsg="boom")]
    with _Pair(P.counter_program(), N.VALUE_JSON, ("_type", COUNTER, 3)) as t:
        t.poll([(0, _batch(0, events[:3], compression="lz4"))])
        assert np.frombuffer(t.dev.get("a"), "<i4").tolist() == [3, 3]
        t.poll([(0, _batch(3, events[3:], compression="lz4"))])
        assert np.frombuffer(t.dev.get("a"), "<i4").tolist() == [5, 5]
        assert np.frombuffer(t.dev.get("ml"), "<i4").tolist() == [1, 3]
        assert np.frombuffer(t.dev.get("n"), "<i4").tolist() == [0, 0]
        assert t.dev.get("x") is None                                # ExceptionThrowingEvent -> unknown_type: the handler threw


def _uuid(rng):
    return str(uuid.UUID(int=int(rng.integers(0, 2**63)) << 64 | int(rng.integers(0, 2**63))))


def _hard_doubles(rng, n):
    """number texts for the slow path: full-precision reprs, 17-digit forms, long midpoint-like digit strings, subnormal and
    overflow edges"""
    out = []
    edges = ["4.9e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "1.7976931348623157e308", "1.7976931348623158e308",
             "1.7976931348623159e308", "-0", "-0.0", "1e-400", "1e400", "9007199254740993", "2.2250738585072011e-308",
             "0." + "0" * 40 + "123456789012345678", "123456789012345678901234567890123456789012345678901234567890"]
    while len(out) < n:
        x = float(np.frombuffer(rng.bytes(8), "<f8")[0])
        if not math.isfinite(x):
            continue
        r = rng.random()
        out.append(repr(x) if r < 0.4 else "%.17g" % x if r < 0.7 else "%.30e" % x if r < 0.9 else edges[int(rng.integers(0, len(edges)))])
    return out


def _bank_json(rng, a, nums):
    if rng.random() < 0.3:
        obj = {"_type": "docs.command.BankAccountCreated", "accountNumber": _uuid(rng), "accountOwner": f"own-{a}", "securityCode": "1234", "balance": 0}
        text = json.dumps(obj, separators=(",", ":")).replace('"balance":0', '"balance":' + nums[int(rng.integers(0, len(nums)))])
    else:
        obj = {"_type": "docs.command.BankAccountUpdated", "accountNumber": _uuid(rng), "newBalance": 0}
        text = json.dumps(obj, separators=(",", ":")).replace('"newBalance":0', '"newBalance":' + nums[int(rng.integers(0, len(nums)))])
    return text.encode()


def test_bank_account_json_through_the_group_by_path():
    rng = np.random.default_rng(5)
    nums = _hard_doubles(rng, 400) + ["%.2f" % (v / 100) for v in rng.integers(-10**8, 10**8, 400)]
    with _Pair(P.bank_account_program(), N.VALUE_JSON, ("_type", BANK)) as t:
        off = {0: 0, 1: 5000}
        for _ in range(3):
            fetches = []
            for p in off:
                data = bytearray()
                for _ in range(4):
                    recs = []
                    for _ in range(int(rng.integers(1, 60))):
                        a = int(rng.integers(0, 50))
                        recs.append((b"acct-%d:%d" % (a, off[p] + len(recs)), _bank_json(rng, a, nums) if rng.random() < 0.95 else None))
                    data += _batch(off[p], recs, compression="lz4" if rng.random() < 0.5 else "none")
                    off[p] += len(recs)
                fetches.append((p, bytes(data)))
            st = t.poll(fetches)
            assert st["n_records"] > 0


def test_json_state_topic_with_tombstones():
    state = ("", [("State", 0, [("count", N.JSON_I32, 16), ("version", N.JSON_I32, 20)])])
    rng = np.random.default_rng(6)
    with _Pair(P.counter_snapshot_restore_program(), N.VALUE_JSON, state, null_type=1) as t:
        off = 0
        for _ in range(3):
            recs = []
            for _ in range(300):
                a = int(rng.integers(0, 40))
                v = None if rng.random() < 0.25 else json.dumps({"aggregateId": f"s{a}", "count": int(rng.integers(-99, 99)), "version": off + len(recs)}).encode()
                recs.append((b"s%d" % a, v))
            st = t.poll([(0, _batch(off, recs[:150], compression="lz4") + _batch(off + 150, recs[150:]))])
            assert st["n_null_values"] > 0
            off += 300
        assert any(v is None for v in t.dev.get_many(t.ing.keys()))


def _pb_varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _pb_event(rng, aid, payload):
    fields = [b"\x0a" + _pb_varint(len(aid)) + aid, b"\x12" + _pb_varint(len(payload)) + payload]
    if rng.random() < 0.3:                                          # unknown fields of every skippable wire type
        fields += [_pb_varint(9 << 3) + _pb_varint(int(rng.integers(0, 2**62))), _pb_varint((10 << 3) | 1) + bytes(8),
                   _pb_varint((11 << 3) | 5) + bytes(4), _pb_varint((12 << 3) | 2) + b"\x02hi"]
    if rng.random() < 0.3:                                          # a repeated payload: the last one wins
        fields.insert(0, b"\x12\x0c" + struct.pack("<IIi", 2, 0, 77))
    if rng.random() < 0.5:
        rng.shuffle(fields)
    return b"".join(fields)


def test_protobuf_events_with_unknown_and_repeated_fields():
    rng = np.random.default_rng(7)
    with _Pair(P.counter_program(), N.VALUE_PROTOBUF_EVENT) as t:
        off = 0
        for _ in range(3):
            recs = []
            for _ in range(400):
                a = int(rng.integers(0, 80))
                payload = struct.pack("<IIi", int(rng.integers(0, 3)), off + len(recs), int(rng.integers(-1000, 1000))) + bytes(int(rng.integers(0, 45)))
                recs.append((b"p%d:%d" % (a, off + len(recs)), _pb_event(rng, b"p%d" % a, payload)))
            t.poll([(0, _batch(off, recs, compression="lz4")), (1, _batch(off, recs[::-1]))])
            off += 400


def test_large_multi_group_poll_with_hard_doubles():
    """8 200 batches of 512 records over 8 partitions (4.2 M records, two groups of 8 192 batches), BankAccount JSON whose
    balances hold the slow-path double corpus. 64 distinct batches are reused at rising base offsets (the CRC does not cover
    the base offset)."""
    rng = np.random.default_rng(8)
    nums = _hard_doubles(rng, 4000)
    distinct = []
    for b in range(64):
        recs = [(b"acct-%d" % int(rng.integers(0, 20000)), _bank_json(rng, 0, nums)) for _ in range(512)]
        distinct.append(_batch(0, recs, compression="lz4" if b % 2 else "none"))
    fetches = []
    n_batches = 8200
    for p in range(8):
        data, off = bytearray(), 0
        for k in range(n_batches // 8 + (1 if p < n_batches % 8 else 0)):
            b = bytearray(distinct[(p * 7 + k) % 64])
            b[0:8] = struct.pack(">q", off)
            data += b
            off += 512
        fetches.append((p, bytes(data)))
    with _Pair(P.bank_account_program(), N.VALUE_JSON, ("_type", BANK), max_keys=1 << 15) as t:
        st = t.poll(fetches)
        assert st["n_batches"] == n_batches and st["n_records"] == n_batches * 512


def test_each_refusal_applies_nothing_and_the_next_poll_folds():
    good = [_counter_ev("CountIncremented", "a", s, incrementBy=2) for s in range(1, 6)]
    T = (CLS + "CountIncremented").encode()
    bad = [b'[1]', b'{"_type":"%s","incrementBy":1.5,"sequenceNumber":1}' % T, b'{"_type":"%s","incrementBy":2147483648,"sequenceNumber":1}' % T,
           b'{"_type":"%s","incrementBy":"1","sequenceNumber":1}' % T, b'{"_type":"nope","sequenceNumber":1}', b'{"sequenceNumber":1}',
           b'{"_type":"%s","incrementBy":1} x' % T, b'{"_type":"%s","incrementBy":01}' % T, b'{"a":"unterminated', b'{"a":"\x01"}',
           b'{"a":' + b"[" * 33 + b"]" * 33 + b"}", b"{" + b",".join(b'"m%d":1' % k for k in range(49)) + b"}", b'{"a":1,}', b'{"a" 1}', b'{"a":tru}',
           b'{"_type":"%s","incrementBy":' % T + b"1" * 64 + b',"sequenceNumber":0}', b'{"_type":"%s","incrementBy":99999999999999999999,"sequenceNumber":0}' % T,
           b'{"a":', b'{"a":[1 2]}', b'{"a":1.}']
    with _Pair(P.counter_program(), N.VALUE_JSON, ("_type", COUNTER, -1)) as t:
        t.poll([(0, _batch(0, good, compression="lz4"))])
        before = (t.dev.export_states().tobytes(), t.dg.offsets(0))
        whys = set()
        for v in bad:
            whys.add(t.refused([(0, _batch(5, good[:2] + [(b"a", v)] + good[2:], compression="lz4"))]))
            assert (t.dev.export_states().tobytes(), t.dg.offsets(0)) == before
        assert len(whys) == len(bad) and all("JSON event: " in w for w in whys)
        t.poll([(0, _batch(5, good, compression="lz4"))])
    # the string members' reasons, on BankAccount events
    U = str(uuid.UUID(int=7))
    upd = '{"_type":"docs.command.BankAccountUpdated","accountNumber":%s,"newBalance":1.5}'
    cre = '{"_type":"docs.command.BankAccountCreated","accountNumber":"%s","accountOwner":%s,"securityCode":"","balance":2}'
    good = [(b"acct", (upd % json.dumps(U)).encode()), (b"acct", (cre % (U, '"Jane"')).encode())]
    bad = [upd % "5", cre % (U, '"\\q"'), upd % '"not-a-uuid"', upd % json.dumps(U[:-1] + "g"), cre % (U, json.dumps("x" * 16))]
    with _Pair(P.bank_account_program(), N.VALUE_JSON, ("_type", BANK)) as t:
        t.poll([(0, _batch(0, good))])
        before = (t.dev.export_states().tobytes(), t.dg.offsets(0))
        for v in bad:
            whys.add(t.refused([(0, _batch(2, [good[0], (b"acct", v.encode()), good[1]]))]))
            assert (t.dev.export_states().tobytes(), t.dg.offsets(0)) == before
        t.poll([(0, _batch(2, good))])
    assert len(whys) == 25                                     # every JSON reason of the host decoder
    with _Pair(P.counter_program(), N.VALUE_PROTOBUF_EVENT) as t:
        for v in (b"\x12\x7f" + bytes(5), b"\x13", b"\x14\x00"):
            assert t.refused([(0, _batch(0, [(b"k", v)]))]) == "value is not a protobuf Event"
        # a missing payload is 0 bytes, refused by the existing 8..56 length check with the device's own wording
        assert "outside 8..56" in t.refused([(0, _batch(0, [(b"k", b"\x0a\x01a")]))], same_text=False)
        t.poll([(0, _batch(0, [(b"k", b"\x12\x0c" + struct.pack("<IIi", 0, 1, 5))]))])


def _mutate(rng, v):
    b = bytearray(v)
    r = rng.random()
    if r < 0.6:
        for _ in range(int(rng.integers(1, 3))):
            b[int(rng.integers(0, len(b)))] = int(rng.choice(list(b'{}[]",:\\ 0123456789-.eE\x00\xff')))
    elif r < 0.8:
        b = b[:int(rng.integers(0, len(b)))]
    else:
        pos = int(rng.integers(0, len(b)))
        del b[pos:pos + int(rng.integers(1, 4))]
    return bytes(b)


def _host_accepts(framing, data):
    probe = Ingest()
    if framing == N.VALUE_JSON:
        probe.set_json_packer("_type", COUNTER, 3)
    probe.set_value_framing(framing)
    try:
        probe.record_batches(0, data)
        return True
    except IngestError:
        return False
    finally:
        probe.close()


@pytest.mark.parametrize("framing", [N.VALUE_JSON, N.VALUE_PROTOBUF_EVENT])
def test_resealed_mutants_are_refused_or_decoded_alike(framing):
    rng = np.random.default_rng(9 + framing)
    if framing == N.VALUE_JSON:
        vals = [_counter_ev(["CountIncremented", "CountDecremented", "NoOpEvent"][k % 3], f"m{k % 9}", k, incrementBy=k, decrementBy=-k)[1] for k in range(60)]
        pair = _Pair(P.counter_program(), framing, ("_type", COUNTER, 3))
    else:
        vals = [_pb_event(rng, b"m%d" % k, struct.pack("<IIi", k % 3, k, k)) for k in range(60)]
        pair = _Pair(P.counter_program(), framing)
    refused = accepted = 0
    with pair as t:
        off = 0
        for i in range(150):
            recs = [(b"m%d" % (k % 9), vals[int(rng.integers(0, len(vals)))]) for k in range(6)]
            recs[int(rng.integers(0, 6))] = (b"m%d" % (i % 9), _mutate(rng, vals[int(rng.integers(0, len(vals)))]))
            fetch = [(0, _batch(off, recs, compression="lz4" if i % 2 else "none"))]
            if _host_accepts(framing, fetch[0][1]):
                t.poll(fetch, skip_stats=("n_new_keys",) if refused else ())   # (ids of a refused poll stay interned on the device)
                off += len(recs)
                accepted += 1
            else:
                t.refused(fetch, same_text=framing == N.VALUE_JSON)   # (a protobuf mutant may fail the length check)
                refused += 1
    assert refused > 20 and accepted > 20


def test_poll_compressing_above_three_times_and_the_next_one():
    """Counter events with 128-bit hex aggregate ids compress about 4.5x: the first such poll needs the exact-layout repeat
    (timing slot [1]) and raises the arena claim to 8x; the next one does not repeat."""
    rng = np.random.default_rng(10)

    def poll(off):
        recs = []
        for k in range(500):
            aid = "%032x" % int(rng.integers(0, 2**62))
            recs.append((aid.encode(), json.dumps({"_type": CLS + "CountIncremented", "aggregateId": aid, "incrementBy": int(rng.integers(0, 9)),
                                                   "sequenceNumber": off + k}, separators=(",", ":")).encode()))
        return [(0, _batch(off, recs, compression="lz4"))]

    with _Pair(P.counter_program(), N.VALUE_JSON, ("_type", COUNTER, 3)) as t:
        st = t.poll(poll(0))
        assert st["n_decompressed_bytes"] > 3 * st["n_compressed_bytes"]
        assert t.dg.last_timing()["decode_walk"] > 0          # slot [1]: the repeat from an exact layout
        st = t.poll(poll(500))
        assert st["n_decompressed_bytes"] > 3 * st["n_compressed_bytes"]
        assert t.dg.last_timing()["decode_walk"] == 0


def test_setter_misuse():
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1024) as dg:
            with pytest.raises(IngestError) as ei:
                dg.set_value_framing(N.VALUE_JSON)            # no packer registered
            assert ei.value.code == N.SGR_ERR_INVALID
            with pytest.raises(IngestError) as ei:
                dg.set_json_packer("_type", [("A", 0, [("x", N.JSON_I32, 8)])])   # would overwrite the aggregate index
            assert ei.value.code == N.SGR_ERR_INVALID
            with pytest.raises(IngestError):
                dg.set_value_framing(7)
            dg.set_json_packer("_type", COUNTER, 3)
            dg.set_value_framing(N.VALUE_JSON)
            dg.submit(0, _batch(0, [_counter_ev("CountIncremented", "a", 1, incrementBy=4)]))
            for call in (lambda: dg.set_value_framing(N.VALUE_PACKED), lambda: dg.set_json_packer("_type", COUNTER, -1)):
                with pytest.raises(IngestError) as ei:
                    call()
                assert ei.value.code == N.SGR_ERR_STATE
            dg.fold()
            assert np.frombuffer(e.get("a"), "<i4").tolist() == [4, 1]
            dg.reset()                                        # the settings survive a reset: a JSON value still decodes
            dg.submit(0, _batch(0, [_counter_ev("CountIncremented", "b", 1, incrementBy=6)]))
            assert dg.fold()["n_records"] == 1
            dg.set_value_framing(N.VALUE_PACKED)
