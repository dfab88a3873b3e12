"""-m gpu: the value-framing corpus of tests/test_value_framing_cpu.py (oracle/value_corpus.py) through the device parse kernel.

The CPU test runs csrc/value_framing.h as a host build; here the same values go through the sm_90a build inside
dg_parse_kernel, next to the host decoder (Ingest) on identical fetches. A mirror program copies every packed byte into the
state (record bytes 0..8 -> row 0..8, record bytes 16..64 -> row 8..56, one CREATE rule per type; a type of 16 or more is a row
with SGR_ST_ERROR), and every value has its own id, so an id's row IS its packed record: the device rows are compared with the
host's, and number texts with Python's float() and int(). Refused values go one per poll among good records, and the device
must give the host's reason and name the refused record. The batch-level half of the file pins which record a batch with
several bad records reports: the lowest, as the host decoder does, whatever thread finds its fault first.
"""
import re
import struct

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import value_corpus as V
from surge_b200 import ReplayEngine
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest, IngestError

pytestmark = pytest.mark.gpu

MIRROR = P.make_program(64, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 0, 8), (N.OP_SET, 8, 16, 48)])] * 16)
LENGTH_TEXT = "packed event value outside 8..56 bytes (u32 type, u32 seq, payload)"   # the device's wording of the 8..56 check


def _why(msg):
    """the reason of a refusal without its location ("partition p offset o: " on the host, "offset o, record r: " on the
    device); the host's 8..56 message (which names the length) in the device's wording"""
    why = re.sub(r"^[A-Z_]+: (partition -?\d+ )?offset -?\d+(, record \d+)?: ", "", msg)
    return LENGTH_TEXT if why.startswith("packed event value of ") else why


class _Pair:
    """A device engine + DeviceIngest and a host engine + Ingest with the mirror program, the same framing and packer."""

    def __init__(self, framing, packer=None, max_keys=1 << 16):
        self.dev, self.host = ReplayEngine(0), ReplayEngine(0)
        self.dev.register_program(MIRROR)
        self.host.register_program(MIRROR)
        self.dg, self.ing = DeviceIngest(self.dev, max_keys), Ingest()
        for g in (self.dg, self.ing):
            if packer is not None:
                g.set_json_packer(*packer)
            g.set_value_framing(framing)
        self.parts = set()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        import torch

        free, total = torch.cuda.mem_get_info(0)
        print(f"device memory in use before the pair closes: {(total - free) / 2**30:.2f} GiB")
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

    def refused(self, p, data):
        """both decoders refuse the one-fetch poll with SGR_ERR_INVALID; returns (host message, device message)"""
        with pytest.raises(IngestError) as hi:
            self.ing.record_batches(p, data)
        with pytest.raises(IngestError) as di:
            self.dg.submit(p, data)
            self.dg.fold()
        assert hi.value.code == di.value.code == N.SGR_ERR_INVALID, (str(hi.value), str(di.value))
        return str(hi.value), str(di.value)

    def applied(self):
        return self.dev.export_states().tobytes(), {p: self.dg.offsets(p) for p in self.parts}

    def rows(self, keys):
        """the device's state rows (u8[n, 56]) and flags of these ids, through sgr_get_batch"""
        states, flags, idx = self.dev.get_many(keys, arrays=True)
        assert (idx >= 0).all()
        return states, flags

    def check(self):
        """whole rows per id (state bytes, flags, err_idx), ids, offsets"""
        keys = self.ing.keys()
        states, flags, idx = self.dev.get_many(keys, arrays=True)
        assert (idx >= 0).all() and len(set(idx.tolist())) == len(keys)
        table, ref = self.dev.export_states(), self.host.export_states()
        assert np.array_equal(table[idx], ref[:len(keys)])
        assert np.array_equal(states, ref[:len(keys), :56]) and np.array_equal(flags, ref[:len(keys), 56:60].copy().view("<u4").ravel())
        assert {p: self.dg.offsets(p) for p in self.parts} == {p: self.ing.offsets(p) for p in self.parts}


def _batch(off, recs, lz4):
    return K.encode_record_batch(off, [(d, k, v) for d, (k, v) in enumerate(recs)], compression="lz4" if lz4 else "none")


def _classify(framing, packer, values):
    """accepted or refused, each value alone in a single-record batch through a host Ingest (as the ASan harness does)"""
    ing = Ingest()
    try:
        if packer is not None:
            ing.set_json_packer(*packer)
        ing.set_value_framing(framing)
        out = []
        for i, v in enumerate(values):
            try:
                ing.record_batches(0, _batch(i, [(b"v%d" % i, v)], False))
                out.append(True)
            except IngestError:
                out.append(False)
        return out
    finally:
        ing.close()


def _json_tables():
    """the JSON corpora of test_json_values_agree_with_the_host_decoder, drawn in its order from its seed"""
    rng = np.random.default_rng(20261015)
    counter = V.counter_values(rng)
    out = {}
    for unknown in (3, -1):
        out[f"counter_unknown{unknown}"] = (N.VALUE_JSON, ("_type", V.COUNTER, unknown), counter + V.mutants(rng, counter, 3000))
    bank = V.bank_values(rng)
    out["bank"] = (N.VALUE_JSON, ("_type", V.BANK), bank + V.mutants(rng, bank, 3000))
    out["upd"] = (N.VALUE_JSON, ("t", V.UPD), V.UPD_VALUES + V.mutants(rng, V.UPD_VALUES, 500))
    out["state"] = (N.VALUE_JSON, ("", V.STATE), V.STATE_VALUES + V.mutants(rng, V.STATE_VALUES, 500))
    return out


def _protobuf_table():
    rng = np.random.default_rng(7)
    good = V.protobuf_good(rng)
    return N.VALUE_PROTOBUF_EVENT, None, good + V.PROTOBUF_HAND + V.mutants(rng, good, 3000)


TABLES = ["counter_unknown3", "counter_unknown-1", "bank", "upd", "state", "protobuf"]


@pytest.mark.parametrize("table", TABLES)
def test_corpus_values_decode_and_refuse_as_on_the_host(table):
    framing, packer, values = _protobuf_table() if table == "protobuf" else _json_tables()[table]
    ok = _classify(framing, packer, values)
    acc = [(b"v%d" % i, v) for i, v in enumerate(values) if ok[i]]
    bad = [(b"v%d" % i, v) for i, v in enumerate(values) if not ok[i]]
    assert acc and bad
    rng = np.random.default_rng(100 + TABLES.index(table))
    with _Pair(framing, packer) as t:
        # accepted values: polls over two partitions, batches of 1..512 records, lz4 and uncompressed alternating (a value
        # starts at an arbitrary offset of the arena and of the wire)
        off, pos, nb = {0: 0, 1: 0}, 0, 0
        order = rng.permutation(len(acc))
        while pos < len(acc):
            fetches = []
            for p in (0, 1):
                data = bytearray()
                for _ in range(int(rng.integers(1, 4))):
                    recs = [acc[j] for j in order[pos:pos + int(rng.integers(1, 513))]]
                    if not recs:
                        break
                    data += _batch(off[p], recs, nb % 2 == 0)
                    pos, off[p], nb = pos + len(recs), off[p] + len(recs), nb + 1
                if data:
                    fetches.append((p, bytes(data)))
            t.poll(fetches)
        # refused values, each in a poll of its own among good records: the host's reason, the refused record named, nothing
        # applied; a good poll after every 64 refusals folds
        before = t.applied()
        for k, (key, v) in enumerate(bad):
            p = k % 2
            recs = [acc[int(j)] for j in rng.integers(0, len(acc), int(rng.integers(0, 24)))]
            at = int(rng.integers(0, len(recs) + 1))
            recs.insert(at, (key, v))
            host_msg, dev_msg = t.refused(p, _batch(off[p], recs, k % 2 == 0))
            assert _why(dev_msg) == _why(host_msg) and f", record {at}: " in dev_msg, (host_msg, dev_msg, v)
            assert t.applied() == before
            if k % 64 == 63 or k == len(bad) - 1:
                recs = [acc[int(j)] for j in rng.integers(0, len(acc), 5)]
                t.poll([(p, _batch(off[p], recs, k % 128 == 63))], skip_stats=("n_new_keys",))   # (ids a refused poll interned)
                off[p] += len(recs)
                before = t.applied()
    print(f"{table}: {len(acc)} values decoded, {len(bad)} refused on the device")


# ------------------------------------------------------------------------------------------------------------------ numbers
def test_every_number_text_is_correctly_rounded_on_the_device():
    """the whole double corpus as {"x":<text>} under one JSON_F64 member at record offset 16 -> row bytes 8..16, bit for bit
    against Python's float()"""
    texts = V.f64_corpus(np.random.default_rng(1234))
    assert len(texts) > 200000
    items = [(b"v%d" % i, b'{"x":%s}' % t.encode()) for i, t in enumerate(texts)]
    with _Pair(N.VALUE_JSON, ("", [("N", 0, [("x", V.F64, 16, 0)])]), max_keys=1 << 19) as t:
        off, nb = {0: 0, 1: 0}, 0
        for lo in range(0, len(items), 1 << 16):                  # four polls of 64 Ki records over two partitions
            fetches = []
            for p, part in enumerate((items[lo:lo + (1 << 15)], items[lo + (1 << 15):lo + (1 << 16)])):
                data = bytearray()
                for b in range(0, len(part), 512):
                    data += _batch(off[p], part[b:b + 512], nb % 2 == 0)
                    off[p], nb = off[p] + len(part[b:b + 512]), nb + 1
                if data:
                    fetches.append((p, bytes(data)))
            assert t.poll(fetches)["n_records"] == min(len(items) - lo, 1 << 16)
        states, flags = t.rows(["v%d" % i for i in range(len(texts))])
        got = states[:, 8:16].copy().view("<u8").ravel()
        want = np.array([struct.unpack("<Q", struct.pack("<d", float(x)))[0] for x in texts], dtype=np.uint64)
        wrong = np.nonzero(got != want)[0]
        assert wrong.size == 0, f"{wrong.size} of {len(texts)} texts:\n" + "\n".join(f"{texts[i]}: got {got[i]:016x} want {want[i]:016x}" for i in wrong[:20])
        assert (flags & N.ST_EXISTS).all() and not (flags & N.ST_ERROR).any()
    print(f"{len(texts)} number texts decoded on the device")


def _int_texts(rng):
    texts = []
    for e in (2**31, -2**31, 2**63, -2**63, 10**18, -10**18, 10**19, -10**19):
        texts += [str(e + d) for d in (-2, -1, 0, 1, 2)]
    texts += ["0", "-0", "1", "-1", "99999999999999999999", "-99999999999999999999", "18446744073709551615", "18446744073709551616",
              "1" + "0" * 40, "-" + "9" * 62]
    for _ in range(300):
        nd = int(rng.choice([1, 5, 9, 10, 11, 18, 19, 19, 20]))
        t = str(int(rng.integers(1, 10))) + "".join(str(int(c)) for c in rng.integers(0, 10, nd - 1))
        texts.append("-" + t if rng.random() < 0.5 else t)
    return texts


@pytest.mark.parametrize("kind", [V.I64, V.I32])
def test_integer_members_match_python_int(kind):
    """I64 and I32 members at the ±2^31 and ±2^63 edges and 19/20-digit texts: accepted ones hold Python's int(), the rest are
    refused one per poll with the host's reason"""
    lo, hi = (-2**63, 2**63 - 1) if kind == V.I64 else (-2**31, 2**31 - 1)
    texts = _int_texts(np.random.default_rng(12 + kind))
    items = [(b"v%d" % i, b'{"x":%s}' % t.encode()) for i, t in enumerate(texts)]
    inside = [i for i, t in enumerate(texts) if lo <= int(t) <= hi]
    outside = [i for i, t in enumerate(texts) if not lo <= int(t) <= hi]
    assert len(inside) > 100 and len(outside) > 50
    with _Pair(N.VALUE_JSON, ("", [("N", 0, [("x", kind, 16, 0)])])) as t:
        recs = [items[i] for i in inside]
        t.poll([(0, _batch(0, recs[:len(recs) // 2], True)), (1, _batch(0, recs[len(recs) // 2:], False))])
        states, _ = t.rows(["v%d" % i for i in inside])
        if kind == V.I64:
            assert states[:, 8:16].copy().view("<i8").ravel().tolist() == [int(texts[i]) for i in inside]
        else:
            assert states[:, 8:12].copy().view("<i4").ravel().tolist() == [int(texts[i]) for i in inside]
            assert not states[:, 12:16].any()
        before = t.applied()
        for k, i in enumerate(outside):
            host_msg, dev_msg = t.refused(0, _batch(len(recs) // 2, [items[inside[k % len(inside)]], items[i]], k % 2 == 0))
            x = int(texts[i])
            want = "integer does not fit an Int" if kind == V.I32 and -2**63 <= x < 2**63 else "integer out of range"
            assert _why(dev_msg) == _why(host_msg) == "JSON event: " + want and ", record 1: " in dev_msg, (texts[i], host_msg, dev_msg)
            assert t.applied() == before


# --------------------------------------------------------------------------------------------------------- deepest frames
def test_a_poll_of_worst_case_frames_at_once():
    """about 100 k records, every one a 48-member object (the most a value may have) with 31 levels of nesting, escaped member
    names and a double for the big-integer path: every resident thread of the parse kernel on its deepest stack at once"""
    rng = np.random.default_rng(11)
    names = [[V.escape_some(rng, f"mé/{j}\U0001F600") for _ in range(4)] for j in range(44)]
    table = [("Deep", 0, [("bal", V.F64, 16, 0), ("n", V.I64, 24, 0)])]
    distinct = []
    for b in range(8):
        recs = []
        for r in range(512):
            x = float(np.frombuffer(rng.bytes(8), "<f8")[0])
            bal = "%.25e" % (x if np.isfinite(x) else 1.0)
            items = [("_type", '"Deep"'), ("bal", bal), ("n", str(int(rng.integers(-2**63, 2**63 - 1)))), ("deep", V.nested(31))]
            items += [(names[j][int(rng.integers(0, 4))], str(j)) for j in range(44)]
            rng.shuffle(items)
            recs.append((b"d%d" % (512 * b + r), V.obj_text(rng, items).encode("utf-8")))
        distinct.append(_batch(0, recs, b % 2 == 0))
    fetches, n_batches = [], 196                                  # 100 352 records; the CRC does not cover the base offset
    for p in range(2):
        data, off = bytearray(), 0
        for k in range(n_batches // 2):
            b = bytearray(distinct[(3 * k + p) % 8])
            b[0:8] = struct.pack(">q", off)
            data += b
            off += 512
        fetches.append((p, bytes(data)))
    with _Pair(N.VALUE_JSON, ("_type", table)) as t:
        st = t.poll(fetches)
        assert st["n_records"] == 512 * n_batches and st["n_new_keys"] == 8 * 512


def test_polls_compressing_above_the_largest_arena_claim():
    """two consecutive JSON polls that compress far above 16x: both need the exact-layout repeat (the claim multiple stops at
    16), and both decode as on the host"""
    T = V.T_INC.encode()

    def poll(off):
        recs = [(b"c%d" % (k % 700), b'{"_type":"%s","incrementBy":%d,"sequenceNumber":%d,"pad":"%s"}' % (T, k % 7, off + k, b"a" * 3000))
                for k in range(2048)]
        return [(0, b"".join(_batch(off + b, recs[b:b + 512], True) for b in range(0, 2048, 512)))]

    with _Pair(N.VALUE_JSON, ("_type", V.COUNTER, 3)) as t:
        for off in (0, 2048):
            st = t.poll(poll(off))
            assert st["n_decompressed_bytes"] > 16 * st["n_compressed_bytes"]
            assert t.dg.last_timing()["decode_walk"] > 0


# -------------------------------------------------------------------------------------- the first failing record of a batch
def _slow_json_refusal():
    """a ~60 KB Counter event whose only fault is a byte after the object: refused only once the whole object is parsed"""
    pad = b",".join([b"12345"] * 10000)
    return b'{"_type":"%s","incrementBy":1,"sequenceNumber":1,"pad":[%s]} x' % (V.T_INC.encode(), pad)


def _counter_recs(n):
    return [(b"k%d" % (k % 97), b'{"_type":"%s","incrementBy":%d,"sequenceNumber":%d}' % (V.T_INC.encode(), k % 5, k)) for k in range(n)]


def _malformed(rec):
    """the encoded record with one stray byte inside its length: the walk passes it, the parse finds it malformed"""
    n, p = K.read_varint(rec, 0)
    body = rec[p:] + b"\x00"
    return K.varint(len(body)) + body


CASES = {
    # record 0 fails slowly (TRAILING_BYTES), record 511 at once (NOT_OBJECT), in another warp
    "json_other_warp": (N.VALUE_JSON, {0: _slow_json_refusal(), 511: b"[1]"}, "JSON event: bytes after the JSON object"),
    # the same with both bad records in one warp
    "json_same_warp": (N.VALUE_JSON, {0: _slow_json_refusal(), 1: b"[1]"}, "JSON event: bytes after the JSON object"),
    # a malformed record (found before any value is looked at) after a JSON refusal
    "malformed_after_json": (N.VALUE_JSON, {0: _slow_json_refusal(), 511: None}, "JSON event: bytes after the JSON object"),
    # protobuf: a value that is no Event (after 60 KB of unknown fields) before one whose payload fails the 8..56 check
    "protobuf_then_length": (N.VALUE_PROTOBUF_EVENT, {0: b"\x08\x01" * 30000 + b"\x13", 511: b"\x0a\x01a"}, "value is not a protobuf Event"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_a_batch_reports_its_first_failing_record(case):
    framing, bad, reason = CASES[case]
    if framing == N.VALUE_JSON:
        packer, recs = ("_type", V.COUNTER, 3), _counter_recs(512)
    else:
        packer, recs = None, [(b"k%d" % (k % 97), b"\x12\x0c" + struct.pack("<IIi", k % 3, k, k)) for k in range(512)]
    malformed = [r for r, v in bad.items() if v is None]
    for r, v in bad.items():
        if v is not None:
            recs[r] = (recs[r][0], v)
    section = b"".join(_malformed(K.encode_record(d, k, v, timestamp_delta=d)) if d in malformed else K.encode_record(d, k, v, timestamp_delta=d)
                       for d, (k, v) in enumerate(recs))
    with _Pair(framing, packer) as t:
        t.poll([(0, _batch(0, _counter_recs(3) if framing == N.VALUE_JSON else recs[1:4], False))])
        before = t.applied()
        for lz4 in (False, True):
            data = K.encode_record_batch(3, [(d, k, v) for d, (k, v) in enumerate(recs)], compression="lz4" if lz4 else "none", records_section=section)
            host_msg, dev_msg = t.refused(0, data)
            print(f"{case} ({'lz4' if lz4 else 'uncompressed'}): host: {host_msg} | device: {dev_msg}")
            assert _why(host_msg) == reason and "offset 3:" in host_msg, host_msg
            assert _why(dev_msg) == reason and "offset 3, record 0: " in dev_msg, dev_msg
            assert t.applied() == before
        t.poll([(0, _batch(3, recs[2:10], True))], skip_stats=("n_new_keys",))


def test_a_record_walk_error_is_reported_before_an_earlier_records_value_error():
    """Known divergence: the device's record walk (lengths, stray bytes, recordsCount) runs before any value is parsed, so a
    batch with a walk error AND an earlier bad value gets the walk's reason on the device and the value's on the host, which
    checks record by record. The code is the same and nothing is applied."""
    recs = _counter_recs(64)
    recs[0] = (recs[0][0], b"[1]")
    section = b"".join(K.encode_record(d, k, v, timestamp_delta=d) for d, (k, v) in enumerate(recs)) + b"\x00"
    with _Pair(N.VALUE_JSON, ("_type", V.COUNTER, 3)) as t:
        t.poll([(0, _batch(0, _counter_recs(3), True))])
        before = t.applied()
        host_msg, dev_msg = t.refused(0, K.encode_record_batch(3, [(d, k, v) for d, (k, v) in enumerate(recs)], records_section=section))
        assert _why(host_msg) == "JSON event: the value is not a JSON object", host_msg
        assert _why(dev_msg) == "stray bytes after the last record", dev_msg
        assert t.applied() == before
