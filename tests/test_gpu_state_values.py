"""-m gpu: JSON state values written on the device (sgr_set_state_writer, sgr_get_batch_values, sgr_export_changes_values,
sgr_scan_values) against the restatement oracle/state_json.py, byte for byte.

Tables come from sgr_put_batch and from a fold. The value reads must give the rows, ids and order of their row-returning twins,
with every value equal to the restatement's for that row and id; pages cut by a small values_cap must together cover an export
exactly once. Refusals (NaN, an overlong string, an ill-formed id, a row with no id, no writer) fail the whole call with the row
named and nothing written. Exported values restored through the device state-topic restore give the same table back."""
import ctypes as C
import math
import os
import re
import struct
import uuid

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import oracle as O
from oracle import state_json as S
from oracle import value_corpus as VC
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200 import synth as SY
from surge_b200.dingest import DeviceIngest
from surge_b200.engine import ReplayEngine
from surge_b200.native import SgrError

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH_ERR = N.ST_CHANGED | N.ST_ERROR


def state_program(sb, f64=()):
    return P.make_program(sb, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])], f64_fields=list(f64))


COUNTER = [("aggregateId", S.ID), ("count", S.I32, 0), ("version", S.I32, 4)]
BANK = [("accountNumber", S.UUID, 0), ("accountOwner", S.PSTR, 16, 16), ("securityCode", S.PSTR, 32, 8), ("balance", S.F64, 40)]
MIXED = [("id", S.ID), ("a", S.I64, 0), ("é\"\\\n", S.F64, 8), ("u", S.UUID, 16), ("s", S.PSTR, 32, 64), ("i", S.I32, 96),
         ("t", S.PSTR, 100, 4), ("z", S.F64, 104), ("last", S.I64, 112)]
ODD_IDS = ['q"uote', "back\\slash", "ctl\x01\x1f\x7f", "tab\tnl\n", "zoë", "日本", "😀", "", "plain"]
BALANCES = [0.0, -0.0, 1100.0, 0.25, -2.5e-7, 1e20, 1.5e21, 1e21, 1.5e-11, 5e-324, 1.7976931348623157e308, 12.34, -99.99]


def writer_of(members):
    return [(m[0], m[1]) if m[1] == S.ID else (m[0], m[1], m[2], m[3] if len(m) > 3 else 0) for m in members]


def pstr(b, slot):
    return bytes([len(b)]) + b + bytes(slot - 1 - len(b))


def bank_row(rng, k, bal=None):
    owners = [b"", "Zoë".encode(), b'a"b\\c', b"\x01\x7f", "日本".encode()]
    b = BALANCES[k % len(BALANCES)] if bal is None else bal
    return rng.bytes(16) + pstr(owners[k % len(owners)], 16) + pstr(b"%d" % (k % 1000), 8) + struct.pack("<d", b) + rng.bytes(8)


def mixed_row(rng, k):
    row = bytearray(rng.bytes(120))
    s = ODD_IDS[k % len(ODD_IDS)].encode()[:63]
    row[32] = len(s)
    row[33:33 + len(s)] = s
    row[100] = k % 4
    row[101:104] = b"abc"
    struct.pack_into("<d", row, 8, float(rng.normal() * 10 ** int(rng.integers(-15, 25))))
    struct.pack_into("<d", row, 104, BALANCES[k % len(BALANCES)])
    return bytes(row)


def put_raw(e, ids, rows, present=None):
    """sgr_put_batch with ids as raw bytes (so that an id can be ill-formed UTF-8)"""
    n = len(ids)
    offs = np.zeros(n + 1, dtype=np.uint32)
    np.cumsum([len(b) for b in ids], out=offs[1:])
    blob = np.frombuffer(b"".join(ids) or b"\0", dtype=np.uint8)
    r = np.ascontiguousarray(np.frombuffer(b"".join(rows), dtype=np.uint8))
    p = np.ones(n, dtype=np.uint8) if present is None else np.asarray(present, dtype=np.uint8)
    e._ck(e._lib.sgr_put_batch(e._h, blob.ctypes.data, offs.ctypes.data, n, r.ctypes.data, p.ctypes.data, None))


def make_engine(prog, members, ids, rows, present=None):
    e = ReplayEngine(0)
    e.register_program(prog)
    e.put_batch(ids, np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(len(ids), -1), present)
    e.set_state_writer(writer_of(members))
    return e


def check_all_reads(e, members, ids, values_cap):
    """get_many_values, export_changes_values and scan_values against the row-returning reads and the restatement"""
    rows, flags, _ = e.get_many(ids + ["never-seen", "x\x00y"], arrays=True)
    got = e.get_many_values(ids + ["never-seen", "x\x00y"])
    for i, k in enumerate(ids + ["never-seen", "x\x00y"]):
        want = S.write_value(members, rows[i].tobytes(), k.encode()) if flags[i] & N.ST_EXISTS else None
        assert got[i] == want, (k, got[i], want)
    # the export: same rows, ids, order and flags as export_changes; pages end inside tiles
    want_pages = [(i.tolist(), f.tolist(), r.copy(), kk) for i, f, _, r, kk in e.export_changes(CH_ERR, page_rows=1 << 20)]
    w_idx = [x for p in want_pages for x in p[0]]
    w_fl = [x for p in want_pages for x in p[1]]
    w_ids = [x for p in want_pages for x in p[3]]
    w_rows = [r for p in want_pages for r in p[2]]
    pages = list(e.export_changes_values(CH_ERR, max_rows=1 << 20, values_cap=values_cap))
    g_idx = [x for p in pages for x in p[0].tolist()]
    assert g_idx == w_idx and len(set(g_idx)) == len(g_idx)
    assert [x for p in pages for x in p[1].tolist()] == w_fl
    assert [x for p in pages for x in p[3]] == w_ids
    vals = [v for p in pages for v in p[4]]
    for k, f, r, v in zip(w_ids, w_fl, w_rows, vals):
        assert v == (S.write_value(members, r.tobytes(), k.encode()) if f & N.ST_EXISTS else None), (k, v)
    # the scan, the same way
    s_want = [(i.tolist(), r.copy(), kk) for i, _, r, kk in e.scan(page_rows=1 << 20)]
    s_pages = list(e.scan_values(max_rows=1 << 20, values_cap=values_cap))
    assert [x for p in s_pages for x in p[0].tolist()] == [x for p in s_want for x in p[0]]
    s_ids = [x for p in s_pages for x in p[2]]
    assert s_ids == [x for p in s_want for x in p[2]]
    for k, r, v in zip(s_ids, [r for p in s_want for r in p[1]], [v for p in s_pages for v in p[3]]):
        assert v == S.write_value(members, r.tobytes(), k.encode())
    return len(pages), len(s_pages)


def test_counter_bank_and_mixed_tables_match_the_restatement():
    rng = np.random.default_rng(1)
    # Counter: ids of every escape class, a tombstone, then a second batch so that CHANGED / None rows mix
    ids = ODD_IDS + ["c-%d" % i for i in range(3000)]
    rows = [struct.pack("<ii", int(rng.integers(-2**31, 2**31)), int(rng.integers(0, 1000))) for _ in ids]
    e = make_engine(P.counter_program(), COUNTER, ids, rows)
    e.put_batch(ids[:500], np.frombuffer(b"".join(rows[:500]), np.uint8).reshape(500, -1)[::-1].copy(), present=[i % 3 != 0 for i in range(500)])
    n_exp, n_scan = check_all_reads(e, COUNTER, ids, values_cap=200)   # a few rows' bytes: pages end inside a tile
    assert n_exp > 5 and n_scan > 50
    e.close()
    # BankAccount: UUID, two strings, a Double at every edge
    ids = [str(uuid.UUID(bytes=rng.bytes(16))) for _ in range(4000)]
    e = make_engine(state_program(64, f64=(40,)), BANK, ids, [bank_row(rng, k) for k in range(len(ids))])
    check_all_reads(e, BANK, ids, values_cap=1000)
    e.close()
    # a 120-byte state with mixed members
    ids = ["m-%d" % i for i in range(2000)] + ODD_IDS
    e = make_engine(state_program(128, f64=(8, 104)), MIXED, ids, [mixed_row(rng, k) for k in range(len(ids))])
    check_all_reads(e, MIXED, ids, values_cap=4096)
    e.close()


def test_folded_table_and_rows_without_ids():
    counts = np.random.default_rng(2).integers(0, 20, size=5000)
    rec, off = SY.counter_csr(len(counts), counts, seed=9, p_throw=0.01)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_events(rec, off)
        e.fold()
        # no key table: every row lacks an id, which a writer without an ID member does not need
        e.set_state_writer(writer_of(COUNTER[1:]))
        got = [(i, v) for p in e.export_changes_values(CH_ERR, values_cap=1 << 20) for i, v in zip(p[0].tolist(), p[4])]
        assert got and all(v == S.write_value(COUNTER[1:], want[i, :8].tobytes(), None) for i, v in got if v is not None)
        e.set_state_writer(writer_of(COUNTER))
        first = next(i for i, v in got if v is not None)
        cur = N.sgr_changes_cursor()
        assert_refused(e, lambda: export_once(e, cur), rf"row \d+ of the page \(aggregate {first}\), member 0 \"aggregateId\": {re.escape(S.NO_ID)}")
        assert cur.next == 0 and cur.token == 0
        e.load_keys(["agg-%d" % g for g in range(len(counts))])
        pages = list(e.export_changes_values(CH_ERR, values_cap=333))
        for p in pages:
            for i, k, v in zip(p[0].tolist(), p[3], p[4]):
                assert v == (S.write_value(COUNTER, want[i, :8].tobytes(), k.encode()) if v is not None else None)
        assert sum(len(p[0]) for p in pages) == len(got)


def export_once(e, cur, cap=1 << 16):
    buf, voffs = np.zeros(cap, np.uint8), np.zeros(1025, np.uint64)
    fl, err, idx, offs, ids = (np.zeros(1024, t) for t in (np.uint32, np.uint32, np.int64, np.uint32, np.uint8))
    ids = np.zeros(1 << 16, np.uint8)
    n = C.c_uint64(7)
    rc = e._lib.sgr_export_changes_values(e._h, CH_ERR, C.byref(cur), 1024, buf.ctypes.data, cap, voffs.ctypes.data, fl.ctypes.data,
                                          err.ctypes.data, idx.ctypes.data, ids.ctypes.data, ids.size, offs.ctypes.data, C.byref(n))
    e._ck(rc)
    return int(n.value), buf, voffs


def assert_refused(e, call, pattern, code=N.SGR_ERR_UNSUPPORTED):
    with pytest.raises(SgrError) as ei:
        call()
    assert ei.value.code == code, str(ei.value)
    assert re.search(pattern, str(ei.value)), str(ei.value)


def test_refusals_capacity_and_writer_lifecycle():
    rng = np.random.default_rng(3)
    ids = ["b-%d" % i for i in range(300)]
    rows = [bank_row(rng, k) for k in range(len(ids))]
    rows[137] = bank_row(rng, 137, bal=float("nan"))
    rows[200] = bank_row(rng, 200, bal=-math.inf)
    e = make_engine(state_program(64, f64=(40,)), BANK, ids, rows)
    # get_batch_values: all or nothing, the lowest refused row named
    assert_refused(e, lambda: e.get_many_values(ids[100:]), rf"row 37 of the batch \(aggregate 137\), member 3 \"balance\": {re.escape(S.F64_NOT_FINITE)}")
    assert e.get_many_values(ids[:100]) == [S.write_value(BANK, rows[i], None) for i in range(100)]
    # ... and writes nothing: every output of a raw call keeps its sentinel
    blob, offs = np.frombuffer(b"b-136b-137b-138", np.uint8), np.array([0, 5, 10, 15], np.uint32)
    buf, voffs, fl, ix, need = np.full(4096, 0xAB, np.uint8), np.full(4, 77, np.uint64), np.full(3, 77, np.uint32), np.full(3, 77, np.int64), C.c_uint64(99)
    rc = e._lib.sgr_get_batch_values(e._h, blob.ctypes.data, offs.ctypes.data, 3, buf.ctypes.data, buf.size, voffs.ctypes.data, fl.ctypes.data,
                                     ix.ctypes.data, C.byref(need))
    assert rc == N.SGR_ERR_UNSUPPORTED
    assert (buf == 0xAB).all() and (voffs == 77).all() and (fl == 77).all() and (ix == 77).all() and need.value == 99
    # a page holding row 137 is refused and the cursor stays
    cur = N.sgr_changes_cursor()
    assert_refused(e, lambda: export_once(e, cur), r"row 137 of the page \(aggregate 137\), member 3")
    assert (cur.next, cur.token) == (0, 0)
    assert_refused(e, lambda: list(e.scan_values()), r"member 3 \"balance\"")
    # capacity: the bytes needed come back, nothing else
    need, voffs, fl = C.c_uint64(), np.full(4, 77, np.uint64), np.full(3, 77, np.uint32)
    blob, offs = np.frombuffer(b"b-0b-1b-2", np.uint8), np.array([0, 3, 6, 9], np.uint32)
    buf = np.zeros(10, np.uint8)
    rc = e._lib.sgr_get_batch_values(e._h, blob.ctypes.data, offs.ctypes.data, 3, buf.ctypes.data, 10, voffs.ctypes.data, fl.ctypes.data, None, C.byref(need))
    assert rc == N.SGR_ERR_CAPACITY and need.value == sum(len(S.write_value(BANK, rows[i], None)) for i in range(3))
    assert (voffs == 77).all() and (fl == 77).all() and not buf.any()
    # a first row whose value alone does not fit a page
    cur = N.sgr_changes_cursor()
    assert_refused(e, lambda: export_once(e, cur, cap=20), "does not fit", N.SGR_ERR_CAPACITY)
    assert (cur.next, cur.token) == (0, 0)
    # an overlong string and an ill-formed id
    bad = bytearray(rows[5])
    bad[16] = 16
    put_raw(e, [b"b-5", b"bad-\xff"], [bytes(bad), rows[6]])
    assert_refused(e, lambda: e.get_many_values(["b-5"]), rf"member 1 \"accountOwner\": {re.escape(S.PSTR_LENGTH)}")
    e.set_state_writer(writer_of([("id", S.ID)] + BANK[:1]))
    assert_refused(e, lambda: list(e.scan_values()), rf"member 0 \"id\": {re.escape(S.ID_UTF8)}")
    # bad tables change nothing; no writer, a cleared writer and a new program all leave reads with SGR_ERR_STATE
    for tbl in ([("x", S.F64, 60)], [("x", S.I32, 2)], [("", S.I32, 0)], [("a", S.I32, 0), ("a", S.I32, 4)], [("i", S.ID), ("j", S.ID)],
                [("p", S.PSTR, 0, 2)], [("k%d" % i, S.I32, 0) for i in range(33)], [("z", 9, 0)]):
        with pytest.raises(SgrError) as ei:
            e.set_state_writer(writer_of(tbl))
        assert ei.value.code == N.SGR_ERR_INVALID
    assert e.get_many_values(["b-0"]) == [S.write_value([("id", S.ID)] + BANK[:1], rows[0], b"b-0")]
    e.set_state_writer([])
    assert_refused(e, lambda: e.get_many_values(["b-0"]), "no state writer", N.SGR_ERR_STATE)
    e.set_state_writer(writer_of(BANK))
    e.register_program(state_program(64, f64=(40,)))
    e.put_batch(["b-0"], np.frombuffer(rows[0], np.uint8).reshape(1, -1))
    assert_refused(e, lambda: e.get_many_values(["b-0"]), "no state writer", N.SGR_ERR_STATE)
    assert_refused(e, lambda: list(e.export_changes_values()), "no state writer", N.SGR_ERR_STATE)
    e.close()


def test_exported_values_restore_to_the_same_table():
    rng = np.random.default_rng(4)
    for prog, members, make_row, n in ((P.counter_program(), COUNTER, None, 3000), (state_program(64, f64=(40,)), BANK, bank_row, 3000),
                                       (state_program(128, f64=(8, 104)), MIXED, mixed_row, 1500)):
        ids = ["r-%d" % i for i in range(n)] + [k for k in ODD_IDS if k]   # (an empty key is a flush marker to a state topic)
        rows = [make_row(rng, k) if make_row else rng.bytes(8) for k in range(len(ids))]
        e = make_engine(prog, members, ids, rows)
        recs = [(k.encode(), v) for p in e.export_changes_values(CH_ERR, values_cap=1 << 16) for k, v in zip(p[3], p[4])]
        assert len(recs) == len(ids) and all(v is not None for _, v in recs)
        restore = [(m[0], m[1], m[2], m[3]) if len(m) > 3 else (m[0], m[1], m[2]) for m in members if m[1] != S.ID]
        with ReplayEngine(0) as f:
            f.register_program(prog)
            with DeviceIngest(f, 1 << 16) as dg:
                dg.set_state_topic(True)
                dg.set_json_packer("", [("State", 0, restore)])
                dg.set_value_framing(N.VALUE_JSON)
                for b in range(0, len(recs), 500):
                    chunk = [(j, k, v) for j, (k, v) in enumerate(recs[b:b + 500])]
                    dg.submit(0, K.encode_record_batch(b, chunk, compression="lz4"))
                dg.fold()
            got, gfl, _ = f.get_many(ids, arrays=True)
        want, wfl, _ = e.get_many(ids, arrays=True)
        assert ((gfl & N.ST_EXISTS) == (wfl & N.ST_EXISTS)).all()
        for i in range(len(ids)):
            assert S.same_row(members, want[i].tobytes(), got[i].tobytes()), (ids[i], want[i], got[i])
        e.close()


def test_device_double_digits_equal_repr_on_two_million_rows():
    rng = np.random.default_rng(5)
    corpus = [float(t) for t in VC.f64_corpus(rng)]
    corpus = [x for x in corpus if math.isfinite(x)]
    rnd = np.frombuffer(rng.bytes(8 * (2_000_000 - len(corpus))), "<f8")
    xs = np.concatenate([np.array(corpus, "<f8"), np.where(np.isfinite(rnd), rnd, 1.0)])
    n = len(xs)
    ids = ["d%d" % i for i in range(n)]
    with ReplayEngine(0) as e:
        e.register_program(state_program(16, f64=(0,)))
        e.put_batch(ids, xs.view(np.uint8).reshape(n, 8))
        e.set_state_writer([("x", N.JSON_F64, 0)])
        got = e.get_many_values(ids)
    bad = [(i, got[i]) for i in range(n) if got[i] != b'{"x":' + S.format_f64(float(xs[i])) + b"}"]
    assert not bad, bad[:5]


def test_jvm_state_values_when_pinned():
    path = os.path.join(ROOT, "tests", "golden", "jvm_vectors.json")
    if not os.path.exists(path):
        pytest.skip("PARITY UNPINNED: tests/golden/jvm_vectors.json (GenVectors.scala on a JVM) is absent")
    import json

    doc = json.load(open(path))
    if "stateValues" not in doc:
        pytest.skip("PARITY UNPINNED: jvm_vectors.json has no stateValues section")
    for case in doc["stateValues"]:
        members = [tuple(m) for m in case["members"]]
        row, agg_id = bytes.fromhex(case["row"]), case.get("id")
        want = case["value"]
        try:
            got = S.write_value(members, row, None if agg_id is None else agg_id.encode()).decode()
        except S.Refused:
            got = "throws"
        assert got == want, case


def _counter_json(key, b):
    """the Python codec of the Counter state: play-json's Json.toJson(State(aggregateId, count, version))"""
    import json

    count, version = struct.unpack_from("<ii", b)
    return json.dumps({"aggregateId": key, "count": count, "version": version}, separators=(",", ":"), ensure_ascii=False).encode()


def _counter_packed(key, v):
    import json

    o = json.loads(v)
    return struct.pack("<ii", o["count"], o["version"])


def test_store_with_a_writer_table_serves_json_values():
    from surge_b200.store import GpuReplayKeyValueStore, StateCodec

    # Counter: the store with the device writer answers as the same store with the Python codec
    ids = ['q"uote', "back\\slash", "zoë", "日本", "😀", "plain"] + ["c-%d" % i for i in range(500)]
    rng = np.random.default_rng(6)
    stores, calls = [], []
    for codec in (StateCodec(_counter_packed, _counter_json), StateCodec(_counter_packed, writer=writer_of(COUNTER))):
        got = []
        st = GpuReplayKeyValueStore("s", P.counter_program(), codec=codec, on_changes=lambda ch, fa, got=got: got.append((sorted(ch), fa)))
        st.init()
        stores.append(st)
        calls.append(got)
    for rnd in range(3):
        batch = [(k, _counter_json(k, struct.pack("<ii", int(rng.integers(-9, 9)), rnd)) if rng.random() < 0.8 else None)
                 for k in rng.choice(ids, 300, replace=False).tolist()]
        for st in stores:
            st.putAll(batch)
        # read-your-writes before the flush, from the unflushed puts
        put_ids = [k for k, _ in batch]
        assert stores[0].get_many(put_ids) == stores[1].get_many(put_ids) == [v for _, v in batch]
        for st in stores:
            st.flush()
        a, b = stores
        assert [a.get(k) for k in ids[:40]] == [b.get(k) for k in ids[:40]]
        assert a.get_many(ids + ["never"]) == b.get_many(ids + ["never"])
        assert list(a.all()) == list(b.all())
        assert list(a.range("c-1", "c-3")) == list(b.range("c-1", "c-3"))
        assert calls[0][-1] == calls[1][-1] and calls[0][-1][0]
    for st in stores:
        st.close()
    # BankAccount: the device writer against the restatement (no Python codec at all)
    ids = [str(uuid.UUID(bytes=rng.bytes(16))) for _ in range(400)]
    rows = {k: bank_row(rng, i)[:56] for i, k in enumerate(ids)}
    got = []
    st = GpuReplayKeyValueStore("b", state_program(64, f64=(40,)), codec=StateCodec(lambda k, v: rows[k], writer=writer_of(BANK)),
                                on_changes=lambda ch, fa: got.append(sorted(ch)))
    st.init()
    st.putAll([(k, b"(any serialized state)") for k in ids])
    st.flush()
    want = {k: S.write_value(BANK, rows[k], None) for k in ids}
    assert st.get_many(ids) == [want[k] for k in ids]
    assert st.get(ids[7]) == want[ids[7]]
    assert list(st.all()) == sorted(want.items(), key=lambda kv: kv[0].encode())
    lo, hi = sorted(ids)[100], sorted(ids)[200]
    assert list(st.range(lo, hi)) == [(k, want[k]) for k in sorted(ids) if lo <= k <= hi]
    assert got == [sorted(want.items())]
    st.delete(ids[0])
    assert st.get(ids[0]) is None                       # read-your-writes of a delete
    st.flush()
    assert st.get(ids[0]) is None and got[-1] == [(ids[0], None)]
    st.close()
