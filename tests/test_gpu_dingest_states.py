"""-m gpu: compacted state topics decoded on the device and applied last write wins (sgr_dingest_set_state_topic).

Every comparison is by id: the device dictionary numbers ids in no promised order, the restatement (oracle/state_topic.py, then
oracle/put_batch.py) in first-appearance order. Per id: the row, its flags and err_idx; then the key table as a set, the
partitions' positions and the poll statistics."""
import ctypes as C
import json
import os
import re
import struct
import subprocess
import threading
import time
import uuid

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import state_topic as S
from oracle import value_corpus as VC
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.engine import ReplayEngine
from surge_b200.ingest import Ingest, IngestError
from surge_b200.native import SgrError
from surge_b200.store import GpuReplayKeyValueStore, StateCodec

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH_ERR = N.ST_CHANGED | N.ST_ERROR
STAT_KEYS = ("n_records", "n_markers", "n_null_values", "n_duplicates", "n_control_batches", "n_aborted_batches", "n_aborted_records")
SPECIAL_F64 = [0.0, -0.0, float("nan"), 1.5, -2.25]


def state_program(sb, kind=N.REC_FIXED64, f64=()):
    """any program will do: a state topic only writes rows"""
    return P.make_program(sb, kind, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])], f64_fields=list(f64))


# name -> (program, Double offsets)
PROGRAMS = {
    "counter": (P.counter_program, ()),
    "bank_account": (lambda: state_program(64, f64=(16,)), (16,)),
    "state128": (lambda: state_program(128, f64=(0, 112)), (0, 112)),
    "var16": (lambda: state_program(96, N.REC_VAR16, (8,)), (8,)),
}


def flags_of(table):
    sb = table.shape[1]
    return table[:, sb - 8:sb - 4].copy().view("<u4").ravel()


def total_stats(dg):
    st = N.sgr_ingest_stats()
    assert dg._lib.sgr_dingest_get_stats(dg._h, C.byref(st)) == N.SGR_OK
    return {n: int(getattr(st, n)) for n, _ in N.sgr_ingest_stats._fields_ if n != "reserved"}


class Restore:
    """A device engine restoring a state topic, and the restatement of the same fetches next to it."""

    def __init__(self, prog, f64=(), framing=N.VALUE_PACKED, packer=None, max_keys=1 << 16):
        self.e = ReplayEngine(0)
        self.e.register_program(prog)
        self.sb = self.e.state_bytes
        self.f64 = f64
        self.dg = DeviceIngest(self.e, max_keys)
        self.dg.set_state_topic(True)
        if packer is not None:
            self.dg.set_json_packer(*packer)
        self.dg.set_value_framing(framing)
        self.framing = S.PROTOBUF if framing == N.VALUE_PROTOBUF_EVENT else S.PACKED
        self.fetches, self.n_recs = [], 0
        self.ids, self.table = [], np.zeros((0, self.sb), np.uint8)
        self.parts, self.new_keys = set(), 0
        self.prev_stats = dict.fromkeys(STAT_KEYS, 0)

    def close(self):
        self.dg.close()
        self.e.close()

    def poll(self, fetches, check=True):
        for p, data, aborted in fetches:
            self.dg.set_aborted(p, aborted)
            self.dg.submit(p, data)
            self.parts.add(p)
        got = self.dg.fold()
        self.new_keys += got["n_new_keys"]
        self.fetches += fetches
        recs, self.nxt, st = S.read_committed_states(self.fetches, self.framing, self.sb - 8)
        new, self.n_recs = recs[self.n_recs:], len(recs)
        self.ids, self.table = S.apply(self.ids, self.table, new, self.f64)
        assert {k: got[k] for k in STAT_KEYS} == {k: st[k] - self.prev_stats[k] for k in STAT_KEYS}
        self.prev_stats = st
        if check:
            self.check()
        return got

    def check(self):
        user = self.sb - 8
        states, fl, idx = self.e.get_many(self.ids, arrays=True)
        assert (idx >= 0).all() and len(set(idx.tolist())) == len(self.ids) == self.new_keys   # the key table, as a set
        want_fl = flags_of(self.table)
        assert np.array_equal(states, self.table[:, :user])
        assert fl.tolist() == want_fl.tolist()
        changes = {}
        for _, f, err, rows, kids in self.e.export_changes(CH_ERR, page_rows=97):
            for i, k in enumerate(kids):
                changes[k] = (int(f[i]), int(err[i]), rows[i].tobytes())
        want = {k: (int(want_fl[i]), 0, self.table[i, :user].tobytes()) for i, k in enumerate(self.ids) if want_fl[i] & CH_ERR}
        assert changes == want
        live = sorted(k for i, k in enumerate(self.ids) if want_fl[i] & N.ST_EXISTS)
        assert sorted(k for pg in self.e.scan(page_rows=53) for k in pg[3]) == live
        assert {p: self.dg.offsets(p) for p in self.parts} == {p: (self.nxt.get(p, 0), self.nxt.get(p, 0)) for p in self.parts}


# ------------------------------------------------------------------ 1, 2: random fetches against the restatement
KEYS = ["id-%d" % i for i in range(30)] + ["acct:%d" % i for i in range(8)] + ["zoë-%d" % i for i in range(6)] + ["日本:%d:x" % i for i in range(4)]


def random_polls(rng, n_polls, n_parts, user, f64, framing):
    """polls of fetches with lz4 and plain batches, flush markers, refetched batches, aborted transactions with their control
    batches, tombstones of known and unknown ids, ids with ':' and non-ASCII bytes, values of every length up to the row"""
    nxt = {p: 0 for p in range(n_parts)}
    sent = {p: [] for p in range(n_parts)}
    polls = []
    for _ in range(n_polls):
        poll = []
        for _ in range(int(rng.integers(3, 9))):
            p = int(rng.integers(0, n_parts))
            roll = rng.random()
            if roll < 0.12 and sent[p]:
                poll.append((p, sent[p][int(rng.integers(0, len(sent[p])))], []))
                continue
            recs = []
            for d in range(int(rng.integers(1, 40))):
                r = rng.random()
                if r < 0.05:
                    recs.append((d, b"", b""))
                    continue
                key = (KEYS[int(rng.integers(0, len(KEYS)))] if r < 0.9 else "ghost-%d" % int(rng.integers(0, 1 << 30))).encode()
                if r < 0.2 or key.startswith(b"ghost"):
                    recs.append((d, key, None))
                    continue
                b = bytearray(rng.integers(0, 3, size=user, dtype=np.uint8).tobytes())   # few values: equal rewrites are common
                for off in f64:
                    b[off:off + 8] = struct.pack("<d", SPECIAL_F64[int(rng.integers(0, len(SPECIAL_F64)))])
                v = bytes(b[:int(rng.integers(0, user + 1))] if rng.random() < 0.3 else b)
                recs.append((d, key, S.encode_state(key, v) if framing == N.VALUE_PROTOBUF_EVENT else v))
            comp = "lz4" if rng.random() < 0.5 else "none"
            if roll < 0.25:
                pid = int(rng.integers(1, 1 << 40))
                data = K.encode_record_batch(nxt[p], recs, compression=comp, producer_id=pid, producer_epoch=0, transactional=True)
                poll.append((p, data + K.encode_control_batch(nxt[p] + len(recs), pid, K.ABORT), [(pid, nxt[p])]))
                nxt[p] += len(recs) + 1
                continue
            data = K.encode_record_batch(nxt[p], recs, compression=comp)
            sent[p].append(data)
            nxt[p] += len(recs)
            poll.append((p, data, []))
        polls.append(poll)
    return polls


@pytest.mark.parametrize("framing", [N.VALUE_PACKED, N.VALUE_PROTOBUF_EVENT], ids=["packed", "protobuf"])
@pytest.mark.parametrize("name", list(PROGRAMS))
def test_random_polls_against_the_restatement(name, framing):
    mk, f64 = PROGRAMS[name]
    rng = np.random.default_rng([len(name), framing])
    r = Restore(mk(), f64, framing)
    try:
        for poll in random_polls(rng, 6, 3, r.sb - 8, f64, framing):
            r.poll(poll)          # every poll checked: CHANGED against the state before it, untouched rows lose their flags
        a_poll_of_holes = [(0, K.encode_record_batch(r.nxt.get(0, 0), [(0, b"", b"")]), [])]
        before = r.e.export_states()
        r.poll(a_poll_of_holes)   # nothing live: nothing applied, the last fold's flags stay; the position advances
        assert np.array_equal(r.e.export_states(), before)
    finally:
        r.close()


def test_bank_account_changed_rule_for_doubles():
    r = Restore(PROGRAMS["bank_account"][0](), (16,))
    d = lambda x, tail=b"\7": b"\1" * 16 + struct.pack("<d", x) + tail * 32   # noqa: E731
    try:
        r.poll([(0, K.encode_record_batch(0, [(0, b"nan", d(float("nan"))), (1, b"zero", d(0.0)), (2, b"same", d(1.0))]), [])])
        r.poll([(0, K.encode_record_batch(3, [(0, b"nan", d(float("nan"))), (1, b"zero", d(-0.0)), (2, b"same", None), (3, b"same", d(1.0))]), [])])
        states, fl, _ = r.e.get_many(["nan", "zero", "same"], arrays=True)
        assert fl.tolist() == [N.ST_EXISTS | N.ST_CHANGED, N.ST_EXISTS, N.ST_EXISTS]
        assert states[1, 16:24].tobytes() == struct.pack("<d", -0.0)
    finally:
        r.close()


# ------------------------------------------------------------------ 3: against the snapshot-event route
def test_json_counter_state_topic_against_the_snapshot_route():
    rng = np.random.default_rng(3)
    ev, st = ReplayEngine(0), ReplayEngine(0)
    try:
        ev.register_program(P.counter_snapshot_restore_program())
        st.register_program(P.counter_program())
        with DeviceIngest(ev, 1 << 12) as de, DeviceIngest(st, 1 << 12) as ds:
            de.set_json_packer("", [("State", 0, [("count", N.JSON_I32, 16), ("version", N.JSON_I32, 20)])])
            de.set_value_framing(N.VALUE_JSON)
            de.set_null_value_type(1)
            ds.set_state_topic(True)
            ds.set_json_packer("", [("State", 0, [("count", N.JSON_I32, 0), ("version", N.JSON_I32, 4)])])
            ds.set_value_framing(N.VALUE_JSON)
            off, ids = 0, ["agg-%d" % i for i in range(200)]
            for _ in range(5):
                recs = []
                for d in range(700):
                    k = ids[int(rng.integers(0, len(ids)))]
                    if rng.random() < 0.15:
                        recs.append((d, k.encode(), None))
                    else:
                        obj = {"aggregateId": k, "count": int(rng.integers(-3, 3)), "version": int(rng.integers(0, 3))}
                        recs.append((d, k.encode(), json.dumps(obj, separators=(",", ":")).encode()))
                data = K.encode_record_batch(off, recs, compression="lz4")
                off += len(recs)
                for g in (de, ds):
                    g.submit(0, data)
                a, b = de.fold(), ds.fold()
                assert {k: a[k] for k in STAT_KEYS} == {k: b[k] for k in STAT_KEYS}
                sa, fa, ia = ev.get_many(ids, arrays=True)
                sb_, fb, ib = st.get_many(ids, arrays=True)
                assert np.array_equal(sa, sb_) and fa.tolist() == fb.tolist()
                assert de.offsets(0) == ds.offsets(0)
    finally:
        ev.close()
        st.close()


# ------------------------------------------------------------------ 4: the JSON state layout against the host decoder
COUNTER_STATE = [("sequenceNumber", N.JSON_I32, 0), ("incrementBy", N.JSON_I32, 4)]
BANK_STATE = [("accountNumber", N.JSON_UUID, 0), ("balance", N.JSON_F64, 16), ("accountOwner", N.JSON_PSTR, 24, 16), ("securityCode", N.JSON_PSTR, 40, 8)]


def _events_layout(members):
    return [(m[0], m[1], m[2] + 16) + tuple(m[3:]) for m in members]


def _why(msg):
    return re.sub(r"^[A-Z_]+: (partition -?\d+ )?offset -?\d+(, record \d+)?: ", "", msg)


@pytest.mark.parametrize("corpus", ["counter", "bank_account"])
def test_json_state_layout_against_the_host_decoder(corpus):
    rng = np.random.default_rng(20261016)
    values = VC.counter_values(rng) if corpus == "counter" else VC.bank_values(rng)
    # (the corpus writes some balances as the repr of a NumPy scalar, "np.float64(1.5)", which every decoder refuses: the same
    # values with the plain number are added, so that BankAccount states are accepted too)
    values += [re.sub(rb"np\.float64\(([^)]*)\)", rb"\1", v) for v in values if b"np.float64(" in v]
    members = COUNTER_STATE if corpus == "counter" else BANK_STATE
    host_packer = ("", [("State", 0, _events_layout(members))])
    accepted, host_rows, host_why = [], {}, {}
    for i, v in enumerate(values):
        ing = Ingest()
        try:
            ing.set_json_packer(*host_packer)
            ing.set_value_framing(N.VALUE_JSON)
            try:
                ing.record_batches(0, K.encode_record_batch(0, [(0, b"v%d" % i, v)]))
                host_rows[i] = ing.pending()[0, 16:64].tobytes()
                accepted.append(i)
            except IngestError as ex:
                host_why[i] = _why(str(ex))
        finally:
            ing.close()
    assert accepted and host_why
    r = Restore(state_program(64), (), N.VALUE_JSON, ("", [("State", 0, members)]))
    try:
        recs = [(d, b"v%d" % i, values[i]) for d, i in enumerate(accepted)]
        off = 0
        for s in range(0, len(recs), 300):
            chunk = [(d - s, k, v) for d, k, v in recs[s:s + 300]]
            r.dg.submit(0, K.encode_record_batch(off, chunk, compression="lz4" if s % 600 else "none"))
            off += len(chunk)
        r.dg.fold()
        states, fl, idx = r.e.get_many(["v%d" % i for i in accepted], arrays=True)
        assert (idx >= 0).all() and (fl == N.ST_EXISTS | N.ST_CHANGED).all()
        for j, i in enumerate(accepted):
            assert states[j, :48].tobytes() == host_rows[i], values[i]
        for i, why in host_why.items():
            table, before = r.e.export_states(), total_stats(r.dg)
            data = K.encode_record_batch(off, [(0, b"good", None), (1, b"bad", values[i])])
            with pytest.raises(IngestError) as ei:
                r.dg.submit(0, data)
                r.dg.fold()
            assert ei.value.code == N.SGR_ERR_INVALID
            assert re.match(r"^[A-Z_]+: offset %d, record 1: " % off, str(ei.value)), str(ei.value)
            assert _why(str(ei.value)) == why
            assert np.array_equal(r.e.export_states(), table) and total_stats(r.dg) == before and r.dg.offsets(0) == (off, off)
    finally:
        r.close()


def test_json_members_past_the_first_48_program_bytes():
    rng = np.random.default_rng(48)
    members = [("big", N.JSON_I64, 48), ("dbl", N.JSON_F64, 56), ("small", N.JSON_I32, 64), ("id", N.JSON_UUID, 68), ("name", N.JSON_PSTR, 84, 36)]
    r = Restore(state_program(128), (), N.VALUE_JSON, ("", [("S", 0, members)]))
    try:
        want, recs = {}, []
        for d in range(400):
            big, small = int(rng.integers(-2**63, 2**63)), int(rng.integers(-2**31, 2**31))
            dbl = float(np.frombuffer(rng.bytes(8), "<f8")[0])
            if not np.isfinite(dbl):
                dbl = 0.25
            u = uuid.UUID(bytes=rng.bytes(16))
            name = "".join(rng.choice(list("abcé日😀"), int(rng.integers(0, 8))))
            obj = {"name": name, "big": big, "dbl": dbl, "small": small, "id": str(u), "other": [1, {"x": "y"}]}
            recs.append((d, b"s%d" % d, json.dumps(obj, ensure_ascii=bool(d % 2)).encode()))
            nb = name.encode()
            row = bytearray(120)
            row[48:68] = struct.pack("<qdi", big, dbl, small)
            row[68:84] = u.bytes
            row[84] = len(nb)
            row[85:85 + len(nb)] = nb
            want["s%d" % d] = bytes(row)
        r.dg.submit(0, K.encode_record_batch(0, recs, compression="lz4"))
        r.dg.fold()
        keys = list(want)
        states, fl, _ = r.e.get_many(keys, arrays=True)
        for j, k in enumerate(keys):
            assert states[j].tobytes() == want[k], k
    finally:
        r.close()


# ------------------------------------------------------------------ 5: refusals
def test_a_value_longer_than_the_row_is_refused_and_applies_nothing():
    r = Restore(P.counter_program())
    try:
        r.poll([(0, K.encode_record_batch(0, [(0, b"a", b"\1" * 8)]), [])])
        table, before = r.e.export_states(), total_stats(r.dg)
        with pytest.raises(IngestError) as ei:
            r.dg.submit(0, K.encode_record_batch(1, [(0, b"b", b"\2" * 8), (1, b"c", b"\3" * 9)], compression="lz4"))
            r.dg.fold()
        assert ei.value.code == N.SGR_ERR_INVALID
        assert "offset 1, record 1: state value of 9 bytes is longer than the 8 program bytes of a row" in str(ei.value)
        assert np.array_equal(r.e.export_states(), table) and total_stats(r.dg) == before and r.dg.offsets(0) == (1, 1)
    finally:
        r.close()


def test_a_full_dictionary_is_a_capacity_error():
    r = Restore(P.counter_program(), max_keys=4)
    try:
        with pytest.raises(IngestError) as ei:
            r.dg.submit(0, K.encode_record_batch(0, [(d, b"k%d" % d, b"\1" * 8) for d in range(5)]))
            r.dg.fold()
        assert ei.value.code == N.SGR_ERR_CAPACITY
    finally:
        r.close()


def test_when_the_mode_can_be_set_and_state_member_tables():
    with ReplayEngine(0) as e:
        e.register_program(state_program(32))
        with DeviceIngest(e, 1 << 10) as dg:
            dg.submit(0, K.encode_record_batch(0, [(0, b"a", b"\0" * 8)]))
            with pytest.raises(IngestError) as ei:
                dg.set_state_topic(True)                       # a poll is pending
            assert ei.value.code == N.SGR_ERR_STATE
            dg.fold()
            with pytest.raises(IngestError) as ei:
                dg.set_state_topic(True)                       # a poll was folded: the dictionary belongs to the events topic
            assert ei.value.code == N.SGR_ERR_STATE
            dg.reset()
            dg.set_state_topic(True)
            for bad in (("_type", [("S", 0, [("x", N.JSON_I32, 0)])]),                          # a discriminator
                        ("", [("S", 0, [("x", N.JSON_I32, 0)]), ("T", 1, [("y", N.JSON_I32, 4)])]),   # two classes
                        ("", [("S", 0, [("x", N.JSON_I64, 20)])]),                          # past state_bytes - 8 = 24
                        ("", [("S", 0, [("x", N.JSON_I32, 2)])])):                          # not on a 4-byte boundary
                with pytest.raises(IngestError) as ei:
                    dg.set_json_packer(*bad)
                assert ei.value.code == N.SGR_ERR_INVALID
            dg.set_json_packer("", [("S", 0, [("x", N.JSON_I64, 16)])])
            with pytest.raises(IngestError) as ei:
                dg.set_state_topic(False)                      # a member table is registered
            assert ei.value.code == N.SGR_ERR_STATE


# ------------------------------------------------------------------ 6: scale
def test_scale_four_million_records_over_two_million_uuids(tmp_path):
    import torch

    t0 = time.perf_counter()
    lib_path = str(tmp_path / "libkv.so")
    subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-o", lib_path, os.path.join(ROOT, "scripts", "kafka_values_encode.c")])
    kv = C.CDLL(lib_path)
    kv.kv_kafka_encode_values_nulls.restype = C.c_int64
    kv.kv_kafka_encode_values_nulls.argtypes = [C.c_void_p] * 5 + [C.c_uint64, C.c_uint32, C.c_int, C.c_int64, C.c_void_p, C.c_uint64]
    rng = np.random.default_rng(66)
    n_ids, n, n_parts = 2 << 20, 4 << 20, 8
    pool = np.array([str(uuid.UUID(bytes=rng.bytes(16))).encode() for _ in range(n_ids)], dtype="S36")
    pick = np.concatenate([rng.permutation(n_ids), rng.integers(0, n_ids, size=n - n_ids)])[rng.permutation(n)]
    part = rng.integers(0, n_parts, size=n)
    rows = rng.integers(0, 4, size=(n, 8), dtype=np.uint8)
    nulls = (rng.random(n) < 0.10).astype(np.uint8)
    fetches, order = [], []
    for p in range(n_parts):
        sel = np.nonzero(part == p)[0]
        order.append(sel)
        keys = np.frombuffer(pool[pick[sel]].tobytes(), np.uint8)
        vals = np.ascontiguousarray(rows[sel]).reshape(-1)
        m = len(sel)
        koff, voff = np.arange(m + 1, dtype=np.uint64) * 36, np.arange(m + 1, dtype=np.uint64) * 8
        nl = np.ascontiguousarray(nulls[sel])
        cap = int(m * (36 + 8 + 32) + 160 * (m // 512 + 1))
        cap += cap // 255 + 1024
        out = np.empty(cap, np.uint8)
        got = kv.kv_kafka_encode_values_nulls(keys.ctypes.data, koff.ctypes.data, vals.ctypes.data, voff.ctypes.data, nl.ctypes.data, m, 512, 1, 0,
                                              out.ctypes.data, cap)
        assert got > 0
        fetches.append(torch.from_numpy(out[:got].copy()).pin_memory())
    arrival = np.concatenate(order)   # submission order: partition 0's records, then partition 1's, ...
    with ReplayEngine(0) as dev, ReplayEngine(0) as ref:
        dev.register_program(P.counter_program())
        ref.register_program(P.counter_program())
        with DeviceIngest(dev, n_ids + 1024, 64 * (n_ids + 1024)) as dg:
            dg.set_state_topic(True)
            low = [torch.cuda.mem_get_info(0)[0]]
            stop = threading.Event()

            def sample():
                while not stop.is_set():
                    low[0] = min(low[0], torch.cuda.mem_get_info(0)[0])
                    time.sleep(0.0005)

            th = threading.Thread(target=sample)
            th.start()
            try:
                t1 = time.perf_counter()
                for p in range(n_parts):
                    dg.submit(p, fetches[p])
                st = dg.fold()
                t_fold = time.perf_counter() - t1
            finally:
                stop.set()
                th.join()
            assert st["n_records"] == n and st["n_null_values"] == int(nulls.sum()) and st["n_new_keys"] == n_ids
            assert all(dg.offsets(p) == (int((part == p).sum()),) * 2 for p in range(n_parts))
            timing = dg.last_timing()
        ids = [k.decode() for k in pool[pick[arrival]]]
        ref.put_batch(ids, rows[arrival], nulls[arrival] == 0)
        all_ids = [k.decode() for k in pool]
        sd, fd, idd = dev.get_many(all_ids, arrays=True)
        sr, fr, _ = ref.get_many(all_ids, arrays=True)
        assert (idd >= 0).all() and len(np.unique(idd)) == n_ids
        assert np.array_equal(sd, sr) and np.array_equal(fd, fr)
        total = torch.cuda.mem_get_info(0)[1]
        print(f"\nstate-topic scale on {torch.cuda.get_device_name(0)}: {n} records / {n_ids} UUID ids in {n_parts} partitions of lz4 "
              f"batches of 512, 10 % tombstones: fold {t_fold:.2f} s (submits + fold, host clock), last_timing {timing}; "
              f"{time.perf_counter() - t0:.1f} s in all; device bytes in use at the peak (whole device) {total - low[0]}")


# ------------------------------------------------------------------ 7: the store
def _store(prog, calls, **kw):
    st = GpuReplayKeyValueStore("s", prog, codec=StateCodec(lambda k, v: v, lambda k, b: b), on_changes=lambda c, f: calls.append((sorted(c), f)), **kw)
    st.init()
    return st


def test_state_topic_store_restores_record_batches_like_puts():
    rng = np.random.default_rng(7)
    prog = state_program(48, f64=(8,))
    polls = random_polls(rng, 4, 2, 40, (8,), N.VALUE_PACKED)
    a_calls, b_calls = [], []
    a, b = _store(prog, a_calls), _store(prog, b_calls)
    try:
        fetched, done = [], 0
        for poll in polls:
            for p, data, aborted in poll:
                a.restore_record_batches(p, data, aborted)
            a.flush()
            fetched += poll
            recs, nxt, _ = S.read_committed_states(fetched)
            for k, v in recs[done:]:          # the same records, restated, through put() / delete()
                b.put(k.decode(), v)
            done = len(recs)
            b.flush()
            assert a_calls[-1] == b_calls[-1]
            assert a.committed_offsets(range(2)) == {p: nxt.get(p, 0) for p in range(2)}
            keys = sorted({k.decode() for k, _ in recs}) + ["nobody"]
            assert [a.get(k) for k in keys] == [b.get(k) for k in keys]
            assert a.get_many(keys) == b.get_many(keys)
            assert list(a.all()) == list(b.all())
        with pytest.raises(SgrError):
            a.put("x", b"\1")                      # fed by record batches: not by put()
        with pytest.raises(SgrError):
            b.restore_record_batches(0, polls[0][0][1])   # fed by put(): not by record batches
    finally:
        a.close()
        b.close()


def test_state_topic_store_max_ids_fails_the_flush():
    calls = []
    st = _store(P.counter_program(), calls, max_ids=3)
    try:
        st.restore_record_batches(0, K.encode_record_batch(0, [(d, b"k%d" % d, b"\1" * 8) for d in range(4)]))
        with pytest.raises(SgrError) as ei:
            st.flush()
        assert ei.value.code == N.SGR_ERR_CAPACITY and calls == []
        assert st.committed_offsets([0]) == {0: 0}
    finally:
        st.close()
