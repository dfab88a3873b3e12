"""-m gpu: the device ingest (csrc/dingest.cu) for fold programs outside the sort-free class. Their polls are grouped on the
device with the dropped records (holes) left out (csrc/group_kernels.cu in hole mode) and folded with prior states. Every case
feeds the same bytes to the device ingest and to the host decoder (csrc/ingest.cpp + sgr_fold_ingested) and compares, per
aggregate id, the whole state row (flags and err_idx included), the ids, the offsets, the poll statistics and the pages of
export_changes; random programs are also checked against the compiled program oracle."""
import struct

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import oracle as O
from oracle import program_corpus as PC
from oracle import program_interp as I
from surge_b200 import ReplayEngine
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest, IngestError

pytestmark = pytest.mark.gpu


def _ev(etype, seq, payload=b""):
    return struct.pack("<II", etype, seq) + payload


def _bank_created(seq, uuid, balance, owner, code):
    return _ev(0, seq, uuid.ljust(16, b"\0")[:16] + struct.pack("<d", balance) + owner.ljust(16, b"\0")[:16] + struct.pack("<q", code))


def _bank_updated(seq, balance):
    return _ev(1, seq, bytes(16) + struct.pack("<d", balance))


def _add(total, st):
    for k, v in st.items():
        total[k] = total.get(k, 0) + v
    return total


def _rows_by_id(e, keys, dev=False):
    """{id: whole state row (user bytes, flags, err_idx)} for the ids `keys`, read from the table the engine exports."""
    table = e.export_states()
    if dev:
        _, _, idx = e.get_many(keys, arrays=True)
        assert (idx >= 0).all(), "an id of the host dictionary is missing on the device"
        assert len(set(idx.tolist())) == len(keys)
        other = np.ones(len(table), bool)
        other[idx] = False
        assert not table[other].any(), "a table row without an id is not empty"
    else:
        idx = np.arange(len(keys))
    return {k: table[i].tobytes() for k, i in zip(keys, idx)}


def _changes(e):
    out = {}
    for idx, flags, err, rows, ids in e.export_changes(N.ST_CHANGED | N.ST_ERROR, page_rows=97):
        for i in range(len(ids)):
            assert ids[i] is not None
            out[ids[i]] = (int(flags[i]), int(err[i]), rows[i].tobytes())
    return out


class _Pair:
    """One device ingest and one host ingest with the same program, polled with the same bytes."""

    def __init__(self, prog, null_type=None, max_keys=1 << 16, rules=None, state_bytes=None, f64=()):
        self.dev, self.host = ReplayEngine(0), ReplayEngine(0)
        self.dev.register_program(prog)
        self.host.register_program(prog)
        self.dg = DeviceIngest(self.dev, max_keys)
        self.ing = Ingest()
        if null_type is not None:
            self.dg.set_null_value_type(null_type)
            self.ing.set_null_value_type(null_type)
        self.rules, self.state_bytes, self.f64 = rules, state_bytes, list(f64)
        self.parts = set()
        self.polls = 0

    def close(self):
        self.dg.close()
        self.ing.close()
        self.dev.close()
        self.host.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def poll(self, fetches, aborted=None, skip_stats=()):
        """One poll of fetches [(partition, bytes)] through both ingests; aborted: {partition: [(producer id, first offset)]}."""
        aborted = aborted or {}
        for p, a in aborted.items():
            self.dg.set_aborted(p, a)
            self.ing.set_aborted(p, a)
        host_st = {}
        for p, d in fetches:
            self.dg.submit(p, d)
            _add(host_st, self.ing.record_batches(p, d))
            self.parts.add(p)
        prior = None
        if self.rules is not None and self.polls:
            prior = self.host.export_states()
        recs = self.ing.pending()
        dev_st = self.dg.fold()
        self.host.fold_ingested(self.ing)
        self.polls += 1
        drop = {"n_trailing_bytes", *skip_stats}
        assert {k: v for k, v in dev_st.items() if k not in drop} == {k: v for k, v in host_st.items() if k not in drop}
        self.check()
        if self.rules is not None:
            self.check_oracle(recs, prior)
        return dev_st

    def keys(self):
        return self.ing.keys()

    def check(self):
        keys = self.keys()
        assert _rows_by_id(self.dev, keys, dev=True) == _rows_by_id(self.host, keys)
        assert {p: self.dg.offsets(p) for p in self.parts} == {p: self.ing.offsets(p) for p in self.parts}
        assert _changes(self.dev) == _changes(self.host)
        ds, hs = self.dev.stats(), self.host.stats()
        if self.polls and self.ing.stats()["n_records"]:
            assert (ds.n_events, ds.n_errors) == (hs.n_events, hs.n_errors)

    def check_oracle(self, recs, prior):
        n_keys = len(self.keys())
        table = np.zeros((n_keys, self.state_bytes), np.uint8)
        if prior is not None:
            table[:min(len(prior), n_keys)] = prior[:n_keys]
        want, _, _ = I.c_fold_arrival_order(self.rules, self.state_bytes, recs, table, self.f64)
        assert np.array_equal(self.host.export_states()[:n_keys], want)


def _batch(off, recs, **kw):
    return K.encode_record_batch(off, [(d, k, v) for d, (k, v) in enumerate(recs)], **kw)


# ----------------------------------------------------------------------------- BankAccount
def _bank_poll(rng, nxt, n_ids, poll):
    """One poll over three partitions: creates, updates (some on aggregates that do not exist yet), flush markers, a refetch
    of the partition's last batch (duplicates) and null values."""
    fetches = []
    for p in sorted(nxt):
        data = bytearray()
        if poll == 0:
            data += _batch(nxt[p], [(b"", b"")])            # the producer's flush marker
            nxt[p] += 1
        for _ in range(int(rng.integers(2, 6))):
            recs = []
            for _ in range(int(rng.integers(1, 40))):
                a = int(rng.integers(0, n_ids)) * 3 + p     # every aggregate lives in one partition
                key = b"acct-%d:%d" % (a, nxt[p] + len(recs))
                u = rng.random()
                if u < 0.35:
                    v = _bank_created(nxt[p] + len(recs), b"u%d" % a, float(rng.integers(-500, 500)) / 4, b"own-%d" % a, int(rng.integers(0, 1 << 40)))
                elif u < 0.9:
                    v = _bank_updated(nxt[p] + len(recs), [0.0, -0.0, 1.5, float(rng.integers(0, 99))][int(rng.integers(0, 4))])
                elif u < 0.95:
                    v = None                                 # a null value: a hole without a tombstone type
                else:
                    key, v = b"", b""                        # a flush marker
                recs.append((key, v))
            last = _batch(nxt[p], recs, compression="lz4" if rng.random() < 0.6 else "none")
            data += last
            nxt[p] += len(recs)
        data += last                                         # refetch: every record of it is a duplicate
        fetches.append((p, bytes(data)))
    return fetches


def test_bank_account_consecutive_polls_match_the_host_decoder():
    rng = np.random.default_rng(61)
    nxt = {0: 0, 1: 10_000, 2: 20_000}
    with _Pair(P.bank_account_program()) as t:
        for poll in range(5):
            st = t.poll(_bank_poll(rng, nxt, 25, poll))
            assert st["n_duplicates"] > 0 and st["n_records"] > 0
        assert t.dev.stats().ms_group > 0                   # grouped on the device, not folded sort-free


def test_snapshot_restore_with_and_without_a_tombstone_type():
    """A 64-byte snapshot-restore program: type 0 sets every state word, type 1 deletes. With a tombstone type null values
    become type-1 events; without one they are holes."""
    prog = P.make_program(64, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 16), (N.OP_SET, 16, 32, 16), (N.OP_SET, 32, 48, 16)]),
                                              (N.TOMBSTONE, [])])
    rules = [(I.CREATE, [(I.OP_SET, 0, 16, 16), (I.OP_SET, 16, 32, 16), (I.OP_SET, 32, 48, 16)]), (I.TOMBSTONE, [])]
    rng = np.random.default_rng(62)
    polls, off = [], 0
    for _ in range(3):
        recs = []
        for _ in range(300):
            a = int(rng.integers(0, 60))
            recs.append((b"snap-%d" % a, None if rng.random() < 0.3 else _ev(0, off + len(recs), bytes(rng.integers(0, 256, 48, dtype=np.uint8)))))
        polls.append([(0, _batch(off, recs[:150], compression="lz4") + _batch(off + 150, recs[150:]))])
        off += 300
    for null_type in (1, None):
        with _Pair(prog, null_type=null_type, rules=rules, state_bytes=64) as t:
            for fetches in polls:
                st = t.poll(fetches)
                assert st["n_null_values"] > 0
            if null_type is not None:
                assert any(v is None for v in t.dev.get_many(t.keys()))


# ----------------------------------------------------------------------------- random programs outside the sort-free class
def _wide_program(rng, kind):
    """(state_bytes, rules, f64) of one kind: class 1 at W = 6 and W = 14 (row programs), 64-bit ops, an f64 field with
    IF_EXISTS, or a draw_program draw that is not sort-free."""
    if kind in ("class1_w6", "class1_w14"):
        w = 6 if kind == "class1_w6" else 14
        return 4 * w + 8, PC.row_program(rng, w, 1, int(rng.integers(2, 9))), []
    if kind == "ops64":
        return 32, [(I.MATERIALISE, [(I.OP_ADD_I64, 0, 16, 8), (I.OP_SET, 8, 4, 4)]), (I.IF_EXISTS, [(I.OP_SUB_I64, 0, 24, 8), (I.OP_SET, 16, 32, 8)]),
                    (I.CREATE, [(I.OP_SET, 0, 40, 16)]), (I.TOMBSTONE, []), (I.THROW, [])], []
    if kind == "f64_if_exists":
        return 48, [(I.CREATE, [(I.OP_SET, 0, 16, 16), (I.OP_SET, 16, 24, 8)]), (I.IF_EXISTS, [(I.OP_SET, 16, 24, 8)]),
                    (I.IF_EXISTS, []), (I.THROW, [])], [16]
    while True:
        sb, rules, f64 = PC.draw_program(rng)
        if sb != 16 or f64 or any(ex == I.IF_EXISTS for ex, _ in rules):
            return sb, rules, f64


def _to_native(sb, rules, f64):
    return P.make_program(sb, N.REC_FIXED64, rules, f64_fields=f64)


def _random_poll(rng, rules, nxt, poll, n_ids=40):
    """Records of random types (throwing ones included) and payloads over two partitions, with markers, null values and a
    refetch; the first and the last record of some aggregates in this poll throw."""
    n_types = len(rules)
    throwing = [t for t, (ex, _) in enumerate(rules) if ex == I.THROW] + [n_types, 255]
    fetches = []
    for p in sorted(nxt):
        per_agg = {}
        recs = []
        for _ in range(int(rng.integers(100, 300))):
            a = int(rng.integers(0, n_ids)) * 2 + p
            u = rng.random()
            if u < 0.04:
                recs.append((b"", b""))
                continue
            if u < 0.08:
                recs.append((b"r-%d" % a, None))
                continue
            t = int(rng.integers(0, n_types)) if rng.random() > 0.05 else int(rng.choice(throwing))
            payload = bytes(rng.integers(0, 256, 48, dtype=np.uint8))
            if rng.random() < 0.3:
                payload = payload[:8] + struct.pack("<d", PC.SPECIAL_F64[int(rng.integers(0, len(PC.SPECIAL_F64)))]) + payload[16:]
            per_agg.setdefault(a, []).append(len(recs))
            recs.append((b"r-%d:%d" % (a, nxt[p] + len(recs)), [t, payload]))
        aggs = sorted(per_agg)
        for a in aggs[:3]:
            recs[per_agg[a][0]][1][0] = throwing[0]         # throws at its first event of the poll
        for a in aggs[3:6]:
            recs[per_agg[a][-1]][1][0] = throwing[-1]       # ... at its last
        recs = [(k, v if v is None or isinstance(v, bytes) else _ev(v[0], nxt[p] + i, v[1])) for i, (k, v) in enumerate(recs)]
        half = len(recs) // 2
        b1 = _batch(nxt[p], recs[:half], compression="lz4")
        b2 = _batch(nxt[p] + half, recs[half:])
        nxt[p] += len(recs)
        fetches.append((p, b1 + b2 + (b2 if poll % 2 else b"")))
    return fetches


@pytest.mark.parametrize("kind", ["class1_w6", "class1_w14", "ops64", "f64_if_exists", "draw"])
def test_random_programs_match_the_host_decoder_and_the_oracle(kind):
    for seed in range(3):
        rng = np.random.default_rng([7100 + seed, len(kind), ord(kind[-1])])
        sb, rules, f64 = _wide_program(rng, kind)
        nxt = {0: 0, 1: 50_000}
        with _Pair(_to_native(sb, rules, f64), rules=rules, state_bytes=sb, f64=f64) as t:
            for poll in range(3):
                t.poll(_random_poll(rng, rules, nxt, poll))
            ds = t.dev.stats()
            assert ds.ms_group > 0


# ----------------------------------------------------------------------------- holes
def test_every_kind_of_hole_in_one_poll():
    prog = P.bank_account_program()
    with _Pair(prog) as t:
        t.poll([(0, _batch(0, [(b"acct-1", _bank_created(0, b"u1", 5.0, b"o1", 1)), (b"acct-2", _bank_created(1, b"u2", 7.0, b"o2", 2)),
                                (b"acct-3", _bank_created(2, b"u3", 9.0, b"o3", 3))]))])
        before = dict(zip(t.keys(), t.dev.get_many(t.keys())))
        # acct-2's only records in this poll are holes (a null value, a duplicate, an aborted update); acct-1 is updated
        p0 = (_batch(0, [(b"acct-2", _bank_updated(1, 99.0))]) +                                # refetch below the position
              _batch(3, [(b"", b"")]) +                                                          # flush marker
              _batch(4, [(b"acct-2", None)]) +                                                   # null value
              _batch(5, [(b"acct-2", _bank_updated(5, 50.0))], producer_id=9, transactional=True) +   # aborted
              K.encode_control_batch(6, 9, K.ABORT) +
              _batch(7, [(b"acct-1", _bank_updated(7, 6.5))], producer_id=10, transactional=True, compression="lz4") +
              K.encode_control_batch(8, 10, K.COMMIT))
        st = t.poll([(0, p0)], aborted={0: [(9, 5)]})
        assert (st["n_records"], st["n_markers"], st["n_null_values"], st["n_duplicates"], st["n_aborted_batches"]) == (1, 1, 1, 1, 1)
        assert st["n_control_batches"] == 2
        after = dict(zip(t.keys(), t.dev.get_many(t.keys())))
        assert after["acct-2"] == before["acct-2"] and after["acct-3"] == before["acct-3"] and after["acct-1"] != before["acct-1"]
        assert set(_changes(t.dev)) == {"acct-1"}            # acct-2 keeps its state and is not CHANGED
        # a poll that is only holes: nothing is folded, the last fold's flags stay (as on the host)
        st = t.poll([(0, _batch(9, [(b"", b""), (b"acct-3", None)]) + _batch(5, [(b"acct-3", _bank_updated(5, 1.0))]))])
        assert st["n_records"] == 0 and st["n_markers"] == 1 and st["n_duplicates"] == 1
        assert set(_changes(t.dev)) == {"acct-1"}


def test_flags_of_aggregates_the_poll_does_not_touch_are_cleared():
    prog = P.bank_account_program()
    with _Pair(prog) as t:
        t.poll([(0, _batch(0, [(b"a", _bank_created(0, b"a", 1.0, b"a", 1)), (b"b", _bank_created(1, b"b", 2.0, b"b", 2)),
                                (b"b", _ev(7, 2))]))])                     # b throws (type 7 is a MatchError)
        ch = _changes(t.dev)
        assert ch["a"][0] & N.ST_CHANGED and ch["b"][0] & N.ST_ERROR and ch["b"][1] == 1
        t.poll([(0, _batch(3, [(b"", b""), (b"c", _bank_created(4, b"c", 3.0, b"c", 3))]))])
        assert set(_changes(t.dev)) == {"c"}
        t.poll([(0, _batch(5, [(b"a", _bank_updated(5, 1.0))]))])        # the same balance: a is not CHANGED, c is cleared
        assert _changes(t.dev) == {}


def test_corrupted_batch_applies_nothing():
    rng = np.random.default_rng(63)
    nxt = {0: 0, 1: 10_000, 2: 20_000}
    good1 = _bank_poll(rng, nxt, 30, 0)
    saved = dict(nxt)
    bad = _bank_poll(rng, nxt, 30, 1)
    nxt = saved
    good2 = _bank_poll(rng, nxt, 30, 1)
    with _Pair(P.bank_account_program()) as t:
        t.poll(good1)
        keys = t.keys()
        before_rows = _rows_by_id(t.dev, keys, dev=True)
        before_changes = _changes(t.dev)
        before_offs = {p: t.dg.offsets(p) for p in nxt}
        broken = list(bad)
        d = bytearray(broken[1][1])
        d[len(d) // 2] ^= 0x10
        broken[1] = (broken[1][0], bytes(d))
        with pytest.raises(IngestError) as ei:
            for p, data in broken:
                t.dg.submit(p, data)
            t.dg.fold()
        assert ei.value.code == N.SGR_ERR_INVALID
        assert _rows_by_id(t.dev, keys, dev=True) == before_rows
        assert _changes(t.dev) == before_changes
        assert {p: t.dg.offsets(p) for p in nxt} == before_offs
        t.poll(good2, skip_stats=("n_new_keys",))            # ids the refused poll interned are reported with this one


# ----------------------------------------------------------------------------- scale and growth
def test_scale_poll_with_holes_and_growth_against_the_oracle():
    """2^24 live records of a class-1 program over 2^20 ids in 8 partitions, about 5 % duplicates (a refetch of each
    partition's first batches in the same poll), after a small first poll: the table grows inside the poll."""
    rules = [(I.CREATE, [(I.OP_SET, 0, 4, 4), (I.OP_ADD_I32, 4, 16, 4)]), (I.IF_EXISTS, [(I.OP_ADD_I32, 4, 16, 4), (I.OP_SET, 8, 4, 4)]),
             (I.IF_EXISTS, [(I.OP_SUB_I32, 12, 16, 4)]), (I.MATERIALISE, [(I.OP_SET, 16, 16, 4)]), (I.THROW, [])]
    sb = 32
    rng = np.random.default_rng(64)
    n, n_ids, parts, rpb = 1 << 24, 1 << 20, 8, 512
    agg = rng.integers(0, n_ids, size=n).astype(np.uint32)
    types = PC.type_mix(rules, n, rng, p_throw=1e-4)
    seqs = np.arange(n, dtype=np.uint32)
    bys = rng.integers(-1000, 1000, size=n).astype(np.int32)
    part = agg % parts
    with _Pair(_to_native(sb, rules, []), max_keys=n_ids + 1024) as t:
        small = []
        for p in range(parts):
            sel = np.arange(p, 64 * parts, parts, dtype=np.uint32)             # 64 ids per partition: a table of 1024 slots
            small.append((p, O.kafka_encode_counter(sel, np.zeros(len(sel), np.uint32), np.arange(len(sel), dtype=np.uint32),
                                                    np.ones(len(sel), np.int32), recs_per_batch=rpb, lz4=True).tobytes()))
        t.poll(small)
        prior = t.host.export_states()
        n_before = t.dev.n_aggregates()
        live = []
        for p in range(parts):
            idx = np.flatnonzero(part == p)
            base = t.ing.offsets(p)[0]
            wire = O.kafka_encode_counter(agg[idx], types[idx], seqs[idx], bys[idx], recs_per_batch=rpb, lz4=True, base_offset=base).tobytes()
            dup = int(len(idx) * 0.05) // rpb * rpb                           # the first batches again: duplicates
            head = O.kafka_encode_counter(agg[idx[:dup]], types[idx[:dup]], seqs[idx[:dup]], bys[idx[:dup]], recs_per_batch=rpb, lz4=True,
                                          base_offset=base).tobytes()
            t.dg.submit(p, wire + head)
            live.append(idx)
        st = t.dg.fold()
        assert st["n_records"] == n and st["n_duplicates"] > 0.04 * n
        assert t.dev.n_aggregates() > n_before
        assert t.dev.stats().ms_group > 0
        # the oracle: the live records in the order the partitions were submitted, dense index = position in `ids`
        ids = t.ing.keys()                                                    # the first poll's ids, in host dense order
        pos = {k: i for i, k in enumerate(ids)}
        for a in np.unique(agg):
            pos.setdefault("agg-%d" % a, len(pos))
        all_ids = list(pos)
        dense = np.array([pos.get("agg-%d" % a, -1) for a in range(n_ids)], dtype=np.int64)
        order = np.concatenate(live)
        recs = np.zeros((n, 64), np.uint8)
        recs[:, 0:4] = types[order].view(np.uint8).reshape(-1, 4)
        recs[:, 4:8] = seqs[order].view(np.uint8).reshape(-1, 4)
        recs[:, 8:16] = dense[agg[order]].astype(np.uint64).view(np.uint8).reshape(-1, 8)
        recs[:, 16:20] = bys[order].view(np.uint8).reshape(-1, 4)
        table = np.zeros((len(all_ids), sb), np.uint8)
        table[:len(ids)] = prior[:len(ids)]
        want, n_events, n_errors = I.c_fold_arrival_order(rules, sb, recs, table)
        _, _, got_idx = t.dev.get_many(all_ids, arrays=True)
        assert (got_idx >= 0).all()
        full = t.dev.export_states()[got_idx]
        assert np.array_equal(full, want)
        ds = t.dev.stats()
        assert (ds.n_events, ds.n_errors) == (n_events, n_errors)


# ----------------------------------------------------------------------------- control
def test_counter_poll_with_holes_stays_sort_free():
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1024) as dg:
            b = _batch(0, [(b"", b""), (b"agg-1:1", _ev(0, 1, struct.pack("<i", 3))), (b"agg-2:2", None)])
            dg.submit(0, b + b)
            st = dg.fold()
            assert (st["n_records"], st["n_markers"], st["n_null_values"], st["n_duplicates"]) == (1, 1, 1, 3)
            s = e.stats()
            assert s.fold_launches == 1 and s.ms_group == 0.0
            assert np.frombuffer(e.get("agg-1"), "<i4").tolist() == [3, 1]


def test_counter_poll_of_holes_only_keeps_the_atomic_fold():
    """A sort-free program keeps today's path for a poll whose records were all dropped: the atomic fold runs and clears the
    last poll's flags (a grouped program folds nothing there, test_every_kind_of_hole_in_one_poll)."""
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1024) as dg:
            dg.submit(0, _batch(0, [(b"agg-1:1", _ev(0, 1, struct.pack("<i", 3)))]))
            dg.fold()
            assert set(_changes(e)) == {"agg-1"}
            dg.submit(0, _batch(1, [(b"", b""), (b"agg-1:2", None)]) + _batch(0, [(b"agg-1:1", _ev(0, 1, struct.pack("<i", 3)))]))
            st = dg.fold()
            assert (st["n_records"], st["n_markers"], st["n_null_values"], st["n_duplicates"]) == (0, 1, 1, 1)
            s = e.stats()
            assert s.fold_launches == 1 and s.ms_group == 0.0
            assert _changes(e) == {}
            assert np.frombuffer(e.get("agg-1"), "<i4").tolist() == [3, 1]


@pytest.mark.parametrize("only_holes", [True, False])
def test_variable_record_programs_are_still_refused(only_holes):
    """SGR_REC_VAR16 programs are refused by the incremental fold, with its message, also for a poll of a flush marker only;
    nothing of the poll is applied."""
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program(N.REC_VAR16))
        with DeviceIngest(e, 1024) as dg:
            recs = [(b"", b"")] + ([] if only_holes else [(b"agg-1:1", _ev(0, 1, struct.pack("<i", 3)))])
            dg.submit(0, _batch(0, recs))
            with pytest.raises(IngestError) as ei:
                dg.fold()
            assert ei.value.code == N.SGR_ERR_UNSUPPORTED
            assert "fixed 64-byte records" in str(ei.value)
            assert dg.offsets(0) == (0, 0)
