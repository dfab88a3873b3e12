"""-m gpu: keyed state writes on the device (sgr_put_batch, csrc/put_batch.cu).

The same stream of state records gives the same table, flags, key table, reads, change pages and scan pages as today's path
(snapshot and tombstone events through sgr_fold_incremental, slots in first-appearance order); wide states and VAR16 programs
match the NumPy restatement (oracle/put_batch.py); put batches and folds scope their flags to themselves; the key-table rules
and the refusals hold; a 4 M-record batch over 2 M UUID ids and a 1 % batch onto it are exact; a state-topic store restores
96-byte states through put() / flush()."""
import ctypes as C
import struct
import threading
import time
import uuid

import numpy as np
import pytest

from oracle import put_batch as O
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.store import GpuReplayKeyValueStore, StateCodec

pytestmark = pytest.mark.gpu

CHANGED_OR_ERROR = N.ST_CHANGED | N.ST_ERROR


def bank_snapshot_program():
    """A BankAccount-shaped 64-byte state (uuid, balance: Double @16, owner, code: 48 program bytes) restored from its state
    topic: type 0 = snapshot (CREATE + SET of the 48 bytes from the record @16), type 1 = tombstone."""
    return P.make_program(64, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 48)]), (N.TOMBSTONE, [])], f64_fields=[16])


# name -> (program with snapshot rules, snapshot type, tombstone type, payload bytes, Double offsets)
SNAPSHOT = {
    "counter": (P.counter_program_with_snapshot_rules, P.COUNTER_SNAPSHOT_TYPE, P.COUNTER_TOMBSTONE_TYPE, 8, ()),
    "bank_account": (bank_snapshot_program, 0, 1, 48, (16,)),
}

SPECIAL_F64 = [0.0, -0.0, float("nan"), 1.5, -2.25, float("inf")]


def payload(rng, nbytes, f64_offsets):
    b = bytearray(rng.integers(0, 4, size=nbytes, dtype=np.uint8).tobytes())   # few values: repeated writes often equal
    for off in f64_offsets:
        b[off:off + 8] = struct.pack("<d", SPECIAL_F64[int(rng.integers(0, len(SPECIAL_F64)))])
    return bytes(b)


def random_batches(rng, n_batches, size, nbytes, f64_offsets):
    """Batches of (id, bytes | None): repeated ids, re-creation after a delete, deletes of ids never seen."""
    pool = [str(uuid.UUID(int=int(rng.integers(0, 1 << 62)) << 64 | i)) for i in range(size * n_batches)]
    seen, out = [], []
    for b in range(n_batches):
        batch = []
        for _ in range(size):
            r = rng.random()
            if seen and r < 0.45:
                k = seen[int(rng.integers(0, len(seen)))]
            elif r < 0.5:
                k = f"unknown-{int(rng.integers(0, 1 << 40))}"
            else:
                k = pool[len(seen) % len(pool)]
            if k not in seen:
                seen.append(k)
            tomb = rng.random() < 0.2 or k.startswith("unknown-")
            batch.append((k, None if tomb else payload(rng, nbytes, f64_offsets)))
        out.append(batch)
    return out


def put(e, batch):
    user = e.state_bytes - 8
    rows = np.zeros((len(batch), user), np.uint8)
    for i, (_, v) in enumerate(batch):
        if v is not None:
            rows[i, :len(v)] = np.frombuffer(v, np.uint8)
    return e.put_batch([k for k, _ in batch], rows, [v is not None for _, v in batch])


class EventArm:
    """Today's path at the engine level: state records as snapshot / tombstone events through sgr_fold_incremental, slots in
    first-appearance order, a table grown by capacity and a key table padded with placeholder ids."""

    def __init__(self, e, snap, tomb):
        self.e, self.snap, self.tomb = e, snap, tomb
        self.keys, self.index, self.cap = [], {}, 0

    def apply(self, batch):
        recs = np.zeros((len(batch), 64), np.uint8)
        for i, (k, v) in enumerate(batch):
            if k not in self.index:
                self.index[k] = len(self.keys)
                self.keys.append(k)
            recs[i, 0:4] = np.frombuffer(np.uint32(self.tomb if v is None else self.snap).tobytes(), np.uint8)
            recs[i, 8:16] = np.frombuffer(np.uint64(self.index[k]).tobytes(), np.uint8)
            if v is not None:
                recs[i, 16:16 + len(v)] = np.frombuffer(v, np.uint8)
        if len(self.keys) > self.cap:
            old = self.e.export_states() if self.cap else None
            self.cap = max(2 * len(self.keys), 1024)
            prior = np.zeros((self.cap, self.e.state_bytes), np.uint8)
            if old is not None:
                prior[:len(old)] = old
            self.e.set_initial_states(prior)
        self.e.fold_incremental(recs)
        self.e.load_keys(self.keys + [f"\0unused-{i}" for i in range(len(self.keys), self.cap)])


def pages(gen):
    return [(p[0].tolist(), p[1].tolist(), [np.asarray(x).tobytes() for x in p[2:-1]], p[-1]) for p in gen]


@pytest.mark.parametrize("name", sorted(SNAPSHOT))
def test_differential_against_snapshot_events(name):
    make, snap, tomb, nbytes, f64 = SNAPSHOT[name]
    rng = np.random.default_rng(11 if name == "counter" else 12)
    batches = random_batches(rng, 5, 3000, nbytes, f64)
    with ReplayEngine(0) as a, ReplayEngine(0) as b:
        a.register_program(make())
        b.register_program(make())
        arm = EventArm(b, snap, tomb)
        n_ids = 0
        for batch in batches:
            n_new = put(a, batch)
            arm.apply(batch)
            assert n_new == len(arm.keys) - n_ids
            n_ids = len(arm.keys)
            ta, tb = a.export_states(), b.export_states()
            assert a.n_aggregates() == n_ids
            assert np.array_equal(ta, tb[:n_ids])
            tail = tb[n_ids:, -8:].copy().view(np.uint32)[:, 0]
            assert not (tail & N.ST_EXISTS).any()
            assert a.get_many(arm.keys, arrays=True)[2].tolist() == list(range(n_ids))   # the ids in index order
            assert a.get_many(arm.keys) == b.get_many(arm.keys)
            assert a.get_many(["never-written"]) == [None]
            assert pages(a.export_changes(CHANGED_OR_ERROR, page_rows=97)) == pages(b.export_changes(CHANGED_OR_ERROR, page_rows=97))
            assert pages(a.scan(page_rows=113)) == pages(b.scan(page_rows=113))
            for k in arm.keys[:20]:
                assert a.get(k) == b.get(k)


def wide_program(sb, kind, f64_offsets):
    return P.make_program(sb, kind, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])], f64_fields=f64_offsets)


@pytest.mark.parametrize("sb,kind,f64", [(64, N.REC_FIXED64, (0, 40)), (96, N.REC_FIXED64, (8, 48, 80)), (128, N.REC_FIXED64, (0, 112)),
                                         (128, N.REC_VAR16, (16, 64)), (96, N.REC_VAR16, ())])
def test_wide_states_against_the_oracle(sb, kind, f64):
    rng = np.random.default_rng(sb + kind)
    user = sb - 8
    batches = random_batches(rng, 4, 2500, user, f64)
    with ReplayEngine(0) as e:
        e.register_program(wide_program(sb, kind, list(f64)))
        ids, table = [], np.zeros((0, sb), np.uint8)
        for batch in batches:
            ids, table, n_new = O.put_batch(ids, table, batch, f64)
            assert put(e, batch) == n_new
            assert np.array_equal(e.export_states(), table)
            assert e.get_many(ids, arrays=True)[2].tolist() == list(range(len(ids)))
        fl = table[:, user:user + 4].copy().view(np.uint32)[:, 0]
        live = sorted((ids[i].encode(), ids[i]) for i in range(len(ids)) if fl[i] & N.ST_EXISTS)
        assert [k for p in e.scan(page_rows=301) for k in p[3]] == [k for _, k in live]


def test_changed_rule_for_doubles_and_repeats():
    """NaN is never equal to itself, 0.0 == -0.0; snap(x), tomb, snap(x) is not CHANGED; a tombstone of None is not CHANGED."""
    sb = 32
    prog = wide_program(sb, N.REC_FIXED64, [0])
    d = lambda x, tail=b"\1" * 16: struct.pack("<d", x) + tail   # noqa: E731
    with ReplayEngine(0) as e:
        e.register_program(prog)
        put(e, [("nan", d(float("nan"))), ("zero", d(0.0)), ("x", d(1.0)), ("gone", d(2.0)), ("none", None)])
        put(e, [("nan", d(float("nan"))), ("zero", d(-0.0)), ("x", d(1.0)), ("x", None), ("x", d(1.0)), ("none", None),
                ("gone", None), ("gone", d(2.0), ), ("gone", None)])
        t = e.export_states()
        fl = t[:, 24:28].copy().view(np.uint32)[:, 0]
        assert fl.tolist() == [N.ST_EXISTS | N.ST_CHANGED, N.ST_EXISTS, N.ST_EXISTS, N.ST_CHANGED, 0]
        assert t[1, :8].tobytes() == struct.pack("<d", -0.0)   # the row's own bytes
        assert not t[3, :24].any()


# ------------------------------------------------------------------ interplay
def counter_rows(values):
    return [(k, None if v is None else struct.pack("<ii", v, 1)) for k, v in values]


def flags(e):
    return e.export_states()[:, 8:12].copy().view(np.uint32)[:, 0].tolist()


def counter_events(slots_by):
    recs = np.zeros((len(slots_by), 64), np.uint8)
    for i, (slot, by) in enumerate(slots_by):
        recs[i, 8:16] = np.frombuffer(np.uint64(slot).tobytes(), np.uint8)
        recs[i, 16:20] = np.frombuffer(np.int32(by).tobytes(), np.uint8)
    return recs


@pytest.mark.parametrize("incremental", [0, 1])
def test_fold_and_put_each_leave_only_their_own_flags(incremental):
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program_with_snapshot_rules())
        e.set_option("incremental", incremental)
        put(e, counter_rows([("a", 1), ("b", 2), ("c", 3)]))
        assert flags(e) == [N.ST_EXISTS | N.ST_CHANGED] * 3
        e.fold_incremental(counter_events([(0, 5)]))
        assert flags(e) == [N.ST_EXISTS | N.ST_CHANGED, N.ST_EXISTS, N.ST_EXISTS]
        put(e, counter_rows([("c", 4), ("d", None)]))
        assert flags(e) == [N.ST_EXISTS, N.ST_EXISTS, N.ST_EXISTS | N.ST_CHANGED, 0]
        e.fold_incremental(counter_events([(1, 1), (3, 1)]))
        assert flags(e) == [N.ST_EXISTS, N.ST_EXISTS | N.ST_CHANGED, N.ST_EXISTS, N.ST_EXISTS | N.ST_CHANGED]
        assert e.get("a") == struct.pack("<ii", 6, 0)
        assert e.get("c") == struct.pack("<ii", 4, 1)


def test_export_in_progress_ends_with_a_put():
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        put(e, counter_rows([(f"k{i}", i) for i in range(100)]))
        it = e.export_changes(N.ST_CHANGED, page_rows=10)
        assert len(next(it)[0]) == 10
        put(e, counter_rows([("k1", 7)]))
        with pytest.raises(N.InvalidStateStoreException):
            next(it)


def test_reads_see_new_ids_without_a_rebuild():
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        first = [f"id-{i}" for i in range(500)]
        put(e, counter_rows([(k, i) for i, k in enumerate(first)]))
        assert e.get_many(first, arrays=True)[2].tolist() == list(range(500))
        assert [k for p in e.scan() for k in p[3]] == sorted(first, key=str.encode)
        more = [f"id-{i}" for i in range(400, 900)]
        put(e, counter_rows([(k, 1) for k in more] + [("id-3", None)]))
        idx = e.get_many(first + more[100:], arrays=True)[2].tolist()
        assert idx == list(range(900))
        live = [k for k in first + more[100:] if k != "id-3"]
        assert [k for p in e.scan(page_rows=64) for k in p[3]] == sorted(live, key=str.encode)
        assert e.get("id-3") is None and e.get("id-899") == struct.pack("<ii", 1, 1)


def test_load_keys_then_puts_append_to_that_table():
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(["k0", "k1", "k2"])
        assert put(e, counter_rows([("k1", 5), ("new", 6), ("k2", None), ("new2", None)])) == 2
        assert e.n_aggregates() == 5
        assert e.get_many(["k0", "k1", "k2", "new", "new2"], arrays=True)[2].tolist() == [0, 1, 2, 3, 4]
        assert e.get_many(["k0", "k1", "new"]) == [None, struct.pack("<ii", 5, 1), struct.pack("<ii", 6, 1)]
        assert put(e, counter_rows([("k0", 1)])) == 0
        assert e.get("k0") == struct.pack("<ii", 1, 1)


def _append_keys(e, owner, keys):
    enc = [k.encode() for k in keys]
    offs = np.zeros(len(enc) + 1, np.uint32)
    np.cumsum([len(b) for b in enc], out=offs[1:])
    blob = np.frombuffer(b"".join(enc) or b"\0", np.uint8)
    assert e._lib.sgr_append_keys(e._h, owner, blob.ctypes.data, offs.ctypes.data, len(enc)) == 0


def test_refusals_apply_nothing():
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.grow_states(2)
        _append_keys(e, C.c_void_p(0x77), ["a", "b"])
        before = e.export_states()
        with pytest.raises(N.InvalidStateStoreException):
            put(e, counter_rows([("a", 1), ("c", 2)]))
        assert np.array_equal(e.export_states(), before)
        assert e.get_many(["a", "b", "c"], arrays=True)[2].tolist() == [0, 1, -1]
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.dist_init(0, 1, None, 1024)
        with pytest.raises(SgrError) as ex:
            put(e, counter_rows([("a", 1)]))
        assert ex.value.code == N.SGR_ERR_UNSUPPORTED
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        rows = np.zeros((2, 8), np.uint8)
        pres = np.ones(2, np.uint8)
        offs = np.array([0, 2, 1], np.uint32)
        blob = np.frombuffer(b"abc", np.uint8)
        assert e._lib.sgr_put_batch(e._h, blob.ctypes.data, offs.ctypes.data, 2, rows.ctypes.data, pres.ctypes.data, None) == N.SGR_ERR_INVALID
        assert e._lib.sgr_put_batch(e._h, blob.ctypes.data, offs.ctypes.data, 0, None, None, None) == 0


# ------------------------------------------------------------------ scale
def lowest_free_while(fn):
    """(fn(), the lowest free device memory a second thread saw while fn ran)."""
    import torch

    low = [torch.cuda.mem_get_info(0)[0]]
    stop = threading.Event()

    def sample():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info(0)[0])
            time.sleep(0.0005)

    th = threading.Thread(target=sample)
    th.start()
    try:
        r = fn()
    finally:
        stop.set()
        th.join()
    return r, low[0]


def expected_counter(ids_s, rows, present, prior_ids, prior):
    """Vectorised restatement for the scale test (the same rules as oracle/put_batch.py, Counter state, no Double fields)."""
    n = len(ids_s)
    uniq, first, inv = np.unique(ids_s, return_index=True, return_inverse=True)
    last = np.full(len(uniq), -1, np.int64)
    np.maximum.at(last, inv, np.arange(n))
    known = {k: i for i, k in enumerate(prior_ids)}
    slot_of_u = np.empty(len(uniq), np.int64)
    new_u = [u for u in range(len(uniq)) if uniq[u].decode() not in known]
    new_u.sort(key=lambda u: first[u])
    for u in range(len(uniq)):
        slot_of_u[u] = known.get(uniq[u].decode(), -1)
    base = len(prior_ids)
    for r, u in enumerate(new_u):
        slot_of_u[u] = base + r
    ids = list(prior_ids) + [uniq[u].decode() for u in new_u]
    table = np.zeros((len(ids), 16), np.uint8)
    table[:len(prior)] = prior
    table[:, 12:16] = 0
    fl = table[:, 8:12].copy().view(np.uint32)[:, 0] & N.ST_EXISTS
    slots = slot_of_u
    old_ex = fl[slots] != 0
    old_rows = table[slots, :8].copy()
    pres = present[last]
    new_rows = np.where(pres[:, None], rows[last], 0).astype(np.uint8)
    changed = np.where(pres, ~old_ex | (new_rows != old_rows).any(axis=1), old_ex)
    newfl = np.where(pres, N.ST_EXISTS, 0) | np.where(changed, N.ST_CHANGED, 0)
    table[:, 8:12] = fl.astype(np.uint32).view(np.uint8).reshape(-1, 4)
    table[slots, :8] = new_rows
    table[slots, 8:12] = newfl.astype(np.uint32).view(np.uint8).reshape(-1, 4)
    return ids, table


def test_scale_four_million_records_over_two_million_uuids():
    t0 = time.perf_counter()
    rng = np.random.default_rng(99)
    n_ids, n = 2 << 20, 4 << 20
    pool = np.array([str(uuid.UUID(bytes=rng.bytes(16))).encode() for _ in range(n_ids)], dtype="S36")
    # every id once (shuffled) and about 30 % of the records repeat one
    pick = np.concatenate([rng.permutation(n_ids), rng.integers(0, n_ids, size=n - n_ids)])
    pick = pick[rng.permutation(n)]
    ids_s = pool[pick]
    rows = rng.integers(0, 256, size=(n, 8), dtype=np.uint8)
    present = rng.random(n) >= 0.05
    keys = [k.decode() for k in ids_s]
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        total = __import__("torch").cuda.mem_get_info(0)[1]
        t1 = time.perf_counter()
        n_new, low0 = lowest_free_while(lambda: e.put_batch(keys, rows, present))
        t_big = time.perf_counter() - t1
        want_ids, want = expected_counter(ids_s, rows, present, [], np.zeros((0, 16), np.uint8))
        assert n_new == len(want_ids) == n_ids
        assert np.array_equal(e.export_states(), want)
        # a 1 % batch onto it: known ids, some new ones, tombstones
        m = n // 100
        extra = np.array([str(uuid.UUID(bytes=rng.bytes(16))).encode() for _ in range(m // 10)], dtype="S36")
        ids2 = np.concatenate([pool[rng.integers(0, n_ids, size=m - len(extra))], extra])[rng.permutation(m)]
        rows2 = rng.integers(0, 4, size=(m, 8), dtype=np.uint8)
        present2 = rng.random(m) >= 0.05
        t1 = time.perf_counter()
        n_new2, low1 = lowest_free_while(lambda: e.put_batch([k.decode() for k in ids2], rows2, present2))
        t_small = time.perf_counter() - t1
        want_ids2, want2 = expected_counter(ids2, rows2, present2, want_ids, want)
        assert n_new2 == len(want_ids2) - len(want_ids)
        assert np.array_equal(e.export_states(), want2)
        sample = [want_ids2[i] for i in rng.integers(0, len(want_ids2), size=5000)]
        idx = {k: i for i, k in enumerate(want_ids2)}
        assert e.get_many(sample, arrays=True)[2].tolist() == [idx[k] for k in sample]
        print(f"\nput_batch scale: {n} records / {n_ids} UUID ids in {t_big:.2f} s, then {m} records in {t_small:.3f} s (wall, "
              f"including the Python encode); {time.perf_counter() - t0:.1f} s in all; device bytes in use at the peak "
              f"(whole device) {total - min(low0, low1)}")


# ------------------------------------------------------------------ the store
def test_state_topic_store_of_96_byte_states():
    sb = 96
    prog = wide_program(sb, N.REC_FIXED64, [8])
    codec = StateCodec(lambda k, v: v, lambda k, b: b)
    calls = []
    st = GpuReplayKeyValueStore("wide", prog, codec=codec, on_changes=lambda ch, fa: calls.append((ch, fa)))
    st.init()
    val = lambda i: bytes([i % 251]) * 88   # noqa: E731
    for i in range(300):
        st.put(f"acct-{i:04d}", val(i))
    st.putAll([("acct-0001", val(7)), ("acct-0002", None)])
    st.delete("acct-0003")
    assert st.get("acct-0001") == val(7)      # read-your-writes before the flush
    st.flush()
    assert st.engine.n_aggregates() == 300
    assert st.get("acct-0001") == val(7) and st.get("acct-0002") is None and st.get("acct-0003") is None
    assert st.get("acct-0299") == val(299) and st.get("nobody") is None
    want = [(f"acct-{i:04d}", val(7) if i == 1 else val(i)) for i in range(300) if i not in (2, 3)]
    assert list(st.all()) == want
    assert list(st.range("acct-0100", "acct-0104")) == [w for w in want if "acct-0100" <= w[0] <= "acct-0104"]
    assert st.approximateNumEntries() == 298
    changed, failed = calls[-1]
    assert failed == [] and sorted(changed) == sorted(want)
    st.put("acct-0001", val(7))       # the same bytes: not a change
    st.put("acct-0005", val(9))
    st.put("acct-0002", val(2))       # re-created
    st.delete("acct-0004")
    st.flush()
    assert sorted(calls[-1][0], key=lambda kv: kv[0]) == [("acct-0002", val(2)), ("acct-0004", None), ("acct-0005", val(9))]
    with pytest.raises(SgrError):
        st.put_event("acct-0001", b"\0" * 64)
    with pytest.raises(ValueError):
        st.put("too-wide", b"\0" * 89)
    st.close()
