"""-m gpu: ids that share one 64-bit tag through every probe (oracle/id_hash.py), on every device user of the id dictionary
(csrc/id_dict.cuh), and the polls after a full device dictionary.

Random ids never share a tag, so every other GPU suite stops its probes at the first tag match. Here clusters of 2, 64 and 3000
ids share one tag, a fourth cluster's home is the last slot of every table up to 2^20 slots (its probes wrap to slot 0), and
the two ids that hash to 0 and 1 both carry tag 1. Everything is compared per id with a plain restatement: the Counter events
folded in Python, the host decoder fed the same bytes, oracle/put_batch.py and oracle/state_topic.py.
"""
import ctypes as C
import struct

import numpy as np
import pytest

from oracle import id_hash as H
from oracle import kafka_batch as K
from oracle import put_batch as PB
from oracle import state_topic as S
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest, IngestError

pytestmark = pytest.mark.gpu

WRAP = (1 << 20) - 1


def _s(ids):
    return [b.decode() for b in ids]


def _clusters(tag):
    """(seen, never seen) ids: clusters of 2, 64 and 3000 plus a wrapping one, each with members held back, a tag-1 pair, one
    half of a second tag-1 pair, random ids, and a near miss of the big cluster (same host shard and tag, other device tag)."""
    c2 = H.cluster(4, tag + b"2-", seed=1)
    c64 = H.cluster(72, tag + b"64-", seed=2)
    c3k = H.cluster(3008, tag + b"3k-", seed=3)
    wrap = H.cluster(40, tag + b"w-", home_mask=WRAP, seed=4)
    pair = H.tag_one_pair(tag + b"1-", seed=5)
    half = H.tag_one_pair(tag + b"h-", seed=6)
    rand = H.random_ids(200, seed=7)
    seen = c2[:2] + c64[:64] + c3k[:3000] + wrap[:32] + pair + half[:1] + rand
    never = c2[2:] + c64[64:] + c3k[3000:] + wrap[32:] + half[1:] + [H.near_miss(c3k[0], seed=8)]
    return _s(seen), _s(never)


def _ev(t, seq, by):
    return struct.pack("<IIi", t, seq, by)


def _events_polls(rng, ids, n_polls=2, n_parts=4, compression="lz4", seq0=1):
    """Polls of fetches [(partition, bytes)] with every id at least once, repeats inside one batch (threads race to intern one
    id), and the Counter's expected rows per id, folded in arrival order."""
    order = list(ids) + [ids[i] for i in rng.integers(0, len(ids), size=2 * len(ids))]
    rng.shuffle(order)
    recs, seq = [], seq0
    for k in order:
        for _ in range(int(rng.integers(1, 5)) if rng.random() < 0.2 else 1):
            recs.append((k, int(rng.integers(0, 3)), seq, int(rng.integers(-1000, 1000))))
            seq += 1
    # cut into batches, batches into polls and partitions
    batches, i = [], 0
    while i < len(recs):
        n = int(rng.integers(1, 60))
        batches.append(recs[i:i + n])
        i += n
    nxt = {p: 0 for p in range(n_parts)}
    polls = [[[] for _ in range(n_parts)] for _ in range(n_polls)]
    for b, batch in enumerate(batches):
        polls[b * n_polls // len(batches)][int(rng.integers(0, n_parts))].append(batch)
    out, arrival = [], []
    for poll in polls:
        fetches = []
        for p, bs in enumerate(poll):
            data = bytearray()
            for batch in bs:
                comp = compression if compression != "mixed" else ("lz4" if rng.random() < 0.5 else "none")
                data += K.encode_record_batch(nxt[p], [(d, f"{k}:{s}".encode(), _ev(t, s, by)) for d, (k, t, s, by) in enumerate(batch)],
                                              compression=comp)
                nxt[p] += len(batch)
                arrival += batch
            if bs:
                fetches.append((p, bytes(data)))
        out.append(fetches)
    return out, arrival, seq


def _counter_rows(arrival, rows=None):
    """Counter (count += by on type 0, -= by on type 1, version = seq on both; type 2 changes nothing but creates the state)."""
    rows = {} if rows is None else dict(rows)
    for k, t, s, by in arrival:
        c, v = rows.get(k, (0, 0))
        if t == 0:
            c, v = (c + by + 2**31) % 2**32 - 2**31, s
        elif t == 1:
            c, v = (c - by + 2**31) % 2**32 - 2**31, s
        rows[k] = (c, v)
    return rows


def _packed(rows):
    return {k: struct.pack("<ii", *v) for k, v in rows.items()}


def _host_states(polls, ids):
    ing = Ingest()
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        for fetches in polls:
            for part, data in fetches:
                ing.record_batches(part, data)
        e.fold_ingested(ing)
        return {k: e.get(k) for k in ids}, ing.keys()


def _scan_ids(e):
    return [k for pg in e.scan(page_rows=509) for k in pg[3]]


def _check_table(e, want, never):
    """want: id -> row bytes (every id with a state); never: ids the engine must not know."""
    keys = list(want)
    states, flags, idx = e.get_many(keys + never, arrays=True)
    n = len(keys)
    assert (idx[:n] >= 0).all() and len(set(idx[:n].tolist())) == n
    assert (idx[n:] == -1).all() and not (flags[n:] & N.ST_EXISTS).any()
    got = {k: states[i, :len(want[k])].tobytes() for i, k in enumerate(keys)}
    assert got == want
    assert e.get_many(never) == [None] * len(never)
    for k in keys[::397] + keys[-3:]:
        assert e.get(k) == want[k], k
    assert _scan_ids(e) == sorted(keys, key=str.encode)


# ------------------------------------------------------------------ device ingest, events topic
@pytest.mark.parametrize("compression", ["none", "lz4", "mixed"])
def test_events_topic_clusters(compression):
    rng = np.random.default_rng({"none": 11, "lz4": 12, "mixed": 13}[compression])
    seen, never = _clusters(b"ev-")
    polls, arrival, _ = _events_polls(rng, seen, compression=compression)
    want = _packed(_counter_rows(arrival))
    host, host_keys = _host_states(polls, seen)
    assert host == want                                  # the host decoder agrees with the restatement
    assert sorted(host_keys) == sorted(seen)
    firsts = []
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1 << 14) as dg:
            for rep in range(2):                         # after a reset the same polls fold to the same states
                got_new, known = [], set()
                for fetches in polls:
                    for part, data in fetches:
                        dg.submit(part, data)
                    got_new.append(dg.fold()["n_new_keys"])
                    ids = {bytes(r[1]).split(b":")[0].decode() for _, d in fetches for b in K.decode_record_batches(d) for r in b["records"]}
                    firsts.append(len(ids - known))
                    known |= ids
                assert got_new == firsts[-len(polls):]
                _check_table(e, want, never)
                dg.reset()
                e.set_initial_states(None)


# ------------------------------------------------------------------ device ingest, state topic
def test_state_topic_clusters():
    rng = np.random.default_rng(21)
    seen, never = _clusters(b"st-")
    nxt = {p: 0 for p in range(3)}
    polls = []
    for _ in range(3):
        fetches = []
        for p in range(3):
            data = bytearray()
            for _ in range(int(rng.integers(4, 12))):
                recs = []
                for d in range(int(rng.integers(1, 200))):
                    k = seen[int(rng.integers(0, len(seen)))].encode()
                    recs.append((d, k, None if rng.random() < 0.15 else rng.integers(0, 4, size=int(rng.integers(0, 9)), dtype=np.uint8).tobytes()))
                data += K.encode_record_batch(nxt[p], recs, compression="lz4" if rng.random() < 0.5 else "none")
                nxt[p] += len(recs)
            fetches.append((p, bytes(data), []))
        polls.append(fetches)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        sb = e.state_bytes
        with DeviceIngest(e, 1 << 14) as dg:
            dg.set_state_topic(True)
            ids, table, done, n_new = [], np.zeros((0, sb), np.uint8), [], 0
            for fetches in polls:
                for p, data, _ in fetches:
                    dg.submit(p, data)
                n_new += dg.fold()["n_new_keys"]
                done += fetches
                recs, _, _ = S.read_committed_states(done, S.PACKED, sb - 8)
                ids, table = S.apply([], np.zeros((0, sb), np.uint8), recs)
                assert n_new == len(ids)
                fl = table[:, sb - 8:sb - 4].copy().view("<u4").ravel()
                want = {k: table[i, :sb - 8].tobytes() for i, k in enumerate(ids) if fl[i] & N.ST_EXISTS}
                _check_table(e, want, never)
                _, _, idx = e.get_many(ids, arrays=True)
                assert (idx >= 0).all() and len(set(idx.tolist())) == len(ids)


# ------------------------------------------------------------------ the engine's id index
def _append(e, owner, ids):
    enc = [k.encode() for k in ids]
    offs = np.zeros(len(enc) + 1, dtype=np.uint32)
    np.cumsum([len(b) for b in enc], out=offs[1:])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    assert e._lib.sgr_append_keys(e._h, owner, blob.ctypes.data, offs.ctypes.data, len(enc)) == 0


def test_engine_index_loads_and_appends_clusters():
    seen, never = _clusters(b"ix-")
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(seen)
        e.grow_states(len(seen))
        assert e.get_many(seen + never, arrays=True)[2].tolist() == list(range(len(seen))) + [-1] * len(never)
    # appends land one cluster across the 1024 -> 2048 -> 4096-slot rehashes
    big = _s(H.cluster(2000, b"grow-", seed=31))
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.grow_states(4096)
        owner = C.c_void_p(0x51)
        have = 0
        for n in (300, 200, 300, 400, 800):
            _append(e, owner, big[have:have + n])
            have += n
            q = big[:have] + big[have:have + 50]
            assert e.get_many(q, arrays=True)[2].tolist() == list(range(have)) + [-1] * len(big[have:have + 50])


def test_a_true_duplicate_inside_a_cluster_is_refused():
    big = _s(H.cluster(300, b"dup-", seed=41))
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.grow_states(1024)
        owner = C.c_void_p(0x77)
        _append(e, owner, big[:100])
        assert e.get_many([big[3]], arrays=True)[2][0] == 3
        _append(e, owner, [big[200], big[42]])
        with pytest.raises(SgrError) as batch:
            e.get_many([big[3]])
        assert batch.value.code == N.SGR_ERR_INVALID and "duplicate aggregate id in key table" in str(batch.value)


# ------------------------------------------------------------------ sgr_put_batch
def test_put_batch_clusters_against_the_restatement():
    rng = np.random.default_rng(51)
    a = _s(H.cluster(1200, b"pa-", seed=52))
    b = _s(H.cluster(400, b"pb-", seed=53))
    pair = _s(H.tag_one_pair(b"pp-", seed=54))
    rand = _s(H.random_ids(100, seed=55))
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        user = e.state_bytes - 8

        def row():
            return None if rng.random() < 0.15 else rng.integers(0, 3, size=user, dtype=np.uint8).tobytes()

        batches = [
            [(k, row()) for k in a[:600] + rand + pair[:1]],                                    # half of cluster a
            [(a[int(i)], row()) for i in rng.integers(0, 1200, size=2400)],                      # a's other half new, first half known
            [(k, row()) for k in rng.permutation(b * 3 + pair * 2).tolist()],                    # new ids of one tag inside one batch
            [(k, None) for k in a[::7] + b[::5]] + [(k, row()) for k in a[::11]],               # tombstones, then rewrites
        ]
        ids, table = [], np.zeros((0, e.state_bytes), np.uint8)
        for batch in batches:
            ids, table, n_new = PB.put_batch(ids, table, batch)
            rows = np.zeros((len(batch), user), np.uint8)
            for i, (_, v) in enumerate(batch):
                if v is not None:
                    rows[i] = np.frombuffer(v, np.uint8)
            assert e.put_batch([k for k, _ in batch], rows, [v is not None for _, v in batch]) == n_new
            assert np.array_equal(e.export_states(), table)
            assert e.get_many(ids, arrays=True)[2].tolist() == list(range(len(ids)))
            fl = table[:, user:user + 4].copy().view("<u4").ravel()
            changes = {}
            for _, f, _, r, kids in e.export_changes(N.ST_CHANGED | N.ST_ERROR, page_rows=211):
                changes.update({k: (int(f[i]), r[i].tobytes()) for i, k in enumerate(kids)})
            assert changes == {k: (int(fl[i]), table[i, :user].tobytes()) for i, k in enumerate(ids) if fl[i] & (N.ST_CHANGED | N.ST_ERROR)}
            assert _scan_ids(e) == sorted((k for i, k in enumerate(ids) if fl[i] & N.ST_EXISTS), key=str.encode)
        assert e.get_many(_s(H.cluster(4, b"pb-", seed=56)), arrays=True)[2].tolist() == [-1] * 4


# ------------------------------------------------------------------ polls after a full device dictionary
def _state_batch(base, ids, rng):
    return K.encode_record_batch(base, [(d, k.encode(), struct.pack("<ii", int(rng.integers(-99, 99)), d)) for d, k in enumerate(ids)],
                                 compression="lz4")


def _event_batch(base, ids, rng, seq):
    return K.encode_record_batch(base, [(d, f"{k}:{seq + d}".encode(), _ev(0, seq + d, int(rng.integers(1, 9)))) for d, k in enumerate(ids)],
                                 compression="lz4")


@pytest.mark.parametrize("bound", ["max_keys", "max_id_bytes"])
@pytest.mark.parametrize("topic", ["events", "state"])
def test_polls_after_a_full_dictionary(topic, bound):
    rng = np.random.default_rng(61 + (topic == "state") + 2 * (bound == "max_keys"))
    cl = _s(H.cluster(160, b"full-" + topic[:1].encode(), seed=62))      # 24-byte ids: 24 arena bytes each
    first, over, fresh = cl[:30], cl[30:130], cl[130:]
    max_keys, max_bytes = (64, 1 << 20) if bound == "max_keys" else (1 << 12, 24 * 64 + 20)
    admitted_max = 64                                                   # either bound admits 64 ids
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        user = e.state_bytes - 8
        with DeviceIngest(e, max_keys, max_bytes) as dg:
            if topic == "state":
                dg.set_state_topic(True)
            off, seq, good = 0, 1, []                                   # good: the fetches of the polls that folded

            def poll(ids, expect_ok):
                """one partition, one fetch of several batches: the fold's stats, or None when it fails with SGR_ERR_CAPACITY"""
                nonlocal off, seq
                data, base = bytearray(), off
                for i in range(0, len(ids), 40):
                    chunk = ids[i:i + 40]
                    data += _state_batch(base, chunk, rng) if topic == "state" else _event_batch(base, chunk, rng, seq)
                    base += len(chunk)
                    seq += len(chunk)
                dg.submit(0, bytes(data))
                try:
                    st = dg.fold()
                except IngestError as ex:
                    assert not expect_ok, str(ex)
                    assert ex.code == N.SGR_ERR_CAPACITY
                    assert dg.offsets(0) == (off, off)
                    return None
                assert expect_ok
                good.append((0, bytes(data), []))
                off = base
                return st

            def want():
                if topic == "state":
                    recs, _, _ = S.read_committed_states(good, S.PACKED, user)
                    ids, table = S.apply([], np.zeros((0, e.state_bytes), np.uint8), recs)
                    return {k: table[i, :user].tobytes() for i, k in enumerate(ids)}
                ing = Ingest()
                with ReplayEngine(0) as h:
                    h.register_program(P.counter_program())
                    for p, d, _ in good:
                        ing.record_batches(p, d)
                    h.fold_ingested(ing)
                    return {k: h.get(k) for k in ing.keys()}

            # 1: a good poll
            assert poll(first * 2, True)["n_new_keys"] == 30
            before = e.get_many(first)
            # 2: 100 new ids of one tag: all race for the last 34 places; refused slots sit among admitted ones
            assert poll(over * 3 + first, False) is None
            assert e.get_many(first) == before
            # 3: known ids only: folds exactly; the ids step 2 admitted become visible, and only those
            st = poll(first, True)
            _, _, idx = e.get_many(over, arrays=True)
            resolved = [k for k, i in zip(over, idx.tolist()) if i >= 0]
            assert st["n_new_keys"] == len(resolved) == admitted_max - 30
            all_idx = e.get_many(first, arrays=True)[2].tolist() + [i for i in idx.tolist() if i >= 0]
            assert sorted(all_idx) == list(range(admitted_max))          # every dense index holds an id that arrived
            assert e.get_many(fresh, arrays=True)[2].tolist() == [-1] * len(fresh)
            w = want()
            assert {k: e.get(k) for k in w} == w
            # 3b: the admitted ids of step 2, wherever they sit in the chain, are known: a poll of them folds
            st = poll(resolved * 2 + first, True)
            assert st["n_new_keys"] == 0
            w = want()
            assert {k: e.get(k) for k in w} == w and sorted(w) == sorted(first + resolved)
            assert _scan_ids(e) == sorted(w, key=str.encode)
            # 4: a new id fails again, and so does an id step 2 refused; nothing is applied
            refused = [k for k in over if k not in set(resolved)]
            assert poll(first + fresh[:1], False) is None
            assert poll(refused[:1] + resolved[:5], False) is None
            assert {k: e.get(k) for k in w} == w
            # 5: after a reset the whole capacity is back
            dg.reset()
            e.set_initial_states(None)
            off, good = 0, []
            assert poll(cl[:admitted_max], True)["n_new_keys"] == admitted_max
            w = want()
            assert {k: e.get(k) for k in w} == w
            assert poll(cl[admitted_max:admitted_max + 1], False) is None
