"""-m gpu: the changed-state export (sgr_export_changes, csrc/changes.cu). Its pages, concatenated, hold exactly the rows of
export_states whose flags meet the selection, in ascending dense index, with the key table's ids: after every fold path, for
16-, 64- and 128-byte states with throwing events, under every page cut by rows and by id bytes, across table generations, and
through the store's on_changes listener."""
import ctypes as C
import struct

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import program_corpus as PC
from oracle import program_interp as I
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest
from surge_b200.store import GpuReplayKeyValueStore

pytestmark = pytest.mark.gpu

TILE = 1024   # kChangesTile (csrc/changes.cuh)
CHANGED_OR_ERROR = N.ST_CHANGED | N.ST_ERROR

COUNTER = [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)]), (I.MATERIALISE, [(I.OP_SUB_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)]),
           (I.MATERIALISE, []), (I.THROW, [])]
BANK = [(I.CREATE, [(I.OP_SET, 0, 16, 16), (I.OP_SET, 16, 32, 8), (I.OP_SET, 24, 40, 16), (I.OP_SET, 40, 56, 8)]),
        (I.IF_EXISTS, [(I.OP_SET, 16, 32, 8)]), (I.TOMBSTONE, []), (I.THROW, [])]
ROW30 = PC.row_program(np.random.default_rng(7), 30, 0, 9)
PROGRAMS = [("counter", 16, COUNTER), ("bank_account", 64, BANK), ("row_128", 128, ROW30)]


def special_ids(n, seed):
    """n distinct ids: "", non-ASCII UTF-8, ids over 256 bytes, ids whose length is a multiple of 8, plain ones."""
    rng = np.random.default_rng(seed)
    ids = ["", "x", "é", "日本語-id", "agg-0" * 60, ("long" * 80) + "a", "eight-by", "sixteen-bytes-id", "ÿĀ"]
    ids += [f"agg-{i}-{int(rng.integers(0, 1 << 30))}" + "z" * int(rng.integers(0, 12)) for i in range(n - len(ids))]
    assert len(set(ids)) == len(ids)
    return ids[:n]


def expected(e, keys, select):
    """(indices, flags, err_idx, rows, ids) of the rows of export_states that `select` picks, with ids from `keys`."""
    sb = e.state_bytes
    table = e.export_states()
    words = table[:, sb - 8:sb].copy().view(np.uint32)
    fl, err = words[:, 0], words[:, 1]
    idx = np.nonzero(fl & select)[0].astype(np.int64)
    rows = table[idx, :sb - 8].copy()
    rows[(fl[idx] & N.ST_EXISTS) == 0] = 0
    ids = [keys[i] if i < len(keys) else None for i in idx]
    return idx, fl[idx], err[idx], rows, ids


def exported(e, select=N.ST_CHANGED, page_rows=None, page_id_bytes=64 << 20):
    pages = list(e.export_changes(select, page_rows, page_id_bytes))
    if not pages:
        return np.zeros(0, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros((0, e.state_bytes - 8), np.uint8), [], []
    cat = [np.concatenate([p[k] for p in pages]) for k in range(4)]
    return (*cat, [k for p in pages for k in p[4]], [len(p[0]) for p in pages])


def check(e, keys, select=N.ST_CHANGED, what="", **page):
    want = expected(e, keys, select)
    got = exported(e, select, **page)
    assert np.array_equal(got[0], want[0]), what
    assert np.array_equal(got[1], want[1]), what
    assert np.array_equal(got[2], want[2]), what
    assert np.array_equal(got[3], want[3]), what
    assert got[4] == want[4], what
    return want, got[5]


def check_all_selections(e, keys, what=""):
    for sel in (N.ST_CHANGED, N.ST_ERROR, CHANGED_OR_ERROR):
        check(e, keys, sel, f"{what} select {sel}")
    return expected(e, keys, CHANGED_OR_ERROR)


def fixed_log(rules, n_agg, seed, p_throw=0.02):
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 12, size=n_agg).astype(np.int64)
    buf, seg, _ = PC.fixed_log(rng, rules, counts, p_throw=p_throw)
    return buf, seg


# ------------------------------------------------------------------ every fold path
@pytest.mark.parametrize("name,sb,rules", PROGRAMS, ids=[p[0] for p in PROGRAMS])
def test_full_fold_kernels(name, sb, rules):
    ids = special_ids(5000, 1)
    buf, seg = fixed_log(rules, len(ids), 2)
    kernels = (0, 1, 2, 3) if name == "counter" else (0, 1, 2)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, rules))
        e.load_keys(ids)
        e.load_events(buf, seg)
        ran = 0
        for k in kernels:
            e.set_option("kernel", k)
            e.set_initial_states(None)
            try:
                e.fold()
            except SgrError as ex:   # a forced kernel that cannot take this program
                assert ex.code == N.SGR_ERR_UNSUPPORTED and k >= 2
                continue
            ran += 1
            _, fl, _, _, _ = check_all_selections(e, ids, f"{name} kernel {k}")
            assert (fl & N.ST_ERROR).any() and (fl & N.ST_CHANGED).any()
            e.fold()                                                         # the same log again, onto its own output
            check_all_selections(e, ids, f"{name} kernel {k}, second fold")
        assert ran >= 2


def test_bank_account_tombstones_are_reported_as_zero_rows():
    ids = special_ids(3000, 3)
    rng = np.random.default_rng(4)
    counts = rng.integers(1, 6, size=len(ids)).astype(np.int64)
    buf, seg, _ = PC.fixed_log(rng, BANK, counts, p_throw=0.02)
    for a in range(len(ids)):
        PC.set_type(buf, seg, a, 0, 0)                                      # first event: CREATE
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(64, N.REC_FIXED64, BANK))
        e.load_keys(ids)
        e.load_events(buf, seg)
        e.fold()
        for a in range(0, len(ids), 3):
            PC.set_type(buf, seg, a, -1, 2)                                 # last event: TOMBSTONE
        e.load_events(buf, seg)
        e.fold()                                                            # from the live states: existing ones become None
        idx, fl, _, rows, _ = check_all_selections(e, ids, "bank")
        tomb = ((fl & N.ST_CHANGED) != 0) & ((fl & N.ST_EXISTS) == 0)
        assert tomb.any() and not rows[tomb].any()


def test_variable_records_vruns():
    rng = np.random.default_rng(5)
    rules = PC.row_program(rng, 2, 0, 3)
    counts = rng.integers(0, 20, size=6000).astype(np.int64)
    buf, seg, rec_off = PC.var_log(rng, rules, counts, 200, p_throw=0.01)
    ids = special_ids(6000, 6)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_VAR16, rules))
        e.load_keys(ids)
        e.load_events_indexed(buf, seg, rec_off)
        e.fold()
        _, fl, _, _, _ = check_all_selections(e, ids, "vruns")
        assert (fl & N.ST_ERROR).any()


@pytest.mark.parametrize("name,sb,rules,bulk", [("counter", 16, COUNTER, 1), ("counter", 16, COUNTER, 0), ("bank_account", 64, BANK, 1)],
                         ids=["counter-bulk", "counter-micro-batch", "bank-grouped"])
def test_fold_unsorted(name, sb, rules, bulk):
    ids = special_ids(4000, 7)
    rng = np.random.default_rng(8)
    buf, _, aggs = PC.fixed_log(rng, rules, rng.integers(0, 12, size=len(ids)).astype(np.int64), p_throw=0.02)
    arrival = np.ascontiguousarray(buf[PC.interleave(rng, aggs)])
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, rules))
        e.set_option("bulk", bulk)
        e.load_keys(ids)
        e.fold_unsorted(arrival, len(ids))
        _, fl, _, _, _ = check_all_selections(e, ids, f"unsorted {name} bulk {bulk}")
        assert (fl & N.ST_ERROR).any()


def _batch(rng, aggs, rules, p_throw=0.05):
    """Records for `aggs` with the program's non-throwing types, and about p_throw of them with type 255 (no rule: a MatchError)."""
    rec = rng.integers(0, 256, size=(len(aggs), 64), dtype=np.uint8)
    ok = np.array([t for t, (ex, _) in enumerate(rules) if ex != I.THROW], dtype=np.uint32)
    t = ok[rng.integers(0, len(ok), size=len(aggs))]
    t[rng.random(len(aggs)) < p_throw] = 255
    rec[:, 0:4] = t.view(np.uint8).reshape(-1, 4)
    rec[:, 4:8] = np.arange(1, len(aggs) + 1, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
    rec[:, 8:16] = np.asarray(aggs, dtype=np.uint64).view(np.uint8).reshape(-1, 8)
    return rec


@pytest.mark.parametrize("name,sb,rules,incremental", [("counter", 16, COUNTER, 0), ("counter", 16, COUNTER, 1), ("bank_account", 64, BANK, 0),
                                                        ("row_128", 128, ROW30, 0)],
                         ids=["counter-atomic", "counter-sorted", "bank-sorted", "row128-sorted"])
def test_fold_incremental_sequences(name, sb, rules, incremental):
    """Each batch touches a subset of the previous one's aggregates: a flag the fold failed to clear would show."""
    n = 5000
    ids = special_ids(n, 10)
    rng = np.random.default_rng(11)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, rules))
        e.set_option("incremental", incremental)
        e.load_keys(ids)
        e.set_initial_states(np.zeros((n, sb), np.uint8))
        touched = np.arange(n)
        for step in range(5):
            touched = np.sort(rng.choice(touched, size=max(len(touched) // 3, 1), replace=False)) if step else touched
            aggs = rng.choice(touched, size=3 * len(touched))
            e.fold_incremental(_batch(rng, aggs, rules))
            idx, fl, _, _, _ = check_all_selections(e, ids, f"{name} incremental step {step}")
            assert set(idx.tolist()) <= set(touched.tolist())


# ------------------------------------------------------------------ ingest paths and the store
def _ev(t, seq, by=0):
    return struct.pack("<IIi", t, seq, by)


def _poll(rng, base, n_batches, key_lo, key_hi, p_throw=0.03):
    out, off = bytearray(), base
    for _ in range(n_batches):
        n = int(rng.integers(1, 40))
        recs = []
        for d in range(n):
            k = int(rng.integers(key_lo, key_hi))
            t = 3 if rng.random() < p_throw else int(rng.integers(0, 3))
            recs.append((d, f"acc-{k}:{off + d}".encode() if k % 7 else f"é-{k}".encode(), _ev(t, off + d, int(rng.integers(0, 1000)))))
        out += K.encode_record_batch(off, recs, compression="lz4")
        off += n
    return bytes(out), off


def test_fold_ingested_polls():
    rng = np.random.default_rng(21)
    ing = Ingest()
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        off = 0
        for p in range(5):
            data, off = _poll(rng, off, 30, 200 * p, 200 * p + 600)          # later polls reuse part of the earlier keys
            ing.record_batches(0, data)
            e.fold_ingested(ing)
            keys = ing.keys()
            idx, fl, _, _, ids = check_all_selections(e, keys, f"ingest poll {p}")
            assert len(idx) and all(k is not None for k in ids[:np.searchsorted(idx, len(keys))])


def test_device_ingest_polls():
    rng = np.random.default_rng(22)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1 << 16) as dg:
            off = 0
            for p in range(4):
                data, off = _poll(rng, off, 30, 300 * p, 300 * p + 700)
                dg.submit(0, data)
                dg.fold()
                # the engine's key table is the device dictionary: the exported ids are checked through get_many's indices
                want = expected(e, [], CHANGED_OR_ERROR)
                got = exported(e, CHANGED_OR_ERROR, page_rows=777)
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
                assert np.array_equal(got[3], want[3])
                known = [k for k in got[4] if k is not None]
                _, _, idx = e.get_many(known, arrays=True)
                assert np.array_equal(idx, got[0][:len(known)]) and len(known) > 0
                assert all(k.startswith(("acc-", "é-")) for k in known)


def test_store_put_event_path_across_growth():
    rng = np.random.default_rng(23)
    calls = []
    st = GpuReplayKeyValueStore("s", P.counter_program(), on_changes=lambda ch, fa: calls.append((ch, fa)))
    st.init()
    ids = special_ids(3000, 24)
    ids.remove("")
    live = 50
    for r in range(6):
        live = min(len(ids), live * 3)                    # new ids every round: the table grows (1024, 2 x ids, ...)
        picked = set()
        for i in rng.integers(0, live, size=2000):
            rec = bytearray(64)
            rec[0:4] = struct.pack("<I", 3 if rng.random() < 0.02 else int(rng.integers(0, 3)))
            rec[4:8] = struct.pack("<I", r + 1)
            rec[16:20] = struct.pack("<i", int(rng.integers(1, 100)))
            st.put_event(f"{ids[i]}:{r}", bytes(rec))
            picked.add(ids[i])
        before = {k: st.get(k) if r else None for k in picked}
        st.flush()
        assert len(calls) == r + 1
        changed, failed = calls[-1]
        e = st.engine
        want = expected(e, st._keys, CHANGED_OR_ERROR)
        keys = {k for k, _ in changed} | {k for k, _ in failed}
        assert keys <= picked
        assert [k for k, _ in changed] == [want[4][j] for j in range(len(want[0])) if want[1][j] & N.ST_CHANGED]
        assert [k for k, _ in failed] == [want[4][j] for j in range(len(want[0])) if want[1][j] & N.ST_ERROR]
        for k, v in changed:
            assert v == st.get(k) and v != before[k]
        for k, err_idx in failed:
            assert st.get(k) == before[k]
            assert isinstance(err_idx, int)
        assert not any(k.startswith("\0unused") for k in keys)
    st.flush()                                            # nothing pending: no fold, no call
    assert len(calls) == 6
    st.close()


def test_store_codec_tombstones_and_ingest_store():
    """Through a codec, a delete() reaches the listener as (id, None); a store fed record batches reports the ingest's ids."""
    from surge_b200.store import StateCodec

    calls = []
    codec = StateCodec(lambda k, v: v[:8].ljust(8, b"\0"), lambda k, b: b"S" + b, 4, 5)
    st = GpuReplayKeyValueStore("c", P.counter_program_with_snapshot_rules(), codec=codec, on_changes=lambda ch, fa: calls.append((ch, fa)))
    st.init()
    st.put("a", b"12345678")
    st.put("b", b"abcdefgh")
    st.flush()
    assert sorted(calls[-1][0]) == [("a", b"S12345678"), ("b", b"Sabcdefgh")] and calls[-1][1] == []
    st.delete("a")
    st.flush()
    assert calls[-1] == ([("a", None)], [])
    assert st.get("a") is None
    st.close()

    calls.clear()
    st2 = GpuReplayKeyValueStore("i", P.counter_program(), on_changes=lambda ch, fa: calls.append((ch, fa)))
    st2.init()
    rng = np.random.default_rng(25)
    data, _ = _poll(rng, 0, 20, 0, 300)
    st2.restore_record_batches(0, data)
    st2.flush()
    changed, failed = calls[-1]
    assert changed and all(st2.get(k) == v for k, v in changed)
    want = expected(st2.engine, st2._ingest.keys(), CHANGED_OR_ERROR)
    assert [k for k, _ in failed] == [want[4][j] for j in range(len(want[0])) if want[1][j] & N.ST_ERROR]
    assert [(k, e) for k, e in failed] == [(want[4][j], int(want[2][j])) for j in range(len(want[0])) if want[1][j] & N.ST_ERROR]
    st2.close()


# ------------------------------------------------------------------ paging
def _table(n, sb, seed, p_changed=0.3, p_error=0.05):
    """A random state table with flags: CHANGED and ERROR on random rows, EXISTS on most."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 256, size=(n, sb), dtype=np.uint8)
    fl = (rng.random(n) < 0.8).astype(np.uint32) * N.ST_EXISTS
    fl |= (rng.random(n) < p_changed).astype(np.uint32) * N.ST_CHANGED
    fl |= (rng.random(n) < p_error).astype(np.uint32) * N.ST_ERROR
    t[:, sb - 8:sb - 4] = fl.view(np.uint8).reshape(-1, 4)
    t[(fl & N.ST_EXISTS) == 0, :sb - 8] = 0
    return t


@pytest.mark.parametrize("page_rows", [1, 7, TILE - 1, TILE, TILE + 1, None])
def test_page_rows(page_rows):
    n = 3 * TILE + 517
    ids = special_ids(n, 30)
    with ReplayEngine(0) as e:
        e.register_program(P.bank_account_program())
        e.load_keys(ids)
        e.set_initial_states(_table(n, 64, 31, p_changed=0.6))
        want, sizes = check(e, ids, CHANGED_OR_ERROR, page_rows=page_rows)
        if page_rows is not None:
            assert all(s == page_rows for s in sizes[:-1]) and 0 < sizes[-1] <= page_rows
        else:
            assert sizes == [len(want[0])]


@pytest.mark.parametrize("cap", [330, 999, 4096, 30_000])
def test_id_byte_caps_cut_inside_tiles(cap):
    n = 4 * TILE + 3
    ids = special_ids(n, 32)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(ids)
        e.set_initial_states(_table(n, 16, 33, p_changed=0.9))
        want, sizes = check(e, ids, N.ST_CHANGED, page_id_bytes=cap)
        # every page is as full as the next id allows
        lens = [len(k.encode()) for k in want[4]]
        pos = 0
        for s in sizes:
            used = sum(lens[pos:pos + s])
            assert used <= cap
            if pos + s < len(lens):
                assert used + lens[pos + s] > cap
            pos += s


@pytest.mark.parametrize("n", [TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE + 1, 1])
def test_table_sizes_around_the_tile(n):
    ids = special_ids(max(n, 12), 34)[:n]
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(ids)
        t = _table(n, 16, 35, p_changed=0.5)
        t[-1, 8:12] = np.frombuffer(np.uint32(N.ST_EXISTS | N.ST_CHANGED).tobytes(), np.uint8)   # the last row is selected
        e.set_initial_states(t)
        for pr in (None, 3, TILE):
            want, _ = check(e, ids, N.ST_CHANGED, f"n {n} page_rows {pr}", page_rows=pr)
            assert want[0][-1] == n - 1


def test_rows_past_the_key_table_and_no_key_table():
    n = 2 * TILE + 10
    with ReplayEngine(0) as e:
        e.register_program(P.bank_account_program())
        e.set_initial_states(_table(n, 64, 36, p_changed=0.5))
        want, _ = check(e, [], CHANGED_OR_ERROR, page_rows=500)                     # no key table: every id is None
        assert want[4] and all(k is None for k in want[4])
        ids = special_ids(TILE + 5, 37)
        e.load_keys(ids)
        want, _ = check(e, ids, CHANGED_OR_ERROR, page_rows=333, page_id_bytes=2000)
        assert any(k is None for k in want[4]) and any(k is not None for k in want[4])
        pages = list(e.export_changes(CHANGED_OR_ERROR, 100))
        assert all(p[4][j] is None for p in pages for j in range(len(p[0])) if p[0][j] >= len(ids))


def test_special_ids_round_trip():
    ids = special_ids(2000, 38)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(ids)
        t = _table(len(ids), 16, 39, p_changed=0.2)
        t[:12, 8:12] = np.frombuffer(np.uint32(N.ST_CHANGED).tobytes(), np.uint8)   # the special ones are all reported
        e.set_initial_states(t)
        for cap in (330, 1 << 20):                                  # (the longest id is 321 bytes)
            want, _ = check(e, ids, N.ST_CHANGED, page_rows=5, page_id_bytes=cap)
            assert want[4][:9] == ids[:9]


# ------------------------------------------------------------------ errors and table generations
def _raw(e, cur, select=N.ST_CHANGED, max_rows=64, ids_cap=4096):
    user = e.state_bytes - 8
    bufs = dict(rows=np.full(max_rows * user, 0xAB, np.uint8), flags=np.full(max_rows, 0xABABABAB, np.uint32),
                err=np.full(max_rows, 0xABABABAB, np.uint32), idx=np.full(max_rows, -7, np.int64),
                ids=np.full(max(ids_cap, 1), 0xAB, np.uint8), offs=np.full(max_rows + 1, 0xABABABAB, np.uint32))
    n = C.c_uint64(12345)
    rc = e._lib.sgr_export_changes(e._h, select, C.byref(cur), max_rows, bufs["rows"].ctypes.data, bufs["flags"].ctypes.data, bufs["err"].ctypes.data,
                                   bufs["idx"].ctypes.data, bufs["ids"].ctypes.data, ids_cap, bufs["offs"].ctypes.data, C.byref(n))
    return rc, bufs, n.value


def _untouched(bufs, n):
    return n == 12345 and (bufs["rows"] == 0xAB).all() and (bufs["idx"] == -7).all() and (bufs["ids"] == 0xAB).all() and (bufs["offs"] == 0xABABABAB).all()


def test_argument_errors_and_capacity():
    ids = ["short", "x" * 500, "y"] + [f"k{i}" for i in range(3000)]
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(ids)
        rc, bufs, n = _raw(e, N.sgr_changes_cursor())
        assert rc == N.SGR_ERR_STATE and _untouched(bufs, n)
        with pytest.raises(N.InvalidStateStoreException):
            list(e.export_changes())
        t = _table(len(ids), 16, 40, p_changed=0.0)
        t[:3, 8:12] = np.frombuffer(np.uint32(N.ST_CHANGED | N.ST_EXISTS).tobytes(), np.uint8)
        e.set_initial_states(t)
        for sel in (0, 8, N.ST_EXISTS, N.ST_CHANGED | 8):
            assert _raw(e, N.sgr_changes_cursor(), select=sel)[0] == N.SGR_ERR_INVALID
        assert _raw(e, N.sgr_changes_cursor(), max_rows=0)[0] == N.SGR_ERR_INVALID
        cur = N.sgr_changes_cursor()
        cur.next = len(ids) + 1
        assert _raw(e, cur)[0] == N.SGR_ERR_INVALID
        cur.next = len(ids)                                              # at the end: an empty, complete page
        rc, bufs, n = _raw(e, cur)
        assert rc == 0 and n == 0 and cur.next == len(ids)
        # the second row's id (500 bytes) alone is past the cap: the first page stops before it, the next one is refused
        cur = N.sgr_changes_cursor()
        rc, bufs, n = _raw(e, cur, ids_cap=100)
        assert rc == 0 and n == 1 and cur.next == 1 and bufs["ids"][:5].tobytes() == b"short"
        saved = (cur.next, cur.token, cur.n_keys)
        rc, bufs, n = _raw(e, cur, ids_cap=100)
        assert rc == N.SGR_ERR_CAPACITY and _untouched(bufs, n) and (cur.next, cur.token, cur.n_keys) == saved
        rc, bufs, n = _raw(e, cur, ids_cap=501)                          # the same export goes on with a larger buffer
        assert rc == 0 and n == 2 and cur.next == len(ids) and list(bufs["idx"][:2]) == [1, 2]


def test_a_new_generation_between_pages_is_refused():
    n = 3 * TILE
    ids = special_ids(n, 41)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(ids)
        t = _table(n, 16, 42, p_changed=0.5)
        e.set_initial_states(t)
        rec = _batch(np.random.default_rng(43), np.arange(0, n, 5), COUNTER)

        def second_page_after(action):
            cur = N.sgr_changes_cursor()
            rc, _, k = _raw(e, cur, max_rows=100)
            assert rc == 0 and k == 100 and cur.token != 0
            action()
            rc, bufs, k = _raw(e, cur, max_rows=100)
            return rc, bufs, k

        rc, bufs, k = second_page_after(lambda: e.get_many(ids[:500]))
        assert rc == 0 and k == 100
        rc, bufs, k = second_page_after(lambda: e.get(ids[3]))
        assert rc == 0 and k == 100
        owner_keys = list(ids)
        rc, bufs, k = second_page_after(lambda: e.fold_incremental(rec))
        assert rc == N.SGR_ERR_STATE and _untouched(bufs, k)
        rc, bufs, k = second_page_after(lambda: e.load_keys(owner_keys))
        assert rc == N.SGR_ERR_STATE and _untouched(bufs, k)
        rc, bufs, k = second_page_after(lambda: e.grow_states(n + 10))
        assert rc == N.SGR_ERR_STATE and _untouched(bufs, k)
        rc, bufs, k = second_page_after(lambda: e.set_initial_states(t))
        assert rc == N.SGR_ERR_STATE and _untouched(bufs, k)
        gen = e.export_changes(N.ST_CHANGED, page_rows=10)
        next(gen)
        e.fold_incremental(rec)
        with pytest.raises(N.InvalidStateStoreException):
            next(gen)


def test_appended_ids_do_not_end_an_export_and_a_routed_engine_is_refused():
    owner = C.c_void_p(0x99)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.grow_states(4000)
        e.set_initial_states(_table(4000, 16, 44, p_changed=0.5))

        def append(keys):
            enc = [k.encode() for k in keys]
            offs = np.zeros(len(enc) + 1, dtype=np.uint32)
            np.cumsum([len(b) for b in enc], out=offs[1:])
            blob = np.frombuffer(b"".join(enc), dtype=np.uint8)
            assert e._lib.sgr_append_keys(e._h, owner, blob.ctypes.data, offs.ctypes.data, len(enc)) == 0

        ids = [f"a-{i}" for i in range(4000)]
        append(ids[:1000])
        cur = N.sgr_changes_cursor()
        rc, bufs, k = _raw(e, cur, max_rows=200, ids_cap=1 << 16)
        assert rc == 0 and cur.n_keys == 1000
        append(ids[1000:])
        got = [int(i) for i in bufs["idx"][:k]]
        while cur.next < 4000:
            rc, bufs, k = _raw(e, cur, max_rows=700, ids_cap=1 << 16)
            assert rc == 0 and cur.n_keys == 4000
            got += [int(i) for i in bufs["idx"][:k]]
        assert got == expected(e, ids, N.ST_CHANGED)[0].tolist()
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.dist_init(0, 1, None, 1024)
        assert _raw(e, N.sgr_changes_cursor())[0] == N.SGR_ERR_UNSUPPORTED


# ------------------------------------------------------------------ scale
def test_scale_two_to_the_24_plus_3():
    n = (1 << 24) + 3
    rng = np.random.default_rng(45)
    blob = np.empty((n, 12), dtype=np.uint8)      # id i = its 12 decimal digits
    v = np.arange(n, dtype=np.int64)
    for d in range(11, -1, -1):
        blob[:, d] = v % 10 + ord("0")
        v //= 10
    offs = (np.arange(n + 1, dtype=np.uint64) * 12).astype(np.uint32)
    states = np.zeros((n, 16), dtype=np.uint8)
    states[:, :8] = rng.integers(0, 256, size=(n, 8), dtype=np.uint8)
    fl = np.full(n, N.ST_EXISTS, dtype=np.uint32)
    pick = rng.random(n) < 0.01
    pick[-1] = True
    fl[pick] |= N.ST_CHANGED
    fl[rng.random(n) < 0.001] |= N.ST_ERROR
    states[:, 8:12] = fl.view(np.uint8).reshape(-1, 4)
    states[:, 12:16] = rng.integers(0, 1 << 31, size=n, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        assert e._lib.sgr_load_keys(e._h, blob.ctypes.data, offs.ctypes.data, n) == 0
        e.set_initial_states(states)
        for sel in (N.ST_CHANGED, CHANGED_OR_ERROR):
            want = np.nonzero(fl & sel)[0]
            for page_rows in (None, 50_000):
                cur, got_idx, got_rows, got_err, got_ids = N.sgr_changes_cursor(), [], [], [], []
                cap = len(want) if page_rows is None else page_rows
                while True:
                    rows = np.zeros((cap, 8), np.uint8)
                    f, er = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
                    ix = np.zeros(cap, np.int64)
                    ib = np.zeros(cap * 12, np.uint8)
                    io = np.zeros(cap + 1, np.uint32)
                    k = C.c_uint64()
                    rc = e._lib.sgr_export_changes(e._h, sel, C.byref(cur), cap, rows.ctypes.data, f.ctypes.data, er.ctypes.data, ix.ctypes.data,
                                                   ib.ctypes.data, ib.nbytes, io.ctypes.data, C.byref(k))
                    assert rc == 0, e._lib.sgr_last_error(e._h)
                    k = k.value
                    got_idx.append(ix[:k]); got_rows.append(rows[:k]); got_err.append(er[:k])
                    assert np.array_equal(io[:k + 1], np.arange(k + 1, dtype=np.uint32) * 12)
                    got_ids.append(ib[:12 * k].reshape(-1, 12))
                    if cur.next == n:
                        break
                gi = np.concatenate(got_idx)
                assert np.array_equal(gi, want)
                assert np.array_equal(np.concatenate(got_rows), states[want, :8])
                assert np.array_equal(np.concatenate(got_err), states[want, 12:16].copy().view(np.uint32).ravel())
                assert np.array_equal(np.concatenate(got_ids), blob[want])
