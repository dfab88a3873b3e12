"""-m gpu: the ordered scan (sgr_scan, csrc/id_order.cu + csrc/changes.cu). Its pages, concatenated, hold exactly the live rows
(SGR_ST_EXISTS) of the key table's ids in Bytes order, with the rows, flags and indices get_many returns for them: for id
families that stress the 8-byte windows of the sort, under every bound and page cut, while the order is extended by appended
ids and rebuilt for new key tables, and at millions of ids. The oracle orders ids with Python's bytes comparison."""
import ctypes as C
import struct
import time

import numpy as np
import pytest

from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest
from surge_b200.store import GpuReplayKeyValueStore

pytestmark = pytest.mark.gpu

TILE = 1024   # kChangesTile (csrc/changes.cuh)


def bkey(s):
    return s.encode("utf-8")


def oracle(ids):
    return sorted(ids, key=bkey)


def uuids(rng, n):
    h = np.frombuffer(b"0123456789abcdef", np.uint8)[rng.integers(0, 16, size=(n, 32))]
    out = np.full((n, 36), ord("-"), np.uint8)
    for dst, src in ((slice(0, 8), slice(0, 8)), (slice(9, 13), slice(8, 12)), (slice(14, 18), slice(12, 16)), (slice(19, 23), slice(16, 20)),
                     (slice(24, 36), slice(20, 32))):
        out[:, dst] = h[:, src]
    ids = [bytes(r).decode() for r in out]
    return list(dict.fromkeys(ids))


def accounts(n, start=0):
    return [f"account-{i:012d}" for i in range(start, start + n)]


def special_ids():
    """Ids that stress the windows: every length 0..300, prefixes of each other, \\0 bytes, a last byte that differs at 8, 16 and 24
    bytes, bytes >= 0x80 and UTF-8 sequences of up to 4 bytes."""
    rng = np.random.default_rng(3)
    ids = ["", "a", "a\0", "a\0\0", "ab", "a\0b", "\0", "\0\0", "\x7f", "\x80", "ÿ", "é", "日本語", "𝄞", "𝄞𝄞", "a𝄞", "😀-id", "\U0010ffff"]
    ids += ["p" * L for L in range(1, 301)]                                    # prefixes of each other, every length
    ids += ["".join(chr(int(c)) for c in rng.integers(97, 100, size=L)) for L in range(0, 301)]
    for L in (8, 16, 24):
        base = "w" * (L - 1)
        ids += [base + c for c in "\0ABz~\x7fé"] + [base, base + "z\0", base + "zz"]
    ids += ["k" * 8 + "\0" * 8, "k" * 8 + "\0" * 7, "k" * 8 + "\0" * 9, "k" * 8, "k" * 16 + "\0"]
    return list(dict.fromkeys(ids))


def table(n, sb, seed, p_exists=0.8, p_error=0.05):
    """A random state table: EXISTS on most rows, ERROR on some (with and without EXISTS), program bytes zero when None."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 256, size=(n, sb), dtype=np.uint8)
    fl = (rng.random(n) < p_exists).astype(np.uint32) * N.ST_EXISTS
    fl |= (rng.random(n) < p_error).astype(np.uint32) * N.ST_ERROR
    fl |= (rng.random(n) < 0.3).astype(np.uint32) * N.ST_CHANGED
    t[:, sb - 8:sb - 4] = fl.view(np.uint8).reshape(-1, 4)
    t[(fl & N.ST_EXISTS) == 0, :sb - 8] = 0
    return t


def scanned(e, frm=None, to=None, page_rows=1 << 20, page_id_bytes=64 << 20):
    pages = list(e.scan(frm, to, page_rows, page_id_bytes))
    if not pages:
        return np.zeros(0, np.int64), np.zeros(0, np.uint32), np.zeros((0, e.state_bytes - 8), np.uint8), [], []
    return (np.concatenate([p[0] for p in pages]), np.concatenate([p[1] for p in pages]), np.concatenate([p[2] for p in pages]),
            [k for p in pages for k in p[3]], [len(p[0]) for p in pages])


def live_ids(e, keys):
    """The keys whose row exists, in oracle order (rows at or past n_agg do not exist)."""
    t = e.export_states()
    fl = t[:, e.state_bytes - 8:e.state_bytes - 4].copy().view(np.uint32).ravel()
    return oracle([k for i, k in enumerate(keys) if i < len(fl) and fl[i] & N.ST_EXISTS])


def check(e, keys, frm=None, to=None, what="", **page):
    """The scan equals the oracle over `keys`, and its rows, flags and indices equal get_many's."""
    want = [k for k in live_ids(e, keys) if (frm is None or bkey(frm) <= bkey(k)) and (to is None or bkey(k) <= bkey(to))]
    idx, fl, rows, ids, sizes = scanned(e, frm, to, **page)
    assert ids == want, what
    if want:
        g_rows, g_fl, g_idx = e.get_many(want, arrays=True)
        assert np.array_equal(idx, g_idx), what
        assert np.array_equal(fl, g_fl), what
        assert np.array_equal(rows, g_rows), what
        assert (fl & N.ST_EXISTS).all()
    return want, sizes


def engine_with(keys, sb=16, seed=1, n_rows=None, **kw):
    e = ReplayEngine(0)
    e.register_program(P.counter_program() if sb == 16 else P.bank_account_program())
    e.load_keys(keys)
    e.set_initial_states(table(len(keys) if n_rows is None else n_rows, sb, seed, **kw))
    return e


# ------------------------------------------------------------------ whole-table order
FAMILIES = {
    "uuid": lambda: uuids(np.random.default_rng(5), 6000),
    "account": lambda: accounts(6000),
    "special": special_ids,
}


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("sb", [16, 64])
def test_whole_table_order(family, sb):
    ids = FAMILIES[family]()
    perm = np.random.default_rng(7).permutation(len(ids))
    ids = [ids[i] for i in perm]                        # dense order unrelated to Bytes order
    with engine_with(ids, sb, 11) as e:
        want, _ = check(e, ids, what=family)
        assert len(want) > len(ids) // 2
    with engine_with(ids, sb, 12, p_exists=1.0) as e:  # every row live: the scan is the whole oracle
        want, _ = check(e, ids, what=family)
        assert want == oracle(ids)


def test_liveness_after_real_folds():
    """Never-created rows, tombstoned rows and IF_EXISTS rows that never materialised are skipped; aggregates whose handler threw
    keep their state and appear with SGR_ST_ERROR."""
    from oracle import program_corpus as PC
    from oracle import program_interp as I

    bank = [(I.CREATE, [(I.OP_SET, 0, 16, 16), (I.OP_SET, 16, 32, 8)]), (I.IF_EXISTS, [(I.OP_SET, 16, 32, 8)]), (I.TOMBSTONE, []), (I.THROW, [])]
    rng = np.random.default_rng(13)
    ids = uuids(rng, 3000)
    counts = rng.integers(1, 6, size=len(ids)).astype(np.int64)
    counts[::10] = 0                                                     # never created
    buf, seg, _ = PC.fixed_log(rng, bank, counts, p_throw=0.0)
    kinds = {}
    for a in range(len(ids)):
        if counts[a] == 0:
            continue
        k = a % 4
        for j in range(int(counts[a])):
            PC.set_type(buf, seg, a, j, 1)                               # IF_EXISTS only: never materialises
        if k >= 1:
            PC.set_type(buf, seg, a, 0, 0)                               # CREATE first
        if k == 2:
            PC.set_type(buf, seg, a, -1, 2)                              # ... and TOMBSTONE last
        kinds[a] = k
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(64, N.REC_FIXED64, bank))
        e.load_keys(ids)
        e.load_events(buf, seg)
        e.fold()
        for a, k in kinds.items():
            if k == 3:
                PC.set_type(buf, seg, a, -1, 3)                          # the second fold throws on its last event: state kept
        e.load_events(buf, seg)
        e.fold()                                                         # onto the live states of the first
        want, _ = check(e, ids, what="bank")
        live = set(want)
        for a, k in kinds.items():
            assert (ids[a] in live) == (k in (1, 3)), (a, k)
        assert not any(ids[a] in live for a in range(0, len(ids), 10))
        _, fl, _, got, _ = scanned(e)
        err = {k for k, f in zip(got, fl) if f & N.ST_ERROR}
        assert err == {ids[a] for a, k in kinds.items() if k == 3}


def test_rows_past_n_agg_and_past_the_key_table():
    ids = uuids(np.random.default_rng(14), 3000)
    with engine_with(ids, 16, 15, n_rows=2000, p_exists=1.0) as e:     # ids 2000.. have no row
        want, _ = check(e, ids)
        assert set(want) == set(ids[:2000])
    with engine_with(ids[:1000], 16, 16, n_rows=2500, p_exists=1.0) as e:   # rows 1000.. have no id
        want, _ = check(e, ids[:1000])
        assert len(want) == 1000


# ------------------------------------------------------------------ bounds
def test_bounds():
    ids = special_ids() + accounts(300) + uuids(np.random.default_rng(17), 500) + ["acc", "acc:1", "acc:2", "acc:~", "acc:~~", "acc;", "acc:"]
    with engine_with(ids, 16, 18) as e:
        live = live_ids(e, ids)
        probes = [None, "", "a", "a\0", "ab", "p" * 7, "p" * 8, "p" * 9, "p" * 500, "account-", "account-000000000150", "account-0000000001500",
                  "acc", "acc:", "b", "w" * 15, "w" * 16, "\U0010ffff" * 3, "zzzz", "é", "\0"] + live[::97]
        for frm in probes:
            for to in probes[::3] + [frm]:
                check(e, ids, frm, to, f"[{frm!r}, {to!r}]", page_rows=37)
        assert scanned(e, "b", "a")[3] == []                              # from > to: empty
        sub = scanned(e, "acc", "acc:~")[3]                              # the substate range of the reference: (id, id + ":~")
        assert sub == [k for k in live if bkey("acc") <= bkey(k) <= bkey("acc:~")] and "acc:1" in sub and "acc:~~" not in sub


def _raw(e, frm, frm_excl, to, max_rows=64, ids_cap=4096):
    user = e.state_bytes - 8
    bufs = dict(rows=np.full(max_rows * user, 0xAB, np.uint8), flags=np.full(max_rows, 0xABABABAB, np.uint32), idx=np.full(max_rows, -7, np.int64),
                ids=np.full(max(ids_cap, 1), 0xAB, np.uint8), offs=np.full(max_rows + 1, 0xABABABAB, np.uint32))
    fb = None if frm is None else C.create_string_buffer(frm, max(len(frm), 1))
    tb = None if to is None else C.create_string_buffer(to, max(len(to), 1))
    n, more = C.c_uint64(12345), C.c_int32(-5)
    rc = e._lib.sgr_scan(e._h, fb, 0 if frm is None else len(frm), frm_excl, tb, 0 if to is None else len(to), max_rows, bufs["rows"].ctypes.data,
                         bufs["flags"].ctypes.data, bufs["idx"].ctypes.data, bufs["ids"].ctypes.data, ids_cap, bufs["offs"].ctypes.data,
                         C.byref(n), C.byref(more))
    return rc, bufs, n.value, more.value


def _untouched(bufs, n, more):
    return n == 12345 and more == -5 and (bufs["rows"] == 0xAB).all() and (bufs["idx"] == -7).all() and (bufs["ids"] == 0xAB).all() \
        and (bufs["offs"] == 0xABABABAB).all()


def test_exclusive_and_empty_lower_bounds():
    ids = ["", "a", "b", "c"]
    with engine_with(ids, 16, 19, p_exists=1.0) as e:
        for frm, excl, want in ((None, 0, ["", "a", "b", "c"]), (b"", 0, ["", "a", "b", "c"]), (b"", 1, ["a", "b", "c"]), (b"a", 1, ["b", "c"]),
                                (b"a", 0, ["a", "b", "c"]), (b"bb", 1, ["c"]), (b"c", 1, [])):
            rc, bufs, n, more = _raw(e, frm, excl, None)
            assert rc == 0 and more == 0
            offs = bufs["offs"][:n + 1]
            got = [bufs["ids"][offs[i]:offs[i + 1]].tobytes().decode() for i in range(n)]
            assert got == want, (frm, excl)


# ------------------------------------------------------------------ paging
@pytest.mark.parametrize("page_rows", [1, 2, TILE - 1, TILE, TILE + 1])
def test_page_rows(page_rows):
    ids = uuids(np.random.default_rng(20), 3 * TILE + 517) + special_ids()
    with engine_with(ids, 64, 21) as e:
        want, sizes = check(e, ids, page_rows=page_rows)
        assert all(s == page_rows for s in sizes[:-1]) and 0 < sizes[-1] <= page_rows
        if page_rows > 2:
            check(e, ids, "account", "f", page_rows=page_rows)


def test_more_is_exact_and_pages_resume():
    ids = accounts(2500)
    with engine_with(ids, 16, 22) as e:
        live = live_ids(e, ids)
        frm, excl, got = None, 0, []
        while True:
            rc, bufs, n, more = _raw(e, frm, excl, None, max_rows=500)
            assert rc == 0
            offs = bufs["offs"][:n + 1]
            page = [bufs["ids"][offs[i]:offs[i + 1]].tobytes() for i in range(n)]
            got += page
            assert more == (len(got) < len(live))
            if not more:
                break
            frm, excl = page[-1], 1
        assert [g.decode() for g in got] == live
        rc, bufs, n, more = _raw(e, None, 0, None, max_rows=len(live), ids_cap=20 * len(live))   # exactly the live rows: none left out
        assert rc == 0 and n == len(live) and more == 0


@pytest.mark.parametrize("cap", [330, 999, 4096, 30_000])
def test_id_byte_caps(cap):
    ids = special_ids() + uuids(np.random.default_rng(23), 4 * TILE)
    with engine_with(ids, 16, 24) as e:
        want, sizes = check(e, ids, page_id_bytes=cap)
        lens = [len(bkey(k)) for k in want]
        pos = 0
        for s in sizes:
            used = sum(lens[pos:pos + s])
            assert used <= cap
            if pos + s < len(lens):
                assert used + lens[pos + s] > cap
            pos += s


def test_capacity_writes_nothing():
    ids = ["a" * 500, "b", "c"]
    with engine_with(ids, 16, 25, p_exists=1.0) as e:
        rc, bufs, n, more = _raw(e, None, 0, None, ids_cap=100)
        assert rc == N.SGR_ERR_CAPACITY and _untouched(bufs, n, more)
        rc, bufs, n, more = _raw(e, b"a" * 500, 1, None, ids_cap=100)   # resumed past it: fine
        assert rc == 0 and n == 2 and more == 0
        rc, bufs, n, more = _raw(e, None, 0, None, max_rows=1, ids_cap=600)
        assert rc == 0 and n == 1 and more == 1


# ------------------------------------------------------------------ maintenance of the order
def _append(e, owner, keys):
    enc = [bkey(k) for k in keys]
    offs = np.zeros(len(enc) + 1, dtype=np.uint32)
    np.cumsum([len(b) for b in enc], out=offs[1:])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    assert e._lib.sgr_append_keys(e._h, owner, blob.ctypes.data, offs.ctypes.data, len(enc)) == 0


def test_appended_ids_merge_into_the_order_and_load_keys_rebuilds():
    rng = np.random.default_rng(26)
    ids = uuids(rng, 3000) + accounts(3000) + special_ids()
    ids = [ids[i] for i in rng.permutation(len(ids))]
    owner = C.c_void_p(0x77)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.set_initial_states(table(len(ids), 16, 27))
        done = 0
        for step in (1, 200, 700, 2500, 5000, len(ids)):                  # several extensions, past the index's rehashes too
            _append(e, owner, ids[done:step])
            done = step
            check(e, ids[:done], what=f"after {done} ids", page_rows=999)
        with ReplayEngine(0) as fresh:
            fresh.register_program(P.counter_program())
            fresh.load_keys(ids)
            fresh.set_initial_states(e.export_states())
            assert scanned(fresh)[3] == scanned(e)[3]
        other = accounts(4000, 10 ** 6)                                    # a new key table: the order is built again
        e.load_keys(other)
        check(e, other, what="after load_keys")
        _append(e, C.c_void_p(0x78), ["zz-new", "aa-new", other[5] + "x"])   # a new owner: its ids replace the table
        check(e, ["zz-new", "aa-new", other[5] + "x"], what="new owner")


def test_host_ingest_polls():
    from oracle import kafka_batch as K

    rng = np.random.default_rng(28)
    ing = Ingest()
    off = 0
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        for p in range(5):
            out = bytearray()
            for _ in range(20):
                n = int(rng.integers(1, 40))
                recs = [(d, f"acc-{int(rng.integers(0, 400 * (p + 1)))}:{off + d}".encode(), struct.pack("<IIi", int(rng.integers(0, 3)), off + d, 1))
                        for d in range(n)]
                out += K.encode_record_batch(off, recs, compression="lz4")
                off += n
            ing.record_batches(0, bytes(out))
            e.fold_ingested(ing)
            check(e, ing.keys(), what=f"poll {p}", page_rows=300)


def test_device_ingest_polls():
    from oracle import kafka_batch as K

    rng = np.random.default_rng(29)
    off = 0
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1 << 16) as dg:
            seen = set()
            for p in range(4):
                out = bytearray()
                for _ in range(20):
                    n = int(rng.integers(1, 40))
                    recs = []
                    for d in range(n):
                        k = f"dev-{int(rng.integers(0, 500 * (p + 1)))}" if d % 5 else f"é-{int(rng.integers(0, 50))}"
                        seen.add(k)
                        recs.append((d, f"{k}:{off + d}".encode(), struct.pack("<IIi", int(rng.integers(0, 3)), off + d, 1)))
                    out += K.encode_record_batch(off, recs, compression="lz4")
                    off += n
                dg.submit(0, bytes(out))
                dg.fold()
                idx, fl, rows, ids, _ = scanned(e, page_rows=333)
                assert ids == oracle(ids) and len(set(ids)) == len(ids) and set(ids) <= seen
                g_rows, g_fl, g_idx = e.get_many(ids, arrays=True)
                assert np.array_equal(g_idx, idx) and np.array_equal(g_fl, fl) and np.array_equal(g_rows, rows)
                t = e.export_states()
                live = t[:, 8:12].copy().view(np.uint32).ravel() & N.ST_EXISTS
                assert len(ids) == int(np.count_nonzero(live[:len(seen)]))


def test_duplicate_ids_and_errors():
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_keys(["a", "b"])
        rc, bufs, n, more = _raw(e, None, 0, None)
        assert rc == N.SGR_ERR_STATE and _untouched(bufs, n, more)
        with pytest.raises(N.InvalidStateStoreException):
            list(e.scan())
        e.set_initial_states(table(3, 16, 30, p_exists=1.0))
        assert _raw(e, None, 0, None, max_rows=0)[0] == N.SGR_ERR_INVALID
        assert scanned(e)[3] == ["a", "b"]
        owner = C.c_void_p(0x79)
        _append(e, owner, ["x", "y", "z"])
        assert scanned(e)[3] == ["x", "y", "z"]
        _append(e, owner, ["w", "y"])                                     # a duplicate appended id, as get_batch refuses it
        with pytest.raises(SgrError) as ex:
            list(e.scan())
        assert ex.value.code == N.SGR_ERR_INVALID and "duplicate aggregate id in key table" in str(ex.value)
        with pytest.raises(SgrError):                                     # and it stays refused
            list(e.scan())
        e.load_keys(["c", "b", "a"])                                      # a new key table without one
        assert scanned(e)[3] == ["a", "b", "c"]
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.dist_init(0, 1, None, 1024)
        assert _raw(e, None, 0, None)[0] == N.SGR_ERR_UNSUPPORTED


def test_scan_waits_for_an_async_fold():
    from oracle import program_corpus as PC

    from oracle import program_interp as I

    rng = np.random.default_rng(31)
    ids = uuids(rng, 200_000)
    counter = [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)])]
    buf, seg, _ = PC.fixed_log(rng, counter, rng.integers(0, 30, size=len(ids)).astype(np.int64), p_throw=0.0)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, counter))
        e.load_keys(ids)
        e.load_events(buf, seg)
        e.fold_async()
        first = scanned(e)
        e.wait()
        second = scanned(e)
        assert first[3] == second[3] and np.array_equal(first[2], second[2])
        assert first[3] == live_ids(e, ids)


# ------------------------------------------------------------------ the store on the device
def test_store_all_range_and_count_match_the_host_algorithm():
    rng = np.random.default_rng(32)
    st = GpuReplayKeyValueStore("s", P.counter_program(), state_formatter=lambda k, b: k.encode() + b"=" + b)
    st.init()
    ids = [k for k in special_ids() if k and ":" not in k] + uuids(rng, 2000)
    for i in rng.integers(0, len(ids), size=6000):
        rec = bytearray(64)
        rec[0:4] = struct.pack("<I", int(rng.integers(0, 3)))
        rec[16:20] = struct.pack("<i", int(rng.integers(1, 100)))
        st.put_event(f"{ids[i]}:1", bytes(rec))
    st.flush()
    st.put("zz-overlay", b"v")
    st.put(ids[3], None)                                                  # hides a device row
    st.put(ids[4], b"over")

    def host_all():
        keys = sorted(set(st._keys) | set(st._overlay) | set(st._unflushed), key=bkey)
        return [(k, st.get(k)) for k in keys if st.get(k) is not None]

    want = host_all()
    assert list(st.all()) == want and len(want) > 100
    assert st.approximateNumEntries() == len(want)
    for frm, to in (("a", "f"), ("", "zzzz"), (ids[5], ids[5]), ("z", "a"), ("p" * 8, "p" * 9)):
        assert list(st.range(frm, to)) == [(k, v) for k, v in want if bkey(frm) <= bkey(k) <= bkey(to)]
    st.close()


# ------------------------------------------------------------------ scale
@pytest.mark.parametrize("family", ["uuid", "account"])
def test_scale_four_million_plus_one_percent(family):
    t0 = time.perf_counter()
    n = 4 << 20
    rng = np.random.default_rng(33)
    ids = uuids(rng, n + n // 100 + 1000) if family == "uuid" else accounts(n + n // 100)
    base, extra = ids[:n], ids[n:n + n // 100]
    ids = base + extra
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        owner = C.c_void_p(0x55)
        _append(e, owner, base)
        states = np.zeros((len(ids), 16), np.uint8)
        fl = np.full(len(ids), N.ST_EXISTS, np.uint32)
        fl[rng.random(len(ids)) < 0.02] = 0
        states[:, 8:12] = fl.view(np.uint8).reshape(-1, 4)
        states[:, :4] = np.arange(len(ids), dtype=np.uint32).view(np.uint8).reshape(-1, 4)
        e.set_initial_states(states)
        total = __import__("torch").cuda.mem_get_info(0)[1]
        first, low0 = lowest_free_while(lambda: [k for p in e.scan(page_rows=1 << 20) for k in p[3]])
        assert first == oracle([k for k, f in zip(base, fl) if f])
        _append(e, owner, extra)
        (idx, _, rows, got, _), low1 = lowest_free_while(lambda: scanned(e))
        want = oracle([k for k, f in zip(ids, fl) if f])
        assert got == want
        assert np.array_equal(rows[:, :4].copy().view(np.uint32).ravel(), idx.astype(np.uint32))
        print(f"\n{family}: {len(ids)} ids, {time.perf_counter() - t0:.1f} s, device bytes in use at the peak of the scans "
              f"(whole device) {total - min(low0, low1)}")


def lowest_free_while(fn):
    """(fn(), the lowest free device memory a second thread saw while fn ran)."""
    import threading

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
