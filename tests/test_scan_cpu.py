"""CPU checks of the ordered scan: the C entry point refuses a NULL engine and NULL arguments before it touches a device; the
round key of the device sort, (word_r, lenclass_r) over 8-byte windows, orders ids exactly as Python's bytes comparison does,
and so does a model of the sort's rounds (group heads, scan, resolution) with the kernels' index arithmetic; and
GpuReplayKeyValueStore.all() / range() / approximateNumEntries() over engine.scan give what the earlier host algorithm (kept
here as the reference) gave. A fake engine stands in for the GPU one."""
import ctypes as C
import functools
import struct

import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

from surge_b200 import native as N
from surge_b200 import store as ST


def test_scan_refuses_a_null_engine_and_null_arguments():
    lib = N.load_library()
    rows = np.zeros(64, np.uint8)
    u32 = np.zeros(8, np.uint32)
    idx = np.zeros(8, np.int64)
    ids = np.zeros(64, np.uint8)
    n, more = C.c_uint64(), C.c_int32()
    full = (4, rows.ctypes.data, u32.ctypes.data, idx.ctypes.data, ids.ctypes.data, 64, u32.ctypes.data, C.byref(n), C.byref(more))
    assert lib.sgr_scan(None, None, 0, 0, None, 0, *full) == N.SGR_ERR_INVALID
    assert lib.sgr_scan(None, b"a", 1, 1, b"b", 1, *full) == N.SGR_ERR_INVALID
    assert lib.sgr_scan(None, None, 0, 0, None, 0, 4, None, None, None, None, 0, None, None, None) == N.SGR_ERR_INVALID


# ------------------------------------------------------------------ the round key
def round_key(b: bytes, r: int):
    """(word_r, lenclass_r) of csrc/id_order.cu: bytes [8r, 8r + 8) big-endian and zero-padded, min(len - 8r, 9)."""
    if len(b) <= 8 * r:
        return 0, 0
    return int.from_bytes(b[8 * r:8 * r + 8].ljust(8, b"\0"), "big"), min(len(b) - 8 * r, 9)


def msd_cmp(a: bytes, b: bytes) -> int:
    """Compare by round keys as the rounds do: a difference decides, an equal key with lenclass <= 8 means equal ids, equal keys
    of class 9 go on to the next window."""
    r = 0
    while True:
        ka, kb = round_key(a, r), round_key(b, r)
        if ka != kb:
            return -1 if ka < kb else 1
        if ka[1] <= 8:
            return 0
        r += 1


def sort_model(ids):
    """The device sort's rounds over a list, with the kernels' arithmetic: keys (group, word, lenclass); old and new group heads;
    an inclusive scan (max, max, sum); resolved ids to group + j - old_start, unresolved ones compacted with group + new_start -
    old_start."""
    m = len(ids)
    out = [None] * m
    act = [(0, i) for i in range(m)]          # (group, id)
    r = 0
    while act:
        keyed = sorted(((g,) + round_key(ids[i], r), i) for g, i in act)
        keys = [k for k, _ in keyed]
        n = len(keys)
        heads = []
        for j, k in enumerate(keys):
            old_head = j == 0 or keys[j - 1][0] != k[0]
            new_head = j == 0 or keys[j - 1] != k
            new_last = j + 1 == n or keys[j + 1] != k
            heads.append((j if old_head else 0, j if new_head else 0, int(not (new_head and new_last) and k[2] == 9)))
        scan, acc = [], (0, 0, 0)
        for h in heads:
            acc = (max(acc[0], h[0]), max(acc[1], h[1]), acc[2] + h[2])
            scan.append(acc)
        nxt = [None] * (scan[-1][2] if scan else 0)
        for j, ((g, _, _), i) in enumerate(keyed):
            before = scan[j - 1][2] if j else 0
            if scan[j][2] == before:
                assert out[g + j - scan[j][0]] is None
                out[g + j - scan[j][0]] = i
            else:
                nxt[scan[j][2] - 1] = (g + scan[j][1] - scan[j][0], i)
        act = nxt
        r += 1
    return [ids[i] for i in out]


_ALPHABET = [0, 1, 0x2f, 0x30, 0x61, 0x7f, 0x80, 0xc3, 0xff]
_byte_strings = st.lists(st.sampled_from(_ALPHABET), max_size=30).map(bytes)


@st.composite
def id_sets(draw):
    """Ids with shared prefixes of every length across multiples of 8, \\0 bytes, ids that are prefixes of each other, "" and
    bytes >= 0x80."""
    base = draw(st.lists(st.sampled_from(_ALPHABET), min_size=40, max_size=40).map(bytes))
    parts = draw(st.lists(st.tuples(st.integers(0, 40), _byte_strings), min_size=1, max_size=40))
    ids = {base[:k] + s for k, s in parts}
    if draw(st.booleans()):
        ids |= {b"", base[:8], base[:16], base[:8] + b"\0", base[:16] + b"\0\0"}
    return sorted(ids, key=lambda _: draw(st.integers(0, 1 << 30)))   # any dense order


@settings(max_examples=300, deadline=None)
@given(id_sets())
def test_round_keys_order_ids_as_bytes_do(ids):
    for a in ids:
        for b in ids[:12]:
            assert msd_cmp(a, b) == (a > b) - (a < b), (a, b)
    assert sorted(ids, key=functools.cmp_to_key(msd_cmp)) == sorted(ids)


@settings(max_examples=300, deadline=None)
@given(id_sets())
def test_sort_rounds_model_equals_sorted(ids):
    assert sort_model(ids) == sorted(ids)


def test_round_keys_on_fixed_cases():
    ids = [b"", b"\0", b"\0\0", b"a", b"a\0", b"a\0\0", b"ab", b"a" * 8, b"a" * 8 + b"\0", b"a" * 9, b"a" * 16, b"a" * 16 + b"\0",
           b"a" * 15 + b"b", b"\x7f", b"\x80", b"\xff" * 9, "é".encode(), "😀".encode()]
    assert sorted(ids, key=functools.cmp_to_key(msd_cmp)) == sorted(ids)
    assert sort_model(ids) == sorted(ids)


# ------------------------------------------------------------------ the store over engine.scan
class FakeEngine:
    """The calls GpuReplayKeyValueStore makes on its engine. `live` maps an id of the loaded key table to its program bytes (a
    live row); scan pages them in Bytes order, get reads them."""

    def __init__(self, device=0):
        self.state_bytes = 16
        self.keys, self.live, self.scans = [], {}, []
        self.closed = False

    def register_program(self, prog):
        self.state_bytes = int(prog.state_bytes)

    def set_initial_states(self, states):
        pass

    def fold_incremental(self, batch):
        pass

    def load_keys(self, keys):
        self.keys = list(keys)

    def export_states(self):
        return np.zeros((0, self.state_bytes), np.uint8)

    def get(self, key):
        return self.live.get(key) if key in self.keys else None

    def scan(self, frm=None, to=None, page_rows=3, page_id_bytes=64 << 20):
        if self.closed:   # a closed engine's handle is NULL: the C call refuses it
            raise N.SgrError(N.SGR_ERR_INVALID, "null argument")
        self.scans.append((frm, to))
        lo = None if frm is None else frm.encode()
        hi = None if to is None else to.encode()
        rows = sorted((k.encode(), i, k) for i, k in enumerate(self.keys) if k in self.live)
        rows = [r for r in rows if (lo is None or lo <= r[0]) and (hi is None or r[0] <= hi)]
        for p in range(0, len(rows), page_rows):
            page = rows[p:p + page_rows]
            yield (np.array([r[1] for r in page], np.int64), np.full(len(page), N.ST_EXISTS, np.uint32),
                   np.array([np.frombuffer(self.live[r[2]], np.uint8) for r in page]).reshape(len(page), 8), [r[2] for r in page])

    def close(self):
        self.closed = True


def reference_all(store):
    """GpuReplayKeyValueStore.all() as it was before engine.scan: every id sorted on the host, then get() per id."""
    with store._lock:
        keys = sorted(set(store._ingest.keys() if store._ingest is not None else store._keys) | set(store._overlay) | set(store._unflushed),
                      key=lambda k: k.encode("utf-8"))
    for k in keys:
        v = store.get(k)
        if v is not None:
            yield k, v


def reference_range(store, frm, to):
    lo, hi = frm.encode("utf-8"), to.encode("utf-8")
    for k, v in reference_all(store):
        if lo <= k.encode("utf-8") <= hi:
            yield k, v


def _event():
    return bytes(64)


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(ST, "ReplayEngine", FakeEngine)


BOUNDS = [("", "\U0010ffff"), ("a", "c"), ("b", "b"), ("c", "a"), ("b\0", "bz"), ("", ""), ("é", "é\0"), ("zz", "zzz")]


def _same_as_reference(st_):
    assert list(st_.all()) == list(reference_all(st_))
    assert st_.approximateNumEntries() == sum(1 for _ in reference_all(st_))
    for frm, to in BOUNDS:
        assert list(st_.range(frm, to)) == list(reference_range(st_, frm, to)), (frm, to)


def test_store_with_overlay_formatter_and_spare_slots(fake):
    from surge_b200 import programs as P

    st_ = ST.GpuReplayKeyValueStore("s", P.counter_program(), state_formatter=lambda k, b: k.encode() + b"=" + b)
    st_.init()
    ids = ["b", "a", "é", "b\0", "", "c", "bb", "ab", "z" * 20, "日本"]
    for k in ids:
        if k:
            st_.put_event(f"{k}:1", _event())
    st_.flush()
    e = st_.engine
    assert e.keys[:len(st_._keys)] == st_._keys and len(e.keys) > len(st_._keys)
    for i, k in enumerate(e.keys):
        if i % 4 != 3:                                        # some never created
            e.live[k] = struct.pack("<Q", i)                 # spare slots too: they must not appear
    _same_as_reference(st_)
    assert all(not k.startswith("\0unused") for k, _ in st_.all())
    st_.put("bz", b"over")                                    # overlay values: new ids, replaced ids, hidden ids
    st_.put("a", b"over-a")
    st_.put("c", None)
    st_.put("00", None)
    _same_as_reference(st_)
    assert dict(st_.all())["a"] == b"over-a" and "c" not in dict(st_.all())
    st_.put_event("new:1", _event())                          # an id the device does not know yet
    _same_as_reference(st_)


def test_store_with_codec_unflushed_puts_and_deletes(fake):
    from surge_b200 import programs as P

    codec = ST.StateCodec(lambda k, v: v[:8].ljust(8, b"\0"), lambda k, b: b"S" + b, 4, 5)
    st_ = ST.GpuReplayKeyValueStore("c", P.counter_program_with_snapshot_rules(), codec=codec)
    st_.init()
    for k in ("a", "b", "c", "d"):
        st_.put(k, k.encode() * 3)
    _same_as_reference(st_)                                   # nothing folded yet: every value is an unflushed put
    st_.flush()
    e = st_.engine
    for k in ("a", "b", "c", "d"):
        e.live[k] = (k.encode() * 3)[:8].ljust(8, b"\0")
    _same_as_reference(st_)
    st_.delete("b")                                           # unflushed delete hides the device row
    st_.put("c", b"newc")                                     # unflushed put answers first
    st_.put("e", b"eeee")                                     # a new id, unflushed
    _same_as_reference(st_)
    assert [k for k, _ in st_.all()] == ["a", "c", "d", "e"]
    assert dict(st_.all())["c"] == b"newc" and dict(st_.all())["a"] == b"Saaa" + bytes(5)


def outcome(entries):
    """(what an iterator yields until it ends or raises, the type of what it raised or None)."""
    got = []
    try:
        for kv in entries:
            got.append(kv)
    except Exception as ex:  # noqa: BLE001
        return got, type(ex)
    return got, None


def _same_outcomes(st_):
    assert outcome(st_.all()) == outcome(reference_all(st_))
    for frm, to in BOUNDS:
        assert outcome(st_.range(frm, to)) == outcome(reference_range(st_, frm, to)), (frm, to)
    def count(f):
        try:
            return f(), None
        except Exception as ex:  # noqa: BLE001
            return None, type(ex)

    assert count(st_.approximateNumEntries) == count(lambda: sum(1 for _ in reference_all(st_)))


def test_store_not_restored_and_closed(fake):
    from surge_b200 import programs as P

    st_ = ST.GpuReplayKeyValueStore("s", P.counter_program())
    st_.init()
    assert list(st_.all()) == [] and st_.approximateNumEntries() == 0
    _same_outcomes(st_)
    st_.put("a", b"v")                                        # an overlay value is readable before any fold
    assert list(st_.all()) == [("a", b"v")]
    _same_outcomes(st_)
    st_.put_event("b:1", _event())
    st_.put_event("é:1", _event())
    got, raised = outcome(st_.all())
    assert got == [("a", b"v")] and raised is ST.InvalidStateStoreException   # the overlay id sorts first, then "b" raises
    assert outcome(st_.range("c", "d")) == ([], ST.InvalidStateStoreException)  # as range() filtering all(): "b" raises anyway
    _same_outcomes(st_)
    st_.flush()
    st_.engine.live["b"] = bytes(8)
    assert [k for k, _ in st_.all()] == ["a", "b"]
    _same_outcomes(st_)
    it = st_.all()
    assert next(it) == ("a", b"v")
    st_.close()                                               # closed while iterating: the next id raises
    with pytest.raises(ST.InvalidStateStoreException):
        next(it)
    assert outcome(st_.all()) == ([], ST.InvalidStateStoreException)
    assert outcome(st_.range("x", "y")) == ([], ST.InvalidStateStoreException)
    with pytest.raises(ST.InvalidStateStoreException):
        st_.approximateNumEntries()
    _same_outcomes(st_)


def test_an_empty_closed_store_yields_nothing(fake):
    from surge_b200 import programs as P

    st_ = ST.GpuReplayKeyValueStore("s", P.counter_program())
    st_.init()
    st_.flush()                                               # folded, with no ids
    st_.close()
    assert list(st_.all()) == [] and list(st_.range("a", "b")) == [] and st_.approximateNumEntries() == 0
    _same_outcomes(st_)


def test_a_closed_store_with_device_rows_only_raises_not_open(fake):
    from surge_b200 import programs as P

    st_ = ST.GpuReplayKeyValueStore("s", P.counter_program())
    st_.init()
    st_.put_event("a:1", _event())
    st_.flush()
    st_.engine.live["a"] = bytes(8)
    st_.close()
    for entries in (st_.all(), st_.range("a", "a"), st_.range("x", "y")):
        with pytest.raises(ST.InvalidStateStoreException, match="is not open"):
            list(entries)
    _same_outcomes(st_)


def test_a_range_asks_the_device_for_its_bounds_only(fake):
    from surge_b200 import programs as P

    st_ = ST.GpuReplayKeyValueStore("s", P.counter_program())
    st_.init()
    st_.put_event("a:1", _event())
    st_.flush()
    st_.engine.live["a"] = bytes(8)
    list(st_.range("a", "b"))
    list(st_.all())
    list(st_.range("b", "a"))                                 # from > to: empty, without a device call
    assert st_.engine.scans == [("a", "b"), (None, None)]
