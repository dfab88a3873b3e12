"""CPU checks of ReplayEngine's read paths over a fake library: the page loops of export_changes(_values) and scan(_values),
and the batched reads get_many / get_many_values. The fake serves a Python table through the calls the engine makes, following
include/sgr.h (max_rows, ids_cap, values_cap, the export cursor, from_exclusive and more, SGR_ERR_CAPACITY), so every page the
engine yields is checked against a dict and a sort."""
import ctypes as C
from itertools import islice

import numpy as np
import pytest

from surge_b200 import native as N
from surge_b200.engine import ReplayEngine

STATE_BYTES = 32
USER = STATE_BYTES - 8
CH, ERR, EX = N.ST_CHANGED, N.ST_ERROR, N.ST_EXISTS


def _at(ptr, dtype, n):
    """n items of dtype at a raw address, writable."""
    dt = np.dtype(dtype)
    return np.frombuffer((C.c_char * (n * dt.itemsize)).from_address(ptr), dtype=dt) if n else np.zeros(0, dt)


def _arg_bytes(buf, n):
    return None if buf is None else bytes(buf.raw[:n])


class FakeLib:
    """The engine's table as Python lists: ids[i] (bytes) for i < n_keys, and per dense index its program bytes (None for a None
    state), flags and err_idx. A row's JSON value is value(i); a None state has none."""

    def __init__(self, ids, states, flags, errs, n_keys):
        self.ids, self.states, self.flags, self.errs, self.n_keys = ids, states, flags, errs, n_keys
        self.index = {ids[i]: i for i in range(n_keys)}
        self.calls = []

    def value(self, i):
        if self.states[i] is None:
            return b""
        return b'{"n":%d,"s":"%s"}' % (i, b"x" * (i % 7) * (40 if i % 23 == 0 else 1))

    def row(self, i):
        return self.states[i] if self.states[i] is not None else bytes(USER)

    # -- lifecycle
    def sgr_create(self, cfg, h):
        h._obj.value = 1
        return N.SGR_OK

    def sgr_destroy(self, h):
        return N.SGR_OK

    def sgr_last_error(self, h):
        return b"fake"

    def sgr_register_program(self, h, prog):
        return N.SGR_OK

    def sgr_states_device(self, h, p, n, sb):
        p._obj.value, n._obj.value, sb._obj.value = 0x1000, len(self.states), STATE_BYTES
        return N.SGR_OK

    # -- batched reads
    def _query(self, blob, offs, n):
        assert blob, "the id blob pointer is never NULL"
        o = _at(offs, np.uint32, n + 1)
        assert o[0] == 0 and np.all(np.diff(o.astype(np.int64)) >= 0)
        raw = C.string_at(blob, int(o[n])) if n else b""
        return [self.index.get(raw[o[i]:o[i + 1]], -1) for i in range(n)]

    def sgr_get_batch(self, h, blob, offs, n, out, cap, flags, indices):
        self.calls.append(("get_batch", n))
        if n == 0:
            return N.SGR_OK
        if cap < n * USER:
            return N.SGR_ERR_CAPACITY
        q = self._query(blob, offs, n)
        rows, fl, ix = _at(out, np.uint8, n * USER).reshape(n, USER), _at(flags, np.uint32, n), _at(indices, np.int64, n)
        for j, i in enumerate(q):
            rows[j] = np.frombuffer(self.row(i), np.uint8) if i >= 0 else 0
            fl[j], ix[j] = (self.flags[i], i) if i >= 0 else (0, -1)
        return N.SGR_OK

    def sgr_get_batch_values(self, h, blob, offs, n, values, values_cap, voffs, flags, indices, values_len):
        self.calls.append(("get_batch_values", values_cap))
        q = self._query(blob, offs, n)
        vals = [self.value(i) if i >= 0 else b"" for i in q]
        need = sum(map(len, vals))
        if values_len is not None:
            values_len._obj.value = need
        if need > values_cap:
            return N.SGR_ERR_CAPACITY
        vo, fl = _at(voffs, np.uint64, n + 1), _at(flags, np.uint32, n)
        vo[0] = 0
        for j, (i, v) in enumerate(zip(q, vals)):
            vo[j + 1] = vo[j] + len(v)
            fl[j] = self.flags[i] if i >= 0 else 0
        _at(values, np.uint8, need)[:] = np.frombuffer(b"".join(vals), np.uint8)
        return N.SGR_OK

    # -- pages
    def _page(self, order, max_rows, out, ids_cap, flags, err, indices, ids, id_offsets, values_cap):
        """Write the rows `order` lists, in that order, until max_rows, ids_cap or values_cap stops the page. Returns the rows
        written, or SGR_ERR_CAPACITY when the first row's id or value alone does not fit."""
        k = used = vused = 0
        for i in order:
            key = self.ids[i] if i < self.n_keys else b""
            val = self.value(i) if values_cap is not None else b""
            if k == max_rows or used + len(key) > ids_cap or vused + len(val) > (values_cap or 0):
                if k == 0:
                    return N.SGR_ERR_CAPACITY
                break
            k, used, vused = k + 1, used + len(key), vused + len(val)
        if k:
            sel = order[:k]
            _at(flags, np.uint32, k)[:] = [self.flags[i] for i in sel]
            _at(indices, np.int64, k)[:] = sel
            if err is not None:
                _at(err, np.uint32, k)[:] = [self.errs[i] for i in sel]
            keys = [self.ids[i] if i < self.n_keys else b"" for i in sel]
            _at(id_offsets, np.uint32, k + 1)[:] = np.cumsum([0] + [len(b) for b in keys])
            _at(ids, np.uint8, used)[:] = np.frombuffer(b"".join(keys), np.uint8)
            if values_cap is None:
                _at(out[0], np.uint8, k * USER)[:] = np.frombuffer(b"".join(self.row(i) for i in sel), np.uint8)
            else:
                vals = [self.value(i) for i in sel]
                _at(out[2], np.uint64, k + 1)[:] = np.cumsum([0] + [len(v) for v in vals])
                _at(out[0], np.uint8, vused)[:] = np.frombuffer(b"".join(vals), np.uint8)
        return k

    def _export(self, select, cur, max_rows, out, flags, err, indices, ids, ids_cap, id_offsets, n_rows, values_cap):
        c = cur._obj
        self.calls.append(("export", c.next, max_rows, ids_cap, values_cap))
        n_agg = len(self.states)
        if select == 0 or select & ~(CH | ERR) or max_rows == 0 or c.next > n_agg:
            return N.SGR_ERR_INVALID
        order = [i for i in range(c.next, n_agg) if self.flags[i] & select]
        k = self._page(order, max_rows, out, ids_cap, flags, err, indices, ids, id_offsets, values_cap)
        if k < 0:
            return k
        c.next = order[k] if k < len(order) else n_agg
        c.token, c.n_keys = 1, self.n_keys
        n_rows._obj.value = k
        return N.SGR_OK

    def sgr_export_changes(self, h, select, cur, max_rows, rows, flags, err, indices, ids, ids_cap, id_offsets, n_rows):
        return self._export(select, cur, max_rows, (rows,), flags, err, indices, ids, ids_cap, id_offsets, n_rows, None)

    def sgr_export_changes_values(self, h, select, cur, max_rows, values, values_cap, voffs, flags, err, indices, ids, ids_cap,
                                  id_offsets, n_rows):
        return self._export(select, cur, max_rows, (values, values_cap, voffs), flags, err, indices, ids, ids_cap, id_offsets,
                            n_rows, values_cap)

    def _scan(self, frm, frm_len, excl, to, to_len, max_rows, out, flags, indices, ids, ids_cap, id_offsets, n_rows, more,
              values_cap):
        lo, hi = _arg_bytes(frm, frm_len), _arg_bytes(to, to_len)
        self.calls.append(("scan", lo, excl, hi, max_rows, ids_cap, values_cap))
        if max_rows == 0:
            return N.SGR_ERR_INVALID
        live = sorted((i for i in range(min(self.n_keys, len(self.states))) if self.flags[i] & EX), key=lambda i: self.ids[i])
        order = [i for i in live if (lo is None or self.ids[i] > lo or (self.ids[i] == lo and not excl))
                 and (hi is None or self.ids[i] <= hi)]
        k = self._page(order, max_rows, out, ids_cap, flags, None, indices, ids, id_offsets, values_cap)
        if k < 0:
            return k
        n_rows._obj.value, more._obj.value = k, int(k < len(order))
        return N.SGR_OK

    def sgr_scan(self, h, frm, frm_len, excl, to, to_len, max_rows, rows, flags, indices, ids, ids_cap, id_offsets, n_rows, more):
        return self._scan(frm, frm_len, excl, to, to_len, max_rows, (rows,), flags, indices, ids, ids_cap, id_offsets, n_rows,
                          more, None)

    def sgr_scan_values(self, h, frm, frm_len, excl, to, to_len, max_rows, values, values_cap, voffs, flags, indices, ids,
                        ids_cap, id_offsets, n_rows, more):
        return self._scan(frm, frm_len, excl, to, to_len, max_rows, (values, values_cap, voffs), flags, indices, ids, ids_cap,
                          id_offsets, n_rows, more, values_cap)


N_AGG, N_KEYS = 300, 280


def make_table(seed=7):
    rng = np.random.default_rng(seed)
    ids = [f"agg-{i:03d}" + "é" * (i % 4) + ":x" * (i % 9 == 0) for i in range(N_KEYS)]
    ids[5], ids[6], ids[7] = "", "a", "ab"   # the empty id, and one id a prefix of another
    flags, states, errs = [], [], []
    for i in range(N_AGG):
        f = int(rng.integers(0, 8))
        flags.append(f)
        states.append(rng.bytes(USER) if f & EX else None)
        errs.append(int(rng.integers(1, 50)) if f & ERR else 0)
    flags[5] = EX | CH
    states[5] = rng.bytes(USER)
    return ids, states, flags, errs


@pytest.fixture
def engine(monkeypatch):
    ids, states, flags, errs = make_table()
    lib = FakeLib([k.encode("utf-8") for k in ids], states, flags, errs, N_KEYS)
    monkeypatch.setattr(N, "load_library", lambda *a, **k: lib)
    e = ReplayEngine(0)
    prog = N.sgr_fold_program()
    prog.state_bytes = STATE_BYTES
    e.register_program(prog)
    e.table = dict(ids=ids, states=states, flags=flags, errs=errs, lib=lib)
    yield e
    e.close()


def _row(t, i):
    return t["states"][i] if t["states"][i] is not None else bytes(USER)


def _id_bytes(ids):
    return sum(len(k.encode("utf-8")) for k in ids if k is not None)


def _bounded(pages):
    """Every table here fits in N_AGG pages: a loop that does not advance fails the comparison instead of running forever."""
    return islice(pages, N_AGG + 1)


PAGES = [(1, 64 << 20), (7, 64 << 20), (None, 64 << 20), (1 << 20, 40), (7, 25)]


@pytest.mark.parametrize("select", [CH, ERR, CH | ERR])
@pytest.mark.parametrize("page_rows,page_id_bytes", PAGES)
def test_export_changes_pages_every_selected_row_once(engine, select, page_rows, page_id_bytes):
    t = engine.table
    want = [i for i in range(N_AGG) if t["flags"][i] & select]
    got, sizes = [], []
    for idx, flags, err, rows, ids in _bounded(engine.export_changes(select, page_rows=page_rows, page_id_bytes=page_id_bytes)):
        assert (idx.dtype, flags.dtype, err.dtype, rows.dtype, rows.shape[1]) == (np.int64, np.uint32, np.uint32, np.uint8, USER)
        assert len(idx) == len(flags) == len(err) == len(rows) == len(ids) > 0
        assert _id_bytes(ids) <= page_id_bytes and (page_rows is None or len(idx) <= page_rows)
        sizes.append(len(idx))
        for j, i in enumerate(idx.tolist()):
            got.append(i)
            assert flags[j] == t["flags"][i] and err[j] == t["errs"][i] and rows[j].tobytes() == _row(t, i)
            assert ids[j] == (t["ids"][i] if i < N_KEYS else None)
    assert got == want
    if page_rows is None:
        assert sizes == [len(want)]
    elif page_id_bytes < 64 << 20:
        assert any(s < page_rows for s in sizes[:-1])   # the id budget cut a page
    else:
        assert sizes == [min(page_rows, len(want) - p) for p in range(0, len(want), page_rows)]


@pytest.mark.parametrize("page_rows,page_id_bytes", PAGES)
@pytest.mark.parametrize("values_cap", [64 << 20, 300])
def test_export_changes_values_pages(engine, page_rows, page_id_bytes, values_cap):
    t, lib = engine.table, engine.table["lib"]
    want = [i for i in range(N_AGG) if t["flags"][i] & (CH | ERR)]
    got, sizes = [], []
    for idx, flags, err, ids, vals in _bounded(engine.export_changes_values(CH | ERR, max_rows=page_rows, values_cap=values_cap,
                                                                             page_id_bytes=page_id_bytes)):
        assert (idx.dtype, flags.dtype, err.dtype) == (np.int64, np.uint32, np.uint32)
        assert len(idx) == len(flags) == len(err) == len(ids) == len(vals) > 0
        assert sum(len(v) for v in vals if v is not None) <= values_cap and _id_bytes(ids) <= page_id_bytes
        sizes.append(len(idx))
        for j, i in enumerate(idx.tolist()):
            got.append(i)
            assert flags[j] == t["flags"][i] and err[j] == t["errs"][i]
            assert ids[j] == (t["ids"][i] if i < N_KEYS else None)
            assert vals[j] == (lib.value(i) if t["states"][i] is not None else None)
    assert got == want
    if values_cap < 64 << 20 and page_rows is None:
        assert len(sizes) > 1   # the value budget cut the pages


def _in_range(t, frm, to):
    live = [i for i in range(N_KEYS) if t["flags"][i] & EX]
    key = lambda i: t["ids"][i].encode("utf-8")   # noqa: E731
    return sorted((i for i in live if (frm is None or key(i) >= frm.encode("utf-8")) and (to is None or key(i) <= to.encode("utf-8"))),
                  key=key)


RANGES = [(None, None), ("", None), ("a", "agg-150"), ("agg-100", None), (None, "agg-050é"), ("agg-2", "agg-1")]


@pytest.mark.parametrize("frm,to", RANGES)
@pytest.mark.parametrize("page_rows,page_id_bytes", [(1, 64 << 20), (7, 64 << 20), (1 << 20, 64 << 20), (1 << 20, 40)])
def test_scan_pages_live_ids_in_bytes_order(engine, frm, to, page_rows, page_id_bytes):
    t, lib = engine.table, engine.table["lib"]
    want = _in_range(t, frm, to)
    lib.calls.clear()
    got, sizes = [], []
    for idx, flags, rows, ids in _bounded(engine.scan(frm, to, page_rows=page_rows, page_id_bytes=page_id_bytes)):
        assert (idx.dtype, flags.dtype, rows.dtype, rows.shape[1]) == (np.int64, np.uint32, np.uint8, USER)
        assert len(idx) == len(flags) == len(rows) == len(ids) > 0
        assert len(idx) <= page_rows and _id_bytes(ids) <= page_id_bytes
        sizes.append(len(idx))
        for j, i in enumerate(idx.tolist()):
            got.append(i)
            assert ids[j] == t["ids"][i] and flags[j] == t["flags"][i] and rows[j].tobytes() == _row(t, i)
    assert got == want
    # each page resumes exclusively after the last id of the page before; the first starts at frm itself
    calls = [c for c in lib.calls if c[0] == "scan"]
    lo0 = None if frm is None else frm.encode("utf-8")
    assert [(c[1], c[2]) for c in calls] == [(lo0, 0)] + [(t["ids"][i].encode("utf-8"), 1) for i in _page_ends(want, sizes)]
    assert all(c[3] == (None if to is None else to.encode("utf-8")) for c in calls)
    if page_id_bytes < 64 << 20 and len(want) > 10:
        assert len(sizes) > 1   # the id budget cut the pages


def _page_ends(want, sizes):
    """The last row of each page but a final one the engine needs no further call after."""
    ends, p = [], 0
    for s in sizes:
        p += s
        ends.append(want[p - 1])
    return ends[:-1]


@pytest.mark.parametrize("frm,to", RANGES[:4])
@pytest.mark.parametrize("page_rows,values_cap", [(1, 64 << 20), (7, 64 << 20), (1 << 20, 64 << 20), (1 << 20, 300)])
def test_scan_values_pages(engine, frm, to, page_rows, values_cap):
    t, lib = engine.table, engine.table["lib"]
    want = _in_range(t, frm, to)
    got, sizes = [], []
    for idx, flags, ids, vals in _bounded(engine.scan_values(frm, to, max_rows=page_rows, values_cap=values_cap)):
        assert (idx.dtype, flags.dtype) == (np.int64, np.uint32)
        assert len(idx) == len(flags) == len(ids) == len(vals) > 0 and len(idx) <= page_rows
        assert sum(len(v) for v in vals) <= values_cap
        sizes.append(len(idx))
        for j, i in enumerate(idx.tolist()):
            got.append(i)
            assert ids[j] == t["ids"][i] and flags[j] == t["flags"][i] and vals[j] == lib.value(i)
    assert got == want
    if values_cap < 64 << 20 and len(want) > 20:
        assert len(sizes) > 1   # the value budget cut the pages


def test_an_id_or_value_too_long_for_its_budget_is_refused(engine):
    for pages in (engine.export_changes(CH | ERR, page_id_bytes=1), engine.scan("agg", page_id_bytes=1),
                  engine.export_changes_values(CH | ERR, values_cap=3), engine.scan_values(values_cap=3)):
        with pytest.raises(N.SgrError) as ex:
            list(pages)
        assert ex.value.code == N.SGR_ERR_CAPACITY


def _queries(t):
    rng = np.random.default_rng(3)
    known = [t["ids"][i] for i in rng.integers(0, N_KEYS, 200)]
    return known + ["", "a", "ab", "nope", "agg-", "agg-290"] + known[:5]


def test_get_many_answers_each_id_as_a_dict_does(engine):
    t = engine.table
    keys = _queries(t)
    pos = {t["ids"][i]: i for i in range(N_KEYS)}
    got = engine.get_many(keys)
    states, flags, indices = engine.get_many(keys, arrays=True)
    assert (states.dtype, states.shape, flags.dtype, indices.dtype) == (np.uint8, (len(keys), USER), np.uint32, np.int64)
    for j, k in enumerate(keys):
        i = pos.get(k)
        assert got[j] == (None if i is None else t["states"][i])
        assert indices[j] == (-1 if i is None else i) and flags[j] == (0 if i is None else t["flags"][i])
        assert states[j].tobytes() == (bytes(USER) if i is None else _row(t, i))
    assert engine.get_many([]) == []
    assert engine.get_many([""]) == [t["states"][5]]


def test_get_many_values_retries_once_with_the_size_the_library_asks_for(engine):
    t, lib = engine.table, engine.table["lib"]
    keys = _queries(t)
    pos = {t["ids"][i]: i for i in range(N_KEYS)}
    want = [None if pos.get(k) is None or t["states"][pos[k]] is None else lib.value(pos[k]) for k in keys]
    lib.calls.clear()
    assert engine.get_many_values(keys) == want
    assert [c[0] for c in lib.calls] == ["get_batch_values"]   # the first budget, 64 bytes an id, fits
    long_keys = [t["ids"][i] for i in range(0, N_KEYS, 23) if t["states"][i] is not None] * 3
    need = sum(len(lib.value(pos[k])) for k in long_keys)
    assert need > 64 * len(long_keys) + 64
    lib.calls.clear()
    assert engine.get_many_values(long_keys) == [lib.value(pos[k]) for k in long_keys]
    assert lib.calls == [("get_batch_values", 64 * len(long_keys) + 64), ("get_batch_values", need)]
    lib.calls.clear()
    with pytest.raises(N.SgrError) as ex:
        engine.get_many_values(long_keys, values_cap=need - 1)
    assert ex.value.code == N.SGR_ERR_CAPACITY and lib.calls == [("get_batch_values", need - 1)]
    assert engine.get_many_values(long_keys, values_cap=need) == [lib.value(pos[k]) for k in long_keys]
    assert engine.get_many_values([]) == []
