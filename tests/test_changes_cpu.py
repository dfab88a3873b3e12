"""CPU checks of the changed-state export: the C entry point refuses a NULL engine and NULL arguments before it touches a
device, and GpuReplayKeyValueStore(on_changes=...) calls its listener once per flush() that folded, with the rows the engine
exports decoded like get(), spare capacity slots left out and failed aggregates with their err_idx. A fake engine stands in
for the GPU one."""
import ctypes as C
import struct

import numpy as np
import pytest

from surge_b200 import native as N
from surge_b200 import store as ST


def test_export_changes_refuses_a_null_engine_and_null_arguments():
    lib = N.load_library()
    cur = N.sgr_changes_cursor()
    rows = np.zeros(64, np.uint8)
    u32 = np.zeros(8, np.uint32)
    idx = np.zeros(8, np.int64)
    ids = np.zeros(64, np.uint8)
    n = C.c_uint64()
    full = (rows.ctypes.data, u32.ctypes.data, u32.ctypes.data, idx.ctypes.data, ids.ctypes.data, 64, u32.ctypes.data, C.byref(n))
    assert lib.sgr_export_changes(None, N.ST_CHANGED, C.byref(cur), 4, *full) == N.SGR_ERR_INVALID
    assert lib.sgr_export_changes(None, N.ST_CHANGED, None, 4, *full) == N.SGR_ERR_INVALID
    assert lib.sgr_export_changes(None, N.ST_CHANGED, C.byref(cur), 4, None, None, None, None, None, 0, None, None) == N.SGR_ERR_INVALID


class FakeEngine:
    """The calls GpuReplayKeyValueStore makes on its engine; export_changes serves `pages`."""

    def __init__(self, device=0):
        self.state_bytes = 16
        self.pages, self.exports, self.folds = [], [], 0
        self.keys = []

    def register_program(self, prog):
        self.state_bytes = int(prog.state_bytes)

    def set_initial_states(self, states):
        pass

    def fold_incremental(self, batch):
        self.folds += 1

    def load_keys(self, keys):
        self.keys = list(keys)

    def export_states(self):
        return np.zeros((0, self.state_bytes), np.uint8)

    def export_changes(self, select=N.ST_CHANGED, page_rows=1 << 20, page_id_bytes=64 << 20):
        self.exports.append(select)
        yield from self.pages

    def close(self):
        pass


def _page(rows):
    """rows: (index, flags, err_idx, program bytes, id)"""
    idx = np.array([r[0] for r in rows], np.int64)
    fl = np.array([r[1] for r in rows], np.uint32)
    err = np.array([r[2] for r in rows], np.uint32)
    data = np.array([np.frombuffer(r[3], np.uint8) for r in rows]).reshape(len(rows), 8)
    return idx, fl, err, data, [r[4] for r in rows]


def _event(t=0):
    rec = bytearray(64)
    rec[0:4] = struct.pack("<I", t)
    return bytes(rec)


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(ST, "ReplayEngine", FakeEngine)


def test_listener_gets_decoded_changes_and_failures_once_per_fold(fake):
    from surge_b200 import programs as P

    calls = []
    st = ST.GpuReplayKeyValueStore("s", P.counter_program(), state_formatter=lambda k, b: k.encode() + b"=" + b,
                                   on_changes=lambda ch, fa: calls.append((ch, fa)))
    st.init()
    for k in ("a", "b", "c"):
        st.put_event(f"{k}:1", _event())
    E, CH, ER = N.ST_EXISTS, N.ST_CHANGED, N.ST_ERROR
    st.engine.pages = [_page([(0, E | CH, 0, b"AAAAAAAA", "a"), (1, CH, 0, bytes(8), "b")]),
                       _page([(2, E | ER, 3, b"CCCCCCCC", "c"), (5, E | CH, 0, b"XXXXXXXX", "\0unused-5"), (9, CH, 0, bytes(8), None)])]
    st.flush()
    assert calls == [([("a", b"a=AAAAAAAA"), ("b", None)], [("c", 3)])]
    assert st.engine.exports == [N.ST_CHANGED | N.ST_ERROR]
    st.flush()                                  # nothing pending: no fold, no call
    assert len(calls) == 1 and st.engine.folds == 1
    st.put_event("a:2", _event())
    st.engine.pages = []
    st.flush()
    assert calls[-1] == ([], []) and len(calls) == 2


def test_without_a_listener_flush_makes_no_export_call(fake):
    from surge_b200 import programs as P

    st = ST.GpuReplayKeyValueStore("s", P.counter_program())
    st.init()
    st.put_event("a:1", _event())
    st.flush()
    assert st.engine.folds == 1 and st.engine.exports == []


def test_overlay_values_are_not_reported(fake):
    from surge_b200 import programs as P

    calls = []
    st = ST.GpuReplayKeyValueStore("s", P.counter_program(), on_changes=lambda ch, fa: calls.append((ch, fa)))
    st.init()
    st.put("kept-in-the-overlay", b"v")         # no codec: an overlay value, never folded
    st.put_event("a:1", _event())
    st.engine.pages = [_page([(0, N.ST_EXISTS | N.ST_CHANGED, 0, b"AAAAAAAA", "a")])]
    st.flush()
    assert calls == [([("a", b"AAAAAAAA")], [])]
    assert st.get("kept-in-the-overlay") == b"v"
