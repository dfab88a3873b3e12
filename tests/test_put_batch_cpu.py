"""No GPU: the rules of sgr_put_batch as the NumPy restatement (oracle/put_batch.py) states them, the argument checks the C ABI
makes before it touches a device, and a state-topic store's refusals (a codec without snapshot rules)."""
import ctypes as C
import struct

import numpy as np
import pytest

from oracle import put_batch as O
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200 import store as ST

EX, CH = O.EXISTS, O.CHANGED


def flags(table):
    sb = table.shape[1]
    return table[:, sb - 8:sb - 4].copy().view(np.uint32)[:, 0].tolist()


def test_last_write_wins_and_first_appearance_indices():
    ids, t, n_new = O.put_batch([], np.zeros((0, 16), np.uint8), [("b", b"\1" * 8), ("a", None), ("b", b"\2" * 8), ("c", b"\3" * 8), ("a", b"\4" * 8)])
    assert ids == ["b", "a", "c"] and n_new == 3
    assert t[:, :8].tolist() == [[2] * 8, [4] * 8, [3] * 8]
    assert flags(t) == [EX | CH] * 3
    ids, t, n_new = O.put_batch(ids, t, [("d", None), ("c", b"\3" * 8), ("b", None), ("e", b"\5" * 8)])
    assert ids == ["b", "a", "c", "d", "e"] and n_new == 2
    assert flags(t) == [CH, EX, EX, 0, EX | CH]      # a unwritten: CHANGED cleared; c rewritten equal; d a tombstone of nothing
    assert not t[0, :8].any() and not t[3, :8].any()


def test_changed_rule_for_double_fields():
    d = lambda x: struct.pack("<d", x) + b"\7" * 16   # noqa: E731
    ids, t, _ = O.put_batch([], np.zeros((0, 32), np.uint8), [("nan", d(float("nan"))), ("zero", d(0.0)), ("x", d(1.0))], f64_offsets=[0])
    ids, t, _ = O.put_batch(ids, t, [("nan", d(float("nan"))), ("zero", d(-0.0)), ("x", d(1.0)), ("x", None), ("x", d(1.0))], f64_offsets=[0])
    assert flags(t) == [EX | CH, EX, EX]
    assert t[1, :8].tobytes() == struct.pack("<d", -0.0)
    # without the Double declaration the same words compare bitwise
    ids, t, _ = O.put_batch(["zero"], np.zeros((1, 32), np.uint8), [("zero", d(0.0))])
    ids, t, _ = O.put_batch(ids, t, [("zero", d(-0.0))])
    assert flags(t) == [EX | CH]


def test_err_idx_and_error_flags_are_cleared():
    t = np.zeros((2, 16), np.uint8)
    t[:, 8:16] = np.frombuffer(struct.pack("<II", EX | CH | O.ERROR, 3) * 1, np.uint8)
    ids, out, _ = O.put_batch(["a", "b"], t, [("a", b"\1" * 8)])
    assert flags(out) == [EX | CH, EX]
    assert not out[:, 12:16].any()


def test_arguments_are_checked_before_any_device():
    lib = N.load_library()
    offs = np.array([0, 1, 2], np.uint32)
    rows = np.zeros(16, np.uint8)
    pres = np.ones(2, np.uint8)
    keys = np.frombuffer(b"ab", np.uint8)
    assert lib.sgr_put_batch(None, keys.ctypes.data, offs.ctypes.data, 2, rows.ctypes.data, pres.ctypes.data, None) == N.SGR_ERR_INVALID
    n_new = C.c_uint64(5)
    assert lib.sgr_put_batch(None, None, None, 0, None, None, C.byref(n_new)) == N.SGR_ERR_INVALID


class FakeEngine:
    def __init__(self, device=0):
        self.state_bytes = 0
        self.calls = []

    def register_program(self, prog):
        self.state_bytes = int(prog.state_bytes)

    def put_batch(self, ids, rows, present=None):
        self.calls.append(("put_batch", list(ids), rows.copy(), list(present)))
        return 0

    def load_keys(self, keys):
        self.calls.append(("load_keys",))

    def __getattr__(self, name):
        def call(*a, **k):
            self.calls.append((name,))
        return call


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(ST, "ReplayEngine", FakeEngine)


def wide_program():
    return P.make_program(96, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])])


def test_state_topic_store_refuses_the_event_feeds(fake):
    st = ST.GpuReplayKeyValueStore("s", wide_program(), codec=ST.StateCodec(lambda k, v: v, lambda k, b: b))
    st.init()
    with pytest.raises(N.SgrError):
        st.put_event("a", b"\0" * 64)
    with pytest.raises(N.SgrError):
        st.restore_record_batches(0, b"")
    with pytest.raises(ValueError):
        st.put("a", b"\0" * 89)
    with pytest.raises(ValueError):
        ST.StateCodec(lambda k, v: v, lambda k, b: b, snapshot_type=4)


def test_state_topic_store_flushes_one_put_batch_and_no_key_table(fake):
    st = ST.GpuReplayKeyValueStore("s", wide_program(), codec=ST.StateCodec(lambda k, v: v, lambda k, b: b))
    st.init()
    st.put("a", b"\1" * 88)            # wider than a 48-byte snapshot record
    st.putAll([("b", b"\2" * 3), ("c", None)])
    assert st.delete("a") == b"\1" * 88
    assert st.get("a") is None and st.get("b") == b"\2" * 3
    st.flush()
    calls = [c for c in st.engine.calls if c[0] in ("put_batch", "load_keys", "fold_incremental", "set_initial_states")]
    assert [c[0] for c in calls] == ["put_batch"]
    _, ids, rows, present = calls[0]
    assert ids == ["a", "b", "c", "a"] and present == [True, True, False, False]
    assert rows[0].tobytes() == b"\1" * 88 and rows[1, :3].tobytes() == b"\2" * 3 and not rows[1, 3:].any()
