"""CPU checks of the batched recovery read: the C entry point refuses a NULL engine, and AggregateStateStore's coalescing reader
(coalesce_reads_us > 0) turns getAggregateBytes calls that arrive within its window into one store.get_many, routes each row to
its own future and hands a batch's failure to every future of that batch. A fake store stands in for the GPU one."""
import ctypes as C
import threading
import time

import pytest

from surge_b200 import native as N
from surge_b200.store import AggregateStateStore


def test_get_batch_refuses_a_null_engine():
    lib = N.load_library()
    offs = (C.c_uint32 * 2)(0, 1)
    out = C.create_string_buffer(64)
    assert lib.sgr_get_batch(None, b"a", offs, 1, out, 64, None, None) == N.SGR_ERR_INVALID
    assert lib.sgr_get_batch(None, None, None, 0, None, 0, None, None) == N.SGR_ERR_INVALID


class FakeStore:
    def __init__(self, fail=None, delay=0.0):
        self.batches, self.gets = [], []
        self.fail, self.delay = fail, delay
        self.lock = threading.Lock()

    def isOpen(self):  # noqa: N802
        return True

    def get(self, key):
        with self.lock:
            self.gets.append(key)
        return f"row:{key}".encode()

    def get_many(self, keys):
        with self.lock:
            self.batches.append(list(keys))
        time.sleep(self.delay)
        if self.fail is not None:
            raise self.fail
        return [None if k.startswith("none") else f"row:{k}".encode() for k in keys]


def test_reads_within_a_window_become_one_get_many():
    st = FakeStore()
    ag = AggregateStateStore(st, threads=4, coalesce_reads_us=200_000)
    try:
        ids = [f"a{i}" for i in range(50)] + ["none-1", "a3"]
        futs = [ag.getAggregateBytes(k) for k in ids]
        got = [f.result(timeout=10) for f in futs]
    finally:
        ag.stop()
    assert len(st.batches) == 1 and sorted(st.batches[0]) == sorted(ids)
    assert st.gets == []
    assert got == [None if k.startswith("none") else f"row:{k}".encode() for k in ids]


def test_results_are_routed_to_their_own_futures_across_windows():
    st = FakeStore()
    ag = AggregateStateStore(st, threads=8, coalesce_reads_us=2_000)
    futs = {}
    try:
        for i in range(400):
            futs[f"k{i}"] = ag.getAggregateBytes(f"k{i}")
            if i % 50 == 0:
                time.sleep(0.01)   # close the window now and then: several batches
        for k, f in futs.items():
            assert f.result(timeout=10) == f"row:{k}".encode()
    finally:
        ag.stop()
    assert len(st.batches) >= 2
    assert sorted(k for b in st.batches for k in b) == sorted(futs)


def test_an_exception_reaches_every_future_of_its_batch():
    err = RuntimeError("device says no")
    st = FakeStore(fail=err)
    ag = AggregateStateStore(st, threads=2, coalesce_reads_us=100_000)
    try:
        futs = [ag.getAggregateBytes(f"x{i}") for i in range(10)]
        for f in futs:
            with pytest.raises(RuntimeError, match="device says no"):
                f.result(timeout=10)
    finally:
        ag.stop()
    assert len(st.batches) == 1


def test_no_window_never_calls_get_many():
    st = FakeStore()
    ag = AggregateStateStore(st, threads=4)
    try:
        futs = [ag.getAggregateBytes(f"p{i}") for i in range(20)]
        assert [f.result(timeout=10) for f in futs] == [f"row:p{i}".encode() for i in range(20)]
    finally:
        ag.stop()
    assert st.batches == [] and sorted(st.gets) == sorted(f"p{i}" for i in range(20))


def test_batch_read_goes_to_get_many_in_one_call():
    st = FakeStore()
    ag = AggregateStateStore(st, threads=2)
    try:
        assert ag.getAggregateBytesBatch(["a", "none-b", "c"]).result(timeout=10) == [b"row:a", None, b"row:c"]
    finally:
        ag.stop()
    assert st.batches == [["a", "none-b", "c"]]
