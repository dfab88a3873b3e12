"""-m gpu: back-to-back asynchronous folds on the record-parallel runs kernel (fold_runs.cu).

Consecutive folds overlap on the device (programmatic dependent launch) and hand out the log in chunks by ticket, so
every result of a pipeline of fold_async calls, queued without a wait in between, is checked bit for bit against the
oracle (and so against one synchronous fold): throwing segments, more of them than the replay list holds, folds on top
of prior states, one segment across thousands of chunks, empty and tiny logs, trailing empty segments, many folds in a
row, and the 64-byte class-1 program.
"""
import uuid

import numpy as np
import pytest

from oracle import oracle as O
from surge_b200 import ReplayEngine
from surge_b200 import formats as F
from surge_b200 import programs as P
from surge_b200 import synth as S

pytestmark = pytest.mark.gpu

# 2 KiB chunks are clamped to the variant's stage count: many chunks even on small logs
CHUNKS = [None, 2048]


def assert_same(got, want, what=""):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:8]}")


def pipelined(prog, rec, off, k, *, chunk=None, init=None, from_none=True, kernel=0):
    """k fold_async calls with no wait in between; returns the table, the stats and one synchronous fold's table.
    Under automatic selection ("kernel" 0) the Counter folds from the head plane (stats().head_plane 1); the same pipeline
    is then run again with "head_plane" 0, on the log, and must give the same tables and counts."""
    arms = []
    for head_plane in ([1, 0] if kernel == 0 else [1]):
        with ReplayEngine(0) as e:
            e.register_program(prog)
            e.set_option("kernel", kernel)
            e.set_option("head_plane", head_plane)
            if chunk is not None:
                e.set_option("run_chunk_bytes", chunk)
            if init is not None:
                e.set_initial_states(init)
            e.load_events(rec, off)
            for _ in range(k):
                if from_none:
                    e.set_initial_states(None)
                e.fold_async()
            e.wait()
            got, st = e.export_states(), e.stats()
            if init is not None:
                e.set_initial_states(init)
            else:
                e.set_initial_states(None)
            e.fold()
            one = e.export_states()
            want_plane = int(kernel == 0 and head_plane == 1)
            assert st.head_plane == want_plane and e.stats().head_plane == want_plane, f"head_plane {st.head_plane}, expected {want_plane}"
        arms.append((got, st, one))
    got, st, one = arms[0]
    for got_log, st_log, one_log in arms[1:]:
        assert_same(got_log, got, "pipelined, head_plane 0 against the plane")
        assert_same(one_log, one, "synchronous, head_plane 0 against the plane")
        assert (st_log.n_events, st_log.n_errors) == (st.n_events, st.n_errors)
    return got, st, one


@pytest.mark.parametrize("chunk", CHUNKS)
def test_pipelined_folds_with_throws(chunk):
    rng = np.random.default_rng(11)
    counts = rng.integers(0, 60, size=30000)
    rec, off = S.counter_csr(len(counts), counts, seed=11, p_throw=0.004)
    want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    assert nerr > 0
    got, st, one = pipelined(P.counter_program(), rec, off, 6, chunk=chunk)
    assert_same(got, want, "pipelined")
    assert_same(one, want, "synchronous")
    assert (st.n_events, st.n_errors) == (nev, nerr)
    assert st.fold_launches == 1 and st.ms_fold > 0


def test_pipelined_folds_replay_list_overflow():
    # more throwing aggregates than the replay list holds (2^20): the host refolds the last fold sequentially
    n_agg = (1 << 20) + 3000
    rec, off = S.counter_csr(n_agg, 1, seed=12, p_incr=0.0, p_decr=0.0, p_throw=1.0)
    want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    assert nerr == n_agg
    got, st, _ = pipelined(P.counter_program(), rec, off, 3)
    assert_same(got, want)
    assert (st.n_events, st.n_errors) == (nev, nerr)


@pytest.mark.parametrize("chunk", CHUNKS)
def test_pipelined_folds_on_prior_states(chunk):
    rng = np.random.default_rng(13)
    counts = rng.integers(0, 40, size=8000)
    counts[100] = 0
    rec, off = S.counter_csr(len(counts), counts, seed=13, p_throw=0.002)
    init, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, *S.counter_csr(len(counts), 3, seed=14))
    want = init
    for _ in range(4):
        want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off, want)
    got, st, one = pipelined(P.counter_program(), rec, off, 4, chunk=chunk, init=init, from_none=False)
    assert_same(got, want, "four folds in place")
    assert (st.n_events, st.n_errors) == (nev, nerr)
    want1, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off, init)
    assert_same(one, want1, "one synchronous fold")


@pytest.mark.parametrize("chunk", CHUNKS)
def test_pipelined_hot_segment_across_thousands_of_chunks(chunk):
    counts = np.full(4000, 5, dtype=np.int64)
    counts[1234] = 400_000  # 25.6 MB: thousands of chunks inside one segment
    counts[-3:] = 0         # trailing empty segments
    rec, off = S.counter_csr(len(counts), counts, seed=15, p_throw=0.00001)
    want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    got, st, one = pipelined(P.counter_program(), rec, off, 3, chunk=chunk)
    assert_same(got, want, "pipelined")
    assert_same(one, want, "synchronous")
    assert (st.n_events, st.n_errors) == (nev, nerr)


@pytest.mark.parametrize("counts", [[0, 0, 0], [1], [3, 0, 0], [0, 0, 2, 0], [64], [0, 128, 0, 0, 0]],
                         ids=["empty", "one-record", "trailing-empty", "leading-empty", "one-step", "one-step-padded"])
def test_pipelined_tiny_logs(counts):
    counts = np.asarray(counts, dtype=np.int64)
    rec, off = S.counter_csr(len(counts), counts, seed=16)
    want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    got, st, one = pipelined(P.counter_program(), rec, off, 5, kernel=2)
    assert_same(got, want, "pipelined")
    assert_same(one, want, "synchronous")
    assert (st.n_events, st.n_errors) == (nev, nerr)


def test_many_pipelined_folds():
    # hundreds of folds in one queue: the counter blocks alternate and every fold cleans the next one's
    rng = np.random.default_rng(17)
    counts = rng.integers(0, 30, size=5000)
    rec, off = S.counter_csr(len(counts), counts, seed=17, p_throw=0.003)
    want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    got, st, _ = pipelined(P.counter_program(), rec, off, 301, chunk=2048)
    assert_same(got, want)
    assert (st.n_events, st.n_errors) == (nev, nerr)


@pytest.mark.parametrize("chunk", CHUNKS)
def test_pipelined_folds_wrap_the_lookback_epoch(chunk):
    # the look-back flags compare against a 32-bit epoch per fold: start a few folds short of 2^32 so the queue wraps it
    # (the flags are cleared on the wrap) with folds still in flight on both sides of it
    rng = np.random.default_rng(19)
    counts = rng.integers(0, 50, size=12000)
    counts[5] = 30_000
    rec, off = S.counter_csr(len(counts), counts, seed=19, p_throw=0.002)
    want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        if chunk is not None:
            e.set_option("run_chunk_bytes", chunk)
        e.load_events(rec, off)
        e.fold()
        e.set_option("lookback_epoch", (1 << 32) - 3)
        for _ in range(7):
            e.set_initial_states(None)
            e.fold_async()
        e.wait()
        assert_same(e.export_states(), want)
        st = e.stats()
        assert (st.n_events, st.n_errors) == (nev, nerr)


def test_small_log_uses_every_warp_slot():
    # a 6.4 MB log (one configs[4]-sized batch) is cut into one-step chunks, as many as the log has steps
    rec, off = S.counter_csr(100_000, 1, seed=20)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    got, st, one = pipelined(P.counter_program(), rec, off, 3)
    assert_same(got, want)
    assert_same(one, want)
    assert st.ms_fold > 0


@pytest.mark.parametrize("chunk", CHUNKS)
def test_pipelined_wide_program(chunk):
    # BankAccount: 64-byte states (W = 14), IF_EXISTS rule (class 1), forced onto the runs kernel
    rng = np.random.default_rng(18)
    n_agg = 3000
    blobs, counts = [], []
    for a in range(n_agg):
        k = int(rng.integers(0, 10)) if a != 7 else 3000
        acct = str(uuid.UUID(int=a + 1))
        evs = []
        for j in range(k):
            if rng.random() < 0.2:
                evs.append(F.bank_created_record(a, j + 1, acct, f"owner{a % 31}", f"{a % 10000:04d}", 10.0 + j))
            else:
                evs.append(F.bank_updated_record(a, j + 1, acct, float(rng.integers(-5, 5))))
        blobs.append(b"".join(evs))
        counts.append(k)
    rec = np.frombuffer(b"".join(blobs), dtype=np.uint8)
    off = F.csr_offsets_from_counts(counts)
    want, _, _ = O.fold_packed(O.MODEL_BANK_ACCOUNT, O.REC_FIXED64, rec, off)
    got, st, one = pipelined(P.bank_account_program(), rec, off, 4, chunk=chunk, kernel=2)
    assert_same(got, want, "pipelined")
    assert_same(one, want, "synchronous")
    assert st.fold_launches == 1
