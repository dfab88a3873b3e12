"""-m gpu: the head plane — the runs fold staging each record's 32-byte head from a dense copy instead of the 64-byte log.

A program whose every record read lies in words 0..7 (RowProgram::head_only: Counter, IntBalance) folds a fixed-record log
with 64-byte aligned segments from the head plane: bytes 0..31 of every record, 32 bytes apart, built behind the copy of
a host load or by the first fold of a borrowed device log. Every case compares whole state tables (err_idx included) and
stats().n_events / n_errors with the compiled program oracle and with the same fold on the log ("head_plane" 0), and reads
stats().head_plane to see which one ran:

  a. Counter and IntBalance on a configs[1]-shaped log, a log that starts past byte 0, empty segments at both ends and in
     the middle, one segment across many chunks, throwing events (the in-kernel replay), a log shorter than one step and a
     log of empty segments only; from None and on prior states; host-loaded and borrowed from a device tensor;
  b. random head-only programs of oracle/program_corpus.py (16- and 32-byte states, class 0 and 1), every head variant;
  c. a program reading word 8 or higher, and every forced kernel option, fold the log;
  d. a new program or a new load drops the plane; overlapped fold_async calls stage it before their griddepcontrol.wait.
"""
import numpy as np
import pytest

from oracle import program_corpus as PC
from oracle import program_interp as I
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P

pytestmark = pytest.mark.gpu

HEAD_WORDS = [1, 4, 5, 6, 7]      # the record words a head-only corpus program may read (0 is the type, 2..3 the aggregate)
N_HEAD_VARIANTS = 5
COUNTER = [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)]),
           (I.MATERIALISE, [(I.OP_SUB_I32, 0, 16, 4), (I.OP_SET, 4, 4, 4)]), (I.MATERIALISE, []), (I.THROW, [])]
INT_BALANCE = [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 16, 4)])]
NAMED = {"counter": (P.counter_program, COUNTER), "int_balance": (P.int_balance_program, INT_BALANCE)}


def same(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:6]}\n got {got[bad[0]].tolist()}\nwant {want[bad[0]].tolist()}")


def check(e, want, nev, nerr, plane, what):
    same(e.export_states(), want, what)
    st = e.stats()
    assert (st.n_events, st.n_errors) == (nev, nerr), f"{what}: stats (n_events, n_errors) = {(st.n_events, st.n_errors)}, oracle {(nev, nerr)}"
    assert st.head_plane == plane, f"{what}: head_plane = {st.head_plane}, expected {plane}"


def oracle(rules, sb, log, seg, prior=None):
    return I.c_fold(rules, sb, log[int(seg[0]):], seg, initial=prior)


def fold(e, prior=None):
    e.set_initial_states(prior)
    e.fold()


def make_log(rng, rules, counts, pad_records=0, p_throw=1e-3):
    buf, seg, _ = PC.fixed_log(rng, rules, np.asarray(counts, np.int64), pad_records=pad_records, p_throw=p_throw)
    return buf.reshape(-1), seg


def shaped_logs(rng, rules):
    """(name, log, seg, plane): the log shapes of case a; plane: whether the fold can take the head plane."""
    out = [("configs1_shape", *make_log(rng, rules, np.full(1 << 16, 32)), 1)]
    counts = rng.geometric(1 / 9, size=40_000) - 1
    out.append(("log_begin_past_0", *make_log(rng, rules, counts, pad_records=37), 1))
    counts = rng.geometric(1 / 20, size=30_000) - 1
    counts[:2000] = 0
    counts[14_000:16_000] = 0
    counts[-2000:] = 0
    counts[rng.integers(0, len(counts), size=3000)] = 0
    out.append(("empty_segments", *make_log(rng, rules, counts), 1))
    counts = rng.geometric(1 / 5, size=5000) - 1
    counts[1234] = 1_500_000                                       # 96 MiB: hundreds of ticketed chunks without a head
    out.append(("one_segment_across_chunks", *make_log(rng, rules, counts, p_throw=0.0), 1))
    out.append(("shorter_than_one_step", *make_log(rng, rules, [3, 0, 5, 1, 0], p_throw=0.0), 1))
    out.append(("empty_segments_only", *make_log(rng, rules, np.zeros(100, np.int64), pad_records=2), 0))
    return out


def prior_of(rng, want):
    prior = want.copy()
    prior[rng.random(len(prior)) < 0.2] = 0
    return prior


# ------------------------------------------------------------------ a. Counter and IntBalance, plane against log
@pytest.mark.parametrize("name", sorted(NAMED))
def test_named_programs_fold_the_same_table_from_the_plane(name):
    import torch

    make, rules = NAMED[name]
    rng = np.random.default_rng(91000 + sum(map(ord, name)))
    for shape, log, seg, plane in shaped_logs(rng, rules):
        want, nev, nerr = oracle(rules, 16, log, seg)
        prior = prior_of(rng, want)
        want2, nev2, nerr2 = oracle(rules, 16, log, seg, prior=prior)
        if shape in ("configs1_shape", "log_begin_past_0", "empty_segments"):
            assert nerr > 0, shape                                 # throwing segments: the in-kernel replay runs
        what = f"{name}, {shape}"
        tables = {}
        for src in ("host", "device"):
            with ReplayEngine(0) as e:
                e.register_program(make())
                if src == "host":
                    e.load_events(log, seg)
                else:
                    e.load_events(torch.from_numpy(log).cuda(), torch.from_numpy(seg.astype(np.int64)).cuda())
                fold(e)
                check(e, want, nev, nerr, plane, f"{what}, {src} load: plane")
                tables[src] = e.export_states()
                fold(e, prior)
                check(e, want2, nev2, nerr2, plane, f"{what}, {src} load: plane on prior states")
                e.set_option("head_plane", 0)
                fold(e)
                check(e, want, nev, nerr, 0, f"{what}, {src} load: log")
                fold(e, prior)
                check(e, want2, nev2, nerr2, 0, f"{what}, {src} load: log on prior states")
        same(tables["device"], tables["host"], f"{what}: borrowed against host-loaded log")


# ------------------------------------------------------------------ b. random head-only programs
@pytest.mark.parametrize("W,cls", [(2, 0), (2, 1), (6, 0), (6, 1)])
def test_random_head_only_programs(W, cls, monkeypatch):
    monkeypatch.setattr(PC, "SOURCE_WORDS", HEAD_WORDS)
    rng = np.random.default_rng(92000 + 10 * W + cls)
    sb = 4 * W + 8
    for i in range(4):
        rules = PC.row_program(rng, W, cls, int(rng.integers(1, len(HEAD_WORDS) + 1)))
        counts = rng.geometric(1 / 12, size=30_000) - 1
        counts[int(rng.integers(0, len(counts)))] = 200_000
        log, seg = make_log(rng, rules, counts, pad_records=int(rng.integers(0, 3)))
        want, nev, nerr = oracle(rules, sb, log, seg)
        prior = prior_of(rng, want)
        want2, nev2, nerr2 = oracle(rules, sb, log, seg, prior=prior)
        what = f"W{W} class {cls} program {i} {rules}"
        with ReplayEngine(0) as e:
            e.register_program(P.make_program(sb, N.REC_FIXED64, rules))
            e.load_events(log, seg)
            for v in range(N_HEAD_VARIANTS) if W == 2 and cls == 0 else [0]:
                e.set_option("head_variant", v)
                fold(e)
                check(e, want, nev, nerr, 1, f"{what}: head variant {v}")
                fold(e, prior)
                check(e, want2, nev2, nerr2, 1, f"{what}: head variant {v} on prior states")


# ------------------------------------------------------------------ c. what keeps the fold on the log
def test_a_program_reading_word_8_or_higher_folds_the_log():
    rng = np.random.default_rng(93000)
    for word in (8, 15):
        rules = [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 4 * word, 4), (I.OP_SET, 4, 4, 4)]), (I.THROW, [])]
        log, seg = make_log(rng, rules, rng.geometric(1 / 10, size=20_000) - 1)
        want, nev, nerr = oracle(rules, 16, log, seg)
        with ReplayEngine(0) as e:
            e.register_program(P.make_program(16, N.REC_FIXED64, rules))
            e.load_events(log, seg)
            fold(e)
            check(e, want, nev, nerr, 0, f"a program reading word {word}")


def test_forced_kernel_options_fold_the_log():
    rng = np.random.default_rng(93100)
    log, seg = make_log(rng, COUNTER, rng.geometric(1 / 10, size=20_000) - 1)
    want, nev, nerr = oracle(COUNTER, 16, log, seg)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_events(log, seg)
        for opt, val in (("kernel", 2), ("kernel", 3), ("kernel", 1)):
            e.set_option(opt, val)
            fold(e)
            check(e, want, nev, nerr, 0, f"{opt} {val}")
        e.set_option("kernel", 0)
        fold(e)
        check(e, want, nev, nerr, 1, "kernel 0")
        e.set_option("run_variant", 0)
        fold(e)
        check(e, want, nev, nerr, 0, "run_variant 0")
        e.set_option("run_variant", -1)   # automatic selection again, as on a fresh engine
        fold(e)
        check(e, want, nev, nerr, 1, "run_variant -1 after run_variant 0")
        with pytest.raises(SgrError) as ei:
            e.set_option("run_variant", -2)
        assert ei.value.code == N.SGR_ERR_INVALID


# ------------------------------------------------------------------ d. the plane's lifetime
def test_new_program_and_new_load_drop_the_plane():
    import torch

    rng = np.random.default_rng(94000)
    word9 = [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 36, 4)]), (I.MATERIALISE, [(I.OP_SET, 4, 4, 4)])]
    logs = [make_log(rng, COUNTER, rng.geometric(1 / 10, size=30_000) - 1, pad_records=k) for k in (0, 5)]
    for src in ("host", "device"):
        with ReplayEngine(0) as e:
            for i, (log, seg) in enumerate(logs):
                what = f"{src} load {i}"
                e.register_program(P.counter_program())
                if src == "host":
                    e.load_events(log, seg)
                else:
                    e.load_events(torch.from_numpy(log).cuda(), torch.from_numpy(seg.astype(np.int64)).cuda())
                fold(e)
                check(e, *oracle(COUNTER, 16, log, seg), 1, f"{what}: Counter")
                e.register_program(P.int_balance_program())
                fold(e)
                check(e, *oracle(INT_BALANCE, 16, log, seg), 1, f"{what}: IntBalance registered after the load")
                e.register_program(P.make_program(16, N.REC_FIXED64, word9))
                fold(e)
                check(e, *oracle(word9, 16, log, seg), 0, f"{what}: a program reading word 9")
                e.register_program(P.counter_program())
                fold(e)
                check(e, *oracle(COUNTER, 16, log, seg), 1, f"{what}: Counter again")


def test_overlapped_folds_from_the_plane():
    rng = np.random.default_rng(95000)
    log, seg = make_log(rng, COUNTER, np.full(1 << 15, 32))
    want, nev, nerr = oracle(COUNTER, 16, log, seg)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_events(log, seg)
        e.set_option("head_plane", 0)
        e.set_initial_states(None)
        e.fold_async()
        e.set_option("head_plane", 1)
        for _ in range(4):                # the first builds nothing (the host load did) but follows a fold of the log
            e.set_initial_states(None)
            e.fold_async()
        e.wait()
        check(e, want, nev, nerr, 1, "four fold_async calls behind a fold of the log")
        e.register_program(P.counter_program())
        for _ in range(3):                # the first rebuilds the plane, the others overlap it
            e.set_initial_states(None)
            e.fold_async()
        e.wait()
        check(e, want, nev, nerr, 1, "three fold_async calls, the first building the plane")
