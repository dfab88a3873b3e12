"""-m gpu: the slot-plane fold's chunk table. A fold from the slot plane starts each ticketed chunk from a per-log table of
first boundaries (engine.cu ensure_chunk_table, fold_runs.cu build_chunk_table_kernel) and loads the next chunk's entry and
boundary window while it folds the current one, instead of searching the offsets at every chunk switch.

Every case is checked against oracle/program_oracle.c (the whole state table, err_idx included, and stats().n_events /
n_errors) and against the same fold with "head_plane" 0 (the log, which searches the offsets). Each slot-plane fold asserts
stats().chunk_table, so a case cannot fall back to the search unnoticed.

  a. run_chunk_bytes 2048 (one step per chunk), 16 KiB, the default and 2^30 (the most steps the warps leave), every projected
     variant at the extremes, on a log with a hot segment over many chunks, throws and runs of empty segments;
  b. segments that end exactly on chunk edges, and empty segments at a chunk's first step;
  c. small logs, where the chunk shrinks to the warp count;
  d. more throwing segments than the replay list holds;
  e. overlapped fold_async calls that change run_chunk_bytes or proj_variant while a fold is pending (the table is rebuilt);
  f. host loads around the 1 M-record plane-build chunk; borrowed logs at several 16-byte address classes;
  g. register_program and a reload with other offsets drop the table with the plane.
"""
import numpy as np
import pytest

from oracle import program_corpus as PC
from oracle import program_interp as I
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import native as N
from surge_b200 import programs as P

pytestmark = pytest.mark.gpu

PROJ_VARIANTS = 4        # fold_runs.cu kProjVariants
STEP_RECS = 256          # records per step of every projected variant (R = 8: 2048 * 8 log bytes)
BUILD_CHUNK = 1 << 20    # records per chunk of a host load's plane build (engine.cu sgr_load_events)


def same(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:6]}\n got {got[bad[0]].tolist()}\nwant {want[bad[0]].tolist()}")


def check(e, want, nev, nerr, plane, what):
    same(e.export_states(), want, what)
    st = e.stats()
    assert (st.n_events, st.n_errors) == (nev, nerr), f"{what}: stats (n_events, n_errors) = {(st.n_events, st.n_errors)}, oracle {(nev, nerr)}"
    expect = (16, 1) if plane else (0, 0)
    assert (st.plane_bytes, st.chunk_table) == expect, f"{what}: (plane_bytes, chunk_table) = {(st.plane_bytes, st.chunk_table)}, expected {expect}"


def oracle(rules, log, seg, prior=None):
    return I.c_fold(rules, 16, log[int(seg[0]):], seg, initial=prior)


def fold(e, prior=None):
    e.set_initial_states(prior)
    e.fold()


def both_ways(e, rules, log, seg, what, prior=None):
    """The fold from the slot plane (chunk table) and from the log (offset search), from `prior`, against the oracle."""
    want = oracle(rules, log, seg, prior)
    for plane in (1, 0, 1):
        e.set_option("head_plane", plane)
        fold(e, prior)
        check(e, *want, plane, f"{what}: {'slot plane' if plane else 'log'}")
    return want


def counts_summing_to(rng, n_rec, p):
    """Per-aggregate counts, geometric with parameter p, that add up to exactly n_rec records."""
    counts = rng.geometric(p, size=n_rec + 1) - 1
    counts[-1] += max(0, n_rec - int(counts.sum()))
    cum = np.cumsum(counts)
    k = int(np.searchsorted(cum, n_rec))
    counts = counts[:k + 1].copy()
    counts[-1] -= int(cum[k]) - n_rec
    return counts


def throw_type(rules):
    return next((t for t, (ex, _) in enumerate(rules) if ex == I.THROW), len(rules))


def hot_log(rng, rules, n_agg=300_000, hot=200_000):
    """About 3.5 M records, enough steps that chunks keep several steps with every warp resident: a calm hot segment of `hot` records across many chunks, a segment whose first record throws, runs of 700 empty
    segments at the start, the middle and the end, from byte 64 * pad."""
    counts = rng.geometric(1 / 12, size=n_agg) - 1
    for a in (0, n_agg // 2, n_agg - 700):
        counts[a:a + 700] = 0
    big, first = 1501, n_agg // 4
    counts[big] = hot
    counts[first] = 5000
    buf, seg, _ = PC.fixed_log(rng, rules, counts, pad_records=int(rng.integers(1, 6)), p_throw=1e-3)
    rec = buf.reshape(-1, 64)[int(seg[big]) // 64:int(seg[big + 1]) // 64]
    types = rec[:, 0:4].copy().view(np.uint32).ravel()
    rec[(types >= len(rules)) | np.isin(types, [t for t, (ex, _) in enumerate(rules) if ex == I.THROW]), 0:4] = 0
    PC.set_type(buf, seg, first, 0, throw_type(rules))
    return buf.reshape(-1), seg


# ------------------------------------------------------------------ a. chunk sizes x projected variants
CHUNKS = [(c, v) for c in (2048, 1 << 30) for v in range(PROJ_VARIANTS)] + [(16384, 0), (131072, 0), (131072, 3)]


@pytest.mark.parametrize("chunk,pv", CHUNKS, ids=[f"chunk{c}-pv{v}" for c, v in CHUNKS])
def test_chunk_sizes(chunk, pv):
    rng = np.random.default_rng(99000 + pv + chunk % 9973)
    rules = PC.head_only_program(rng, 2, 0, int(rng.integers(2, 5)))
    log, seg = hot_log(rng, rules)
    what = f"run_chunk_bytes {chunk}, proj_variant {pv}"
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.set_option("run_chunk_bytes", chunk)
        e.set_option("proj_variant", pv)
        e.load_events(log, seg)
        want = both_ways(e, rules, log, seg, what)
        both_ways(e, rules, log, seg, f"{what}, on its own result", prior=want[0])


# ------------------------------------------------------------------ b. segment boundaries on chunk edges
@pytest.mark.parametrize("chunk_steps", [1, 2, 3])
def test_boundaries_on_chunk_edges(chunk_steps):
    """Segments of whole chunks, segments that end one record before or after an edge, and runs of empty segments right at
    a chunk's first record. The log has about 3000 chunks, more than there are resident warps, so the chunk keeps its size."""
    rng = np.random.default_rng(99100 + chunk_steps)
    rules = PC.head_only_program(rng, 2, 0, 3)
    ch = chunk_steps * STEP_RECS
    counts, total = [], 0
    while total < 3000 * ch:
        kind = int(rng.integers(0, 4))
        if kind == 0:
            counts += [ch * int(rng.integers(1, 4))]                       # whole chunks: ends on an edge
        elif kind == 1:
            counts += [0] * int(rng.integers(1, 40)) + [ch]                # empty segments at the chunk's first record
        else:
            n = ch - total % ch + int(rng.choice([-1, 0, 1]))              # around the next edge
            counts += [n if n > 0 else ch]
        total += counts[-1]
    counts[len(counts) // 3] = 25 * ch                                    # one segment over many chunks
    counts += [0] * 5
    buf, seg, _ = PC.fixed_log(rng, rules, np.asarray(counts), pad_records=0, p_throw=5e-4)
    log = buf.reshape(-1)
    ends = (seg[1:] - seg[0]) // 64
    assert ((ends % ch == 0) & (np.diff(seg) > 0)).sum() > 100, "segments ending on chunk edges"
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.set_option("run_chunk_bytes", chunk_steps * STEP_RECS * 64)
        e.load_events(log, seg)
        both_ways(e, rules, log, seg, f"chunks of {chunk_steps} steps, boundaries on their edges")


# ------------------------------------------------------------------ c. small logs
@pytest.mark.parametrize("pv", [0, 3])
@pytest.mark.parametrize("n_rec", [1, 255, 257, 5000, 200_000])
def test_small_logs(n_rec, pv):
    """Fewer steps than resident warps: chunks shrink to one step (NSTAGE - 1 for deeper variants)."""
    rng = np.random.default_rng(99200 + n_rec + pv)
    rules = PC.head_only_program(rng, 2, 0, 4)
    counts = counts_summing_to(rng, n_rec, 1 / 6)
    buf, seg, _ = PC.fixed_log(rng, rules, counts, pad_records=2, p_throw=1e-3)
    log = buf.reshape(-1)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.set_option("proj_variant", pv)
        e.load_events(log, seg)
        both_ways(e, rules, log, seg, f"{n_rec} records, proj_variant {pv}")


# ------------------------------------------------------------------ d. replay-list overflow
def test_replay_list_overflow():
    """More throwing aggregates than the replay list holds (2^20): the host refolds the whole log sequentially."""
    rng = np.random.default_rng(99300)
    rules = PC.head_only_program(rng, 2, 0, 4)
    n_throw = (1 << 20) + 3000
    counts = rng.integers(1, 3, size=n_throw + 100_000)
    counts[5] = 6000
    buf, seg, _ = PC.fixed_log(rng, rules, counts, pad_records=1, p_throw=0.0)
    rec = buf.reshape(-1, 64)
    rec[np.asarray(seg[:n_throw] // 64, np.int64), 0:4] = np.frombuffer(np.uint32(len(rules)).tobytes(), np.uint8)
    log = buf.reshape(-1)
    want, nev, nerr = oracle(rules, log, seg)
    assert nerr == n_throw
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.set_option("run_chunk_bytes", 16384)
        e.load_events(log, seg)
        for p in (1, 0):
            e.set_option("head_plane", p)
            fold(e)
            same(e.export_states(), want, f"replay overflow, head_plane {p}")
            st = e.stats()
            assert (st.n_events, st.n_errors) == (nev, nerr)
            with pytest.raises(SgrError) as ei:
                fold(e, want)
            assert ei.value.code == N.SGR_ERR_UNSUPPORTED


# ------------------------------------------------------------------ e. the table rebuilt under pending folds
def test_table_rebuilt_between_pending_folds():
    """fold_async calls queued without a wait, each folding onto the table the one before it wrote, with run_chunk_bytes or
    proj_variant changed between them: each change rebuilds the table behind the fold still running."""
    rng = np.random.default_rng(99400)
    rules = PC.head_only_program(rng, 2, 0, 3)
    log, seg = hot_log(rng, rules)
    chain = [(131072, 0), (131072, 0), (2048, 0), (2048, 0), (2048, 3), (1 << 30, 3), (1 << 30, 1), (16384, 1), (131072, 0),
             (131072, 0)]
    wants = [oracle(rules, log, seg)]
    for _ in chain[1:]:
        wants.append(oracle(rules, log, seg, prior=wants[-1][0]))
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.load_events(log, seg)
        e.set_initial_states(None)
        for chunk, pv in chain:
            e.set_option("run_chunk_bytes", chunk)
            e.set_option("proj_variant", pv)
            e.fold_async()
        e.wait()
        check(e, *wants[-1], 1, f"{len(chain)} overlapped folds: {chain}")


# ------------------------------------------------------------------ f. host loads, borrowed logs
@pytest.mark.parametrize("n_rec", [BUILD_CHUNK - 1, BUILD_CHUNK + 1], ids=["1Mrec-1", "1Mrec+1"])
def test_host_load_across_the_build_chunk(n_rec):
    rng = np.random.default_rng(99500 + n_rec % 1000)
    rules = PC.head_only_program(rng, 2, 0, 4)
    counts = counts_summing_to(rng, n_rec, 1 / 9)
    rec, seg0, _ = PC.fixed_log(rng, rules, counts, p_throw=2e-4)
    tail = rng.integers(0, 256, size=480, dtype=np.uint8)
    for begin in (0, 208):
        log = np.concatenate([rng.integers(0, 256, size=begin, dtype=np.uint8), rec.reshape(-1), tail])
        seg = seg0 + np.uint64(begin)
        with ReplayEngine(0) as e:
            e.register_program(P.make_program(16, N.REC_FIXED64, rules))
            e.set_option("run_chunk_bytes", 16384)
            e.load_events(log, seg)
            both_ways(e, rules, log, seg, f"host load of {n_rec} records from byte {begin}")


def test_borrowed_log_at_16_byte_address_classes():
    import torch

    rng = np.random.default_rng(99600)
    rules = PC.head_only_program(rng, 2, 0, 4)
    counts = rng.geometric(1 / 8, size=25_000) - 1
    counts[321] = 50_000
    buf, seg, _ = PC.fixed_log(rng, rules, counts, pad_records=1, p_throw=1e-3)
    log = buf.reshape(-1)
    big = torch.zeros(len(log) + 512, dtype=torch.uint8, device="cuda")
    offs = torch.from_numpy(seg.astype(np.int64)).cuda()
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.set_option("run_chunk_bytes", 16384)
        for shift in (0, 16, 48, 112, 240):
            dev = big[shift:shift + len(log)]
            dev.copy_(torch.from_numpy(log))
            assert dev.data_ptr() % 256 == shift
            e.load_events(dev, offs)
            both_ways(e, rules, log, seg, f"device log at address {shift} (mod 256)")


# ------------------------------------------------------------------ g. the table is dropped with the plane
def test_table_dropped_by_register_program_and_reload():
    """A reload of the same bytes under other offsets, or another program, must not fold from the old table: the chunk
    size is the same, only the boundaries moved."""
    rng = np.random.default_rng(99700)
    rules = [PC.head_only_program(rng, 2, 0, 4) for _ in range(2)]
    counts = rng.geometric(1 / 10, size=30_000) - 1
    counts[777] = 8000
    buf, seg, _ = PC.fixed_log(rng, rules[0], counts, pad_records=2, p_throw=0.0)
    log = buf.reshape(-1)
    seg2 = seg.copy()
    inner = seg2[1:-1]
    seg2[1:-1] = np.sort(seg[0] + 64 * rng.integers(0, (int(seg[-1]) - int(seg[0])) // 64, size=len(inner)).astype(np.uint64))
    with ReplayEngine(0) as e:
        e.set_option("run_chunk_bytes", 16384)
        for i, (r, s) in enumerate([(0, seg), (0, seg2), (1, seg2), (0, seg2), (0, seg)]):
            e.register_program(P.make_program(16, N.REC_FIXED64, rules[r]))
            e.load_events(log, s)
            for _ in range(2):
                want = oracle(rules[r], log, s)
                fold(e)
                check(e, *want, 1, f"load {i}: program {r}, offsets {'moved' if s is seg2 else 'as drawn'}")
        # register_program alone, the log kept
        e.register_program(P.make_program(16, N.REC_FIXED64, rules[1]))
        fold(e)
        check(e, *oracle(rules[1], log, seg), 1, "register_program on a loaded log")
