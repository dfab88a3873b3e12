"""-m gpu: random sort-free fold programs through the routed push path and the single-engine sort-free paths.

tests/test_gpu_dist.py checks the multi-rank push path (route_push.cu + bulk_fold.cu) with one program, the Counter, whose
only set word is `version = seq` over seq 1..k: "the last SET by arrival index" and "the largest value" agree there, it only
uses the (add, set) entry layout, and its compact record is 16 bytes. Here the programs come from
oracle/program_corpus.py draw_sort_free_program: every entry layout with and without tombstones, 2..7 slots (16- and
32-byte compact records), rules without ops, SUB, ADDs of 0, and logs whose set values are random, with MatchError types
up to 2^32 - 1. Each routed case runs R loopback ranks (R engines on cuda:0, one host thread per rank), feeding every
aggregate from one chosen rank as a Kafka key does, and compares every rank's table, the ranks' hash sum and their event
and error counts with oracle/program_interp.py c_fold over the global CSR log.

Part B folds the same kind of programs on one engine over logs of 2 M records: fold_unsorted on the bulk kernels and on
the micro-batch kernel, and three micro-batches onto the live table, against c_fold_arrival_order.
"""
import numpy as np
import pytest

from oracle import program_corpus as PC
from oracle import program_interp as I
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import dist as D
from surge_b200 import native as N
from surge_b200 import programs as P

pytestmark = pytest.mark.gpu


def _torch():
    import torch

    return torch


def same(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:6]}\n got {got[bad[:3]].tolist()}\nwant {want[bad[:3]].tolist()}")


# ------------------------------------------------------------------ loopback ranks
def Ranks(rules, part, feeds, chunks, force_route=False):
    """R loopback ranks on cuda:0. feeds[r]: rank r's records in arrival order (global aggregate index at +8). The receive
    capacity is R x chunks x the longest chunk of any rank, so no region can overflow whatever the partition table."""
    torch = _torch()
    cap = len(feeds) * chunks * max(D.chunk_records(len(f), chunks) for f in feeds) + 1024

    def engine():
        e = ReplayEngine(0)
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.set_option("push_chunks", chunks)
        if force_route:
            e.set_option("force_route", 1)
        return e

    return D.LoopbackRanks(engine, part, [torch.from_numpy(np.ascontiguousarray(f).reshape(-1)).to("cuda:0") for f in feeds], cap)


def exchange_bytes(fused, n_slots):
    return 64 if fused == 2 else 16 if (1 + n_slots) * 4 <= 16 else 32


def check_ranks(ranks, chunks, want, nev, nerr, fused, n_slots, what):
    total, n_seen = 0, 0
    for r, e in enumerate(ranks.engines):
        gl = e.dist_local_aggregates().astype(np.int64)
        same(e.export_states(), want[gl], f"{what}, rank {r}")
        h = e.states_hash()
        if len(gl) == 0:
            assert h == 0, f"{what}, rank {r} owns nothing"
        total = (total + h) % (1 << 64)
        n_seen += len(gl)
        assert e.stats().fold_launches == 2 * chunks + 1, f"{what}, rank {r}: the push path did not run"
        assert e.dist_stats().exchange_record_bytes == exchange_bytes(fused, n_slots), what
    assert n_seen == len(want), what
    assert total == D.states_hash(want), what
    got = (sum(e.stats().n_events for e in ranks.engines), sum(e.stats().n_errors for e in ranks.engines))
    assert got == (nev, nerr), f"{what}: (n_events, n_errors) {got}, oracle {(nev, nerr)}"


def split_feeds(rng, rec, off, source_of, R):
    """Arrival order (aggregates interleaved, each one's records in log order), then rank r gets the records of the
    aggregates whose source is r."""
    counts = np.diff(off.astype(np.int64)) // 64
    aggs = np.repeat(np.arange(len(counts), dtype=np.uint64), counts)
    perm = PC.interleave(rng, aggs)
    src = np.asarray(source_of)[aggs[perm].astype(np.int64)]
    arrival = rec[perm]
    return [arrival[src == r] for r in range(R)]


def routed_case(seed, p_throw, n_agg=3000, n_rec=40_000, hot_len=5000, **program):
    rng = np.random.default_rng(seed)
    rules, n_slots = PC.draw_sort_free_program(rng, **program)
    rec, off, _ = PC.draw_sort_free_log(rng, rules, n_agg, n_rec, hot_len, p_throw=p_throw)
    want, nev, nerr = I.c_fold(rules, 16, rec, off)
    return rng, rules, n_slots, rec, off, want, nev, nerr


def run_and_check(rng, rules, n_slots, rec, off, want, nev, nerr, R, fused_modes=(2, 3), chunks=4, part=None, source_of=None,
                  what="", expect_repeat=None):
    n_agg = len(off) - 1
    part = rng.integers(0, 32, size=n_agg).astype(np.uint32) if part is None else part
    source_of = rng.integers(0, R, size=n_agg) if source_of is None else source_of
    feeds = split_feeds(rng, rec, off, source_of, R)
    what = f"{what} R={R} chunks={chunks} rules={rules}"
    with Ranks(rules, part, feeds, chunks) as ranks:
        for fused in fused_modes:
            for rnd in range(2):                     # twice: epochs, scratch hygiene, region reuse
                errors, repeated, times = ranks.run(fused)
                assert not any(errors), (what, errors, "entered, returned:", times)
                check_ranks(ranks, chunks, want, nev, nerr, fused, n_slots, f"{what} fused={fused} round {rnd}")
                if expect_repeat is not None:
                    assert repeated == expect_repeat, f"{what}: ordered repeat {repeated}"


@pytest.mark.parametrize("seed", range(24))
@pytest.mark.parametrize("throws", [False, True], ids=["no_throws", "throws"])
def test_random_programs_on_loopback_ranks(seed, throws):
    """24 drawn programs (layouts cycle, 2..7 slots), fused 2 and 3, R = 2, 3, 8; with throws every run goes through the
    ordered repeat and replays throwing aggregates from 64-, 16- and 32-byte records."""
    layout = PC.LAYOUTS[seed % 4]
    args = routed_case(61000 + seed + 100 * throws, 0.002 if throws else 0.0, layout=layout,
                       tombstones=layout == ("set", "set") and seed % 8 >= 4, n_src=1 + seed % 6)
    assert (args[-1] > 0) == throws
    for R in (2, 3, 8):
        run_and_check(*args, R=R, what=f"seed {seed}", expect_repeat=throws)


@pytest.mark.parametrize("R", [5, 16])
@pytest.mark.parametrize("layout", PC.LAYOUTS + ["tombstones"])
def test_every_layout_at_larger_rank_counts(R, layout):
    """One program per entry layout at R = 16 (kMaxRanks) and R = 5 (not a power of two)."""
    tomb = layout == "tombstones"
    args = routed_case(62000 + 10 * R + (PC.LAYOUTS + ["tombstones"]).index(layout), 0.001, n_agg=4000, n_rec=60_000,
                       layout=("set", "set") if tomb else layout, tombstones=tomb, n_src=5)
    run_and_check(*args, R=R, what=f"layout {layout}")


@pytest.mark.parametrize("chunks", [1, 3, 16, 256])
def test_push_chunks(chunks):
    """1 and 256 (kMaxChunks) chunks. The hot aggregate holds more than chunks x 1024 records and nearly all of its source
    rank's log, so it spans every non-empty chunk of that rank with several tiles per chunk. The other ranks' logs are shorter
    than chunks x 1024 records at 16 and 256 chunks, so most of their chunks are empty and still flag."""
    hot = max(5000, chunks * 1024 + 1000)
    args = routed_case(63000 + chunks, 0.001, n_agg=3000, n_rec=30_000, hot_len=hot, layout=("set", "set"), tombstones=True, n_src=4)
    run_and_check(*args, R=4, chunks=chunks, what=f"chunks {chunks}")


def test_one_tile_per_cta_fold_grid():
    """push_fold_blocks_per_sm = 0: the routed fold launches one CTA per tile (bulk_fold.cu, blocks_per_sm == ~0) instead of
    a grid of 2 CTAs per SM, so a low-priority fold yields the SMs to the partition kernels between tiles."""
    args = routed_case(63500, 0.001, layout=("set", "set"), tombstones=True, n_src=5)
    knobs = ReplayEngine(0)
    try:
        knobs.set_option("push_fold_blocks_per_sm", 0)
        for R in (3, 8):
            run_and_check(*args, R=R, what="push_fold_blocks_per_sm 0", expect_repeat=True)
    finally:
        knobs.set_option("push_fold_blocks_per_sm", 2)
        knobs.close()


def test_skewed_sources():
    """Rank 0 is fed nothing, rank 1 fewer than 256 records, rank 3 most of the log."""
    rng, rules, n_slots, rec, off, want, nev, nerr = routed_case(64000, 0.001, layout=("add", "set"), n_src=3)
    counts = np.diff(off.astype(np.int64)) // 64
    source_of = np.full(len(counts), 3)
    small = np.nonzero((counts > 0) & (counts < 20))[0][:10]
    source_of[small] = 1
    source_of[rng.choice(np.nonzero(source_of == 3)[0], size=len(counts) // 10, replace=False)] = 2
    assert 0 < counts[small].sum() < 256
    rng2 = np.random.default_rng(1)
    feeds = split_feeds(rng2, rec, off, source_of, 4)
    assert len(feeds[0]) == 0 and 0 < len(feeds[1]) < 256 and len(feeds[3]) > len(rec) // 2
    run_and_check(rng2, rules, n_slots, rec, off, want, nev, nerr, R=4, source_of=source_of, what="skewed sources")


def test_fewer_partitions_than_ranks():
    """Three partitions over five ranks: ranks 3 and 4 own no aggregate (empty table, hash 0) and still feed records."""
    rng, rules, n_slots, rec, off, want, nev, nerr = routed_case(65000, 0.001, layout=("set", "add"), n_src=5)
    part = rng.integers(0, 3, size=len(off) - 1).astype(np.uint32)
    source_of = rng.integers(0, 5, size=len(off) - 1)
    run_and_check(rng, rules, n_slots, rec, off, want, nev, nerr, R=5, part=part, source_of=source_of, what="3 partitions")


@pytest.mark.parametrize("pull,staged,tile", [(0, 1, 1024), (0, 0, 256), (1, 1, 512), (1, 0, 1024), (1, 0, 256), (0, 1, 512), (1, 1, 1024), (1, 1, 256), (1, 0, 512)])
def test_exchange_variants_with_a_seven_slot_tombstone_program(pull, staged, tile):
    """Remote stores vs remote loads, staged vs direct partition kernel, every tile size, with a 7-slot (set, set) program
    with tombstones: 32-byte compact records through both partition kernels (the staged one runs in the ordered repeat)."""
    args = routed_case(66000 + pull * 7 + staged * 3 + tile, 0.001, layout=("set", "set"), tombstones=True, n_src=6)
    assert args[2] == 7
    knobs = ReplayEngine(0)
    try:
        knobs.set_option("push_pull", pull); knobs.set_option("push_staged", staged); knobs.set_option("push_tile", tile)
        run_and_check(*args, R=4, chunks=3, what=f"pull {pull} staged {staged} tile {tile}", expect_repeat=True)
    finally:
        knobs.set_option("push_pull", 1); knobs.set_option("push_staged", -1); knobs.set_option("push_tile", 512)
        knobs.close()


def refused_everywhere(ranks, fused, what):
    errors, _, _ = ranks.run(fused)
    assert all(isinstance(x, SgrError) and x.code == N.SGR_ERR_UNSUPPORTED for x in errors), (what, errors)
    return errors


def test_compact_exchange_refuses_eight_slots():
    """A program that reads 7 record words besides the type does not fit a 32-byte compact record: fused 3 is refused on
    every rank, fused 2 is exact on the same ranks afterwards."""
    rng, rules, n_slots, rec, off, want, nev, nerr = routed_case(67000, 0.001, layout=("set", "set"), n_src=7)
    assert n_slots == 8
    feeds = split_feeds(rng, rec, off, rng.integers(0, 4, size=len(off) - 1), 4)
    with Ranks(rules, rng.integers(0, 32, size=len(off) - 1).astype(np.uint32), feeds, 4) as ranks:
        refused_everywhere(ranks, 3, "8 slots, fused 3")
        for _ in range(2):
            errors, _, _ = ranks.run(2)
            assert not any(errors), errors
            check_ranks(ranks, 4, want, nev, nerr, 2, n_slots, "8 slots, fused 2")


OUTSIDE_SORT_FREE = {
    "if_exists": [(I.CREATE, [(I.OP_SET, 0, 16, 4)]), (I.IF_EXISTS, [(I.OP_ADD_I32, 4, 20, 4)]), (I.THROW, [])],
    "set_and_added_word": [(I.MATERIALISE, [(I.OP_SET, 0, 16, 4)]), (I.MATERIALISE, [(I.OP_ADD_I32, 0, 20, 4)])],
}


@pytest.mark.parametrize("name", list(OUTSIDE_SORT_FREE))
def test_programs_outside_the_sort_free_class_are_refused_on_loopback_ranks(name):
    """Loopback ranks have no NCCL communicator for the scatter + group-by path: refused on the host, every fused mode."""
    rules = OUTSIDE_SORT_FREE[name]
    assert PC.bulk_layout(rules) is None
    rng = np.random.default_rng(68000)
    rec, off, _ = PC.draw_sort_free_log(rng, rules, 500, 5000, 100)
    feeds = split_feeds(rng, rec, off, rng.integers(0, 3, size=500), 3)
    with Ranks(rules, rng.integers(0, 32, size=500).astype(np.uint32), feeds, 2) as ranks:
        for fused in (0, 1, 2, 3):
            refused_everywhere(ranks, fused, f"{name} fused {fused}")


# bytes 8..15 of a record are its aggregate index: global when fed, rewritten by every exchange mode
HEADER_READ = [(I.MATERIALISE, [(I.OP_SET, 0, 8, 8)]), (I.MATERIALISE, [(I.OP_SET, 0, 16, 4), (I.OP_SET, 4, 12, 4)]), (I.THROW, [])]


def test_a_program_reading_the_aggregate_field_is_refused_when_routed():
    """Refused with SGR_ERR_UNSUPPORTED before any launch: on 4 loopback ranks (fused 2 and 3) and on one rank with
    force_route (every fused mode). On one engine the same program folds to what the oracle says: the dense index."""
    assert PC.bulk_layout(HEADER_READ) is not None
    rng = np.random.default_rng(69000)
    n_agg = 2000
    rec, off, _ = PC.draw_sort_free_log(rng, HEADER_READ, n_agg, 30_000, 3000, p_throw=0.001)
    feeds = split_feeds(rng, rec, off, rng.integers(0, 4, size=n_agg), 4)
    part = rng.integers(0, 32, size=n_agg).astype(np.uint32)
    with Ranks(HEADER_READ, part, feeds, 4) as ranks:
        for fused in (2, 3):
            errors = refused_everywhere(ranks, fused, f"R=4 fused {fused}")
            assert all("8..15" in str(x) for x in errors), errors
    everything = [np.concatenate(feeds)]
    with Ranks(HEADER_READ, np.zeros(n_agg, np.uint32), everything, 4, force_route=True) as one:
        for fused in (0, 1, 2, 3):
            refused_everywhere(one, fused, f"force_route fused {fused}")
    arrival = rec[PC.interleave(rng, np.repeat(np.arange(n_agg, dtype=np.uint64), np.diff(off.astype(np.int64)) // 64))]
    want, nev, nerr = I.c_fold_arrival_order(HEADER_READ, 16, arrival, None, n_agg=n_agg)
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, HEADER_READ))
        e.fold_unsorted(arrival, n_agg)
        same(e.export_states(), want, "header read, fold_unsorted")
        assert (e.stats().n_events, e.stats().n_errors) == (nev, nerr)
        half = len(arrival) // 2
        table, _, _ = I.c_fold_arrival_order(HEADER_READ, 16, arrival[:half], None, n_agg=n_agg)
        table, nev2, nerr2 = I.c_fold_arrival_order(HEADER_READ, 16, arrival[half:], table)
        e.fold_unsorted(arrival[:half], n_agg)
        e.fold_incremental(arrival[half:])
        same(e.export_states(), table, "header read, fold_incremental")
        assert (e.stats().n_events, e.stats().n_errors) == (nev2, nerr2)


# ------------------------------------------------------------------ part B: one engine, logs of 2 M records
N_REC_B = 2_000_000
N_AGG_B = 400_000


def arrival_log(seed, rules, n_rec=N_REC_B, n_agg=N_AGG_B, hot_len=200_000, p_throw=2e-4):
    rng = np.random.default_rng(seed)
    rec, off, _ = PC.draw_sort_free_log(rng, rules, n_agg, n_rec, hot_len, p_throw=p_throw)
    return rec[PC.interleave(rng, np.repeat(np.arange(n_agg, dtype=np.uint64), np.diff(off.astype(np.int64)) // 64))]


def check(e, want, nev, nerr, what):
    same(e.export_states(), want, what)
    st = e.stats()
    assert (st.n_events, st.n_errors) == (nev, nerr), f"{what}: stats {(st.n_events, st.n_errors)}, oracle {(nev, nerr)}"


def scale_programs():
    out = {}
    for i, layout in enumerate(PC.LAYOUTS):
        out["-".join(layout)] = PC.draw_sort_free_program(np.random.default_rng(70000 + i), layout=layout, tombstones=False)[0]
    out["set-set-tombstones"] = PC.draw_sort_free_program(np.random.default_rng(70010), layout=("set", "set"), tombstones=True, n_src=6)[0]
    # a word that one rule sets and another adds: outside the bulk layouts, the micro-batch kernel's general mode
    base = PC.draw_sort_free_program(np.random.default_rng(70020), layout=("set", "add"), tombstones=False, n_types=5)[0]
    out["set-and-added"] = base + [(I.MATERIALISE, [(I.OP_ADD_I32, 0, 24, 4)])]
    return out


SCALE = scale_programs()


@pytest.mark.parametrize("name", list(SCALE))
def test_one_engine_at_scale(name):
    """fold_unsorted with the bulk kernels (two launches), with the micro-batch kernel from None (bulk = 0), on the smallest
    bulk grid; then three micro-batches onto the live table, the middle ones with a replay budget so small that throwing
    slots leave the in-kernel replay."""
    rules = SCALE[name]
    bulk = PC.bulk_layout(rules) is not None
    assert bulk == (name != "set-and-added")
    log = arrival_log(71000 + list(SCALE).index(name), rules)
    want, nev, nerr = I.c_fold_arrival_order(rules, 16, log, None, n_agg=N_AGG_B)
    assert nerr > 0
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(16, N.REC_FIXED64, rules))
        e.fold_unsorted(log, N_AGG_B)
        check(e, want, nev, nerr, f"{name} fold_unsorted")
        if bulk:
            assert e.stats().fold_launches == 2
            try:
                e.set_option("bulk_blocks_per_sm", 1)
                e.fold_unsorted(log, N_AGG_B)
                check(e, want, nev, nerr, f"{name} bulk_blocks_per_sm 1")
            finally:
                e.set_option("bulk_blocks_per_sm", 0)
            e.set_option("bulk", 0)
            e.fold_unsorted(log, N_AGG_B)
            check(e, want, nev, nerr, f"{name} bulk 0")
            e.set_option("bulk", 1)
        table = want
        for b, (n, budget) in enumerate([(600_000, 1 << 24), (20_000, 1), (1_000_000, 1)]):
            batch = arrival_log(71100 + b, rules, n_rec=n, hot_len=n // 8, p_throw=1e-3)
            e.set_option("replay_budget", budget)
            table, nev_b, nerr_b = I.c_fold_arrival_order(rules, 16, batch, table)
            e.fold_incremental(batch)
            check(e, table, nev_b, nerr_b, f"{name} micro-batch {b} ({n} records, replay budget {budget})")
        e.set_option("replay_budget", 1 << 24)
