"""-m gpu: the multi-rank path (route + exchange + fold) and the sort-free bulk fold, bit-exact against the oracle.

Three layers:
  * the bulk sort-free fold on one engine (sgr_fold_unsorted on a large arrival-order log);
  * LOOPBACK ranks: R engines on cuda:0 inside this process, each one rank of an R-rank job, pushing into each other's receive
    regions through plain device pointers — the whole pipelined push path (partition in shared memory, look-back, arrival
    flags, chunked fold) runs on ONE GPU, so the driver's single-GPU box exercises it;
  * real ranks under torchrun over NCCL + CUDA IPC when the box has >= 2 GPUs (scripts/dist_check.py).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import dist as D
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200 import synth as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch():
    import torch

    return torch


def assert_same(got, want, what=""):
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).any(axis=1))[0]
        raise AssertionError(f"{what}: {len(bad)} of {len(want)} states differ; first {bad[:8]}\n"
                             f"got  {got[bad[:4]].tolist()}\nwant {want[bad[:4]].tolist()}")


# ------------------------------------------------------------------ bulk sort-free fold (one engine)
@pytest.mark.parametrize("n_agg,max_events,p_throw,seed", [(1, 5, 0.0, 1), (50, 300, 0.0, 2), (3000, 60, 0.002, 3), (20000, 40, 0.0005, 4)])
@pytest.mark.parametrize("bulk", [1, 0])
def test_bulk_fold_counter(n_agg, max_events, p_throw, seed, bulk):
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, max_events + 1, size=n_agg)
    rec, off = S.counter_csr(n_agg, counts, seed=seed, p_throw=p_throw)
    want, nev, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    arrival = S.interleave_arrival(rec, seed=seed + 10)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.set_option("bulk", bulk)
        e.fold_unsorted(arrival, n_agg)
        st = e.stats()
        assert_same(e.export_states(), want, f"bulk={bulk}")
        assert (st.n_events, st.n_errors) == (nev, nerr)
        # a second fold on the same engine: the scratch was left clean
        e.fold_unsorted(arrival, n_agg)
        assert_same(e.export_states(), want, f"bulk={bulk}, second fold")
        assert e.states_hash() == D.states_hash(want)


@pytest.mark.parametrize("unroll,hints", [(1, 0), (2, 1), (4, 0)])
def test_bulk_fold_tuning_variants_agree(unroll, hints):
    rng = np.random.default_rng(9)
    counts = rng.integers(0, 50, size=5000)
    rec, off = S.counter_csr(5000, counts, seed=9, p_throw=0.001)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    arrival = S.interleave_arrival(rec, seed=19)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.set_option("bulk_unroll", unroll)
        e.set_option("bulk_hints", hints)
        try:
            e.fold_unsorted(arrival, 5000)
            assert_same(e.export_states(), want, f"unroll {unroll} hints {hints}")
        finally:
            e.set_option("bulk_unroll", 4)
            e.set_option("bulk_hints", 1)


def test_bulk_fold_other_programs():
    """IntBalance (add-only), multilanguage Counter (MatchError on unknown types), snapshot restore (set-only + tombstones)."""
    from surge_b200 import formats as F

    rng = np.random.default_rng(5)
    n_agg = 4000
    # IntBalance: one event type, add only
    counts = rng.integers(0, 30, size=n_agg)
    n = int(counts.sum())
    agg = np.repeat(np.arange(n_agg, dtype=np.uint64), counts)
    rec = F.counter_records(np.zeros(n, dtype=np.uint32), np.arange(n, dtype=np.uint32), agg, rng.integers(-(1 << 31), 1 << 31, size=n).astype(np.int32))
    off = F.csr_offsets_from_counts(counts)
    want, _, _ = O.fold_packed(O.MODEL_INT_BALANCE, O.REC_FIXED64, rec, off)
    arr = S.interleave_arrival(rec, seed=6)
    with ReplayEngine(0) as e:
        e.register_program(P.int_balance_program())
        e.fold_unsorted(arr, n_agg)
        assert_same(e.export_states(), want, "IntBalance")
    # multilanguage Counter: types >= 2 are MatchErrors
    rec2, off2 = S.counter_csr(n_agg, counts, seed=7, p_throw=0.0)   # has NoOp (type 2) events: they throw in this model
    want2, nev2, nerr2 = O.fold_packed(O.MODEL_ML_COUNTER, O.REC_FIXED64, rec2, off2)
    with ReplayEngine(0) as e:
        e.register_program(P.ml_counter_program())
        e.fold_unsorted(S.interleave_arrival(rec2, seed=8), n_agg)
        assert_same(e.export_states(), want2, "ml counter")
        assert (e.stats().n_events, e.stats().n_errors) == (nev2, nerr2)


def test_bulk_fold_snapshot_restore_is_last_write_wins():
    """a7: the state topic as a fold — both words set-only, tombstones (32-byte scratch entries, has_none)."""
    from oracle import program_interp as I

    from surge_b200 import formats as F

    rng = np.random.default_rng(11)
    n_agg, n = 3000, 40000
    rec = np.zeros(n, dtype=F.REC64)
    rec["type"] = (rng.random(n) < 0.15).astype(np.uint32)            # 0 snapshot, 1 tombstone
    rec["agg"] = rng.integers(0, n_agg, size=n).astype(np.uint64)
    rec["seq"] = np.arange(n, dtype=np.uint32)
    rec["arg0"] = rng.integers(-(1 << 31), 1 << 31, size=n).astype(np.int32)
    rec["arg1"] = rng.integers(0, 1 << 31, size=n).astype(np.int32)
    prog = P.counter_snapshot_restore_program()
    order = np.argsort(rec["agg"], kind="stable")
    counts = np.bincount(rec["agg"].astype(np.int64), minlength=n_agg)
    rules = [(I.CREATE, [(I.OP_SET, 0, 16, 4), (I.OP_SET, 4, 20, 4)]), (I.TOMBSTONE, [])]
    want = I.fold(rules, 16, rec[order], F.csr_offsets_from_counts(counts))
    with ReplayEngine(0) as e:
        e.register_program(prog)
        e.fold_unsorted(rec, n_agg)
        assert_same(e.export_states(), want, "snapshot restore")


def test_states_hash_matches_the_numpy_twin():
    rng = np.random.default_rng(3)
    counts = rng.integers(0, 20, size=1234)
    rec, off = S.counter_csr(1234, counts, seed=3)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_events(rec, off)
        e.fold()
        st = e.export_states()
        assert e.states_hash() == D.states_hash(st)
        assert e.states_hash() != D.states_hash(st[::-1].copy())   # the index is part of the hash


def test_routed_log_generators_agree():
    torch = _torch()
    n_global, epa, seed = 5000, 7, 3
    for world in (1, 3):
        for rank in range(world):
            dev = S.routed_log_device(rank, world, n_global, epa, seed, "cuda:0").cpu().numpy()
            g = np.arange(rank, n_global, world)
            host, _ = S.routed_events_host(g, epa, seed)
            host = host.copy()
            host["agg"] = np.repeat(g, epa).astype(np.uint64)
            # device order: event k of every aggregate before event k+1
            want = host.view(np.int32).reshape(len(g), epa, 16).transpose(1, 0, 2).reshape(-1, 16)
            assert np.array_equal(dev, want)


# ------------------------------------------------------------------ loopback ranks: the push pipeline on one GPU
def _loopback_job(R, n_global, rec_all, part, fused, chunks, capacity, prog=None, seed=4):
    """Run an R-rank route + fold with every rank on cuda:0. rec_all: CSR records with GLOBAL agg; rank r feeds the
    aggregates whose source partition (agg % 64) % R == r, in an interleaved arrival order."""
    torch = _torch()
    arrival = S.interleave_arrival(rec_all, seed=seed)
    src = (arrival["agg"] % 64).astype(np.int64) % R
    feeds = [torch.from_numpy(arrival[src == r].view(np.uint8).reshape(-1).copy()).to("cuda:0") for r in range(R)]

    def engine():
        e = ReplayEngine(0)
        e.register_program(prog or P.counter_program())
        e.set_option("push_chunks", chunks)
        return e

    ranks = D.LoopbackRanks(engine, part, feeds, capacity)
    again_rounds = 0
    for _round in range(2):       # twice: epochs, scratch hygiene, region reuse
        errors, repeated, _ = ranks.run(fused)
        again_rounds += repeated
        if any(errors):
            break
    ranks.engines[0].again_rounds = again_rounds
    return ranks.engines, errors


def _check_loopback(engines, want, R):
    total_hash = 0
    n_seen = 0
    for r, e in enumerate(engines):
        got = e.export_states()
        gl = e.dist_local_aggregates().astype(np.int64)
        assert_same(got, want[gl], f"rank {r}/{R}")
        total_hash = (total_hash + e.states_hash()) % (1 << 64)
        n_seen += len(gl)
    assert n_seen == len(want)
    assert total_hash == D.states_hash(want)


@pytest.mark.parametrize("R", [2, 4, 8])
@pytest.mark.parametrize("fused", [2, 3])
def test_loopback_push_pipeline_matches_oracle(R, fused):
    n_global, rng = 30000, np.random.default_rng(R * 10 + fused)
    counts = rng.integers(0, 40, size=n_global)
    rec, off = S.counter_csr(n_global, counts, seed=R, p_throw=0.0)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    part = D.partitions_for_keys([f"agg-{g}" for g in range(n_global)], 32)
    cap = int(len(rec) / R * 1.5) + 8 * R * 4 * 1024
    engines, errors = _loopback_job(R, n_global, rec, part, fused, chunks=4, capacity=cap)
    try:
        assert not any(errors), errors
        _check_loopback(engines, want, R)
        ds = engines[0].dist_stats()
        assert ds.exchange_record_bytes == (64 if fused == 2 else 16)
    finally:
        for e in engines:
            e.close()


@pytest.mark.parametrize("pull,staged,tile", [(0, 1, 1024), (0, 0, 256), (1, 1, 512), (1, 0, 1024), (1, 0, 256), (0, 1, 512), (1, 1, 1024), (1, 1, 256), (1, 0, 512)])
def test_loopback_exchange_variants_agree(pull, staged, tile):
    """remote stores vs remote loads, staged vs direct partition kernel, every tile size: the same tables."""
    R, n_global = 4, 20000
    rng = np.random.default_rng(pull * 7 + staged * 3 + tile)
    counts = rng.integers(0, 35, size=n_global)
    rec, off = S.counter_csr(n_global, counts, seed=tile + pull, p_throw=0.001)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    part = D.partitions_for_keys([f"agg-{g}" for g in range(n_global)], 32)
    knobs = ReplayEngine(0)
    try:
        knobs.set_option("push_pull", pull); knobs.set_option("push_staged", staged); knobs.set_option("push_tile", tile)
        for fused in (2, 3):
            engines, errors = _loopback_job(R, n_global, rec, part, fused, chunks=3, capacity=int(len(rec) / R * 1.6) + 200000)
            try:
                assert not any(errors), errors
                _check_loopback(engines, want, R)
            finally:
                for e in engines:
                    e.close()
    finally:
        knobs.set_option("push_pull", 1); knobs.set_option("push_staged", -1); knobs.set_option("push_tile", 512)
        knobs.close()


def test_loopback_push_with_throwing_events_replays_exactly():
    R, n_global = 4, 12000
    rng = np.random.default_rng(77)
    counts = rng.integers(0, 30, size=n_global)
    rec, off = S.counter_csr(n_global, counts, seed=77, p_throw=0.002)
    want, _, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    assert nerr > 0
    part = D.partitions_for_keys([f"agg-{g}" for g in range(n_global)], 32)
    for fused in (2, 3):
        engines, errors = _loopback_job(R, n_global, rec, part, fused, chunks=3, capacity=int(len(rec) / R * 1.6) + 200000)
        try:
            assert not any(errors), errors
            _check_loopback(engines, want, R)
            assert sum(e.stats().n_errors for e in engines) == nerr
            assert engines[0].again_rounds == 2     # both rounds went through the ordered repeat
        finally:
            for e in engines:
                e.close()


def test_loopback_region_overflow_fails_on_every_rank_without_writing_out_of_bounds():
    """ADVICE r1 (dist.cu:369): a receive region that would overflow must not be written past, and the ranks fail together."""
    R, n_global = 2, 20000
    counts = np.full(n_global, 10)
    rec, off = S.counter_csr(n_global, counts, seed=5)
    part = D.partitions_for_keys([f"agg-{g}" for g in range(n_global)], 32)
    # capacity for a quarter of what arrives
    engines, errors = _loopback_job(R, n_global, rec, part, 2, chunks=2, capacity=len(rec) // R // 4)
    try:
        assert all(isinstance(x, SgrError) for x in errors), errors
        assert all(x.code == N.SGR_ERR_CAPACITY for x in errors), [x.code for x in errors]
    finally:
        for e in engines:
            e.close()


def test_force_route_single_rank_push():
    """nranks == 1 with force_route: the push kernel, flags and chunked fold with one destination."""
    torch = _torch()
    n_global = 9000
    rng = np.random.default_rng(8)
    counts = rng.integers(0, 25, size=n_global)
    rec, off = S.counter_csr(n_global, counts, seed=8, p_throw=0.001)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    arrival = S.interleave_arrival(rec, seed=9)
    feed = torch.from_numpy(arrival.view(np.uint8).reshape(-1).copy()).to("cuda:0")
    for fused in (2, 3):
        with ReplayEngine(0) as e:
            e.register_program(P.counter_program())
            e.set_option("force_route", 1)
            e.set_option("push_chunks", 5)
            e.dist_init(0, 1, None, len(arrival) + 5 * 1024)
            e.dist_set_partitions(np.zeros(n_global, dtype=np.uint32))
            e.dist_route_and_fold(feed, fused)
            assert_same(e.export_states(), want, f"fused {fused}")


# ------------------------------------------------------------------ real ranks (NCCL + CUDA IPC) when the box has them
@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_gpu_route_and_fold_under_torchrun(world):
    torch = _torch()
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, the box has {torch.cuda.device_count()}")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29611 + world), os.path.join(ROOT, "scripts", "dist_check.py"), "300000", "20"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    lines = [ln for ln in r.stdout.splitlines() if "parity=" in ln]
    assert len(lines) >= world * 3, r.stdout[-3000:]
    assert all("parity=True" in ln for ln in lines), "\n".join(lines)
    assert "hash_ok=True" in r.stdout
