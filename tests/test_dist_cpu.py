"""CPU tests of the N>1 host logic (gloo, world_size 2): ownership tables, stable routing, the exchange plan.
The device kernels (csrc/dist.cu) mirror surge_b200.dist.route_on_host; here the numpy mirror is driven through a real
2-process all-to-all and checked against the single-process oracle, so the routing contract is pinned without a GPU."""
import os
import socket
import sys
import threading

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank: int, world: int, port: int, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import oracle as O
    from surge_b200 import dist as D
    from surge_b200 import formats as F
    from surge_b200 import synth as S

    n_global, n_src = 3000, 16
    rng = np.random.default_rng(1)
    counts = rng.integers(0, 12, size=n_global)
    rec, off = S.counter_csr(n_global, counts, seed=2, p_throw=0.01)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    arrival = S.interleave_arrival(rec, seed=3)
    mine = arrival[((arrival["agg"] % n_src) % world) == rank]        # this rank's source partitions, arrival order
    part = D.partitions_for_keys([f"agg-{g}" for g in range(n_global)], 32)
    owner, local, globals_of = D.owner_and_local_index(part, world)
    sends = D.route_on_host(mine, owner, local, world)
    # counts all-gather, then the all-to-all of packed records
    cnt = torch.tensor([len(s) for s in sends], dtype=torch.int64)
    allc = [torch.zeros(world, dtype=torch.int64) for _ in range(world)]
    dist.all_gather(allc, cnt)
    recv_counts = [int(allc[s][rank]) for s in range(world)]
    send_t = torch.from_numpy(np.concatenate(sends).view(np.uint8).reshape(-1).copy())
    recv_t = torch.zeros(sum(recv_counts) * 64, dtype=torch.uint8)
    dist.all_to_all_single(recv_t, send_t, [c * 64 for c in recv_counts], [len(s) * 64 for s in sends])
    got_rec = recv_t.numpy().view(F.REC64)
    n_local = len(globals_of[rank])
    grouped, goff = O.group_by_agg(got_rec, n_local)
    states, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, grouped, goff)
    ok = np.array_equal(states, want[globals_of[rank].astype(np.int64)])
    total = torch.tensor([len(got_rec)], dtype=torch.int64)
    dist.all_reduce(total)
    ret[rank] = (bool(ok), int(total[0]) == len(rec), n_local)
    dist.destroy_process_group()


def test_two_rank_routing_matches_single_process_fold():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert all(ret[r][0] for r in range(world)), dict(ret)
    assert all(ret[r][1] for r in range(world))
    assert sum(ret[r][2] for r in range(world)) == 3000


def test_owner_tables_follow_the_reference_partitioner():
    from oracle import surge_model as M
    from surge_b200 import dist as D

    keys = [f"agg-{g}:{g % 7}" for g in range(200)]
    part = D.partitions_for_keys(keys, 32, up_to_colon=True)
    for k, p in zip(keys, part):
        assert p == M.partition_for_key(M.partition_string_up_to_colon(k), 32)
    owner, local, globals_of = D.owner_and_local_index(part, 4)
    assert (owner == part % 4).all()
    for r in range(4):
        assert (owner[globals_of[r]] == r).all() and (local[globals_of[r]] == np.arange(len(globals_of[r]))).all()


def test_topic_partitions_split_over_ranks_need_no_exchange():
    """Feeding from the topic: rank r takes the partitions p % nranks == r; because the partition of a record IS
    partitionForKey(aggregate id), every aggregate's records land on exactly one rank and ranks share no aggregate."""
    from surge_b200 import dist as D

    keys = [f"agg-{i}" for i in range(5000)]
    n_part, nranks = 32, 4
    part = D.partitions_for_keys(keys, n_part)
    owners = {}
    for r in range(nranks):
        mine = set(D.partitions_of_rank(r, nranks, n_part))
        assert mine == {p for p in range(n_part) if p % nranks == r}
        for k, p in zip(keys, part.tolist()):
            if p in mine:
                assert k not in owners
                owners[k] = r
    assert len(owners) == len(keys)
    owner, _, _ = D.owner_and_local_index(part, nranks)          # the routed path's owner table says the same
    assert [owners[k] for k in keys] == owner.tolist()


# ------------------------------------------------------------------ the loopback-ranks driver, on fake engines
class _FakeRank:
    """One rank for surge_b200.dist.LoopbackRanks, without a library or a GPU: it records the calls the driver makes, and its
    dist_route_and_fold returns or raises what answer(rank, push_ordered) says (None, or an exception to raise)."""

    def __init__(self, answer):
        self.answer, self.rank, self.log, self.push_ordered, self.calls, self.closed = answer, None, [], 0, [], False

    def dist_init(self, rank, nranks, unique_id, capacity):
        self.rank = rank
        self.log.append(("init", rank, nranks, unique_id, capacity))

    def dist_set_partitions(self, part):
        self.log.append(("partitions", len(part)))

    def dist_recv_base(self):
        return 0x1000 * (self.rank + 1)

    def dist_set_peers(self, bases):
        self.log.append(("peers", list(bases)))

    def dist_reserve(self, n):
        self.log.append(("reserve", n))

    def set_option(self, name, value):
        assert name == "push_ordered"
        self.push_ordered = value

    def dist_route_and_fold(self, feed, fused):
        self.calls.append((fused, self.push_ordered))
        ex = self.answer(self.rank, self.push_ordered)
        if ex is not None:
            raise ex

    def close(self):
        self.closed = True


def _fake_ranks(answer, R=3):
    from surge_b200 import dist as D

    feeds = [np.zeros(64 * (r + 1), np.uint8) for r in range(R)]
    return D.LoopbackRanks(lambda: _FakeRank(answer), np.zeros(10, np.uint32), feeds, 4096)


def _again():
    from surge_b200 import native as N

    return N.SgrError(N.SGR_ERR_AGAIN, "throwing aggregates")


def test_loopback_ranks_set_up_and_run_without_a_repeat():
    with _fake_ranks(lambda r, ordered: None) as ranks:
        bases = [0x1000, 0x2000, 0x3000]
        for r, e in enumerate(ranks.engines):
            assert e.log == [("init", r, 3, None, 4096), ("partitions", 10), ("peers", bases), ("reserve", r + 1)]
        errors, repeated, times = ranks.run(2)
        assert errors == [None] * 3 and not repeated
        assert all(e.calls == [(2, 0)] and e.push_ordered == 0 for e in ranks.engines)
        assert all(0 <= t[0] <= t[1] for t in times)
    assert all(e.closed for e in ranks.engines)


def test_loopback_ranks_repeat_in_order_when_every_rank_says_again():
    with _fake_ranks(lambda r, ordered: None if ordered else _again()) as ranks:
        errors, repeated, _ = ranks.run(3)
        assert errors == [None] * 3 and repeated
        assert all(e.calls == [(3, 0), (3, 1)] and e.push_ordered == 0 for e in ranks.engines)


def test_loopback_ranks_refuse_again_next_to_another_error():
    from surge_b200 import native as N

    other = N.SgrError(N.SGR_ERR_CAPACITY, "a source rank reported a full receive region")
    with _fake_ranks(lambda r, ordered: _again() if r == 0 else other if r == 1 else None) as ranks:
        with pytest.raises(AssertionError) as info:
            ranks.run(2)
        assert "SGR_ERR_AGAIN" in str(info.value) and "SGR_ERR_CAPACITY" in str(info.value)
        assert all(len(e.calls) == 1 and e.push_ordered == 0 for e in ranks.engines)


def test_loopback_ranks_report_a_rank_that_hangs():
    release, threads = threading.Event(), []

    def answer(r, ordered):
        if r == 2:
            threads.append(threading.current_thread())
            release.wait()
        return None

    try:
        with _fake_ranks(answer) as ranks:
            with pytest.raises(AssertionError, match="hung"):
                ranks.run(2, timeout=0.2)
            assert all(e.push_ordered == 0 for e in ranks.engines)
    finally:
        release.set()
        for t in threads:
            t.join(timeout=10)
    assert len(threads) == 1 and not threads[0].is_alive()


def test_loopback_ranks_reset_push_ordered_when_a_rank_raises():
    def answer(r, ordered):
        if not ordered:
            return _again()
        return RuntimeError("lost rank") if r == 1 else None

    with _fake_ranks(answer) as ranks:
        errors, repeated, _ = ranks.run(2)
        assert repeated and errors[0] is None and errors[2] is None and str(errors[1]) == "lost rank"
        assert all(e.calls == [(2, 0), (2, 1)] and e.push_ordered == 0 for e in ranks.engines)
