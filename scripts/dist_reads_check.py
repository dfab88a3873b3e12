"""Reads of a routed rank under torchrun: every rank folds its share of one global Counter log (fused 2, then fused 0), loads
its rank key table (sgr_dist_load_keys) and checks the batched read, the changed-state export and the scan of its own engine
against the oracle's table for the ids it owns; ids it does not own must be unknown.

  torchrun --nproc-per-node N scripts/dist_reads_check.py [n_global]

Uses the oracle as the checker only (tests/test_gpu_dist_reads.py runs this script)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from surge_b200 import ReplayEngine
from surge_b200 import dist as D
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200 import synth as S


def check_reads(e, ids, want, owned):
    user = want.shape[1] - 8
    fl_want = want[:, user:user + 4].copy().view(np.uint32).reshape(-1)
    rows, fl, idx = e.get_many(ids, arrays=True)
    gl = e.dist_local_aggregates().astype(np.int64)
    ok = bool((idx[~owned] == -1).all() and (fl[~owned] == 0).all())
    ok &= bool(np.array_equal(gl[idx[owned]], np.nonzero(owned)[0]) and np.array_equal(rows[owned], want[owned, :user]))
    ok &= bool(np.array_equal(fl[owned], fl_want[owned]))
    exported = np.sort(np.concatenate([gl[p[0]] for p in e.export_changes(N.ST_CHANGED | N.ST_ERROR)] or [np.zeros(0, np.int64)]))
    ok &= bool(np.array_equal(exported, np.nonzero(owned & ((fl_want & (N.ST_CHANGED | N.ST_ERROR)) != 0))[0]))
    scanned = [k for p in e.scan() for k in p[3]]
    ok &= scanned == sorted((ids[g] for g in np.nonzero(owned & ((fl_want & N.ST_EXISTS) != 0))[0]), key=str.encode)
    return ok


def main():
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1)); lr = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(lr)
    dev = f"cuda:{lr}"
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device(dev))
    n_global = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000
    from oracle import oracle as O

    rng = np.random.default_rng(17)
    counts = rng.integers(0, 12, size=n_global)
    rec, off = S.counter_csr(n_global, counts, seed=5, p_throw=0.0005)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off, threads=8)
    ids = [f"acct-{g}" + (":" + str(g % 7) if g % 5 == 0 else "") for g in range(n_global)]
    part = D.partitions_for_keys(ids, 32)
    owned = (part % world) == rank
    arrival = S.interleave_arrival(rec, seed=6)
    mine = arrival[(arrival["agg"] % 64).astype(np.int64) % world == rank]
    local_rec = torch.from_numpy(mine.view(np.uint8).reshape(-1).copy()).to(dev)
    cap = int(len(rec) / world * 1.5) + 16 * 1024 * world * 8
    all_ok = True
    for fused in ([2, 0] if world > 1 else [2]):
        e = ReplayEngine(lr)
        e.register_program(P.counter_program())
        if world == 1:
            e.set_option("force_route", 1)
        e.set_option("push_chunks", 8)
        D.exchange_ids(e, rank, world, cap, fused=True)
        e.dist_set_partitions(part)
        if world > 1:
            dist.barrier()
        e.dist_route_and_fold(local_rec, fused)
        e.dist_load_keys(ids)
        ok = check_reads(e, ids, want, owned)
        all_ok &= ok
        print(f"[rank {rank}/{world}] fused={fused} owned={int(owned.sum())} reads_ok={ok}", flush=True)
        e.close()
        if world > 1:
            dist.barrier()
    if world > 1:
        dist.destroy_process_group()
    if not all_ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
