"""Reads of a routed table: 4 loopback ranks (one routed rebuild split four ways on one card) against one engine holding the same
table, 10 M Counter aggregates with UUID ids. Host clocks around calls that end in a device synchronisation:
  1. dist_load_keys on each rank plus the first read, which builds the rank's device id index (one engine: load_keys + first read);
  2. routed reads (surge_b200/dist.py read_routed: every id to its owner's get_many) in 100 batches of 100 k random ids, against
     get_many on the one engine over the same batches;
  3. a full changed-state export and a full scan on each rank, against the same on the one engine.
Prints the card name and power limit, then one JSON line.

    python scripts/dist_reads_bench.py [--n 10000000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from surge_b200 import ReplayEngine  # noqa: E402
from surge_b200 import dist as D  # noqa: E402
from surge_b200 import native as N  # noqa: E402
from surge_b200 import programs as P  # noqa: E402
from surge_b200 import synth as S  # noqa: E402

R = 4
CH_ERR = N.ST_CHANGED | N.ST_ERROR


def card() -> dict:
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return {"card": name, "power_limit": pl}


def uuid_ids(n: int, seed: int):
    h = np.random.default_rng(seed).integers(0, 256, size=(n, 16), dtype=np.uint8).tobytes().hex()
    return [f"{h[i:i + 8]}-{h[i + 8:i + 12]}-{h[i + 12:i + 16]}-{h[i + 16:i + 20]}-{h[i + 20:i + 32]}" for i in range(0, 32 * n, 32)]


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def rebuild(n: int, part: np.ndarray):
    """The loopback ranks after one routed fold (fused 2) of a Counter log, and one engine after fold_unsorted of the same log."""
    import torch

    rec, _ = S.counter_csr(n, np.random.default_rng(1).integers(1, 4, size=n), seed=2)
    arrival = S.interleave_arrival(rec, seed=3)
    src = (arrival["agg"] % 64).astype(np.int64) % R
    feeds = [torch.from_numpy(arrival[src == r].view(np.uint8).reshape(-1).copy()).to("cuda:0") for r in range(R)]
    cap = int(len(rec) / R * 1.5) + 64 * 1024 * R

    def engine():
        e = ReplayEngine(0)
        e.register_program(P.counter_program())
        return e

    ranks = D.LoopbackRanks(engine, part, feeds, cap)
    errors, _, _ = ranks.run(2)
    assert not any(errors), errors
    one = ReplayEngine(0)
    one.register_program(P.counter_program())
    one.fold_unsorted(arrival, n)
    return ranks.engines, one


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--batches", type=int, default=100)
    ap.add_argument("--batch", type=int, default=100_000)
    a = ap.parse_args()
    info = card()
    print(f"card: {info['card']}, power limit {info['power_limit']}", flush=True)
    ids = uuid_ids(a.n, 4)
    part = D.partitions_for_keys(ids, 32)
    ranks, one = rebuild(a.n, part)
    res = {"n_aggregates": a.n, "ranks": R, **info}
    probe = ids[:1000]
    res["load_keys_and_first_read_s"] = {
        "ranks": [timed(lambda e=e: (e.dist_load_keys(ids), e.get_many(probe, arrays=True)))[0] for e in ranks],
        "one_engine": timed(lambda: (one.load_keys(ids), one.get_many(probe, arrays=True)))[0]}
    rng = np.random.default_rng(5)
    batches = [[ids[i] for i in rng.integers(0, a.n, size=a.batch)] for _ in range(a.batches)]
    D.read_routed(ranks, batches[0], 32)    # warm-up
    one.get_many(batches[0], arrays=True)
    t_routed = sum(timed(lambda q=q: D.read_routed(ranks, q, 32, arrays=True))[0] for q in batches)
    t_one = sum(timed(lambda q=q: one.get_many(q, arrays=True))[0] for q in batches)
    # parity of the last batch
    got, want = D.read_routed(ranks, batches[-1], 32, arrays=True), one.get_many(batches[-1], arrays=True)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    res["get_many_s"] = {"batches": a.batches, "ids_per_batch": a.batch, "routed": t_routed, "one_engine": t_one}

    def count(pages, k):
        return sum(len(p[k]) for p in pages)

    exp = [timed(lambda e=e: count(e.export_changes(CH_ERR), 0)) for e in ranks]
    scan = [timed(lambda e=e: count(e.scan(), 0)) for e in ranks]
    exp1, scan1 = timed(lambda: count(one.export_changes(CH_ERR), 0)), timed(lambda: count(one.scan(), 0))
    assert sum(x[1] for x in exp) == exp1[1] and sum(x[1] for x in scan) == scan1[1]
    res["export_changes_s"] = {"ranks": [x[0] for x in exp], "one_engine": exp1[0], "rows": exp1[1]}
    res["scan_s"] = {"ranks": [x[0] for x in scan], "one_engine": scan1[0], "rows": scan1[1]}
    print(json.dumps(res), flush=True)
    for e in ranks + [one]:
        e.close()


if __name__ == "__main__":
    main()
