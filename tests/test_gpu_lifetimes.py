"""-m gpu: a handle's destroy call gives back the device memory it took (include/sgr.h: sgr_destroy frees engine memory).

Each case runs the same work three times, destroying every handle after each cycle, and reads the device's free memory once the
torch allocator has returned its cache. The first cycle absorbs what stays loaded for the process (kernel modules, library
state); the second and the third must end within 2 MiB of where the first ended. A buffer, stream or event that a destroy call
missed would leave the second and third cycles lower, by its size each time.
  (a) one engine: load, fold, incremental fold, batched read, changed-state export, scan, put batch and a value-returning read
      under a state writer;
  (b) a device ingest with a JSON packer: submits and folds of lz4 and uncompressed fetches, several polls;
  (c) two loopback routed ranks: the pipelined route and fold, then their rank key tables, batched reads and scans.
The test also passes on the code before the host resources got owner types (devbuf.h): no leak on a success path was known
there. It keeps the owners honest from here on. On an H100 80GB HBM3 every case ended its three cycles at the same free memory,
to the byte.
"""
import gc
import json

import numpy as np
import pytest

from oracle import kafka_batch as K
from surge_b200 import ReplayEngine
from surge_b200 import dist as D
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200 import synth as S
from surge_b200.dingest import DeviceIngest

pytestmark = pytest.mark.gpu

SLACK = 2 << 20
CH_ERR = N.ST_CHANGED | N.ST_ERROR
CLS = "surge.core.TestBoundedContext."
COUNTER_JSON = [(CLS + "CountIncremented", 0, [("incrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)]),
                (CLS + "CountDecremented", 1, [("decrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)])]
COUNTER_WRITER = [("aggregateId", N.JSON_ID), ("count", N.JSON_I32, 0), ("version", N.JSON_I32, 4)]


def free_after_release():
    import torch

    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(0)[0]


def engine_cycle():
    n_agg = 20000
    rng = np.random.default_rng(1)
    rec, off = S.counter_csr(n_agg, rng.integers(0, 24, size=n_agg), seed=2, p_throw=0.002)
    ids = [f"agg-{g}" for g in range(n_agg)]
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        e.load_events(rec, off)
        e.fold()
        e.load_keys(ids)
        e.fold_incremental(S.interleave_arrival(rec, seed=3)[:50000].copy())
        rows = e.get_many(ids[::7])
        changed = sum(len(p[0]) for p in e.export_changes(CH_ERR, page_rows=4099))
        scanned = sum(len(p[0]) for p in e.scan(page_rows=4099))
        fresh = [f"put-{i}" for i in range(3000)]
        n_new = e.put_batch(ids[:3000] + fresh, np.zeros((6000, 8), dtype=np.uint8))
        e.set_state_writer(COUNTER_WRITER)
        values = e.get_many_values(ids[:5000] + fresh[:1000])
    assert n_new == len(fresh) and changed and 0 < scanned <= n_agg and any(r is not None for r in rows)
    return len(rows), changed, scanned, n_new, sum(len(v) for v in values if v is not None)


def counter_event(name, agg, seq, **kw):
    return (f"{agg}:{seq}".encode(), json.dumps({"_type": CLS + name, "aggregateId": agg, **kw, "sequenceNumber": seq},
                                                separators=(",", ":")).encode())


def ingest_cycle():
    rng = np.random.default_rng(4)
    folded = []
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1 << 16) as dg:
            dg.set_json_packer("_type", COUNTER_JSON, -1)
            dg.set_value_framing(N.VALUE_JSON)
            seq, off = {}, {0: 0, 1: 0}
            for poll in range(3):
                for part in (0, 1):
                    events = []
                    for agg in rng.integers(0, 2000 * (poll + 1), size=3000):
                        key = f"acct-{part}-{agg}"
                        seq[key] = seq.get(key, 0) + 1
                        events.append(counter_event("CountIncremented", key, seq[key], incrementBy=int(agg % 5)))
                    for lo in range(0, len(events), 500):
                        chunk = events[lo:lo + 500]
                        dg.submit(part, K.encode_record_batch(off[part], [(d, k, v) for d, (k, v) in enumerate(chunk)],
                                                              compression="lz4" if lo % 1000 else "none"))
                        off[part] += len(chunk)
                folded.append(dg.fold()["n_records"])
            assert all(e.get(k) is not None for k in list(seq)[:500])
    assert folded == [6000, 6000, 6000]
    return tuple(folded)


def routed_cycle():
    import torch

    n_agg, chunks = 30000, 4
    rng = np.random.default_rng(5)
    rec, _ = S.counter_csr(n_agg, rng.integers(0, 16, size=n_agg), seed=6)
    arrival = np.ascontiguousarray(S.interleave_arrival(rec, seed=7)).view(np.uint8).reshape(-1, 64)
    aggs = arrival[:, 8:16].copy().view(np.uint64).reshape(-1)
    feeds = [arrival[aggs % 2 == r] for r in range(2)]   # each aggregate comes from one rank, in log order
    ids = [f"acct-{g:x}" + ":q" * (g % 3) for g in range(n_agg)]
    part = D.partitions_for_keys(ids, 32)
    cap = 2 * chunks * max(D.chunk_records(len(f), chunks) for f in feeds) + 1024

    def engine():
        e = ReplayEngine(0)
        e.register_program(P.counter_program())
        e.set_option("push_chunks", chunks)
        return e

    dev_feeds = [torch.from_numpy(np.ascontiguousarray(f).reshape(-1)).to("cuda:0") for f in feeds]
    with D.LoopbackRanks(engine, part, dev_feeds, cap) as ranks:
        errors, _, _ = ranks.run(2)
        assert not any(errors), errors
        for e in ranks.engines:
            e.dist_load_keys(ids)
        rows = D.read_routed(ranks.engines, ids[::5], 32)
        scanned = sum(1 for _ in D.merge_scans(ranks.engines, page_rows=3001))
    assert any(r is not None for r in rows) and 0 < scanned <= n_agg
    return len(rows), scanned


@pytest.mark.parametrize("cycle", [engine_cycle, ingest_cycle, routed_cycle], ids=["engine", "device_ingest", "loopback_ranks"])
def test_destroy_returns_device_memory(cycle):
    free_after_release()   # (the context and the torch allocator exist before the first reading)
    results, free = [], []
    for _ in range(3):
        results.append(cycle())
        free.append(free_after_release())
    assert results[1] == results[0] and results[2] == results[0], results
    drift = [free[0] - f for f in free[1:]]
    print(f"\n{cycle.__name__}: free device memory after each cycle {free}, drift after cycles 2 and 3 {drift} bytes")
    assert all(abs(d) <= SLACK for d in drift), f"free device memory after cycles 2 and 3 moved by {drift} bytes from cycle 1"
