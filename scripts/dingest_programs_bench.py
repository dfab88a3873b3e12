"""Wire-format end to end per fold program: the device ingest (sgr_dingest_*) against the host decoder (sgr_ingest_* +
sgr_fold_ingested) on the same bytes, for Counter (sort-free: the control), BankAccount (64-byte state, f64, IF_EXISTS) and a
class-1 program of 14 state words from oracle/program_corpus.row_program.

The input has bench.py's e2e shape: 2^20 aggregates x 32 events in 32 partitions of lz4 batches of 512 records (65,536 batches),
in pinned host memory. Each partition also starts with a flush marker and ends with a refetch of its first 5 % of batches
(duplicates), so the poll holds holes. Every step is a rebuild from offset 0 into an empty table. Host clocks around calls that
end in a device synchronisation, after warm-up steps. The group-by's share is the engine's ms_group (device events around the
K5 group-by) over the step. Prints the card name and power limit first, then one JSON line per arm and decoder.

    python scripts/dingest_programs_bench.py [--steps 5] [--host-steps 2] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import kafka_batch as K  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import program_corpus as PC  # noqa: E402
from scripts.get_batch_bench import card  # noqa: E402
from surge_b200 import ReplayEngine  # noqa: E402
from surge_b200 import native as N  # noqa: E402
from surge_b200 import programs as P  # noqa: E402
from surge_b200.dingest import DeviceIngest  # noqa: E402
from surge_b200.ingest import Ingest  # noqa: E402

N_AGG, EPA, N_PART, RPB = 1 << 20, 32, 32, 512


def arms(rng):
    """(name, program, event types per record of the [N_AGG, EPA] log)."""
    counter = rng.integers(0, 3, size=(N_AGG, EPA)).astype(np.uint32)
    bank = np.ones((N_AGG, EPA), np.uint32)
    bank[:, 0] = 0                                            # BankAccountCreated, then BankAccountUpdated
    bank[rng.random(N_AGG) < 0.05, 0] = 1                     # some updates of accounts that do not exist
    rules = PC.row_program(rng, 14, 1, 8)
    wide = PC.type_mix(rules, N_AGG * EPA, rng).reshape(N_AGG, EPA)
    wide[:, 0] = 0                                            # type 0 is the class-1 program's CREATE
    return [("counter", P.counter_program(), counter), ("bank_account", P.bank_account_program(), bank),
            ("class1_w14", P.make_program(64, N.REC_FIXED64, rules), wide)]


def encode(types, rng):
    """32 partitions of wire bytes in pinned memory: a flush marker, the log's lz4 batches, then a refetch of the first 5 %."""
    import torch

    agg = np.repeat(np.arange(N_AGG, dtype=np.uint32), EPA).reshape(N_AGG, EPA)
    seq = np.tile(np.arange(1, EPA + 1, dtype=np.uint32), (N_AGG, 1))
    by = rng.integers(-1000, 1000, size=(N_AGG, EPA)).astype(np.int32)
    # arrival order: event k of every aggregate before event k + 1 of any aggregate of the partition
    def one(p):
        sl = slice(p, None, N_PART)
        a, t, s, b = (x[sl].T.reshape(-1) for x in (agg, types, seq, by))
        body = O.kafka_encode_counter(a, t, s, b, recs_per_batch=RPB, lz4=True, base_offset=1).tobytes()
        dup = (len(a) // 20) // RPB * RPB
        head = O.kafka_encode_counter(a[:dup], t[:dup], s[:dup], b[:dup], recs_per_batch=RPB, lz4=True, base_offset=1).tobytes()
        return K.encode_record_batch(0, [(0, b"", b"")]) + body + head
    with ThreadPoolExecutor(max_workers=min(N_PART, os.cpu_count() or 1)) as ex:
        wires = list(ex.map(one, range(N_PART)))
    pinned = []
    for w in wires:
        t = torch.empty(len(w), dtype=torch.uint8, pin_memory=True)
        t.numpy()[:] = np.frombuffer(w, np.uint8)
        pinned.append(t)
    return pinned, sum(len(w) for w in wires)


def run_device(prog, pinned, steps, warmup):
    with ReplayEngine(0) as e:
        e.register_program(prog)
        with DeviceIngest(e, N_AGG + 1024) as dg:
            def step():
                e.set_initial_states(None)
                dg.reset()
                for p, t in enumerate(pinned):
                    dg.submit(p, t)
                return dg.fold()
            for _ in range(warmup):
                step()
            ms, group, fold_slot = [], [], []
            for _ in range(steps):
                t0 = time.perf_counter()
                st = step()
                ms.append((time.perf_counter() - t0) * 1e3)
                group.append(float(e.stats().ms_group))
                fold_slot.append(dg.last_timing()["grow_fold_append_keys"])
            return ms, st, {"ms_group": group, "grow_fold_append_keys_ms": fold_slot}, e.export_states()


def run_host(prog, pinned, steps, warmup):
    fetches = [(p, t.numpy()) for p, t in enumerate(pinned)]
    with ReplayEngine(0) as e:
        e.register_program(prog)
        def step():
            e.set_initial_states(None)
            ing = Ingest()
            try:
                ing.record_batches_mt(fetches)
                e.fold_ingested(ing)
                return ing.stats()
            finally:
                ing.close()
        for _ in range(warmup):
            step()
        ms = []
        for _ in range(steps):
            t0 = time.perf_counter()
            st = step()
            ms.append((time.perf_counter() - t0) * 1e3)
        return ms, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--host-steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--arms", default="counter,bank_account,class1_w14")
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    rng = np.random.default_rng(2024)
    for name, prog, types in arms(rng):
        if name not in args.arms.split(","):
            continue
        pinned, wire_bytes = encode(types, rng)
        ms, st, timing, dev_table = run_device(prog, pinned, args.steps, args.warmup)
        n = int(st["n_records"])
        med = float(np.median(ms))
        print(json.dumps({"arm": name, "decoder": "device", "events": n, "holes": int(st["n_markers"] + st["n_duplicates"]),
                          "wire_bytes": int(wire_bytes), "ms_per_step": ms, "median_ms": med, "events_per_s": n / med * 1e3,
                          "group_share_of_step": float(np.median(timing["ms_group"])) / med, **timing}), flush=True)
        hms, hst = run_host(prog, pinned, args.host_steps, args.warmup)
        hmed = float(np.median(hms))
        print(json.dumps({"arm": name, "decoder": "host", "events": int(hst["n_records"]), "ms_per_step": hms, "median_ms": hmed,
                          "events_per_s": int(hst["n_records"]) / hmed * 1e3}), flush=True)
        del pinned, dev_table


if __name__ == "__main__":
    main()
