"""Restore of a compacted STATE topic on the device (sgr_dingest_set_state_topic) against the events-mode route with snapshot rules.

The topic: 10 M UUID ids, one record per id, then 10 % updates and 2 % tombstones of random ids, in 32 partitions of lz4
batches of 512 records, from pinned host memory. Every step is a rebuild from offset 0 into an empty table; the host clock runs
around fold() (the submits before it launch the decode chains behind their copies), after a warm-up. Workloads:
  counter_packed     Counter state (16 bytes): the 8 program bytes as the value; state mode only (no type header for events)
  counter_json       Json.toJson(State) = {"aggregateId","count","version"}; state mode, and events mode through
                     counter_snapshot_restore_program + set_null_value_type(1) (the route before state mode)
  bank_json          BankAccount (64 bytes) as {"accountNumber","accountOwner","securityCode","balance"}; state mode only
                     (56 program bytes: more than a snapshot event carries)
  state128_packed    a 128-byte state, 120 program bytes as the value; state mode only
Per cell: fold ms/step, records/s over the fold, submit ms, and slots [0] / [1] / [4] of sgr_dingest_last_timing. Prints the
card name and power limit first, then one JSON line per cell. Records are encoded by scripts/kafka_values_encode.c in worker
processes, compiled into a temporary directory.

    python scripts/dingest_states_bench.py [--steps 3] [--warmup 1] [--ids 10000000] [--workloads a,b]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import multiprocessing as mp
import os
import struct
import subprocess
import sys
import tempfile
import time
import uuid

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_PART, RPB = 32, 512
WORKLOADS = ["counter_packed", "counter_json", "bank_json", "state128_packed"]
_lib = None


def _encoder(libdir):
    global _lib
    if _lib is None:
        _lib = C.CDLL(os.path.join(libdir, "libkv.so"))
        _lib.kv_kafka_encode_values_nulls.restype = C.c_int64
        _lib.kv_kafka_encode_values_nulls.argtypes = [C.c_void_p] * 5 + [C.c_uint64, C.c_uint32, C.c_int, C.c_int64, C.c_void_p, C.c_uint64]
    return _lib


def _value(workload, aid, count, version, rng):
    if workload == "counter_packed":
        return struct.pack("<ii", count, version)
    if workload == "counter_json":
        return ('{"aggregateId":"%s","count":%d,"version":%d}' % (aid, count, version)).encode()
    if workload == "bank_json":
        return ('{"accountNumber":"%s","accountOwner":"owner-%s","securityCode":"1234","balance":%.2f}' % (aid, aid[:8], count / 100)).encode()
    return struct.pack("<ii", count, version) + bytes([version & 7]) * 112   # state128_packed: 120 program bytes


def encode_partition(args):
    """one partition's wire bytes: every id of the partition once, then 10 % updates and 2 % tombstones of random ids"""
    workload, p, n_ids, libdir, seed = args
    rng = np.random.default_rng([seed, p])
    ids = [str(uuid.UUID(int=(a * 0x9E3779B97F4A7C15F39CC0605CEDC835 + 0x1234) & ((1 << 128) - 1))) for a in range(p, n_ids, N_PART)]
    m = len(ids)
    order = np.concatenate([np.arange(m), rng.integers(0, m, size=m // 10), rng.integers(0, m, size=m // 50)])
    nulls = np.zeros(len(order), np.uint8)
    nulls[m + m // 10:] = 1
    counts = rng.integers(-10**6, 10**6, size=len(order))
    keys, vals = [], []
    for j, a in enumerate(order):
        keys.append(ids[a].encode())
        vals.append(b"" if nulls[j] else _value(workload, ids[a], int(counts[j]), j, rng))
    n = len(keys)
    key_offs = np.zeros(n + 1, np.uint64)
    key_offs[1:] = np.cumsum([len(x) for x in keys])
    val_offs = np.zeros(n + 1, np.uint64)
    val_offs[1:] = np.cumsum([len(x) for x in vals])
    kb, vb = np.frombuffer(b"".join(keys), np.uint8), np.frombuffer(b"".join(vals) or b"\0", np.uint8)
    cap = int(key_offs[-1] + val_offs[-1]) + 32 * n + 160 * (n // RPB + 1)
    cap += cap // 255 + 1024
    out = np.empty(cap, np.uint8)
    got = _encoder(libdir).kv_kafka_encode_values_nulls(kb.ctypes.data, key_offs.ctypes.data, vb.ctypes.data, val_offs.ctypes.data, nulls.ctypes.data,
                                                        n, RPB, 1, 0, out.ctypes.data, cap)
    if got < 0:
        raise RuntimeError(f"kv_kafka_encode_values_nulls failed ({got})")
    return out[:got].tobytes()


def encode(workload, n_ids, libdir, seed):
    import torch

    ctx = mp.get_context("spawn")
    with ctx.Pool(min(N_PART, os.cpu_count() or 1)) as pool:
        wires = pool.map(encode_partition, [(workload, p, n_ids, libdir, seed) for p in range(N_PART)])
    pinned = []
    for w in wires:
        t = torch.empty(len(w), dtype=torch.uint8, pin_memory=True)
        t.numpy()[:] = np.frombuffer(w, np.uint8)
        pinned.append(t)
    return pinned, sum(len(w) for w in wires)


def program(workload, mode):
    from surge_b200 import native as N
    from surge_b200 import programs as P

    if mode == "events":
        return P.counter_snapshot_restore_program()
    if workload == "bank_json":
        return P.bank_account_program()
    if workload == "state128_packed":
        return P.make_program(128, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])])
    return P.counter_program()


def setup(g, workload, mode):
    from surge_b200 import native as N

    if mode == "events":   # the route before state mode: JSON snapshots as events of a program with snapshot rules
        g.set_json_packer("", [("State", 0, [("count", N.JSON_I32, 16), ("version", N.JSON_I32, 20)])])
        g.set_value_framing(N.VALUE_JSON)
        g.set_null_value_type(1)
        return
    g.set_state_topic(True)
    if workload == "counter_json":
        g.set_json_packer("", [("State", 0, [("count", N.JSON_I32, 0), ("version", N.JSON_I32, 4)])])
        g.set_value_framing(N.VALUE_JSON)
    elif workload == "bank_json":
        g.set_json_packer("", [("BankAccount", 0, [("accountNumber", N.JSON_UUID, 0), ("balance", N.JSON_F64, 16), ("accountOwner", N.JSON_PSTR, 24, 16),
                                                    ("securityCode", N.JSON_PSTR, 40, 8)])])
        g.set_value_framing(N.VALUE_JSON)


def run(workload, mode, pinned, n_ids, steps, warmup):
    from surge_b200 import ReplayEngine
    from surge_b200.dingest import DeviceIngest

    with ReplayEngine(0) as e:
        e.register_program(program(workload, mode))
        with DeviceIngest(e, n_ids + 1024, 48 * (n_ids + 1024)) as dg:   # (36-byte UUID ids)
            setup(dg, workload, mode)
            fold_ms, submit_ms, slots, st = [], [], [], None
            for k in range(warmup + steps):
                e.set_initial_states(None)
                dg.reset()
                t0 = time.perf_counter()
                for p, t in enumerate(pinned):
                    dg.submit(p, t)
                t1 = time.perf_counter()
                st = dg.fold()
                t2 = time.perf_counter()
                if k >= warmup:
                    submit_ms.append((t1 - t0) * 1e3)
                    fold_ms.append((t2 - t1) * 1e3)
                    tm = dg.last_timing()
                    slots.append((tm["wait_copies_and_chains"], tm["decode_walk"], tm["grow_fold_append_keys"]))
            return fold_ms, submit_ms, slots, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ids", type=int, default=10_000_000)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    from scripts.get_batch_bench import card

    print(json.dumps(card()), flush=True)
    with tempfile.TemporaryDirectory() as libdir:
        subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-o", os.path.join(libdir, "libkv.so"), os.path.join(ROOT, "scripts", "kafka_values_encode.c")])
        for w in args.workloads.split(","):
            pinned, wire_bytes = encode(w, args.ids, libdir, 2026)
            for mode in (("state", "events") if w == "counter_json" else ("state",)):
                fold_ms, submit_ms, slots, st = run(w, mode, pinned, args.ids, args.steps, args.warmup)
                n = int(st["n_records"])
                med = float(np.median(fold_ms))
                s = np.median(np.asarray(slots), axis=0)
                print(json.dumps({"workload": w, "mode": mode, "records": n, "tombstones": int(st["n_null_values"]), "new_ids": int(st["n_new_keys"]),
                                  "wire_bytes": wire_bytes, "fold_ms_per_step": fold_ms, "fold_median_ms": med, "records_per_s": n / med * 1e3,
                                  "submit_median_ms": float(np.median(submit_ms)), "slot0_copies_and_chains_ms": float(s[0]),
                                  "slot1_exact_repeat_ms": float(s[1]), "slot4_grow_apply_ms": float(s[2])}), flush=True)
            del pinned


if __name__ == "__main__":
    main()
