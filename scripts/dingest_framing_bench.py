"""Device ingest of protobuf-wrapped and play-json event values against the host decoder, on the same bytes.

bench.py's e2e shape: 2^20 aggregates x 32 events in 32 partitions of lz4 batches of 512 records, from pinned host memory,
every step a rebuild from offset 0 into an empty table. Keys are "<uuid>:<seq>". The same events are written five ways:
  packed         u32 type, u32 seq, i32 by (the control: no conversion)
  protobuf       the multilanguage Event { aggregateId, payload = the packed event }
  json_counter   play-json Counter events (TestBoundedContext), compact separators
  json_bank_money      BankAccount events, balances with two decimals
  json_bank_precise    BankAccount events, balances the repr of random doubles (the exact slow path of the double parse)
  protobuf_json        the multilanguage Counter's events as its gateway writes them: Event { aggregateId, payload = the
                       play-json event (the multilanguage TestBoundedContext) }, SGR_VALUE_PROTOBUF_JSON
  protobuf_json_state  a state-topic restore of the same aggregates: one State { aggregateId, payload = the play-json
                       AggregateState } per aggregate, keyed by the id (device only: the host decoder has no state-topic mode)
Per workload: wire bytes per event, device ms/step and events/s, timing slots [0] (copies + decode chains), [1] (the repeat
from an exact arena layout) and [4] (growth + fold) of sgr_dingest_last_timing, and the host decoder (sgr_ingest_record_batches_mt
+ sgr_fold_ingested) on the same bytes. The first device step is a warm-up: it also raises the arena claim for the framing.
Records are encoded in worker processes by scripts/kafka_values_encode.c, compiled into a temporary directory. Prints the card
name and power limit, then one JSON line per workload.

    python scripts/dingest_framing_bench.py [--steps 3] [--host-steps 1] [--aggregates 1048576] [--workloads a,b]
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

EPA, N_PART, RPB = 32, 32, 512
WORKLOADS = ["packed", "protobuf", "json_counter", "json_bank_money", "json_bank_precise", "protobuf_json", "protobuf_json_state"]
CLS = "surge.core.TestBoundedContext."
ML_CLS = "com.ukg.surge.multilanguage.TestBoundedContext."
_lib = None


def _encoder(libdir):
    global _lib
    if _lib is None:
        _lib = C.CDLL(os.path.join(libdir, "libkv.so"))
        _lib.kv_kafka_encode_values.restype = C.c_int64
        _lib.kv_kafka_encode_values.argtypes = [C.c_void_p] * 4 + [C.c_uint64, C.c_uint32, C.c_int, C.c_int64, C.c_void_p, C.c_uint64]
    return _lib


def _pb_varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def _ids(aggs):
    return [str(uuid.UUID(int=(a * 0x9E3779B97F4A7C15F39CC0605CEDC835 + 0x1234) & ((1 << 128) - 1))) for a in aggs]


def _pb(aid, payload):
    """the multilanguage Event / State { aggregateId = 1, payload = 2 }"""
    a = aid.encode()
    return b"\x0a" + _pb_varint(len(a)) + a + b"\x12" + _pb_varint(len(payload)) + payload


def _value(workload, aid, k, kind, by, dbl):
    seq = k + 1
    if workload == "protobuf_json":
        name, member = (("CountIncremented", "incrementBy"), ("CountDecremented", "decrementBy"))[kind % 2]
        return _pb(aid, ('{"_type":"%s%s","aggregateId":"%s","%s":%d,"sequenceNumber":%d}' % (ML_CLS, name, aid, member, by, seq)).encode())
    if workload == "protobuf_json_state":
        return _pb(aid, ('{"aggregateId":"%s","count":%d,"version":%d}' % (aid, by, EPA)).encode())
    if workload in ("packed", "protobuf"):
        packed = struct.pack("<IIi", kind, seq, by)
        if workload == "packed":
            return packed
        return _pb(aid, packed)
    if workload == "json_counter":
        name = ("CountIncremented", "CountDecremented", "NoOpEvent")[kind]
        member = ('"incrementBy":%d,' % by, '"decrementBy":%d,' % by, "")[kind]
        return ('{"_type":"%s%s","aggregateId":"%s",%s"sequenceNumber":%d}' % (CLS, name, aid, member, seq)).encode()
    if workload == "json_bank_money":
        bal = "%.2f" % (by / 100)
    else:
        bal = repr(dbl)
    if k == 0:
        return ('{"_type":"docs.command.BankAccountCreated","accountNumber":"%s","accountOwner":"owner-%s","securityCode":"1234","balance":%s}'
                % (aid, aid[:8], bal)).encode()
    return ('{"_type":"docs.command.BankAccountUpdated","accountNumber":"%s","newBalance":%s}' % (aid, bal)).encode()


def encode_partition(args):
    """one partition's wire bytes: event k of every aggregate of the partition before event k + 1 of any"""
    workload, p, n_agg, libdir, seed = args
    rng = np.random.default_rng([seed, p])
    aggs = list(range(p, n_agg, N_PART))
    ids = _ids(aggs)
    kinds = rng.integers(0, 3, (EPA, len(aggs)))
    bys = rng.integers(-10**6, 10**6, (EPA, len(aggs)))
    dbls = rng.integers(0, 2**64, (EPA, len(aggs)), dtype=np.uint64).view("<f8")   # random bits: every exponent
    dbls[~np.isfinite(dbls)] = 0.1
    keys, vals = [], []
    for k in range(1 if workload == "protobuf_json_state" else EPA):   # (a state topic: one record per aggregate, keyed by the id)
        for j, aid in enumerate(ids):
            keys.append(aid.encode() if workload == "protobuf_json_state" else b"%s:%d" % (aid.encode(), k + 1))
            vals.append(_value(workload, aid, k, int(kinds[k, j]), int(bys[k, j]), float(dbls[k, j])))
    n = len(keys)
    key_offs = np.zeros(n + 1, np.uint64)
    key_offs[1:] = np.cumsum([len(x) for x in keys])
    val_offs = np.zeros(n + 1, np.uint64)
    val_offs[1:] = np.cumsum([len(x) for x in vals])
    kb, vb = np.frombuffer(b"".join(keys), np.uint8), np.frombuffer(b"".join(vals), np.uint8)
    cap = int(key_offs[-1] + val_offs[-1]) + 32 * n + 160 * (n // RPB + 1)
    cap += cap // 255 + 1024
    out = np.empty(cap, np.uint8)
    got = _encoder(libdir).kv_kafka_encode_values(kb.ctypes.data, key_offs.ctypes.data, vb.ctypes.data, val_offs.ctypes.data, n, RPB, 1, 0,
                                                  out.ctypes.data, cap)
    if got < 0:
        raise RuntimeError(f"kv_kafka_encode_values failed ({got})")
    return out[:got].tobytes()


def encode(workload, n_agg, libdir, seed):
    import torch

    ctx = mp.get_context("spawn")
    with ctx.Pool(min(N_PART, os.cpu_count() or 1)) as pool:
        wires = pool.map(encode_partition, [(workload, p, n_agg, libdir, seed) for p in range(N_PART)])
    pinned = []
    for w in wires:
        t = torch.empty(len(w), dtype=torch.uint8, pin_memory=True)
        t.numpy()[:] = np.frombuffer(w, np.uint8)
        pinned.append(t)
    return pinned, sum(len(w) for w in wires)


def setup(g, workload):
    from surge_b200 import native as N

    if workload == "protobuf":
        g.set_value_framing(N.VALUE_PROTOBUF_EVENT)
    elif workload == "json_counter":
        g.set_json_packer("_type", [(CLS + "CountIncremented", 0, [("incrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)]),
                                    (CLS + "CountDecremented", 1, [("decrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)]),
                                    (CLS + "NoOpEvent", 2, [("sequenceNumber", N.JSON_I32, 4)])], unknown_type=3)
        g.set_value_framing(N.VALUE_JSON)
    elif workload.startswith("json_bank"):
        g.set_json_packer("_type", [("docs.command.BankAccountCreated", 0, [("accountNumber", N.JSON_UUID, 16), ("balance", N.JSON_F64, 32),
                                                                             ("accountOwner", N.JSON_PSTR, 40, 16), ("securityCode", N.JSON_PSTR, 56, 8)]),
                                    ("docs.command.BankAccountUpdated", 1, [("accountNumber", N.JSON_UUID, 16), ("newBalance", N.JSON_F64, 32)])])
        g.set_value_framing(N.VALUE_JSON)
    elif workload == "protobuf_json":
        g.set_json_packer("_type", [(ML_CLS + "CountIncremented", 0, [("incrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)]),
                                    (ML_CLS + "CountDecremented", 1, [("decrementBy", N.JSON_I32, 16), ("sequenceNumber", N.JSON_I32, 4)])])
        g.set_value_framing(N.VALUE_PROTOBUF_JSON)
    elif workload == "protobuf_json_state":
        g.set_state_topic(True)
        g.set_json_packer("", [("AggregateState", 0, [("count", N.JSON_I32, 0), ("version", N.JSON_I32, 4)])])
        g.set_value_framing(N.VALUE_PROTOBUF_JSON)


def program(workload):
    from surge_b200 import programs as P

    if workload.startswith("protobuf_json"):
        return P.ml_counter_program()
    return P.bank_account_program() if workload.startswith("json_bank") else P.counter_program()


def run_device(workload, pinned, n_agg, steps, warmup):
    from surge_b200 import ReplayEngine
    from surge_b200.dingest import DeviceIngest

    with ReplayEngine(0) as e:
        e.register_program(program(workload))
        with DeviceIngest(e, n_agg + 1024, 48 * (n_agg + 1024)) as dg:   # (36-byte UUID ids)
            setup(dg, workload)

            def step():
                e.set_initial_states(None)
                dg.reset()
                for p, t in enumerate(pinned):
                    dg.submit(p, t)
                return dg.fold()
            for _ in range(warmup):
                step()
            ms, slots = [], []
            for _ in range(steps):
                t0 = time.perf_counter()
                st = step()
                ms.append((time.perf_counter() - t0) * 1e3)
                tm = dg.last_timing()
                slots.append((tm["wait_copies_and_chains"], tm["decode_walk"], tm["grow_fold_append_keys"]))
            return ms, st, slots


def run_host(workload, pinned, steps):
    from surge_b200 import ReplayEngine
    from surge_b200.ingest import Ingest

    fetches = [(p, t.numpy()) for p, t in enumerate(pinned)]
    with ReplayEngine(0) as e:
        e.register_program(program(workload))
        ms, st = [], None
        for _ in range(steps):
            e.set_initial_states(None)
            ing = Ingest()
            try:
                setup(ing, workload)
                t0 = time.perf_counter()
                ing.record_batches_mt(fetches)
                e.fold_ingested(ing)
                ms.append((time.perf_counter() - t0) * 1e3)
                st = ing.stats()
            finally:
                ing.close()
        return ms, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--host-steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--aggregates", type=int, default=1 << 20)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    from scripts.get_batch_bench import card

    print(json.dumps(card()), flush=True)
    with tempfile.TemporaryDirectory() as libdir:
        subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-o", os.path.join(libdir, "libkv.so"), os.path.join(ROOT, "scripts", "kafka_values_encode.c")])
        for w in args.workloads.split(","):
            pinned, wire_bytes = encode(w, args.aggregates, libdir, 2026)
            ms, st, slots = run_device(w, pinned, args.aggregates, args.steps, args.warmup)
            state_topic = w == "protobuf_json_state"
            hms, hst = run_host(w, pinned, args.host_steps) if not state_topic else ([float("nan")], None)
            n = int(st["n_records"])
            assert state_topic or int(hst["n_records"]) == n, (hst, st)
            med, hmed = float(np.median(ms)), float(np.median(hms))
            s = np.median(np.asarray(slots), axis=0)
            print(json.dumps({"workload": w, "events": n, "wire_bytes_per_event": wire_bytes / n, "device_ms_per_step": ms, "device_median_ms": med,
                              "device_events_per_s": n / med * 1e3, "slot0_copies_and_chains_ms": float(s[0]), "slot1_exact_repeat_ms": float(s[1]),
                              "slot1_share": float(s[1]) / med, "slot4_grow_fold_ms": float(s[2]), "host_ms_per_step": hms,
                              "host_events_per_s": n / hmed * 1e3, "host_over_device": hmed / med,
                              "decompressed_over_compressed": int(st["n_decompressed_bytes"]) / max(1, int(st["n_compressed_bytes"]))}), flush=True)
            del pinned

if __name__ == "__main__":
    main()
