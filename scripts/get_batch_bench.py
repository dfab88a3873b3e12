"""Recovery reads: sgr_get_batch (device id index) against a loop of sgr_get (host snapshot + host KeyTable).

Setup per program: 10 M aggregate ids of 36 bytes in an engine's key table (appended, as an ingest does), a state table of random
states. Measured with host clocks around calls that end in a device synchronisation, after warm-ups, three repeats each:
  1. per-call ms of sgr_get_batch at 1, 1 k, 100 k and 1 M random ids, against a loop of sgr_get over the same ids with a warm
     snapshot;
  2. the first read after a fold that appended 1 % new ids: the batch path (index extension + read of 100 k ids) against the
     point path (snapshot copy + KeyTable rebuild + one read, then the other reads of the same ids).
Prints the card name and power limit first, then one JSON line per measurement; --out also writes them to a file.

    python scripts/get_batch_bench.py [--n 10000000] [--out results.jsonl]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from surge_b200 import ReplayEngine  # noqa: E402
from surge_b200 import programs as P  # noqa: E402

ID_BYTES = 36


def ids_blob(lo: int, hi: int) -> np.ndarray:
    """ids lo..hi-1 as 36 ASCII bytes each: 'agg-' and 32 decimal digits."""
    blob = np.empty((hi - lo, ID_BYTES), dtype=np.uint8)
    blob[:, :4] = np.frombuffer(b"agg-", np.uint8)
    v = np.arange(lo, hi, dtype=np.int64)
    for d in range(ID_BYTES - 1, 3, -1):
        blob[:, d] = v % 10 + ord("0")
        v //= 10
    return blob


def offsets(n: int) -> np.ndarray:
    return (np.arange(n + 1, dtype=np.uint64) * ID_BYTES).astype(np.uint32)


def card() -> dict:
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return {"card": name, "power_limit": pl}


class Reader:
    def __init__(self, e: ReplayEngine):
        self.e, self.lib, self.h = e, e._lib, e._h
        self.user = e.state_bytes - 8

    def batch(self, blob: np.ndarray) -> float:
        n = blob.shape[0]
        q = np.ascontiguousarray(blob).reshape(-1)
        qo = offsets(n)
        out = np.empty(n * self.user, dtype=np.uint8)
        fl = np.empty(n, dtype=np.uint32)
        t = time.perf_counter()
        rc = self.lib.sgr_get_batch(self.h, q.ctypes.data, qo.ctypes.data, n, out.ctypes.data, out.nbytes, fl.ctypes.data, None)
        dt = time.perf_counter() - t
        assert rc == 0, self.lib.sgr_last_error(self.h)
        return dt * 1e3

    def points(self, blob: np.ndarray) -> float:
        keys = [bytes(r) for r in blob]
        buf = C.create_string_buffer(128)
        outlen, exists = C.c_uint32(), C.c_int32()
        get, h = self.lib.sgr_get, self.h
        t = time.perf_counter()
        for k in keys:
            rc = get(h, k, ID_BYTES, buf, 128, C.byref(outlen), C.byref(exists))
            if rc:
                raise RuntimeError(self.lib.sgr_last_error(h))
        return (time.perf_counter() - t) * 1e3


def run(name: str, prog, n: int, emit) -> None:
    rng = np.random.default_rng(1)
    extra = n // 100
    cap = n + 4 * extra
    owner = C.c_void_p(0x5eed)
    with ReplayEngine(0) as e:
        e.register_program(prog)
        sb = e.state_bytes
        states = rng.integers(0, 256, size=(cap, sb), dtype=np.uint8)
        states[:, sb - 8:sb - 4] = np.frombuffer(np.uint32(1).tobytes(), np.uint8)   # every state exists
        e.set_initial_states(states)
        del states
        blob, offs = ids_blob(0, n), offsets(n)   # (named: ctypes gets their addresses, they must outlive the call)
        assert e._lib.sgr_append_keys(e._h, owner, blob.ctypes.data, offs.ctypes.data, n) == 0
        r = Reader(e)
        t_index = r.batch(blob[:1])         # builds the device index from all ids
        t_snap = r.points(blob[:1])         # builds the host KeyTable and snapshot
        emit({"program": name, "what": "first read after loading the key table", "n_ids": n, "batch_ms": t_index, "point_ms": t_snap})
        for k in (1, 1000, 100_000, 1_000_000):
            pick = rng.integers(0, n, size=k)
            q = blob[pick]
            r.batch(q); r.points(q[: min(k, 1000)])   # warm-up
            b = [r.batch(q) for _ in range(3)]
            p = [r.points(q) for _ in range(3)]
            emit({"program": name, "what": "per call, warm", "n_ids": k, "batch_ms": b, "point_loop_ms": p})
        # first read after a fold that appended 1 % new ids
        have = n
        rec = np.zeros((extra, 64), dtype=np.uint8)
        for rep in range(3):
            new, new_offs = ids_blob(have, have + extra), offsets(extra)
            assert e._lib.sgr_append_keys(e._h, owner, new.ctypes.data, new_offs.ctypes.data, extra) == 0
            rec[:, 8:16] = np.arange(have, have + extra, dtype=np.uint64).view(np.uint8).reshape(-1, 8)
            e.fold_incremental(rec)
            have += extra
            q = np.concatenate([blob[rng.integers(0, n, size=99_000)], new[:1000]])   # mostly old ids, some of the new ones
            tb = r.batch(q)
            tp_first = r.points(q[:1])
            tp_rest = r.points(q[1:])
            emit({"program": name, "what": "first read after a fold appending 1% new ids", "repeat": rep, "n_ids_total": have, "n_read": len(q),
                  "batch_ms": tb, "point_first_ms": tp_first, "point_rest_ms": tp_rest})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit(card())
    for name, prog in (("counter", P.counter_program()), ("bank_account", P.bank_account_program())):
        run(name, prog, a.n, emit)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
