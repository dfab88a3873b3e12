"""Keyed state writes: sgr_put_batch against today's state-topic path (snapshot / tombstone events through sgr_fold_incremental,
the key table reloaded with sgr_load_keys whenever it grew), for 10 M UUID ids in batches of 100 k and of 10 M.

    python scripts/put_batch_bench.py [--ids 10000000] [--repeat 3]

Counter (16-byte state) runs both paths; the 128-byte state runs sgr_put_batch only (a snapshot record carries at most 48
program bytes). Each batch's arrays are built before the clock starts: the times are the C calls (upload, device work, host key
table), wall clock. One JSON line per (state, batch size, path): min / median / max of the total over --repeat runs."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time
import uuid

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from surge_b200 import ReplayEngine  # noqa: E402
from surge_b200 import native as N  # noqa: E402
from surge_b200 import programs as P  # noqa: E402


def id_blob(ids):
    enc = [k.encode() for k in ids]
    offs = np.zeros(len(enc) + 1, np.uint32)
    np.cumsum([len(b) for b in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc), np.uint8), offs


def put_path(sb, batches):
    with ReplayEngine(0) as e:
        e.register_program(P.make_program(sb, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])]))
        t0 = time.perf_counter()
        for blob, offs, rows, present in batches:
            n_new = C.c_uint64()
            e._ck(e._lib.sgr_put_batch(e._h, blob.ctypes.data, offs.ctypes.data, len(present), rows.ctypes.data, present.ctypes.data, C.byref(n_new)))
        return time.perf_counter() - t0


def snapshot_path(batches, all_ids):
    """all_ids: (blob, offsets) of every id; a key table of the first n ids is its prefix (the store also pads the table to the
    capacity with placeholder ids, which this leaves out: the times favour today's path)."""
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program_with_snapshot_rules())
        cap, n_keys = 0, 0
        t0 = time.perf_counter()
        for recs, n_after in batches:
            if n_after > cap:
                cap = max(2 * n_after, 1024)
                e.grow_states(cap)
            e.fold_incremental(recs)
            if n_after != n_keys:
                blob, offs = all_ids
                e._ck(e._lib.sgr_load_keys(e._h, blob.ctypes.data, offs.ctypes.data, n_after))
                n_keys = n_after
        return time.perf_counter() - t0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ids", type=int, default=10_000_000)
    ap.add_argument("--repeat", type=int, default=3)
    args = ap.parse_args()
    rng = np.random.default_rng(1)
    ids = [str(uuid.UUID(bytes=rng.bytes(16))) for _ in range(args.ids)]
    for batch in (100_000, args.ids):
        cuts = list(range(0, args.ids, batch))
        for sb in (16, 128):
            user = sb - 8
            staged = []
            for c in cuts:
                blob, offs = id_blob(ids[c:c + batch])
                rows = rng.integers(0, 256, size=(len(offs) - 1, user), dtype=np.uint8)
                staged.append((blob, offs, rows, np.ones(len(offs) - 1, np.uint8)))
            times = sorted(put_path(sb, staged) for _ in range(args.repeat))
            print(json.dumps({"state_bytes": sb, "batch": batch, "path": "sgr_put_batch", "ids": args.ids,
                              "s_min": times[0], "s_median": times[len(times) // 2], "s_max": times[-1]}), flush=True)
            if sb != 16:
                continue
            recs_batches = []
            for k, c in enumerate(cuts):
                part = staged[k]
                n = len(part[3])
                recs = np.zeros((n, 64), np.uint8)
                recs[:, 0:4] = np.frombuffer(np.uint32(P.COUNTER_SNAPSHOT_TYPE).tobytes(), np.uint8)
                recs[:, 8:16] = np.arange(c, c + n, dtype=np.uint64).view(np.uint8).reshape(-1, 8)
                recs[:, 16:24] = part[2][:, :8]
                recs_batches.append((recs, c + n))
            all_ids = id_blob(ids)
            times = sorted(snapshot_path(recs_batches, all_ids) for _ in range(args.repeat))
            print(json.dumps({"state_bytes": sb, "batch": batch, "path": "snapshot events + sgr_fold_incremental + sgr_load_keys",
                              "ids": args.ids, "s_min": times[0], "s_median": times[len(times) // 2], "s_max": times[-1]}), flush=True)


if __name__ == "__main__":
    main()
