"""Changed-state export: sgr_export_changes (compaction on the device) against export_states(bitmaps=True) + a numpy filter + an
id lookup (the whole table over PCIe, then the host finds the changed rows and their ids).

Setup per program: 10 M aggregate ids of 36 bytes appended to an engine's key table (as an ingest does), a state table of random
existing states. For each changed fraction (0.1 %, 1 %, 10 %, 100 %) one incremental batch touches that many distinct
aggregates, then both exports run three times; a full export through sgr_export_changes is paged at 2^20 rows and 64 MiB of ids.
Host clocks around calls that end in a device synchronisation, after a warm-up. Also: the first export after a fold that
appended 1 % new ids, which includes extending the device id index.
Prints the card name and power limit first, then one JSON line per measurement; --out also writes them to a file.

    python scripts/changes_bench.py [--n 10000000] [--out results.jsonl]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.get_batch_bench import ID_BYTES, card, ids_blob, offsets  # noqa: E402
from surge_b200 import ReplayEngine  # noqa: E402
from surge_b200 import native as N  # noqa: E402
from surge_b200 import programs as P  # noqa: E402

PAGE_ROWS = 1 << 20
PAGE_ID_BYTES = 64 << 20


class Exporter:
    def __init__(self, e: ReplayEngine):
        self.e, self.lib, self.h = e, e._lib, e._h
        user = e.state_bytes - 8
        self.rows = np.empty((PAGE_ROWS, user), np.uint8)
        self.flags, self.err = np.empty(PAGE_ROWS, np.uint32), np.empty(PAGE_ROWS, np.uint32)
        self.idx = np.empty(PAGE_ROWS, np.int64)
        self.ids = np.empty(PAGE_ID_BYTES, np.uint8)
        self.offs = np.empty(PAGE_ROWS + 1, np.uint32)

    def changes(self, n_agg: int):
        """(ms, rows, pages) of one full export of the CHANGED rows."""
        cur, n, rows, pages = N.sgr_changes_cursor(), C.c_uint64(), 0, 0
        t = time.perf_counter()
        while True:
            rc = self.lib.sgr_export_changes(self.h, N.ST_CHANGED, C.byref(cur), PAGE_ROWS, self.rows.ctypes.data, self.flags.ctypes.data,
                                             self.err.ctypes.data, self.idx.ctypes.data, self.ids.ctypes.data, PAGE_ID_BYTES,
                                             self.offs.ctypes.data, C.byref(n))
            assert rc == 0, self.lib.sgr_last_error(self.h)
            rows += n.value
            pages += 1
            if cur.next >= n_agg:
                break
        return (time.perf_counter() - t) * 1e3, rows, pages

    def whole_table(self, blob: np.ndarray):
        """(ms, rows): export_states with bitmaps, the changed rows' indices from the bitmap, their rows and ids gathered."""
        t = time.perf_counter()
        table, _, changed, _ = self.e.export_states(bitmaps=True)
        idx = np.nonzero(np.unpackbits(changed, bitorder="little")[:len(table)])[0]
        rows = table[idx]
        ids = blob[idx[idx < len(blob)]]
        dt = (time.perf_counter() - t) * 1e3
        del table, rows, ids
        return dt, len(idx)


def touch(n_touch: int, n: int, rng, sb: int) -> np.ndarray:
    """One record per aggregate for n_touch distinct aggregates below n: Counter increments, BankAccount balance updates."""
    aggs = rng.choice(n, size=n_touch, replace=False) if n_touch < n else np.arange(n)
    rec = np.zeros((n_touch, 64), dtype=np.uint8)
    rec[:, 0:4] = np.frombuffer(np.uint32(0 if sb == 16 else 1).tobytes(), np.uint8)
    rec[:, 4:8] = np.frombuffer(np.uint32(7).tobytes(), np.uint8)
    rec[:, 8:16] = aggs.astype(np.uint64).view(np.uint8).reshape(-1, 8)
    rec[:, 16:24] = rng.integers(1, 1 << 62, size=n_touch, dtype=np.int64).view(np.uint8).reshape(-1, 8)
    rec[:, 32:40] = rng.integers(1, 1 << 62, size=n_touch, dtype=np.int64).view(np.uint8).reshape(-1, 8)
    return rec


def run(name: str, prog, n: int, emit) -> None:
    rng = np.random.default_rng(1)
    extra = n // 100
    cap = n + 4 * extra
    owner = C.c_void_p(0x5eed)
    with ReplayEngine(0) as e:
        e.register_program(prog)
        sb = e.state_bytes
        states = rng.integers(0, 256, size=(cap, sb), dtype=np.uint8)
        states[:, sb - 8:sb] = 0
        states[:, sb - 8:sb - 4] = np.frombuffer(np.uint32(N.ST_EXISTS).tobytes(), np.uint8)   # every state exists, nothing changed
        e.set_initial_states(states)
        del states
        blob, offs = ids_blob(0, n), offsets(n)
        assert e._lib.sgr_append_keys(e._h, owner, blob.ctypes.data, offs.ctypes.data, n) == 0
        x = Exporter(e)
        e.fold_incremental(touch(1000, n, rng, sb))
        t_first, _, _ = x.changes(cap)                      # builds the device index from all ids
        emit({"program": name, "what": "first export after loading the key table", "n_ids": n, "export_changes_ms": t_first})
        for frac in (0.001, 0.01, 0.1, 1.0):
            k = int(n * frac)
            e.fold_incremental(touch(k, n, rng, sb))
            x.changes(cap); x.whole_table(blob)             # warm-up
            c = [x.changes(cap) for _ in range(3)]
            w = [x.whole_table(blob) for _ in range(3)]
            assert all(r == c[0][1] for _, r, _ in c) and all(r == c[0][1] for _, r in w), (c, w)
            emit({"program": name, "what": "full export of the changed rows", "n_agg": cap, "changed": c[0][1], "fraction": frac,
                  "pages": c[0][2], "export_changes_ms": [m for m, _, _ in c], "export_states_filter_ms": [m for m, _ in w]})
        have, all_ids = n, blob
        for rep in range(3):
            new, new_offs = ids_blob(have, have + extra), offsets(extra)
            all_ids = np.concatenate([all_ids, new])
            assert e._lib.sgr_append_keys(e._h, owner, new.ctypes.data, new_offs.ctypes.data, extra) == 0
            rec = touch(extra, have, rng, sb)
            rec[:, 8:16] = np.arange(have, have + extra, dtype=np.uint64).view(np.uint8).reshape(-1, 8)   # the new aggregates
            e.fold_incremental(np.concatenate([rec, touch(extra, have, rng, sb)]))
            have += extra
            tc, rows, _ = x.changes(cap)
            tw, _ = x.whole_table(all_ids)
            emit({"program": name, "what": "first export after a fold appending 1% new ids", "repeat": rep, "n_ids_total": have,
                  "changed": rows, "export_changes_ms": tc, "export_states_filter_ms": tw})


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
    emit({"id_bytes": ID_BYTES, "page_rows": PAGE_ROWS, "page_id_bytes": PAGE_ID_BYTES})
    for name, prog in (("counter", P.counter_program()), ("bank_account", P.bank_account_program())):
        run(name, prog, a.n, emit)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
