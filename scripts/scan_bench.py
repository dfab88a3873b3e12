"""Ordered scan: sgr_scan (an id order kept on the device, pages compacted there) against the store's earlier host path (sort
every id on the host, then one sgr_get per id) and against export_states + a host sort of the ids + a numpy gather.

Two id families of --n ids each (10 M by default), appended to an engine's key table as an ingest does, dense order unrelated to
Bytes order: 36-byte UUID strings, which the sort mostly resolves in its first 8-byte window, and 'account-%012d', whose shared
prefix takes it through three windows. Each family runs with Counter (16-byte) and BankAccount (64-byte) tables, every state
existing. Measured, with host clocks around calls that end in a device synchronisation:
  - building the order from every id at the first scan (the id index is built by a get_batch before it, and timed apart);
  - extending it at the first scan after a fold that appended 1 % new ids (index extension again timed apart);
  - all(): every row through sgr_scan in pages of 2^20 rows, three repeats;
  - ranges returning 10, 1 k and 100 k rows, three repeats each from random starting ids;
  - export_states + a host argsort of the ids + a numpy gather of the rows, once;
  - the host path at --host-n ids (1 M by default; it is far too slow at 10 M): a sort of the Python strings and one sgr_get each.
Device memory: the order (free memory before and after it is built) and the peak while it is built (free memory sampled by a
second thread during the build). Prints the card name and power limit first, then one JSON line per measurement.

    python scripts/scan_bench.py [--n 10000000] [--host-n 1000000] [--out results.jsonl]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.get_batch_bench import card  # noqa: E402
from surge_b200 import ReplayEngine  # noqa: E402
from surge_b200 import native as N  # noqa: E402
from surge_b200 import programs as P  # noqa: E402

PAGE_ROWS = 1 << 20
PAGE_ID_BYTES = 64 << 20


def family_blob(name: str, lo: int, hi: int, rng) -> np.ndarray:
    """ids lo..hi-1 of a family as fixed-width rows of bytes."""
    n = hi - lo
    if name == "uuid":
        hexd = np.frombuffer(b"0123456789abcdef", np.uint8)[rng.integers(0, 16, size=(n, 32))]
        out = np.full((n, 36), ord("-"), np.uint8)
        out[:, 0:8], out[:, 9:13], out[:, 14:18], out[:, 19:23], out[:, 24:36] = hexd[:, 0:8], hexd[:, 8:12], hexd[:, 12:16], hexd[:, 16:20], hexd[:, 20:32]
        return out
    out = np.empty((n, 20), np.uint8)
    out[:, :8] = np.frombuffer(b"account-", np.uint8)
    v = lo + rng.permutation(n).astype(np.int64)   # appended in an order unrelated to Bytes order
    for d in range(19, 7, -1):
        out[:, d] = v % 10 + ord("0")
        v //= 10
    return out


def append(e, owner, blob: np.ndarray) -> None:
    offs = (np.arange(len(blob) + 1, dtype=np.uint64) * blob.shape[1]).astype(np.uint32)
    flat = np.ascontiguousarray(blob).reshape(-1)
    assert e._lib.sgr_append_keys(e._h, owner, flat.ctypes.data, offs.ctypes.data, len(blob)) == 0, e._lib.sgr_last_error(e._h)


class Scanner:
    def __init__(self, e: ReplayEngine, max_rows: int):
        self.e, self.lib, self.h = e, e._lib, e._h
        self.rows = np.empty((max_rows, e.state_bytes - 8), np.uint8)
        self.flags, self.idx = np.empty(max_rows, np.uint32), np.empty(max_rows, np.int64)
        self.ids = np.empty(PAGE_ID_BYTES, np.uint8)
        self.offs = np.empty(max_rows + 1, np.uint32)
        self.max_rows = max_rows

    def page(self, frm, excl, to, max_rows):
        n, more = C.c_uint64(), C.c_int32()
        fb = None if frm is None else C.create_string_buffer(frm, max(len(frm), 1))
        tb = None if to is None else C.create_string_buffer(to, max(len(to), 1))
        rc = self.lib.sgr_scan(self.h, fb, 0 if frm is None else len(frm), excl, tb, 0 if to is None else len(to), max_rows, self.rows.ctypes.data,
                               self.flags.ctypes.data, self.idx.ctypes.data, self.ids.ctypes.data, PAGE_ID_BYTES, self.offs.ctypes.data,
                               C.byref(n), C.byref(more))
        assert rc == 0, self.lib.sgr_last_error(self.h)
        k = n.value
        return k, more.value, (self.ids[self.offs[k - 1]:self.offs[k]].tobytes() if k else None)

    def scan(self, frm=None, to=None):
        """(ms, rows, pages) of one full scan of [frm, to] in pages of max_rows."""
        t = time.perf_counter()
        rows = pages = 0
        excl = 0
        while True:
            k, more, last = self.page(frm, excl, to, self.max_rows)
            rows += k
            pages += 1
            if not more:
                break
            frm, excl = last, 1
        return (time.perf_counter() - t) * 1e3, rows, pages


def timed_with_peak(fn):
    """(ms, result, lowest free device memory seen while fn ran)."""
    import torch

    low = [torch.cuda.mem_get_info(0)[0]]
    stop = threading.Event()

    def sample():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info(0)[0])
            time.sleep(0.0002)

    th = threading.Thread(target=sample)
    th.start()
    t = time.perf_counter()
    try:
        r = fn()
    finally:
        dt = (time.perf_counter() - t) * 1e3
        stop.set()
        th.join()
    return dt, r, low[0]


def touch_new(lo: int, hi: int, sb: int) -> np.ndarray:
    rec = np.zeros((hi - lo, 64), dtype=np.uint8)
    rec[:, 0:4] = np.frombuffer(np.uint32(0 if sb == 16 else 1).tobytes(), np.uint8)
    rec[:, 4:8] = np.frombuffer(np.uint32(7).tobytes(), np.uint8)
    rec[:, 8:16] = np.arange(lo, hi, dtype=np.uint64).view(np.uint8).reshape(-1, 8)
    rec[:, 16:24] = 5
    return rec


def warm_up() -> None:
    """Load the scan's kernels (the sort, the merge, the bounds) once, so that no measurement includes module loading."""
    rng = np.random.default_rng(3)
    owner = C.c_void_p(0x3)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        states = np.zeros((4096, 16), np.uint8)
        states[:, 8:12] = np.frombuffer(np.uint32(N.ST_EXISTS).tobytes(), np.uint8)
        e.set_initial_states(states)
        for fam in ("uuid", "account"):
            append(e, owner, family_blob(fam, 0, 2000, rng))
            Scanner(e, 100).scan()
            append(e, owner, family_blob(fam, 2000, 4000, rng))
            Scanner(e, 100).scan(b"a", b"b")
            owner = C.c_void_p(0x4)


def run(fam: str, prog_name: str, prog, n: int, emit) -> None:
    import torch

    rng = np.random.default_rng(1)
    extra = n // 100
    cap = n + extra
    owner = C.c_void_p(0x5eed)
    base = family_blob(fam, 0, n, rng)
    tag = {"family": fam, "program": prog_name, "id_bytes": base.shape[1]}
    with ReplayEngine(0) as e:
        e.register_program(prog)
        sb = e.state_bytes
        states = rng.integers(0, 256, size=(cap, sb), dtype=np.uint8)
        states[:, sb - 8:sb] = 0
        states[:, sb - 8:sb - 4] = np.frombuffer(np.uint32(N.ST_EXISTS).tobytes(), np.uint8)
        e.set_initial_states(states)
        del states
        append(e, owner, base)
        t = time.perf_counter()
        e.get_many([bytes(base[0]).decode()])                      # builds the device id index
        t_index = (time.perf_counter() - t) * 1e3
        x1 = Scanner(e, 1)
        free0 = torch.cuda.mem_get_info(0)[0]
        t_build, _, low = timed_with_peak(lambda: x1.page(None, 0, None, 1))
        free1 = torch.cuda.mem_get_info(0)[0]
        emit({**tag, "what": "order built from every id at the first scan (a 1-row page)", "n_ids": n, "scan_ms": t_build,
              "index_build_ms": t_index, "order_bytes": free0 - free1, "peak_bytes_during_build": free0 - low})
        x = Scanner(e, PAGE_ROWS)
        x.scan()                                                      # warm-up
        runs = [x.scan() for _ in range(3)]
        assert all(r == n for _, r, _ in runs), runs
        emit({**tag, "what": "all() through sgr_scan", "rows": n, "pages": runs[0][2], "scan_ms": [m for m, _, _ in runs]})
        order = np.argsort(base.view(f"S{base.shape[1]}").ravel(), kind="stable")   # (no \0 in these ids: S compares them right)
        for k in (10, 1000, 100_000):
            xs = Scanner(e, k)
            ts = []
            for s in rng.integers(0, n - k, size=4):
                frm, to = bytes(base[order[s]]), bytes(base[order[s + k - 1]])
                dt, got, _ = xs.scan(frm, to)
                assert got == k, (got, k)
                ts.append(dt)
            emit({**tag, "what": f"range returning {k} rows", "scan_ms": ts[1:]})   # (the first one warms the page size up)
        t = time.perf_counter()
        table = e.export_states()
        perm = np.argsort(base.view(f"S{base.shape[1]}").ravel(), kind="stable")
        rows = table[perm]
        t_host = (time.perf_counter() - t) * 1e3
        del table, rows, perm
        emit({**tag, "what": "export_states + host argsort of the ids + numpy gather", "rows": n, "ms": t_host})
        # a fold that appends 1 % new ids, then the first scan after it
        new = family_blob(fam, n, cap, rng)
        append(e, owner, new)
        e.fold_incremental(touch_new(n, cap, sb))
        t = time.perf_counter()
        e.get_many([bytes(new[0]).decode()])
        t_index = (time.perf_counter() - t) * 1e3
        free0 = torch.cuda.mem_get_info(0)[0]
        t_ext, _, low = timed_with_peak(lambda: x1.page(None, 0, None, 1))
        emit({**tag, "what": "order extended at the first scan after a fold appending 1% new ids", "n_ids_total": cap, "scan_ms": t_ext,
              "index_extension_ms": t_index, "peak_bytes_during_extension": free0 - low})
        dt, got, pages = x.scan()
        assert got == cap
        emit({**tag, "what": "all() through sgr_scan after the extension", "rows": got, "pages": pages, "scan_ms": dt})


def host_path(fam: str, prog_name: str, prog, n: int, emit) -> None:
    """The store's earlier all(): every id sorted in Python, then one sgr_get per id."""
    rng = np.random.default_rng(2)
    blob = family_blob(fam, 0, n, rng)
    keys = [bytes(r).decode() for r in blob]
    with ReplayEngine(0) as e:
        e.register_program(prog)
        sb = e.state_bytes
        states = rng.integers(0, 256, size=(n, sb), dtype=np.uint8)
        states[:, sb - 8:sb] = 0
        states[:, sb - 8:sb - 4] = np.frombuffer(np.uint32(N.ST_EXISTS).tobytes(), np.uint8)
        e.set_initial_states(states)
        e.load_keys(keys)
        e.get(keys[0])                                                # host key table and snapshot in place
        t = time.perf_counter()
        got = 0
        for k in sorted(keys, key=lambda s: s.encode("utf-8")):
            got += e.get(k) is not None
        dt = (time.perf_counter() - t) * 1e3
        assert got == n
        x = Scanner(e, PAGE_ROWS)
        dts = x.scan()[0]
        emit({"family": fam, "program": prog_name, "what": "host path: Python sort + one sgr_get per id (the earlier all())", "rows": n,
              "host_ms": dt, "scan_ms_same_table_first_scan": dts})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--host-n", type=int, default=1_000_000)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    lines = []

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)

    emit(card())
    emit({"page_rows": PAGE_ROWS, "page_id_bytes": PAGE_ID_BYTES})
    warm_up()
    for fam in ("uuid", "account"):
        for name, prog in (("counter", P.counter_program()), ("bank_account", P.bank_account_program())):
            run(fam, name, prog, a.n, emit)
            host_path(fam, name, prog, a.host_n, emit)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
