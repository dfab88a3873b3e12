"""Measure the JSON state value reads (sgr_get_batch_values, sgr_export_changes_values, sgr_scan_values) on one GPU.

Tables: 10 M Counter rows and 10 M BankAccount rows, both with UUID ids, written by sgr_put_batch. Timed, each beside its
row-returning twin:
  get_many_values   100 batches of 100 k ids, and one batch of 10 M ids       (twin: get_many(arrays=True))
  export            a full export_changes_values of the table                  (twin: export_changes)
  scan              a full scan_values                                          (twin: scan)
the same three reads again with each value wrapped in the multilanguage protobuf State (sgr_set_state_writer_framing
SGR_VALUE_PROTOBUF_JSON: what a multilanguage store hands its gateway), reported under "protobuf_json" beside the JSON arms,
and a CPU restatement: the same csrc/state_writer.h compiled for the host (g++ -O3, one thread per core) writing the values
of the rows get_many returned. This is NOT the JVM's writeState: it says what the same code costs on the host's cores.
Reported per call: rows/s, value bytes/s, pages, with the card's name and power limit. The host build goes to a temporary
directory; nothing is written into the tree.

    python scripts/state_values_bench.py [--rows 10000000] [--json out.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time
import uuid

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from surge_b200 import native as N  # noqa: E402
from surge_b200 import programs as P  # noqa: E402
from surge_b200.engine import ReplayEngine  # noqa: E402

HOST_SRC = r'''
#include <stdint.h>
#include <string.h>
#include <thread>
#include <vector>
#include "state_writer.h"
using namespace sgr;
// members: n x {kind, off, len}, names NUL-separated; rows n_rows x user; ids with u32 offsets (or null); out: value bytes
extern "C" uint64_t sw_host_write(const uint32_t* m3, const char* names, uint32_t nm, const uint8_t* rows, uint32_t user, uint64_t n_rows,
                                  const uint8_t* ids, const uint32_t* id_offs, uint8_t* out, uint64_t out_cap, int threads) {
  std::vector<sw::Member> mem(nm);
  std::vector<uint8_t> lits;
  for (uint32_t i = 0; i < nm; ++i) {
    const size_t nl = strlen(names);
    sw::Member& m = mem[i];
    m.kind = (uint8_t)m3[3 * i]; m.off = (uint16_t)m3[3 * i + 1]; m.len = m3[3 * i + 2];
    m.lit_off = (uint32_t)lits.size();
    lits.push_back(i ? ',' : '{');
    const size_t at = lits.size();
    lits.resize(at + sw::str_len((const uint8_t*)names, nl));
    sw::str_write(lits.data() + at, (const uint8_t*)names, nl);
    lits.push_back(':');
    m.lit_len = (uint32_t)(lits.size() - m.lit_off);
    names += nl + 1;
  }
  std::vector<uint64_t> total(threads, 0);
  std::vector<std::thread> pool;
  const uint64_t per = (n_rows + threads - 1) / threads, slice = out_cap / threads;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&, t] {
      uint8_t* o = out + t * slice;
      uint8_t* end = o + slice;
      for (uint64_t r = t * per; r < n_rows && r < (t + 1) * per; ++r) {
        const uint8_t* row = rows + r * user;
        const uint8_t* id = ids ? ids + id_offs[r] : nullptr;
        const uint64_t il = ids ? id_offs[r + 1] - id_offs[r] : 0;
        uint64_t len = 1; uint32_t why = 0;
        for (uint32_t k = 0; k < nm && !why; ++k) len += sw::member_len(mem[k], row, id, il, ids != nullptr, &why);
        if (why || (uint64_t)(end - o) < len) continue;
        for (uint32_t k = 0; k < nm; ++k) o = sw::member_write(o, mem[k], lits.data(), row, id, il);
        *o++ = '}';
        total[t] += len;
      }
    });
  for (auto& th : pool) th.join();
  uint64_t s = 0;
  for (uint64_t v : total) s += v;
  return s;
}
'''


def host_writer(tmp):
    src = os.path.join(tmp, "sw_host.cpp")
    lib = os.path.join(tmp, "libsw_host.so")
    with open(src, "w") as f:
        f.write(HOST_SRC)
    subprocess.run(["g++", "-O3", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "surge_b200", "csrc"), src, "-o", lib, "-lpthread"], check=True)
    h = C.CDLL(lib)
    h.sw_host_write.restype = C.c_uint64
    h.sw_host_write.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_uint64, C.c_int]
    return h


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def model(name, n, rng):
    if name == "counter":
        prog = P.counter_program()
        members = [("aggregateId", N.JSON_ID), ("count", N.JSON_I32, 0), ("version", N.JSON_I32, 4)]
        rows = rng.integers(-1000, 1000, size=(n, 8), dtype=np.int32).astype(np.int32).view(np.uint8)[:, :8].copy()
    else:
        prog = P.make_program(64, N.REC_FIXED64, [(N.CREATE, [(N.OP_SET, 0, 16, 4)]), (N.TOMBSTONE, [])], f64_fields=[40])
        members = [("accountNumber", N.JSON_UUID, 0), ("accountOwner", N.JSON_PSTR, 16, 16), ("securityCode", N.JSON_PSTR, 32, 8), ("balance", N.JSON_F64, 40)]
        rows = np.zeros((n, 56), np.uint8)
        rows[:, :16] = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
        rows[:, 16] = 8
        rows[:, 17:25] = np.frombuffer(b"Jane Doe", np.uint8)
        rows[:, 32] = 4
        rows[:, 33:37] = np.frombuffer(b"1234", np.uint8)
        rows[:, 40:48] = (rng.random(n) * 1e6).round(2).view(np.uint8).reshape(n, 8)
    return prog, members, rows


def run(name, n, host, threads):
    rng = np.random.default_rng(1)
    prog, members, rows = model(name, n, rng)
    ids = [str(uuid.UUID(bytes=rng.bytes(16))) for _ in range(n)]
    out = {"model": name, "rows": n}
    with ReplayEngine(0) as e:
        e.register_program(prog)
        e.put_batch(ids, rows)
        e.set_state_writer(members)
        e.get_many_values(ids[:1000])   # warm: index, scratch, pinned staging
        e.get_many(ids[:1000], arrays=True)
        batch = 100_000
        t_rows, _ = timed(lambda: [e.get_many(ids[i:i + batch], arrays=True) for i in range(0, min(n, 100 * batch), batch)])
        t_vals, vals = timed(lambda: [e.get_many_values(ids[i:i + batch]) for i in range(0, min(n, 100 * batch), batch)])
        nb = min(n, 100 * batch)
        vbytes = sum(len(v) for page in vals for v in page if v)
        out["get_100k"] = {"rows_per_s": nb / t_vals, "value_bytes_per_s": vbytes / t_vals, "twin_rows_per_s": nb / t_rows}
        t_rows, got = timed(lambda: e.get_many(ids, arrays=True))
        t_vals, vals = timed(lambda: e.get_many_values(ids))
        vbytes = sum(len(v) for v in vals if v)
        out["get_all"] = {"rows_per_s": n / t_vals, "value_bytes_per_s": vbytes / t_vals, "twin_rows_per_s": n / t_rows}
        for what, vf, rf in (("export", lambda: list(e.export_changes_values(N.ST_CHANGED, max_rows=1 << 20, values_cap=256 << 20)),
                              lambda: list(e.export_changes(N.ST_CHANGED, page_rows=1 << 20))),
                             ("scan", lambda: list(e.scan_values(max_rows=1 << 20, values_cap=256 << 20)), lambda: list(e.scan(page_rows=1 << 20)))):
            t_rows, _ = timed(rf)
            t_vals, pages = timed(vf)
            vb = sum(len(v) for p in pages for v in p[-1] if v)
            out[what] = {"rows_per_s": n / t_vals, "value_bytes_per_s": vb / t_vals, "pages": len(pages), "twin_rows_per_s": n / t_rows}
        # the same reads under the protobuf wrapping (one length pass and one write pass, as the JSON arms)
        e.set_state_writer_framing(N.VALUE_PROTOBUF_JSON)
        e.get_many_values(ids[:1000])
        pb = {}
        t_vals, pvals = timed(lambda: [e.get_many_values(ids[i:i + batch]) for i in range(0, nb, batch)])
        pb["get_100k"] = {"rows_per_s": nb / t_vals, "value_bytes_per_s": sum(len(v) for page in pvals for v in page if v) / t_vals}
        t_vals, pvals = timed(lambda: e.get_many_values(ids))
        pb["get_all"] = {"rows_per_s": n / t_vals, "value_bytes_per_s": sum(len(v) for v in pvals if v) / t_vals}
        for what, vf in (("export", lambda: list(e.export_changes_values(N.ST_CHANGED, max_rows=1 << 20, values_cap=256 << 20))),
                         ("scan", lambda: list(e.scan_values(max_rows=1 << 20, values_cap=256 << 20)))):
            t_vals, pages = timed(vf)
            pb[what] = {"rows_per_s": n / t_vals, "value_bytes_per_s": sum(len(v) for p in pages for v in p[-1] if v) / t_vals, "pages": len(pages)}
        out["protobuf_json"] = pb
        e.set_state_writer_framing(N.VALUE_JSON)
        # CPU restatement over the rows get_many returned
        states = np.ascontiguousarray(got[0])
        m3 = np.array([[m[1], m[2] if len(m) > 2 else 0, m[3] if len(m) > 3 else 0] for m in members], np.uint32)
        names = b"".join(m[0].encode() + b"\0" for m in members)
        enc = [k.encode() for k in ids]
        offs = np.zeros(n + 1, np.uint32)
        np.cumsum([len(b) for b in enc], out=offs[1:])
        blob = np.frombuffer(b"".join(enc), np.uint8)
        has_id = any(m[1] == N.JSON_ID for m in members)
        buf = np.empty(vbytes + 64 * threads * 1024 + (1 << 20), np.uint8)
        t_host, hb = timed(lambda: host.sw_host_write(m3.ctypes.data, names, len(members), states.ctypes.data, states.shape[1], n,
                                                     blob.ctypes.data if has_id else None, offs.ctypes.data if has_id else None, buf.ctypes.data,
                                                     buf.size, threads))
        out["cpu_restatement"] = {"rows_per_s": n / t_host, "value_bytes_per_s": hb / t_host, "threads": threads}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    name = torch.cuda.get_device_name(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    threads = os.cpu_count() or 1
    with tempfile.TemporaryDirectory() as tmp:
        host = host_writer(tmp)
        res = {"gpu": name, "power_limit": q, "results": [run(m, a.rows, host, threads) for m in ("counter", "bank_account")]}
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
