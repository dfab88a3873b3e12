"""-m gpu: the reads of a routed rank (sgr_dist_load_keys). After a routed rebuild each rank holds the aggregates it owns,
partitionForKey(id) % R == rank, in local slots; with its rank key table the batched reads, the changed-state export, the
scan and their JSON-value twins serve those rows by id. Every case is checked against a single engine fed the same log with
fold_unsorted + load_keys, and against the oracle's table (oracle/program_interp.py, oracle/oracle.py, oracle/state_json.py).

Loopback ranks (R engines on cuda:0, one host thread per rank) run the pipelined push path; one rank with fused 0 runs the
group-by path that takes every program; real ranks run under torchrun when the box has the GPUs (scripts/dist_reads_check.py).
"""
import ctypes as C
import os
import subprocess
import sys
import threading
import uuid

import numpy as np
import pytest

from oracle import oracle as O
from oracle import program_corpus as PC
from oracle import program_interp as I
from oracle import state_json as SJ
from surge_b200 import ReplayEngine, SgrError
from surge_b200 import dist as D
from surge_b200 import formats as F
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200 import synth as S
from surge_b200.dingest import DeviceIngest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH_ERR = N.ST_CHANGED | N.ST_ERROR
NUM_PARTITIONS = 32


def _torch():
    import torch

    return torch


def make_ids(n, seed):
    """Distinct ids with a shared prefix and varied length; every fourth one has a ':' (partitionForKey hashes what precedes it)."""
    rng = np.random.default_rng(seed)
    pad = rng.integers(0, 12, size=n)
    tail = rng.integers(0, 6, size=n)
    return [f"acct-{g:x}" + "z" * int(pad[g]) + (":" + "q" * int(tail[g]) if g % 4 == 1 else "") for g in range(n)]


def split_feeds(rng, rec, R):
    """Arrival order (aggregates interleaved, each one's records in log order); every aggregate is fed by one random rank."""
    rec = np.ascontiguousarray(rec).view(np.uint8).reshape(-1, 64)
    aggs = rec[:, 8:16].copy().view(np.uint64).reshape(-1)
    arrival = rec[PC.interleave(rng, aggs)]
    n_agg = int(aggs.max()) + 1 if len(aggs) else 0
    source_of = rng.integers(0, R, size=max(n_agg, 1))
    src = source_of[arrival[:, 8:16].copy().view(np.uint64).reshape(-1).astype(np.int64)]
    return arrival, [arrival[src == r] for r in range(R)]


def Ranks(prog, part, feeds, chunks=4):
    """R loopback ranks on cuda:0 holding `prog`, partition table `part`, feeds[r] in arrival order (global index at +8)."""
    torch = _torch()
    cap = len(feeds) * chunks * max(D.chunk_records(len(f), chunks) for f in feeds) + 1024

    def engine():
        e = ReplayEngine(0)
        e.register_program(prog)
        e.set_option("push_chunks", chunks)
        return e

    return D.LoopbackRanks(engine, part, [torch.from_numpy(np.ascontiguousarray(f).reshape(-1)).to("cuda:0") for f in feeds], cap)


def fold(ranks, fused):
    """Every rank's route_and_fold, which must succeed; returns whether the ordered repeat ran."""
    errors, repeated, _ = ranks.run(fused)
    assert not any(errors), errors
    return repeated


def single_engine(prog, arrival, n_global, ids):
    """The reference: one engine, the whole log, the whole key table."""
    e = ReplayEngine(0)
    e.register_program(prog)
    e.fold_unsorted(np.ascontiguousarray(arrival), n_global)
    e.load_keys(ids)
    return e


def flags_of(table):
    user = table.shape[1] - 8
    return table[:, user:user + 4].copy().view(np.uint32).reshape(-1)


def export_set(e, page_rows, page_id_bytes, local_to_global=None):
    out = {}
    for idx, fl, err, rows, ids in e.export_changes(CH_ERR, page_rows=page_rows, page_id_bytes=page_id_bytes):
        for i, k in enumerate(ids):
            assert k not in out, k
            g = int(idx[i]) if local_to_global is None else int(local_to_global[idx[i]])
            out[k] = (g, rows[i].tobytes(), int(fl[i]), int(err[i]))
    return out


def scan_raw(e, frm, exclusive, to, page_rows=97):
    """sgr_scan paged by hand, so that the first page can take an exclusive lower bound: [(id, index, flags, row)]."""
    user = e.state_bytes - 8
    lo = None if frm is None else frm.encode()
    hi = None if to is None else to.encode()
    hi_buf = None if hi is None else C.create_string_buffer(hi, max(len(hi), 1))
    n, more = C.c_uint64(), C.c_int32()
    got = []
    while True:
        rows = np.empty((page_rows, user), np.uint8)
        flags = np.empty(page_rows, np.uint32)
        idx = np.empty(page_rows, np.int64)
        offs = np.empty(page_rows + 1, np.uint32)
        blob = np.empty(1 << 16, np.uint8)
        lo_buf = None if lo is None else C.create_string_buffer(lo, max(len(lo), 1))
        rc = e._lib.sgr_scan(e._h, lo_buf, 0 if lo is None else len(lo), exclusive, hi_buf, 0 if hi is None else len(hi), page_rows,
                             rows.ctypes.data, flags.ctypes.data, idx.ctypes.data, blob.ctypes.data, blob.size, offs.ctypes.data,
                             C.byref(n), C.byref(more))
        assert rc == 0, (rc, e._lib.sgr_last_error(e._h))
        k = int(n.value)
        raw = blob[:int(offs[k])].tobytes() if k else b""
        for i in range(k):
            got.append((raw[offs[i]:offs[i + 1]].decode(), int(idx[i]), int(flags[i]), rows[i].tobytes()))
        if k:
            lo, exclusive = raw[offs[k - 1]:offs[k]], 1
        if not more.value:
            return got


def check_rank_reads(engines, single, ids, want, rng, what):
    """Every read of every rank against the oracle's table `want` and the single engine."""
    R = len(engines)
    n = len(ids)
    user = want.shape[1] - 8
    owner = D.partitions_for_keys(ids, NUM_PARTITIONS) % np.uint32(R)
    want_fl = flags_of(want)
    gls = [e.dist_local_aggregates().astype(np.int64) for e in engines]
    assert sorted(np.concatenate(gls).tolist()) == list(range(n)), what
    # batched reads: owned ids from the rank's rows, foreign ids unknown
    for r, e in enumerate(engines):
        rows, fl, idx = e.get_many(ids, arrays=True)
        mine = owner == r
        assert (idx[~mine] == -1).all() and (fl[~mine] == 0).all() and not rows[~mine].any(), f"{what}: rank {r} answers a foreign id"
        assert np.array_equal(gls[r][idx[mine]], np.nonzero(mine)[0]), f"{what}: rank {r} indices"
        assert np.array_equal(rows[mine], want[mine, :user]), f"{what}: rank {r} rows"
        assert np.array_equal(fl[mine], want_fl[mine]), f"{what}: rank {r} flags"
    s_rows, s_fl, _ = single.get_many(ids, arrays=True)
    r_rows, r_fl, _ = D.read_routed(engines, ids, NUM_PARTITIONS, arrays=True)
    assert np.array_equal(r_rows, s_rows) and np.array_equal(r_fl, s_fl), f"{what}: read_routed"
    assert D.read_routed(engines, ids[:50], NUM_PARTITIONS) == single.get_many(ids[:50])
    # the changed-state export: the ranks' pages together are the single engine's export, each id on one rank
    s_exp = export_set(single, 1 << 20, 64 << 20)
    for page_rows in (7, 1000):
        union = {}
        for r, e in enumerate(engines):
            part = export_set(e, page_rows, 40, gls[r])      # 40 id bytes: most pages end on the id budget
            assert not set(part) & set(union), f"{what}: an id exported by two ranks"
            union.update(part)
        assert union == s_exp, f"{what}: export with pages of {page_rows}"
    # the scan: each rank its own live ids in Bytes order, merged into the single engine's scan
    live = (want_fl & N.ST_EXISTS) != 0
    pos = {k: g for g, k in enumerate(ids)}
    for r, e in enumerate(engines):
        got = [k for p in e.scan(page_rows=333) for k in p[3]]
        assert got == sorted((ids[g] for g in np.nonzero(live & (owner == r))[0]), key=str.encode), f"{what}: rank {r} scan"
    s_scan = [(k, int(f), st.tobytes()) for idx, fl, rows, kk in single.scan() for k, f, st in zip(kk, fl, rows)]
    assert [(k, f, row) for k, _, _, f, row in D.merge_scans(engines, page_rows=333)] == s_scan, f"{what}: merge_scans"
    # 20 random [from, to] bounds, half of them with an exclusive lower bound, some of them ids no rank holds
    live_keys = sorted((ids[g].encode() for g in np.nonzero(live)[0]))
    keys = sorted(k.encode() for k in ids)
    for b in range(20):
        a, z = sorted(rng.integers(0, n, size=2).tolist())
        frm = None if b == 0 else keys[a] + (b"" if b % 3 else b"z")
        to = None if b == 1 else keys[z]
        exclusive = b % 2
        want_ids = [k.decode() for k in live_keys if (frm is None or (k > frm if exclusive else k >= frm)) and (to is None or k <= to)]
        frm = None if frm is None else frm.decode()
        to = None if to is None else to.decode()
        per_rank = [scan_raw(e, frm, exclusive, to) for e in engines]
        for r, got in enumerate(per_rank):
            assert [k for k, _, _, _ in got] == [k for k in want_ids if owner[pos[k]] == r], f"{what}: rank {r} bounds {frm!r} {to!r} {exclusive}"
        merged = sorted((x for got in per_rank for x in got), key=lambda x: x[0].encode())
        single_rows = scan_raw(single, frm, exclusive, to)
        assert [k for k, _, _, _ in single_rows] == want_ids
        assert [(k, f, row) for k, _, f, row in merged] == [(k, f, row) for k, _, f, row in single_rows], f"{what}: bounds {frm!r} {to!r}"


# ------------------------------------------------------------------ 1. loopback ranks, sort-free programs
PROGRAMS = ["counter"] + ["-".join(layout) for layout in PC.LAYOUTS]


def sort_free_case(name, throws, n_agg=3000):
    rng = np.random.default_rng(81000 + PROGRAMS.index(name) + 100 * throws)
    if name == "counter":
        counts = rng.integers(0, 30, size=n_agg)
        rec, off = S.counter_csr(n_agg, counts, seed=int(rng.integers(1 << 20)), p_throw=0.002 if throws else 0.0)
        want, _, nerr = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
        return rng, P.counter_program(), np.ascontiguousarray(rec).view(np.uint8).reshape(-1, 64), want, nerr
    layout = tuple(name.split("-"))
    rules, _ = PC.draw_sort_free_program(rng, layout=layout, tombstones=layout == ("set", "set"))
    rec, off, _ = PC.draw_sort_free_log(rng, rules, n_agg, 40_000, 3000, p_throw=0.002 if throws else 0.0)
    want, _, nerr = I.c_fold(rules, 16, rec, off)
    return rng, P.make_program(16, N.REC_FIXED64, rules), rec, want, nerr


@pytest.mark.parametrize("throws", [False, True], ids=["no_throws", "throws"])
@pytest.mark.parametrize("name", PROGRAMS)
def test_loopback_ranks_serve_their_rows_by_id(name, throws):
    rng, prog, rec, want, nerr = sort_free_case(name, throws)
    assert (nerr > 0) == throws
    n_global = len(want)
    ids = make_ids(n_global, 7)
    part = D.partitions_for_keys(ids, NUM_PARTITIONS)
    for R in (2, 3, 8):
        arrival, feeds = split_feeds(rng, rec, R)
        single = single_engine(prog, arrival, n_global, ids)
        try:
            assert np.array_equal(single.export_states(), want)
            with Ranks(prog, part, feeds) as ranks:
                for e in ranks.engines:
                    e.dist_load_keys(ids)
                for fused in (2, 3):
                    assert fold(ranks, fused) == throws
                    check_rank_reads(ranks.engines, single, ids, want, rng, f"{name} R={R} fused={fused}")
        finally:
            single.close()


# ------------------------------------------------------------------ 2. one rank on the group-by path, wider programs, values
COUNTER_JSON = [("aggregateId", SJ.ID), ("count", SJ.I32, 0), ("version", SJ.I32, 4)]
BANK_JSON = [("id", SJ.ID), ("accountNumber", SJ.UUID, 0), ("accountOwner", SJ.PSTR, 24, 16), ("securityCode", SJ.PSTR, 40, 8),
             ("balance", SJ.F64, 16)]
STATE_128B = [(I.CREATE, [(I.OP_SET, 0, 16, 48), (I.OP_SET, 64, 16, 48)]), (I.IF_EXISTS, [(I.OP_ADD_I64, 112, 24, 8)]),
              (I.IF_EXISTS, []), (I.THROW, [])]


def writer_of(members):
    return [(m[0], m[1]) if m[1] == SJ.ID else (m[0], m[1], m[2], m[3] if len(m) > 3 else 0) for m in members]


def bank_log(rng, n_agg):
    blobs = []
    for a in range(n_agg):
        acct = str(uuid.UUID(int=int(rng.integers(1, 2**62))))
        for j in range(int(rng.integers(0, 8))):
            if j == 0 or rng.random() < 0.2:
                blobs.append(F.bank_created_record(a, j + 1, acct, f"owner{a % 97}", f"{a % 10000:04d}", 1000.0 + 0.25 * j))
            else:
                blobs.append(F.bank_updated_record(a, j + 1, acct, [float(j), -0.0, 0.0, 1e300, 12.5][int(rng.integers(0, 5))]))
    return np.frombuffer(b"".join(blobs), dtype=np.uint8).reshape(-1, 64)


def one_rank(prog, part, arrival, fused=0, force_route=False):
    """A routed engine of one rank (dist_init(0, 1)): local index == global index."""
    torch = _torch()
    e = ReplayEngine(0)
    e.register_program(prog)
    if force_route:
        e.set_option("force_route", 1)
        e.set_option("push_chunks", 3)
    e.dist_init(0, 1, None, len(arrival) + 3 * 1024 + 1024)
    e.dist_set_partitions(part)
    feed = torch.from_numpy(np.ascontiguousarray(arrival).reshape(-1).copy()).to("cuda:0")
    e.dist_route_and_fold(feed, fused)
    e._feed = feed
    return e


def check_values(e, single, ids, members):
    """get_many_values, export_changes_values and scan_values of the rank equal the single engine's and the restatement."""
    e.set_state_writer(writer_of(members))
    single.set_state_writer(writer_of(members))
    probe = ids + ["never-seen"]
    got = e.get_many_values(probe)
    assert got == single.get_many_values(probe)
    rows, fl, _ = single.get_many(probe, arrays=True)
    assert got == [SJ.write_value(members, rows[i].tobytes(), k.encode()) if fl[i] & N.ST_EXISTS else None for i, k in enumerate(probe)]
    flat = lambda pages: [(i, k, v) for p in pages for i, k, v in zip(p[0].tolist(), p[3], p[4])]   # noqa: E731
    assert flat(e.export_changes_values(CH_ERR, max_rows=500, values_cap=3000)) == flat(single.export_changes_values(CH_ERR))
    flat_s = lambda pages: [(i, k, v) for p in pages for i, k, v in zip(p[0].tolist(), p[2], p[3])]   # noqa: E731
    assert flat_s(e.scan_values(max_rows=300, values_cap=2000)) == flat_s(single.scan_values())


def check_one_rank_reads(e, single, ids, want, what):
    user = want.shape[1] - 8
    assert np.array_equal(e.export_states(), want), what
    assert np.array_equal(e.dist_local_aggregates(), np.arange(len(ids))), what
    for k, got in zip(ids[:200], [e.get(k) for k in ids[:200]]):
        assert got == single.get(k), (what, k)
    rows, fl, idx = e.get_many(ids + ["never-seen"], arrays=True)
    s = single.get_many(ids + ["never-seen"], arrays=True)
    assert all(np.array_equal(a, b) for a, b in zip((rows, fl, idx), s)), what
    assert np.array_equal(rows[:-1], want[:, :user]), what
    assert export_set(e, 13, 64) == export_set(single, 1 << 20, 64 << 20), what
    assert [p[3] for p in e.scan(page_rows=77)] == [p[3] for p in single.scan(page_rows=77)], what
    assert scan_raw(e, ids[5], 1, ids[900]) == scan_raw(single, ids[5], 1, ids[900]), what


@pytest.mark.parametrize("name", ["bank", "state_128B", "class1", "counter"])
def test_one_rank_group_by_path_and_state_values(name):
    rng = np.random.default_rng(82000 + len(name))
    n_agg = 3000
    if name == "bank":
        prog, sb = P.bank_account_program(), 64
        rec = bank_log(rng, n_agg)
        counts = np.bincount(rec[:, 8:16].copy().view(np.uint64).reshape(-1).astype(np.int64), minlength=n_agg)
        want, _, _ = O.fold_packed(O.MODEL_BANK_ACCOUNT, O.REC_FIXED64, rec, F.csr_offsets_from_counts(counts))
    elif name == "counter":
        prog, sb = P.counter_program(), 16
        rec, off = S.counter_csr(n_agg, rng.integers(0, 20, size=n_agg), seed=5, p_throw=0.01)
        want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
        rec = np.ascontiguousarray(rec).view(np.uint8).reshape(-1, 64)
    else:
        sb, rules = (128, STATE_128B) if name == "state_128B" else (16, PC.row_program(rng, 2, 1, 3))
        prog = P.make_program(sb, N.REC_FIXED64, rules)
        buf, seg, _ = PC.fixed_log(rng, rules, rng.integers(0, 15, size=n_agg), p_throw=0.003)
        want, _, _ = I.c_fold(rules, sb, buf, seg)
        rec = buf
    ids = [str(uuid.UUID(int=int(x))) for x in rng.integers(1, 2**62, size=n_agg)] if name == "bank" else make_ids(n_agg, 3)
    arrival, _ = split_feeds(rng, rec, 1)
    part = D.partitions_for_keys(ids, NUM_PARTITIONS)
    single = single_engine(prog, arrival, n_agg, ids)
    e = one_rank(prog, part, arrival)
    try:
        assert np.array_equal(single.export_states(), want)
        e.dist_load_keys(ids)
        check_one_rank_reads(e, single, ids, want, name)
        if name == "bank":
            check_values(e, single, ids, BANK_JSON)
        elif name == "counter":
            check_values(e, single, ids, COUNTER_JSON)
        if name == "counter":
            for fused in (2, 3):      # the push path with one destination
                f = one_rank(prog, np.zeros(n_agg, np.uint32), arrival, fused=fused, force_route=True)
                try:
                    f.dist_load_keys(ids)
                    check_one_rank_reads(f, single, ids, want, f"force_route fused {fused}")
                    check_values(f, single, ids, COUNTER_JSON)
                finally:
                    f.close()
    finally:
        e.close()
        single.close()


# ------------------------------------------------------------------ 3. lifecycle and refusals
def raw_load(e, blob, offs, n):
    return e._lib.sgr_dist_load_keys(e._h, blob, offs, n)


def encode(ids):
    enc = [k.encode() for k in ids]
    offs = np.zeros(len(enc) + 1, np.uint32)
    np.cumsum([len(b) for b in enc], out=offs[1:])
    return np.frombuffer(b"".join(enc) or b"\0", np.uint8).copy(), offs


READS = {     # the writer first: the value reads need one
    "set_state_writer": lambda e, ids: e.set_state_writer(writer_of(COUNTER_JSON)),
    "get_many": lambda e, ids: e.get_many(ids, arrays=True),
    "get_many_values": lambda e, ids: e.get_many_values(ids),
    "export_changes": lambda e, ids: list(e.export_changes(CH_ERR)),
    "export_changes_values": lambda e, ids: list(e.export_changes_values(CH_ERR)),
    "scan": lambda e, ids: list(e.scan()),
    "scan_values": lambda e, ids: list(e.scan_values()),
}


def reads(e, ids):
    """Each read once: the code it returns (0 on success)."""
    out = {}
    for name, call in READS.items():
        try:
            call(e, ids)
            out[name] = 0
        except SgrError as ex:
            out[name] = ex.code
    return out


def export_page(e, cur, max_rows=100):
    rows = np.empty((max_rows, 8), np.uint8)
    fl, err = np.empty(max_rows, np.uint32), np.empty(max_rows, np.uint32)
    idx = np.empty(max_rows, np.int64)
    offs = np.empty(max_rows + 1, np.uint32)
    blob = np.empty(1 << 16, np.uint8)
    n = C.c_uint64()
    return e._lib.sgr_export_changes(e._h, CH_ERR, C.byref(cur), max_rows, rows.ctypes.data, fl.ctypes.data, err.ctypes.data, idx.ctypes.data,
                                     blob.ctypes.data, blob.size, offs.ctypes.data, C.byref(n))


def test_lifecycle_and_refusals():
    rng = np.random.default_rng(83000)
    n_agg = 2000
    rec, off = S.counter_csr(n_agg, rng.integers(1, 10, size=n_agg), seed=6)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off)
    arrival, _ = split_feeds(rng, rec, 1)
    ids = make_ids(n_agg, 11)
    part = D.partitions_for_keys(ids, NUM_PARTITIONS)
    blob, offs = encode(ids)
    refused = {k: N.SGR_ERR_UNSUPPORTED for k in READS}
    first3 = [want[g, :8].tobytes() if flags_of(want)[g] & N.ST_EXISTS else None for g in range(3)]
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        assert raw_load(e, blob.ctypes.data, offs.ctypes.data, n_agg) == N.SGR_ERR_NOT_LOADED     # no sgr_dist_init
        e.dist_init(0, 1, None, len(arrival) + 4096)
        assert raw_load(e, blob.ctypes.data, offs.ctypes.data, n_agg) == N.SGR_ERR_NOT_LOADED     # no partition table
    e = one_rank(P.counter_program(), part, arrival)
    try:
        assert reads(e, ids) == refused
        e.dist_load_keys(ids)
        assert set(reads(e, ids).values()) == {0}
        assert e.get_many(ids[:3]) == first3
        # refused loads leave the key table as it was
        bad = offs.copy()
        bad[7] = bad[8] + 1
        for args in [(blob.ctypes.data, offs.ctypes.data, n_agg - 1), (blob.ctypes.data, None, n_agg), (None, offs.ctypes.data, n_agg),
                     (blob.ctypes.data, bad.ctypes.data, n_agg)]:
            assert raw_load(e, *args) == N.SGR_ERR_INVALID, args
            assert e.get_many(ids[:3]) == first3
        # an export page in flight across dist_load_keys, and across a second route_and_fold
        for between in (lambda: e.dist_load_keys(ids), lambda: e.dist_route_and_fold(e._feed, 0)):
            cur = N.sgr_changes_cursor()
            assert export_page(e, cur) == 0 and 0 < cur.next < n_agg
            between()
            assert export_page(e, cur) == N.SGR_ERR_STATE
        assert np.array_equal(e.export_states(), want)
        # still refused with rank keys: writes that number new ids
        with pytest.raises(SgrError) as ex:
            e.put_batch(["new-id"], np.zeros((1, 8), np.uint8))
        assert ex.value.code == N.SGR_ERR_UNSUPPORTED
        with DeviceIngest(e, 1 << 12) as dg:
            with pytest.raises(SgrError) as ex:
                dg.set_state_topic(True)
            assert ex.value.code == N.SGR_ERR_UNSUPPORTED
        # each of these ends the rank key table
        for end in (lambda: e.dist_set_partitions(part), lambda: e.load_keys(ids),
                    lambda: e._lib.sgr_append_keys(e._h, C.c_void_p(0x51), blob.ctypes.data, offs.ctypes.data, 10)):
            e.dist_load_keys(ids)
            assert e.get_many(ids[:1]) == first3[:1]
            end()
            assert reads(e, ids) == refused
        e.dist_load_keys(ids)
        e.dist_init(0, 1, None, len(arrival) + 4096)
        assert reads(e, ids) == refused
        assert e.get(ids[0]) is None          # the host path finds no id either
    finally:
        e.close()
    # duplicate ids: refused when this rank owns both (as sgr_load_keys), unseen when another rank owns them
    dup = ["x", "y", "x", "z", "w", "w"]
    dpart = np.array([0, 1, 1, 0, 1, 1], np.uint32)
    for r in (0, 1):
        with ReplayEngine(0) as d:
            d.register_program(P.counter_program())
            d.dist_init(r, 2, None, 4096)
            d.dist_set_partitions(dpart)
            if r == 1:
                with pytest.raises(SgrError) as ex:
                    d.dist_load_keys(dup)
                assert ex.value.code == N.SGR_ERR_INVALID and "duplicate" in str(ex.value)
                continue
            d.dist_load_keys(dup)
            d.grow_states(2)
            assert d.get_many(["x", "z", "y", "w"], arrays=True)[2].tolist() == [0, 1, -1, -1]


# ------------------------------------------------------------------ 4. scale
def test_four_million_aggregates_on_four_ranks():
    torch = _torch()
    n_global, R = 4 << 20, 4
    rng = np.random.default_rng(84000)
    rec, off = S.counter_csr(n_global, rng.integers(0, 4, size=n_global), seed=12, p_throw=1e-5)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off, threads=8)
    ids = [f"agg-{g}" for g in range(n_global)]
    part = D.partitions_for_keys(ids, NUM_PARTITIONS)
    arrival, feeds = split_feeds(rng, rec, R)
    single = single_engine(P.counter_program(), arrival, n_global, ids)
    del rec, arrival
    low = [torch.cuda.mem_get_info(0)[0]]
    stop = threading.Event()

    def sample():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info(0)[0])
            stop.wait(0.005)

    try:
        with Ranks(P.counter_program(), part, feeds) as ranks:
            fold(ranks, 2)
            th = threading.Thread(target=sample)
            th.start()
            try:
                for e in ranks.engines:
                    e.dist_load_keys(ids)
                for b in range(0, n_global, 1 << 20):
                    q = ids[b:b + (1 << 20)]
                    got = D.read_routed(ranks.engines, q, NUM_PARTITIONS, arrays=True)
                    s = single.get_many(q, arrays=True)
                    assert np.array_equal(got[0], s[0]) and np.array_equal(got[1], s[1]), b
                    assert np.array_equal(got[0], want[b:b + len(q), :8])
                total_export, total_scan = 0, 0
                s_idx = np.concatenate([p[0] for p in single.export_changes(CH_ERR)])
                for e in ranks.engines:
                    gl = e.dist_local_aggregates().astype(np.int64)
                    for idx, fl, _, rows, kk in e.export_changes(CH_ERR):
                        g = gl[idx]
                        assert np.array_equal(rows, want[g, :8]) and kk[0] == ids[g[0]] and kk[-1] == ids[g[-1]]
                        total_export += len(idx)
                    prev = b""
                    for idx, _, rows, kk in e.scan():
                        g = gl[idx]
                        assert np.array_equal(rows, want[g, :8]) and kk[0].encode() > prev
                        prev = kk[-1].encode()
                        total_scan += len(idx)
                assert total_export == len(s_idx)
                assert total_scan == int(((flags_of(want) & N.ST_EXISTS) != 0).sum())
            finally:
                stop.set()
                th.join()
            free, total = torch.cuda.mem_get_info(0)
            print(f"4 M aggregates on 4 loopback ranks: lowest free device memory during the reads {low[0] / 2**30:.2f} GiB "
                  f"of {total / 2**30:.2f} GiB (peak in use {(total - low[0]) / 2**30:.2f} GiB)")
    finally:
        single.close()


# ------------------------------------------------------------------ 5. real ranks
@pytest.mark.parametrize("world", [2, 4, 8])
def test_rank_reads_under_torchrun(world):
    torch = _torch()
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, the box has {torch.cuda.device_count()}")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29711 + world), os.path.join(ROOT, "scripts", "dist_reads_check.py"), "200000"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    lines = [ln for ln in r.stdout.splitlines() if "reads_ok=" in ln]
    assert len(lines) == 2 * world and all("reads_ok=True" in ln for ln in lines), r.stdout[-3000:]   # fused 2 and 0
