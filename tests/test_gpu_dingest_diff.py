"""-m gpu: differential tests of the device record-batch decoder (csrc/dingest.cu, csrc/dingest_kernels.cu, csrc/lz4_fast.h) on
input its own encoders never write. The plain restatement (oracle/kafka_batch.py: lz4_frame_decompress, decode_record_batches,
read_committed_pack, then oracle.fold_incremental or surge_model.ktable_restore) says which states, ids and offsets are right;
the host decoder (csrc/ingest.cpp) is the second opinion on statistics, on refusals and wherever the restatement is
deliberately permissive. Every comparison is exact."""
import contextlib
import ctypes as C
import struct

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import oracle as O
from oracle import surge_model as M
from oracle import wire_corpus as W
from surge_b200 import ReplayEngine
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest, IngestError

pytestmark = pytest.mark.gpu

SETTINGS = {"default": {}, "groups_of_64": {"SGR_DINGEST_GROUP": "64"}}


@contextlib.contextmanager
def _device(max_keys=1 << 14, program=None, null_type=None):
    with ReplayEngine(0) as e:
        e.register_program(program or P.counter_program())
        with DeviceIngest(e, max_keys) as dg:
            if null_type is not None:
                dg.set_null_value_type(null_type)
            yield e, dg


def _expected(fetches, aborted=None):
    """Restatement of a sequence of accepted fetches [(partition, bytes)] (aborted: {partition: [(producer id, first offset)]}
    announced with the partition's first fetch): ({id: Counter state bytes or None}, next offsets)."""
    announce = dict(aborted or {})
    recs, keys, nxt = K.read_committed_pack([(p, d, announce.pop(p, [])) for p, d in fetches])
    st = O.fold_incremental(O.MODEL_COUNTER, recs, np.zeros((len(keys), 16), np.uint8))
    flags = st[:, 8:12].copy().view("<u4").ravel()
    return {k.decode(): (st[i, :8].tobytes() if flags[i] & N.ST_EXISTS else None) for i, k in enumerate(keys)}, nxt


def _assert_table(e, want):
    for k, v in want.items():
        assert e.get(k) == v, k


def _add(total, st):
    for k, v in st.items():
        total[k] = total.get(k, 0) + v
    return total


def _host_poll(ing, fetches):
    """The host decoder's statistics for one poll (summed over its fetches)."""
    total = {}
    for p, d in fetches:
        _add(total, ing.record_batches(p, d))
    ing.mark_folded()
    return total


def _same_stats(dev, host, skip=()):
    drop = {"n_trailing_bytes", *skip}
    assert {k: v for k, v in dev.items() if k not in drop} == {k: v for k, v in host.items() if k not in drop}


def _host_ids(ing):
    """Every id of the host dictionary that is valid UTF-8 (engine.get takes a str)."""
    kp, op, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
    assert ing._lib.sgr_ingest_keys(ing.handle, C.byref(kp), C.byref(op), C.byref(n)) == N.SGR_OK
    if not n.value:
        return []
    offs = np.ctypeslib.as_array(C.cast(op, C.POINTER(C.c_uint32)), shape=(n.value + 1,)).copy()
    raw = C.string_at(kp, int(offs[-1])) if offs[-1] else b""
    out = []
    for i in range(n.value):
        try:
            out.append(raw[offs[i]:offs[i + 1]].decode("utf-8"))
        except UnicodeDecodeError:
            pass
    return out


# ----------------------------------------------------------------------------- 1. hostile lz4 against the restatement
def test_hostile_lz4_on_the_device_matches_the_restatement():
    rng = np.random.default_rng(101)
    nxt = {p: p * 1_000_000 for p in range(4)}
    fetches, ing, n_ids = [], Ingest(), 0
    with _device() as (e, dg):
        for poll in range(3):
            this = []
            for p in nxt:
                data, nxt[p] = W.hostile_batches(rng, 20, nxt[p], p_lz4=0.9)
                if (poll + p) % 2:
                    data += K.encode_record_batch(nxt[p], [], last_offset_delta=3, compression="lz4")   # emptied by compaction
                    nxt[p] += 4
                this.append((p, data))
            for p, d in this:
                dg.submit(p, d)
            st = dg.fold()
            n_ids += st["n_new_keys"]
            fetches += this
            want, want_next = _expected(fetches)
            assert want_next == nxt
            _assert_table(e, want)
            assert n_ids == len(want)                 # no id the restatement does not have
            assert e.get("tenant-0042/aggregate-999") is None
            assert {p: dg.offsets(p) for p in nxt} == {p: (n, n) for p, n in nxt.items()}
            _same_stats(st, _host_poll(ing, this))
        assert st["n_decompressed_bytes"] > 0 and st["n_records"] > 500


# ----------------------------------------------------------------------------- 2. ring geometry, one chain per poll and many
def _ring_polls():
    """Records of 7 bytes (null key, null value) up to ~400 bytes (long headers), so the walk advances its input ring by 0, 1,
    2, ... 8 and more 16-byte chunks per record (advance and seek); stored and literal runs past 128 bytes; batch starts at
    every residue mod 16."""
    rng = np.random.default_rng(202)
    polls, nxt = [], {0: 0, 1: 5000}
    for _ in range(2):
        this = []
        for p in nxt:
            data, nxt[p] = W.hostile_batches(rng, 60, nxt[p], max_records=12, p_lz4=0.5, long_headers=True)
            data += K.encode_record_batch(nxt[p], [(d, None, None) for d in range(40)])
            nxt[p] += 40
            short = [(d, b"s%d" % (d % 5), _ev(d % 3, nxt[p] + d, 1)[:8] + bytes(d % 30)) for d in range(40)]   # 16..47 bytes
            data += K.encode_record_batch(nxt[p], short, compression="lz4" if p else "none")
            nxt[p] += 40
            this.append((p, data))
        polls.append(this)
    return polls, nxt


def _sections(fetch):
    """(lz4 frame or None, records section) of every batch of a fetch."""
    out = []
    for s in W.batch_starts(fetch):
        body = fetch[s + 61:s + 12 + struct.unpack_from(">i", fetch, s + 8)[0]]
        lz4 = struct.unpack_from(">h", fetch, s + 21)[0] & 7 == 3
        out.append((body, K.lz4_frame_decompress(body)) if lz4 else (None, body))
    return out


def _record_lengths(section):
    """Wire length of every record of a records section, its length varint included."""
    q, out = 0, []
    while q < len(section):
        ln, body = K.read_varint(section, q)
        out.append(body - q + ln)
        q = body + ln
    return out


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_ring_geometry_gives_the_same_table_under_every_load_path(monkeypatch, setting):
    for k, v in SETTINGS[setting].items():
        monkeypatch.setenv(k, v)
    polls, nxt = _ring_polls()
    assert {s % 16 for poll in polls for _, d in poll for s in W.batch_starts(d)} == set(range(16))
    secs = [s for poll in polls for _, d in poll for s in _sections(d)]
    lens = [n for _, sec in secs for n in _record_lengths(sec)]
    assert min(lens) == 7 and {n // 16 for n in lens} >= set(range(9)) and max(lens) > 300   # 0..8 chunks a record, and seeks
    seqs = [e for f, _ in secs if f for e in W.lz4_frame_sequences(f)]
    assert any(e["lit"] > 128 for e in seqs if not e["stored"]) and any(e["lit"] > 128 for e in seqs if e["stored"])
    ing, fetches = Ingest(), []
    with _device() as (e, dg):
        for this in polls:
            for p, d in this:
                dg.submit(p, d)
            st = dg.fold()
            fetches += this
            _same_stats(st, _host_poll(ing, this))
        want, want_next = _expected(fetches)
        assert want_next == nxt
        _assert_table(e, want)
        assert {p: dg.offsets(p) for p in nxt} == {p: (n, n) for p, n in nxt.items()}


# ----------------------------------------------------------------------------- 3. record-layout edges
def _run_host(polls, null_type=None, aborted=None):
    ing = Ingest()
    if null_type is not None:
        ing.set_null_value_type(null_type)
    for p, a in (aborted or {}).items():
        ing.set_aborted(p, a)
    out = []
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        for fetches in polls:
            try:
                st = {}
                for s in ing.record_batches_mt(fetches, threads=1):
                    _add(st, s)
            except IngestError as ex:
                out.append(("refused", ex.code))
                continue
            e.fold_ingested(ing)
            out.append(("ok", {k: e.get(k) for k in _host_ids(ing)}, {p: ing.offsets(p) for p, _ in fetches}, st))
    return out


def _run_device(polls, ids, null_type=None, aborted=None):
    out = []
    with _device(null_type=null_type) as (e, dg):
        for p, a in (aborted or {}).items():
            dg.set_aborted(p, a)
        for fetches in polls:
            try:
                for p, d in fetches:
                    dg.submit(p, d)
                st = dg.fold()
            except IngestError as ex:
                out.append(("refused", ex.code))
                continue
            out.append(("ok", {k: e.get(k) for k in ids}, {p: dg.offsets(p) for p, _ in fetches}, st))
    return out


def _ev(t, s, by=1, extra=b""):
    return struct.pack("<IIi", t, s, by) + extra


def _section(*recs):
    return b"".join(W.record(*r) for r in recs)


def _edge_cases():
    b = K.encode_record_batch
    rs = [(d, b"r:%d" % d, _ev(d % 3, d, d)) for d in range(6)]
    ts = _section((0, b"t:0", _ev(0, 0, 3), (), -2**63), (1, b"t:1", _ev(0, 1, 4), (), -5), (2, b"t:2", _ev(1, 2, 1), (), 2**62))
    many = [(b"h%d" % i, None if i % 7 == 0 else bytes([i]) * (i % 5)) for i in range(50)]
    hs = _section((0, b"h:0", _ev(0, 0, 1), ()), (1, b"h:1", _ev(0, 1, 2), [(b"", b"x")]), (2, b"h:2", _ev(0, 2, 3), many),
                  (3, b"h:3", _ev(0, 3, 4), [(b"big", b"\xab" * 300), (b"null", None)]))
    keys = [(0, b":x", _ev(0, 0, 5)), (1, b"nocolon", _ev(0, 1, 6)), (2, b"a:b:c", _ev(0, 2, 7)), (3, b"K" * 1024 + b":1", _ev(0, 3, 8)),
            (4, b"L" * 4096, _ev(0, 4, 9)), (5, "ключ-é✓:1".encode(), _ev(0, 5, 10)), (6, None, _ev(0, 6, 11)), (7, b"", _ev(0, 7, 12)),
            (8, b":x", _ev(1, 8, 1))]
    nulls = [(0, b"n:0", _ev(0, 0, 2)), (1, b"n:1", None), (2, b"m:2", None)]
    # offset gaps: lastOffsetDelta past the last record, an emptied batch, an offset delta of 2^31 - 1
    gaps = b(0, rs[:3], last_offset_delta=9) + b(10, [], last_offset_delta=4, compression="lz4") + \
        b(15, [(0, b"g:0", _ev(0, 0, 1)), (2**31 - 1, b"g:1", _ev(0, 1, 1))])
    first = b"".join(b(o, [(d, b"d:%d" % (o + d), _ev(0, o + d, 1)) for d in range(5)], compression="lz4") for o in (0, 5, 10, 15))
    refetch = b"".join(b(o, [(d, b"d:%d" % (o + d), _ev(0, o + d, 1)) for d in range(5)], compression="lz4") for o in (10, 15, 20))
    part = b(0, rs[:4]) + b(4, rs[:2])[:-3]    # a trailing partial batch: left for the next fetch
    # regressions: inputs on which the device and the host decoder once disagreed
    good = b(0, rs[:4])
    short = bytearray(good)
    struct.pack_into(">i", short, 57, 5)                 # recordsCount 5 over 4 records
    huge = bytearray(b(0, rs[:4], compression="lz4"))
    struct.pack_into(">i", huge, 57, 2**31 - 1)
    ctl_snappy = bytearray(K.encode_control_batch(5, 3, K.ABORT))
    ctl_snappy[22] |= 2
    txn = lambda o, n: b(o, [(d, b"x:%d" % (o + d), _ev(0, o + d, 1)) for d in range(n)], producer_id=7, producer_epoch=0, transactional=True)  # noqa: E731
    abort_lz4 = b(2, [(0, struct.pack(">hh", 0, K.ABORT), struct.pack(">hi", 0, 0))], producer_id=7, producer_epoch=0, transactional=True,
                  control=True, compression="lz4")
    body = b"\x00" + K.varlong(0) + K.varint(0) + K.varint(3) + b"t:1" + K.varint(12) + _ev(0, 1, 1) + K.varint(0) + b"\xee"
    tail_in_record = K.varint(len(body)) + body          # a byte after the headers, inside the record's length
    two = _section((0, b"s:0", _ev(0, 0, 1)), (1, b"s:1", _ev(0, 1, 1)))
    blank = [(d, b"", b"") for d in range(4)]      # (recordsCount and lastOffsetDelta of a caller-built records section)
    # batches of an aborted transaction (producer 7 from offset 0): CRC-checked, then skipped unread
    txn_lz4 = lambda o, n, **kw: b(o, [(d, b"x:%d" % (o + d), _ev(0, o + d, 1)) for d in range(n)], producer_id=7, producer_epoch=0,  # noqa: E731
                                   transactional=True, compression="lz4", **kw)
    damaged_aborted = bytearray(txn(0, 2))
    damaged_aborted[-1] ^= 1
    after_abort = K.encode_control_batch(2, 7, K.ABORT) + b(3, [(0, b"y:3", _ev(0, 3, 1))])
    return {
        # name: (polls, null value type, expected refusal code or None)
        "value_8_and_56_bytes": ([[(0, b(0, [(0, b"v:8", _ev(0, 1)[:8]), (1, b"v:56", _ev(0, 2, 7, bytes(range(44))))]))]], None, None),
        "value_7_bytes": ([[(0, b(0, [(0, b"v:7", _ev(0, 1)[:7])]))]], None, N.SGR_ERR_INVALID),
        "value_57_bytes": ([[(0, b(0, [(0, b"v:57", _ev(0, 1, 1, bytes(45)))], compression="lz4"))]], None, N.SGR_ERR_INVALID),
        "keys": ([[(0, b(0, keys)), (1, b(0, keys, compression="lz4"))]], None, None),
        "null_values_dropped": ([[(0, b(0, nulls, compression="lz4"))]], None, None),
        "null_values_as_tombstones": ([[(0, b(0, nulls, compression="lz4"))]], 2, None),
        "timestamp_deltas": ([[(0, b(0, blank[:3], records_section=ts)), (1, b(0, blank[:3], records_section=ts, compression="lz4"))]], None, None),
        "headers": ([[(0, b(0, blank[:4], records_section=hs)), (1, b(0, blank[:4], records_section=hs, compression="lz4"))]], None, None),
        "offset_gaps_and_empty_batches": ([[(0, gaps)], [(0, b(2**31 + 15, [(0, b"g:2", _ev(0, 2, 1))]))]], None, None),
        "refetch_overlapping_the_folded_range": ([[(0, first)], [(0, refetch)]], None, None),
        "partial_trailing_batch": ([[(0, part)]], None, None),
        "gzip": ([[(0, b(0, rs, compression="gzip"))]], None, N.SGR_ERR_UNSUPPORTED),
        "snappy": ([[(0, b(0, rs, compression="snappy"))]], None, N.SGR_ERR_UNSUPPORTED),
        "zstd": ([[(0, b(0, rs, compression="zstd"))]], None, N.SGR_ERR_UNSUPPORTED),
        "magic_v1": ([[(0, b(0, rs, magic=1))]], None, N.SGR_ERR_UNSUPPORTED),
        "byte_after_a_records_headers": ([[(0, b(0, blank[:1], records_section=tail_in_record, compression="lz4"))]], None, N.SGR_ERR_INVALID),
        "stray_bytes_after_the_last_record": ([[(0, b(0, blank[:2], records_section=two + b"\x00\x00"))]], None, N.SGR_ERR_INVALID),
        "refetch_of_a_damaged_batch": ([[(0, good)], [(0, W.reseal(short))]], None, N.SGR_ERR_INVALID),
        "records_count_past_what_the_batch_holds": ([[(0, W.reseal(huge))]], None, N.SGR_ERR_INVALID),
        "control_batch_with_an_unsupported_codec": ([[(0, W.reseal(ctl_snappy))]], None, N.SGR_ERR_UNSUPPORTED),
        "lz4_abort_marker_ends_the_transaction": ([[(0, txn(0, 2) + abort_lz4 + txn(3, 2))]], None, None, {0: [(7, 0)]}),
        "aborted_batch_with_a_damaged_crc": ([[(0, bytes(damaged_aborted) + after_abort)]], None, N.SGR_ERR_INVALID, {0: [(7, 0)]}),
        "aborted_lz4_batch_is_skipped_unread": ([[(0, txn_lz4(0, 2, headers=[(b"h", b"v" * 40)]) + after_abort)]], None, None, {0: [(7, 0)]}),
        "aborted_batch_with_an_unsupported_codec": ([[(0, b(0, rs[:2], producer_id=7, producer_epoch=0, transactional=True, compression="zstd") +
                                                      after_abort)]], None, None, {0: [(7, 0)]}),
    }


# the restatement decompresses every batch, aborted ones included, and knows no codec but lz4: the host decides these alone
HOST_ONLY = {"aborted_batch_with_an_unsupported_codec"}


@pytest.mark.parametrize("name", list(_edge_cases()))
def test_record_layout_edge(name):
    polls, null_type, refusal, *rest = _edge_cases()[name]
    aborted = rest[0] if rest else None
    host = _run_host(polls, null_type, aborted)
    ids = sorted({k for o in host if o[0] == "ok" for k in o[1]})
    dev = _run_device(polls, ids, null_type, aborted)
    for i, (h, d) in enumerate(zip(host, dev)):
        if h[0] == "refused" or d[0] == "refused":
            assert d == h, (i, d, h)
            continue
        assert d[1] == h[1], i
        assert d[2] == h[2], i
        _same_stats(d[3], h[3])
    if refusal is not None:
        assert host[-1] == ("refused", refusal)
    else:
        assert all(o[0] == "ok" for o in host)
        if null_type is None and name not in HOST_ONLY:
            want, nxt = _expected([f for poll in polls for f in poll], aborted)
            assert {k: v for k, v in host[-1][1].items()} == want
            assert {p: o for p, o in host[-1][2].items()} == {p: (n, n) for p, n in nxt.items() if p in host[-1][2]}


def test_several_bad_batches_in_one_fetch_are_refused_by_both():
    """The check order holds per batch (include/sgr.h): a fetch of [lz4 batch with a damaged CRC, zstd batch] is refused by both
    decoders, the host with the CRC of the first batch, the device with the codec its header walk meets in the second."""
    bad = bytearray(K.encode_record_batch(0, [(0, b"a:0", _ev(0, 0, 1))], compression="lz4"))
    bad[-1] ^= 1
    polls = [[(0, K.encode_record_batch(0, [(0, b"z:0", _ev(0, 0, 1))]))],
             [(0, bytes(bad) + K.encode_record_batch(1, [(0, b"b:1", _ev(0, 1, 1))], compression="zstd"))]]
    host = _run_host(polls)
    dev = _run_device(polls, ["z"])
    assert host[1] == ("refused", N.SGR_ERR_INVALID) and dev[1] == ("refused", N.SGR_ERR_UNSUPPORTED)
    assert host[0][0] == dev[0][0] == "ok" and dev[0][1] == host[0][1]


def test_keys_edge_ids():
    """The ids the edge batches intern: the empty id of ":x", whole keys without a colon, the part before the first colon."""
    polls = _edge_cases()["keys"][0]
    with _device() as (e, dg):
        for p, d in polls[0]:
            dg.submit(p, d)
        st = dg.fold()
        assert st["n_new_keys"] == 6 and st["n_markers"] == 4 and st["n_records"] == 14
        assert np.frombuffer(e.get(""), "<i4").tolist() == [2 * (5 - 1), 8]
        assert e.get("a") is not None and e.get("nocolon") is not None and e.get("L" * 4096) is not None and e.get("K" * 1024) is not None
        assert e.get("ключ-é✓") is not None and e.get("a:b") is None


# ----------------------------------------------------------------------------- 4. resealed mutants, device against host
class _Pair:
    """A long-lived host decoder + engine and a long-lived device ingest + engine fed the same polls."""

    def __init__(self):
        self.stack = contextlib.ExitStack()
        self.ing = Ingest()
        self.eh = self.stack.enter_context(ReplayEngine(0))
        self.eh.register_program(P.counter_program())
        self.ed, self.dg = self.stack.enter_context(_device(max_keys=1 << 16))

    def close(self):
        self.stack.close()
        self.ing.close()

    def _hash(self):
        try:
            return self.ed.states_hash()
        except N.InvalidStateStoreException:      # no table yet: nothing was ever folded
            return None

    def poll(self, part, data):
        try:
            st_h = self.ing.record_batches(part, data)
            self.eh.fold_ingested(self.ing)
            host = ("ok", st_h)
        except IngestError as ex:
            host = ("refused", ex.code)
        before = self._hash(), self.dg.offsets(part)
        try:
            self.dg.submit(part, data)
            dev = ("ok", self.dg.fold())
        except IngestError as ex:
            dev = ("refused", ex.code)
            assert (self._hash(), self.dg.offsets(part)) == before     # nothing of a refused poll is applied
        return host, dev


def _mutants(rng):
    cases = [d for kind, d in W.batch_mutants(rng, 1500) if kind == 0]
    hostile, _ = W.hostile_batches(rng, 40, 0, max_records=20)
    starts = W.batch_starts(hostile) + [len(hostile)]
    protos = [hostile[a:z] for a, z in zip(starts, starts[1:])]
    for _ in range(700):
        b = bytearray(protos[int(rng.integers(0, len(protos)))])
        for _ in range(int(rng.integers(1, 4))):
            pos = int(rng.integers(61 if rng.random() < 0.8 else 21, len(b)))
            b[pos] = int(rng.integers(0, 256)) if rng.random() < 0.5 else b[pos] ^ (1 << int(rng.integers(0, 8)))
        cases.append(W.reseal(b))
    return cases


def test_resealed_mutants_are_refused_alike_or_decoded_alike():
    rng = np.random.default_rng(404)
    cases = _mutants(rng)
    pair, disagree, n_ok, n_refused = _Pair(), [], 0, 0
    try:
        for i, data in enumerate(cases):
            part = 0 if i % 4 == 0 else i          # every fourth onto one long-lived partition (duplicates), the rest fresh
            n_ids = len(_host_ids(pair.ing))
            host, dev = pair.poll(part, data)
            if host[0] != dev[0] or (host[0] == "refused" and host[1] != dev[1]):
                disagree.append((i, part, host if host[0] == "refused" else "ok", dev if dev[0] == "refused" else "ok"))
                pair.close()
                pair = _Pair()                   # the two sides no longer share a history: start both again
                continue
            assert pair.dg.offsets(part) == pair.ing.offsets(part), i
            if host[0] == "refused":
                n_refused += 1
                continue
            n_ok += 1
            # (a refused device poll may leave ids in the dictionary that the next good poll reports as new)
            _same_stats(dev[1], host[1], skip=("n_new_keys",))
            ids = _host_ids(pair.ing)
            for k in ids[n_ids:] + ids[:: max(1, len(ids) // 32)]:
                assert pair.ed.get(k) == pair.eh.get(k), (i, k)
        assert not disagree, f"{len(disagree)} of {len(cases)} polls: {disagree[:12]}"
        for k in _host_ids(pair.ing):
            assert pair.ed.get(k) == pair.eh.get(k), k
        assert n_ok > 100 and n_refused > 500, (n_ok, n_refused)
        # the long-lived device ingest still folds a good poll exactly
        good, nxt = W.hostile_batches(rng, 10, 0)
        host, dev = pair.poll(10**6, good)
        assert host[0] == dev[0] == "ok"
        want, _ = _expected([(10**6, good)])
        for k, v in want.items():
            assert pair.ed.get(k) == pair.eh.get(k), k
        assert pair.dg.offsets(10**6) == (nxt, nxt)
    finally:
        pair.close()


# ----------------------------------------------------------------------------- 5. state-topic restore through the device
def test_state_topic_restore_through_the_device():
    """Device twin of test_gpu_parity.test_state_topic_restore_from_raw_record_batches: the compacted STATE topic (a snapshot
    per write, a null value deletes) as hostile lz4 batches, folded with the snapshot-restore program, equals the KTable
    restatement after every poll."""
    rng = np.random.default_rng(612)
    history, off = [], 0
    with _device(program=P.counter_snapshot_restore_program(), null_type=1) as (e, dg):
        for poll in range(4):
            blob = bytearray()
            for b in range(5):
                recs = []
                for d in range(int(rng.integers(50, 300))):
                    key = f"agg-{int(rng.integers(0, 500))}"
                    if rng.random() < 0.1:
                        recs.append((d, key.encode(), None))
                        history.append((key, None))
                    else:
                        c, v = int(rng.integers(-2**31, 2**31)), int(rng.integers(0, 1000))
                        recs.append((d, key.encode(), struct.pack("<IIii", 0, 0, c, v)))
                        history.append((key, (c, v)))
                opts = W.FRAME_OPTIONS[(poll * 5 + b) % len(W.FRAME_OPTIONS)]
                blob += K.encode_record_batch(off, recs, compression="lz4", lz4_frame=lambda body, o=opts: W.hostile_lz4_frame(body, rng, **o))
                off += len(recs)
            dg.submit(0, bytes(blob))
            st = dg.fold()
            assert st["n_null_values"] == sum(1 for _, v in history[-st["n_records"]:] if v is None)
            table = M.ktable_restore(history)
            for key in {k for k, _ in history}:
                got, want = e.get(key), table.get(key)
                assert (got is None) == (want is None), key
                if want is not None:
                    assert tuple(np.frombuffer(got, "<i4").tolist()) == want, key
        assert dg.offsets(0) == (off, off)
