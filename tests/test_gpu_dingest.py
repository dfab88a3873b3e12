"""-m gpu: the device record-batch decode (csrc/dingest_kernels.cu) against the host decoder (csrc/ingest.cpp) and the oracle:
the same wire bytes must give the same states per aggregate id, the same offsets for the lag gate and the same statistics."""
import struct

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import oracle as O
from surge_b200 import ReplayEngine
from surge_b200 import native as N
from surge_b200 import programs as P
from surge_b200.dingest import DeviceIngest
from surge_b200.ingest import Ingest, IngestError

pytestmark = pytest.mark.gpu


def _ev(t, seq, by=0, extra=b""):
    return struct.pack("<IIi", t, seq, by) + extra


def _stream(rng, n_batches, n_keys, compression, base=0, max_per_batch=60):
    out, off = bytearray(), base
    for _ in range(n_batches):
        n = int(rng.integers(1, max_per_batch))
        recs = []
        for d in range(n):
            k = int(rng.integers(0, n_keys))
            key = f"agg-{k}:{off + d}".encode() if rng.random() < 0.7 else f"agg-{k}".encode()
            recs.append((d, key, _ev(int(rng.integers(0, 3)), off + d, int(rng.integers(-2**31, 2**31)), bytes(int(rng.integers(0, 45))))))
        out += K.encode_record_batch(off, recs, compression=compression, headers=[(b"aggregate_id", b"x"), (b"n", None)])
        off += n
    return bytes(out), off


def _states_by_id(engine, keys):
    st = engine.export_states()
    return {k: st[i].tobytes() for i, k in enumerate(keys)}


def _host_fold(fetches, aborted=None):
    ing = Ingest()
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        for part, data in fetches:
            if aborted and part in aborted:
                ing.set_aborted(part, aborted[part])
            ing.record_batches(part, data)
        e.fold_ingested(ing)
        keys = ing.keys()
        return {k: e.get(k) for k in keys}, {p: ing.offsets(p) for p, _ in fetches}, ing


def _device_fold(fetches, aborted=None, max_keys=1 << 16):
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, max_keys) as dg:
            stats = []
            for part, data in fetches:
                if aborted and part in aborted:
                    dg.set_aborted(part, aborted[part])
                stats.append(dg.submit(part, data))
            total = dg.fold()
            offs = {p: dg.offsets(p) for p, _ in fetches}
            return e, dg, total, offs, stats


@pytest.mark.parametrize("compression", ["none", "lz4"])
def test_device_decode_matches_the_host_decoder(compression):
    rng = np.random.default_rng(11)
    fetches = []
    for part in range(4):
        data, _ = _stream(rng, 25, 200, compression, base=part * 1000)
        fetches.append((part, data))
    want, want_offs, host = _host_fold(fetches)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 4096) as dg:
            for part, data in fetches:
                dg.submit(part, data)
            st = dg.fold()
            assert st["n_records"] == len(host.pending()) or st["n_records"] > 0
            for k, v in want.items():
                assert e.get(k) == v, k
            assert e.get("agg-nope") is None
            assert {p: dg.offsets(p) for p, _ in fetches} == want_offs
            assert st["n_new_keys"] == len(want)
            # a second poll onto the live table, with duplicates of the tail of the first one
            more = [(p, _stream(rng, 5, 300, compression, base=want_offs[p][0])[0]) for p, _ in fetches]
            for part, data in more:
                dg.submit(part, data)
            dg.fold()
            hw = Ingest()
            with ReplayEngine(0) as e2:
                e2.register_program(P.counter_program())
                for part, data in fetches + more:
                    hw.record_batches(part, data)
                e2.fold_ingested(hw)
                for k in hw.keys():
                    assert e.get(k) == e2.get(k), k


def test_read_committed_markers_null_values_and_duplicates():
    p0 = K.encode_record_batch(0, [(0, b"", b"")]) + K.encode_record_batch(1, [(0, b"a:1", _ev(0, 1, 1)), (1, b"a:2", _ev(0, 2, 1))], compression="lz4",
                                                                          producer_id=5, transactional=True) + K.encode_control_batch(3, 5, K.COMMIT)
    p1 = K.encode_record_batch(10, [(0, b"b:1", _ev(0, 1, 9))], producer_id=6, transactional=True) + K.encode_control_batch(11, 6, K.ABORT) + \
        K.encode_record_batch(12, [(0, b"c:1", _ev(2, 1, 0)), (1, b"d:1", None)])
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 64) as dg:
            s0 = dg.submit(0, p0)
            assert (s0["n_batches"], s0["n_control_batches"]) == (3, 1)
            dg.set_aborted(1, [(6, 10)])
            s1 = dg.submit(1, p1 + b"\x00" * 7)     # a trailing partial batch is left for the next fetch
            assert s1["n_aborted_batches"] == 1 and s1["n_trailing_bytes"] == 7
            assert dg.offsets(0) == (0, 0)          # submitted, not folded: the gate stays shut
            st = dg.fold()
            assert (st["n_records"], st["n_markers"], st["n_null_values"]) == (3, 1, 1)
            assert dg.offsets(0) == (4, 4) and dg.offsets(1) == (14, 14)
            assert np.frombuffer(e.get("a"), dtype="<i4").tolist() == [2, 2]
            assert e.get("b") is None and e.get("d") is None
            assert np.frombuffer(e.get("c"), dtype="<i4").tolist() == [0, 0]
            # refetch from offset 1: everything below the position is a duplicate
            dg.submit(0, p0[len(K.encode_record_batch(0, [(0, b"", b"")])):] + K.encode_record_batch(4, [(0, b"a:3", _ev(1, 3, 1))]))
            st = dg.fold()
            assert st["n_records"] == 1 and st["n_duplicates"] == 2
            assert np.frombuffer(e.get("a"), dtype="<i4").tolist() == [1, 3]


def test_corruption_fails_the_poll_and_applies_nothing():
    rng = np.random.default_rng(3)
    good, nxt = _stream(rng, 6, 40, "lz4")
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1024) as dg:
            dg.submit(0, good)
            dg.fold()
            before = {k: e.get(k) for k in [f"agg-{i}" for i in range(40)]}
            more, _ = _stream(rng, 4, 40, "lz4", base=nxt)
            for flip in (len(more) // 2, 70, len(more) - 3):
                bad = bytearray(more)
                bad[flip] ^= 0x20
                with pytest.raises(IngestError) as ei:
                    dg.submit(0, bytes(bad))
                    dg.fold()
                assert ei.value.code == N.SGR_ERR_INVALID
                assert dg.offsets(0) == (nxt, nxt)
                assert {k: e.get(k) for k in before} == before
            dg.submit(0, more)
            assert dg.fold()["n_records"] > 0


def test_dictionary_overflow_is_reported():
    rng = np.random.default_rng(4)
    data, _ = _stream(rng, 10, 500, "none")
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 16) as dg:
            dg.submit(0, data)
            with pytest.raises(IngestError) as ei:
                dg.fold()
            assert ei.value.code == N.SGR_ERR_CAPACITY


def test_large_log_from_the_fast_encoder_matches_the_oracle():
    """200 k aggregates x 8 events through 8 partitions of lz4 batches: device decode + fold vs the CPU oracle on the same events."""
    from surge_b200 import synth as S

    n_agg, epa = 200_000, 8
    rec, off = S.counter_csr(n_agg, epa, seed=21)
    want, _, _ = O.fold_packed(O.MODEL_COUNTER, O.REC_FIXED64, rec, off, threads=8)
    part = (rec["agg"] % 8).astype(np.int64)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, 1 << 18) as dg:
            for p in range(8):
                sel = rec[part == p]
                wire = O.kafka_encode_counter(sel["agg"].astype(np.uint32), sel["type"], sel["seq"], sel["arg0"], recs_per_batch=500, lz4=True)
                dg.submit(p, wire)
            st = dg.fold()
            assert st["n_records"] == n_agg * epa and st["n_new_keys"] == n_agg
            for g in list(range(0, n_agg, 997)) + [n_agg - 1]:
                assert e.get(f"agg-{g}") == want[g, :8].tobytes(), g


def _compare_with_host(fetches, max_keys=1 << 14):
    want, want_offs, host = _host_fold(fetches)
    with ReplayEngine(0) as e:
        e.register_program(P.counter_program())
        with DeviceIngest(e, max_keys) as dg:
            for part, data in fetches:
                dg.submit(part, data)
            st = dg.fold()
            for k, v in want.items():
                assert e.get(k) == v, k
            assert {p: dg.offsets(p) for p, _ in fetches} == want_offs
            assert st["n_new_keys"] == len(want)
            return st, dg.last_timing()


@pytest.mark.parametrize("compression", ["none", "lz4"])
def test_small_groups_chain_on_several_streams(monkeypatch, compression):
    """SGR_DINGEST_GROUP=64: a poll of ~600 batches becomes ~10 chains (descriptors, CRC + arena claim, decode, parse) spread over
    the group streams while later fetches are still being copied; buffers grow between groups and must keep their content."""
    monkeypatch.setenv("SGR_DINGEST_GROUP", "64")
    rng = np.random.default_rng(31)
    fetches = []
    for part in range(6):
        data, _ = _stream(rng, 100, 3000, compression, base=part * 100000, max_per_batch=40)
        fetches.append((part, data))
    st, _ = _compare_with_host(fetches)
    assert st["n_batches"] == 600


def test_arena_overflow_falls_back_to_an_exact_layout():
    """Batches that compress far better than the 3x the arena is sized for: the device-side claims overflow, the poll is decoded
    again from a host-side layout and the result is the same."""
    protos = [K.encode_record_batch(0, [(d, b"agg-%d" % ((i + d) % 5), _ev(0, d, 1 + i, b"\x00" * 40)) for d in range(400)], compression="lz4") for i in range(4)]
    parts = []
    for i in range(320):   # baseOffset sits in front of the CRC'd region: the same batch bytes serve at any offset
        parts.append(struct.pack(">q", 400 * i) + protos[i % 4][8:])
    one = b"".join(parts)
    fetches = [(0, one)]
    st, _ = _compare_with_host(fetches)
    assert st["n_decompressed_bytes"] > 3.2 * len(one), (st["n_decompressed_bytes"], len(one))


def test_forty_byte_records_walk_through_the_ring():
    """Records of ~38 bytes make the record walk advance its input ring by three 16-byte chunks per record, every record, in every
    lane — the access pattern that exposed two asynchronous copies aimed at one ring slot (csrc/dingest_kernels.cu, RingIn::advance).
    Several polls of 600 batches x 512 records against the host decoder."""
    rng = np.random.default_rng(77)
    n = 512 * 600
    for rep in range(3):
        agg = rng.integers(0, 150_000, size=n).astype(np.uint32)
        wire = O.kafka_encode_counter(agg, rng.integers(0, 3, size=n).astype(np.uint32), (np.arange(n, dtype=np.uint32) + 3_000_000 * (rep + 1)),
                                      rng.integers(0, 1 << 31, size=n).astype(np.int32), recs_per_batch=512, lz4=True).tobytes()
        want, want_offs, _ = _host_fold([(0, wire)])
        with ReplayEngine(0) as e:
            e.register_program(P.counter_program())
            with DeviceIngest(e, 1 << 18) as dg:
                dg.submit(0, wire)
                st = dg.fold()
                assert st["n_records"] == n and st["n_new_keys"] == len(want)
                keys = list(want)
                for k in keys[::37] + keys[-5:]:
                    assert e.get(k) == want[k], k
                assert dg.offsets(0) == want_offs[0]
