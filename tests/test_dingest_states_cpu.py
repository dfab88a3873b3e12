"""No GPU: the restatement of the device ingest's state-topic mode (oracle/state_topic.py), pinned to the events-mode restatement
(oracle/kafka_batch.read_committed_pack) on keys without ':' and to hand-computed cases, and the ABI argument checks of
sgr_dingest_set_state_topic that need no device."""
import random
import struct

import numpy as np
import pytest

from oracle import kafka_batch as K
from oracle import put_batch as PB
from oracle import state_topic as S
from surge_b200 import native as N

EX, CH = PB.EXISTS, PB.CHANGED


def flags(table):
    sb = table.shape[1]
    return table[:, sb - 8:sb - 4].copy().view(np.uint32)[:, 0].tolist()


def random_fetches(seed, n_parts=3, n_batches=12, colon=False):
    """Fetches over several partitions with flush markers, null values, refetched batches and aborted transactions."""
    rng = random.Random(seed)
    fetches = []
    nxt = {p: 0 for p in range(n_parts)}
    sent = {p: [] for p in range(n_parts)}
    for _ in range(n_batches):
        p = rng.randrange(n_parts)
        roll = rng.random()
        if roll < 0.15 and sent[p]:
            fetches.append((p, rng.choice(sent[p]), []))          # a refetch below the position: duplicates
            continue
        recs = []
        for d in range(rng.randrange(1, 9)):
            kind = rng.random()
            if kind < 0.1:
                recs.append((d, b"", b""))                           # the producer's flush marker
                continue
            key = b"id-%d" % rng.randrange(12) + (b":%d" % d if colon else b"")
            val = None if kind < 0.25 else bytes(rng.randrange(256) for _ in range(rng.randrange(8, 57)))
            recs.append((d, key, val))
        comp = rng.choice(["none", "lz4"])
        if roll < 0.3:
            pid = 1000 + len(fetches)
            data = K.encode_record_batch(nxt[p], recs, compression=comp, producer_id=pid, producer_epoch=0, transactional=True)
            ctl = K.encode_control_batch(nxt[p] + len(recs), pid, K.ABORT)
            fetches.append((p, data + ctl, [(pid, nxt[p])]))
            nxt[p] += len(recs) + 1
            continue
        data = K.encode_record_batch(nxt[p], recs, compression=comp)
        sent[p].append(data)
        nxt[p] += len(recs)
        fetches.append((p, data, []))
    return fetches


@pytest.mark.parametrize("seed", range(6))
def test_pinned_to_the_events_restatement_without_colons(seed):
    fetches = random_fetches(seed)
    recs, nxt, st = S.read_committed_states(fetches)
    arr, keys, nxt_ev = K.read_committed_pack(fetches)
    assert nxt == nxt_ev
    live = [(k, v) for k, v in recs if v is not None]
    assert len(live) == len(arr)
    for (k, v), row in zip(live, arr):
        idx = int(row[8:16].view(np.uint64)[0])
        assert keys[idx] == k
        assert row[0:8].tobytes() + row[16:64].tobytes() == v + b"\0" * (56 - len(v))
    assert st["n_records"] == len(recs) and st["n_null_values"] == len(recs) - len(live)
    # the events restatement interns ids in first-seen order of its live records: the same ids as the state records' rows
    assert keys == list(dict.fromkeys(k for k, _ in live))


def test_whole_key_is_the_id_and_tombstones_of_unknown_ids_make_none_rows():
    recs = [(0, b"a:1", b"\1" * 8), (1, b"ghost", None), (2, b"a", b"\2" * 8)]
    fetch = [(0, K.encode_record_batch(0, recs), [])]
    got, nxt, st = S.read_committed_states(fetch)
    assert got == [(b"a:1", b"\1" * 8), (b"ghost", None), (b"a", b"\2" * 8)] and nxt == {0: 3}
    ids, t = S.apply([], np.zeros((0, 16), np.uint8), got)
    assert ids == ["a:1", "ghost", "a"]
    assert flags(t) == [EX | CH, 0, EX | CH] and not t[1, :8].any()


def test_snap_tomb_snap_of_one_id_and_one_id_in_two_partitions():
    f = [(0, K.encode_record_batch(0, [(0, b"x", b"\5" * 4), (1, b"x", None)]), []),
         (1, K.encode_record_batch(0, [(0, b"x", b"\6" * 4)]), []),
         (0, K.encode_record_batch(2, [(0, b"y", b"\7" * 8)]), [])]
    recs, nxt, _ = S.read_committed_states(f)
    assert nxt == {0: 3, 1: 1}
    ids, t = S.apply([], np.zeros((0, 16), np.uint8), recs)
    assert ids == ["x", "y"]
    assert t[0, :8].tobytes() == b"\6" * 4 + b"\0" * 4 and flags(t) == [EX | CH, EX | CH]   # partition 1's write is the last
    # the same id rewritten with its bytes in a later poll: not CHANGED; a poll without live records applies nothing
    ids2, t2 = S.apply(ids, t, [(b"x", b"\5" * 4), (b"x", None), (b"x", b"\6" * 4)])
    assert flags(t2) == [EX, EX]
    ids3, t3 = S.apply(ids2, t2, [])
    assert np.array_equal(t3, t2) and ids3 == ids2


def test_protobuf_state_framing_and_length_refusal():
    v = S.encode_state(b"agg", b"\1\2\3")
    assert S.protobuf_payload(v) == b"\1\2\3"
    assert S.protobuf_payload(b"") == b""
    with pytest.raises(S.Refused):
        S.protobuf_payload(b"\x0a\x05ab")
    f = [(0, K.encode_record_batch(7, [(0, b"k", b"\0" * 8), (1, b"k", b"\0" * 9)]), [])]
    with pytest.raises(S.Refused, match=r"offset 7, record 1: state value of 9 bytes is longer than the 8 program bytes"):
        S.read_committed_states(f, row_bytes=8)
    recs, _, _ = S.read_committed_states([(0, K.encode_record_batch(0, [(0, b"k", S.encode_state(b"k", struct.pack("<q", -5)))]), [])],
                                         framing=S.PROTOBUF, row_bytes=8)
    assert recs == [(b"k", struct.pack("<q", -5))]


def test_markers_duplicates_and_aborted_records_are_counted():
    data = K.encode_record_batch(0, [(0, b"", b""), (1, None, b"x"), (2, b"a", b"\1")])
    pid = 9
    aborted = K.encode_record_batch(3, [(0, b"b", b"\2")], producer_id=pid, producer_epoch=0, transactional=True)
    ctl = K.encode_control_batch(4, pid, K.ABORT)
    recs, nxt, st = S.read_committed_states([(0, data + aborted + ctl, [(pid, 3)]), (0, data, [])])
    assert recs == [(b"a", b"\1")] and nxt == {0: 5}
    assert st["n_markers"] == 2 and st["n_duplicates"] == 3 and st["n_aborted_records"] == 1 and st["n_control_batches"] == 1


def test_set_state_topic_checks_its_handle_before_any_device():
    lib = N.load_library()
    assert lib.sgr_dingest_set_state_topic(None, 1) == N.SGR_ERR_INVALID
    assert lib.sgr_dingest_set_state_topic(None, 0) == N.SGR_ERR_INVALID
