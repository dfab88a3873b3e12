"""The host decoder's id dictionary (ShardedDict in csrc/ingest.cpp) with ids built to collide (oracle/id_hash.py).

ShardedDict keeps the low 32 bits of hash_bytes as a slot's tag and home and the top 6 bits as its shard. Clusters that share
the whole 64-bit hash, and near misses that share only those 38 bits, reach its "same tag, other bytes" branch, both against
admitted ids and against the provisional ids of the call being decoded; the two ids that hash to 0 and 1 sit next to them.
Polls of such ids mixed with random ones, over several partitions and fetches, through record_batches and through
record_batches_mt with 7 threads, must give oracle/kafka_batch.py's pending records and keys in first-seen order.
"""
import struct

import numpy as np
import pytest

from oracle import id_hash as H
from oracle import kafka_batch as K
from surge_b200.ingest import Ingest


def _ids():
    big = H.cluster(1500, b"hc-", seed=1)
    near = [H.near_miss(big[0], seed=s) for s in range(40)]             # one host tag, 41 device tags
    return [b.decode() for b in big + near + H.cluster(64, b"hw-", home_mask=(1 << 20) - 1, seed=2) + H.tag_one_pair(b"h1-", seed=3)
            + H.random_ids(300, seed=4)]


def _rounds(rng, ids, n_rounds=4, n_parts=4):
    nxt = {p: 0 for p in range(n_parts)}
    first = list(rng.permutation(ids))                                  # every id arrives, then ids drawn at random
    rounds = []
    for _ in range(n_rounds):
        fetches = []
        for p in range(n_parts):
            data = bytearray()
            for _ in range(int(rng.integers(2, 8))):
                recs = []
                for d in range(int(rng.integers(1, 120))):
                    k = first.pop() if first and rng.random() < 0.8 else ids[int(rng.integers(0, len(ids)))]
                    recs.append((d, f"{k}:{nxt[p] + d}".encode(), struct.pack("<IIi", int(rng.integers(0, 3)), nxt[p] + d, d)))
                data += K.encode_record_batch(nxt[p], recs, compression="lz4" if rng.random() < 0.5 else "none")
                nxt[p] += len(recs)
            fetches.append((p, bytes(data)))
        rounds.append(fetches)
    return rounds


@pytest.mark.parametrize("threads", [0, 7], ids=["serial", "mt7"])
def test_host_decoder_over_colliding_ids(threads):
    rng = np.random.default_rng(5 + threads)
    ids = _ids()
    ing = Ingest()
    done = []
    for fetches in _rounds(rng, ids):
        if threads:
            ing.record_batches_mt(fetches, threads=threads)
        else:
            for p, data in fetches:
                ing.record_batches(p, data)
        done += [(p, d, []) for p, d in fetches]
        want, want_keys, want_next = K.read_committed_pack(done)
        assert ing.keys() == [k.decode() for k in want_keys]
        assert np.array_equal(ing.pending(), want)
        assert {p: ing.offsets(p)[0] for p, _ in fetches} == {p: want_next[p] for p, _ in fetches}
    assert sorted(ing.keys()) == sorted(ids)
