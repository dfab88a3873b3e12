"""CPU checks of the host router for routed reads (surge_b200/dist.py read_routed, merge_scans) over fake ranks, and of the
ctypes prototype of sgr_dist_load_keys against include/sgr.h."""
import ctypes as C
import os
import re

import numpy as np

from surge_b200 import dist as D
from surge_b200 import native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class FakeRank:
    """What a rank with its rank key table answers: its own ids (partition % R == rank) from a dict, in local-slot order."""

    state_bytes = 16

    def __init__(self, table, rank, R, num_partitions):
        ids = list(table)
        own = D.partitions_for_keys(ids, num_partitions) % R == rank
        self.ids = [k for k, o in zip(ids, own) if o]
        self.table = {k: table[k] for k in self.ids}
        self.asked = []

    def get_many(self, keys, arrays=False):
        assert arrays
        self.asked += list(keys)
        n = len(keys)
        states, flags, idx = np.zeros((n, 8), np.uint8), np.zeros(n, np.uint32), np.full(n, -1, np.int64)
        for i, k in enumerate(keys):
            if k in self.table:
                idx[i] = self.ids.index(k)
                row = self.table[k]
                if row is not None:
                    states[i] = np.frombuffer(row, np.uint8)
                    flags[i] = N.ST_EXISTS
        return states, flags, idx

    def scan(self, frm=None, to=None, page_rows=1 << 20):
        keys = sorted((k for k, v in self.table.items() if v is not None and (frm is None or k.encode() >= frm.encode())
                       and (to is None or k.encode() <= to.encode())), key=str.encode)
        for p in range(0, len(keys), page_rows):
            page = keys[p:p + page_rows]
            yield (np.array([self.ids.index(k) for k in page], np.int64), np.full(len(page), N.ST_EXISTS, np.uint32),
                   np.array([np.frombuffer(self.table[k], np.uint8) for k in page]).reshape(-1, 8), page)


def make_table(n, seed):
    rng = np.random.default_rng(seed)
    ids = [f"k-{g}" + "é" * (g % 3) + (":x" if g % 5 == 0 else "") for g in range(n)]
    return {k: (None if rng.random() < 0.2 else rng.bytes(8)) for k in ids}


def test_read_routed_sends_each_id_to_its_owner_and_keeps_query_order():
    table = make_table(500, 1)
    for R in (1, 3, 8):
        ranks = [FakeRank(table, r, R, 32) for r in range(R)]
        rng = np.random.default_rng(R)
        q = [list(table)[i] for i in rng.integers(0, len(table), size=300)] + ["nobody", "k-1"]
        assert D.read_routed(ranks, q, 32) == [table.get(k) for k in q]
        for e in ranks:
            e.asked = []
        states, flags, idx = D.read_routed(ranks, q, 32, arrays=True)
        assert [bool(f & N.ST_EXISTS) for f in flags] == [table.get(k) is not None for k in q]
        assert (idx[[i for i, k in enumerate(q) if k not in table]] == -1).all()
        owner = D.partitions_for_keys(q, 32) % R
        for r, e in enumerate(ranks):
            assert e.asked == [k for k, o in zip(q, owner) if o == r]
    assert D.read_routed([FakeRank(table, 0, 1, 32)], [], 32) == []


def test_merge_scans_is_one_bytes_ordered_stream():
    table = make_table(700, 2)
    live = sorted((k for k, v in table.items() if v is not None), key=str.encode)
    for R in (1, 2, 5):
        ranks = [FakeRank(table, r, R, 32) for r in range(R)]
        got = list(D.merge_scans(ranks, page_rows=17))
        assert [k for k, *_ in got] == live
        assert all(row == table[k] and fl == N.ST_EXISTS for k, _, _, fl, row in got)
        assert all(ranks[r].ids[i] == k for k, r, i, _, _ in got)
        frm, to = live[100], live[400]
        assert [k for k, *_ in D.merge_scans(ranks, frm, to, page_rows=9)] == live[100:401]


def test_dist_load_keys_prototype_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sgr.h")).read(), flags=re.S)
    decl = re.search(r"int32_t\s+sgr_dist_load_keys\s*\(([^)]*)\)", src)
    assert decl, "sgr_dist_load_keys is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in decl.group(1).split(",")]
    assert params == ["sgr_engine* e", "const uint8_t* keys", "const uint32_t* key_offsets", "uint64_t n_global"]
    (restype, argtypes), = [(r, a) for n, r, a in N.ABI if n == "sgr_dist_load_keys"]
    assert restype is C.c_int32
    assert argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
