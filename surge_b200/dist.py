"""Host-side plumbing of the multi-GPU replay: one process per GPU, torch.distributed only for the
rendezvous (NCCL unique id, CUDA IPC handles, barriers); the data path is the engine's own
route kernel + NCCL / peer-memory exchange (csrc/dist.cu).

Ownership mirrors the reference: aggregateId -> partition (KafkaPartitionProvider.partitionForKey,
modules/common/src/main/scala/surge/kafka/KafkaPartitioner.scala:7-9) -> owner = partition % nranks.
"""
from __future__ import annotations

import ctypes as C
import heapq
import threading
import time
from typing import Callable, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import native as N
from .engine import _id_batch, _rows_or_none


def partitions_for_keys(keys: Sequence[str], num_partitions: int, up_to_colon: bool = True) -> np.ndarray:
    """partition_of[i] = abs(MurmurHash3.stringHash(keys[i].takeWhile(_ != ':')) % num_partitions)."""
    lib = N.load_library()
    blob, offs = _id_batch([k.encode("utf-8") for k in keys])
    out = np.zeros(len(offs) - 1, dtype=np.uint32)
    rc = lib.sgr_partitions_for_keys(blob.ctypes.data, offs.ctypes.data, len(out), num_partitions, 1 if up_to_colon else 0, out.ctypes.data)
    if rc != 0:
        raise ValueError(f"sgr_partitions_for_keys -> {rc}")
    return out


def owner_and_local_index(partition_of_agg: np.ndarray, nranks: int) -> Tuple[np.ndarray, np.ndarray, List[np.ndarray]]:
    """numpy mirror of the device tables (csrc/dist.cu): owner rank, local dense index on the owner, and per rank
    the global indices of its local slots. Used by the CPU (gloo) tests of the routing logic."""
    owner = (np.asarray(partition_of_agg, dtype=np.uint32) % np.uint32(nranks)).astype(np.uint8)
    local = np.zeros(len(owner), dtype=np.uint32)
    globals_of = []
    for r in range(nranks):
        idx = np.nonzero(owner == r)[0]
        local[idx] = np.arange(len(idx), dtype=np.uint32)
        globals_of.append(idx.astype(np.uint32))
    return owner, local, globals_of


def route_on_host(records: np.ndarray, owner: np.ndarray, local: np.ndarray, nranks: int) -> List[np.ndarray]:
    """Stable partition of REC64 records by owner with the agg field rewritten to the owner's local index:
    what K4 (route_scatter) produces, as numpy. Returns one array per destination rank."""
    agg = records["agg"].astype(np.int64)
    o = owner[agg]
    out = []
    for r in range(nranks):
        sel = records[o == r].copy()           # boolean mask keeps order: stable
        sel["agg"] = local[agg[o == r]]
        out.append(sel)
    return out


def _splitmix64(x: np.ndarray) -> np.ndarray:
    x = (x + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def states_hash(states: np.ndarray, global_ids: Optional[np.ndarray] = None) -> int:
    """numpy twin of sgr_states_hash (csrc/bulk_fold.cu states_hash_kernel): sum over slots of
    mix(id, state bytes) mod 2^64 — order independent, so per-rank hashes of a routed table add up to the hash of the
    whole table under global aggregate indices."""
    st = np.ascontiguousarray(states).view(np.uint8)
    n = st.shape[0]
    if n == 0:
        return 0
    words = st.reshape(n, -1).view(np.uint64)
    ids = np.arange(n, dtype=np.uint64) if global_ids is None else np.asarray(global_ids).astype(np.uint64)
    with np.errstate(over="ignore"):
        h = _splitmix64(ids)
        for k in range(words.shape[1]):
            h = _splitmix64(h ^ words[:, k])
        return int(h.sum(dtype=np.uint64))


def partitions_of_rank(rank: int, nranks: int, num_partitions: int) -> List[int]:
    """Topic partitions a rank consumes when the store is fed from the topic itself (surge_b200/ingest.py): the broker has already
    done the shuffle — every record of an aggregate sits in partition partitionForKey(id) — so rank r decodes and folds the
    partitions p with p % nranks == r and NO exchange between GPUs is needed; the same owner rule as the routed path."""
    return [p for p in range(num_partitions) if p % nranks == rank]


def exchange_ids(engine, rank: int, nranks: int, recv_capacity_records: int, fused: bool = True) -> None:
    """Rendezvous over torch.distributed: NCCL unique id from rank 0, then (fused path) the IPC handles."""
    import torch.distributed as dist

    lib = N.load_library()
    uid = [None]
    if rank == 0 and nranks > 1:
        buf = C.create_string_buffer(128)
        rc = lib.sgr_dist_unique_id(buf)
        if rc != 0:
            raise N.SgrError(rc, (lib.sgr_last_error(None) or b"").decode())
        uid = [bytes(buf.raw)]
    if nranks > 1:
        dist.broadcast_object_list(uid, src=0)
    engine.dist_init(rank, nranks, uid[0], recv_capacity_records)
    if fused and nranks > 1:
        mine = engine.dist_ipc_export()
        handles: List[Optional[bytes]] = [None] * nranks
        dist.all_gather_object(handles, mine)
        engine.dist_ipc_import(handles)


def chunk_records(n: int, chunks: int) -> int:
    """A rank's chunk length on the push path (csrc/route_push.cu chunk_records) for a log of n records cut into `chunks`
    chunks: whole multiples of 1024 records."""
    c = -(-n // chunks)
    return -(-c // 1024) * 1024


class LoopbackRanks:
    """The ranks of one routed job inside this process, every one an engine on the same device (sgr_dist_init without a unique
    id), set up as include/sgr.h asks: every rank learns every rank's receive base, and reserves the push path's buffers for
    its feed up front, because nothing may allocate while a peer's wait kernel spins. new_engine() returns a new engine with
    its program registered and its options set; feeds[r] is rank r's device tensor of 64-byte records in arrival order, with
    the global aggregate index at +8. The engines are the caller's to read and are closed with the ranks."""

    def __init__(self, new_engine: Callable[[], object], part: np.ndarray, feeds: Sequence, capacity: int):
        R = len(feeds)
        self.engines: List = []
        self.feeds = list(feeds)
        try:
            for r in range(R):
                e = new_engine()
                self.engines.append(e)
                e.dist_init(r, R, None, capacity)
                e.dist_set_partitions(part)
            if R > 1:
                bases = [e.dist_recv_base() for e in self.engines]
                for e in self.engines:
                    e.dist_set_peers(bases)
            for e, f in zip(self.engines, self.feeds):
                e.dist_reserve(f.nbytes // 64)
        except BaseException:
            self.close()
            raise

    def close(self) -> None:
        for e in self.engines:
            e.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def run(self, fused: int, timeout: float = 120.0):
        """Every rank's dist_route_and_fold(feed, fused) on a thread of its own. A rank that meets a throwing aggregate
        returns SGR_ERR_AGAIN: real ranks agree over NCCL to repeat the exchange in log order, loopback ranks leave that to
        their caller, so when every rank returned either nothing or SGR_ERR_AGAIN, every rank repeats the call once with
        option push_ordered = 1. push_ordered is 0 again on return, whatever happened. A rank still inside its call after
        `timeout` seconds fails an assertion, and so does SGR_ERR_AGAIN next to another error.

        Returns (errors, repeated, times) of the last attempt: each rank's exception or None, whether the ordered repeat ran,
        and when each rank entered and left its call, in seconds after the threads were started."""
        R = len(self.engines)
        repeated = False
        try:
            for _attempt in range(2):
                errors, times = [None] * R, [None] * R
                t0 = time.monotonic()

                def one(r):
                    start = time.monotonic()
                    try:
                        self.engines[r].dist_route_and_fold(self.feeds[r], fused)
                    except Exception as ex:  # noqa: BLE001 — reported to the caller with the rank's other outcomes
                        errors[r] = ex
                    times[r] = (round(start - t0, 4), round(time.monotonic() - t0, 4))

                th = [threading.Thread(target=one, args=(r,)) for r in range(R)]
                for t in th:
                    t.start()
                for t in th:
                    t.join(timeout=timeout)
                assert not any(t.is_alive() for t in th), ("a loopback rank hung", "entered, returned:", times)
                again = [getattr(x, "code", None) == N.SGR_ERR_AGAIN for x in errors]
                if not any(again):
                    break
                assert all(x is None or a for x, a in zip(errors, again)), (errors, "entered, returned:", times)
                repeated = True
                for e in self.engines:
                    e.set_option("push_ordered", 1)
        finally:
            for e in self.engines:
                e.set_option("push_ordered", 0)
        return errors, repeated, times


def read_routed(engines: Sequence, ids: Sequence[str], num_partitions: int, arrays: bool = False):
    """getAggregateBytes for many ids over the ranks of one routed table, each rank holding its rank key table
    (ReplayEngine.dist_load_keys): every id goes to its owner, rank partitionForKey(id) % len(engines), as the Surge router sends
    a command to the node that owns the id's partition, and the answers come back in query order. For ranks inside one process;
    a real rank reads its own engine only. Returns what get_many returns: a list of Optional[bytes], or with arrays=True
    (states u8[n, state_bytes - 8], flags u32[n], indices i64[n]) where an index is a local slot of the owner (-1: unknown)."""
    R = len(engines)
    owner = partitions_for_keys(ids, num_partitions) % np.uint32(R)
    n = len(ids)
    user = engines[0].state_bytes - 8
    states = np.zeros((n, user), dtype=np.uint8)
    flags = np.zeros(n, dtype=np.uint32)
    indices = np.full(n, -1, dtype=np.int64)
    for r, e in enumerate(engines):
        pos = np.nonzero(owner == r)[0]
        if len(pos):
            states[pos], flags[pos], indices[pos] = e.get_many([ids[i] for i in pos], arrays=True)
    return (states, flags, indices) if arrays else _rows_or_none(states, flags)


def merge_scans(engines: Sequence, frm: Optional[str] = None, to: Optional[str] = None,
                page_rows: int = 1 << 20) -> Iterator[Tuple[str, int, int, int, bytes]]:
    """One scan of [frm, to] over the ranks of one routed table: the ranks' ordered pages (ReplayEngine.scan on each rank key
    table) merged into one stream in Bytes order of the ids, as range / all over every node's KTable would be. Each rank holds
    distinct ids, so the merge only interleaves. Yields (id, rank, local index, flags, program bytes) per live aggregate."""
    def rows(r, e):
        for idx, fl, st, page_ids in e.scan(frm, to, page_rows=page_rows):
            for i, k in enumerate(page_ids):
                yield k.encode("utf-8"), k, r, int(idx[i]), int(fl[i]), st[i].tobytes()

    for _, k, r, idx, fl, row in heapq.merge(*(rows(r, e) for r, e in enumerate(engines))):
        yield k, r, idx, fl, row
