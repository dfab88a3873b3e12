"""ctypes wrapper over the C oracle (oracle/sgr_oracle.c). TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
import this; nothing under surge_b200/ does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liborc.so")

MODEL_COUNTER, MODEL_BANK_ACCOUNT, MODEL_INT_BALANCE, MODEL_ML_COUNTER = 0, 1, 2, 3
REC_FIXED64, REC_VAR16 = 0, 1
ST_EXISTS, ST_CHANGED, ST_ERROR = 1, 2, 4


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "sgr_oracle.c")
    hdr = os.path.join(_HERE, "sgr_oracle.h")
    enc = os.path.join(_HERE, "kafka_encode.c")
    prg = os.path.join(_HERE, "program_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(f) for f in (src, hdr, enc, prg)):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-B"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        u8p, u64p = C.c_void_p, C.c_void_p
        L.orc_state_bytes.restype = C.c_uint32
        L.orc_state_bytes.argtypes = [C.c_int]
        L.orc_fold_packed.restype = C.c_int
        L.orc_fold_packed.argtypes = [C.c_int, C.c_uint32, u8p, u64p, C.c_uint64, u8p, u8p, u64p, u64p]
        L.orc_fold_packed_mt.restype = C.c_int
        L.orc_fold_packed_mt.argtypes = [C.c_int, C.c_uint32, u8p, u64p, C.c_uint64, u8p, u8p, C.c_int, u64p, u64p]
        L.orc_fold_packed_mt_pinned.restype = C.c_int
        L.orc_fold_packed_mt_pinned.argtypes = [C.c_int, C.c_uint32, u8p, u64p, C.c_uint64, u8p, u8p, C.c_int, u64p, u64p]
        L.orc_place_log_mt.restype = C.c_int
        L.orc_place_log_mt.argtypes = [u8p, u8p, u64p, C.c_uint64, C.c_int]
        L.orc_kafka_encode_bound.restype = C.c_uint64
        L.orc_kafka_encode_bound.argtypes = [C.c_uint64, C.c_uint32]
        L.orc_kafka_encode_counter.restype = C.c_int64
        L.orc_kafka_encode_counter.argtypes = [u8p, u8p, u8p, u8p, C.c_uint64, C.c_uint32, C.c_int, C.c_int64, u8p, C.c_uint64]
        L.orc_fold_incremental.restype = C.c_int
        L.orc_fold_incremental.argtypes = [C.c_int, u8p, C.c_uint64, u8p, C.c_uint64]
        L.orc_group_by_agg.restype = C.c_int
        L.orc_group_by_agg.argtypes = [u8p, C.c_uint64, C.c_uint64, u8p, u64p]
        L.orc_scala_string_hash.restype = C.c_int32
        L.orc_scala_string_hash.argtypes = [C.c_void_p, C.c_uint32]
        L.orc_partition_for_key.restype = C.c_int32
        L.orc_partition_for_key.argtypes = [C.c_void_p, C.c_uint32, C.c_int32]
        L.orc_take_while_not_colon.restype = C.c_uint32
        L.orc_take_while_not_colon.argtypes = [C.c_void_p, C.c_uint32]
        # fold programs (oracle/program_oracle.c, bound in oracle/program_interp.py)
        L.orc_prog_fold.restype = C.c_int
        L.orc_prog_fold.argtypes = [u8p, u8p, u64p, C.c_uint64, u8p, u8p, u64p, u64p]
        L.orc_prog_fold_var.restype = C.c_int
        L.orc_prog_fold_var.argtypes = [u8p, C.c_uint32, u8p, u64p, C.c_uint64, u8p, u8p, u64p, u64p]
        L.orc_prog_fold_arrival.restype = C.c_int
        L.orc_prog_fold_arrival.argtypes = [u8p, u8p, C.c_uint64, u8p, C.c_uint64, u64p, u64p]
        _lib = L
    return _lib


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def state_bytes(model: int) -> int:
    return int(lib().orc_state_bytes(model))


def fold_packed(model: int, record_kind: int, events: np.ndarray, seg_offsets: np.ndarray,
                initial_states: Optional[np.ndarray] = None, threads: int = 1, pinned: bool = False) -> Tuple[np.ndarray, int, int]:
    """Returns (states[n_agg, state_bytes] u8, n_events, n_errors). pinned: worker t runs on CPU t (see place_log)."""
    events = np.ascontiguousarray(events).view(np.uint8).reshape(-1)
    seg_offsets = np.ascontiguousarray(seg_offsets, dtype=np.uint64)
    n_agg = len(seg_offsets) - 1
    sb = state_bytes(model)
    out = np.zeros((n_agg, sb), dtype=np.uint8)
    if initial_states is not None:
        initial_states = np.ascontiguousarray(initial_states).view(np.uint8).reshape(n_agg, sb)
    nev, nerr = C.c_uint64(0), C.c_uint64(0)
    if threads > 1:
        fn = lib().orc_fold_packed_mt_pinned if pinned else lib().orc_fold_packed_mt
        rc = fn(model, record_kind, _ptr(events), _ptr(seg_offsets), n_agg, _ptr(initial_states),
                                      _ptr(out), threads, C.addressof(nev), C.addressof(nerr))
    else:
        rc = lib().orc_fold_packed(model, record_kind, _ptr(events), _ptr(seg_offsets), n_agg, _ptr(initial_states),
                                   _ptr(out), C.addressof(nev), C.addressof(nerr))
    if rc != 0:
        raise ValueError("oracle: malformed input")
    return out, int(nev.value), int(nerr.value)


def place_log(events: np.ndarray, seg_offsets: np.ndarray, threads: int) -> np.ndarray:
    """NUMA-aware copy of a CSR log for the CPU arm of bench.py: the copy is written by the pinned workers that will later
    fold it (same byte sharding), so first touch puts every worker's range on its own node."""
    events = np.ascontiguousarray(events).view(np.uint8).reshape(-1)
    seg_offsets = np.ascontiguousarray(seg_offsets, dtype=np.uint64)
    dst = np.empty(events.size, dtype=np.uint8)   # fresh mapping: pages untouched until the workers write them
    if lib().orc_place_log_mt(_ptr(dst), _ptr(events), _ptr(seg_offsets), len(seg_offsets) - 1, threads) != 0:
        raise ValueError("oracle: placement failed")
    return dst


def kafka_encode_counter(agg: np.ndarray, types: np.ndarray, seqs: np.ndarray, bys: np.ndarray, recs_per_batch: int = 512, lz4: bool = True,
                         base_offset: int = 0, out: Optional[np.ndarray] = None) -> np.ndarray:
    """Producer-side bytes of one partition of the Counter events topic (oracle/kafka_encode.c): consecutive RecordBatch v2
    structures of recs_per_batch records, key "agg-<n>:<seq>", value = packed (type, seq, by). Returns a uint8 view of `out`
    (allocated when None). Test / bench INPUT construction only."""
    agg = np.ascontiguousarray(agg, dtype=np.uint32); types = np.ascontiguousarray(types, dtype=np.uint32)
    seqs = np.ascontiguousarray(seqs, dtype=np.uint32); bys = np.ascontiguousarray(bys, dtype=np.int32)
    n = len(agg)
    bound = int(lib().orc_kafka_encode_bound(n, recs_per_batch))
    if out is None:
        out = np.empty(bound, dtype=np.uint8)
    got = lib().orc_kafka_encode_counter(_ptr(agg), _ptr(types), _ptr(seqs), _ptr(bys), n, recs_per_batch, 1 if lz4 else 0, base_offset, _ptr(out), out.size)
    if got < 0:
        raise ValueError("kafka_encode: output buffer too small")
    return out[:got]


def group_by_agg(records: np.ndarray, n_agg: int) -> Tuple[np.ndarray, np.ndarray]:
    records = np.ascontiguousarray(records).view(np.uint8).reshape(-1, 64)
    n = records.shape[0]
    out = np.zeros_like(records)
    offs = np.zeros(n_agg + 1, dtype=np.uint64)
    if lib().orc_group_by_agg(_ptr(records), n, n_agg, _ptr(out), _ptr(offs)) != 0:
        raise ValueError("oracle: aggregate index out of range")
    return out, offs


def fold_incremental(model: int, records: np.ndarray, states: np.ndarray) -> np.ndarray:
    records = np.ascontiguousarray(records).view(np.uint8).reshape(-1, 64)
    sb = state_bytes(model)
    states = np.ascontiguousarray(states).view(np.uint8).reshape(-1, sb).copy()
    if lib().orc_fold_incremental(model, _ptr(records), records.shape[0], _ptr(states), states.shape[0]) != 0:
        raise ValueError("oracle: malformed input")
    return states


def _utf16(s: str) -> np.ndarray:
    return np.frombuffer(s.encode("utf-16-le"), dtype=np.uint16).copy()


def scala_string_hash(s: str) -> int:
    u = _utf16(s)
    return int(lib().orc_scala_string_hash(_ptr(u) if len(u) else None, len(u)))


def partition_for_key(s: str, n: int, up_to_colon: bool = False) -> int:
    u = _utf16(s)
    k = len(u)
    if up_to_colon and k:
        k = int(lib().orc_take_while_not_colon(_ptr(u), k))
    return int(lib().orc_partition_for_key(_ptr(u) if len(u) else None, k, n))
