"""Ingest: Kafka RecordBatch bytes -> packed event records, over the C ABI (include/sgr.h, "ingest" section).

Host-side mirror of what sits in front of the state store in the reference: the read_committed consumer
(modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:38) and the lag gate's view of how far the
store has consumed (modules/common/src/main/scala/surge/kafka/KafkaAdminClient.scala:36-56). All decoding happens in
libsgr.so; this class only moves pointers.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import native as N


class IngestError(N.SgrError):
    pass


def _as_pointer(data) -> C.c_void_p:
    """Address of a bytes-like object's buffer, without copying it (the decoder only reads)."""
    if not len(data):
        return C.c_void_p(None)
    if isinstance(data, bytes):
        return C.cast(C.c_char_p(data), C.c_void_p)
    return C.c_void_p(np.frombuffer(data, dtype=np.uint8).ctypes.data)


def json_events(events: Sequence[Tuple[str, int, Sequence[Tuple]]]):
    """the sgr_json_event array of a JSON packer (Ingest.set_json_packer's `events`)"""
    arr = (N.sgr_json_event * max(len(events), 1))()
    for i, (type_name, event_type, fields) in enumerate(events):
        arr[i].type_name = type_name.encode("utf-8")
        arr[i].event_type = event_type
        arr[i].n_fields = len(fields)
        if len(fields) > 8:
            raise IngestError(N.SGR_ERR_INVALID, "at most 8 numeric members per event")
        for j, spec in enumerate(fields):
            name, kind, dst_off = spec[:3]
            arr[i].fields[j].name = name.encode("utf-8")
            arr[i].fields[j].kind = kind
            arr[i].fields[j].dst_off = dst_off
            arr[i].fields[j].len = spec[3] if len(spec) > 3 else 0      # slot size of a JSON_PSTR member
    return arr


def _stats(st) -> Dict[str, int]:
    return {n: int(getattr(st, n)) for n, _ in N.sgr_ingest_stats._fields_ if n != "reserved"}


def _set_aborted(check, fn, handle, partition: int, aborted: Sequence[Tuple[int, int]]) -> None:
    """fn: sgr_ingest_set_aborted or sgr_dingest_set_aborted; `check` raises on its return code"""
    if not aborted:
        return
    pids = np.asarray([a[0] for a in aborted], dtype=np.int64)
    offs = np.asarray([a[1] for a in aborted], dtype=np.int64)
    check(fn(handle, partition, pids.ctypes.data, offs.ctypes.data, len(aborted)))


def _offsets(check, fn, handle, partition: int) -> Tuple[int, int]:
    """(decoded_next, folded_next) through fn = sgr_ingest_offsets or sgr_dingest_offsets"""
    d, f = C.c_int64(), C.c_int64()
    check(fn(handle, partition, C.byref(d), C.byref(f)))
    return d.value, f.value


class Ingest:
    def __init__(self):
        self._lib = N.load_library()
        self._h = C.c_void_p()
        rc = self._lib.sgr_ingest_create(C.byref(self._h))
        if rc != N.SGR_OK:
            raise IngestError(rc, "sgr_ingest_create failed")

    def close(self) -> None:
        if self._h:
            self._lib.sgr_ingest_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    def _check(self, rc: int) -> None:
        if rc != N.SGR_OK:
            msg = self._lib.sgr_ingest_last_error(self._h)
            raise IngestError(rc, msg.decode("utf-8", "replace") if msg else "")

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def set_value_framing(self, framing: int) -> None:
        """How a record value wraps its event (include/sgr.h SGR_VALUE_*): N.VALUE_PACKED, the value is the packed event;
        N.VALUE_PROTOBUF_EVENT, the protobuf Event{aggregateId, payload} of the multilanguage module, whose payload is the packed
        event; N.VALUE_JSON, a flat JSON object read through the member table of set_json_packer; N.VALUE_PROTOBUF_JSON, the
        multilanguage Event whose payload is such a JSON object (what the gateway writes for an app that serializes its events as
        JSON). The two JSON framings need set_json_packer first. Event.aggregateId is not read: the record key is the id."""
        self._check(self._lib.sgr_ingest_set_value_framing(self._h, framing))

    def set_json_packer(self, discriminator: str, events: Sequence[Tuple[str, int, Sequence[Tuple[str, int, int]]]], unknown_type: int = -1) -> None:
        """events = [(class name, event type index, [(member name, N.JSON_I32 | JSON_I64 | JSON_F64 | JSON_UUID, record byte offset) or
        (member name, N.JSON_PSTR, record byte offset, slot bytes)])].
        Switches nothing by itself: follow with set_value_framing(N.VALUE_JSON) or set_value_framing(N.VALUE_PROTOBUF_JSON)."""
        self._check(self._lib.sgr_ingest_set_json_packer(self._h, discriminator.encode("utf-8"), json_events(events), len(events), unknown_type))

    def set_null_value_type(self, event_type: int) -> None:
        """State-topic mode: null-valued records become events of `event_type` (the program's tombstone rule); -1 drops them."""
        self._check(self._lib.sgr_ingest_set_null_value_type(self._h, event_type))

    def set_dictionary_limits(self, max_ids: int, max_id_bytes: int) -> None:
        """Fail with SGR_ERR_CAPACITY once a call could carry the id dictionary past these bounds (defaults 2^31 ids, 4 GiB)."""
        self._check(self._lib.sgr_ingest_set_dictionary_limits(self._h, max_ids, max_id_bytes))

    def set_aborted(self, partition: int, aborted: Sequence[Tuple[int, int]]) -> None:
        """aborted = [(producer_id, first_offset)] from the fetch response."""
        _set_aborted(self._check, self._lib.sgr_ingest_set_aborted, self._h, partition, aborted)

    def record_batches(self, partition: int, data: bytes) -> Dict[str, int]:
        st = N.sgr_ingest_stats()
        self._check(self._lib.sgr_ingest_record_batches(self._h, partition, _as_pointer(data), len(data), C.byref(st)))
        return _stats(st)

    def record_batches_mt(self, fetches: Sequence[Tuple[int, bytes]], threads: int = 0) -> List[Dict[str, int]]:
        """Several fetches [(partition, bytes)] in one call, decoded on `threads` host threads (0 = one per partition,
        capped by the host's cores); same outcome as calling record_batches on each in order."""
        import os

        n = len(fetches)
        if not n:
            return []
        parts = (C.c_int32 * n)(*[p for p, _ in fetches])
        ptrs = (C.c_void_p * n)(*[_as_pointer(d) for _, d in fetches])     # borrowed for the call: `fetches` keeps the bytes alive
        lens = (C.c_uint64 * n)(*[len(d) for _, d in fetches])
        st = (N.sgr_ingest_stats * n)()
        thr = threads or min(len({p for p, _ in fetches}), os.cpu_count() or 1)
        self._check(self._lib.sgr_ingest_record_batches_mt(self._h, n, parts, ptrs, lens, thr, st))
        return [_stats(s) for s in st]

    def pending(self) -> np.ndarray:
        """Copy of the pending packed records, [n, 64] uint8."""
        p = C.c_void_p()
        n = C.c_uint64()
        self._check(self._lib.sgr_ingest_pending(self._h, C.byref(p), C.byref(n)))
        if not n.value:
            return np.zeros((0, 64), dtype=np.uint8)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value * 64,)).reshape(-1, 64).copy()

    def keys(self) -> List[str]:
        kp, op = C.c_void_p(), C.c_void_p()
        n = C.c_uint64()
        self._check(self._lib.sgr_ingest_keys(self._h, C.byref(kp), C.byref(op), C.byref(n)))
        if not n.value:
            return []
        offs = np.ctypeslib.as_array(C.cast(op, C.POINTER(C.c_uint32)), shape=(n.value + 1,)).copy()
        raw = C.string_at(kp, int(offs[-1])) if offs[-1] else b""
        return [raw[offs[i]:offs[i + 1]].decode("utf-8") for i in range(n.value)]

    def mark_folded(self) -> None:
        self._check(self._lib.sgr_ingest_mark_folded(self._h))

    def offsets(self, partition: int) -> Tuple[int, int]:
        """(decoded_next, folded_next): next offset to fetch, and the offset to commit for the lag gate."""
        return _offsets(self._check, self._lib.sgr_ingest_offsets, self._h, partition)

    def stats(self) -> Dict[str, int]:
        st = N.sgr_ingest_stats()
        self._check(self._lib.sgr_ingest_get_stats(self._h, C.byref(st)))
        return _stats(st)
