"""DeviceIngest: Kafka RecordBatch bytes -> folded state table with the decode ON THE GPU (include/sgr.h "device ingest").

The same input and the same outcome as Ingest + ReplayEngine.fold_ingested (surge_b200/ingest.py), but only the wire bytes cross
PCIe: CRC-32C, lz4, record parsing, id interning and the fold run on the engine's device (csrc/dingest_kernels.cu). The host
walks batch headers and keeps the read_committed bookkeeping of the consumer the reference configures
(modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:38).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Sequence, Tuple

from . import native as N
from .ingest import IngestError, _as_pointer, _offsets, _set_aborted, _stats, json_events


class DeviceIngest:
    def __init__(self, engine, max_keys: int, max_id_bytes: int = 0):
        self._lib = N.load_library()
        self._engine = engine
        self._h = C.c_void_p()
        eh = getattr(engine, "_h", None)
        if not isinstance(eh, C.c_void_p) or not eh:
            raise IngestError(N.SGR_ERR_INVALID, "a device ingest needs an open ReplayEngine")
        rc = self._lib.sgr_dingest_create(engine._h, int(max_keys), int(max_id_bytes), C.byref(self._h))
        if rc != N.SGR_OK:
            raise IngestError(rc, "sgr_dingest_create failed")
        self._keep = []   # submitted buffers stay alive until the fold (the H2D copy may be asynchronous)

    def close(self) -> None:
        if self._h:
            self._lib.sgr_dingest_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc: int) -> None:
        if rc != N.SGR_OK:
            msg = self._lib.sgr_dingest_last_error(self._h)
            raise IngestError(rc, msg.decode("utf-8", "replace") if msg else "")

    def set_null_value_type(self, event_type: int) -> None:
        self._check(self._lib.sgr_dingest_set_null_value_type(self._h, event_type))

    def set_value_framing(self, framing: int) -> None:
        """N.VALUE_PACKED, N.VALUE_PROTOBUF_EVENT, N.VALUE_JSON or N.VALUE_PROTOBUF_JSON (the last two after set_json_packer), as
        Ingest.set_value_framing. In state-topic mode N.VALUE_PROTOBUF_JSON reads the multilanguage State, whose payload is the
        app's JSON state, into the row through the member table."""
        self._check(self._lib.sgr_dingest_set_value_framing(self._h, framing))

    def set_json_packer(self, discriminator: str, events: Sequence[Tuple[str, int, Sequence[Tuple]]], unknown_type: int = -1) -> None:
        """The member table of JSON values, with the arguments of Ingest.set_json_packer."""
        self._check(self._lib.sgr_dingest_set_json_packer(self._h, discriminator.encode("utf-8"), json_events(events), len(events), unknown_type))

    def set_state_topic(self, on: bool = True) -> None:
        """Decode a compacted state topic (include/sgr.h sgr_dingest_set_state_topic): the whole key is the id, a value is the
        program bytes of a row (after its framing), null deletes, and fold() applies the poll last write wins. Set it before the
        first fold and before set_json_packer, whose member offsets then are program byte offsets."""
        self._check(self._lib.sgr_dingest_set_state_topic(self._h, 1 if on else 0))

    def set_aborted(self, partition: int, aborted: Sequence[Tuple[int, int]]) -> None:
        _set_aborted(self._check, self._lib.sgr_dingest_set_aborted, self._h, partition, aborted)

    def submit(self, partition: int, data) -> Dict[str, int]:
        """bytes of one fetch response (bytes, numpy uint8 array, or a pinned torch uint8 tensor): header walk + H2D copy."""
        st = N.sgr_ingest_stats()
        if hasattr(data, "data_ptr"):
            ptr, n = C.c_void_p(data.data_ptr()), int(data.numel())
        else:
            ptr, n = _as_pointer(data), len(data)
        self._keep.append(data)
        self._check(self._lib.sgr_dingest_submit(self._h, partition, ptr, n, C.byref(st)))
        return _stats(st)

    def fold(self) -> Dict[str, int]:
        """decode + intern + fold everything submitted since the last fold; returns the poll's statistics."""
        st = N.sgr_ingest_stats()
        try:
            self._check(self._lib.sgr_dingest_fold(self._h, C.byref(st)))
        finally:
            self._keep = []
        return _stats(st)

    def last_timing(self) -> Dict[str, float]:
        ms = (C.c_float * 8)()
        self._check(self._lib.sgr_dingest_last_timing(self._h, ms))
        # [0] is the wait for the copies and every group's CRC -> decode -> parse chain, [1] only the repeat from an exact arena
        # layout (0 normally), [2] unused (its key stays so that recorded results keep their shape)
        return dict(zip(("wait_copies_and_chains", "decode_walk", "parse_intern", "keys_gather", "grow_fold_append_keys", "total"), [float(x) for x in ms[:6]]))

    def reset(self) -> None:
        """Forget dictionary, positions and statistics: the next poll rebuilds from offset 0."""
        self._keep = []
        self._check(self._lib.sgr_dingest_reset(self._h))

    def offsets(self, partition: int) -> Tuple[int, int]:
        return _offsets(self._check, self._lib.sgr_dingest_offsets, self._h, partition)
