"""TEST INFRASTRUCTURE — restatement of the device ingest's state-topic mode (include/sgr.h sgr_dingest_set_state_topic).

A compacted state topic (SurgeStateStoreConsumer.scala:57-76) read the way a read_committed consumer reads it, then applied the
way sgr_put_batch applies a batch (oracle/put_batch.py):
  * fetches [(partition, bytes, aborted [(producer_id, first_offset)])] are decoded as oracle/kafka_batch.read_committed_pack
    decodes them: CRC, control batches, aborted transactions, duplicates below the partition's position, the positions;
  * the id is the WHOLE key (no cut at ':'); a null or empty key is the producer's flush marker and is dropped;
  * a null value is a tombstone; any other value, after its framing, is the row's program bytes (at most state_bytes - 8):
    packed values are the bytes themselves, protobuf values are the `payload` (field 2) of the multilanguage
    `State { string aggregateId = 1; bytes payload = 2; }`;
  * a poll is one put batch of its live records in arrival order; a poll without live records applies nothing.
Never imported by surge_b200/."""
from __future__ import annotations

import struct
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import kafka_batch as K
from . import put_batch as PB

PACKED, PROTOBUF = 0, 1


class Refused(ValueError):
    pass


def _uvarint(b: bytes, p: int) -> Tuple[int, int]:
    x = shift = 0
    for _ in range(10):
        if p >= len(b):
            raise Refused("value is not a protobuf Event")
        c = b[p]
        p += 1
        x |= (c & 0x7F) << shift
        if not c & 0x80:
            return x, p
        shift += 7
    raise Refused("value is not a protobuf Event")


def protobuf_payload(v: bytes) -> bytes:
    """The last field 2 of wire type 2 (empty when there is none), as the device's unwrap reads it."""
    p, out = 0, b""
    while p < len(v):
        tag, p = _uvarint(v, p)
        wt = tag & 7
        if wt == 0:
            _, p = _uvarint(v, p)
        elif wt == 1 or wt == 5:
            n = 8 if wt == 1 else 4
            if len(v) - p < n:
                raise Refused("value is not a protobuf Event")
            p += n
        elif wt == 2:
            ln, p = _uvarint(v, p)
            if ln > len(v) - p:
                raise Refused("value is not a protobuf Event")
            if tag >> 3 == 2:
                out = v[p:p + ln]
            p += ln
        else:
            raise Refused("value is not a protobuf Event")
    return out


def encode_state(aggregate_id: bytes, payload: bytes) -> bytes:
    """The multilanguage State message: aggregateId = 1, payload = 2."""
    return K._uvar(0x0A) + K._uvar(len(aggregate_id)) + aggregate_id + K._uvar(0x12) + K._uvar(len(payload)) + payload


def read_committed_states(fetches: Iterable[Tuple[int, bytes, Sequence[Tuple[int, int]]]], framing: int = PACKED, row_bytes: int = 120):
    """(records [(id bytes, program bytes | None)] in arrival order, next offset per partition, statistics)."""
    recs: List[Tuple[bytes, Optional[bytes]]] = []
    nxt: Dict[int, int] = {}
    aborting: Dict[int, set] = {}
    pending: Dict[int, list] = {}
    st = dict(n_records=0, n_markers=0, n_null_values=0, n_duplicates=0, n_control_batches=0, n_aborted_batches=0, n_aborted_records=0)
    for partition, buf, aborted in fetches:
        pend = pending.setdefault(partition, [])
        pend.extend((fo, pid) for pid, fo in aborted)
        pend.sort()
        act = aborting.setdefault(partition, set())
        for b in K.decode_record_batches(buf):
            while pend and pend[0][0] <= b["last_offset"]:
                act.add(pend.pop(0)[1])
            if b["control"]:
                st["n_control_batches"] += 1
                if struct.unpack(">hh", b["records"][0][1][:4])[1] == K.ABORT:
                    act.discard(b["producer_id"])
            elif b["transactional"] and b["producer_id"] in act:
                st["n_aborted_batches"] += 1
                st["n_aborted_records"] += len(b["records"])
            else:
                for r, (od, key, val) in enumerate(b["records"]):
                    if partition in nxt and b["base_offset"] + od < nxt[partition]:
                        st["n_duplicates"] += 1
                        continue
                    if not key:
                        st["n_markers"] += 1
                        continue
                    if val is not None:
                        if framing == PROTOBUF:
                            val = protobuf_payload(val)
                        if len(val) > row_bytes:
                            raise Refused(f"offset {b['base_offset']}, record {r}: state value of {len(val)} bytes is longer than the "
                                          f"{row_bytes} program bytes of a row (state_bytes - 8)")
                    else:
                        st["n_null_values"] += 1
                    st["n_records"] += 1
                    recs.append((bytes(key), None if val is None else bytes(val)))
            nxt[partition] = max(nxt.get(partition, 0), b["last_offset"] + 1)
    return recs, nxt, st


def apply(ids: List[str], states: np.ndarray, records: Sequence[Tuple[bytes, Optional[bytes]]], f64_offsets: Sequence[int] = ()):
    """One poll on the table (oracle/put_batch.py layout); ids are the UTF-8 texts of the keys. No live records: unchanged."""
    if not records:
        return list(ids), states.copy()
    ids, out, _ = PB.put_batch(ids, states, [(k.decode("utf-8"), v) for k, v in records], f64_offsets)
    return ids, out
