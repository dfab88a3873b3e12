"""TEST INFRASTRUCTURE — the multilanguage gateway's JSON topics (SGR_VALUE_PROTOBUF_JSON), restated apart from the product.

Every business app of the reference serializes its events and states as flat JSON, and the multilanguage gateway wraps them in
the protobuf `Event` / `State { string aggregateId = 1; bytes payload = 2; }`
(modules/multilanguage/src/main/scala/com/ukg/surge/multilanguage/GenericSurgeCommandBusinessLogic.scala:25-38). This module
holds what the tests compare such topics with:
  * the C# SDK sample's event handler, restated from its C# source as oracle/surge_model.py restates the Scala samples;
  * the three reference models' JSON member tables (events and states), the layouts Ingest.set_json_packer takes;
  * pbjson_corpus: protobuf-wrapped JSON values and hostile variants of both layers, for the host and device decoders;
  * read_committed_states for a state topic under the protobuf-wrapped JSON framing: oracle/state_topic.py's read of the
    fetches, then each State's payload mapped to program bytes with Python's json module.
Never imported by surge_b200/."""
from __future__ import annotations

import json
import struct
import uuid
from dataclasses import dataclass
from typing import Iterable, Optional, Sequence, Tuple

from . import state_topic as S
from . import value_corpus as V
from .surge_model import jvm_int

I32, I64, F64, UUID, PSTR = 0, 1, 2, 3, 4          # = surge_b200.native.JSON_*

# ------------------------------------------------------------------------------------------------ C# SDK sample
# modules/multilanguage-csharp-sdk/Sample/Model.cs:7-60 (Newtonsoft.Json, JsonSubtypes discriminator "Type")
@dataclass(frozen=True)
class Account:
    amount: int


@dataclass(frozen=True)
class MoneyWithdrawn:
    Amount: int


@dataclass(frozen=True)
class MoneyDeposited:
    Amount: int


@dataclass(frozen=True)
class OtherBankEvent:
    """any BankEvent that is neither subtype (the base class's Type, or one a later app version adds)"""
    Type: str


def csharp_bank_event_handler(state: Optional[Account], bank_event) -> Optional[Account]:
    """Sample/Program.cs:62-80 (CqrsModel.EventHandler). C# int arithmetic is unchecked: it wraps as a JVM Int does."""
    balance = state.amount if state is not None else 0
    if isinstance(bank_event, MoneyWithdrawn):
        return Account(jvm_int(balance - bank_event.Amount))
    if isinstance(bank_event, MoneyDeposited):
        return Account(jvm_int(balance + bank_event.Amount))
    return None


def csharp_bank_event(obj: dict):
    """JsonConvert.DeserializeObject<BankEvent> of one events-topic payload (Program.cs:27-32)."""
    if obj["Type"] == "MoneyWithdrawn":
        return MoneyWithdrawn(obj["Amount"])
    if obj["Type"] == "MoneyDeposited":
        return MoneyDeposited(obj["Amount"])
    return OtherBankEvent(obj["Type"])


# ------------------------------------------------------------------------------------------------ member tables
# (class name, event type, [(member, kind, record offset[, slot bytes])]) for the events topics; [(member, kind, program offset)]
# for the state topics (no discriminator, one class)
ML_COUNTER_EVENTS = ("_type", [("com.ukg.surge.multilanguage.TestBoundedContext.CountIncremented", 0, [("incrementBy", I32, 16), ("sequenceNumber", I32, 4)]),
                               ("com.ukg.surge.multilanguage.TestBoundedContext.CountDecremented", 1, [("decrementBy", I32, 16), ("sequenceNumber", I32, 4)])])
ML_COUNTER_STATE = [("count", I32, 0), ("version", I32, 4)]
INT_BALANCE_EVENTS = ("", [("MoneyDeposited", 0, [("amount", I32, 16)])])
INT_BALANCE_STATE = [("balance", I32, 0)]
CSHARP_BANK_EVENTS = ("Type", [("MoneyWithdrawn", 0, [("Amount", I32, 16)]), ("MoneyDeposited", 1, [("Amount", I32, 16)])])
CSHARP_BANK_UNKNOWN_TYPE = 2
CSHARP_ACCOUNT_STATE = [("amount", I32, 0)]


def json_row(obj: dict, members: Sequence[Tuple], row_bytes: int) -> bytes:
    """The program bytes a state's JSON object gives under a member table [(name, kind, program offset[, slot bytes])]."""
    row = bytearray(row_bytes)
    for m in members:
        name, kind, off = m[0], m[1], m[2]
        v = obj[name]
        if kind == I32:
            row[off:off + 4] = struct.pack("<i", v)
        elif kind == I64:
            row[off:off + 8] = struct.pack("<q", v)
        elif kind == F64:
            row[off:off + 8] = struct.pack("<d", float(v))
        elif kind == UUID:
            row[off:off + 16] = uuid.UUID(v).bytes
        else:
            b = v.encode("utf-8")
            assert len(b) <= m[3] - 1
            row[off] = len(b)
            row[off + 1:off + 1 + len(b)] = b
    return bytes(row)


def read_committed_states(fetches: Iterable[Tuple[int, bytes, Sequence[Tuple[int, int]]]], members: Sequence[Tuple], row_bytes: int):
    """oracle/state_topic.read_committed_states for SGR_VALUE_PROTOBUF_JSON: (records [(id bytes, program bytes | None)] in
    arrival order, next offset per partition, statistics). Each live value is a protobuf State whose payload is a JSON object;
    the State's aggregateId is not read (the key is the id)."""
    recs, nxt, st = S.read_committed_states(fetches, S.PROTOBUF, row_bytes=1 << 30)
    return [(k, None if v is None else json_row(json.loads(v), members, row_bytes)) for k, v in recs], nxt, st


# ------------------------------------------------------------------------------------------------ value corpus
def _uv(v):
    return V.pb_varint(v)


def _field2(payload, wire_type=2):
    if wire_type == 2:
        return b"\x12" + _uv(len(payload)) + payload
    if wire_type == 0:
        return b"\x10" + _uv(len(payload))
    return (b"\x11" + bytes(8)) if wire_type == 1 else (b"\x15" + bytes(4))


def padded(json_bytes, n):
    """the same object with whitespace before its closing brace: exactly n bytes"""
    assert len(json_bytes) <= n
    return json_bytes[:-1] + b" " * (n - len(json_bytes)) + b"}"


def pbjson_corpus(rng, json_values, Event):
    """SGR_VALUE_PROTOBUF_JSON values: the JSON values wrapped as `Event` (a protobuf message class with the multilanguage Event's
    fields, built by the caller from the protobuf runtime), then hostile variants of both layers: truncated tags and lengths,
    wire types 3, 4, 6 and 7, field 2 missing, repeated or of another wire type, unknown fields before and after, payloads of
    127, 128, 16383 and 16384 bytes, and byte mutations of the messages and of the JSON inside them."""
    wrapped = [Event(aggregateId=f"agg-{d}", payload=v).SerializeToString() for d, v in enumerate(json_values)]
    out = list(wrapped)
    good = json_values[:200]
    for d, v in enumerate(good):
        w = wrapped[d]
        out.append(w[:int(rng.integers(0, min(len(w), 12) + 1))])                      # a truncated tag or length
        out.append(b"\x12" + b"\xff" * int(rng.integers(1, 4)))                        # a length varint that never ends
        for wt in (3, 4, 6, 7):                                                        # wire types nobody may skip
            out.append(bytes([(9 << 3) | wt]) + w)
            out.append(w + bytes([(9 << 3) | wt]))
        out.append(b"\x0a\x03abc")                                                     # field 2 missing: an empty payload
        out.append(b"\x0a\x03abc" + _field2(v, int(rng.choice([0, 1, 5]))))            # field 2 of another wire type: skipped
        out.append(_field2(b"[1,2]") + _field2(v))                                     # repeated: the last one wins
        out.append(_field2(v) + _field2(b"{\"x\":"))
        unk = _uv((int(rng.integers(3, 1000)) << 3) | 0) + _uv(int(rng.integers(0, 2**63)))
        unk += _uv((77 << 3) | 1) + bytes(8) + _uv((78 << 3) | 5) + bytes(4) + _uv((79 << 3) | 2) + b"\x02hi"
        out.append(unk + w)                                                            # unknown fields before
        out.append(w + unk)                                                            # ... and after
    for n in (127, 128, 16383, 16384):                                                 # payload lengths around the varint steps
        for v in good[:8]:
            if len(v) <= n:
                out.append(Event(aggregateId="p", payload=padded(v, n)).SerializeToString())
    out += V.mutants(rng, wrapped, 3000)                                               # bytes of both layers
    out += [Event(aggregateId="m", payload=m).SerializeToString() for m in V.mutants(rng, json_values, 2000)]
    return out
