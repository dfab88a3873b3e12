"""Host-side mirror of the reference's state-store boundary, over the C ABI.

Reference interfaces mirrored here (same names, argument meaning and error behaviour; paths relative to the
reference checkout, COMMON = modules/common/src/main/scala/surge):

  SurgeKafkaStreamsPersistencePlugin { createSupplier(storeName); enableLogging }
      COMMON/kafka/streams/SurgeKafkaStreamsPersistencePlugin.scala:12-15
  SurgeKafkaStreamsPersistencePluginLoader.load(config)                       same file, :27-50
  KeyValueBytesStoreSupplier.get(): KeyValueStore[Bytes, Array[Byte]]         (Kafka Streams; in-tree example
      modules/common/src/test/scala/surge/kafka/streams/SingleExceptionThrowingKeyValueStore.scala:18-91)
  AggregateStateStoreKafkaStreams.getAggregateBytes(aggregateId): Future[Option[Array[Byte]]]
      COMMON/kafka/streams/AggregateStateStoreKafkaStreams.scala:83-85
  ThreadPools.ioBoundContext (32 threads)                                     COMMON/kafka/streams/ThreadPools.scala:9-11

The JVM shim (shim/scala) is the real drop-in; this module is its executable twin for the toolchain this
image has, and is what the parity tests drive. It adds nothing to the data path: every fold runs in
libsgr.so on the GPU.
"""
from __future__ import annotations

import importlib
import threading
import time
from concurrent.futures import Future, ThreadPoolExecutor
from typing import Callable, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import native as N
from .engine import ReplayEngine
from .ingest import Ingest

STATE_STORE_PLUGIN_KEY = "surge.kafka-streams.state-store-plugin"


class InvalidStateStoreException(N.InvalidStateStoreException):
    pass


# --------------------------------------------------------------------------- plugin + loader
class SurgeKafkaStreamsPersistencePlugin:
    """trait SurgeKafkaStreamsPersistencePlugin (SurgeKafkaStreamsPersistencePlugin.scala:12-15)."""

    def createSupplier(self, storeName: str) -> "KeyValueBytesStoreSupplier":  # noqa: N802,N803 - reference names
        raise NotImplementedError

    @property
    def enableLogging(self) -> bool:  # noqa: N802
        raise NotImplementedError


class SurgeKafkaStreamsPersistencePluginLoader:
    """object SurgeKafkaStreamsPersistencePluginLoader (same file, :27-50): reads
    `surge.kafka-streams.state-store-plugin`, then `<name>.plugin-class`, instantiates it with the no-arg
    constructor. DEVIATION (deliberate): the reference silently falls back to RocksDB on any failure
    (:34-39,45-47); a GPU store that silently turns into RocksDB would void every measurement, so this loader
    raises instead."""

    @staticmethod
    def load(config: Dict[str, str]) -> SurgeKafkaStreamsPersistencePlugin:
        name = config.get(STATE_STORE_PLUGIN_KEY)
        if not name:
            raise KeyError(f"{STATE_STORE_PLUGIN_KEY} is not set")
        cls_path = config.get(f"{name}.plugin-class")
        if not cls_path:
            raise KeyError(f"{name}.plugin-class is not set")
        mod, _, cls = cls_path.rpartition(".")
        plugin = getattr(importlib.import_module(mod), cls)()
        if not isinstance(plugin, SurgeKafkaStreamsPersistencePlugin):
            raise TypeError(f"{cls_path} is not a SurgeKafkaStreamsPersistencePlugin")
        return plugin


class KeyValueBytesStoreSupplier:
    def __init__(self, name: str, factory: Callable[[str], "GpuReplayKeyValueStore"]):
        self._name, self._factory = name, factory

    def name(self) -> str:
        return self._name

    def get(self) -> "GpuReplayKeyValueStore":
        return self._factory(self._name)

    def metricsScope(self) -> str:  # noqa: N802
        return "gpu-replay"


class GpuReplayPersistencePlugin(SurgeKafkaStreamsPersistencePlugin):
    """Config-selected drop-in:  surge.kafka-streams.state-store-plugin = "gpu-replay"
                                 gpu-replay.plugin-class = "surge_b200.store.GpuReplayPersistencePlugin"
    enableLogging = false: Kafka Streams must not restore this store from a changelog — it rebuilds from the
    events topic (SurgeStateStoreConsumer.scala:63-75)."""

    program_factory: Optional[Callable[[], N.sgr_fold_program]] = None  # set by the model registration
    device: int = 0

    def createSupplier(self, storeName: str) -> KeyValueBytesStoreSupplier:  # noqa: N802,N803
        if GpuReplayPersistencePlugin.program_factory is None:
            raise N.SgrError(N.SGR_ERR_NO_PROGRAM, "no fold program registered for the model (GpuReplayPersistencePlugin.program_factory)")
        return KeyValueBytesStoreSupplier(storeName, lambda n: GpuReplayKeyValueStore(n, GpuReplayPersistencePlugin.program_factory(),
                                                                                      GpuReplayPersistencePlugin.device))

    @property
    def enableLogging(self) -> bool:  # noqa: N802
        return False


# --------------------------------------------------------------------------- the store
def aggregate_id_of_record_key(key: str) -> str:
    """Event record keys are model-defined ("<aggId>:<seq>" in core TestBoundedContext.scala:160, or the bare id);
    the aggregate is key.takeWhile(_ != ':') under the default partitioner (KafkaPartitioner.scala:38-42)."""
    i = key.find(":")
    return key if i < 0 else key[:i]


class StateCodec:
    """serialized state bytes (what the state topic and the actors hold) <-> the packed program bytes of the GPU table
    (trait GpuStateCodec of shim/scala GpuReplayPersistencePlugin.scala). snapshot_type / tombstone_type are the two extra rules of
    the registered fold program (programs.counter_program_with_snapshot_rules); a codec without them (both None) makes the store
    a state-topic store, whose state records go to the table through sgr_put_batch (no extra rules, states of any width).
    writer: a JSON state writer table for ReplayEngine.set_state_writer, [(name, N.JSON_*, program offset[, slot bytes])] or
    (name, N.JSON_ID): the store's reads and on_changes then take the model's JSON value from the device (sgr_get_batch_values,
    sgr_scan_values, sgr_export_changes_values) instead of calling from_packed, which becomes optional.
    writer_framing: how the device wraps those values, N.VALUE_JSON (the JSON value itself, the default) or N.VALUE_PROTOBUF_JSON
    (the multilanguage protobuf State around it: what a multilanguage store holds, ReplayEngine.set_state_writer_framing)."""

    def __init__(self, to_packed: Callable[[str, bytes], bytes], from_packed: Optional[Callable[[str, bytes], bytes]] = None,
                 snapshot_type: Optional[int] = None, tombstone_type: Optional[int] = None, writer: Optional[Sequence[Tuple]] = None,
                 writer_framing: int = N.VALUE_JSON):
        if (snapshot_type is None) != (tombstone_type is None):
            raise ValueError("a codec names both the snapshot and the tombstone type, or neither")
        if from_packed is None and writer is None:
            raise ValueError("a codec decodes rows with from_packed, or has the device write them with a writer table")
        self.to_packed, self.from_packed, self.snapshot_type, self.tombstone_type = to_packed, from_packed, snapshot_type, tombstone_type
        self.writer = None if writer is None else list(writer)
        self.writer_framing = writer_framing

    @property
    def state_topic(self) -> bool:
        """No snapshot rules: put()/delete() are applied by sgr_put_batch."""
        return self.snapshot_type is None


class GpuReplayKeyValueStore:
    """KeyValueStore[Bytes, Array[Byte]] whose content is the GPU-folded state table.

    write side (one stream thread in the reference): restore()/put_event() batch packed 64-byte event records;
    flush() folds the batch on the GPU (first batch: group + full fold, later batches: incremental fold).
    put()/delete() of *state* records keep KTable semantics — last write wins per key, null deletes
    (SurgeStateStoreConsumer.scala:57-76) — as an overlay over the folded table.
    read side (32-thread pool in the reference): get() is thread-safe.
    """

    def __init__(self, name: str, program: N.sgr_fold_program, device: int = 0, state_formatter: Optional[Callable[[str, bytes], bytes]] = None,
                 codec: Optional[StateCodec] = None,
                 on_changes: Optional[Callable[[List[Tuple[str, Optional[bytes]]], List[Tuple[str, int]]], None]] = None,
                 max_ids: int = 1 << 20):
        self._name = name
        # on_changes(changed, failed): called once by every flush() that folded, before it returns, with what the reference's
        # actors would publish for that fold (PersistentActor.scala:252-263): changed = [(id, serialized state or None)], decoded
        # like get(), None for a state that became None; failed = [(id, err_idx)] for the aggregates whose handler threw. Values
        # put() keeps in the overlay (a store without a codec) are not folded, so they are never reported.
        self._on_changes = on_changes
        # with a codec, put()/delete() are records of the STATE topic folded on the GPU as snapshot / tombstone events (feed (i) of
        # the Scala store): flush() — which Kafka Streams calls before it commits offsets — makes them readable from the table.
        # A codec without snapshot rules makes a state-topic store: flush() hands the pending records to one sgr_put_batch,
        # which numbers new ids on the device in first-appearance order (the order _slot follows), so no key table is loaded.
        # A state-topic store may instead restore the topic's raw record batches (restore_record_batches): a DeviceIngest in
        # state-topic mode decodes and applies them on the device, its id dictionary bounded by max_ids
        self._codec = codec
        self._max_ids = int(max_ids)
        self._dingest = None
        self._state_topic = codec is not None and codec.state_topic
        self._puts: List[Tuple[str, Optional[bytes]]] = []   # a state-topic store's pending records, packed, in arrival order
        self._unflushed: Dict[str, Optional[bytes]] = {}
        self._engine = ReplayEngine(device)
        self._engine.register_program(program)
        # with a writer table, values leave the device as the model's JSON state and the host codec is not called
        self._writer = codec is not None and codec.writer is not None
        if self._writer:
            self._engine.set_state_writer(codec.writer)
            if codec.writer_framing != N.VALUE_JSON:
                self._engine.set_state_writer_framing(codec.writer_framing)
        self._formatter = state_formatter
        self._keys: List[str] = []
        self._index: Dict[str, int] = {}
        self._pending: List[np.ndarray] = []
        self._overlay: Dict[str, Optional[bytes]] = {}
        self._folded = False
        self._capacity = 0
        self._open = False
        self._lock = threading.RLock()
        self._restore_callback = None
        self._keys_loaded = (-1, -1)
        self._ingest: Optional[Ingest] = None  # set once the store is fed raw record batches

    # -- lifecycle (StateStore)
    def name(self) -> str:
        return self._name

    def init(self, context=None, root=None) -> None:
        """Registers the restore callback the way the in-tree example does (context.register(root, (k, v) => ...),
        SingleExceptionThrowingKeyValueStore.scala:84-86)."""
        self._open = True
        self._restore_callback = lambda key, value: self.put_event(key, value)
        if context is not None and hasattr(context, "register"):
            context.register(root, self._restore_callback)

    def persistent(self) -> bool:
        return False

    def isOpen(self) -> bool:  # noqa: N802
        return self._open

    def close(self) -> None:
        with self._lock:
            self._open = False
            if self._dingest is not None:
                self._dingest.close()
            self._engine.close()

    # -- event ingestion
    def _slot(self, aggregate_id: str) -> int:
        i = self._index.get(aggregate_id)
        if i is None:
            i = len(self._keys)
            self._index[aggregate_id] = i
            self._keys.append(aggregate_id)
        return i

    def put_event(self, record_key: Optional[str], packed_event: bytes) -> None:
        """One record of the events topic: key -> aggregate id, value = the model's packed 64-byte event."""
        if not record_key:  # the producer's empty-key flush markers (KafkaProducerActorImpl.scala:321-329) are dropped
            return
        if len(packed_event) != 64:
            raise ValueError("packed events are 64 bytes")
        with self._lock:
            if self._ingest is not None:
                raise N.SgrError(N.SGR_ERR_INVALID, "this store is already fed through restore_record_batches")
            if self._state_topic:
                raise N.SgrError(N.SGR_ERR_INVALID, "this store is fed through put() of state records (its codec has no snapshot rules)")
            rec = np.frombuffer(packed_event, dtype=np.uint8).copy()
            agg_id = aggregate_id_of_record_key(record_key)
            rec[8:16] = np.frombuffer(np.uint64(self._slot(agg_id)).tobytes(), dtype=np.uint8)
            self._pending.append(rec)
            self._unflushed.pop(agg_id, None)   # an event supersedes an unflushed snapshot view

    def restore(self, records: Iterable[Tuple[Optional[str], bytes]]) -> None:
        for k, v in records:
            self.put_event(k, v)
        self.flush()

    def restore_record_batches(self, partition: int, data: bytes, aborted: Sequence[Tuple[int, int]] = ()) -> Dict[str, int]:
        """Raw bytes of one fetch response for `partition` (a concatenation of Kafka RecordBatch v2), plus the
        response's aborted transactions [(producerId, firstOffset)]: decoded natively as a read_committed consumer
        would (SurgeStateStoreConsumer.scala:38) into the pending batch. flush() folds it. A store is fed either this
        way or through put_event, not both (each keeps its own id dictionary).
        A state-topic store (codec without snapshot rules) takes the fetches of the compacted state topic: decoded and applied
        last write wins on the device (DeviceIngest in state-topic mode), fed this way or through put()/delete(), not both."""
        with self._lock:
            if self._state_topic:
                if self._keys:
                    raise N.SgrError(N.SGR_ERR_INVALID, "this store is already fed through put() / delete() of state records")
                if self._dingest is None:
                    from .dingest import DeviceIngest

                    self._dingest = DeviceIngest(self._engine, self._max_ids, 64 * self._max_ids)
                    self._dingest.set_state_topic(True)
                self._dingest.set_aborted(partition, aborted)
                return self._dingest.submit(partition, data)
            if self._keys:
                raise N.SgrError(N.SGR_ERR_INVALID, "this store is already fed through put_event")
            if self._ingest is None:
                self._ingest = Ingest()
            self._ingest.set_aborted(partition, aborted)
            return self._ingest.record_batches(partition, data)

    def committed_offsets(self, partitions: Iterable[int]) -> Dict[int, int]:
        """Per partition, the offset below which every record is inside the state table: what the consumer acting for
        this store commits for the streams application id, so that the producer's lag check
        (KafkaProducerActorImpl.scala:684-708 -> KafkaAdminClient.consumerLag, KafkaAdminClient.scala:44-56) reaches zero
        exactly when get() can serve the state."""
        with self._lock:
            fed = self._dingest if self._dingest is not None else self._ingest
            if fed is None:
                return {int(p): 0 for p in partitions}
            return {int(p): fed.offsets(int(p))[1] for p in partitions}

    def flush(self) -> None:
        with self._lock:
            if self._ingest is not None:
                self._engine.fold_ingested(self._ingest)
                self._folded = True
                self._report_changes()
                return
            if self._dingest is not None:
                self._dingest.fold()
                self._folded = True
                self._report_changes()
                return
            if self._state_topic:
                self._flush_puts()
                return
            if not self._pending and self._folded:
                return
            batch = np.concatenate(self._pending) if self._pending else np.zeros(0, dtype=np.uint8)
            self._pending = []
            n_keys = len(self._keys)
            if not self._folded or n_keys > self._capacity:
                # (re)build: carry the current table into a larger one, then append the batch
                prior = None
                if self._folded:
                    old = self._engine.export_states()
                    self._capacity = max(2 * n_keys, 1024)
                    prior = np.zeros((self._capacity, self._engine.state_bytes), dtype=np.uint8)
                    prior[: len(old)] = old
                else:
                    self._capacity = max(2 * n_keys, 1024)
                    prior = np.zeros((self._capacity, self._engine.state_bytes), dtype=np.uint8)
                self._engine.set_initial_states(prior)
                self._folded = True
            self._engine.fold_incremental(batch)
            if self._keys_loaded != (n_keys, self._capacity):
                self._engine.load_keys(self._keys + [f"\0unused-{i}" for i in range(n_keys, self._capacity)])
                self._keys_loaded = (n_keys, self._capacity)
            self._unflushed.clear()
            self._report_changes()

    def _flush_puts(self) -> None:
        """A state-topic store's flush: every pending record in one sgr_put_batch (the first flush creates the table)."""
        if not self._puts and self._folded:
            return
        puts, self._puts = self._puts, []
        if puts:
            user = self._engine.state_bytes - 8
            rows = np.zeros((len(puts), user), dtype=np.uint8)
            present = np.zeros(len(puts), dtype=bool)
            for i, (_, packed) in enumerate(puts):
                if packed is not None:
                    rows[i, :len(packed)] = np.frombuffer(packed, dtype=np.uint8)
                    present[i] = True
            self._engine.put_batch([k for k, _ in puts], rows, present)
        else:
            self._engine.grow_states(0)   # nothing restored: an empty table, readable
        self._folded = True
        self._unflushed.clear()
        self._report_changes()

    def _report_changes(self) -> None:
        """on_changes for the fold that just ran: its CHANGED and ERROR rows, paged from the device (sgr_export_changes, or
        sgr_export_changes_values with a writer table). Spare capacity slots (ids past the ones this store assigned) never appear."""
        if self._on_changes is None:
            return
        n_ids = None if self._ingest is not None or self._dingest is not None else len(self._keys)
        changed: List[Tuple[str, Optional[bytes]]] = []
        failed: List[Tuple[str, int]] = []
        if self._writer:
            pages = ((idx, flags, err, vals, ids) for idx, flags, err, ids, vals in self._engine.export_changes_values(N.ST_CHANGED | N.ST_ERROR))
        else:
            pages = self._engine.export_changes(N.ST_CHANGED | N.ST_ERROR)
        for idx, flags, err, rows, ids in pages:
            for i, key in enumerate(ids):
                if key is None or (n_ids is not None and idx[i] >= n_ids):
                    continue
                if flags[i] & N.ST_CHANGED:
                    if not flags[i] & N.ST_EXISTS:
                        changed.append((key, None))
                    else:
                        changed.append((key, rows[i] if self._writer else self._decode(key, rows[i].tobytes())))
                if flags[i] & N.ST_ERROR:
                    failed.append((key, int(err[i])))
        self._on_changes(changed, failed)

    # -- KeyValueStore
    def _state_record(self, key: str, value: Optional[bytes]) -> None:
        rec = np.zeros(64, dtype=np.uint8)
        rec[0:4] = np.frombuffer(np.uint32(self._codec.tombstone_type if value is None else self._codec.snapshot_type).tobytes(), dtype=np.uint8)
        rec[8:16] = np.frombuffer(np.uint64(self._slot(key)).tobytes(), dtype=np.uint8)
        if value is not None:
            packed = self._codec.to_packed(key, value)
            if len(packed) > 48:
                raise ValueError("snapshot records carry at most 48 program bytes")
            rec[16:16 + len(packed)] = np.frombuffer(packed, dtype=np.uint8)
        self._pending.append(rec)
        self._unflushed[key] = value

    def _state_put(self, key: str, value: Optional[bytes]) -> None:
        packed = None
        if value is not None:
            packed = self._codec.to_packed(key, value)
            if len(packed) > self._engine.state_bytes - 8:
                raise ValueError(f"the state packs to {len(packed)} bytes; the program holds {self._engine.state_bytes - 8}")
        self._slot(key)
        self._puts.append((key, packed))
        self._unflushed[key] = value

    def put(self, key: str, value: Optional[bytes]) -> None:
        if not key:      # the producer's flush record: empty key, empty value (KafkaProducerActorImpl.scala:321-329)
            return
        with self._lock:
            if self._dingest is not None:
                raise N.SgrError(N.SGR_ERR_INVALID, "this store is already fed through restore_record_batches")
            if self._state_topic:
                self._state_put(key, value)
            elif self._codec is not None:
                self._state_record(key, value)
            else:
                self._overlay[key] = value

    def putIfAbsent(self, key: str, value: bytes) -> Optional[bytes]:  # noqa: N802
        with self._lock:
            cur = self.get(key)
            if cur is None:
                self.put(key, value)
            return cur

    def putAll(self, entries: Sequence[Tuple[str, Optional[bytes]]]) -> None:  # noqa: N802
        for k, v in entries:
            self.put(k, v)

    def delete(self, key: str) -> Optional[bytes]:
        with self._lock:
            cur = self.get(key)
            self.put(key, None)
            return cur

    def get(self, key: str) -> Optional[bytes]:
        if not self._open:
            raise InvalidStateStoreException(N.SGR_ERR_STATE, f"store {self._name} is not open")
        if key in self._overlay:
            return self._overlay[key]
        if key in self._unflushed:            # read-your-writes between put() and flush()
            return self._unflushed[key]
        if not self._folded:
            raise InvalidStateStoreException(N.SGR_ERR_STATE, f"store {self._name} has not been restored yet")
        if self._writer:
            return self._engine.get_many_values([key])[0]
        return self._decode(key, self._engine.get(key))

    def _decode(self, key: str, b: Optional[bytes]) -> Optional[bytes]:
        if b is None:
            return None
        if self._codec is not None:
            return self._codec.from_packed(key, b)
        return self._formatter(key, b) if self._formatter else b

    def get_many(self, keys: Sequence[str]) -> List[Optional[bytes]]:
        """get() for many keys: each key is answered from the overlay, then the unflushed puts, like get(); the rest go to the
        device in one sgr_get_batch call and through the codec / formatter (or, with a writer table, as JSON values from one
        sgr_get_batch_values call)."""
        if not self._open:
            raise InvalidStateStoreException(N.SGR_ERR_STATE, f"store {self._name} is not open")
        keys = list(keys)
        out: List[Optional[bytes]] = [None] * len(keys)
        rest = []
        for i, key in enumerate(keys):
            if key in self._overlay:
                out[i] = self._overlay[key]
            elif key in self._unflushed:
                out[i] = self._unflushed[key]
            else:
                rest.append(i)
        if rest:
            if not self._folded:
                raise InvalidStateStoreException(N.SGR_ERR_STATE, f"store {self._name} has not been restored yet")
            if self._writer:
                for i, v in zip(rest, self._engine.get_many_values([keys[i] for i in rest])):
                    out[i] = v
            else:
                for i, b in zip(rest, self._engine.get_many([keys[i] for i in rest])):
                    out[i] = self._decode(keys[i], b)
        return out

    def all(self) -> Iterator[Tuple[str, bytes]]:
        return self._entries(None, None, decode=True)

    def range(self, frm: str, to: str) -> Iterator[Tuple[str, bytes]]:
        return self._entries(frm, to, decode=True)

    def _entries(self, frm: Optional[str], to: Optional[str], decode: bool) -> Iterator[Tuple[str, Optional[bytes]]]:
        """(id, value) of the live entries with frm <= id <= to (None: that end open) in Bytes order, the order a
        KeyValueStore[Bytes, _] iterates in: unsigned lexicographic over the UTF-8 bytes. The device pages of engine.scan are
        merged with the overlay and the unflushed puts, which answer first as in get(); a None there hides the device row. decode:
        values as get() returns them (with a writer table, the device's JSON values of engine.scan_values), else the packed
        program bytes."""
        lo = None if frm is None else frm.encode("utf-8")
        hi = None if to is None else to.encode("utf-8")

        def inside(kb: bytes) -> bool:
            return (lo is None or lo <= kb) and (hi is None or kb <= hi)

        def check_open():
            if not self._open:
                raise InvalidStateStoreException(N.SGR_ERR_STATE, f"store {self._name} is not open")

        with self._lock:
            host = dict(self._unflushed)
            host.update(self._overlay)
            if not self._open:
                # as the earlier get() per id: a closed store raises at its first id and yields nothing when it holds none
                if host or (self._ingest.keys() if self._ingest is not None else self._keys):
                    check_open()
                return
            folded = self._folded
            # the ids in the engine's key table (a state-topic store's table has no spare slots)
            n_ids = None if self._ingest is not None or self._state_topic else max(self._keys_loaded[0], 0)
            unread = [] if folded else [k for k in (self._ingest.keys() if self._ingest is not None else self._keys) if k not in host]
        hosted = sorted((kb, k, v) for k, v in host.items() if inside(kb := k.encode("utf-8")))
        values = decode and self._writer

        def device() -> Iterator[Tuple[bytes, str, Optional[bytes]]]:
            if not folded:
                # not restored yet: get() of a device id raises. The earlier range() filtered all(), so the first such id raises
                # where it sorts, in the range or not, after the overlay and unflushed entries of the range that sort before it
                for kb, k in sorted((k.encode("utf-8"), k) for k in unread):
                    yield kb, k, None
                    raise InvalidStateStoreException(N.SGR_ERR_STATE, f"store {self._name} has not been restored yet")
                return
            if lo is not None and hi is not None and lo > hi:
                return
            try:
                if values:
                    pages = ((idx, vals, ids) for idx, _, ids, vals in self._engine.scan_values(frm, to))
                else:
                    pages = ((idx, rows, ids) for idx, _, rows, ids in self._engine.scan(frm, to))
                for idx, rows, ids in pages:
                    for i, k in enumerate(ids):
                        if n_ids is None or idx[i] < n_ids:   # spare capacity slots are not this store's ids
                            yield k.encode("utf-8"), k, rows[i] if values else rows[i].tobytes()
            except N.SgrError:
                check_open()   # closed while the iteration ran: what get() raised for the next id
                raise

        dev = device()
        h = 0
        for kb, k, packed in dev:
            while h < len(hosted) and hosted[h][0] < kb:
                check_open()
                if hosted[h][2] is not None:
                    yield hosted[h][1], hosted[h][2]
                h += 1
            check_open()
            if h < len(hosted) and hosted[h][0] == kb:
                if hosted[h][2] is not None:
                    yield k, hosted[h][2]
                h += 1
                continue
            if packed is None:   # (an id of a store that has not been restored: the device iterator raises next)
                continue
            v = self._decode(k, packed) if decode and not values else packed
            if v is not None:
                yield k, v
        for _, k, v in hosted[h:]:
            check_open()
            if v is not None:
                yield k, v

    def restoreAll(self, records: Iterable[Tuple[Optional[str], bytes]]) -> None:  # noqa: N802
        """BatchingStateRestoreCallback.restoreAll(Collection[KeyValue[bytes, bytes]]): Kafka Streams hands the restore
        consumer's polls over in batches; one batch = one GPU fold."""
        self.restore(records)

    def approximateNumEntries(self) -> int:  # noqa: N802
        return sum(1 for _ in self._entries(None, None, decode=False))

    @property
    def engine(self) -> ReplayEngine:
        return self._engine


class AggregateStateStore:
    """The narrow seam PersistentActor consumes (AggregateStateStoreKafkaStreams.scala:83-89):
    getAggregateBytes(aggregateId): Future[Option[Array[Byte]]] served from a 32-thread pool (ThreadPools.scala:9-11).

    coalesce_reads_us > 0: getAggregateBytes calls that arrive within that many microseconds of the first one are answered together
    by one store.get_many (one device call), each future with its own row, or every future of the batch with the batch's
    exception. A node that starts makes one recovery read per aggregate that receives a command; this turns those one-id calls
    into batches without changing the callers. 0 (the default): every call is one store.get on the pool."""

    def __init__(self, store: GpuReplayKeyValueStore, threads: int = 32, coalesce_reads_us: int = 0):
        self._store = store
        self._pool = ThreadPoolExecutor(max_workers=threads, thread_name_prefix="surge-io")
        self._window_s = coalesce_reads_us / 1e6
        self._batch_lock = threading.Lock()
        self._batch: Optional[List[Tuple[str, Future]]] = None   # reads waiting for the open window

    def getAggregateBytes(self, aggregateId: str) -> "Future[Optional[bytes]]":  # noqa: N802,N803
        if self._window_s <= 0:
            return self._pool.submit(self._store.get, aggregateId)
        fut: Future = Future()
        with self._batch_lock:
            opens = self._batch is None
            if opens:
                self._batch = []
            self._batch.append((aggregateId, fut))
        if opens:
            self._pool.submit(self._read_window)
        return fut

    def _read_window(self) -> None:
        time.sleep(self._window_s)
        with self._batch_lock:
            batch, self._batch = self._batch, None
        live = [(k, f) for k, f in batch if f.set_running_or_notify_cancel()]
        if not live:
            return
        try:
            rows = self._store.get_many([k for k, _ in live])
        except BaseException as ex:  # noqa: BLE001 - every caller of the batch sees its failure
            for _, f in live:
                f.set_exception(ex)
            return
        for (_, f), row in zip(live, rows):
            f.set_result(row)

    def getAggregateBytesBatch(self, aggregateIds: Sequence[str]) -> "Future[List[Optional[bytes]]]":  # noqa: N802,N803
        """Recovery reads of many ids in one device call (store.get_many)."""
        return self._pool.submit(self._store.get_many, list(aggregateIds))

    def healthCheck(self) -> dict:  # noqa: N802
        return {"name": "aggregate-state-store", "status": "up" if self._store.isOpen() else "down"}

    def stop(self) -> None:
        self._pool.shutdown(wait=True)
