// GpuReplayPersistencePlugin.scala — the config-selected drop-in behind Surge's state-store seam.
//
//   surge.kafka-streams.state-store-plugin = "gpu-replay"
//   gpu-replay.plugin-class = "surge.gpu.GpuReplayPersistencePlugin"
//
// Implements, without touching SurgeCommand / AggregateRef / SurgeModel:
//   trait SurgeKafkaStreamsPersistencePlugin { def createSupplier(storeName: String): KeyValueBytesStoreSupplier; def enableLogging: Boolean }
//     modules/common/src/main/scala/surge/kafka/streams/SurgeKafkaStreamsPersistencePlugin.scala:12-15
// and returns a KeyValueStore[Bytes, Array[Byte]] shaped like the in-tree example
//     modules/common/src/test/scala/surge/kafka/streams/SingleExceptionThrowingKeyValueStore.scala:18-91.
//
// HOW THE STORE IS FED (the data flow of INTEGRATION.md §1; round-1 review: the previous version parked state records in a JVM
// map and waited for a changelog restore that withLoggingDisabled() guarantees never fires):
//
//   (i)  STATE TOPIC — what Kafka Streams does with this store today. The topology is builder.table(stateTopic, materialized)
//        (SurgeStateStoreConsumer.scala:57-76): the stream thread calls put(aggregateId, serializedState) for every record of
//        the compacted state topic, null = delete (SurgeModel.scala:62-64), then flush() before it commits the offsets of the
//        streams application id. Here put() turns the record into one SNAPSHOT event (or TOMBSTONE) of the registered fold
//        program and flush() folds the batch on the GPU: last write wins per key, exactly the KTable. Because the fold happens
//        inside flush(), the offsets Kafka Streams commits afterwards cover only state that get() can already serve — the lag
//        gate of KafkaProducerActorImpl.scala:684-708 (KafkaAdminClient.consumerLag, KafkaAdminClient.scala:44-56) keeps its
//        meaning with no extra code (SURVEY §8 f2).
//   (ii) EVENTS TOPIC — the rebuild Surge cannot do today (SURVEY §0.2). EventsTopicRebuilder (same package) consumes the events
//        topic with a plain read_committed consumer and calls putEvent(); the same flush() folds events and snapshots in
//        arrival order onto the live table.
//
// The GPU table holds fixed-size packed structs; the topic holds the model's serialized bytes (aggregateWriteFormatting,
// SurgeModel.scala:57-65). A GpuStateCodec registered next to the fold program converts in both directions; a model without one
// cannot use this plugin (sgr_register_program declines it) and keeps the stock RocksDB store.
//
// NOT COMPILED HERE (no JDK / sbt / jars in the build image). The executable twin that the parity tests drive is
// surge_b200/store.py; both are thin adapters over the same C ABI (include/sgr.h).
package surge.gpu

import java.nio.{ ByteBuffer, ByteOrder }
import java.util
import java.util.concurrent.ConcurrentHashMap
import java.util.concurrent.locks.ReentrantReadWriteLock

import org.apache.kafka.common.utils.Bytes
import org.apache.kafka.streams.KeyValue
import org.apache.kafka.streams.errors.InvalidStateStoreException
import org.apache.kafka.streams.processor.{ ProcessorContext, StateStore }
import org.apache.kafka.streams.state.{ KeyValueBytesStoreSupplier, KeyValueIterator, KeyValueStore }
import org.slf4j.LoggerFactory
import surge.kafka.streams.SurgeKafkaStreamsPersistencePlugin

/** serialized state bytes (what the topic and the actors hold) <-> the packed program bytes of the GPU table */
trait GpuStateCodec {

  /** program bytes of the state struct: sgr_fold_program.state_bytes - 8. At most 48 with snapshot rules (one fixed 64-byte
   *  snapshot record carries them at +16); a registration without them (state-topic store, sgr_put_batch) takes up to 120. */
  def programBytes: Int

  /** aggregateReadFormatting.readState, then the packed layout of surge_b200/formats.py for the model */
  def toPacked(aggregateId: String, serialized: Array[Byte]): Array[Byte]

  /** the inverse: aggregateWriteFormatting.writeState of the state the packed bytes stand for */
  def fromPacked(aggregateId: String, packed: Array[Byte]): Array[Byte]
}

/** A model registers the declarative form of its handleEvent once, next to the JVM handler: the fold program (its rules for the
 *  model's event classes PLUS one CREATE+SET rule `snapshotType` that copies program bytes from +16 and one TOMBSTONE rule
 *  `tombstoneType`; surge_b200/dsl.py emits both with `with_snapshot_rules`) and the codec. */
object GpuFoldPrograms {
  /** snapshotType / tombstoneType of a registration without snapshot rules */
  final val NoSnapshotRules = -1
  /** one member of a JSON state writer table (sgr_set_state_writer): kind SGR_JSON_* (0 I32, 1 I64, 2 F64, 3 UUID, 4 PSTR, 5 the
   *  aggregate id), program byte offset, PSTR slot bytes */
  final case class WriterMember(name: String, kind: Int, offset: Int = 0, len: Int = 0)
  final case class Registration(program: ByteBuffer, codec: GpuStateCodec, snapshotType: Int, tombstoneType: Int, writer: Seq[WriterMember] = Nil) {
    /** no snapshot rules: the store takes records of the STATE topic only, applied on the device by sgr_put_batch */
    def stateTopic: Boolean = snapshotType == NoSnapshotRules
  }
  @volatile private var registration: Option[Registration] = None
  def register(packedSgrFoldProgram: ByteBuffer, codec: GpuStateCodec, snapshotType: Int, tombstoneType: Int): Unit = {
    if (snapshotType == NoSnapshotRules || tombstoneType == NoSnapshotRules) {
      require(snapshotType == tombstoneType, "a registration names both the snapshot and the tombstone type, or neither")
      require(codec.programBytes > 0 && codec.programBytes <= 120 && codec.programBytes % 4 == 0, "a state holds at most 120 program bytes")
    } else {
      require(codec.programBytes > 0 && codec.programBytes <= 48 && codec.programBytes % 4 == 0, "snapshot records carry at most 48 program bytes")
    }
    registration = Some(Registration(packedSgrFoldProgram, codec, snapshotType, tombstoneType))
  }
  /** a state-topic store: no snapshot rules, states of any width the engine folds */
  def register(packedSgrFoldProgram: ByteBuffer, codec: GpuStateCodec): Unit =
    register(packedSgrFoldProgram, codec, NoSnapshotRules, NoSnapshotRules)
  /** a state-topic store whose reads, iterators and onChanges take the model's JSON state from the device writer: the codec's
   *  fromPacked is not called (its toPacked still packs what put() receives) */
  def register(packedSgrFoldProgram: ByteBuffer, codec: GpuStateCodec, writer: Seq[WriterMember]): Unit = {
    require(writer.nonEmpty && writer.size <= 32, "a writer table holds 1 to 32 members")
    register(packedSgrFoldProgram, codec, NoSnapshotRules, NoSnapshotRules)
    registration = registration.map(_.copy(writer = writer))
  }
  def current: Registration = registration.getOrElse(throw new IllegalStateException("no GPU fold program registered for this model"))
}

class GpuReplayPersistencePlugin extends SurgeKafkaStreamsPersistencePlugin {
  private val log = LoggerFactory.getLogger(getClass)
  // No changelog: the source topic IS the log of this table (SurgeStateStoreConsumer.scala:63-75 builds the topology
  // withLoggingDisabled() and unoptimised in that case, so every state record reaches put()).
  override def enableLogging: Boolean = false

  override def createSupplier(storeName: String): KeyValueBytesStoreSupplier = {
    // The loader swallows every failure and falls back to RocksDB (SurgeKafkaStreamsPersistencePlugin.scala:34-47):
    // be loud here so a silent fallback is visible in the logs, and fail in the constructor path rather than later.
    GpuFoldPrograms.current
    log.warn(s"GPU replay state store '$storeName' selected; if RocksDB metrics appear the plugin failed to load")
    new KeyValueBytesStoreSupplier {
      override def name(): String = storeName
      override def get(): KeyValueStore[Bytes, Array[Byte]] = new GpuReplayKeyValueStore(storeName)
      override def metricsScope(): String = "gpu-replay"
    }
  }
}

/** onChanges(changed, failed): called once by every flush() that folded, before it returns, with what the reference's actors
 *  would publish for that fold (PersistentActor.scala:252-263): changed = (id, serialized state through the codec, or null for a
 *  state that became None), failed = (id, err_idx) for the aggregates whose handler threw. Rebuilding a state topic from the
 *  events topic produces these records; producing them to Kafka is the caller's. */
class GpuReplayKeyValueStore(storeName: String, onChanges: Option[(Seq[(String, Array[Byte])], Seq[(String, Int)]) => Unit] = None)
    extends KeyValueStore[Bytes, Array[Byte]] {
  private val log = LoggerFactory.getLogger(getClass)
  private val reg = GpuFoldPrograms.current
  private var handle: Long = 0L
  @volatile private var open = false
  // write side: ONE thread (the Kafka Streams stream thread, or the rebuilder's poll thread) — guarded by `lock` against the
  // 32 reader threads of ThreadPools.ioBoundContext that call get()/all()/range()
  private val lock = new ReentrantReadWriteLock()
  private val pending = new java.io.ByteArrayOutputStream()
  private var pendingRecords = 0L
  // a state-topic store's pending records in arrival order: (id, packed program bytes, or null for a tombstone)
  private val statePuts = new util.ArrayList[(String, Array[Byte])]()
  private val keyIndex = new util.HashMap[String, java.lang.Long]() // aggregate id -> dense slot (first-seen order)
  private val keys = new util.ArrayList[String]()
  // read-your-writes between put() and flush(): the not-yet-folded value of a key (None = deleted)
  private val unflushed = new ConcurrentHashMap[String, Option[Array[Byte]]]()
  private var capacity = 0L
  private var folded = false
  private var loadedKeys = -1

  private def check(rc: Int): Unit = if (rc != Native.OK) {
    val msg = Native.lastError(handle)
    if (rc == Native.ERR_STATE) throw new InvalidStateStoreException(msg) else throw new RuntimeException(s"sgr error $rc: $msg")
  }

  override def name(): String = storeName
  // like the in-memory stores of Kafka Streams: nothing on local disk, the table is rebuilt from the topic after a restart
  override def persistent(): Boolean = false
  override def isOpen: Boolean = open

  override def init(context: ProcessorContext, root: StateStore): Unit = {
    handle = Native.create(0) // throws when there is no usable GPU: no CPU fallback, the stream thread dies loudly
    check(Native.registerProgram(handle, reg.program))
    if (reg.writer.nonEmpty) {
      val t = new java.io.ByteArrayOutputStream()
      reg.writer.foreach { m =>
        val name = m.name.getBytes("UTF-8")
        t.write(ByteBuffer.allocate(16).order(ByteOrder.LITTLE_ENDIAN).putInt(m.kind).putInt(m.offset).putInt(m.len).putInt(name.length).array())
        t.write(name)
      }
      val tb = ByteBuffer.allocateDirect(math.max(t.size(), 1)); tb.put(t.toByteArray); tb.flip()
      check(Native.setStateWriter(handle, tb, t.size().toLong, reg.writer.size))
    }
    // The restore callback exists for stores with a changelog (SingleExceptionThrowingKeyValueStore.scala:84-86). This store has
    // none (enableLogging = false), so Kafka Streams never calls it; it is registered because StateStore.init must register the
    // root store, and it does the right thing if a future topology does restore through it.
    context.register(root, (key: Array[Byte], value: Array[Byte]) => put(Bytes.wrap(key), value))
    open = true
  }

  // ---------------------------------------------------------------- write side
  private def slotOf(aggregateId: String): Long = {
    var s = keyIndex.get(aggregateId)
    if (s == null) { s = java.lang.Long.valueOf(keys.size().toLong); keyIndex.put(aggregateId, s); keys.add(aggregateId) }
    s.longValue()
  }

  private def appendRecord(eventType: Int, seq: Int, slot: Long, payload: Array[Byte]): Unit = {
    val rec = ByteBuffer.allocate(64).order(ByteOrder.LITTLE_ENDIAN)
    rec.putInt(0, eventType); rec.putInt(4, seq); rec.putLong(8, slot)
    if (payload != null) { rec.position(16); rec.put(payload, 0, math.min(payload.length, 48)) }
    pending.write(rec.array()); pendingRecords += 1
  }

  /** (i) one record of the STATE topic: KTable semantics, last write wins, null deletes (SurgeStateStoreConsumer.scala:57-76) */
  override def put(key: Bytes, value: Array[Byte]): Unit = {
    val id = new String(key.get(), "UTF-8")
    if (id.isEmpty) return // the producer's flush record: empty key, empty value (KafkaProducerActorImpl.scala:321-329)
    lock.writeLock().lock()
    try {
      if (reg.stateTopic) {
        val packed = if (value == null) null else reg.codec.toPacked(id, value)
        require(packed == null || packed.length <= reg.codec.programBytes, "the packed state is wider than the program's bytes")
        slotOf(id) // (the device numbers new ids in first-appearance order too: keys stays the key table)
        statePuts.add(id -> packed)
      } else if (value == null) appendRecord(reg.tombstoneType, 0, slotOf(id), null)
      else appendRecord(reg.snapshotType, 0, slotOf(id), reg.codec.toPacked(id, value))
      unflushed.put(id, Option(value))
    } finally lock.writeLock().unlock()
  }

  /** (ii) one record of the EVENTS topic: value = the model's packed event (u32 type, u32 seq, payload; formats.py) */
  def putEvent(recordKey: String, packedEvent: Array[Byte]): Unit = if (recordKey != null && recordKey.nonEmpty) {
    require(packedEvent.length >= 8 && packedEvent.length <= 56, "packed event: u32 type, u32 seq, up to 48 payload bytes")
    val id = recordKey.takeWhile(_ != ':') // PartitionStringUpToColon, KafkaPartitioner.scala:38-42
    val b = ByteBuffer.wrap(packedEvent).order(ByteOrder.LITTLE_ENDIAN)
    if (reg.stateTopic) throw new IllegalStateException("this store takes records of the state topic only (no snapshot rules registered)")
    lock.writeLock().lock()
    try {
      appendRecord(b.getInt(0), b.getInt(4), slotOf(id), util.Arrays.copyOfRange(packedEvent, 8, packedEvent.length))
      unflushed.remove(id) // an event supersedes an unflushed snapshot view: readers see the folded table again after flush()
    } finally lock.writeLock().unlock()
  }

  override def putIfAbsent(key: Bytes, value: Array[Byte]): Array[Byte] = { val cur = get(key); if (cur == null) put(key, value); cur }
  override def putAll(entries: util.List[KeyValue[Bytes, Array[Byte]]]): Unit = entries.forEach(kv => put(kv.key, kv.value))
  override def delete(key: Bytes): Array[Byte] = { val cur = get(key); put(key, null); cur }

  /** Kafka Streams calls this before it commits offsets: everything put() so far is folded when it returns. */
  override def flush(): Unit = {
    lock.writeLock().lock()
    try {
      if (reg.stateTopic) { flushPuts(); return }
      if (pendingRecords == 0L && folded) return
      val batch = pending.toByteArray; pending.reset()
      val n = pendingRecords; pendingRecords = 0L
      if (!folded || keys.size() > capacity) growTable()
      if (n > 0) {
        val direct = ByteBuffer.allocateDirect(batch.length); direct.put(batch); direct.flip()
        check(Native.foldIncremental(handle, direct, n))
      }
      if (keys.size() != loadedKeys) loadKeyTable() // new ids inside the current capacity
      unflushed.clear()
      onChanges.foreach(reportChanges)
    } finally lock.writeLock().unlock()
  }

  /** A state-topic store's flush: every pending record in ONE sgr_put_batch, which interns new ids on the device and grows the
   *  table to them; no key table is loaded. */
  private def flushPuts(): Unit = {
    if (statePuts.isEmpty && folded) return
    val n = statePuts.size()
    if (n == 0) check(Native.growStates(handle, 0L)) // nothing to restore: an empty table, readable
    else {
      val user = reg.program.duplicate().order(ByteOrder.LITTLE_ENDIAN).getInt(0) - 8
      val blob = new java.io.ByteArrayOutputStream()
      val offs = ByteBuffer.allocateDirect((n + 1) * 4).order(ByteOrder.LITTLE_ENDIAN)
      val rows = ByteBuffer.allocateDirect(math.max(n * user, 1))
      val present = ByteBuffer.allocateDirect(n)
      offs.putInt(0)
      var i = 0
      while (i < n) {
        val (id, packed) = statePuts.get(i)
        blob.write(id.getBytes("UTF-8")); offs.putInt(blob.size())
        if (packed != null) { rows.position(i * user); rows.put(packed) }
        present.put(i, (if (packed != null) 1 else 0).toByte)
        i += 1
      }
      val kb = ByteBuffer.allocateDirect(math.max(blob.size(), 1)); kb.put(blob.toByteArray); kb.flip(); offs.flip(); rows.clear()
      Native.putBatch(handle, kb, offs, n.toLong, rows, user + 8, present) // throws on failure
      statePuts.clear()
    }
    capacity = keys.size().toLong; loadedKeys = keys.size(); folded = true
    unflushed.clear()
    onChanges.foreach(reportChanges)
  }

  /** The CHANGED and ERROR rows of the fold that just ran, paged from the device (sgr_export_changes); spare capacity slots
   *  (past the ids this store assigned) are left out. */
  private def reportChanges(listener: (Seq[(String, Array[Byte])], Seq[(String, Int)]) => Unit): Unit = {
    val user = reg.program.duplicate().order(ByteOrder.LITTLE_ENDIAN).getInt(0) - 8 // state_bytes is the first field
    val pageRows = 65536
    val cursor = ByteBuffer.allocateDirect(32).order(ByteOrder.LITTLE_ENDIAN)
    val rows = ByteBuffer.allocateDirect(user * pageRows)
    val flags = ByteBuffer.allocateDirect(4 * pageRows).order(ByteOrder.LITTLE_ENDIAN)
    val errs = ByteBuffer.allocateDirect(4 * pageRows).order(ByteOrder.LITTLE_ENDIAN)
    val indices = ByteBuffer.allocateDirect(8 * pageRows).order(ByteOrder.LITTLE_ENDIAN)
    val idOffsets = ByteBuffer.allocateDirect(4 * (pageRows + 1)).order(ByteOrder.LITTLE_ENDIAN)
    val ids = ByteBuffer.allocateDirect(4 << 20)
    val changed = scala.collection.mutable.ArrayBuffer[(String, Array[Byte])]()
    val failed = scala.collection.mutable.ArrayBuffer[(String, Int)]()
    val values = if (writes) ByteBuffer.allocateDirect(16 << 20) else null
    val valueOffsets = if (writes) ByteBuffer.allocateDirect(8 * (pageRows + 1)).order(ByteOrder.LITTLE_ENDIAN) else null
    do {
      val n = (if (writes) Native.exportChangesValues(handle, 2 | 4, cursor, pageRows.toLong, values, valueOffsets, flags, errs, indices, ids, idOffsets)
               else Native.exportChanges(handle, 2 | 4, cursor, pageRows.toLong, rows, flags, errs, indices, ids, idOffsets)).toInt // CHANGED | ERROR
      var i = 0
      while (i < n) {
        val slot = indices.getLong(8 * i)
        if (slot < keys.size()) { // the key table is this store's ids in slot order
          val id = keys.get(slot.toInt)
          val fl = flags.getInt(4 * i)
          if ((fl & 2) != 0) changed += id -> (if ((fl & 1) != 0 && writes) valueAt(values, valueOffsets, i)
          else if ((fl & 1) != 0) {
            val packed = new Array[Byte](user)
            rows.position(i * user); rows.get(packed)
            reg.codec.fromPacked(id, packed)
          } else null)
          if ((fl & 4) != 0) failed += id -> errs.getInt(4 * i)
        }
        i += 1
      }
    } while (cursor.getLong(0) < capacity) // next == n_agg: the export is complete
    listener(changed.toSeq, failed.toSeq)
  }

  /** with a writer table the device writes the model's JSON state (sgr_*_values) and fromPacked is not called */
  private def writes: Boolean = reg.writer.nonEmpty

  /** value i of a page of JSON values (u64 offsets) */
  private def valueAt(values: ByteBuffer, valueOffsets: ByteBuffer, i: Int): Array[Byte] = {
    val lo = valueOffsets.getLong(8 * i).toInt; val hi = valueOffsets.getLong(8 * (i + 1)).toInt
    val v = new Array[Byte](hi - lo)
    values.position(lo); values.get(v)
    v
  }

  /** Make room for the keys seen so far: the table is resized on the device, content kept, new slots None (sgr_grow_states). */
  private def growTable(): Unit = {
    val newCapacity = math.max(2L * keys.size(), 1024L)
    check(Native.growStates(handle, newCapacity))
    capacity = newCapacity
    folded = true
    loadKeyTable()
  }

  /** key table for sgr_get: ids in slot order, unused slots get unreachable placeholder keys */
  private def loadKeyTable(): Unit = {
    val blob = new java.io.ByteArrayOutputStream()
    val offs = ByteBuffer.allocateDirect((capacity.toInt + 1) * 4).order(ByteOrder.LITTLE_ENDIAN)
    offs.putInt(0)
    var i = 0
    while (i < capacity) {
      val bytes = (if (i < keys.size()) keys.get(i) else " unused-" + i).getBytes("UTF-8")
      blob.write(bytes); offs.putInt(blob.size()); i += 1
    }
    val kb = ByteBuffer.allocateDirect(math.max(blob.size(), 1)); kb.put(blob.toByteArray); kb.flip(); offs.flip()
    check(Native.loadKeys(handle, kb, offs, capacity))
    loadedKeys = keys.size()
  }

  // ---------------------------------------------------------------- read side
  /** The recovery read: AggregateStateStoreKafkaStreams.getAggregateBytes ends here (KafkaStreamsKeyValueStore.scala:24-26).
   *  A fresh array every time, as RocksDB returns (SURVEY §8b ownership). */
  override def get(key: Bytes): Array[Byte] = {
    if (!open) throw new InvalidStateStoreException(s"store $storeName is not open")
    val id = new String(key.get(), "UTF-8")
    val u = unflushed.get(id)
    if (u != null) return u.map(_.clone()).orNull
    if (!folded) return null // nothing was ever put: an empty table, not an error (KTable miss)
    if (writes) return getBatch(Seq(key)).head
    val packed = Native.get(handle, key.get()) // null == None; InvalidStateStoreException while the table is being rebuilt
    if (packed == null) null else reg.codec.fromPacked(id, packed)
  }

  /** get() for many keys: unflushed puts answer first, the rest go to the device in one sgr_get_batch call. */
  def getBatch(batch: Seq[Bytes]): Seq[Array[Byte]] = {
    if (!open) throw new InvalidStateStoreException(s"store $storeName is not open")
    val ids = batch.map(k => new String(k.get(), "UTF-8"))
    val out = new Array[Array[Byte]](batch.size)
    val rest = ids.indices.filter { i =>
      val u = unflushed.get(ids(i))
      if (u != null) out(i) = u.map(_.clone()).orNull
      u == null
    }
    if (rest.nonEmpty && folded) {
      val user = reg.program.duplicate().order(ByteOrder.LITTLE_ENDIAN).getInt(0) - 8 // state_bytes is the first field
      val offs = ByteBuffer.allocateDirect(4 * (rest.size + 1)).order(ByteOrder.LITTLE_ENDIAN)
      val blob = new java.io.ByteArrayOutputStream()
      offs.putInt(0)
      rest.foreach { i => blob.write(batch(i).get()); offs.putInt(blob.size()) }
      val kb = ByteBuffer.allocateDirect(math.max(blob.size(), 1)); kb.put(blob.toByteArray); kb.flip(); offs.flip()
      val flags = ByteBuffer.allocateDirect(4 * rest.size).order(ByteOrder.LITTLE_ENDIAN)
      if (writes) {
        val valueOffsets = ByteBuffer.allocateDirect(8 * (rest.size + 1)).order(ByteOrder.LITTLE_ENDIAN)
        var values = ByteBuffer.allocateDirect(64 * rest.size + 64)
        var r = Native.getBatchValues(handle, kb, offs, rest.size.toLong, values, valueOffsets, flags)
        if (r < 0) { values = ByteBuffer.allocateDirect((-r).toInt); r = Native.getBatchValues(handle, kb, offs, rest.size.toLong, values, valueOffsets, flags) }
        rest.zipWithIndex.foreach { case (i, j) => if ((flags.getInt(4 * j) & 1) != 0) out(i) = valueAt(values, valueOffsets, j) }
        return out.toSeq
      }
      val rows = ByteBuffer.allocateDirect(user * rest.size)
      check(Native.getBatch(handle, kb, offs, rest.size.toLong, rows, flags))
      rest.zipWithIndex.foreach { case (i, r) =>
        if ((flags.getInt(4 * r) & 1) != 0) { // SGR_ST_EXISTS
          val packed = new Array[Byte](user)
          rows.position(r * user); rows.get(packed)
          out(i) = reg.codec.fromPacked(ids(i), packed)
        }
      }
    }
    out.toSeq
  }

  /** The live entries in Bytes order (unsigned lexicographic over the UTF-8 bytes) with from <= id <= to (null: that end open):
   *  pages of sgr_scan, pulled from the device as the iterator advances, merged with the unflushed puts, which answer first as
   *  in get() (a deleted one hides the device row). Each page resumes after the last id of the one before, so a fold between two
   *  pages is fine. */
  private def orderedIterator(from: Bytes, to: Bytes): KeyValueIterator[Bytes, Array[Byte]] = {
    if (!open) throw new InvalidStateStoreException(s"store $storeName is not open")
    def inside(b: Bytes) = (from == null || from.compareTo(b) <= 0) && (to == null || b.compareTo(to) <= 0)
    lock.readLock().lock()
    val (host, nIds, deviceReadable) =
      try {
        val m = new util.TreeMap[Bytes, Option[Array[Byte]]]() // Bytes.compareTo is the store order of Kafka Streams
        unflushed.forEach((k, v) => { val b = Bytes.wrap(k.getBytes("UTF-8")); if (inside(b)) m.put(b, v) })
        // the ids the engine's key table names: `keys` runs ahead of it between putEvent() and the end of flush(), and a slot
        // the fold has filled still carries its spare-slot placeholder id until loadKeyTable() has run
        (m.entrySet().toArray(new Array[util.Map.Entry[Bytes, Option[Array[Byte]]]](0)), math.max(loadedKeys, 0).toLong, folded)
      } finally lock.readLock().unlock()
    val user = reg.program.duplicate().order(ByteOrder.LITTLE_ENDIAN).getInt(0) - 8 // state_bytes is the first field
    val pageRows = 4096
    new KeyValueIterator[Bytes, Array[Byte]] {
      private val rows = ByteBuffer.allocateDirect(user * pageRows)
      private val flags = ByteBuffer.allocateDirect(4 * pageRows).order(ByteOrder.LITTLE_ENDIAN)
      private val indices = ByteBuffer.allocateDirect(8 * pageRows).order(ByteOrder.LITTLE_ENDIAN)
      private val idOffsets = ByteBuffer.allocateDirect(4 * (pageRows + 1)).order(ByteOrder.LITTLE_ENDIAN)
      private val ids = ByteBuffer.allocateDirect(1 << 20)
      private val values = if (writes) ByteBuffer.allocateDirect(4 << 20) else null
      private val valueOffsets = if (writes) ByteBuffer.allocateDirect(8 * (pageRows + 1)).order(ByteOrder.LITTLE_ENDIAN) else null
      private val toBytes = if (to == null) null else to.get()
      private var resume: Array[Byte] = if (from == null) null else from.get()
      private var resumeExclusive = false
      private var deviceMore = deviceReadable // an empty table before the first flush, as get() answers
      private val pageKeys = scala.collection.mutable.ArrayBuffer[Bytes]()
      private val pageValues = scala.collection.mutable.ArrayBuffer[Array[Byte]]()
      private var d = 0
      private var h = 0
      private var nextKv: KeyValue[Bytes, Array[Byte]] = _

      private def fillPage(): Unit = while (d >= pageKeys.size && deviceMore) {
        pageKeys.clear(); pageValues.clear(); d = 0
        val r = if (writes) Native.scanValues(handle, resume, resumeExclusive, toBytes, pageRows.toLong, values, valueOffsets, flags, indices, ids, idOffsets)
                else Native.scan(handle, resume, resumeExclusive, toBytes, pageRows.toLong, rows, flags, indices, ids, idOffsets)
        val n = (r >> 1).toInt
        deviceMore = (r & 1) != 0
        var i = 0
        while (i < n) {
          val lo = idOffsets.getInt(4 * i); val hi = idOffsets.getInt(4 * (i + 1))
          val idBytes = new Array[Byte](hi - lo)
          ids.position(lo); ids.get(idBytes)
          if (indices.getLong(8 * i) < nIds) { // spare capacity slots are not this store's ids
            val value = if (writes) valueAt(values, valueOffsets, i) else {
              val packed = new Array[Byte](user)
              rows.position(i * user); rows.get(packed)
              reg.codec.fromPacked(new String(idBytes, "UTF-8"), packed)
            }
            if (value != null) { pageKeys += Bytes.wrap(idBytes); pageValues += value } // a null value is skipped, as get() => null was
          }
          if (i == n - 1) { resume = idBytes; resumeExclusive = true }
          i += 1
        }
      }

      private def advance(): Unit = {
        nextKv = null
        while (nextKv == null) {
          fillPage()
          val dk = if (d < pageKeys.size) pageKeys(d) else null
          val hk = if (h < host.length) host(h).getKey else null
          if (dk == null && hk == null) return
          if (dk == null || (hk != null && hk.compareTo(dk) <= 0)) {
            if (dk != null && hk.equals(dk)) d += 1 // the unflushed value answers for this id
            host(h).getValue.foreach(v => nextKv = new KeyValue(hk, v.clone()))
            h += 1
          } else {
            nextKv = new KeyValue(dk, pageValues(d))
            d += 1
          }
        }
      }
      advance()
      override def hasNext: Boolean = nextKv != null
      override def next(): KeyValue[Bytes, Array[Byte]] = {
        if (nextKv == null) throw new java.util.NoSuchElementException
        val r = nextKv; advance(); r
      }
      override def peekNextKey(): Bytes = { if (nextKv == null) throw new java.util.NoSuchElementException; nextKv.key }
      override def close(): Unit = ()
    }
  }

  override def range(from: Bytes, to: Bytes): KeyValueIterator[Bytes, Array[Byte]] = orderedIterator(from, to)
  override def all(): KeyValueIterator[Bytes, Array[Byte]] = orderedIterator(null, null)

  /** upper bound, like RocksDB's estimate: ids ever seen (deleted ones included until the next rebuild) + unflushed new ones */
  override def approximateNumEntries(): Long = {
    lock.readLock().lock()
    try {
      var n = keys.size().toLong
      unflushed.keySet().forEach(k => if (!keyIndex.containsKey(k)) n += 1)
      n
    } finally lock.readLock().unlock()
  }

  override def close(): Unit = {
    lock.writeLock().lock()
    try { open = false; if (handle != 0L) Native.destroy(handle); handle = 0L }
    finally lock.writeLock().unlock()
    log.info(s"GPU replay state store '$storeName' closed")
  }
}

/** The coalescing reader of surge_b200/store.py AggregateStateStore(coalesce_reads_us > 0): getAggregateBytes calls that arrive
 *  within `windowMicros` of the first one are answered by one getBatch (one device call); each promise gets its own row, or the
 *  batch's exception. The one-id-per-call recovery reads of PersistentActor reach the batch path without a change on their side. */
class CoalescingAggregateReader(store: GpuReplayKeyValueStore, windowMicros: Long)(implicit ec: scala.concurrent.ExecutionContext) {
  private val lock = new Object
  private var waiting: List[(String, scala.concurrent.Promise[Option[Array[Byte]]])] = Nil
  private var open = false

  def getAggregateBytes(aggregateId: String): scala.concurrent.Future[Option[Array[Byte]]] = {
    val p = scala.concurrent.Promise[Option[Array[Byte]]]()
    val first = lock.synchronized { waiting = (aggregateId, p) :: waiting; val f = !open; open = true; f }
    if (first) scala.concurrent.Future {
      Thread.sleep(windowMicros / 1000, ((windowMicros % 1000) * 1000).toInt)
      val batch = lock.synchronized { val b = waiting.reverse; waiting = Nil; open = false; b }
      try {
        val rows = store.getBatch(batch.map { case (id, _) => Bytes.wrap(id.getBytes("UTF-8")) })
        batch.zip(rows).foreach { case ((_, pr), row) => pr.success(Option(row)) }
      } catch { case e: Throwable => batch.foreach { case (_, pr) => pr.failure(e) } }
    }
    p.future
  }
}
