// Native.scala — JNI face of libsgr.so (include/sgr.h). One `external` per C entry point, same order, same meaning.
// NOT COMPILED IN THIS REPOSITORY'S IMAGE (no JDK / sbt / Surge jars); shipped as the binding a maintainer adds
// next to modules/common. The C side of these stubs is shim/jni/sgr_jni.c.
package surge.gpu

import java.nio.ByteBuffer

object Native {
  System.loadLibrary("sgr_jni") // links libsgr.so

  // status codes of include/sgr.h
  final val OK = 0
  final val ERR_STATE = -8 // -> org.apache.kafka.streams.errors.InvalidStateStoreException

  @native def create(device: Int): Long                                            // sgr_create
  @native def destroy(handle: Long): Int                                           // sgr_destroy
  @native def lastError(handle: Long): String                                      // sgr_last_error
  @native def registerProgram(handle: Long, program: ByteBuffer): Int              // sgr_register_program (packed sgr_fold_program)
  @native def loadEvents(handle: Long, events: ByteBuffer, nbytes: Long, segOffsets: ByteBuffer, nAgg: Long): Int // sgr_load_events
  @native def loadUnsorted(handle: Long, records: ByteBuffer, nRecords: Long, nAgg: Long): Int // sgr_load_unsorted
  @native def setInitialStates(handle: Long, states: ByteBuffer, nAgg: Long): Int  // sgr_set_initial_states
  @native def fold(handle: Long): Int                                              // sgr_fold
  @native def foldIncremental(handle: Long, records: ByteBuffer, nRecords: Long): Int // sgr_fold_incremental
  @native def loadKeys(handle: Long, keys: ByteBuffer, keyOffsets: ByteBuffer, nAgg: Long): Int // sgr_load_keys
  /** returns null for None, the program bytes otherwise; throws on a non-OK status */
  @native def get(handle: Long, key: Array[Byte]): Array[Byte]                     // sgr_get
  /** n ids (keys[keyOffsets(i) until keyOffsets(i+1)], u32 offsets) in one device call: row i of `out` = program bytes
   * (stateBytes - 8, zero for None / unknown), flags(i) = SGR_ST_* (0 for an unknown id); returns the status */
  @native def getBatch(handle: Long, keys: ByteBuffer, keyOffsets: ByteBuffer, n: Long, out: ByteBuffer, flags: ByteBuffer): Int // sgr_get_batch
  /** n state-topic records in arrival order (ids as for getBatch): row i = rows[i * (stateBytes - 8), +stateBytes - 8), or a
   * tombstone when present(i) == 0; the last write per id wins on the device. Returns the ids appended to the key table (in
   * first-appearance order); throws InvalidStateStoreException when the key table mirrors an ingest */
  @native def putBatch(handle: Long, keys: ByteBuffer, keyOffsets: ByteBuffer, n: Long, rows: ByteBuffer, stateBytes: Int, present: ByteBuffer): Long // sgr_put_batch
  @native def exportStates(handle: Long, out: ByteBuffer, changedBits: ByteBuffer): Int // sgr_export_states
  /** one page of the rows whose flags meet `select` (SGR_ST_CHANGED = 2 | SGR_ST_ERROR = 4), from the cursor (4 u64: next, token,
   * nKeys, reserved; start with zeros) on: row i = rows (stateBytes - 8), flags(i), errIdx(i), indices(i) and its id
   * ids[idOffsets(i) until idOffsets(i+1)]; the ids buffer's capacity is the page's id-byte budget. Returns the rows written and
   * advances the cursor (next == nAgg: done); throws InvalidStateStoreException when the table changed since the first page */
  @native def exportChanges(handle: Long, select: Int, cursor: ByteBuffer, maxRows: Long, rows: ByteBuffer, flags: ByteBuffer, errIdx: ByteBuffer,
                            indices: ByteBuffer, ids: ByteBuffer, idOffsets: ByteBuffer): Long // sgr_export_changes
  /** one page of the live rows (SGR_ST_EXISTS) whose id lies in [from, to] (null: that end open; fromExclusive leaves from out),
   * in Bytes order of the ids: row i = rows (stateBytes - 8), flags(i), indices(i) and its id ids[idOffsets(i) until
   * idOffsets(i+1)]; the ids buffer's capacity is the page's id-byte budget. Returns 2 * rows written + 1 when a live row in range
   * was left out (continue from the page's last id, exclusive), + 0 when the scan is complete */
  @native def scan(handle: Long, from: Array[Byte], fromExclusive: Boolean, to: Array[Byte], maxRows: Long, rows: ByteBuffer, flags: ByteBuffer,
                   indices: ByteBuffer, ids: ByteBuffer, idOffsets: ByteBuffer): Long // sgr_scan
  /** the JSON state writer (sgr_set_state_writer): per member (little endian) u32 SGR_JSON_* kind (5 = the aggregate id), u32
   *  program byte offset, u32 PSTR slot bytes, u32 name length, the UTF-8 name; nMembers == 0 clears it */
  @native def setStateWriter(handle: Long, table: ByteBuffer, tableBytes: Long, nMembers: Int): Int // sgr_set_state_writer
  /** how the value reads wrap the JSON value: 2 = the JSON itself (default), 3 = the multilanguage protobuf State{aggregateId,
   *  payload = the JSON} a multilanguage store hands the gateway; survives setStateWriter, reset by registerProgram */
  @native def setStateWriterFraming(handle: Long, framing: Int): Int                // sgr_set_state_writer_framing
  /** getBatch with JSON values: value i = values[valueOffsets(i) until valueOffsets(i+1)] (u64 offsets), empty for None / unknown
   *  ids; returns the value bytes written, or -(bytes needed) when values is too small */
  @native def getBatchValues(handle: Long, keys: ByteBuffer, keyOffsets: ByteBuffer, n: Long, values: ByteBuffer, valueOffsets: ByteBuffer,
                             flags: ByteBuffer): Long // sgr_get_batch_values
  /** exportChanges with JSON values in place of rows; the values buffer's capacity is the page's value-byte budget */
  @native def exportChangesValues(handle: Long, select: Int, cursor: ByteBuffer, maxRows: Long, values: ByteBuffer, valueOffsets: ByteBuffer,
                                  flags: ByteBuffer, errIdx: ByteBuffer, indices: ByteBuffer, ids: ByteBuffer, idOffsets: ByteBuffer): Long // sgr_export_changes_values
  /** scan with JSON values in place of rows */
  @native def scanValues(handle: Long, from: Array[Byte], fromExclusive: Boolean, to: Array[Byte], maxRows: Long, values: ByteBuffer,
                         valueOffsets: ByteBuffer, flags: ByteBuffer, indices: ByteBuffer, ids: ByteBuffer, idOffsets: ByteBuffer): Long // sgr_scan_values
  @native def partitionForKey(key: Array[Byte], numPartitions: Int, upToColon: Boolean): Int // sgr_partition_for_key_utf8

  // raw record batches in, committed offsets out (include/sgr.h "ingest")
  @native def ingestCreate(): Long                                                 // sgr_ingest_create
  @native def ingestDestroy(ingest: Long): Int                                     // sgr_ingest_destroy
  @native def ingestSetValueFraming(ingest: Long, framing: Int): Int               // sgr_ingest_set_value_framing (0 packed, 1 protobuf Event, 2 JSON, 3 protobuf Event of JSON)
  /** the JSON member table of framings 2 and 3, little endian: i32 unknownType, u32 length + discriminator, u32 nClasses, per class
   *  u32 length + class name, u32 eventType, u32 nMembers (<= 8), per member u32 kind (SGR_JSON_*), u32 record offset, u32 PSTR
   *  slot bytes, u32 length + member name */
  @native def ingestSetJsonPacker(ingest: Long, table: ByteBuffer, tableBytes: Long): Int // sgr_ingest_set_json_packer
  @native def ingestSetNullValueType(ingest: Long, eventType: Int): Int            // sgr_ingest_set_null_value_type (state-topic tombstones)
  @native def ingestSetAborted(ingest: Long, partition: Int, producerIds: Array[Long], firstOffsets: Array[Long]): Int // sgr_ingest_set_aborted
  /** decodes one fetch response's bytes for `partition`; returns the number of packed records appended; throws on malformed input */
  @native def ingestRecordBatches(ingest: Long, partition: Int, data: ByteBuffer, nbytes: Long): Long // sgr_ingest_record_batches
  @native def foldIngested(handle: Long, ingest: Long): Int                        // sgr_fold_ingested
  @native def growStates(handle: Long, nAgg: Long): Int                            // sgr_grow_states
  /** Array(decodedNext, foldedNext) */
  @native def ingestOffsets(ingest: Long, partition: Int): Array[Long]             // sgr_ingest_offsets

  // the same bytes decoded ON THE DEVICE: only the wire bytes cross PCIe (include/sgr.h "device ingest")
  @native def dingestCreate(handle: Long, maxKeys: Long, maxIdBytes: Long): Long   // sgr_dingest_create (maxIdBytes 0 = 32 per id)
  @native def dingestDestroy(dingest: Long): Int                                   // sgr_dingest_destroy
  @native def dingestSetNullValueType(dingest: Long, eventType: Int): Int          // sgr_dingest_set_null_value_type
  @native def dingestSetValueFraming(dingest: Long, framing: Int): Int             // sgr_dingest_set_value_framing (0 packed, 1 protobuf Event, 2 JSON, 3 protobuf Event of JSON)
  /** as ingestSetJsonPacker; in state-topic mode (set it first) the offsets are program byte offsets */
  @native def dingestSetJsonPacker(dingest: Long, table: ByteBuffer, tableBytes: Long): Int // sgr_dingest_set_json_packer
  @native def dingestSetStateTopic(dingest: Long, on: Int): Int                    // sgr_dingest_set_state_topic (1: compacted state topic, before the first fold)
  @native def dingestSetAborted(dingest: Long, partition: Int, producerIds: Array[Long], firstOffsets: Array[Long]): Int // sgr_dingest_set_aborted
  /** queues one fetch response's bytes (a DIRECT buffer, untouched until dingestFold returns); returns the data batches queued */
  @native def dingestSubmit(dingest: Long, partition: Int, data: ByteBuffer, nbytes: Long): Long // sgr_dingest_submit
  /** CRC, lz4, parse, intern and fold of everything submitted, all or nothing; Array(recordsFolded, newAggregateIds) */
  @native def dingestFold(dingest: Long): Array[Long]                              // sgr_dingest_fold
  /** Array(decodedNext, foldedNext) */
  @native def dingestOffsets(dingest: Long, partition: Int): Array[Long]           // sgr_dingest_offsets
  @native def dingestReset(dingest: Long): Int                                     // sgr_dingest_reset
}
