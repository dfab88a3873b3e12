// SegmentFileRebuilder.scala — rebuilds a GPU state table from the LOG SEGMENT FILES of the events topic (INTEGRATION.md §4).
//
// The public KafkaConsumer hands out deserialized records; the device decoder wants RecordBatch bytes. A partition directory
// holds exactly those: `<baseOffset>.log` is a plain sequence of RecordBatch v2 structures (what a fetch response carries), and
// `<baseOffset>.txnindex` lists the aborted transactions that intersect the segment (34-byte entries: int16 version,
// int64 producerId, int64 firstOffset, int64 lastOffset, int64 lastStableOffset) — what a read_committed consumer
// (modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:38) gets in the fetch response. So a bulk
// rebuild maps the files, announces the aborted transactions and submits the bytes; CRC-32C, lz4, the transaction markers, the
// producer's flush records (modules/command-engine/core/src/main/scala/surge/internal/kafka/KafkaProducerActorImpl.scala:321-329),
// record parsing, id interning and the fold all run on the device (Native.dingest*).
//
// The executable twin is surge_b200/segments.py (tests/test_segments_cpu.py: segment boundaries, chunk cuts, an aborted
// transaction, a preallocated tail, a torn last batch). NOT COMPILED HERE (no JDK / sbt / jars in the build image).
package surge.gpu

import java.io.{ File, RandomAccessFile }
import java.nio.{ ByteBuffer, ByteOrder }
import java.nio.channels.FileChannel
import java.util.zip.CRC32C

import org.slf4j.LoggerFactory

object SegmentFileRebuilder {
  private val SegmentName = """^(\d{20})\.log$""".r
  final case class Segment(baseOffset: Long, log: File, txnIndex: Option[File])
  final case class AbortedTxn(producerId: Long, firstOffset: Long, lastOffset: Long, lastStableOffset: Long)

  def segments(partitionDir: File): Seq[Segment] =
    Option(partitionDir.listFiles()).getOrElse(Array.empty[File]).toSeq.flatMap { f =>
      f.getName match {
        case SegmentName(base) =>
          val tx = new File(partitionDir, base + ".txnindex")
          Some(Segment(base.toLong, f, if (tx.exists()) Some(tx) else None))
        case _ => None
      }
    }.sortBy(_.baseOffset)

  /** a torn tail entry is ignored, like the broker's recovery does */
  def readTxnIndex(f: File): Seq[AbortedTxn] = {
    val raf = new RandomAccessFile(f, "r")
    try {
      val n = (raf.length() / 34).toInt
      (0 until n).map { _ =>
        val version = raf.readShort()
        require(version == 0, s"${f.getName}: aborted-transaction entry version $version")
        AbortedTxn(raf.readLong(), raf.readLong(), raf.readLong(), raf.readLong())
      }
    } finally raf.close()
  }

  /** end (exclusive) of the last whole batch that starts at or after `from`, cut after about `chunkBytes`; `from` if none */
  private def chunkEnd(buf: ByteBuffer, from: Int, limit: Int, chunkBytes: Int): Int = {
    var pos = from
    while (limit - pos >= 12) {
      val length = buf.getInt(pos + 8) // big-endian, like the wire
      if (length <= 0 || pos.toLong + 12 + length > limit) return pos // preallocated zeros / a torn write: not log
      pos += 12 + length
      if (pos - from >= chunkBytes) return pos
    }
    pos
  }

  private def crcHolds(buf: ByteBuffer, begin: Int, end: Int): Boolean = {
    if (end - begin < 61) return false
    val crc = new CRC32C
    val body = buf.duplicate(); body.position(begin + 21); body.limit(end)
    crc.update(body)
    crc.getValue == (buf.getInt(begin + 17) & 0xffffffffL)
  }
}

/** One rebuild of one engine from partition directories `partition -> dir`. Not thread-safe; run it on the thread that owns the
 *  engine's mutating calls (the store's flush lock in GpuReplayKeyValueStore). */
final class SegmentFileRebuilder(engine: Long, maxAggregates: Long, chunkBytes: Int = 64 << 20, pollBytes: Long = 1L << 30,
                                 valueFraming: Int = 0,      // sgr_dingest_set_value_framing: 0 packed, 1 protobuf Event (State)
                                 stateTopic: Boolean = false) { // sgr_dingest_set_state_topic: the partitions hold the compacted state topic
  import SegmentFileRebuilder._
  private val log = LoggerFactory.getLogger(getClass)
  // (JSON needs a member table, which has no JNI binding: checked before the handle exists, so a refusal leaks nothing)
  require(valueFraming == 0 || valueFraming == 1, s"value framing $valueFraming: 0 (packed) or 1 (protobuf Event)")
  private val dingest = Native.dingestCreate(engine, maxAggregates, 0L)
  if (stateTopic) {   // before the first submit: the mode is fixed once a poll was folded
    val rc = Native.dingestSetStateTopic(dingest, 1)
    if (rc != 0) {
      Native.dingestDestroy(dingest)
      throw new IllegalStateException(s"sgr_dingest_set_state_topic failed: $rc")
    }
  }
  if (valueFraming != 0) {
    val rc = Native.dingestSetValueFraming(dingest, valueFraming)
    if (rc != 0) {
      Native.dingestDestroy(dingest)
      throw new IllegalStateException(s"sgr_dingest_set_value_framing($valueFraming) failed: $rc")
    }
  }

  /** decoded == folded position per partition afterwards; returns events folded */
  def rebuild(partitions: Map[Int, File], fromOffsets: Map[Int, Long] = Map.empty): Long = {
    var folded = 0L
    var queued = 0L
    // mapped segments must stay mapped (and untouched) until the fold that consumes them has returned
    var inFlight = List.empty[ByteBuffer]
    def foldNow(): Unit = if (queued > 0) {
      val Array(records, newIds) = Native.dingestFold(dingest)
      folded += records
      log.info(s"rebuild: folded $records records, $newIds new aggregates")
      queued = 0L; inFlight = Nil
    }
    for ((partition, dir) <- partitions.toSeq.sortBy(_._1)) {
      val segs = segments(dir)
      val from = fromOffsets.getOrElse(partition, 0L)
      val needed = segs.zipWithIndex.collect { case (s, i) if i + 1 == segs.size || segs(i + 1).baseOffset > from => s }
      for (seg <- needed) {
        seg.txnIndex.foreach { f =>
          val aborted = readTxnIndex(f)
          if (aborted.nonEmpty) Native.dingestSetAborted(dingest, partition, aborted.map(_.producerId).toArray, aborted.map(_.firstOffset).toArray)
        }
        val ch = FileChannel.open(seg.log.toPath)
        try {
          val size = ch.size()
          require(size <= Int.MaxValue, s"${seg.log}: segments above 2 GiB are not produced by Kafka")
          if (size > 0) {
            val buf = ch.map(FileChannel.MapMode.READ_ONLY, 0, size).order(ByteOrder.BIG_ENDIAN) // a direct buffer
            var limit = size.toInt
            var pos = 0
            var last = false
            while (!last) {
              var end = chunkEnd(buf, pos, limit, chunkBytes)
              last = end == pos || chunkEnd(buf, end, limit, 1) == end
              if (last && (seg eq needed.last) && end > pos) {
                // the active segment may end in a torn write: drop a final batch whose CRC does not hold
                var b = pos; var lastBatch = pos
                while (b < end) { lastBatch = b; b += 12 + buf.getInt(b + 8) }
                if (!crcHolds(buf, lastBatch, end)) end = lastBatch
              }
              if (end > pos) {
                val slice = buf.duplicate(); slice.position(pos); slice.limit(end)
                Native.dingestSubmit(dingest, partition, slice.slice(), (end - pos).toLong)
                inFlight ::= buf
                queued += end - pos
                if (queued >= pollBytes) foldNow()
              }
              pos = end
            }
          }
        } finally ch.close()
      }
    }
    foldNow()
    folded
  }

  /** Array(decodedNext, foldedNext) of a partition after rebuild() */
  def offsets(partition: Int): Array[Long] = Native.dingestOffsets(dingest, partition)
  def close(): Unit = Native.dingestDestroy(dingest)
}
