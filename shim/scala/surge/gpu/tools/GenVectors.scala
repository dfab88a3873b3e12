// GenVectors.scala — prints the known-answer vectors this repository could not produce in its build image (no JVM):
//   a8  scala.util.hashing.MurmurHash3.stringHash (scala-library 2.13.8) behind KafkaPartitionProvider.partitionForKey
//       (modules/common/src/main/scala/surge/kafka/KafkaPartitioner.scala:7-9,38-42)
//   a9  the exact bytes play-json 2.9.2 writes for the sample states (modules/surge-docs/src/test/scala/docs/command/
//       BankAccountSurgeModel.scala:26-28; modules/command-engine/core/src/test/scala/surge/core/TestBoundedContext.scala:153-160)
//   a9  stateValues: the same states as rows of the engine's JSON state writer (sgr_set_state_writer) with the bytes play-json
//       writes for them, or "throws" where it refuses (tests/test_gpu_state_values.py compares oracle/state_json.py with them)
//   f1  kafka-clients 3.2.3 MemoryRecords bytes: RecordBatch v2, none / lz4, transactional data batch, control batch
// as one JSON document on stdout:
//
//   scala-cli run --dep com.typesafe.play::play-json:2.9.2 --dep org.apache.kafka:kafka-clients:3.2.3 GenVectors.scala > tests/golden/jvm_vectors.json
//   (or: sbt "surge-common/Test/runMain surge.gpu.tools.GenVectors" from a Surge checkout with this file on the test classpath)
//
// tests/test_jvm_vectors.py consumes the file when it exists (and says "unpinned" loudly when it does not): the day anyone runs
// this on a JVM box, rows a8 / a9 / f1 of SURVEY §8 move from "parity unpinned" to pinned.
package surge.gpu.tools

import java.nio.ByteBuffer
import java.nio.charset.StandardCharsets.UTF_8

import org.apache.kafka.common.record.{ CompressionType, ControlRecordType, EndTransactionMarker, MemoryRecords, MemoryRecordsBuilder, RecordBatch, SimpleRecord, TimestampType }
import play.api.libs.json.{ Json, OFormat }

import scala.util.hashing.MurmurHash3

object GenVectors {
  private def hex(b: Array[Byte]): String = b.map(x => f"${x & 0xff}%02x").mkString
  private def hex(b: ByteBuffer): String = { val a = new Array[Byte](b.remaining()); b.duplicate().get(a); hex(a) }

  // the sample states, as the reference declares them
  final case class State(aggregateId: String, count: Int, version: Int) // core TestBoundedContext.scala:32
  implicit val stateFormat: OFormat[State] = Json.format
  final case class BankAccount(accountNumber: java.util.UUID, accountOwner: String, securityCode: String, balance: Double) // docs BankAccount.scala
  implicit val bankFormat: OFormat[BankAccount] = Json.format

  private def keys: Seq[String] = {
    val rnd = new scala.util.Random(20240923L)
    val ascii = (0 until 400).map(i => s"agg-$i") ++ (0 until 200).map(_ => rnd.alphanumeric.take(1 + rnd.nextInt(40)).mkString)
    val colon = (0 until 150).map(i => s"agg-$i:${rnd.nextInt(1000)}") ++ Seq(":", "a:", ":b", "a:b:c", "")
    val bmp = (0 until 150).map(_ => (0 until (1 + rnd.nextInt(12))).map(_ => (0x00A1 + rnd.nextInt(0x2FFF)).toChar).mkString)
    val astral = (0 until 100).map(_ => (0 until (1 + rnd.nextInt(6))).map(_ => new String(Character.toChars(0x1F300 + rnd.nextInt(0x2FF)))).mkString) // surrogate pairs
    val uuids = (0 until 100).map(_ => new java.util.UUID(rnd.nextLong(), rnd.nextLong()).toString)
    ascii ++ colon ++ bmp ++ astral ++ uuids
  }

  private def batch(compression: CompressionType, baseOffset: Long, records: Seq[SimpleRecord], producerId: Long = RecordBatch.NO_PRODUCER_ID, transactional: Boolean = false): ByteBuffer = {
    val buf = ByteBuffer.allocate(1 << 16)
    val epoch: Short = if (producerId == RecordBatch.NO_PRODUCER_ID) RecordBatch.NO_PRODUCER_EPOCH else 0
    val seq = if (producerId == RecordBatch.NO_PRODUCER_ID) RecordBatch.NO_SEQUENCE else 0
    val b: MemoryRecordsBuilder = MemoryRecords.builder(buf, RecordBatch.MAGIC_VALUE_V2, compression, TimestampType.CREATE_TIME, baseOffset, 1000L, producerId, epoch, seq, transactional, RecordBatch.NO_PARTITION_LEADER_EPOCH)
    records.foreach(b.append)
    b.build().buffer()
  }

  def main(args: Array[String]): Unit = {
    val hashes = keys.map { k =>
      val upTo = k.takeWhile(_ != ':')
      Json.obj("key" -> k, "utf16" -> k.map(_.toInt), "stringHash" -> MurmurHash3.stringHash(k), "stringHashUpToColon" -> MurmurHash3.stringHash(upTo),
        "partitionOf32" -> math.abs(MurmurHash3.stringHash(upTo) % 32), "partitionOf7" -> math.abs(MurmurHash3.stringHash(upTo) % 7))
    }
    val states = Seq(State("a", 0, 0), State("agg-17", 4, 4), State("x", -5, 2147483647), State("é\"\\", Int.MinValue, 1)).map { s =>
      Json.obj("state" -> Json.toJson(s), "bytes_hex" -> hex(Json.toJson(s).toString().getBytes(UTF_8)))
    }
    val accounts = Seq(1100.0, 1000.25, 0.1, -0.0, 1e21, 1e-7, 123456789.125, Double.MinPositiveValue, Double.MaxValue).map { bal =>
      val a = BankAccount(new java.util.UUID(0x0123456789abcdefL, 0x0fedcba987654321L), "Jane Doe", "1234", bal)
      Json.obj("balance_bits" -> java.lang.Double.doubleToRawLongBits(bal).toString, "bytes_hex" -> hex(Json.toJson(a).toString().getBytes(UTF_8)))
    }
    // stateValues: {members: [[name, kind, program offset(, slot bytes)]], row: program bytes hex, id: aggregate id or null,
    // value: play-json's text or "throws"}; kinds as include/sgr.h SGR_JSON_* (0 I32, 2 F64, 3 UUID, 4 PSTR, 5 ID)
    def le(n: Int) = ByteBuffer.allocate(n).order(java.nio.ByteOrder.LITTLE_ENDIAN)
    def pstr(s: String, slot: Int): Array[Byte] = { val b = s.getBytes(UTF_8); val a = new Array[Byte](slot); a(0) = b.length.toByte; System.arraycopy(b, 0, a, 1, b.length); a }
    def written(v: => play.api.libs.json.JsValue): String = try v.toString() catch { case _: Throwable => "throws" }
    val bankMembers = Json.arr(Json.arr("accountNumber", 3, 0), Json.arr("accountOwner", 4, 16, 16), Json.arr("securityCode", 4, 32, 8), Json.arr("balance", 2, 40))
    val bankBalances = Seq(0.0, -0.0, 1100.0, 0.25, -2.5e-7, 1e20, 1.5e21, 1e21, 1.5e-11, 5e-324, 1e-10, 9.999999999999999e-11, 1.7976931348623157e308,
      12.34, -99.99, 0.1, 1e22, 1e23, Double.NaN, Double.PositiveInfinity, Double.NegativeInfinity)
    val bankValues = bankBalances.zipWithIndex.map { case (bal, i) =>
      val u = new java.util.UUID(0x0123456789abcdefL + i, 0x0fedcba987654321L)
      val owner = Seq("Jane Doe", "Zoë", "a\"b\\c", "\u0001\u007f", "日本")(i % 5)
      val r = new Array[Byte](48)
      val ub = ByteBuffer.allocate(16).putLong(u.getMostSignificantBits).putLong(u.getLeastSignificantBits).array()
      System.arraycopy(ub, 0, r, 0, 16)
      System.arraycopy(pstr(owner, 16), 0, r, 16, 16)
      System.arraycopy(pstr((1000 + i).toString, 8), 0, r, 32, 8)
      System.arraycopy(le(8).putDouble(bal).array(), 0, r, 40, 8)
      Json.obj("members" -> bankMembers, "row" -> hex(r), "id" -> play.api.libs.json.JsNull,
        "value" -> written(Json.toJson(BankAccount(u, owner, (1000 + i).toString, bal))))
    }
    val counterMembers = Json.arr(Json.arr("aggregateId", 5), Json.arr("count", 0, 0), Json.arr("version", 0, 4))
    val counterIds = Seq("a", "q\"uote", "back\\slash", "ctl\u0001\u001f\u007f", "tab\tnl\nff\fcr\rbs\b", "zoë", "日本", "\ud83d\ude00", "", "agg-17")
    val counterValues = counterIds.zipWithIndex.map { case (id, i) =>
      val s = State(id, i * 7 - 20, Seq(0, 1, Int.MaxValue, Int.MinValue)(i % 4))
      Json.obj("members" -> counterMembers, "row" -> hex(le(8).putInt(s.count).putInt(s.version).array()), "id" -> id, "value" -> written(Json.toJson(s)))
    }
    def ev(t: Int, seq: Int, by: Int): Array[Byte] = ByteBuffer.allocate(12).order(java.nio.ByteOrder.LITTLE_ENDIAN).putInt(t).putInt(seq).putInt(by).array()
    val recs = (0 until 20).map(i => new SimpleRecord(1000L + i, s"agg-${i % 5}:$i".getBytes(UTF_8), ev(i % 3, i + 1, i * 7 - 3)))
    val flush = new SimpleRecord(1000L, "".getBytes(UTF_8), "".getBytes(UTF_8)) // KafkaProducerActorImpl.scala:321-329
    val control = MemoryRecords.withEndTransactionMarker(40L, 1000L, RecordBatch.NO_PARTITION_LEADER_EPOCH, 77L, 0.toShort, new EndTransactionMarker(ControlRecordType.ABORT, 0)).buffer()
    val batches = Json.obj(
      "none" -> hex(batch(CompressionType.NONE, 0L, recs)),
      "lz4" -> hex(batch(CompressionType.LZ4, 20L, recs)),
      "with_flush_record" -> hex(batch(CompressionType.NONE, 60L, flush +: recs.take(3))),
      "transactional_pid77" -> hex(batch(CompressionType.LZ4, 30L, recs.take(10), producerId = 77L, transactional = true)),
      "abort_marker_pid77" -> hex(control),
      "records" -> recs.map(r => Json.obj("key" -> new String(r.key().array(), UTF_8), "value_hex" -> hex(r.value().array()))))
    println(Json.prettyPrint(Json.obj("scala" -> util.Properties.versionNumberString, "stringHash" -> hashes, "counterStateJson" -> states, "bankAccountJson" -> accounts, "recordBatches" -> batches,
      "stateValues" -> (bankValues ++ counterValues))))
  }
}
