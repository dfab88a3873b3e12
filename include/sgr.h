/*
 * sgr.h — C ABI of the H100 batched event-replay engine ("surge gpu replay").
 *
 * This is the drop-in boundary for ONE path of UltimateSoftware/surge: rebuilding
 * aggregate state by folding each aggregate's ordered event log through the model's
 * event handler, and the AggregateStateStore recovery read that consumes the result.
 * The reference has no FFI of its own (pure Scala/JVM); each entry point below names
 * the JVM interface a JNI stub would bind it behind (paths relative to the reference
 * checkout, see INTEGRATION.md for the stubs):
 *
 *   CORE  = modules/command-engine/core/src/main/scala/surge
 *   SDSL  = modules/command-engine/scaladsl/src/main/scala/surge/scaladsl
 *   COMMON= modules/common/src/main/scala/surge
 *
 * Conventions
 *   - plain C, no C++/CUDA/torch types cross this boundary;
 *   - every function returns an int32 status (SGR_OK == 0, negative == error class);
 *     the message for the calling thread's last error on an engine is sgr_last_error(engine)
 *     (errno-style, thread-local: concurrent readers never share a message buffer);
 *   - buffers are caller-allocated and caller-owned in both directions; the engine
 *     never frees caller memory and only sgr_destroy frees engine memory;
 *   - "_device" variants take CUDA device pointers on the engine's device and BORROW
 *     them (no copy) — the caller keeps them alive until the next load or destroy;
 *   - load/fold calls are serialised by the caller (the Kafka Streams stream thread in
 *     the reference, COMMON/kafka/streams/KafkaStreamManagerActor.scala:106-133);
 *     sgr_get / sgr_get_index may be called concurrently from many threads (the
 *     reference reads the store from a 32-thread pool,
 *     COMMON/kafka/streams/ThreadPools.scala:9-11).
 *   - there is NO CPU fallback: without a usable CUDA device sgr_create fails.
 */
#ifndef SGR_H
#define SGR_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGR_ABI_VERSION 1

/* ------------------------------------------------------------------ status codes */
#define SGR_OK                 0
#define SGR_ERR_INVALID       -1   /* bad argument / malformed buffer (IllegalArgumentException) */
#define SGR_ERR_NO_DEVICE     -2   /* no CUDA device / extension unusable: fail loudly, never fall back */
#define SGR_ERR_CUDA          -3   /* a CUDA call failed; message carries cudaGetErrorString */
#define SGR_ERR_NO_PROGRAM    -4   /* fold requested before sgr_register_program */
#define SGR_ERR_NOT_LOADED    -5   /* fold/get requested before any load */
#define SGR_ERR_UNSUPPORTED   -6   /* model cannot be expressed as a fold program: decline the plugin */
#define SGR_ERR_OOM           -7
#define SGR_ERR_STATE         -8   /* store not readable now (maps to InvalidStateStoreException,
                                      COMMON/kafka/streams/SurgeAggregateStore.scala:31-46) */
#define SGR_ERR_DIST          -9   /* NCCL / peer-memory failure */
#define SGR_ERR_CAPACITY     -10   /* caller buffer too small */
#define SGR_ERR_AGAIN        -11   /* loopback ranks only: repeat the call on every rank with option "push_ordered" = 1 */

/* ------------------------------------------------------------------ packed formats
 *
 * Fixed record (SGR_REC_FIXED64): 64 bytes, little-endian, 16-byte aligned in the log
 *   +0  u32 type      event type = index into the program's rule table
 *   +4  u32 seq       sequence number (Counter: sequenceNumber)
 *   +8  u64 agg       dense aggregate index (or global index before routing). A program may read it like any
 *                     other bytes, except on a routed engine: there sgr_dist_route_and_fold refuses a program
 *                     with an op reading any of bytes 8..15 (SGR_ERR_UNSUPPORTED), see the multi-GPU block
 *   +16 u8  payload[48]  program-defined view (Counter: i32 by @16;
 *                        BankAccount: uuid @16, f64 balance @32, owner @40, code @56)
 *
 * Variable record (SGR_REC_VAR16): 16-byte header + payload padded to 16 bytes
 *   +0  u32 type   +4 u32 seq   +8 u32 payload_len (unpadded)   +12 u32 agg
 *   +16 payload, padded with zeros up to a multiple of 16
 *   A record is at most 528 bytes (16 + payload_len, before padding) unless option "max_record_bytes" (16..2064,
 *   set before the load) says otherwise; a longer record is a malformed event: the handler throws at it.
 *
 * CSR: u64 seg_offsets[n_agg+1], BYTE offsets into the event log; segment i is
 *   [seg_offsets[i], seg_offsets[i+1]); every offset is a multiple of 16 so that
 *   each segment is a legal source for a 1-D TMA bulk copy.
 *   Fixed records: a segment may start at any multiple of 16, and its whole records fold at their
 *   actual byte positions (seg_offsets[i] + 64*k), whatever the log start or the device address.
 *   A segment whose length is not a multiple of 64 ends in a trailing partial record of 16, 32 or
 *   48 bytes: a malformed event, at which the handler throws — SGR_ST_ERROR, err_idx = the number
 *   of whole records before it, the prior state kept. As for any other throw, n_events counts the
 *   records applied and n_errors counts the aggregate. Option "kernel" 2 and 3 (the record-parallel
 *   kernels) take only logs whose every offset is seg_offsets[0] (mod 64); they refuse any other
 *   with SGR_ERR_UNSUPPORTED, and automatic selection folds it on the lane-sequential kernel.
 *
 * State table: n_agg structs of state_bytes (multiple of 16, <= SGR_MAX_STATE_BYTES).
 *   The program owns bytes [0, state_bytes-8); the engine owns the trailing 8:
 *   +state_bytes-8  u32 flags   (SGR_ST_EXISTS | SGR_ST_CHANGED | SGR_ST_ERROR)
 *   +state_bytes-4  u32 err_idx (index, within the aggregate's batch, of the event that
 *                                threw; 0 when no error)
 *   A state that does not exist (Scala None) has all program bytes zero.
 */
#define SGR_REC_FIXED64 0u
#define SGR_REC_VAR16   1u

#define SGR_ST_EXISTS   1u
#define SGR_ST_CHANGED  2u   /* newState != oldState: the publish rule of
                                CORE/internal/persistence/PersistentActor.scala:252-257 */
#define SGR_ST_ERROR    4u   /* handler threw: state kept at its pre-batch value
                                (PersistentActor.scala:260-263,303-309) */

#define SGR_MAX_STATE_BYTES 128u
#define SGR_MAX_TYPES        16u
#define SGR_MAX_OPS           8u

/* ------------------------------------------------------------------ fold program
 *
 * Declarative form of AggregateCommandModel.handleEvent(Option[Agg], Evt): Option[Agg]
 * (SDSL/command/CommandModels.scala:14). A JVM closure cannot run on a GPU, so a model
 * registers, next to its handler, one rule per event type:
 *
 *   exists_rule   what happens to Option-ness before the field ops run
 *     SGR_IF_EXISTS    None stays None and the ops are skipped   (aggregate.map(_.copy(..)))
 *     SGR_MATERIALISE  None becomes the all-zero default state    (agg.getOrElse(State(id,0,0)))
 *     SGR_CREATE       state is reset to the default, then ops    (Some(Agg(evt fields)))
 *     SGR_TOMBSTONE    state becomes None                          (handler returns None)
 *     SGR_THROW        the handler throws                          (ExceptionThrowingEvent)
 *   ops           word-granular field transfers record -> state, applied in order.
 *                 All offsets/lengths are byte counts and multiples of 4.
 *
 * An event whose type is >= n_types is a scala.MatchError, i.e. SGR_THROW.
 *
 * Instance identity: a rule with field ops, SGR_CREATE, and SGR_MATERIALISE on None build a NEW state instance
 * (Scala constructor / copy); SGR_IF_EXISTS / SGR_MATERIALISE without ops on an existing state hand the same instance
 * back (`current`). The publish rule compares with the case-class equals, which starts with `this eq that`: an
 * aggregate with no events in the fold, or only instance-preserving ones, is never SGR_ST_CHANGED — even if one of its
 * Double fields holds a NaN — while a new instance compares field by field (NaN != NaN, 0.0 == -0.0).
 */
#define SGR_IF_EXISTS    0u
#define SGR_MATERIALISE  1u
#define SGR_CREATE       2u
#define SGR_TOMBSTONE    3u
#define SGR_THROW        4u

#define SGR_OP_SET      0u  /* state[dst .. dst+len) = record[src .. src+len)   (bit copy; f64, strings) */
#define SGR_OP_ADD_I32  1u  /* state.i32[dst] += record.i32[src]   two's-complement wrap (JVM Int)  */
#define SGR_OP_SUB_I32  2u  /* state.i32[dst] -= record.i32[src]                                     */
#define SGR_OP_ADD_I64  3u  /* state.i64[dst] += record.i64[src]   wrap (JVM Long)                    */
#define SGR_OP_SUB_I64  4u

typedef struct sgr_op {
  uint8_t  opcode;     /* SGR_OP_* */
  uint8_t  reserved;
  uint16_t dst_off;    /* byte offset into the state struct (program area) */
  uint16_t src_off;    /* byte offset into the record, header included */
  uint16_t len;        /* bytes; SET: any multiple of 4; I32 ops: 4; I64 ops: 8 */
} sgr_op;

typedef struct sgr_rule {
  uint8_t exists_rule; /* SGR_IF_EXISTS .. SGR_THROW */
  uint8_t n_ops;       /* <= SGR_MAX_OPS */
  uint8_t reserved[6];
  sgr_op  ops[SGR_MAX_OPS];
} sgr_rule;

typedef struct sgr_fold_program {
  uint32_t state_bytes;   /* multiple of 16, 16..SGR_MAX_STATE_BYTES, includes the 8 engine bytes */
  uint32_t record_kind;   /* SGR_REC_FIXED64 | SGR_REC_VAR16 */
  uint32_t n_types;       /* <= SGR_MAX_TYPES */
  uint32_t n_f64_fields;  /* <= 8: state fields that are JVM Doubles; they are bit-copied by SGR_OP_SET
                             but compare with == for the publish rule (0.0 == -0.0, NaN != NaN), as
                             Scala case-class equality does in PersistentActor.scala:257 */
  uint16_t f64_field_off[8];
  sgr_rule rules[SGR_MAX_TYPES];
} sgr_fold_program;

/* ------------------------------------------------------------------ engine */
typedef struct sgr_engine sgr_engine;   /* opaque */

typedef struct sgr_config {
  int32_t  device;          /* CUDA device ordinal */
  uint32_t flags;           /* reserved, 0 */
  uint64_t reserved[6];
} sgr_config;

typedef struct sgr_stats {
  uint64_t n_aggregates;    /* segments folded by the last fold */
  uint64_t n_events;        /* events consumed by the last fold */
  uint64_t event_bytes;     /* stored event-record bytes read by the last fold */
  uint64_t algorithmic_bytes;/* event_bytes + 8*(n_agg+1) + state_bytes*n_agg (+ prior states read) */
  uint64_t n_errors;        /* aggregates whose handler threw */
  uint64_t n_long_segments; /* always 0 (kept for ABI layout; no fold skips long segments) */
  float    ms_h2d;          /* host->device copy of the last load (0 for _device loads) */
  float    ms_group;        /* stable group-by of the last unsorted load */
  float    ms_fold;         /* device time of the last fold (all its kernels); a record-parallel fold queued behind a
                               fold of the same log (sgr_fold_async) overlaps it and is timed from its first CTA's entry
                               to its last warp's exit by %globaltimer, every other fold by CUDA events around it */
  float    ms_d2h;          /* device->host copy of the last export */
  uint32_t fold_launches;   /* kernels launched by the last fold */
  uint32_t reserved[7];
} sgr_stats;

int32_t sgr_abi_version(void);

/* Create an engine bound to one CUDA device. Replaces the construction of the state
 * store inside the engine pipeline (CORE/internal/domain/SurgeMessagePipeline.scala:68-78). */
int32_t sgr_create(const sgr_config* cfg, sgr_engine** out);
int32_t sgr_destroy(sgr_engine* e);
const char* sgr_last_error(const sgr_engine* e);   /* e may be NULL: last create error */

/* Register the declarative form of the model's event handler
 * (SDSL/command/CommandModels.scala:14; core entry
 * CORE/internal/domain/AggregateProcessingModel.scala:21). */
int32_t sgr_register_program(sgr_engine* e, const sgr_fold_program* prog);

/* Load a CSR-ordered event log (host buffers; copied to HBM). The log is what
 * AggregateRef.applyEvents would be handed per aggregate, for every aggregate at once
 * (SDSL/common/AggregateRefBaseTrait.scala:23-28). */
int32_t sgr_load_events(sgr_engine* e, const void* events, uint64_t nbytes,
                        const uint64_t* seg_offsets, uint64_t n_agg);
int32_t sgr_load_events_device(sgr_engine* e, const void* d_events, uint64_t nbytes,
                               const uint64_t* d_seg_offsets, uint64_t n_agg);

/* Variable records with a record directory: rec_offsets[n_records+1] are the byte offsets of every record in log order
 * (the packer knows them for free). With it the log is cut into record-balanced spans, so skewed (Zipf) keys do not
 * serialise one lane; without it (sgr_load_events) variable records are folded one lane per aggregate. */
int32_t sgr_load_events_indexed(sgr_engine* e, const void* events, uint64_t nbytes, const uint64_t* seg_offsets, uint64_t n_agg,
                                const uint64_t* rec_offsets, uint64_t n_records);
int32_t sgr_load_events_indexed_device(sgr_engine* e, const void* d_events, uint64_t nbytes, const uint64_t* d_seg_offsets,
                                       uint64_t n_agg, const uint64_t* d_rec_offsets, uint64_t n_records);

/* Load records in ARRIVAL order (a Kafka partition log interleaves aggregates) and group
 * them, stably, by aggregate index into CSR form on the device. n_agg is the number of
 * dense aggregate indices (records carry agg < n_agg). Fixed 64-byte records only. */
int32_t sgr_load_unsorted(sgr_engine* e, const void* records, uint64_t n_records, uint64_t n_agg);
int32_t sgr_load_unsorted_device(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_agg);

/* Rebuild every state from an arrival-order log in one call (the shape of a Kafka partition log: aggregates
 * interleaved, each aggregate's own order kept), without exposing a CSR log afterwards. Programs inside the
 * transformer algebra with add-only / set-only words need no grouping at all (integer-atomic fold); others are grouped
 * and folded as sgr_load_unsorted + sgr_fold would. */
int32_t sgr_fold_unsorted(sgr_engine* e, const void* records, uint64_t n_records, uint64_t n_agg);
int32_t sgr_fold_unsorted_device(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_agg);

/* Prior states for an incremental fold (None everywhere if never called):
 * the actor's state before ApplyEvents, PersistentActor.scala:245-264. states may be NULL to reset. */
int32_t sgr_set_initial_states(sgr_engine* e, const void* states, uint64_t n_agg);

/* Fold every aggregate's segment left to right in event order:
 * events.foldLeft(state)(handleEvent), SDSL/command/CommandModels.scala:25-28. */
int32_t sgr_fold(sgr_engine* e);

/* The same fold without host synchronisation: sgr_fold_async enqueues the kernels on the engine's
 * stream and returns; sgr_wait blocks until they finish and collects the statistics. Any call that
 * reads results (get/export/stats) waits implicitly. */
int32_t sgr_fold_async(sgr_engine* e);
int32_t sgr_wait(sgr_engine* e);

/* Append one micro-batch (arrival order, fixed records) to the live state table: group by
 * aggregate, fold onto the current states, write back (PersistentActor.doApplyEvent on a
 * live actor, PersistentActor.scala:245-264). Requires a prior fold or set_initial_states. */
int32_t sgr_fold_incremental(sgr_engine* e, const void* records, uint64_t n_records);
int32_t sgr_fold_incremental_device(sgr_engine* e, const void* d_records, uint64_t n_records);

/* Key table: UTF-8 aggregate ids, key i = keys[key_offsets[i] .. key_offsets[i+1]).
 * Not read by the fold; only by sgr_get. */
int32_t sgr_load_keys(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n_agg);

/* Point lookup of folded state bytes by aggregate id: the recovery read
 * AggregateStateStoreKafkaStreams.getAggregateBytes(aggregateId): Future[Option[Array[Byte]]]
 * (COMMON/kafka/streams/AggregateStateStoreKafkaStreams.scala:83-85). *exists == 0 is None.
 * Thread-safe against a published snapshot. Copies the program bytes (state_bytes-8). */
int32_t sgr_get(sgr_engine* e, const uint8_t* key, uint32_t klen,
                void* out, uint32_t cap, uint32_t* outlen, int32_t* exists);
int32_t sgr_get_index(sgr_engine* e, uint64_t agg, void* out, uint32_t cap,
                      uint32_t* outlen, int32_t* exists, uint32_t* flags, uint32_t* err_idx);

/* Recovery reads of many aggregate ids in one call, served from the device table (getAggregateBytes for a batch).
 * Key i = keys[key_offsets[i] .. key_offsets[i+1]). Row i of `out` (state_bytes-8 bytes) = program bytes of key i,
 * all zero when the state is None or the id is unknown. flags (optional, n x u32): the state's SGR_ST_* flags, 0 for an
 * unknown id. indices (optional, n x i64): dense index, or -1 for an unknown id.
 * Answers what sgr_get / sgr_get_index answer for each id, from the same key table (sgr_load_keys, or the ids an ingest
 * appended). The ids are looked up in an index on the device, extended by the first call after ids are appended (only the new
 * ids are uploaded) and rebuilt after sgr_load_keys or a new ingest; the host snapshot of sgr_get is not used. The call holds
 * the engine's operation lock throughout and waits for an sgr_fold_async first: every row of a batch comes from one table
 * generation, and batch readers serialise (one call should carry many ids). SGR_ERR_STATE before any fold; SGR_ERR_INVALID on
 * non-monotone key_offsets or a duplicate id in the key table; SGR_ERR_CAPACITY (nothing written) when
 * cap < n * (state_bytes - 8); SGR_ERR_UNSUPPORTED on a routed engine without a current rank key table (sgr_dist_load_keys),
 * whose rows are local slots. n == 0 is a no-op. */
int32_t sgr_get_batch(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n,
                      void* out, uint64_t cap, uint32_t* flags, int64_t* indices);

/* Keyed state writes: a batch of state-topic records applied to the table on the device, the KTable a state topic restores
 * (SurgeStateStoreConsumer.scala:57-76: last write wins per key, a null value deletes, SurgeModel.scala:62-64).
 * Record i, in arrival order: id keys[key_offsets[i] .. key_offsets[i+1]) (any bytes, "" included), and either the row
 * rows + i * (state_bytes - 8) (the program bytes) or, when present[i] == 0, a tombstone (its row is not read).
 * The table ends as if each record had been folded in order as a snapshot event (SGR_CREATE + SET of every program byte) or a
 * SGR_TOMBSTONE event: the last record per id decides its row. A row gets SGR_ST_EXISTS and its own bytes; a tombstone leaves
 * None (program bytes zero, no EXISTS). SGR_ST_CHANGED compares the end state with the state before the batch, field by
 * field, as a new instance: Double fields with == (NaN is never equal to itself, 0.0 == -0.0), the rest bitwise. So
 * snap(x), tomb, snap(x) on an existing x is not CHANGED, nor is a tombstone of a None state. The rows the batch writes have
 * SGR_ST_ERROR and err_idx cleared. The call is a fold for everything scoped to the last fold: the rows it does not write lose
 * CHANGED and ERROR, the generation advances (an export in progress ends with SGR_ERR_STATE; sgr_get snapshots are refreshed).
 * Ids: known ids are looked up in the device id index of sgr_get_batch. New ids get dense indices n_keys, n_keys + 1, ... in
 * order of first appearance in the batch (a tombstone of an unknown id is one too, with a None row), are inserted into that
 * index and appended to the key table sgr_get / sgr_get_batch / sgr_export_changes / sgr_scan read, and the table grows to
 * hold them (new rows None, as sgr_grow_states). *n_new_ids (optional): the ids appended. Works for every program (16 to 128
 * byte states, FIXED64 or VAR16 records: rows are states, not records), and on an engine without a table, which it creates.
 * Key table: one of sgr_load_keys, one built by earlier put batches, or none. SGR_ERR_STATE (nothing applied) when it mirrors
 * an ingest's id dictionary (sgr_fold_ingested, the device ingest, sgr_append_keys), which numbers new ids itself;
 * SGR_ERR_UNSUPPORTED on a routed engine (sgr_dist_init), with or without a rank key table: a new id would need a global
 * aggregate index and an owner, which only the partition table can give.
 * All or nothing: SGR_ERR_INVALID on NULL arguments, non-monotone key_offsets or a duplicate id in the key table;
 * SGR_ERR_CAPACITY when the key table would reach 2^32 - 1 ids or pass 4 GiB of id bytes; SGR_ERR_UNSUPPORTED for n >= 2^32;
 * n == 0 is a no-op. Holds the operation lock and waits for an sgr_fold_async, as sgr_get_batch does. */
int32_t sgr_put_batch(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n,
                      const void* rows, const uint8_t* present, uint64_t* n_new_ids);

/* Changed-state export: the aggregates the last fold changed (SGR_ST_CHANGED, "newState != oldState") or failed (SGR_ST_ERROR,
 * the handler threw and the state was kept), with their ids, compacted on the device and handed over in pages: what the
 * reference's actors publish to the state topic after a poll (PersistentActor.scala:252-263), without copying the whole table.
 * select: a non-empty subset of SGR_ST_CHANGED | SGR_ST_ERROR; a row is reported when flags & select != 0.
 * A page holds the selected rows in ascending dense index from cur->next on, at most max_rows of them and at most ids_cap id
 * bytes; cur->next comes back as the first selected row that did not fit, or n_agg when the scan reached the end. Row i of the
 * page: rows[i] (state_bytes - 8 bytes; all zero for a None state, the tombstone case CHANGED without EXISTS), flags[i],
 * err_idx[i], indices[i] (its dense index) and its id ids[id_offsets[i] .. id_offsets[i+1]) from the key table sgr_get /
 * sgr_get_batch read. A row at or past cur->n_keys has no id: a zero-length span, told apart from the id "" by its index.
 * Buffers: rows max_rows x (state_bytes - 8), flags / err_idx max_rows x u32, indices max_rows x i64, id_offsets max_rows + 1
 * u32, ids ids_cap bytes (NULL when ids_cap == 0); *n_rows = the rows written.
 * One export is one table generation: start with cur = {0}; the first page records the generation and the key-table epoch in
 * cur->token and later pages pass it back. After any fold, grow or sgr_set_initial_states, or sgr_load_keys or a new ingest
 * owner, a later page fails with SGR_ERR_STATE and writes nothing. Appended ids and reads do not end an export.
 * Holds the operation lock and waits for an sgr_fold_async, as sgr_get_batch does. SGR_ERR_STATE before any fold;
 * SGR_ERR_INVALID on NULL arguments, a bad select, max_rows == 0 or cur->next > n_agg; SGR_ERR_CAPACITY (nothing written,
 * the cursor unchanged) when the first selected row's id alone exceeds ids_cap; SGR_ERR_UNSUPPORTED on a routed engine
 * without a current rank key table (sgr_dist_load_keys), whose rows are local slots. */
typedef struct sgr_changes_cursor {
  uint64_t next;     /* in/out: first dense index not yet reported; 0 starts an export; n_agg when the export is complete */
  uint64_t token;    /* in/out: 0 on the first page; the engine sets it and later pages pass it back */
  uint64_t n_keys;   /* out: size of the key table the page was read against */
  uint64_t reserved;
} sgr_changes_cursor;
int32_t sgr_export_changes(sgr_engine* e, uint32_t select, sgr_changes_cursor* cur, uint64_t max_rows, void* rows,
                           uint32_t* flags, uint32_t* err_idx, int64_t* indices, uint8_t* ids, uint64_t ids_cap,
                           uint32_t* id_offsets, uint64_t* n_rows);

/* Ordered scan of the live table: the rows whose state exists (SGR_ST_EXISTS), in Bytes order of their aggregate ids (unsigned
 * lexicographic over the UTF-8 bytes, a prefix before any longer id), whose id lies in [from, to]: Kafka Streams'
 * KeyValueStore.range / all over the store's Bytes keys, served from the table on the device.
 * Bounds: from == NULL is no lower bound; a non-NULL from with from_len 0 is the id "", which from_exclusive != 0 leaves out
 * (from_exclusive drops the id equal to from, whatever it is). to == NULL is no upper bound; to is inclusive. from > to gives an
 * empty page.
 * A page holds, from the lower bound on, at most max_rows rows and at most ids_cap id bytes. Row i of the page: rows[i]
 * (state_bytes - 8 program bytes), flags[i] (SGR_ST_*; EXISTS is always set, ERROR when the last fold's handler threw and kept
 * the state), indices[i] (its dense index) and its id ids[id_offsets[i] .. id_offsets[i+1]). *n_rows = the rows written; *more
 * = 1 exactly when a live row in range was left out of the page.
 * Pages carry no cursor: the caller continues with the page's last id as from and from_exclusive = 1. Each page is read against
 * one table generation (the call holds the operation lock and waits for an sgr_fold_async, as sgr_get_batch does), but the
 * pages of one scan may come from different generations when folds run between them. An id live at both ends of such a scan
 * is reported exactly once; one created or deleted in between may or may not appear.
 * Rows: the ids of the key table sgr_get_batch reads (sgr_load_keys, or the ids an ingest appended). Rows at or past n_agg,
 * rows without SGR_ST_EXISTS and rows past the key table never appear. The order lives on the device next to the id index
 * and is brought up to date by the first scan after the key table changes: appended ids are sorted and merged in, a replaced
 * key table is ordered again.
 * Buffers: rows max_rows x (state_bytes - 8), flags max_rows x u32 (optional), indices max_rows x i64 (optional), id_offsets
 * max_rows + 1 u32, ids ids_cap bytes (NULL when ids_cap == 0).
 * SGR_ERR_STATE before any fold; SGR_ERR_INVALID on NULL buffers, max_rows == 0 or a duplicate id in the key table;
 * SGR_ERR_CAPACITY (nothing written) when the first row's id alone exceeds ids_cap; SGR_ERR_UNSUPPORTED on a routed engine
 * without a current rank key table (sgr_dist_load_keys), whose rows are local slots, and for tables of 2^32 - 1 rows or more. */
int32_t sgr_scan(sgr_engine* e, const uint8_t* from, uint32_t from_len, int32_t from_exclusive, const uint8_t* to, uint32_t to_len,
                 uint64_t max_rows, void* rows, uint32_t* flags, int64_t* indices, uint8_t* ids, uint64_t ids_cap,
                 uint32_t* id_offsets, uint64_t* n_rows, int32_t* more);

/* Export the whole state table (n_agg * state_bytes) and, optionally, bitmaps
 * (bit i of byte i/8, LSB first). Any out pointer may be NULL. */
int32_t sgr_export_states(sgr_engine* e, void* out, uint64_t cap,
                          uint8_t* exists_bits, uint8_t* changed_bits, uint8_t* error_bits);
/* Device pointer to the live state table (borrowed; valid until the next load/destroy). */
int32_t sgr_states_device(sgr_engine* e, void** d_states, uint64_t* n_agg, uint32_t* state_bytes);
/* Device pointers to the engine's CSR event log (after any load). */
int32_t sgr_events_device(sgr_engine* e, void** d_events, uint64_t* nbytes, uint64_t** d_seg_offsets);

int32_t sgr_get_stats(sgr_engine* e, sgr_stats* out);

/* Tuning knob for measurements: which fold kernel variant to launch
 * (0 = default; see DESIGN.md "kernel variants"). */
int32_t sgr_set_option(sgr_engine* e, const char* name, int64_t value);

/* The CUDA stream (cudaStream_t) the engine launches on, so callers can record events. */
int32_t sgr_stream(sgr_engine* e, void** stream);

/* Measurement probe (scripts/fold_ceiling.py): enqueue on `stream` one launch that stages `bytes` of the device buffer
 * `buf` into shared memory the way the default record-parallel fold does, and does nothing else. Warps take fixed
 * spans (ticketed = 0) or chunks of chunk_bytes by ticket (ticketed = 1); ctl: 2 device u64, zero before the launch. */
int32_t sgr_probe_read(const void* buf, uint64_t bytes, int32_t ticketed, uint64_t chunk_bytes, void* ctl, void* stream);

/* ------------------------------------------------------------------ multi-GPU (one process per GPU, one node)
 * Aggregates are hash-partitioned across ranks exactly as Surge shards them across nodes
 * (aggregateId -> partition -> owner): partition_of_agg[g] is
 * KafkaPartitionProvider.partitionForKey of global aggregate g (COMMON/kafka/KafkaPartitioner.scala:7-9)
 * and the owner rank is partition % nranks. Each rank feeds the records of ITS source partitions in arrival
 * order (records carry the GLOBAL aggregate index at +8); one exchange over NVLink replaces the broker
 * shuffle (KafkaProducerHelperCommon.getPartitionFor, COMMON/kafka/KafkaProducer.scala:45-57). */
typedef struct sgr_dist_stats {
  uint64_t n_sent, n_sent_remote, n_recv, n_local_aggregates;
  float ms_count, ms_counts_exchange, ms_scatter, ms_exchange, ms_group, ms_fold;
  float ms_pipeline;               /* fused >= 2: device time of the whole overlapped route + exchange + fold */
  uint32_t exchange_record_bytes;  /* bytes per record that crossed NVLink (64, or the projected size with fused == 3) */
  uint32_t reserved[4];
} sgr_dist_stats;

int32_t sgr_dist_unique_id(void* out128);                       /* rank 0: a 128-byte NCCL unique id to hand to the others */
int32_t sgr_dist_init(sgr_engine* e, int32_t rank, int32_t nranks, const void* unique_id128,
                      uint64_t recv_capacity_records);
int32_t sgr_dist_set_partitions(sgr_engine* e, const uint32_t* partition_of_agg, uint64_t n_global_agg);
/* fused path: every rank exports its receive buffer (64-byte CUDA IPC handle), the host exchanges the
 * handles, every rank imports all nranks of them (own slot ignored). */
int32_t sgr_dist_ipc_export(sgr_engine* e, void* out64);
int32_t sgr_dist_ipc_import(sgr_engine* e, const void* handles64_by_rank);
/* Route + exchange + (group-by) + fold.
 *   fused == 0  count + pack, one NCCL all-to-all (grouped ncclSend/ncclRecv), then the fold;
 *   fused == 1  count, then the route kernel writes each record straight into its owner's receive buffer over NVLink;
 *   fused == 2  ONE pass, pipelined: the log is cut into chunks (option "push_chunks", the same on every rank); a push kernel
 *               partitions each chunk in shared memory and writes every owner's run contiguously into that owner's receive
 *               region over NVLink, an arrival flag per (source, chunk) follows, and the owner folds chunk c while chunk c+1 is
 *               still in flight. No count pass, no send buffer, no host synchronisation inside. Needs the peers' receive buffers
 *               (IPC import) and a program in the sort-free class (16-byte state, class 0, every word add-only or set-only) —
 *               other programs silently take fused == 1. Receive regions have a fixed capacity of
 *               recv_capacity / (nranks * push_chunks) records per (source, chunk): a region that would overflow fails the call
 *               with SGR_ERR_CAPACITY on EVERY rank (nothing is written out of bounds); retry with fused <= 1 or more capacity.
 *               Option "push_pull" (default 1): the source partitions into ITS OWN buffer and the owner's fold reads those
 *               regions over NVLink (remote loads: only the 32-byte sectors the fold touches cross the link); 0: the source
 *               writes into the owner's buffer (remote stores). By default a CTA takes its place inside a region with one
 *               atomicAdd per owner and every record carries its index within the chunk, which is the only order the
 *               sort-free fold needs; when any rank meets a throwing aggregate (the exact replay wants positional log order)
 *               every rank repeats the exchange in ordered mode (decoupled look-back) — automatically on real ranks, by
 *               SGR_ERR_AGAIN + option "push_ordered" on loopback ranks.
 *   fused == 3  as 2, but only the record words the fold program reads cross NVLink (u32 local index + slot words:
 *               16 bytes per record for the Counter model); a program that reads more than 7 record words (event type
 *               included) is refused with SGR_ERR_UNSUPPORTED, use fused == 2.
 * On a routed engine (nranks > 1, or option "force_route") what arrives in a record's aggregate field depends on the mode (the
 * owner's local index, the record's index within its chunk, or the global index), so a program with an op that reads any of
 * record bytes 8..15 is refused with SGR_ERR_UNSUPPORTED on every rank, before anything is launched or exchanged. */
int32_t sgr_dist_route_and_fold(sgr_engine* e, const void* d_records, uint64_t n_records, int32_t fused);
/* Several ranks inside ONE process on one device ("loopback", for single-GPU tests of the multi-rank logic): sgr_dist_init with
 * unique_id128 == NULL and nranks > 1 creates such a rank; the ranks hand each other their receive allocation as plain device
 * pointers (sgr_dist_recv_base -> sgr_dist_set_peers) and the caller runs every rank's sgr_dist_route_and_fold(fused >= 2)
 * concurrently (one host thread per rank), with a barrier of its own between calls. fused <= 1 needs NCCL and is refused.
 * The ranks' streams share the device's hardware queues, so inside the call each loopback rank enqueues all of its partition
 * and flag kernels, then waits on the host for its peers to do the same (at most 60 s, else SGR_ERR_DIST), and only then
 * enqueues the kernels that wait for arrival flags: a waiting kernel never stands in a queue ahead of a flag it waits for. */
int32_t sgr_dist_recv_base(sgr_engine* e, void** base);
/* Allocate everything sgr_dist_route_and_fold(fused >= 2) needs for logs of up to max_records records now (after
 * sgr_dist_set_partitions and the "push_chunks" option), so that the call itself allocates nothing. Optional for real ranks;
 * loopback ranks share one device, where an allocation can wait for another rank's kernel: call it on every rank first. */
int32_t sgr_dist_reserve(sgr_engine* e, uint64_t max_records);
int32_t sgr_dist_set_peers(sgr_engine* e, void* const* recv_bases_by_rank);
/* 64-bit order-independent hash of the live state table: sum over slots of mix(aggregate index, state bytes) mod 2^64, the
 * index being the GLOBAL aggregate index on a routed engine — so the sum of the ranks' hashes does not depend on how many ranks
 * there are. The parity check of the multi-GPU runs (bench.py, tests/test_gpu_dist.py; twin: surge_b200/dist.py states_hash). */
int32_t sgr_states_hash(sgr_engine* e, uint64_t* out);
int32_t sgr_dist_get_stats(sgr_engine* e, sgr_dist_stats* out);
/* global aggregate index of each local state slot (host copy, n_local u32) */
int32_t sgr_dist_local_aggregates(sgr_engine* e, uint32_t* out, uint64_t cap, uint64_t* n_local);
/* The key table of a routed rank: keys[key_offsets[g] .. key_offsets[g+1]) is the id of GLOBAL aggregate g, for every g of the
 * partition table (n_global == the n_global_agg of sgr_dist_set_partitions). The engine keeps the ids of the aggregates this
 * rank owns, in local-slot order: id i of the rank's key table is that of global aggregate sgr_dist_local_aggregates()[i].
 * Each Surge node answers getAggregateBytes, range and all from the KTable partitions it owns; with this table a rank does the
 * same from its rows. sgr_get, sgr_get_batch(_values), sgr_export_changes(_values), sgr_scan(_values) and sgr_set_state_writer
 * then serve the rank as they serve one engine, over the rank's rows: a dense index is a local slot (the row order of
 * sgr_export_states), and an id another rank owns is unknown, as a KTable miss is. After sgr_dist_route_and_fold every row is
 * flagged, so sgr_export_changes(SGR_ST_CHANGED | SGR_ST_ERROR) pages the rank's share of a republished state topic.
 * The ids are gathered on the host and installed as sgr_load_keys installs a table: ingest ids are dropped, the key-table
 * epoch advances (an export in progress ends with SGR_ERR_STATE) and the device id index and id order are rebuilt by the
 * next read. The table stays current until sgr_dist_init, sgr_dist_set_partitions, sgr_load_keys, sgr_append_keys or an
 * ingest replaces it; after that the reads are refused again until this call is repeated.
 * The partition table is the caller's contract: when it disagrees with KafkaPartitionProvider.partitionForKey of the ids, a
 * rank holds ids the router would never send it.
 * SGR_ERR_NOT_LOADED before sgr_dist_init and sgr_dist_set_partitions; SGR_ERR_INVALID (the key table unchanged) on NULL
 * arguments, non-monotone key_offsets, n_global different from the partition table's size, or two equal ids among the ones
 * this rank owns (as sgr_load_keys). sgr_put_batch and the state-topic mode of the device ingest stay refused on a routed
 * engine: they number new ids themselves, which a partition table cannot hold. */
int32_t sgr_dist_load_keys(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n_global);

/* ------------------------------------------------------------------ ingest: Kafka record batches -> packed records (SURVEY §8 f1, f2)
 * What feeds the store today is a Kafka consumer in read_committed mode
 * (COMMON/kafka/streams/SurgeStateStoreConsumer.scala:38; the plain wrapper is COMMON/kafka/KafkaConsumer.scala:48-105,120-132)
 * over a topic whose producer compresses with lz4 (modules/common/src/main/resources/reference.conf:124) and writes inside
 * transactions. sgr_ingest decodes the raw bytes of a fetch response / log segment — a concatenation of RecordBatch
 * (magic 2) structures — into the engine's fixed 64-byte records in arrival order, interning aggregate ids
 * (key.takeWhile(_ != ':'), COMMON/kafka/KafkaPartitioner.scala:38-42) as dense indices in first-seen order.
 *   - verifies each batch's CRC-32C; decodes compression none and lz4 (gzip/snappy/zstd: SGR_ERR_UNSUPPORTED);
 *   - skips control batches, and data batches of aborted transactions announced with sgr_ingest_set_aborted
 *     (the fetch response's abortedTransactions list), the way a read_committed consumer does;
 *   - drops records with a null/empty key: the producer's flush markers
 *     (CORE/internal/kafka/KafkaProducerActorImpl.scala:321-329);
 *   - a trailing partial batch is left undecoded (n_trailing_bytes), as fetch responses may end with one;
 *   - records below the partition's decoded position are counted as duplicates and skipped (refetch after restart);
 *   - record value = the model's packed event: u32 type, u32 seq (little endian) + up to 48 payload bytes — as is, inside the
 *     multilanguage protobuf Event, or produced from a flat JSON object by a registered member table (sgr_ingest_set_value_framing).
 * A malformed batch fails the whole call and leaves the pending log and the partition position untouched.
 * The RecordBatch framing is third-party (org.apache.kafka:kafka-clients:3.2.3) and the reference holds no broker bytes:
 * its byte-level parity is UNPINNED (see oracle/kafka_batch.py); lz4, xxHash32, CRC-32C and the protobuf framing are pinned
 * against real implementations.
 *
 * Lag gate (f2): actors trust the store only once the consumer group of the streams applicationId has no lag
 * (CORE/internal/kafka/KafkaProducerActorImpl.scala:530-540,684-708; COMMON/kafka/KafkaAdminClient.scala:36-56).
 * sgr_ingest_offsets reports, per partition, the next offset to fetch (decoded_next) and the offset below which every
 * record is inside the state table (folded_next) — the value whoever consumes on the store's behalf commits. */
typedef struct sgr_ingest sgr_ingest;

typedef struct sgr_ingest_stats {
  uint64_t n_bytes;              /* bytes consumed (whole batches) */
  uint64_t n_trailing_bytes;     /* bytes of a trailing partial batch left undecoded (last call only) */
  uint64_t n_batches;
  uint64_t n_records;            /* packed records appended to the pending log */
  uint64_t n_markers;            /* null/empty-key records dropped */
  uint64_t n_null_values;        /* keyed records with a null value: dropped, or turned into tombstone events
                                    (sgr_ingest_set_null_value_type) */
  uint64_t n_control_batches;
  uint64_t n_aborted_batches, n_aborted_records;
  uint64_t n_duplicates;         /* records below the partition's decoded position */
  uint64_t n_new_keys;
  uint64_t n_compressed_bytes, n_decompressed_bytes;
  uint64_t reserved[3];
} sgr_ingest_stats;

int32_t sgr_ingest_create(sgr_ingest** out);
int32_t sgr_ingest_destroy(sgr_ingest* g);
const char* sgr_ingest_last_error(const sgr_ingest* g);
/* How the record value wraps the packed event. SGR_VALUE_PACKED (default): the value IS `u32 type, u32 seq, payload`.
 * SGR_VALUE_PROTOBUF_EVENT: the value is the multilanguage module's protobuf `Event { string aggregateId = 1; bytes payload = 2; }`
 * (modules/multilanguage-protocol/src/main/protobuf/multilanguage-protocol.proto:17-20, written by
 * modules/multilanguage/src/main/scala/com/ukg/surge/multilanguage/GenericSurgeCommandBusinessLogic.scala:30-33) and the packed
 * event is its payload. The framing is pinned against the protobuf runtime in tests/test_ingest_cpu.py. */
#define SGR_VALUE_PACKED          0
#define SGR_VALUE_PROTOBUF_EVENT  1
#define SGR_VALUE_JSON            2
int32_t sgr_ingest_set_value_framing(sgr_ingest* g, int32_t framing);

/* SGR_VALUE_JSON: the value is a flat JSON object as the reference's sample models write their events with play-json,
 * e.g. {"_type":"...CountIncremented","aggregateId":"a","incrementBy":1,"sequenceNumber":4}
 * (modules/command-engine/core/src/test/scala/surge/core/TestBoundedContext.scala:44-56 formats, :159-161 writer).
 * The model registers the discriminator member, the event type index of each class name and where each numeric member
 * lands in the packed record (record byte offsets: 4 = the sequence number, 16..63 = payload). Members are found by name —
 * order, whitespace and extra members do not matter; with an empty discriminator exactly one class is registered and every
 * value is that class (a state topic: Json.toJson(agg) carries no discriminator); an unknown class name becomes event type `unknown_type` (a
 * scala.MatchError in the handler) or, with -1, fails the call. Doubles are parsed correctly rounded (strtod), as
 * java.lang.Double.parseDouble does. The exact bytes play-json writes are NOT pinned (no JVM here); the parser is checked
 * against Python's json module on both well-formed and hostile input. */
#define SGR_JSON_I32  0u
#define SGR_JSON_I64  1u
#define SGR_JSON_F64  2u
#define SGR_JSON_UUID 3u   /* "8-4-4-4-12" string (java.util.UUID.toString) -> 16 bytes, most significant first */
#define SGR_JSON_PSTR 4u   /* string -> length byte + UTF-8 bytes, zero padded to `len` bytes (must fit: len - 1 bytes at most) */
#define SGR_JSON_MAX_FIELDS 8u
typedef struct sgr_json_field { const char* name; uint8_t kind; uint8_t reserved; uint16_t dst_off; uint32_t len; /* PSTR slot */ } sgr_json_field;
typedef struct sgr_json_event {
  const char* type_name;     /* value of the discriminator member */
  uint32_t event_type;       /* index into the fold program's rules */
  uint32_t n_fields;
  sgr_json_field fields[SGR_JSON_MAX_FIELDS];
} sgr_json_event;
int32_t sgr_ingest_set_json_packer(sgr_ingest* g, const char* discriminator, const sgr_json_event* events, uint32_t n_events,
                                   int32_t unknown_type);
/* Compacted STATE topic (what the reference restores from today, COMMON/kafka/streams/SurgeStateStoreConsumer.scala:57-76): a keyed
 * record with a null value deletes the key (CORE/internal/SurgeModel.scala:62-64). With event_type >= 0 such a record becomes an
 * event of that type (the program's SGR_TOMBSTONE rule) instead of being dropped; -1 (default) drops it. */
int32_t sgr_ingest_set_null_value_type(sgr_ingest* g, int32_t event_type);
/* The id dictionary holds at most 2^31 ids and 4 GiB of id bytes (32-bit fields). A call that could exceed a bound fails with
 * SGR_ERR_CAPACITY before anything is applied (every id of the call is counted as new: conservative). Lower bounds can be set
 * to fail earlier (operators; tests). */
int32_t sgr_ingest_set_dictionary_limits(sgr_ingest* g, uint64_t max_ids, uint64_t max_id_bytes);
/* aborted transactions of the next fetch of `partition`: (producerId, firstOffset) pairs */
int32_t sgr_ingest_set_aborted(sgr_ingest* g, int32_t partition, const int64_t* producer_ids, const int64_t* first_offsets, uint64_t n);
int32_t sgr_ingest_record_batches(sgr_ingest* g, int32_t partition, const void* data, uint64_t nbytes, sgr_ingest_stats* stats);
/* n fetches in one call. CRC, decompression and parsing run on up to `threads` host threads (the fetches of one partition
 * stay on one thread, in call order); ids are interned and records appended afterwards in call order, so the outcome is
 * identical to n single calls. All or nothing: one malformed fetch and nothing is applied. stats: n entries or NULL. */
int32_t sgr_ingest_record_batches_mt(sgr_ingest* g, uint32_t n, const int32_t* partitions, const void* const* datas,
                                     const uint64_t* nbytes, uint32_t threads, sgr_ingest_stats* stats);
/* Where the pending log lives (default malloc/free). sgr_fold_ingested installs page-locked host memory so that the copy of
 * a poll to the device is one DMA at full PCIe rate; content already pending is carried over. */
int32_t sgr_ingest_set_allocator(sgr_ingest* g, void* (*alloc_fn)(size_t), void (*free_fn)(void*));
/* the pending packed records (borrowed until the next ingest call) and the id dictionary (key i = dense index i) */
int32_t sgr_ingest_pending(sgr_ingest* g, const void** records, uint64_t* n_records);
int32_t sgr_ingest_keys(sgr_ingest* g, const uint8_t** keys, const uint32_t** key_offsets, uint64_t* n_keys);
/* the pending records are inside the state table now: drop them, advance folded_next to decoded_next */
int32_t sgr_ingest_mark_folded(sgr_ingest* g);
int32_t sgr_ingest_offsets(sgr_ingest* g, int32_t partition, int64_t* decoded_next, int64_t* folded_next);
int32_t sgr_ingest_get_stats(sgr_ingest* g, sgr_ingest_stats* out);   /* totals since create */

/* Resize the live state table to n_agg slots on the device, keeping its content; new slots are None.
 * (A KTable grows as new keys appear; never shrinks.) */
int32_t sgr_grow_states(sgr_engine* e, uint64_t n_agg);
/* Fold everything pending in `g` onto the live table (growing it for new aggregate ids), publish the id dictionary
 * to sgr_get, and mark the ingest folded: poll -> sgr_ingest_record_batches -> sgr_fold_ingested is the whole restore loop. */
int32_t sgr_fold_ingested(sgr_engine* e, sgr_ingest* g);

/* Append ids to the key table sgr_get reads: the ids of dense indices [n, n + n_new) where n is the number of ids `owner` has
 * appended so far (a different owner starts a new table). owner is an opaque tag: the id dictionary the table mirrors. */
int32_t sgr_append_keys(sgr_engine* e, const void* owner, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n_new);

/* ------------------------------------------------------------------ device ingest: the same decode ON THE GPU
 * Same input (raw bytes of fetch responses, RecordBatch magic 2, compression none / lz4, read_committed semantics) and the same
 * outcome as sgr_ingest_* + sgr_fold_ingested, but only the WIRE bytes cross PCIe: CRC-32C, lz4, record parsing, id interning and
 * the fold run on the engine's device (csrc/dingest_kernels.cu); the host walks the 61-byte batch headers and keeps the
 * read_committed bookkeeping (control batches, aborted transactions, partition positions). csrc/ingest.cpp is its checker
 * (tests/test_gpu_dingest.py: identical states, ids, offsets and statistics on the same bytes).
 *   - value framing: as the host ingest's (sgr_dingest_set_value_framing, sgr_dingest_set_json_packer): the packed event, the
 *     protobuf Event's payload or a flat JSON object through a registered member table, converted inside the parse kernel with
 *     the host decoder's results and refusal texts ("offset N, record r: JSON event: unknown event class"). Both settings survive
 *     sgr_dingest_reset and are refused with SGR_ERR_STATE between a submit and its fold. JSON compresses better than packed
 *     values: under protobuf / JSON framing a poll that needed the exact-layout repeat raises the arena claim for the next polls
 *     (to the power of two at or above the ratio it showed, at most 16x the wire bytes);
 *   - every fixed-record program is accepted. Dropped records (flush markers, duplicates, null values without a tombstone type)
 *     stay in place as holes. Sort-free programs skip the holes in the atomic fold; the others group the live records on the
 *     device first (K5, holes left out), at one extra pass over the poll's records. err_idx counts the aggregate's live events of
 *     the poll, as the host decoder does. For those others a poll whose records were all dropped folds nothing and leaves the
 *     last fold's flags, as the host decoder does; a sort-free program runs its fold and clears them. All or nothing covers
 *     refusals before the fold (corruption, dictionary full); an error inside the fold itself (a CUDA failure, a replay-list
 *     overflow) can leave the previous poll's CHANGED / ERROR flags already cleared;
 *   - dense indices are stable per id but follow no arrival-order promise (they come from an atomic counter);
 *   - polls are processed in groups of SGR_DINGEST_GROUP (default 8192) batches, each group one chain of launches on one of eight
 *     streams; batches decompress into an arena of 3x the wire bytes (a poll that compresses better is decoded a second time from
 *     an exact layout — correct, slower); SGR_DINGEST_TIMING=1 prints each group's device timeline to stderr;
 *   - the id dictionary is sized at creation: max_keys ids, max_id_bytes id bytes (0 = 32 per id); exceeding either fails the
 *     poll with SGR_ERR_CAPACITY and applies nothing;
 *   - a refused poll applies nothing to the table, the positions or the statistics, but ids it interned stay in the device
 *     dictionary (they count against max_keys, and the next good poll reports them in n_new_keys);
 *   - after SGR_ERR_CAPACITY the dictionary holds at most max_keys ids in at most max_id_bytes id bytes, and each of them is an
 *     id that arrived; a later poll of ids it holds folds as usual, and a poll with an id it did not admit fails again, until
 *     sgr_dingest_reset;
 *   - refusals follow the host decoder, which checks each batch in the order Kafka's consumer does: the CRC-32C first (a damaged
 *     batch is SGR_ERR_INVALID whatever else it claims); a batch of an aborted transaction is then skipped unread (its codec is
 *     not looked at, it is not decompressed); any other batch is SGR_ERR_UNSUPPORTED for a codec other than none / lz4, control
 *     batches included. A batch entirely below the partition's position is decoded and checked like any other, its records
 *     counting as duplicates. A control batch may be lz4-compressed; its marker is read after decompression. The order holds
 *     per batch: in a fetch with several bad batches the device may report the header-level refusal of a later batch (magic,
 *     codec, length) where the host reports the content error (CRC, lz4, records) of an earlier one. Either way nothing of the
 *     poll is applied;
 *   - inside a batch, a refused record (malformed, its value refused by the framing, outside 8..56 bytes, id too long) is
 *     reported as the host reports it: the batch's lowest such record, with the host's reason ("offset N, record r: ..."),
 *     whichever record the device happened to check first. The record walk (a record length that runs past the batch, stray
 *     bytes after the last record, a recordsCount that does not fit) runs over the whole batch before any record is parsed,
 *     so a batch with a walk error AND an earlier refused record gets the walk's reason on the device and that record's on
 *     the host, which checks record by record. The code (SGR_ERR_INVALID) is the same and nothing is applied.
 * poll loop:  sgr_dingest_set_aborted* -> sgr_dingest_submit(partition, bytes)* -> sgr_dingest_fold.
 * `data` of a submit must stay valid until the fold returns (with page-locked memory the copy is one asynchronous DMA). */
typedef struct sgr_dingest sgr_dingest;
int32_t sgr_dingest_create(sgr_engine* e, uint64_t max_keys, uint64_t max_id_bytes, sgr_dingest** out);
int32_t sgr_dingest_destroy(sgr_dingest* g);
const char* sgr_dingest_last_error(const sgr_dingest* g);
int32_t sgr_dingest_set_null_value_type(sgr_dingest* g, int32_t event_type);
/* as sgr_ingest_set_value_framing / sgr_ingest_set_json_packer, validated alike; SGR_ERR_STATE while a poll is pending */
int32_t sgr_dingest_set_value_framing(sgr_dingest* g, int32_t framing);          /* SGR_VALUE_PACKED | _PROTOBUF_EVENT | _JSON */
int32_t sgr_dingest_set_json_packer(sgr_dingest* g, const char* discriminator, const sgr_json_event* events,
                                    uint32_t n_events, int32_t unknown_type);
/* Decode a compacted STATE topic instead of an events topic (on != 0; 0 goes back to events). The reference recovers by having
 * Kafka Streams restore the state topic into a KTable (SurgeStateStoreConsumer.scala:57-76): key = the aggregate id as written
 * (SurgeModel.scala:64), value = the serialized state, null deletes, the last write per key wins.
 * When: SGR_ERR_STATE while a poll is pending, after any successful fold since create or sgr_dingest_reset (one dictionary and
 * one set of positions belong to one topic), and once a JSON member table is registered (its offsets mean different things in
 * the two modes: set the mode first). SGR_ERR_UNSUPPORTED on a routed engine (sgr_dist_init), with or without a rank key
 * table, as sgr_put_batch: the restore numbers new ids itself. The mode
 * survives sgr_dingest_reset, as the value framing does.
 * Records: everything a read_committed consumer does stays as in events mode (CRC first, control batches, aborted
 * transactions, a trailing partial batch, duplicates below the partition's position, the positions of the lag gate). Then:
 *   - the id is the WHOLE key, with no cut at ':' (shorter than 2^24 bytes);
 *   - a null or empty key is the producer's flush marker: dropped, counted in n_markers. (The reference's KTable would hold
 *     an entry for the empty key written by the producer's flush record, KafkaProducerActorImpl.scala:321-329; here it stays
 *     a dropped marker, as everywhere in this library);
 *   - a null value is a tombstone, counted in n_null_values and in n_records; sgr_dingest_set_null_value_type has no effect;
 *   - any other value, after its framing, gives the row's program bytes: SGR_VALUE_PACKED, the value itself, 0 to
 *     state_bytes - 8 bytes, zero-padded; SGR_VALUE_PROTOBUF_EVENT, the payload of the multilanguage
 *     `State { string aggregateId = 1; bytes payload = 2; }` (Event's field numbers); SGR_VALUE_JSON, the members of the
 *     registered table at PROGRAM byte offsets;
 *   - a framed value longer than state_bytes - 8 is refused: "offset N, record r: state value of L bytes is longer than the
 *     P program bytes of a row (state_bytes - 8)";
 *   - n_records counts the live records: rows plus tombstones.
 * JSON member table in this mode (sgr_dingest_set_json_packer, with a program registered): an empty discriminator and exactly
 * one class (Json.toJson(state) writes no discriminator; its event_type and unknown_type are ignored); each member needs
 * dst_off % 4 == 0, a size that is a multiple of 4 and at least 4, and dst_off + size <= state_bytes - 8, else SGR_ERR_INVALID.
 * Apply: the poll is one sgr_put_batch over its live records in arrival order (submission order, then batch order, then record
 * order): the last record per id decides its row (EXISTS with its bytes, or None for a tombstone); CHANGED compares with the
 * state before the poll (Double fields with ==, the rest bitwise); the rows written have ERROR and err_idx cleared; rows the
 * poll does not write lose CHANGED and ERROR; the generation advances and the rows written are what the next operation clears;
 * an unknown id, one seen only in a tombstone included, gets a None row; the table grows to hold new ids. Dense indices come
 * from the device dictionary, with no first-appearance promise; new ids reach the key table as in events mode, so sgr_get,
 * sgr_get_batch, sgr_export_changes and sgr_scan read them. Every program works: 16- to 128-byte states, FIXED64 or VAR16.
 * All or nothing as an events poll: a refusal applies nothing to the table, the positions or the statistics. A poll whose
 * records were all dropped applies nothing to the table and leaves the last fold's flags (as an n == 0 put batch); its
 * positions still advance. Slot [4] of sgr_dingest_last_timing is table growth + the apply. */
int32_t sgr_dingest_set_state_topic(sgr_dingest* g, int32_t on);
int32_t sgr_dingest_set_aborted(sgr_dingest* g, int32_t partition, const int64_t* producer_ids, const int64_t* first_offsets, uint64_t n);
int32_t sgr_dingest_submit(sgr_dingest* g, int32_t partition, const void* data, uint64_t nbytes, sgr_ingest_stats* stats);
/* decode + intern + fold everything submitted since the last fold onto the engine's live table (grown as ids appear), publish
 * the new ids to sgr_get, advance the partitions' positions. All or nothing. stats (optional): this poll's totals. */
int32_t sgr_dingest_fold(sgr_dingest* g, sgr_ingest_stats* stats);
int32_t sgr_dingest_offsets(sgr_dingest* g, int32_t partition, int64_t* decoded_next, int64_t* folded_next);
/* Forget everything (dictionary, partition positions, statistics): the next poll starts a rebuild from offset 0 with dense
 * indices from 0. The engine's table is the caller's to reset (sgr_set_initial_states(e, NULL, 0)). */
int32_t sgr_dingest_reset(sgr_dingest* g);
/* host-clock milliseconds of the last sgr_dingest_fold: [0] wait for the copies and for every group's chain (CRC, lz4 decode +
 * record walk, record parse + id interning — launched by the submits behind the copies), [1] a repeat from an exact arena
 * layout when the arena claims were too small (normally 0), [2] unused, [3] launch of the new ids' gather and download,
 * [4] table growth + fold, with the ids handed to the key table by a helper thread meanwhile, [5] the whole call. */
int32_t sgr_dingest_last_timing(sgr_dingest* g, float* ms8);
int32_t sgr_dingest_get_stats(sgr_dingest* g, sgr_ingest_stats* out);

/* ------------------------------------------------------------------ state values: rows written as the model's JSON state
 * The store's reads and the records a republish produces are the model's serialized state (getAggregateBytes; the state topic's
 * value, aggregateWriteFormatting.writeState, SurgeModel.scala:57-65). With a writer table the engine writes that value on the
 * device, as Json.toJson(state) writes a case class of flat members: {"name":value,...}, members in table order, no whitespace
 * (csrc/state_writer.h; restatement oracle/state_json.py):
 *   SGR_JSON_I32 / _I64  plain decimal;  SGR_JSON_UUID  8-4-4-4-12 lowercase hex, most significant byte first;
 *   SGR_JSON_PSTR        a string of the slot's first length-byte bytes (padding ignored);
 *   SGR_JSON_F64         the shortest decimal that rounds back to the double (Python's repr digits, Double.toString's from
 *                        JDK 19 on), trailing zeros stripped, plain for 1e-10 <= |v| <= 1e20, else BigDecimal.toString's
 *                        scientific form (1.5E+21, 1E-11); 0.0 and -0.0 are 0;
 *   SGR_JSON_ID          (writer tables only) the row's aggregate id; dst_off and len are ignored.
 * Strings escape '"', '\\' and \b \t \n \f \r by their short forms and other characters below U+0020 as \u00XX (uppercase hex);
 * every other byte is written as it is. Every value parses back to its row through the state-topic restore (JSON members,
 * sgr_dingest_set_state_topic) and through any JSON parser, doubles equal by == (so -0.0 comes back as 0.0). The exact bytes
 * play-json writes are NOT pinned (no JVM here): member order, integers, UUIDs and escaping follow a restatement, the digits
 * of doubles are repr's, their layout is our reading of play-json's serializer.
 * A row cannot be written, and the JVM's writeState throws too, when an F64 member holds NaN or an infinity, a PSTR length byte
 * exceeds len - 1 or its bytes are not well-formed UTF-8, or (ID member) the id is not well-formed UTF-8 or the row has no id in
 * the key table. */
#define SGR_JSON_ID 5u
/* Register the writer table: members in value order, at most 32. Each non-ID member needs dst_off % 4 == 0, a size (I32 4,
 * I64 / F64 8, UUID 16, PSTR len) that is a multiple of 4 and at least 4, and dst_off + size <= state_bytes - 8, as a state
 * topic's JSON member table does; at most one SGR_JSON_ID member; names non-empty, well-formed UTF-8 and distinct. The restore's
 * table for the same values is this table without its ID member. n_members == 0 clears the writer. SGR_ERR_NO_PROGRAM before
 * sgr_register_program, and a later sgr_register_program clears the writer; SGR_ERR_INVALID on a bad table (nothing changes);
 * SGR_ERR_UNSUPPORTED on a routed engine without a current rank key table (sgr_dist_load_keys). */
int32_t sgr_set_state_writer(sgr_engine* e, const sgr_json_field* members, uint32_t n_members);
/* Three reads that return values instead of rows. Each matches its twin (sgr_get_batch, sgr_export_changes, sgr_scan) in
 * locking, table generation, id-index update, paging, cursor / token and error codes, with the rows replaced by values
 * (values_cap bytes) and value_offsets (rows + 1 u64): row i's value is values[value_offsets[i] .. value_offsets[i + 1]). A
 * None row (no SGR_ST_EXISTS in flags; in an export, the tombstone: the (id, null) record) has an empty span. flags is required.
 * SGR_ERR_STATE when no writer is set. A row that cannot be written fails the call with SGR_ERR_UNSUPPORTED and nothing written
 * (for a page, the cursor unchanged); the message names the lowest such row (its position in the batch or page and its dense
 * index), the member and the reason.
 * sgr_get_batch_values: all or nothing; an unknown id has an empty span, flags 0 and index -1. SGR_ERR_CAPACITY (nothing
 * written but *values_len, optional, = the bytes needed) when the values need more than values_cap bytes.
 * sgr_export_changes_values / sgr_scan_values: a page also ends before the first selected row whose value does not fit in
 * what is left of values_cap (cur->next names that row; *more is 1); SGR_ERR_CAPACITY (nothing written, the cursor unchanged)
 * when the first row's value alone does not fit. */
int32_t sgr_get_batch_values(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n, uint8_t* values, uint64_t values_cap,
                             uint64_t* value_offsets, uint32_t* flags, int64_t* indices, uint64_t* values_len);
int32_t sgr_export_changes_values(sgr_engine* e, uint32_t select, sgr_changes_cursor* cur, uint64_t max_rows, uint8_t* values,
                                  uint64_t values_cap, uint64_t* value_offsets, uint32_t* flags, uint32_t* err_idx, int64_t* indices,
                                  uint8_t* ids, uint64_t ids_cap, uint32_t* id_offsets, uint64_t* n_rows);
int32_t sgr_scan_values(sgr_engine* e, const uint8_t* from, uint32_t from_len, int32_t from_exclusive, const uint8_t* to, uint32_t to_len,
                        uint64_t max_rows, uint8_t* values, uint64_t values_cap, uint64_t* value_offsets, uint32_t* flags, int64_t* indices,
                        uint8_t* ids, uint64_t ids_cap, uint32_t* id_offsets, uint64_t* n_rows, int32_t* more);

/* building blocks, exported for the known-answer tests */
uint32_t sgr_crc32c(const void* data, uint64_t nbytes);            /* RFC 3720 CRC-32C (SSE4.2 when present) */
uint32_t sgr_crc32c_portable(const void* data, uint64_t nbytes);   /* table-driven twin */
uint32_t sgr_xxh32(const void* data, uint64_t nbytes, uint32_t seed);
int32_t sgr_lz4_frame_decode(const void* src, uint64_t nbytes, void* out, uint64_t cap, uint64_t* out_len);

/* ------------------------------------------------------------------ partitioner
 * KafkaPartitionProvider.partitionForKey = abs(MurmurHash3.stringHash(s) % n)
 * (COMMON/kafka/KafkaPartitioner.scala:7-9) over key.takeWhile(_ != ':')
 * (PartitionStringUpToColon, :38-42). Host-side, UTF-16 code units. */
int32_t sgr_string_hash_utf16(const uint16_t* units, uint32_t n);
int32_t sgr_partition_for_key_utf8(const uint8_t* key, uint32_t klen, uint32_t num_partitions,
                                   int32_t up_to_colon, int32_t* partition);
int32_t sgr_partitions_for_keys(const uint8_t* keys, const uint32_t* key_offsets, uint64_t n, uint32_t num_partitions,
                                int32_t up_to_colon, uint32_t* partition_of);

#ifdef __cplusplus
}
#endif
#endif /* SGR_H */
