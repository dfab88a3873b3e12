// dingest.cu — host side of the device record-batch decode (include/sgr.h "device ingest"; kernels: dingest_kernels.cu).
//
// The host keeps exactly what is sequential and tiny: the walk over the 61-byte RecordBatch headers of a fetch (boundaries, a
// trailing partial batch, magic), the read_committed bookkeeping of org.apache.kafka consumers (control batches, the aborted
// transactions a fetch response announces) and the partition positions for the lag gate
// (modules/command-engine/core/src/main/scala/surge/internal/kafka/KafkaProducerActorImpl.scala:684-708). The wire bytes go to
// the device as they are; CRC, lz4, record parsing, id interning and the fold never touch the CPU.
//
// Call sequence per poll:   sgr_dingest_submit(partition, fetch bytes)*  ->  sgr_dingest_fold()
// submit = header walk + one asynchronous H2D copy of the fetch (page-locked source memory makes it a single DMA). Whenever
//          `group_batches` data batches have accumulated, their whole chain
//              descriptors up -> crc_size (claims each batch's arena slot) -> decode_walk -> parse + intern
//          is enqueued on one of a few streams behind the copy that brought the group's last byte: no host round trip inside
//          the chain, so groups decode while later fetches are still crossing PCIe and while the host walks their headers.
// fold   = the chain of the remainder, one synchronisation, the verdicts (any error: nothing of the poll is applied), table
//          growth, new ids to the engine's key table, the fold of the decoded records onto the live table (sort-free programs
//          skip the holes in the atomic fold, the others group the live records first); only then do the partitions'
//          positions advance. All or nothing.
// The arena the batches decompress into is sized from the wire bytes (3x); if a poll compresses better than that the claims
// overflow, the flag comes back with the verdicts and the poll is decoded again from an exact host-side layout. Protobuf and
// JSON values (sgr_dingest_set_value_framing) are converted to packed events inside the parse kernel (value_framing.h); JSON
// compresses better than packed values, so under those framings the claim multiple adapts (claim_mult).
// A compacted STATE topic (sgr_dingest_set_state_topic) takes the same chain; its parse writes rows of program bytes, and the
// fold applies them last write wins with sgr_put_batch's kernels (put_decoded_poll) instead of folding events.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <map>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "../../include/sgr.h"
#include "devbuf.h"
#include "dingest_kernels.cuh"
#include "engine_internal.h"
#include "record_batch.h"

using namespace sgr;

struct sgr_dingest {
  sgr_engine* eng = nullptr;
  cudaStream_t stream = nullptr;
  std::string last_error;
  std::map<int32_t, PartitionState> parts;  // committed view (after the last successful fold)
  std::map<int32_t, PartitionState> staged; // view after the submissions of the current poll
  int32_t null_value_type = -1;
  int32_t value_framing = SGR_VALUE_PACKED;
  DevBuf json_table;                        // SGR_VALUE_JSON: member table (vf::Class[], vf::Field[], names) on the device
  vf::Table json{};                         // ... its view; n_classes == 0 until a packer is registered
  // arena claim of an lz4 batch, in multiples of its compressed size: 3 for packed values; under protobuf / JSON framing raised
  // after a poll that needed the exact-layout repeat, to the power of two at or above the largest ratio it showed (at most 16)
  uint32_t claim_mult = 3;
  // a compacted STATE topic (sgr_dingest_set_state_topic): the whole key is the id, a value is the program bytes of a row, null
  // deletes; a poll is applied last write wins (put_decoded_poll) instead of folded. Fixed before the first fold.
  bool state_topic = false;
  bool folded = false;                      // a fold succeeded since create / sgr_dingest_reset
  uint32_t row_bytes = 0;                   // state mode: program bytes of a row (state_bytes - 8), read when a poll's first group launches
  uint32_t json_row_end = 0;                // state mode: end of the registered JSON members in the row
  // staged submissions: the fetches of one poll accumulate in `wire`, whose first wire_used bytes are taken
  DevBuf wire;
  uint64_t wire_used = 0;
  // descriptors of the poll's data batches, in PAGE-LOCKED memory: every copy of them is a true asynchronous DMA (a copy from
  // pageable memory makes the host wait for the stream, which serialised the submissions behind each other's CRC kernels)
  struct PinnedBatches {
    HostBuf buf;
    size_t n = 0, cap = 0;
    bool reserve(size_t want) {   // (keeps the first n descriptors)
      if (want <= cap) return true;
      size_t c = cap ? cap : 4096;
      while (c < want) c *= 2;
      HostBuf nb;
      if (nb.alloc(c * sizeof(DgBatch), cudaHostAllocMapped) != cudaSuccess) return false;
      if (n) memcpy(nb.p, buf.p, n * sizeof(DgBatch));
      buf = std::move(nb);
      cap = c;
      return true;
    }
    size_t size() const { return n; }
    bool empty() const { return n == 0; }
    void clear() { n = 0; }
    DgBatch* data() { return (DgBatch*)buf.p; }
    DgBatch& operator[](size_t i) { return data()[i]; }
  } batches;
  uint64_t n_record_slots = 0;
  sgr_ingest_stats poll{};                  // statistics of the current poll (host-side parts)
  sgr_ingest_stats total{};
  struct Sub { uint32_t batch_begin, batch_end; uint64_t nbytes; cudaEvent_t copied; };
  std::vector<Sub> subs;                    // the submissions of the current poll, in order
  std::vector<Event> event_pool;
  Stream copy_stream;                       // H2D copies of the wire bytes: they overlap the decode of earlier submissions
  // device scratch
  DevBuf arena, d_batches;
  DevBuf rec_off, rec_batch, out;           // per record slot; they keep their content when a later group needs them larger
  DevBuf st_idx, st_present;                // ... state mode: the slot's dense index (~0u: hole) and 0 / 1 (tombstone / row)
  DevBuf key_offs_dev, key_bytes_dev, key_scan_tmp;
  // chains of launches per group of batches
  uint64_t launched_batches = 0;            // batches of this poll whose chain has been launched
  uint32_t group_batches = 8192;            // SGR_DINGEST_GROUP
  static constexpr int kGroupStreams = 8;
  Stream gstream[kGroupStreams];
  std::vector<Event> group_events;          // pool; the first n_groups are this poll's "group done" events
  uint32_t n_groups = 0;
  uint64_t launched_records = 0;            // record slots covered by the launched chains
  // SGR_DINGEST_TIMING: per group the device times (ms since the poll's first copy was queued) at which its bytes had landed,
  // its CRC + size pass, its decode and its parse ended; printed to stderr by sgr_dingest_fold
  std::vector<Event> tl_events;             // 4 per group
  Event tl_origin;                          // the poll's origin
  HostBuf h_keys;                           // page-locked landing area of the new ids
  // device dictionary
  DevBuf tags, slot_idx, key_ref, id_arena, ctl;
  uint64_t slots = 0, max_keys = 0, arena_cap = 0;
  uint64_t keys_on_host = 0;                // ids already appended to the engine's key table
  uint64_t id_bytes_on_host = 0;            // ... and the id-arena bytes they occupy
  Event keys_landed;
  uint64_t generation = 0;                  // bumped by sgr_dingest_reset: a new dictionary is a new owner of the engine's key table
  HostBuf h_ctl;                            // page-locked landing area
  bool timing_syncs = false;                // SGR_DINGEST_TIMING=1: record the per-group device timeline (tl_events)
  float ms[8] = {};                         // last fold: [0] wait for the copies and every chain [1] exact-layout repeat [2] unused
                                            //            [3] keys to host [4] table growth + fold [5] total
};

namespace {
template <class... A> int32_t dfail(sgr_dingest* g, int32_t code, const char* fmt, A... a) { return g ? set_error(&g->last_error, code, fmt, a...) : code; }
#define DG_TRY(g, call)                                                                                          \
  do {                                                                                                           \
    cudaError_t _e = (call);                                                                                     \
    if (_e == cudaErrorMemoryAllocation) (void)cudaGetLastError();   /* not sticky: the engine's next launch check must not see it */ \
    if (_e != cudaSuccess) return dfail((g), _e == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(_e)); \
  } while (0)

// grow an event pool to n events
cudaError_t grow_pool(std::vector<Event>& pool, size_t n, unsigned flags) {
  while (pool.size() < n) {
    Event ev;
    if (const cudaError_t e = cudaEventCreateWithFlags(ev.put(), flags)) return e;
    pool.push_back(std::move(ev));
  }
  return cudaSuccess;
}

std::string dg_err_text(const sgr_dingest* g, uint32_t e) {
  if ((e & 0xffu) == DG_VALUE_FRAMING) {   // the host decoder's text: JSON reasons follow "JSON event: "
    const uint32_t why = e >> 8;
    return std::string(why == vf::NOT_PROTOBUF ? "" : "JSON event: ") + vf::reason_text(why);
  }
  if ((e & 0xffu) == DG_STATE_LENGTH) {
    char buf[160];
    const uint32_t len = e >> 8;
    snprintf(buf, sizeof buf, "state value of %s%u bytes is longer than the %u program bytes of a row (state_bytes - 8)", len == 0xffffffu ? "at least " : "",
             len, g->row_bytes);
    return buf;
  }
  switch (e) {
    case DG_CRC: return "CRC-32C mismatch";
    case DG_LZ4_HEADER: return "bad LZ4 frame header";
    case DG_LZ4_BLOCK: return "LZ4 frame / block truncated or inconsistent";
    case DG_LZ4_SEQUENCE: return "malformed LZ4 sequence";
    case DG_LZ4_CHECKSUM: return "LZ4 checksum mismatch";
    case DG_LZ4_TOO_LARGE: return "LZ4 block decodes past its maximum size";
    case DG_RECORD_LENGTH: return "record length runs past the batch";
    case DG_RECORD_MALFORMED: return "record is malformed";
    case DG_RECORD_COUNT: return "recordsCount does not fit the batch";
    case DG_VALUE_LENGTH: return "packed event value outside 8..56 bytes (u32 type, u32 seq, payload)";
    case DG_ID_LENGTH: return "aggregate id too long";
    case DG_STRAY_BYTES: return "stray bytes after the last record";
  }
  return "unknown";
}

cudaError_t sync_all(sgr_dingest* g) {
  cudaError_t e = cudaSuccess, x;
  if (g->copy_stream && (x = cudaStreamSynchronize(g->copy_stream)) != cudaSuccess) e = x;
  for (cudaStream_t s : g->gstream) if (s && (x = cudaStreamSynchronize(s)) != cudaSuccess) e = x;
  if (g->stream && (x = cudaStreamSynchronize(g->stream)) != cudaSuccess) e = x;
  return e;
}

// per-poll device counters back to zero: [2] markers [3] null values [4] duplicates [5] dictionary overflow [6] records written,
// [8] arena bytes claimed, [10] arena overflow; [0] keys / [1] id bytes / [9] arena capacity persist
cudaError_t reset_poll_counters(sgr_dingest* g) {
  cudaError_t e = cudaMemsetAsync((unsigned long long*)g->ctl.p + 2, 0, 5 * 8, g->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync((unsigned long long*)g->ctl.p + 8, 0, 8, g->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync((unsigned long long*)g->ctl.p + 10, 0, 8, g->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(g->stream);   // group streams of the next poll must see it
  return e;
}

void clear_poll(sgr_dingest* g) {
  g->wire_used = 0; g->batches.clear(); g->n_record_slots = 0; g->poll = sgr_ingest_stats{}; g->subs.clear();
  g->launched_batches = 0; g->n_groups = 0; g->launched_records = 0;
}

void discard_poll(sgr_dingest* g) {
  sync_all(g);   // no copy may still be landing in the buffer the next poll reuses, no chain still running
  reset_poll_counters(g);
  clear_poll(g);
  g->staged = g->parts;
}

DgParse parse_args(sgr_dingest* g) {
  DgParse p{};
  p.wire = (const uint8_t*)g->wire.p; p.arena = (const uint8_t*)g->arena.p;
  p.batches = (DgBatch*)g->d_batches.p;
  p.rec_off = (const uint32_t*)g->rec_off.p; p.rec_batch = (const uint32_t*)g->rec_batch.p; p.out = (uint8_t*)g->out.p; p.null_value_type = g->null_value_type;
  p.value_framing = g->value_framing; p.json = g->json;
  p.dict.tags = (unsigned long long*)g->tags.p; p.dict.slot_idx = (uint32_t*)g->slot_idx.p; p.dict.key_ref = (uint2*)g->key_ref.p;
  p.dict.arena = (uint8_t*)g->id_arena.p; p.dict.ctl = (unsigned long long*)g->ctl.p; p.dict.slots_mask = g->slots - 1;
  p.dict.max_keys = g->max_keys; p.dict.arena_cap = g->arena_cap;
  p.state_topic = g->state_topic; p.row_bytes = g->row_bytes;
  p.idx = (uint32_t*)g->st_idx.p; p.present = (uint8_t*)g->st_present.p;
  return p;
}

// Grow a buffer to at least want_bytes, doubling from 1 MiB, keeping its first keep_bytes. Anything that moves waits for every
// stream first (kernels in flight hold the old address).
cudaError_t grow_keeping(sgr_dingest* g, DevBuf& b, uint64_t keep_bytes, uint64_t want_bytes) {
  if (want_bytes <= b.cap) return cudaSuccess;
  cudaError_t e = sync_all(g);
  if (e != cudaSuccess) return e;
  uint64_t cap = b.cap ? b.cap : (1ull << 20);
  while (cap < want_bytes) cap *= 2;
  return b.grow_keep(cap, keep_bytes, g->stream);
}

cudaError_t set_arena_capacity(sgr_dingest* g) {
  const unsigned long long cap = g->arena.cap >= 512 ? g->arena.cap - 512 : 0;   // (the walk's ring reads 256 bytes past a slot)
  return cudaMemcpy((unsigned long long*)g->ctl.p + 9, &cap, 8, cudaMemcpyHostToDevice);
}

// (state values compress like JSON events: a state topic adapts the claim whatever its framing)
uint32_t claim_multiple(const sgr_dingest* g) { return g->value_framing == SGR_VALUE_PACKED && !g->state_topic ? 3u : g->claim_mult; }

// Enqueue descriptors-up -> crc_size (+ arena claim) -> decode_walk -> parse for the batches [launched_batches, batch_end) —
// record slots [launched_records, rec_end) — behind `landed` (the copy of the last fetch that contributes to the group).
int32_t launch_group(sgr_dingest* g, uint64_t batch_end, uint64_t rec_end, cudaEvent_t landed) {
  const uint64_t b0 = g->launched_batches, nb = batch_end - b0;
  if (!nb) return SGR_OK;
  const uint64_t r0 = g->launched_records;
  if (g->state_topic && !g->n_groups) {   // the poll's rows take the program's width, fixed until its fold
    uint32_t sb = 0;
    bool routed = false;
    const int32_t rc = engine_program_state_bytes(g->eng, &sb, &routed);
    if (rc || !sb) return dfail(g, rc ? rc : SGR_ERR_NO_PROGRAM, "state topic: register a fold program first");
    if (routed) return dfail(g, SGR_ERR_UNSUPPORTED, "state topic: the rows of a routed engine are local slots");
    if (g->json_row_end > sb - 8) return dfail(g, SGR_ERR_STATE, "state topic: the JSON members end at program byte %u, past the program's %u", g->json_row_end, sb - 8);
    g->row_bytes = sb - 8;
  }
  const uint64_t stride = g->state_topic ? g->row_bytes : 64;
  DG_TRY(g, grow_keeping(g, g->d_batches, b0 * sizeof(DgBatch), batch_end * sizeof(DgBatch) + 64));
  DG_TRY(g, grow_keeping(g, g->rec_off, r0 * 4, rec_end * 4 + 64));
  DG_TRY(g, grow_keeping(g, g->rec_batch, r0 * 4, rec_end * 4 + 64));
  DG_TRY(g, grow_keeping(g, g->out, r0 * stride, rec_end * stride + 64));
  if (g->state_topic) {
    DG_TRY(g, grow_keeping(g, g->st_idx, r0 * 4, rec_end * 4 + 64));
    DG_TRY(g, grow_keeping(g, g->st_present, r0, rec_end + 64));
  }
  const uint64_t arena_want = (uint64_t)claim_multiple(g) * g->wire.cap + 512;
  if (g->arena.cap < arena_want) {
    DG_TRY(g, grow_keeping(g, g->arena, b0 ? g->arena.cap : 0, arena_want));
    DG_TRY(g, set_arena_capacity(g));
  }
  DG_TRY(g, grow_pool(g->group_events, g->n_groups + 1, cudaEventDisableTiming));
  cudaStream_t s = g->gstream[g->n_groups % sgr_dingest::kGroupStreams];
  DG_TRY(g, cudaStreamWaitEvent(s, landed, 0));
  const Event* tl = nullptr;
  if (g->timing_syncs) {
    DG_TRY(g, grow_pool(g->tl_events, 4 * (size_t)(g->n_groups + 1), cudaEventDefault));
    tl = g->tl_events.data() + 4 * (size_t)g->n_groups;
    DG_TRY(g, cudaEventRecord(tl[0], s));
  }
  DgBatch* db = (DgBatch*)g->d_batches.p + b0;
  {
    void* mapped = nullptr;   // the descriptors go up by a kernel: a copy-engine transfer would queue behind every fetch of the poll
    DG_TRY(g, cudaHostGetDevicePointer(&mapped, g->batches.data() + b0, 0));
    DG_TRY(g, dg_copy_from_mapped_host(mapped, db, nb * sizeof(DgBatch), s));
  }
  if (rec_end > r0) DG_TRY(g, cudaMemsetAsync((uint32_t*)g->rec_batch.p + r0, 0xff, (rec_end - r0) * 4, s));
  DG_TRY(g, dg_launch_crc_size_fast((const uint8_t*)g->wire.p, db, (uint32_t)nb, (unsigned long long*)g->ctl.p + 8, claim_multiple(g), s));
  if (tl) DG_TRY(g, cudaEventRecord(tl[1], s));
  DG_TRY(g, dg_launch_decode_walk_fast((const uint8_t*)g->wire.p, (uint8_t*)g->arena.p, db, (uint32_t)nb, (uint32_t)b0, (uint32_t*)g->rec_off.p, (uint32_t*)g->rec_batch.p, (unsigned long long*)g->ctl.p + 8, s));
  if (tl) DG_TRY(g, cudaEventRecord(tl[2], s));
  DgParse p = parse_args(g);
  p.n_batches = (uint32_t)batch_end; p.rec_begin = (uint32_t)r0; p.n_records = (uint32_t)rec_end;
  DG_TRY(g, dg_launch_parse(p, s));
  if (tl) DG_TRY(g, cudaEventRecord(tl[3], s));
  DG_TRY(g, cudaEventRecord(g->group_events[g->n_groups], s));
  ++g->n_groups;
  g->launched_batches = batch_end; g->launched_records = rec_end;
  return SGR_OK;
}
}  // namespace

extern "C" {

int32_t sgr_dingest_create(sgr_engine* e, uint64_t max_keys, uint64_t max_id_bytes, sgr_dingest** out) {
  if (!e || !out || !max_keys) return SGR_ERR_INVALID;
  *out = nullptr;
  void* st = nullptr;
  if (sgr_stream(e, &st) != SGR_OK) return SGR_ERR_INVALID;
  std::unique_ptr<sgr_dingest> g(new sgr_dingest());   // (a failure below frees whatever was made)
  g->eng = e; g->stream = (cudaStream_t)st;
  g->timing_syncs = getenv("SGR_DINGEST_TIMING") != nullptr;
  if (const char* gb = getenv("SGR_DINGEST_GROUP")) { const long v = atol(gb); if (v >= 64 && v <= (1l << 24)) g->group_batches = (uint32_t)v; }
  if (dg_prepare() != cudaSuccess) return SGR_ERR_CUDA;
  if (cudaStreamCreateWithFlags(g->copy_stream.put(), cudaStreamNonBlocking) != cudaSuccess) return SGR_ERR_CUDA;
  for (Stream& s : g->gstream)
    if (cudaStreamCreateWithFlags(s.put(), cudaStreamNonBlocking) != cudaSuccess) return SGR_ERR_CUDA;
  g->max_keys = max_keys;
  g->slots = 1024;
  while (g->slots < 2 * max_keys) g->slots *= 2;          // load factor <= 0.5
  g->arena_cap = max_id_bytes ? max_id_bytes : 32 * max_keys;
  cudaError_t ce;
  if ((ce = g->tags.reserve(g->slots * 8)) != cudaSuccess || (ce = g->slot_idx.reserve(g->slots * 4)) != cudaSuccess ||
      (ce = g->key_ref.reserve(max_keys * 8)) != cudaSuccess || (ce = g->id_arena.reserve(g->arena_cap + 64)) != cudaSuccess ||
      (ce = g->ctl.reserve(128)) != cudaSuccess || (ce = g->h_ctl.alloc(256, cudaHostAllocDefault)) != cudaSuccess ||
      (ce = cudaMemsetAsync(g->tags.p, 0, g->slots * 8, g->stream)) != cudaSuccess || (ce = cudaMemsetAsync(g->slot_idx.p, 0, g->slots * 4, g->stream)) != cudaSuccess ||
      (ce = cudaMemsetAsync(g->ctl.p, 0, 128, g->stream)) != cudaSuccess || (ce = cudaStreamSynchronize(g->stream)) != cudaSuccess)
    return ce == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA;
  *out = g.release();
  return SGR_OK;
}

int32_t sgr_dingest_destroy(sgr_dingest* g) {
  if (!g) return SGR_OK;
  sync_all(g);
  delete g;
  return SGR_OK;
}

const char* sgr_dingest_last_error(const sgr_dingest* g) { return g ? g->last_error.c_str() : "null device-ingest handle"; }

int32_t sgr_dingest_set_null_value_type(sgr_dingest* g, int32_t event_type) {
  if (!g || event_type >= (int32_t)SGR_MAX_TYPES) return dfail(g, SGR_ERR_INVALID, "event type out of range");
  g->null_value_type = event_type < 0 ? -1 : event_type;
  return SGR_OK;
}

// Both settings are refused while a poll is pending: its groups were parsed at submit time, and the exact-layout repeat parses
// again at fold time; one poll must not be decoded two ways.
int32_t sgr_dingest_set_value_framing(sgr_dingest* g, int32_t framing) {
  if (!g || (framing != SGR_VALUE_PACKED && framing != SGR_VALUE_PROTOBUF_EVENT && framing != SGR_VALUE_JSON)) return dfail(g, SGR_ERR_INVALID, "unknown value framing %d", framing);
  if (!g->subs.empty()) return dfail(g, SGR_ERR_STATE, "the value framing cannot change between a submit and its fold");
  if (framing == SGR_VALUE_JSON && !g->json.n_classes) return dfail(g, SGR_ERR_INVALID, "register a JSON packer first (sgr_dingest_set_json_packer)");
  g->value_framing = framing;
  return SGR_OK;
}

int32_t sgr_dingest_set_state_topic(sgr_dingest* g, int32_t on) {
  if (!g) return SGR_ERR_INVALID;
  if (!g->subs.empty()) return dfail(g, SGR_ERR_STATE, "the topic mode cannot change between a submit and its fold");
  if (g->folded) return dfail(g, SGR_ERR_STATE, "the topic mode is fixed once a poll was folded (sgr_dingest_reset first)");
  if (g->json.n_classes) return dfail(g, SGR_ERR_STATE, "set the topic mode before the JSON packer: its offsets mean different things in the two modes");
  uint32_t sb = 0;
  bool routed = false;
  if (engine_program_state_bytes(g->eng, &sb, &routed) != SGR_OK) return dfail(g, SGR_ERR_INVALID, "engine");
  if (routed) return dfail(g, SGR_ERR_UNSUPPORTED, "the rows of a routed engine are local slots: a state topic does not map ids to them");
  g->state_topic = on != 0;
  return SGR_OK;
}

int32_t sgr_dingest_set_json_packer(sgr_dingest* g, const char* discriminator, const sgr_json_event* events, uint32_t n_events, int32_t unknown_type) {
  if (!g || !discriminator || (n_events && !events)) return dfail(g, SGR_ERR_INVALID, "null argument");
  if (!g->subs.empty()) return dfail(g, SGR_ERR_STATE, "the JSON packer cannot change between a submit and its fold");
  if (unknown_type >= (int32_t)SGR_MAX_TYPES) return dfail(g, SGR_ERR_INVALID, "unknown_type out of range");
  if (!*discriminator && n_events != 1) return dfail(g, SGR_ERR_INVALID, "without a discriminator member exactly one class can be registered");
  // state topic: Json.toJson(state) writes no discriminator, the one class is the state; members land at program byte offsets
  uint32_t row_limit = 0, row_end = 0;
  if (g->state_topic) {
    if (*discriminator) return dfail(g, SGR_ERR_INVALID, "a state topic's JSON values carry no discriminator member");
    bool routed = false;
    if (engine_program_state_bytes(g->eng, &row_limit, &routed) != SGR_OK || !row_limit) return dfail(g, SGR_ERR_NO_PROGRAM, "state topic: register a fold program first");
    row_limit -= 8;
  }
  // the table goes to the device as classes, fields, then the names
  std::vector<vf::Class> classes;
  std::vector<vf::Field> fields;
  std::string names = discriminator;
  for (uint32_t i = 0; i < n_events; ++i) {
    const sgr_json_event& e = events[i];
    if (!e.type_name || e.event_type >= SGR_MAX_TYPES || e.n_fields > SGR_JSON_MAX_FIELDS) return dfail(g, SGR_ERR_INVALID, "JSON event %u: bad type name, type index or field count", i);
    classes.push_back(vf::Class{(uint32_t)names.size(), (uint32_t)strlen(e.type_name), e.event_type, (uint32_t)fields.size(), e.n_fields});
    names += e.type_name;
    for (uint32_t f = 0; f < e.n_fields; ++f) {
      const sgr_json_field& jf = e.fields[f];
      // state topic: anywhere in the row's program bytes
      const uint32_t size = json_member_size(jf);
      const bool ok = size && (g->state_topic ? (uint64_t)jf.dst_off + size <= row_limit : json_event_slot_ok(jf, size));
      if (!ok) return dfail(g, SGR_ERR_INVALID, "JSON %s %u field %u: bad name, kind, length or %s offset", g->state_topic ? "state" : "event", i, f,
                            g->state_topic ? "program byte" : "record");
      row_end = std::max(row_end, jf.dst_off + size);
      fields.push_back(vf::Field{(uint32_t)names.size(), (uint32_t)strlen(jf.name), jf.kind, jf.dst_off, size});
      names += jf.name;
    }
  }
  const size_t cls_bytes = classes.size() * sizeof(vf::Class), fld_bytes = fields.size() * sizeof(vf::Field);
  std::vector<uint8_t> blob(cls_bytes + fld_bytes + names.size() + 1);
  if (cls_bytes) memcpy(blob.data(), classes.data(), cls_bytes);
  if (fld_bytes) memcpy(blob.data() + cls_bytes, fields.data(), fld_bytes);
  memcpy(blob.data() + cls_bytes + fld_bytes, names.data(), names.size());
  DG_TRY(g, sync_all(g));   // (no kernel of an earlier poll may still read the old table)
  DevBuf nb;
  DG_TRY(g, nb.reserve(blob.size()));
  DG_TRY(g, cudaMemcpy(nb.p, blob.data(), blob.size(), cudaMemcpyHostToDevice));
  g->json_table = std::move(nb);
  const uint8_t* base = (const uint8_t*)g->json_table.p;
  g->json = vf::Table{base + cls_bytes + fld_bytes, (const vf::Class*)base, (const vf::Field*)(base + cls_bytes), (uint32_t)classes.size(), 0,
                      (uint32_t)strlen(discriminator), unknown_type < 0 ? -1 : unknown_type};
  g->json_row_end = row_end;
  return SGR_OK;
}

int32_t sgr_dingest_set_aborted(sgr_dingest* g, int32_t partition, const int64_t* producer_ids, const int64_t* first_offsets, uint64_t n) {
  if (!g || (n && (!producer_ids || !first_offsets))) return dfail(g, SGR_ERR_INVALID, "null argument");
  g->staged[partition].announce_aborted(producer_ids, first_offsets, n);
  return SGR_OK;
}

// Walk the batch headers of one fetch; data batches that a read_committed consumer would deliver are queued for the device.
int32_t sgr_dingest_submit(sgr_dingest* g, int32_t partition, const void* data, uint64_t nbytes, sgr_ingest_stats* stats) {
  if (!g || (!data && nbytes)) return dfail(g, SGR_ERR_INVALID, "null argument");
  const uint8_t* buf = (const uint8_t*)data;
  PartitionState ps = g->staged[partition];   // work on a copy: a malformed fetch leaves the staged view untouched
  sgr_ingest_stats st{};
  std::vector<DgBatch> add;
  uint64_t slots = 0, pos = 0;
  for (BatchHeader h;; pos += h.total) {
    if (const int32_t rc = frame_batch(partition, buf, nbytes, pos, &h, &g->last_error)) return rc;
    if (!h.total) break;   // a trailing partial batch: the next fetch repeats it
    if (const int32_t rc = read_batch_fields(partition, &h, &g->last_error)) return rc;
    ++st.n_batches;
    const bool aborted_batch = ps.reach(h);
    if (h.control) {
      // tiny and never compressed by the broker: read on the host (CRC included), it only steers the bookkeeping. Read as the
      // host decoder reads it: a codec other than none / lz4 is refused, an lz4 one is decompressed, the key must fit.
      ++st.n_control_batches;
      if (sgr_crc32c(h.b + 21, h.total - 21) != h.stored_crc) return dfail(g, SGR_ERR_INVALID, "partition %d offset %lld: CRC-32C mismatch in a control batch", partition, (long long)h.base_offset);
      if (h.codec != 0 && h.codec != 3) return dfail(g, SGR_ERR_UNSUPPORTED, "partition %d offset %lld: compression codec %d (none and lz4 are decoded)", partition, (long long)h.base_offset, h.codec);
      const uint8_t* r = h.b + kBatchHeader; const uint8_t* end = h.b + h.total;
      std::vector<uint8_t> plain;
      if (h.codec == 3) {
        uint64_t n = 0;
        if (sgr_lz4_frame_decode(r, h.total - kBatchHeader, nullptr, 0, &n) == SGR_ERR_INVALID) return dfail(g, SGR_ERR_INVALID, "partition %d offset %lld: bad lz4 frame in a control batch", partition, (long long)h.base_offset);
        plain.resize(n);
        if (n && sgr_lz4_frame_decode(r, h.total - kBatchHeader, plain.data(), n, &n) != SGR_OK) return dfail(g, SGR_ERR_INVALID, "partition %d offset %lld: bad lz4 frame in a control batch", partition, (long long)h.base_offset);
        st.n_compressed_bytes += h.total - kBatchHeader; st.n_decompressed_bytes += n;
        r = plain.data(); end = r + n;
      }
      ps.apply_control(h, r, (uint64_t)(end - r));
    } else if (aborted_batch) {
      // skipped unread, as Kafka's consumer skips it, but only after its CRC: a damaged batch is refused here as on the host
      if (sgr_crc32c(h.b + 21, h.total - 21) != h.stored_crc) return dfail(g, SGR_ERR_INVALID, "partition %d offset %lld: CRC-32C mismatch in an aborted batch", partition, (long long)h.base_offset);
      ++st.n_aborted_batches; st.n_aborted_records += (uint64_t)h.records_count;
    } else {
      // A batch entirely below the position (a refetch) is decoded and checked like any other and its records count as
      // duplicates, as the host decoder and Kafka's consumer do: skipping it unread would accept damage the host refuses.
      if (h.codec != 0 && h.codec != 3) {
        // the CRC comes first, as on the host and in Kafka's consumer: a damaged batch is invalid whatever its codec says
        if (sgr_crc32c(h.b + 21, h.total - 21) != h.stored_crc) return dfail(g, SGR_ERR_INVALID, "partition %d offset %lld: CRC-32C mismatch", partition, (long long)h.base_offset);
        return dfail(g, SGR_ERR_UNSUPPORTED, "partition %d offset %lld: compression codec %d (none and lz4 are decoded)", partition, (long long)h.base_offset, h.codec);
      }
      // Every record is at least 7 bytes and lz4 expands at most 255-fold: a recordsCount beyond that is refused here, before the
      // poll sizes its per-record buffers by it (the decode kernels then check the exact bound, as the host decoder does).
      const uint64_t max_section = h.codec == 3 ? (h.total - kBatchHeader) * 255ull + 64 : h.total - kBatchHeader;
      if ((uint64_t)h.records_count > max_section / 7 + 1) return dfail(g, SGR_ERR_INVALID, "partition %d offset %lld: recordsCount %d does not fit the batch", partition, (long long)h.base_offset, h.records_count);
      DgBatch d{};
      d.src_off = g->wire_used + pos; d.base_offset = h.base_offset; d.min_offset = ps.seen ? ps.decoded_next : INT64_MIN;
      d.total_len = (uint32_t)h.total; d.n_records = (uint32_t)h.records_count; d.codec = (uint16_t)h.codec; d.stored_crc = h.stored_crc;
      d.rec_base = (uint32_t)(g->n_record_slots + slots);
      slots += (uint64_t)h.records_count;
      if (h.codec == 3) st.n_compressed_bytes += h.total - kBatchHeader;
      add.push_back(d);
    }
    ps.close(h);
  }
  st.n_bytes = pos; st.n_trailing_bytes = nbytes - pos;
  if (g->n_record_slots + slots >= (1ull << 32)) return dfail(g, SGR_ERR_CAPACITY, "more than 2^32 records in one poll");
  sgr_dingest::Sub sub{};
  sub.batch_begin = (uint32_t)g->batches.size(); sub.batch_end = sub.batch_begin + (uint32_t)add.size(); sub.nbytes = pos;
  DG_TRY(g, grow_pool(g->event_pool, g->subs.size() + 1, cudaEventDisableTiming));
  sub.copied = g->event_pool[g->subs.size()];
  if (g->timing_syncs && g->subs.empty()) {
    if (!g->tl_origin) DG_TRY(g, cudaEventCreate(g->tl_origin.put()));
    DG_TRY(g, cudaEventRecord(g->tl_origin, g->copy_stream));
  }
  if (pos) {
    DG_TRY(g, grow_keeping(g, g->wire, g->wire_used, g->wire_used + pos + 272));   // (the input ring reads up to 256 bytes past a batch)
    DG_TRY(g, cudaMemcpyAsync((uint8_t*)g->wire.p + g->wire_used, buf, pos, cudaMemcpyHostToDevice, g->copy_stream));
    g->wire_used += (pos + 15) & ~15ull;
  }
  DG_TRY(g, cudaEventRecord(sub.copied, g->copy_stream));
  g->subs.push_back(sub);
  if (!add.empty()) {
    if (g->batches.n + add.size() > g->batches.cap) {   // the pinned array moves: nothing may still be copying from / into it
      DG_TRY(g, sync_all(g));
      if (!g->batches.reserve(g->batches.n + add.size())) return dfail(g, SGR_ERR_OOM, "page-locked descriptor array");
    }
    memcpy(g->batches.data() + g->batches.n, add.data(), add.size() * sizeof(DgBatch));
    g->batches.n += add.size();
    if (g->batches.n - g->launched_batches >= g->group_batches) {
      const int32_t rc = launch_group(g, g->batches.n, g->n_record_slots + slots, sub.copied);
      if (rc) { discard_poll(g); return rc; }
    }
  }
  g->n_record_slots += slots;
  g->staged[partition] = ps;
  add_stats(&g->poll, st);   // (n_decompressed_bytes: lz4 control batches; data batches add theirs at the fold)
  g->poll.n_trailing_bytes = st.n_trailing_bytes;
  if (stats) *stats = st;
  return SGR_OK;
}

int32_t sgr_dingest_fold(sgr_dingest* g, sgr_ingest_stats* stats) {
  if (!g) return SGR_ERR_INVALID;
  const uint32_t nb = (uint32_t)g->batches.size();
  const uint32_t nrec = (uint32_t)g->n_record_slots;
  sgr_ingest_stats st = g->poll;
  unsigned long long* h = (unsigned long long*)g->h_ctl.p;
  typedef std::chrono::steady_clock Clk;
  const Clk::time_point t_begin = Clk::now();
  Clk::time_point t_last = t_begin;
  auto lap = [&](int i) { const Clk::time_point now = Clk::now(); g->ms[i] += std::chrono::duration<float, std::milli>(now - t_last).count(); t_last = now; };
  memset(g->ms, 0, sizeof g->ms);
  if (nb) {
    DgParse p = parse_args(g);
    // ---- chains: launch the remainder, wait for every group, bring the verdicts back
    { const int32_t rc = launch_group(g, nb, nrec, g->subs.back().copied); if (rc) { discard_poll(g); return rc; } }
    for (uint32_t k = 0; k < g->n_groups; ++k) DG_TRY(g, cudaStreamWaitEvent(g->stream, g->group_events[k], 0));
    DG_TRY(g, cudaMemcpyAsync(g->batches.data(), g->d_batches.p, (size_t)nb * sizeof(DgBatch), cudaMemcpyDeviceToHost, g->stream));
    DG_TRY(g, cudaMemcpyAsync(h, g->ctl.p, 128, cudaMemcpyDeviceToHost, g->stream));
    DG_TRY(g, cudaStreamSynchronize(g->stream));
    lap(0);
    if (g->timing_syncs && g->tl_origin) {
      for (uint32_t k = 0; k < g->n_groups; ++k) {
        float t[4] = {0, 0, 0, 0};
        for (int j = 0; j < 4; ++j) cudaEventElapsedTime(&t[j], g->tl_origin, g->tl_events[4 * (size_t)k + j]);
        fprintf(stderr, "[dingest] group %u: landed %.2f  crc+size %.2f  decode+walk %.2f  parse %.2f ms\n", k, t[0], t[1], t[2], t[3]);
      }
    }
    if (h[10]) {
      // the arena claims overflowed (the poll compresses better than 3x): lay the arena out exactly and decode + parse again.
      // Ids the first attempt interned stay (an id is an id); its records are overwritten slot for slot.
      // (exact sizes first: the claim mode never measured them)
      DG_TRY(g, dg_launch_crc_size_fast((const uint8_t*)g->wire.p, (DgBatch*)g->d_batches.p, nb, nullptr, 0, g->stream));
      DG_TRY(g, cudaMemcpyAsync(g->batches.data(), g->d_batches.p, (size_t)nb * sizeof(DgBatch), cudaMemcpyDeviceToHost, g->stream));
      DG_TRY(g, cudaStreamSynchronize(g->stream));
      uint64_t need = 0;
      double ratio = 0;
      for (uint32_t i = 0; i < nb; ++i) {
        DgBatch& b = g->batches[i];
        if (b.err == DG_ARENA_FULL) b.err = DG_OK;
        if (b.err) { const int32_t rc = dfail(g, SGR_ERR_INVALID, "offset %lld: %s", (long long)b.base_offset, dg_err_text(g, b.err).c_str()); discard_poll(g); return rc; }
        b.rec_err = kNoRecErr;
        if (b.codec == 3) {
          b.arena_off = need; need += ((uint64_t)b.dsize + 15) & ~15ull;
          ratio = std::max(ratio, (double)b.dsize / (double)std::max<uint64_t>(1, b.total_len - kBatchHeader));
        }
      }
      if (g->value_framing != SGR_VALUE_PACKED || g->state_topic)
        while (g->claim_mult < 16 && (double)g->claim_mult < ratio) g->claim_mult = g->claim_mult < 4 ? 4 : 2 * g->claim_mult;
      DG_TRY(g, grow_keeping(g, g->arena, 0, need + 512));
      DG_TRY(g, set_arena_capacity(g));
      p = parse_args(g);
      h[2] = h[3] = h[4] = h[5] = h[6] = 0; h[8] = need; h[10] = 0;
      DG_TRY(g, cudaMemcpyAsync((unsigned long long*)g->ctl.p + 2, h + 2, 5 * 8, cudaMemcpyHostToDevice, g->stream));
      DG_TRY(g, cudaMemcpyAsync((unsigned long long*)g->ctl.p + 8, h + 8, 8, cudaMemcpyHostToDevice, g->stream));
      DG_TRY(g, cudaMemcpyAsync((unsigned long long*)g->ctl.p + 10, h + 10, 8, cudaMemcpyHostToDevice, g->stream));
      DG_TRY(g, cudaMemsetAsync(g->rec_batch.p, 0xff, (size_t)nrec * 4 + 4, g->stream));
      DG_TRY(g, cudaMemcpyAsync(g->d_batches.p, g->batches.data(), (size_t)nb * sizeof(DgBatch), cudaMemcpyHostToDevice, g->stream));
      DG_TRY(g, dg_launch_decode_walk_fast((const uint8_t*)g->wire.p, (uint8_t*)g->arena.p, (DgBatch*)g->d_batches.p, nb, 0, (uint32_t*)g->rec_off.p, (uint32_t*)g->rec_batch.p, nullptr, g->stream));
      p.n_batches = nb; p.rec_begin = 0; p.n_records = nrec;
      DG_TRY(g, dg_launch_parse(p, g->stream));
      DG_TRY(g, cudaMemcpyAsync(g->batches.data(), g->d_batches.p, (size_t)nb * sizeof(DgBatch), cudaMemcpyDeviceToHost, g->stream));
      DG_TRY(g, cudaMemcpyAsync(h, g->ctl.p, 128, cudaMemcpyDeviceToHost, g->stream));
      DG_TRY(g, cudaStreamSynchronize(g->stream));
      lap(1);
    }
    for (uint32_t i = 0; i < nb; ++i) if (g->batches[i].codec == 3 && !g->batches[i].err) st.n_decompressed_bytes += g->batches[i].dsize;
    // a batch-level error (CRC, lz4, the record walk) first, else the batch's lowest refused record; the walk's errors therefore
    // win over an earlier record's value error, where the host decoder, checking record by record, names that record (same code)
    for (uint32_t i = 0; i < nb; ++i)
      if (g->batches[i].err || g->batches[i].rec_err != kNoRecErr) {
        const DgBatch& b = g->batches[i];
        const uint32_t record = b.rec_err == kNoRecErr ? 0u : (uint32_t)(b.rec_err >> 32), code = b.err ? b.err : (uint32_t)b.rec_err;
        const int32_t rc = dfail(g, SGR_ERR_INVALID, "offset %lld, record %u: %s", (long long)b.base_offset, record, dg_err_text(g, code).c_str());
        // ids interned by this failed poll stay in the dictionary (harmless: an id is an id); the records are dropped
        discard_poll(g); return rc;
      }
    if (h[5]) {
      const int32_t rc = dfail(g, SGR_ERR_CAPACITY, "device id dictionary full (%llu ids / %llu id bytes allowed): create the device ingest with larger bounds", (unsigned long long)g->max_keys, (unsigned long long)g->arena_cap);
      discard_poll(g); return rc;
    }
    // ctl[0] and ctl[1] also count the claims a full dictionary refused (intern): the ids admitted are the first max_keys dense
    // indices at most, their bytes within arena_cap
    const uint64_t n_keys = std::min<uint64_t>(h[0], g->max_keys), id_bytes = std::min<uint64_t>(h[1], g->arena_cap);
    st.n_markers = h[2]; st.n_null_values = h[3]; st.n_duplicates += h[4]; st.n_records = h[6]; st.n_new_keys = n_keys - g->keys_on_host;   // (ids a failed poll interned become visible with the next good one)
    // ---- grow the table for the new ids, hand their names to the engine's key table, fold
    if (const int32_t rc = grow_states_for_ids(g->eng, n_keys, g->max_keys)) {
      dfail(g, rc, "engine: %s", sgr_last_error(g->eng)); discard_poll(g); return rc;
    }
    lap(4);
    // The new ids, gathered on the device into dense-index order, come down in two copies queued BEHIND nothing the fold needs
    // and IN FRONT of the fold's kernels; a helper thread hands them to the engine's key table while this thread runs the fold.
    std::thread appender;
    int32_t rc_append = SGR_OK;
    if (n_keys > g->keys_on_host) {
      const uint64_t add = n_keys - g->keys_on_host;
      const uint64_t id_bytes_max = id_bytes - g->id_bytes_on_host;   // (an upper bound: arena entries are padded to 8 bytes)
      DG_TRY(g, g->key_offs_dev.reserve((add + 2) * 4));
      DG_TRY(g, g->key_bytes_dev.reserve(id_bytes_max + 64));
      uint32_t* d_offs = (uint32_t*)g->key_offs_dev.p;
      DG_TRY(g, dg_gather_keys(p.dict, g->keys_on_host, (uint32_t)add, d_offs, (uint8_t*)g->key_bytes_dev.p, g->key_scan_tmp, g->stream));
      const uint64_t h_need = (add + 2) * 4 + id_bytes_max + 64;
      if (g->h_keys.cap < h_need) DG_TRY(g, g->h_keys.alloc(2 * h_need, cudaHostAllocDefault));
      uint32_t* h_offs = (uint32_t*)g->h_keys.p;
      uint8_t* h_bytes = (uint8_t*)g->h_keys.p + (add + 2) * 4;
      DG_TRY(g, cudaMemcpyAsync(h_offs, d_offs, (add + 1) * 4, cudaMemcpyDeviceToHost, g->stream));
      if (id_bytes_max) DG_TRY(g, cudaMemcpyAsync(h_bytes, g->key_bytes_dev.p, id_bytes_max, cudaMemcpyDeviceToHost, g->stream));
      if (!g->keys_landed) DG_TRY(g, cudaEventCreateWithFlags(g->keys_landed.put(), cudaEventDisableTiming));
      DG_TRY(g, cudaEventRecord(g->keys_landed, g->stream));
      int dev = 0;
      cudaGetDevice(&dev);
      const void* owner = (const char*)g + g->generation;
      appender = std::thread([g, dev, owner, h_offs, h_bytes, add, &rc_append]() {
        cudaSetDevice(dev);
        if (cudaEventSynchronize(g->keys_landed) != cudaSuccess) { rc_append = SGR_ERR_CUDA; return; }
        rc_append = sgr_append_keys(g->eng, owner, h_bytes, h_offs, add);
      });
    }
    lap(3);
    int32_t rc_fold = SGR_OK;
    if (nrec && g->state_topic) rc_fold = put_decoded_poll(g->eng, g->out.p, (const uint32_t*)g->st_idx.p, (const uint8_t*)g->st_present.p, nrec, st.n_records);
    else if (nrec) rc_fold = fold_decoded_poll(g->eng, g->out.p, nrec, st.n_records);
    if (appender.joinable()) appender.join();
    if (rc_fold) { dfail(g, rc_fold, "engine: %s", sgr_last_error(g->eng)); discard_poll(g); return rc_fold; }
    if (rc_append) { dfail(g, rc_append, "engine: %s", sgr_last_error(g->eng)); discard_poll(g); return rc_append; }
    g->keys_on_host = n_keys; g->id_bytes_on_host = id_bytes;
  }
  lap(4);
  g->ms[5] = std::chrono::duration<float, std::milli>(Clk::now() - t_begin).count();
  // ---- commit: the staged positions become the live ones and everything decoded is folded
  for (auto& kv : g->staged) { kv.second.folded_next = kv.second.decoded_next; }
  g->parts = g->staged;
  g->folded = true;
  if (nb) DG_TRY(g, reset_poll_counters(g));
  clear_poll(g);
  add_stats(&g->total, st);
  if (stats) *stats = st;
  return SGR_OK;
}

int32_t sgr_dingest_reset(sgr_dingest* g) {
  if (!g) return SGR_ERR_INVALID;
  discard_poll(g);
  g->parts.clear(); g->staged.clear(); g->total = sgr_ingest_stats{}; g->keys_on_host = 0; g->id_bytes_on_host = 0; ++g->generation;
  g->folded = false;   // (the topic mode stays, as the value framing does)
  DG_TRY(g, cudaMemsetAsync(g->tags.p, 0, g->slots * 8, g->stream));
  DG_TRY(g, cudaMemsetAsync(g->slot_idx.p, 0, g->slots * 4, g->stream));
  DG_TRY(g, cudaMemsetAsync(g->ctl.p, 0, 9 * 8, g->stream));                                  // ([9], the arena's capacity, stays)
  DG_TRY(g, cudaMemsetAsync((unsigned long long*)g->ctl.p + 10, 0, 8, g->stream));
  DG_TRY(g, cudaStreamSynchronize(g->stream));                                                   // the group streams must see it
  return SGR_OK;
}

int32_t sgr_dingest_offsets(sgr_dingest* g, int32_t partition, int64_t* decoded_next, int64_t* folded_next) {
  return g ? partition_offsets(g->parts, partition, decoded_next, folded_next) : SGR_ERR_INVALID;
}

int32_t sgr_dingest_last_timing(sgr_dingest* g, float* ms8) {
  if (!g || !ms8) return SGR_ERR_INVALID;
  memcpy(ms8, g->ms, sizeof g->ms);
  return SGR_OK;
}

int32_t sgr_dingest_get_stats(sgr_dingest* g, sgr_ingest_stats* out) {
  if (!g || !out) return SGR_ERR_INVALID;
  *out = g->total;
  return SGR_OK;
}

}  // extern "C"
