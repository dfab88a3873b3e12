// engine.cu — the C ABI of include/sgr.h over the CUDA kernels (host side of the boundary).
//
// No CPU fallback lives here: every compute entry point launches a kernel on the engine's
// device or fails with a status code. Nothing in this file includes or links oracle/.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/sgr.h"
#include "bulk_fold.cuh"
#include "changes.cuh"
#include "devbuf.h"
#include "dist.cuh"
#include "engine_internal.h"
#include "fold_kernels.cuh"
#include "fold_rows.cuh"
#include "group_kernels.cuh"
#include "id_index.cuh"
#include "id_order.cuh"
#include "incremental.cuh"
#include "keytable.h"
#include "put_batch.cuh"
#include "route_push.cuh"
#include "state_values.cuh"

using namespace sgr;

namespace {
thread_local std::string g_create_error;
thread_local std::string t_last_error;
thread_local const sgr_engine* t_last_engine = nullptr;

// host snapshot of the state table that sgr_get reads (published after a fold)
struct Snapshot {
  std::vector<uint8_t> states;
  uint64_t n_agg = 0;
  uint32_t state_bytes = 0;
};

// sgr_engine::gb_dev begins with u64 control words that kernels write and one copy brings back to the host:
//   [kCtlDup], [kCtlNoSlot]        the id index insert's duplicate ids and ids that found no free slot (id_index_settle)
//   [kCtlGatherBad]                id_index_gather's largest out-of-range index + 1
//   [kCtlCut, kCtlCut + 4)         changes_count_cut's page cut, indexed by kChCtl* (changes.cuh)
//   [kCtlRange, kCtlRange + 2)     sgr_scan's range of positions (id_order_bounds)
// id_index_update zeroes the words before kCtlCut, and sgr_get_batch's results follow them. The scan's bounds and the page of
// sgr_export_changes / sgr_scan start at byte kPayloadOff.
constexpr size_t kCtlDup = 0, kCtlNoSlot = 1, kCtlGatherBad = 2, kCtlCut = 4, kCtlRange = 8, kPayloadOff = 96;

// Which rows carry the CHANGED/ERROR flags the last operation set, so that the next one clears only those (clear_flagged). The
// lists stay in the engine's buffers: a host list in inc_prev_ids, a device list in inc_touched[next ^ 1] with its count in the
// matching inc_counters block.
struct FlaggedRows {
  enum Kind { kWholeTable, kNothing, kHostList, kDeviceList };
  Kind kind = kWholeTable;
  uint64_t n = 0;       // kHostList: the list's length
  uint32_t upper = 0;   // kDeviceList: a bound on the list's length
  int next = 0;         // the inc_touched buffer the next atomic micro-batch writes its list to
  void forget() { kind = kWholeTable; }
  void nothing() { kind = kNothing; }
  void host_list(uint64_t count) { kind = kHostList; n = count; }
  void device_list(uint32_t bound) { kind = kDeviceList; upper = bound; next ^= 1; }
};

// The fold enqueue_fold launched, for finish_fold: which kernel, on what, and where its counters are.
struct PendingFold {
  enum Kernel { kSequential, kRows, kRuns, kVarRuns };
  Kernel kernel = kSequential;
  bool stamped = false;   // timed by the kernel itself (counters[8], [9]) rather than by ev0 / ev1
  bool prior = false;     // folded onto the live table in place
  uint64_t n_seg = 0, event_bytes = 0;
  const uint8_t* events = nullptr; const uint64_t* offsets = nullptr; const uint32_t* ids = nullptr;
  const void* counters = nullptr;
};
}  // namespace

struct sgr_engine {
  int device = 0;
  int num_sms = 0;
  Stream stream;
  Event ev0, ev1;

  bool has_program = false;
  sgr_fold_program program{};
  DevProgram dprog{};

  // CSR event log: owned buffers or borrowed pointers
  DevBuf own_events, own_offsets, own_rec_offsets;
  const uint64_t* d_rec_offsets = nullptr;   // record directory (variable records), or null
  uint64_t n_rec = 0;
  const uint8_t* d_events = nullptr;
  const uint64_t* d_offsets = nullptr;
  uint64_t event_bytes = 0;
  uint64_t n_agg = 0;
  bool loaded = false;
  uint32_t max_record_bytes = 64;

  DevBuf states;        // n_agg * state_bytes, live table
  bool states_valid = false;  // holds prior states (set_initial_states or a previous fold)
  uint64_t states_n = 0;
  DevBuf counters;      // 8 x u64
  GroupScratch group;   // K5 scratch
  DevBuf inc_records, inc_offsets, inc_ids, inc_prev_ids;  // K6
  // sort-free K6 (incremental.cu)
  DevBuf inc_scratch, inc_touched[2], inc_err_ids, inc_counters;
  uint64_t inc_scratch_slots = 0;
  FlaggedRows flagged;

  // record-parallel path (fold_rows.cu)
  bool row_ok = false;            // program is inside the transformer algebra
  RowProgram row_prog{};
  int row_max_grid = 0;
  int run_max_grid = 0, run_max_grid_variant = -1;
  int64_t opt_run_variant = 0;
  DevBuf part_flags, part_data, redo_ids;
  DevBuf run_counters;            // 2 x 16 u64, ping-pong; the runs kernel zeroes the other block itself
  int run_counter_idx = 0;
  int64_t opt_run_chunk_bytes = 131072; // runs kernel: bytes of log per ticket (rounded to whole steps, at least NSTAGE);
                                        // on configs[1] 128 KiB beat 32 KiB and 512 KiB (scripts/fold_ceiling.py)
  uint32_t epoch = 0;
  size_t part_flags_cap_seen = 0;
  bool offsets_aligned64 = false; // every segment offset == log_begin (mod 64)
  uint64_t log_begin = 0, log_end = 0, max_seg_bytes = 0;
  bool fold_pending = false;      // a fold was enqueued and not yet finished (it is `pending`)
  PendingFold pending;
  Event ev2, ev3;

  int64_t opt_kernel = 0;         // 0 auto (runs if the program allows), 1 lane-sequential TMA kernel (fold_kernels.cu),
                                  // 2 force runs (fold_runs.cu), 3 record-per-lane rows (fold_rows.cu)
  int64_t opt_variant = -1;
  int64_t opt_long_threshold = 0;
  int64_t opt_var_stages = 1;     // 1 stage leaves shared memory for the most resident warps per SM (2 or 3 trade warps for depth)
  int64_t opt_var_stage_bytes = 12288;  // smem bytes staged per 32-record step of the variable-record kernel
  int64_t opt_replay_budget = 1ll << 24;  // K6: in-kernel replay of throwing slots only while n_err * n stays below this
                                          // (beyond it one group-by of the batch is cheaper)
  int64_t opt_force_route = 0;    // profiling aid: run K4 even on a single rank
  int64_t opt_incremental = 0;    // 0 auto (sort-free K6 when the program allows), 1 force the sort-based path
  int64_t opt_max_record_bytes = 528;

  // sort-free fold of large arrival-order logs (bulk_fold.cu)
  bool bulk_ok = false;
  BulkLayout bulk_lay{};
  DevBuf bulk_scratch, bulk_err_ids, bulk_counters, hash_out;
  uint64_t bulk_scratch_slots = 0;
  int64_t opt_bulk = 1;           // 0: keep arrival-order logs on the single-launch micro-batch kernel (incremental.cu)
  int64_t opt_push_ordered = 0;   // 1: positions inside the exchange regions follow the log from the first attempt (look-back)
  int64_t opt_push_chunks = 16;   // chunks of the pipelined route + exchange + fold (route_push.cu); the same on every rank

  sgr_stats stats{};

  Owned<DistState*, dist_destroy> dist;   // this rank's routing state (sgr_dist_init), or none
  sgr_dist_stats dstats{};

  std::shared_ptr<const KeyTable> keys;   // swapped atomically: sgr_get readers never see a table being rebuilt
  // ids handed over by sgr_fold_ingested: appended per poll (the dictionary is append-only), hashed lazily by the first
  // sgr_get that follows — a restore polls thousands of times before anybody reads
  std::mutex keys_mu;
  std::vector<uint8_t> ing_key_bytes;
  std::vector<uint32_t> ing_key_offs;
  const void* ing_keys_from = nullptr;      // whose dictionary the appended ids mirror (an sgr_ingest or an sgr_dingest)
  std::atomic<bool> keys_stale{false};
  uint64_t keys_epoch = 0;                  // bumped (under keys_mu) whenever the key table is replaced rather than appended to
  // (under keys_mu) the key table is this rank's, built by sgr_dist_load_keys for the current partition table: the reads
  // serve a routed engine only while it is set
  bool rank_keys = false;
  // sgr_get_batch: the device id index, kept up to date lazily like the host KeyTable (under op_mu, then keys_mu), and its
  // staging: one page-locked buffer (ids and queries up, results down) and one device buffer (queries, results) that begins
  // with the control words named by kCtl* (above)
  IdIndex id_index;
  HostBuf gb_host;
  DevBuf gb_dev;
  DevBuf ch_tiles;                          // sgr_export_changes, sgr_scan: per-tile totals and bases (changes.cuh)
  IdOrder id_order;                         // sgr_scan: the index's ids in Bytes order, brought up to date by the first scan after they change
  // sgr_put_batch: the batch's scratch (put_batch.cuh), and the last-write word of each table row (u32, zero between batches)
  DevBuf pb_scratch, pb_last;
  uint64_t pb_last_n = 0;                   // rows pb_last covers
  // sgr_set_state_writer: the writer table (writer.n == 0: none; its literals in writer_lits) and the member names for refusal
  // messages; the scratch and the values of the value-returning reads (state_values.cuh)
  SwWriter writer{};
  DevBuf writer_lits;
  std::vector<std::string> writer_names;
  DevBuf sv_scratch, sv_values;
  // Every call that changes the engine (loads, folds, table growth) and the snapshot refresh of a reader hold op_mu:
  // a reader never sees a table being freed or swapped, and a snapshot is only marked clean for the generation it copied.
  std::recursive_mutex op_mu;
  std::atomic<uint64_t> generation{0};
  std::shared_ptr<Snapshot> snapshot;
  std::atomic<bool> snapshot_dirty{true};
};

namespace {

// serialises engine mutation against the snapshot refresh of concurrent readers (ADVICE r1: reader threads touched a table
// the stream thread was freeing); recursive because public entry points call each other (sgr_fold_ingested)
struct OpLock {
  std::unique_lock<std::recursive_mutex> l;
  explicit OpLock(sgr_engine* e) { if (e) l = std::unique_lock<std::recursive_mutex>(e->op_mu); }
};

int32_t fail(sgr_engine* e, int32_t code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  // errno-style: the message belongs to the calling thread (sgr_get runs on a 32-thread pool in the reference; two failing
  // readers must not race on one string). sgr_last_error(e) answers for the last failure of THIS thread on e.
  if (e) { t_last_error = buf; t_last_engine = e; } else g_create_error = buf;
  return code;
}
#define CUDA_TRY(e, call)                                                                         \
  do {                                                                                            \
    cudaError_t _err = (call);                                                                    \
    if (_err != cudaSuccess)                                                                      \
      return fail((e), _err == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA, "%s: %s", #call, \
                  cudaGetErrorString(_err));                                                      \
  } while (0)

int32_t use_device(sgr_engine* e) {
  CUDA_TRY(e, cudaSetDevice(e->device));
  return SGR_OK;
}

int32_t compile_program(sgr_engine* e, const sgr_fold_program* p, DevProgram* d) {
  if (p->state_bytes < 16 || p->state_bytes > SGR_MAX_STATE_BYTES || p->state_bytes % 16)
    return fail(e, SGR_ERR_INVALID, "state_bytes %u must be a multiple of 16 in [16,%u]", p->state_bytes, SGR_MAX_STATE_BYTES);
  if (p->record_kind != SGR_REC_FIXED64 && p->record_kind != SGR_REC_VAR16)
    return fail(e, SGR_ERR_INVALID, "unknown record_kind %u", p->record_kind);
  if (p->n_types == 0 || p->n_types > SGR_MAX_TYPES) return fail(e, SGR_ERR_INVALID, "n_types %u out of range", p->n_types);
  if (p->n_f64_fields > 8) return fail(e, SGR_ERR_INVALID, "n_f64_fields %u > 8", p->n_f64_fields);
  memset(d, 0, sizeof *d);
  d->state_words = p->state_bytes / 4;
  d->user_words = d->state_words - 2;
  d->record_kind = p->record_kind;
  d->n_types = p->n_types;
  d->n_f64 = p->n_f64_fields;
  const uint32_t user_bytes = p->state_bytes - 8;
  for (uint32_t f = 0; f < p->n_f64_fields; ++f) {
    if (p->f64_field_off[f] % 4 || p->f64_field_off[f] + 8u > user_bytes)
      return fail(e, SGR_ERR_INVALID, "f64 field %u at offset %u outside the program area", f, p->f64_field_off[f]);
    d->f64_word[f] = p->f64_field_off[f] / 4;
  }
  const uint32_t max_src = p->record_kind == SGR_REC_FIXED64 ? 64u : 0xfffcu;
  for (uint32_t t = 0; t < p->n_types; ++t) {
    const sgr_rule& r = p->rules[t];
    if (r.exists_rule > SGR_THROW) return fail(e, SGR_ERR_INVALID, "rule %u: bad exists_rule %u", t, r.exists_rule);
    if (r.n_ops > SGR_MAX_OPS) return fail(e, SGR_ERR_INVALID, "rule %u: n_ops %u > %u", t, r.n_ops, SGR_MAX_OPS);
    DevRule& dr = d->rules[t];
    dr.exists_rule = r.exists_rule;
    dr.n_ops = (r.exists_rule == SGR_TOMBSTONE || r.exists_rule == SGR_THROW) ? 0 : r.n_ops;
    dr.min_len = 16;
    for (uint32_t i = 0; i < dr.n_ops; ++i) {
      const sgr_op& o = r.ops[i];
      if (o.opcode > SGR_OP_SUB_I64) return fail(e, SGR_ERR_UNSUPPORTED, "rule %u op %u: opcode %u", t, i, o.opcode);
      uint32_t len = o.len;
      if (o.opcode == SGR_OP_ADD_I32 || o.opcode == SGR_OP_SUB_I32) { if (len != 4) return fail(e, SGR_ERR_INVALID, "rule %u op %u: i32 op needs len 4", t, i); }
      else if (o.opcode == SGR_OP_ADD_I64 || o.opcode == SGR_OP_SUB_I64) { if (len != 8) return fail(e, SGR_ERR_INVALID, "rule %u op %u: i64 op needs len 8", t, i); }
      if (len == 0 || len % 4 || o.dst_off % 4 || o.src_off % 4)
        return fail(e, SGR_ERR_INVALID, "rule %u op %u: offsets and length must be non-zero multiples of 4", t, i);
      if (o.dst_off + len > user_bytes) return fail(e, SGR_ERR_INVALID, "rule %u op %u: writes past the program area", t, i);
      if (o.src_off + len > max_src) return fail(e, SGR_ERR_INVALID, "rule %u op %u: reads past the record", t, i);
      if (o.src_off + len > dr.min_len) dr.min_len = o.src_off + len;
      dr.ops[i] = pack_op(o.opcode, len / 4, o.dst_off / 4, o.src_off / 4);
    }
  }
  return SGR_OK;
}

int32_t finish_fold(sgr_engine* e);

void mark_dirty(sgr_engine* e) { e->generation.fetch_add(1, std::memory_order_acq_rel); e->snapshot_dirty.store(true, std::memory_order_release); }

int32_t ensure_states(sgr_engine* e, uint64_t n_agg) {
  const size_t need = (size_t)n_agg * e->program.state_bytes;
  if (e->states_n != n_agg || e->states.cap < need) {
    CUDA_TRY(e, e->states.reserve(need));
    e->states_n = n_agg;
    e->states_valid = false;
  }
  return SGR_OK;
}

// publish a host snapshot of the live state table for sgr_get
int32_t refresh_snapshot(sgr_engine* e, std::shared_ptr<Snapshot>* out) {
  // readers (sgr_get on the store's 32-thread pool) and the stream thread's loads/folds exclude each other here
  std::lock_guard<std::recursive_mutex> g(e->op_mu);
  if (!e->snapshot_dirty.load(std::memory_order_acquire) && e->snapshot) { *out = e->snapshot; return SGR_OK; }
  const uint64_t gen = e->generation.load(std::memory_order_acquire);
  if (!e->states_valid) return fail(e, SGR_ERR_STATE, "state store is not readable: no fold has completed");
  int32_t rc = use_device(e); if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  auto s = std::make_shared<Snapshot>();
  s->n_agg = e->states_n; s->state_bytes = e->program.state_bytes;
  s->states.resize((size_t)s->n_agg * s->state_bytes);
  CUDA_TRY(e, cudaMemcpyAsync(s->states.data(), e->states.p, s->states.size(), cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  std::atomic_store(&e->snapshot, s);
  // clean only for the generation that was copied (op_mu makes a concurrent bump impossible today; the check keeps it so)
  if (e->generation.load(std::memory_order_acquire) == gen) e->snapshot_dirty.store(false, std::memory_order_release);
  *out = s;
  return SGR_OK;
}

constexpr uint64_t kRedoCap = 1u << 20;

// Reserve the look-back partials of a record-parallel launch of up to n_warps_max warps (`words` u32 of part_data per warp) and
// the replay list, and move to a new epoch. The flags are cleared when their buffer is new and when the epoch wraps to 0.
int32_t begin_lookback(sgr_engine* e, uint64_t n_warps_max, uint64_t words) {
  CUDA_TRY(e, e->part_flags.reserve(n_warps_max * 4 + 256));
  CUDA_TRY(e, e->part_data.reserve(n_warps_max * words * 4 + 256));
  CUDA_TRY(e, e->redo_ids.reserve(kRedoCap * 4));
  if (e->epoch == 0 || e->part_flags_cap_seen != e->part_flags.cap) {
    CUDA_TRY(e, cudaMemsetAsync(e->part_flags.p, 0, e->part_flags.cap, e->stream));
    e->part_flags_cap_seen = e->part_flags.cap;
  }
  ++e->epoch;
  if (e->epoch == 0) { CUDA_TRY(e, cudaMemsetAsync(e->part_flags.p, 0, e->part_flags.cap, e->stream)); e->epoch = 1; }
  return SGR_OK;
}

// Enqueue the exact replay of the segments a record-parallel kernel listed in redo_ids (throwing or malformed) on the
// sequential kernel; their count lives on the device (counters[3]).
int32_t launch_replay(sgr_engine* e, const uint8_t* d_events, const uint64_t* d_offsets, const uint32_t* d_ids, const uint8_t* states_in,
                      unsigned long long* counters) {
  FoldArgs a{};
  a.events = d_events; a.seg_offsets = d_offsets; a.seg_ids = d_ids; a.n_seg = kRedoCap; a.seg_list = (const uint32_t*)e->redo_ids.p;
  a.n_seg_dev = counters + 3; a.states_in = states_in; a.states_out = (uint8_t*)e->states.p; a.counters = counters;
  FoldLaunchInfo info{};
  cudaError_t le = launch_fold_stream(a, e->dprog, -1, 8, e->max_record_bytes, e->stream, &info);
  if (le != cudaSuccess) return fail(e, SGR_ERR_CUDA, "replay launch: %s", cudaGetErrorString(le));
  return SGR_OK;
}

// Enqueue one fold on the engine's stream (no host synchronisation).
int32_t enqueue_fold(sgr_engine* e, const uint8_t* d_events, const uint64_t* d_offsets, const uint32_t* d_ids,
                     uint64_t n_seg, bool use_prior, uint64_t event_bytes, bool aligned64, uint64_t log_begin, uint64_t log_end) {
  const uint8_t* states_in = use_prior ? (const uint8_t*)e->states.p : nullptr;
  // 64-byte states: the transformer scan moves 16 registers per lane per step and the lane-per-aggregate TMA kernel is
  // faster on balanced logs (BankAccount); the record-parallel kernel is taken when a
  // long segment would otherwise serialise one lane
  const bool wide_balanced = e->row_prog.user_words == 14 && e->opt_kernel == 0 && d_offsets == e->d_offsets && e->max_seg_bytes <= (256u << 10);
  bool use_rows = e->row_ok && !wide_balanced && e->program.record_kind == SGR_REC_FIXED64 && aligned64 && e->opt_kernel != 1 && n_seg < (1ull << 32) && n_seg > 0;
  if ((e->opt_kernel == 2 || e->opt_kernel == 3) && !use_rows && n_seg > 0)
    return fail(e, SGR_ERR_UNSUPPORTED, "record-parallel kernel cannot take this program/log");
  if (use_rows && e->opt_kernel == 3 && (e->row_prog.user_words != 2 || e->row_prog.cls != 0 || e->row_prog.n_slots > 6 || e->row_prog.f64_mask))
    return fail(e, SGR_ERR_UNSUPPORTED, "the record-per-lane kernel takes 16-byte class-0 programs only");
  const bool runs = use_rows && e->opt_kernel != 3;
  unsigned long long* counters = (unsigned long long*)e->counters.p;
  if (runs) {
    if (!e->run_counters.p) {
      CUDA_TRY(e, e->run_counters.reserve(256));
      CUDA_TRY(e, cudaMemsetAsync(e->run_counters.p, 0, 256, e->stream));
    }
    counters = (unsigned long long*)e->run_counters.p + 16 * e->run_counter_idx;
  } else {
    CUDA_TRY(e, cudaMemsetAsync(e->counters.p, 0, 64, e->stream));
  }
  // A runs fold queued right behind a runs fold of the same log overlaps it (programmatic dependent launch): before its
  // griddepcontrol.wait it reads only the log, the offsets and the program, which the fold before it does not write. Behind
  // anything else (a group-by or decode kernel that writes the log, a copy) it is launched plainly.
  const bool overlap = runs && e->fold_pending && e->pending.kernel == PendingFold::kRuns && e->pending.events == d_events &&
                       e->pending.offsets == d_offsets && e->pending.ids == d_ids;
  // an overlapping fold stamps its own start and end (counters[8], [9]): an event between two folds would keep the next
  // one from starting while this one drains. Every other fold is timed by CUDA events around its launch.
  if (!overlap) CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
  uint32_t launches = 0;
  PendingFold::Kernel kernel = PendingFold::kSequential;
  const bool use_var = e->row_ok && e->row_prog.user_words == 2 && e->row_prog.cls == 0 && e->program.record_kind == SGR_REC_VAR16 && e->d_rec_offsets && d_offsets == e->d_offsets && !use_prior &&
                       !d_ids && e->opt_kernel != 1 && n_seg > 0 && n_seg < (1ull << 32) && e->n_rec > 0;
  if (use_var) {
    int threads = 0; size_t smem = 0; uint32_t stage = 0;
    const int max_grid = vruns_config(e->num_sms, e->max_record_bytes, (uint32_t)e->opt_var_stage_bytes, (int)e->opt_var_stages, &threads, &smem, &stage);
    if (max_grid > 0) {
      int32_t rc = begin_lookback(e, (uint64_t)max_grid * (threads / 32), 8); if (rc) return rc;
      CUDA_TRY(e, cudaMemsetAsync(e->states.p, 0, (size_t)n_seg * e->program.state_bytes, e->stream));
      VarArgs v{};
      v.events = d_events; v.rec_offsets = e->d_rec_offsets; v.n_rec = e->n_rec; v.seg_offsets = d_offsets; v.n_seg = n_seg;
      v.states_out = (uint8_t*)e->states.p; v.counters = counters; v.redo_ids = (uint32_t*)e->redo_ids.p; v.redo_cap = kRedoCap;
      v.part_flags = (uint32_t*)e->part_flags.p; v.part_data = (uint32_t*)e->part_data.p; v.epoch = e->epoch; v.stage_bytes = stage;
      const uint64_t steps = (e->n_rec + 31) / 32;
      uint64_t want = (steps + (threads / 32) - 1) / (threads / 32);
      const int grid = (int)(want < (uint64_t)max_grid ? want : (uint64_t)max_grid);
      cudaError_t le = launch_fold_vruns(v, e->row_prog, (int)e->opt_var_stages, grid, threads, smem, e->stream);
      if (le != cudaSuccess) return fail(e, SGR_ERR_CUDA, "fold_vruns launch: %s", cudaGetErrorString(le));
      rc = launch_replay(e, d_events, d_offsets, d_ids, states_in, counters); if (rc) return rc;
      launches = 2;
      kernel = PendingFold::kVarRuns;
    }
  }
  if (n_seg && kernel != PendingFold::kVarRuns) {
    if (use_rows) {
      const bool v1 = e->opt_kernel == 3;
      const int rv = (int)e->opt_run_variant;
      if (v1 && !e->row_max_grid) e->row_max_grid = row_kernel_max_grid(e->num_sms, e->row_prog);
      if (!v1 && e->run_max_grid_variant != rv) { e->run_max_grid = run_kernel_max_grid(e->num_sms, rv, e->row_prog); e->run_max_grid_variant = rv; }
      const int max_grid = v1 ? e->row_max_grid : e->run_max_grid;
      const int wpc = v1 ? kRowThreads / 32 : run_warps_per_cta();
      const uint64_t step_bytes = v1 ? 2048 : (uint64_t)run_variant_step_bytes(rv, e->row_prog);
      const uint64_t steps = (log_end - log_begin + step_bytes - 1) / step_bytes;
      // the runs kernel publishes a look-back partial per chunk of chunk_steps steps, the rows kernel one per warp; a
      // small log is cut into smaller chunks, so that every resident warp gets one
      const uint64_t chunk_steps = v1 ? 1 : run_variant_chunk_steps(rv, e->row_prog, (uint64_t)e->opt_run_chunk_bytes, steps, (uint64_t)max_grid * wpc);
      const uint64_t n_chunks = (steps + chunk_steps - 1) / chunk_steps;
      const uint64_t n_parts = v1 ? (uint64_t)max_grid * wpc : n_chunks;
      int32_t rc = begin_lookback(e, n_parts, e->row_prog.user_words + 2); if (rc) return rc;
      RowArgs r{};
      r.events = d_events; r.seg_offsets = d_offsets; r.seg_ids = d_ids; r.n_seg = n_seg;
      r.log_begin = log_begin; r.log_end = log_end;
      r.states_in = states_in; r.states_out = (uint8_t*)e->states.p;
      r.counters = counters;
      r.counters_next = runs ? (unsigned long long*)e->run_counters.p + 16 * (e->run_counter_idx ^ 1) : nullptr;
      r.redo_ids = (uint32_t*)e->redo_ids.p; r.redo_cap = kRedoCap;
      r.part_flags = (uint32_t*)e->part_flags.p; r.part_data = (uint32_t*)e->part_data.p; r.epoch = e->epoch;
      r.chunk_steps = chunk_steps;
      uint64_t want = (n_chunks + wpc - 1) / wpc;
      if (want == 0) want = 1;  // all segments empty: one CTA still writes every (None) state
      const int grid = (int)(want < (uint64_t)max_grid ? want : (uint64_t)max_grid);
      cudaError_t le = v1 ? launch_fold_rows(r, e->row_prog, grid, e->stream) : launch_fold_runs(r, e->row_prog, rv, grid, overlap, e->stream);
      if (le != cudaSuccess) return fail(e, SGR_ERR_CUDA, "fold launch: %s", cudaGetErrorString(le));
      if (runs) {
        e->run_counter_idx ^= 1;  // the kernel replays throwing segments itself and cleans the other block
        launches = 1;
      } else {
        rc = launch_replay(e, d_events, d_offsets, d_ids, states_in, counters); if (rc) return rc;
        launches = 2;
      }
      kernel = runs ? PendingFold::kRuns : PendingFold::kRows;
    } else {
      FoldArgs a{};
      a.events = d_events; a.seg_offsets = d_offsets; a.seg_ids = d_ids; a.n_seg = n_seg;
      a.states_in = states_in; a.states_out = (uint8_t*)e->states.p;
      a.counters = counters;
      a.long_threshold = (uint64_t)e->opt_long_threshold;
      FoldLaunchInfo info{};
      cudaError_t le = launch_fold_stream(a, e->dprog, (int)e->opt_variant, e->num_sms, e->max_record_bytes, e->stream, &info);
      if (le != cudaSuccess) return fail(e, SGR_ERR_CUDA, "fold launch: %s", cudaGetErrorString(le));
      launches = 1;
    }
  }
  if (!overlap) CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  e->fold_pending = true;
  e->pending = PendingFold{kernel, overlap, use_prior, n_seg, event_bytes, d_events, d_offsets, d_ids, counters};
  e->stats.fold_launches = launches;
  return SGR_OK;
}

// Wait for the enqueued fold and collect its statistics.
int32_t finish_fold(sgr_engine* e) {
  if (!e->fold_pending) return SGR_OK;
  e->fold_pending = false;
  PendingFold& p = e->pending;
  unsigned long long h[16] = {};
  CUDA_TRY(e, cudaMemcpyAsync(h, p.counters, p.kernel == PendingFold::kRuns ? 128 : 64, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  // stamped: from the first CTA's entry (~counters[8]) to the last warp's exit, both %globaltimer nanoseconds
  if (p.stamped) e->stats.ms_fold = (h[8] && h[9] > ~h[8]) ? (float)((double)(h[9] - ~h[8]) * 1e-6) : 0.f;
  else CUDA_TRY(e, cudaEventElapsedTime(&e->stats.ms_fold, e->ev0, e->ev1));
  if ((p.kernel == PendingFold::kVarRuns && h[7]) || (p.kernel != PendingFold::kSequential && h[3] > kRedoCap)) {
    // the variable-record kernel's directory/header view disagreed with the CSR, or more aggregates threw than the replay
    // list holds: the CSR is the source of truth, fold everything again on the sequential kernel
    if (p.prior) {
      // the kernel has already overwritten the non-throwing aggregates in place: the table is half-applied. It must not be
      // served, and a retry must not double-apply — invalidate it (reads fail with SGR_ERR_STATE until the next full fold)
      e->states_valid = false; mark_dirty(e);
      return fail(e, SGR_ERR_UNSUPPORTED, "replay list overflow on an in-place incremental fold: state table invalidated, rebuild it");
    }
    FoldArgs a{};
    a.events = p.events; a.seg_offsets = p.offsets; a.seg_ids = p.ids; a.n_seg = p.n_seg;
    a.states_out = (uint8_t*)e->states.p; a.counters = (unsigned long long*)e->counters.p;
    CUDA_TRY(e, cudaMemsetAsync(e->counters.p, 0, 64, e->stream));
    CUDA_TRY(e, cudaEventRecord(e->ev2, e->stream));
    FoldLaunchInfo info{};
    cudaError_t le = launch_fold_stream(a, e->dprog, -1, e->num_sms, e->max_record_bytes, e->stream, &info);
    if (le != cudaSuccess) return fail(e, SGR_ERR_CUDA, "fold launch: %s", cudaGetErrorString(le));
    CUDA_TRY(e, cudaEventRecord(e->ev3, e->stream));
    CUDA_TRY(e, cudaMemcpyAsync(h, e->counters.p, 64, cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(e, cudaStreamSynchronize(e->stream));
    float ms2 = 0; CUDA_TRY(e, cudaEventElapsedTime(&ms2, e->ev2, e->ev3));
    e->stats.ms_fold += ms2; e->stats.fold_launches += 1;
    // h now holds the sequential kernel's counters, which count only the events before each throw
    p.kernel = PendingFold::kSequential;
  }
  const uint64_t n_seg = p.n_seg;
  e->stats.n_aggregates = n_seg;
  switch (p.kernel) {
    case PendingFold::kSequential: e->stats.n_events = h[0]; break;
    // the runs kernel counts every record, the replay takes back what followed a throw; the rows kernel skips throwing
    // segments, the replay adds what preceded the throw; the variable-record kernel does both
    case PendingFold::kRuns: e->stats.n_events = h[0] - h[4]; break;
    case PendingFold::kRows: e->stats.n_events = h[0] + h[5]; break;
    case PendingFold::kVarRuns: e->stats.n_events = h[0] - h[4] + h[5]; break;
  }
  e->stats.n_errors = h[1];
  e->stats.n_long_segments = h[2];
  e->stats.event_bytes = p.event_bytes;
  e->stats.algorithmic_bytes = p.event_bytes + 8 * (n_seg + 1) + (uint64_t)e->program.state_bytes * n_seg * (p.prior ? 2 : 1) + (p.ids ? 4 * n_seg : 0);
  return SGR_OK;
}

}  // namespace

// ================================================================== C ABI
extern "C" {

int32_t sgr_abi_version(void) { return SGR_ABI_VERSION; }

const char* sgr_last_error(const sgr_engine* e) {
  if (!e) return g_create_error.c_str();
  return t_last_engine == e ? t_last_error.c_str() : "";
}

int32_t sgr_create(const sgr_config* cfg, sgr_engine** out) {
  if (!out) return fail(nullptr, SGR_ERR_INVALID, "out is NULL");
  *out = nullptr;
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(nullptr, SGR_ERR_NO_DEVICE, "no CUDA device (%s); the replay engine has no CPU fallback",
                ce != cudaSuccess ? cudaGetErrorString(ce) : "device count 0");
  const int dev = cfg ? cfg->device : 0;
  if (dev < 0 || dev >= ndev) return fail(nullptr, SGR_ERR_NO_DEVICE, "device %d out of range (have %d)", dev, ndev);
  cudaDeviceProp prop;
  if ((ce = cudaGetDeviceProperties(&prop, dev)) != cudaSuccess)
    return fail(nullptr, SGR_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(ce));
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, SGR_ERR_NO_DEVICE, "device %d is sm_%d%d; kernels are built for sm_90a only", dev, prop.major, prop.minor);
  std::unique_ptr<sgr_engine> e(new sgr_engine());
  e->device = dev;
  e->num_sms = prop.multiProcessorCount;
  if ((ce = cudaSetDevice(dev)) != cudaSuccess) return fail(nullptr, SGR_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(ce));
  if ((ce = cudaStreamCreateWithFlags(e->stream.put(), cudaStreamNonBlocking)) != cudaSuccess ||
      (ce = cudaEventCreate(e->ev0.put())) != cudaSuccess || (ce = cudaEventCreate(e->ev1.put())) != cudaSuccess ||
      (ce = cudaEventCreate(e->ev2.put())) != cudaSuccess || (ce = cudaEventCreate(e->ev3.put())) != cudaSuccess ||
      (ce = e->counters.reserve(64)) != cudaSuccess)
    return fail(nullptr, SGR_ERR_CUDA, "engine setup: %s", cudaGetErrorString(ce));
  *out = e.release();
  return SGR_OK;
}

int32_t sgr_destroy(sgr_engine* e) {
  if (!e) return SGR_OK;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  delete e;   // (its members free the buffers, the rank state, the events and, last, the stream)
  return SGR_OK;
}

int32_t sgr_register_program(sgr_engine* e, const sgr_fold_program* prog) {
  OpLock op_lock(e);
  if (!e || !prog) return fail(e, SGR_ERR_INVALID, "null argument");
  DevProgram d;
  int32_t rc = compile_program(e, prog, &d);
  if (rc) return rc;
  e->program = *prog; e->dprog = d; e->has_program = true;
  e->row_ok = build_row_program(d, &e->row_prog);
  e->bulk_ok = e->row_ok && prog->record_kind == SGR_REC_FIXED64 && bulk_layout_for(e->row_prog, &e->bulk_lay);
  e->bulk_scratch_slots = 0;
  e->row_max_grid = 0; e->run_max_grid_variant = -1;
  e->states_valid = false; e->states_n = 0;
  e->writer.n = 0;   // its offsets belonged to the old program
  mark_dirty(e);
  return SGR_OK;
}

static int32_t before_load(sgr_engine* e) {
  int32_t rc = use_device(e); if (rc) return rc;
  return finish_fold(e);
}

struct Upload { void* dst; const void* src; size_t bytes; };

// Copy host buffers to the device between the events t0 and t1, wait for them, and record the span as stats.ms_h2d.
static int32_t upload_timed(sgr_engine* e, cudaEvent_t t0, cudaEvent_t t1, std::initializer_list<Upload> uploads) {
  CUDA_TRY(e, cudaEventRecord(t0, e->stream));
  for (const Upload& u : uploads) CUDA_TRY(e, cudaMemcpyAsync(u.dst, u.src, u.bytes, cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(e, cudaEventRecord(t1, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  CUDA_TRY(e, cudaEventElapsedTime(&e->stats.ms_h2d, t0, t1));
  return SGR_OK;
}

static int32_t after_load(sgr_engine* e, const uint8_t* d_events, const uint64_t* d_offsets, uint64_t nbytes, uint64_t n_agg) {
  e->d_events = d_events; e->d_offsets = d_offsets; e->event_bytes = nbytes; e->n_agg = n_agg; e->loaded = true;
  e->d_rec_offsets = nullptr; e->n_rec = 0;
  // variable records: the format caps a record at 16+512 bytes unless the caller raises
  // "max_record_bytes"; a longer record is flagged as a malformed event by the kernel, never mis-parsed
  e->max_record_bytes = e->program.record_kind == SGR_REC_VAR16 ? (uint32_t)e->opt_max_record_bytes : 64u;
  e->offsets_aligned64 = false; e->log_begin = 0; e->log_end = nbytes;
  if (e->program.record_kind == SGR_REC_FIXED64) {
    cudaError_t ce = inspect_offsets(d_offsets, n_agg, (unsigned long long*)e->counters.p, e->stream, &e->offsets_aligned64,
                                     &e->log_begin, &e->log_end, &e->max_seg_bytes);
    if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "offset inspection: %s", cudaGetErrorString(ce));
  }
  return SGR_OK;
}

int32_t sgr_load_events(sgr_engine* e, const void* events, uint64_t nbytes, const uint64_t* seg_offsets, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e || (!events && nbytes) || !seg_offsets) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program before loading events");
  if (seg_offsets[n_agg] > nbytes) return fail(e, SGR_ERR_INVALID, "seg_offsets[n_agg]=%llu exceeds nbytes=%llu",
                                               (unsigned long long)seg_offsets[n_agg], (unsigned long long)nbytes);
  for (uint64_t i = 0; i <= n_agg; ++i) {
    if (seg_offsets[i] % 16) return fail(e, SGR_ERR_INVALID, "seg_offsets[%llu] is not a multiple of 16", (unsigned long long)i);
    if (i && seg_offsets[i] < seg_offsets[i - 1]) return fail(e, SGR_ERR_INVALID, "seg_offsets not monotone at %llu", (unsigned long long)i);
  }
  int32_t rc = before_load(e); if (rc) return rc;
  CUDA_TRY(e, e->own_events.reserve(nbytes));
  CUDA_TRY(e, e->own_offsets.reserve((n_agg + 1) * 8));
  rc = upload_timed(e, e->ev0, e->ev1, {{e->own_events.p, events, nbytes}, {e->own_offsets.p, seg_offsets, (n_agg + 1) * 8}});
  if (rc) return rc;
  e->stats.ms_group = 0;
  return after_load(e, (const uint8_t*)e->own_events.p, (const uint64_t*)e->own_offsets.p, nbytes, n_agg);
}

int32_t sgr_load_events_device(sgr_engine* e, const void* d_events, uint64_t nbytes, const uint64_t* d_seg_offsets, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e || (!d_events && nbytes) || !d_seg_offsets) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program before loading events");
  if (((uintptr_t)d_events) % 16) return fail(e, SGR_ERR_INVALID, "device event log must be 16-byte aligned");
  int32_t rc = before_load(e); if (rc) return rc;
  e->stats.ms_h2d = 0; e->stats.ms_group = 0;
  return after_load(e, (const uint8_t*)d_events, d_seg_offsets, nbytes, n_agg);
}

int32_t sgr_load_events_indexed(sgr_engine* e, const void* events, uint64_t nbytes, const uint64_t* seg_offsets, uint64_t n_agg,
                                const uint64_t* rec_offsets, uint64_t n_records) {
  OpLock op_lock(e);
  if (!rec_offsets) return fail(e, SGR_ERR_INVALID, "null record directory");
  int32_t rc = sgr_load_events(e, events, nbytes, seg_offsets, n_agg);
  if (rc) return rc;
  for (uint64_t i = 0; i < n_records; ++i)
    if (rec_offsets[i + 1] < rec_offsets[i] || rec_offsets[i] % 16) return fail(e, SGR_ERR_INVALID, "record directory is not monotone / 16-byte aligned at %llu", (unsigned long long)i);
  if (rec_offsets[0] != seg_offsets[0] || rec_offsets[n_records] != seg_offsets[n_agg]) return fail(e, SGR_ERR_INVALID, "record directory and CSR cover different byte ranges");
  CUDA_TRY(e, e->own_rec_offsets.reserve((n_records + 1) * 8));
  CUDA_TRY(e, cudaMemcpyAsync(e->own_rec_offsets.p, rec_offsets, (n_records + 1) * 8, cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  e->d_rec_offsets = (const uint64_t*)e->own_rec_offsets.p; e->n_rec = n_records;
  return SGR_OK;
}

int32_t sgr_load_events_indexed_device(sgr_engine* e, const void* d_events, uint64_t nbytes, const uint64_t* d_seg_offsets, uint64_t n_agg,
                                       const uint64_t* d_rec_offsets, uint64_t n_records) {
  OpLock op_lock(e);
  if (!d_rec_offsets) return fail(e, SGR_ERR_INVALID, "null record directory");
  int32_t rc = sgr_load_events_device(e, d_events, nbytes, d_seg_offsets, n_agg);
  if (rc) return rc;
  e->d_rec_offsets = d_rec_offsets; e->n_rec = n_records;   // consistency with the CSR is checked by the kernel at every segment head
  return SGR_OK;
}

static int32_t load_unsorted_impl(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_agg) {
  if (e->program.record_kind != SGR_REC_FIXED64) return fail(e, SGR_ERR_UNSUPPORTED, "unsorted loads take fixed 64-byte records");
  if (n_agg >= (1ull << 32) || n_records >= (1ull << 32)) return fail(e, SGR_ERR_UNSUPPORTED, "group-by is limited to 2^32 records/aggregates");
  CUDA_TRY(e, e->own_events.reserve(n_records * 64));
  CUDA_TRY(e, e->own_offsets.reserve((n_agg + 1) * 8));
  CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
  unsigned long long bad = 0;
  cudaError_t ce = group_by_agg_stable(e->group, (const uint8_t*)d_records, n_records, n_agg, (uint8_t*)e->own_events.p,
                                       (uint64_t*)e->own_offsets.p, nullptr, nullptr, (unsigned long long*)e->counters.p, e->stream, &bad);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "group-by: %s", cudaGetErrorString(ce));
  CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  CUDA_TRY(e, cudaEventElapsedTime(&e->stats.ms_group, e->ev0, e->ev1));
  if (bad) return fail(e, SGR_ERR_INVALID, "%llu records carry an aggregate index >= n_agg", bad);
  return after_load(e, (const uint8_t*)e->own_events.p, (const uint64_t*)e->own_offsets.p, n_records * 64, n_agg);
}

int32_t sgr_load_unsorted_device(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e || (!d_records && n_records)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program before loading events");
  int32_t rc = before_load(e); if (rc) return rc;
  e->stats.ms_h2d = 0;
  return load_unsorted_impl(e, d_records, n_records, n_agg);
}

int32_t sgr_load_unsorted(sgr_engine* e, const void* records, uint64_t n_records, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e || (!records && n_records)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program before loading events");
  int32_t rc = before_load(e); if (rc) return rc;
  CUDA_TRY(e, e->inc_records.reserve(n_records * 64));
  rc = upload_timed(e, e->ev0, e->ev1, {{e->inc_records.p, records, n_records * 64}}); if (rc) return rc;
  return load_unsorted_impl(e, e->inc_records.p, n_records, n_agg);
}

int32_t sgr_set_initial_states(sgr_engine* e, const void* states, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e) return SGR_ERR_INVALID;
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  // NULL only says "the next fold starts from None everywhere": no device work, no wait
  if (!states) { e->states_valid = false; mark_dirty(e); return SGR_OK; }
  int32_t rc = before_load(e); if (rc) return rc;
  rc = ensure_states(e, n_agg); if (rc) return rc;
  CUDA_TRY(e, cudaMemcpyAsync(e->states.p, states, (size_t)n_agg * e->program.state_bytes, cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  e->states_valid = true;
  e->flagged.forget();
  mark_dirty(e);
  return SGR_OK;
}

static int32_t fold_begin(sgr_engine* e, bool pipelined) {
  if (!e) return SGR_ERR_INVALID;
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "no fold program registered");
  if (!e->loaded) return fail(e, SGR_ERR_NOT_LOADED, "no event log loaded");
  int32_t rc = use_device(e); if (rc) return rc;
  // back-to-back asynchronous folds of the same log are queued without a host round trip;
  // only the last one is waited on (sgr_wait) and has its statistics collected
  if (!pipelined) { rc = finish_fold(e); if (rc) return rc; }
  const bool prior = e->states_valid && e->states_n == e->n_agg;
  rc = ensure_states(e, e->n_agg); if (rc) return rc;
  rc = enqueue_fold(e, e->d_events, e->d_offsets, nullptr, e->n_agg, prior, e->event_bytes, e->offsets_aligned64, e->log_begin, e->log_end);
  if (rc) return rc;
  e->states_valid = true;
  e->flagged.forget();
  mark_dirty(e);
  return SGR_OK;
}

int32_t sgr_fold(sgr_engine* e) {
  OpLock op_lock(e);
  int32_t rc = fold_begin(e, false); if (rc) return rc;
  return finish_fold(e);
}

int32_t sgr_fold_async(sgr_engine* e) { OpLock op_lock(e); return fold_begin(e, true); }

int32_t sgr_wait(sgr_engine* e) {
  OpLock op_lock(e);
  if (!e) return SGR_ERR_INVALID;
  int32_t rc = use_device(e); if (rc) return rc;
  return finish_fold(e);
}

// Exact replay of the slots that saw a throwing event in a sort-free fold: the batch is grouped once (K5) and exactly those
// slots are folded sequentially onto their untouched prior states (exact err_idx, state kept: PersistentActor.scala:260-263).
// h_throwing / h_dropped: aggregates in error, events dropped after their throw.
static int32_t replay_throwing_slots(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_agg, const uint32_t* d_err_ids,
                                     uint64_t n_err, unsigned long long* h_throwing, unsigned long long* h_dropped) {
  DevBuf& grouped = e->group.batch_records;
  CUDA_TRY(e, grouped.reserve(n_records * 64));
  CUDA_TRY(e, e->inc_offsets.reserve((n_agg + 2) * 8));
  unsigned long long bad = 0;
  cudaError_t ce = group_by_agg_stable(e->group, (const uint8_t*)d_records, n_records, n_agg, (uint8_t*)grouped.p, (uint64_t*)e->inc_offsets.p,
                                       nullptr, nullptr, (unsigned long long*)e->counters.p, e->stream, &bad);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "group-by (replay): %s", cudaGetErrorString(ce));
  CUDA_TRY(e, cudaMemsetAsync(e->counters.p, 0, 64, e->stream));
  FoldArgs a{};
  a.events = (const uint8_t*)grouped.p; a.seg_offsets = (const uint64_t*)e->inc_offsets.p; a.n_seg = n_err;
  a.seg_list = d_err_ids; a.states_in = (const uint8_t*)e->states.p; a.states_out = (uint8_t*)e->states.p;
  a.counters = (unsigned long long*)e->counters.p;
  FoldLaunchInfo info{};
  cudaError_t le2 = launch_fold_stream(a, e->dprog, -1, e->num_sms, e->max_record_bytes, e->stream, &info);
  if (le2 != cudaSuccess) return fail(e, SGR_ERR_CUDA, "replay launch: %s", cudaGetErrorString(le2));
  unsigned long long h2[8];
  CUDA_TRY(e, cudaMemcpyAsync(h2, e->counters.p, 64, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  *h_throwing = h2[1]; *h_dropped = h2[4];
  return SGR_OK;
}

// Enqueue the clear of the flags e->flagged names, before an operation sets its own. The atomic micro-batch (`atomic`) clears a
// device list in its own kernel and clears nothing on a fresh table; it gets back the bound on the list it is to clear (0:
// none). Every other operation clears a host list, or else the whole table.
static uint32_t clear_flagged(sgr_engine* e, bool atomic) {
  const FlaggedRows& f = e->flagged;
  if (atomic && f.kind == FlaggedRows::kDeviceList) return f.upper;
  if (atomic && f.kind == FlaggedRows::kNothing) return 0;
  const bool list = !atomic && f.kind == FlaggedRows::kHostList;
  clear_batch_flags((uint8_t*)e->states.p, e->program.state_bytes, list ? (const uint32_t*)e->inc_prev_ids.p : nullptr, list ? f.n : e->states_n,
                    e->stream);
  return 0;
}

// The program folds sort-free on integer atomics (incremental.cu, bulk_fold.cu), both as micro-batches and as arrival-order logs.
// (a 16-byte state that is one JVM Double compares with ==, not bitwise: it takes the sort-based path)
static bool folds_sort_free(const sgr_engine* e) {
  return e->row_ok && e->row_prog.user_words == 2 && e->row_prog.cls == 0 && !e->row_prog.f64_mask && e->opt_kernel != 1 &&
         e->opt_kernel != 3 && e->opt_incremental != 1;
}

// sort-free path for programs inside the transformer algebra (incremental.cu)
static int32_t fold_incremental_atomic(sgr_engine* e, const void* d_records, uint64_t n_records) {
  const uint64_t n_agg = e->states_n;
  if (n_records >= (1ull << 32)) return fail(e, SGR_ERR_UNSUPPORTED, "micro-batches are limited to 2^32 records");
  if (e->inc_scratch_slots != n_agg) {
    CUDA_TRY(e, e->inc_scratch.reserve(inc_scratch_bytes(n_agg)));
    CUDA_TRY(e, cudaMemsetAsync(e->inc_scratch.p, 0, inc_scratch_bytes(n_agg), e->stream));
    e->inc_scratch_slots = n_agg;
  }
  // sized by the table, not by the batch: the previous batch's list must survive a larger next batch
  CUDA_TRY(e, e->inc_touched[0].reserve((n_agg + 1) * 4)); CUDA_TRY(e, e->inc_touched[1].reserve((n_agg + 1) * 4));
  CUDA_TRY(e, e->inc_err_ids.reserve((n_agg + 1) * 4));
  CUDA_TRY(e, e->inc_counters.reserve(256));
  const int next = e->flagged.next;
  unsigned long long* cur = (unsigned long long*)e->inc_counters.p + 8 * next;
  unsigned long long* prev = (unsigned long long*)e->inc_counters.p + 8 * (next ^ 1);
  CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
  CUDA_TRY(e, cudaMemsetAsync(cur, 0, 64, e->stream));
  const uint32_t prev_upper = clear_flagged(e, true);
  cudaError_t le = launch_incremental_atomic((const uint8_t*)d_records, (uint32_t)n_records, n_agg, e->inc_scratch.p, (uint8_t*)e->states.p,
                                             (uint32_t*)e->inc_touched[next].p, (uint32_t*)e->inc_err_ids.p,
                                             (const uint32_t*)e->inc_touched[next ^ 1].p, prev + 5, prev_upper, e->row_prog, cur, (unsigned long long)e->opt_replay_budget, e->stream);
  if (le != cudaSuccess) return fail(e, SGR_ERR_CUDA, "incremental launch: %s", cudaGetErrorString(le));
  CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  unsigned long long h[8];
  CUDA_TRY(e, cudaMemcpyAsync(h, cur, 64, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  CUDA_TRY(e, cudaEventElapsedTime(&e->stats.ms_fold, e->ev0, e->ev1));
  if (h[4]) return fail(e, SGR_ERR_INVALID, "%llu records carry an aggregate index >= n_agg; the batch was not applied", h[4]);
  if (h[2]) {
    // too many throwing slots to re-scan the batch for each: group the batch once and replay exactly those slots
    // on the sequential kernel (their states are still the pre-batch ones)
    unsigned long long thr = 0, drop = 0;
    int32_t rr = replay_throwing_slots(e, d_records, n_records, n_agg, (const uint32_t*)e->inc_err_ids.p, h[3], &thr, &drop);
    if (rr) return rr;
    h[1] = thr; h[6] = drop;   // throwing slots, events dropped after their throw
  }
  e->flagged.device_list((uint32_t)h[5]);
  e->stats.ms_group = 0;
  e->stats.n_aggregates = h[5]; e->stats.n_errors = h[1]; e->stats.n_events = n_records - h[6];
  e->stats.event_bytes = n_records * 64; e->stats.n_long_segments = 0;
  e->stats.algorithmic_bytes = n_records * 64 + 2 * (uint64_t)e->program.state_bytes * h[5];
  e->stats.fold_launches = 1;
  mark_dirty(e);
  return SGR_OK;
}

// holes: the batch is a poll of the device ingest, whose dropped records stay in place with agg == ~0, and n_live of its
// records are not holes. The sort-free kernel skips holes; the group-by leaves them out of the CSR, so they are neither folded,
// nor counted as events, nor in err_idx. A grouped poll without live records folds nothing: the last fold's flags stay.
static int32_t fold_incremental_impl(sgr_engine* e, const void* d_records, uint64_t n_records, bool holes, uint64_t n_live) {
  if (e->program.record_kind != SGR_REC_FIXED64) return fail(e, SGR_ERR_UNSUPPORTED, "incremental batches take fixed 64-byte records");
  if (!e->states_valid) return fail(e, SGR_ERR_NOT_LOADED, "incremental fold needs a live state table (fold or set_initial_states first)");
  { int32_t rc0 = finish_fold(e); if (rc0) return rc0; }
  if (folds_sort_free(e)) return fold_incremental_atomic(e, d_records, n_records);
  const uint64_t n_agg = e->states_n;
  if (holes && (n_agg >= (1ull << 32) || n_records >= (1ull << 32)))
    return fail(e, SGR_ERR_UNSUPPORTED, "group-by is limited to 2^32 records/aggregates");
  if (holes && n_live == 0) return SGR_OK;
  if (e->flagged.kind != FlaggedRows::kHostList) e->flagged.forget();   // this batch rewrites rows a device list does not name
  CUDA_TRY(e, e->inc_offsets.reserve((n_records + 2) * 8));
  CUDA_TRY(e, e->inc_ids.reserve((n_records + 1) * 4));
  DevBuf& grouped = e->group.batch_records;
  CUDA_TRY(e, grouped.reserve(n_records * 64));
  CUDA_TRY(e, cudaEventRecord(e->ev2, e->stream));
  clear_flagged(e, false);
  unsigned long long bad = 0, n_holes = 0;
  uint64_t n_touched = 0;
  cudaError_t ce = group_by_agg_stable(e->group, (const uint8_t*)d_records, n_records, n_agg, (uint8_t*)grouped.p,
                                       (uint64_t*)e->inc_offsets.p, (uint32_t*)e->inc_ids.p, &n_touched,
                                       (unsigned long long*)e->counters.p, e->stream, &bad, holes ? &n_holes : nullptr);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "group-by: %s", cudaGetErrorString(ce));
  CUDA_TRY(e, cudaEventRecord(e->ev3, e->stream));
  if (bad) return fail(e, SGR_ERR_INVALID, "%llu records carry an aggregate index >= n_agg", bad);
  const uint64_t live_bytes = (n_records - n_holes) * 64;
  int32_t rc = enqueue_fold(e, (const uint8_t*)grouped.p, (const uint64_t*)e->inc_offsets.p, (const uint32_t*)e->inc_ids.p, n_touched, true,
                            live_bytes, true, 0, live_bytes);
  if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  CUDA_TRY(e, cudaEventElapsedTime(&e->stats.ms_group, e->ev2, e->ev3));
  std::swap(e->inc_ids, e->inc_prev_ids);
  e->flagged.host_list(n_touched);
  mark_dirty(e);
  return SGR_OK;
}

static int32_t fold_incremental_device(sgr_engine* e, const void* d_records, uint64_t n_records, bool holes, uint64_t n_live) {
  OpLock op_lock(e);
  if (!e || (!d_records && n_records)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "no fold program registered");
  int32_t rc = use_device(e); if (rc) return rc;
  e->stats.ms_h2d = 0;
  return fold_incremental_impl(e, d_records, n_records, holes, n_live);
}

int32_t sgr_fold_incremental_device(sgr_engine* e, const void* d_records, uint64_t n_records) {
  return fold_incremental_device(e, d_records, n_records, false, n_records);
}

int32_t sgr_fold_incremental(sgr_engine* e, const void* records, uint64_t n_records) {
  OpLock op_lock(e);
  if (!e || (!records && n_records)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "no fold program registered");
  int32_t rc = use_device(e); if (rc) return rc;
  CUDA_TRY(e, e->inc_records.reserve(n_records * 64));
  CUDA_TRY(e, cudaMemcpyAsync(e->inc_records.p, records, n_records * 64, cudaMemcpyHostToDevice, e->stream));
  return fold_incremental_impl(e, e->inc_records.p, n_records, false, n_records);
}

// Replace the key table (sgr_load_keys, sgr_dist_load_keys): any ingest mirror is dropped, and `rank` records whether the new
// table is a routed rank's.
static int32_t install_keys(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n_agg, bool rank) {
  std::string err;
  auto kt = std::make_shared<KeyTable>();
  if (!kt->build(keys, key_offsets, n_agg, &err)) return fail(e, SGR_ERR_INVALID, "%s", err.c_str());
  std::lock_guard<std::mutex> lk(e->keys_mu);
  e->ing_keys_from = nullptr; e->ing_key_bytes.clear(); e->ing_key_offs.clear();
  ++e->keys_epoch;
  e->rank_keys = rank;
  e->keys_stale.store(false, std::memory_order_release);
  std::atomic_store(&e->keys, std::shared_ptr<const KeyTable>(kt));
  return SGR_OK;
}

int32_t sgr_load_keys(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n_agg) {
  if (!e || !key_offsets || (!keys && n_agg && key_offsets[n_agg])) return fail(e, SGR_ERR_INVALID, "null argument");
  return install_keys(e, keys, key_offsets, n_agg, false);
}

// A new rank or partition table (sgr_dist_init, sgr_dist_set_partitions) moves the rows: the rank key table no longer names
// them, so it is dropped (sgr_get finds no id) and the reads are refused until sgr_dist_load_keys runs again.
static void drop_rank_keys(sgr_engine* e) {
  std::lock_guard<std::mutex> lk(e->keys_mu);
  if (!e->rank_keys) return;
  e->rank_keys = false;
  ++e->keys_epoch;
  std::atomic_store(&e->keys, std::shared_ptr<const KeyTable>());
}

// Grow the live table to n_agg rows (no fewer than it holds), keeping the rows of a valid table and making the others None, in a
// new buffer of at least min_bytes only when the old one is too small (no device-wide synchronisation by cudaFree otherwise).
static int32_t grow_table(sgr_engine* e, uint64_t n_agg, size_t min_bytes) {
  const size_t sb = e->program.state_bytes, need = (size_t)n_agg * sb;
  const uint64_t have = e->states_valid ? e->states_n : 0;
  if (e->states.cap < need) {
    CUDA_TRY(e, e->states.grow_keep(need > min_bytes ? need : min_bytes, have * sb, e->stream));
  }
  CUDA_TRY(e, cudaMemsetAsync((uint8_t*)e->states.p + have * sb, 0, need - have * sb, e->stream));
  e->states_n = n_agg;
  e->states_valid = true;
  return SGR_OK;
}

int32_t sgr_grow_states(sgr_engine* e, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e) return SGR_ERR_INVALID;
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  int32_t rc = use_device(e); if (rc) return rc;
  rc = before_load(e); if (rc) return rc;
  if (e->states_valid && n_agg <= e->states_n) return SGR_OK;
  rc = grow_table(e, n_agg, 0); if (rc) return rc;
  e->flagged.forget();
  mark_dirty(e);
  return SGR_OK;
}

static void* pinned_alloc(size_t n) { void* p = nullptr; return cudaHostAlloc(&p, n, cudaHostAllocPortable) == cudaSuccess ? p : nullptr; }
static void pinned_free(void* p) { cudaFreeHost(p); }

// The key table follows an append-only id dictionary kept elsewhere (host ingest, device ingest). Appends ids [first, n) of
// keys / key_offsets: first is 0 for a slice of new ids, or the ids already mirrored when they hold the owner's whole
// dictionary. A new owner starts the mirror again and bumps keys_epoch. The hash index is rebuilt lazily by the first sgr_get
// that follows (a restore polls thousands of times before anybody reads).
static void append_keys(sgr_engine* e, const void* owner, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n, bool whole_dictionary) {
  std::lock_guard<std::mutex> lk(e->keys_mu);
  if (e->ing_keys_from != owner || e->rank_keys) {
    e->ing_keys_from = owner; e->ing_key_bytes.clear(); e->ing_key_offs.assign(1, 0u); ++e->keys_epoch;
  }
  e->rank_keys = false;
  const uint64_t first = whole_dictionary ? e->ing_key_offs.size() - 1 : 0;
  if (n <= first) return;
  e->ing_key_bytes.insert(e->ing_key_bytes.end(), keys + key_offsets[first], keys + key_offsets[n]);
  const uint32_t shift = e->ing_key_offs.back() - key_offsets[first];
  const size_t old = e->ing_key_offs.size();
  e->ing_key_offs.resize(old + (n - first));
  uint32_t* dst = e->ing_key_offs.data() + old;
  for (uint64_t i = first; i < n; ++i) dst[i - first] = key_offsets[i + 1] + shift;
  e->keys_stale.store(true, std::memory_order_release);
}

int32_t sgr_append_keys(sgr_engine* e, const void* owner, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n_new) {
  if (!e || !key_offsets || (!keys && n_new && key_offsets[n_new])) return fail(e, SGR_ERR_INVALID, "null argument");
  append_keys(e, owner, keys, key_offsets, n_new, false);
  return SGR_OK;
}

int32_t sgr_fold_ingested(sgr_engine* e, sgr_ingest* g) {
  OpLock op_lock(e);
  if (!e || !g) return fail(e, SGR_ERR_INVALID, "null argument");
  { int32_t rc0 = use_device(e); if (rc0) return rc0; }
  // from now on the ingest decodes straight into page-locked memory (what is pending right now is moved once)
  if (sgr_ingest_set_allocator(g, pinned_alloc, pinned_free)) return fail(e, SGR_ERR_OOM, "ingest: %s", sgr_ingest_last_error(g));
  const void* recs = nullptr; uint64_t n_records = 0;
  const uint8_t* keys = nullptr; const uint32_t* key_offsets = nullptr; uint64_t n_keys = 0;
  if (sgr_ingest_pending(g, &recs, &n_records) || sgr_ingest_keys(g, &keys, &key_offsets, &n_keys))
    return fail(e, SGR_ERR_INVALID, "ingest: %s", sgr_ingest_last_error(g));
  { int32_t rc = grow_states_for_ids(e, n_keys, UINT64_MAX); if (rc) return rc; }
  if (n_records) { int32_t rc = sgr_fold_incremental(e, recs, n_records); if (rc) return rc; }
  if (n_keys) append_keys(e, g, keys, key_offsets, n_keys, true);
  sgr_ingest_mark_folded(g);
  return SGR_OK;
}

int32_t sgr_get_index(sgr_engine* e, uint64_t agg, void* out, uint32_t cap, uint32_t* outlen, int32_t* exists,
                      uint32_t* flags, uint32_t* err_idx) {
  if (!e) return SGR_ERR_INVALID;
  std::shared_ptr<Snapshot> s = std::atomic_load(&e->snapshot);
  if (!s || e->snapshot_dirty.load(std::memory_order_acquire)) {
    int32_t rc = refresh_snapshot(e, &s); if (rc) return rc;
  }
  if (agg >= s->n_agg) return fail(e, SGR_ERR_INVALID, "aggregate index %llu out of range", (unsigned long long)agg);
  const uint8_t* st = s->states.data() + agg * s->state_bytes;
  uint32_t fl, ei;
  memcpy(&fl, st + s->state_bytes - 8, 4); memcpy(&ei, st + s->state_bytes - 4, 4);
  const uint32_t user = s->state_bytes - 8;
  if (flags) *flags = fl;
  if (err_idx) *err_idx = ei;
  if (exists) *exists = (fl & SGR_ST_EXISTS) ? 1 : 0;
  if (outlen) *outlen = (fl & SGR_ST_EXISTS) ? user : 0;
  if ((fl & SGR_ST_EXISTS) && out) {
    if (cap < user) return fail(e, SGR_ERR_CAPACITY, "buffer of %u bytes is smaller than the state (%u)", cap, user);
    memcpy(out, st, user);
  }
  return SGR_OK;
}

int32_t sgr_get(sgr_engine* e, const uint8_t* key, uint32_t klen, void* out, uint32_t cap, uint32_t* outlen, int32_t* exists) {
  if (!e || (!key && klen)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (e->keys_stale.load(std::memory_order_acquire)) {
    std::lock_guard<std::mutex> lk(e->keys_mu);
    if (e->keys_stale.load(std::memory_order_relaxed)) {
      auto fresh = std::make_shared<KeyTable>();
      std::string err;
      if (!fresh->build(e->ing_key_bytes.data(), e->ing_key_offs.data(), e->ing_key_offs.size() - 1, &err)) return fail(e, SGR_ERR_INVALID, "%s", err.c_str());
      std::atomic_store(&e->keys, std::shared_ptr<const KeyTable>(fresh));
      e->keys_stale.store(false, std::memory_order_release);
    }
  }
  std::shared_ptr<const KeyTable> kt = std::atomic_load(&e->keys);
  int64_t idx = kt ? kt->find(key, klen) : -1;
  if (idx < 0) {  // unknown aggregate id: Option.empty, like a KTable miss
    if (exists) *exists = 0;
    if (outlen) *outlen = 0;
    // still surface "store not readable" the way the reference does
    std::shared_ptr<Snapshot> s = std::atomic_load(&e->snapshot);
    if (!s || e->snapshot_dirty.load(std::memory_order_acquire)) { int32_t rc = refresh_snapshot(e, &s); if (rc) return rc; }
    return SGR_OK;
  }
  return sgr_get_index(e, (uint64_t)idx, out, cap, outlen, exists, nullptr, nullptr);
}

static size_t round16(size_t v) { return (v + 15) & ~(size_t)15; }

// Grow the page-locked staging buffer to at least `bytes` (1.5x, so that slowly growing pages do not reallocate every time). The
// old block is freed before the new one is allocated: the stream must not be reading from or writing to gb_host.
static int32_t ensure_pinned(sgr_engine* e, size_t bytes) {
  if (bytes > e->gb_host.cap) CUDA_TRY(e, e->gb_host.alloc(bytes + bytes / 2, cudaHostAllocPortable));
  return SGR_OK;
}

// Whether the rows of e are named by its key table: always on one engine, on a routed one only under a rank key table.
static bool keys_name_rows(sgr_engine* e) {
  if (!e->dist) return true;
  std::lock_guard<std::mutex> lk(e->keys_mu);
  return e->rank_keys;
}

// The start of every device read, in this order: refuse a routed engine without a rank key table, wait for an enqueued fold,
// fail before any fold, and fail a read of JSON values (`values`) without a state writer. `api`: the entry point's name without
// "sgr_". Caller holds op_mu.
static int32_t begin_read(sgr_engine* e, const char* api, bool values) {
  if (!keys_name_rows(e))
    return fail(e, SGR_ERR_UNSUPPORTED, "the rows of a routed engine are local slots: sgr_%s does not map them to ids without a "
                "rank key table (call sgr_dist_load_keys)", api);
  int32_t rc = use_device(e); if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  if (!e->states_valid) return fail(e, SGR_ERR_STATE, "state store is not readable: no fold has completed");
  if (values && !e->writer.n) return fail(e, SGR_ERR_STATE, "sgr_%s: no state writer is set (sgr_set_state_writer)", api);
  return SGR_OK;
}

// Bring the device id index up to the key table sgr_get would read (the ids an ingest appended, else the table of
// sgr_load_keys, or none): ids appended since the last call are staged at the front of the page-locked buffer and inserted; a
// replaced table is indexed from id 0. Also makes room for `host_extra` page-locked bytes behind the staged ids (the caller's,
// at gb_host.p + gb_host.cap - host_extra) and `dev_bytes` in gb_dev, whose words before kCtlCut are zeroed for the insert's
// control words. Enqueued on the stream only: the caller synchronises and hands those words to id_index_settle. Caller holds
// op_mu, and the stream is idle.
static int32_t id_index_update(sgr_engine* e, size_t host_extra, size_t dev_bytes) {
  IdIndex& x = e->id_index;
  std::lock_guard<std::mutex> lk(e->keys_mu);
  std::shared_ptr<const KeyTable> kt;
  const uint8_t* kb = nullptr; const uint32_t* ko = nullptr; uint64_t kn = 0;
  if (!e->ing_key_offs.empty()) { kb = e->ing_key_bytes.data(); ko = e->ing_key_offs.data(); kn = e->ing_key_offs.size() - 1; }
  else if ((kt = std::atomic_load(&e->keys))) { kb = kt->bytes(); ko = kt->offsets(); kn = kt->size(); }
  if (kn >= 0xffffffffull) return fail(e, SGR_ERR_UNSUPPORTED, "the device id index holds fewer than 2^32 - 1 ids");
  if (!x.valid || x.epoch != e->keys_epoch || kn < x.n) { x.n = 0; x.arena_used = 0; x.epoch = e->keys_epoch; ++x.builds; }
  bool mono = true;
  const size_t ids = kn > x.n ? round16(id_index_stage_bytes(ko, x.n, kn, &mono)) : 0;
  if (!mono) { x.valid = false; return fail(e, SGR_ERR_INVALID, "key_offsets not monotone"); }
  int32_t rc = ensure_pinned(e, ids + host_extra); if (rc) return rc;
  CUDA_TRY(e, e->gb_dev.reserve(dev_bytes));
  CUDA_TRY(e, cudaMemsetAsync(e->gb_dev.p, 0, 8 * kCtlCut, e->stream));
  if (kn > x.n) {
    x.valid = false;   // until the insert reports no duplicate id
    cudaError_t ce = id_index_append(x, kb, ko, kn, e->gb_host.p, (unsigned long long*)e->gb_dev.p + kCtlDup, e->stream);
    if (ce != cudaSuccess) return fail(e, ce == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA, "id index: %s", cudaGetErrorString(ce));
  }
  return SGR_OK;
}

// The insert's control words, copied back after a synchronisation. Either one leaves the index to be rebuilt by the next call.
static int32_t id_index_settle(sgr_engine* e, const unsigned long long* ctl) {
  IdIndex& x = e->id_index;
  if (ctl[kCtlDup]) { x.valid = false; return fail(e, SGR_ERR_INVALID, "duplicate aggregate id in key table"); }
  if (ctl[kCtlNoSlot]) { x.valid = false; return fail(e, SGR_ERR_CUDA, "id index: %llu ids found no free slot", ctl[kCtlNoSlot]); }
  x.valid = true;
  return SGR_OK;
}

// Where read_batch_front left a batch. Device, at dd: the results (`down` bytes: the id index's control words, then indices at
// r_idx, flags at r_flags, program bytes at r_rows) | query offsets | query bytes (at q_ids). Page-locked, at hd (behind the
// staged ids and queries): room for the results, then for sgr_get_batch_values' value control words.
struct BatchRead {
  std::unique_lock<std::recursive_mutex> op_lock;
  uint8_t* hd = nullptr;
  uint8_t* dd = nullptr;
  size_t down = 0, q_ids = 0, r_idx = 0, r_flags = 0, r_rows = 0;
};

// The front of sgr_get_batch and sgr_get_batch_values, after their output checks: the key checks, begin_read, the refusal of a
// batch whose program bytes do not fit in rows_cap bytes, then (n > 0) the staging of the queries and the probe + gather.
// `values`: the batch is read as JSON values. `api`: the entry point's name without "sgr_".
static int32_t read_batch_front(sgr_engine* e, const char* api, bool values, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n,
                                uint64_t rows_cap, BatchRead* b) {
  if ((n && !key_offsets) || (n && !keys && key_offsets[n] != key_offsets[0])) return fail(e, SGR_ERR_INVALID, "null argument");
  for (uint64_t i = 0; i < n; ++i)
    if (key_offsets[i + 1] < key_offsets[i]) return fail(e, SGR_ERR_INVALID, "key_offsets not monotone at %llu", (unsigned long long)i);
  // one table generation for the whole batch: no load or fold runs while it is read, and an enqueued fold is waited for
  b->op_lock = std::unique_lock<std::recursive_mutex>(e->op_mu);
  int32_t rc = begin_read(e, api, values); if (rc) return rc;
  const uint32_t sb = e->program.state_bytes, user = sb - 8;
  if (rows_cap / user < n) return fail(e, SGR_ERR_CAPACITY, "%llu rows of %u bytes do not fit in %llu bytes", (unsigned long long)n, user, (unsigned long long)rows_cap);
  if (!n) return SGR_OK;
  const uint64_t q0 = key_offsets[0], q_bytes = key_offsets[n] - q0;
  b->q_ids = round16((n + 1) * 4);
  const size_t up = b->q_ids + round16(q_bytes);
  b->r_idx = 8 * kCtlCut; b->r_flags = b->r_idx + n * 8; b->r_rows = b->r_flags + round16(n * 4); b->down = b->r_rows + round16(n * user);
  const size_t host = up + b->down + (values ? 8 * kSvCtlWords : 0);
  rc = id_index_update(e, host, b->down + up); if (rc) return rc;
  uint8_t* hq = (uint8_t*)e->gb_host.p + (e->gb_host.cap - host);   // (behind the ids: the stream may still be copying them)
  b->hd = hq + up;
  uint8_t* dd = b->dd = (uint8_t*)e->gb_dev.p;
  uint32_t* qo = (uint32_t*)hq;
  for (uint64_t i = 0; i <= n; ++i) qo[i] = key_offsets[i] - (uint32_t)q0;
  if (q_bytes) memcpy(hq + b->q_ids, keys + q0, q_bytes);
  CUDA_TRY(e, cudaMemcpyAsync(dd + b->down, hq, up, cudaMemcpyHostToDevice, e->stream));
  cudaError_t ce = id_index_probe(e->id_index, dd + b->down + b->q_ids, (const uint32_t*)(dd + b->down), n, (long long*)(dd + b->r_idx), e->stream);
  if (ce == cudaSuccess)
    ce = id_index_gather((const uint8_t*)e->states.p, sb, e->states_n, (const long long*)(dd + b->r_idx), n, dd + b->r_rows,
                         (uint32_t*)(dd + b->r_flags), (unsigned long long*)dd + kCtlGatherBad, e->stream);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "%s launch: %s", api, cudaGetErrorString(ce));
  return SGR_OK;
}

int32_t sgr_get_batch(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n, void* out, uint64_t cap, uint32_t* flags,
                      int64_t* indices) {
  if (!e || (n && !out)) return fail(e, SGR_ERR_INVALID, "null argument");
  BatchRead b;
  int32_t rc = read_batch_front(e, "get_batch", false, keys, key_offsets, n, cap, &b);
  if (rc || !n) return rc;
  CUDA_TRY(e, cudaMemcpyAsync(b.hd, b.dd, b.down, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  const unsigned long long* ctl = (const unsigned long long*)b.hd;
  rc = id_index_settle(e, ctl); if (rc) return rc;
  if (ctl[kCtlGatherBad]) return fail(e, SGR_ERR_INVALID, "aggregate index %llu out of range", ctl[kCtlGatherBad] - 1);
  memcpy(out, b.hd + b.r_rows, n * (e->program.state_bytes - 8));
  if (flags) memcpy(flags, b.hd + b.r_flags, n * 4);
  if (indices) memcpy(indices, b.hd + b.r_idx, n * 8);
  return SGR_OK;
}

// The message of a row the state writer refuses: `what` names the row's place, ctl holds state_values_measure's control words.
static int32_t writer_refusal(sgr_engine* e, const char* api, const char* what, const unsigned long long* ctl) {
  const uint32_t member = (uint32_t)(ctl[kSvStatus] >> 8), why = (uint32_t)(ctl[kSvStatus] & 0xff);
  return fail(e, SGR_ERR_UNSUPPORTED, "%s: row %llu of the %s (aggregate %lld), member %u \"%s\": %s", api, ctl[kSvRefused], what,
              (long long)ctl[kSvIndex], member, member < e->writer_names.size() ? e->writer_names[member].c_str() : "", sw::reason_text(why));
}

int32_t sgr_set_state_writer(sgr_engine* e, const sgr_json_field* members, uint32_t n_members) {
  OpLock op_lock(e);
  if (!e || (n_members && !members)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program before its state writer");
  if (!keys_name_rows(e))
    return fail(e, SGR_ERR_UNSUPPORTED, "the rows of a routed engine are local slots: a state writer does not map ids to them without "
                "a rank key table (call sgr_dist_load_keys)");
  if (n_members > sw::kMaxMembers) return fail(e, SGR_ERR_INVALID, "%u members: a state writer takes at most %u", n_members, sw::kMaxMembers);
  const uint32_t user = e->program.state_bytes - 8;
  SwWriter w{};
  std::vector<uint8_t> lits;
  std::vector<std::string> names;
  bool has_id = false;
  for (uint32_t i = 0; i < n_members; ++i) {
    const sgr_json_field& f = members[i];
    const size_t nl = f.name ? strlen(f.name) : 0;
    if (!nl || !sw::utf8_ok((const uint8_t*)f.name, nl)) return fail(e, SGR_ERR_INVALID, "member %u: the name is empty or not well-formed UTF-8", i);
    for (uint32_t k = 0; k < i; ++k)
      if (names[k] == f.name) return fail(e, SGR_ERR_INVALID, "member %u: the name \"%s\" is member %u's too", i, f.name, k);
    sw::Member& m = w.m[i];
    m.kind = f.kind;
    if (f.kind == SGR_JSON_ID) {
      if (has_id) return fail(e, SGR_ERR_INVALID, "member %u: a second SGR_JSON_ID member", i);
      has_id = true;
    } else {
      // the checks of a state topic's JSON member table (sgr_dingest_set_json_packer), so that the restore can read what is written
      const uint32_t size = f.kind == SGR_JSON_I32 ? 4u : f.kind == SGR_JSON_UUID ? 16u : f.kind == SGR_JSON_PSTR ? f.len : 8u;
      if (f.kind > SGR_JSON_PSTR || f.dst_off % 4 || size < 4 || size % 4 || (uint64_t)f.dst_off + size > user)
        return fail(e, SGR_ERR_INVALID, "member %u \"%s\": bad kind, length or program byte offset", i, f.name);
      m.off = f.dst_off;
      m.len = size;
    }
    m.lit_off = (uint32_t)lits.size();
    lits.push_back(i ? ',' : '{');
    const size_t at = lits.size();
    lits.resize(at + sw::str_len((const uint8_t*)f.name, nl));
    sw::str_write(lits.data() + at, (const uint8_t*)f.name, nl);
    lits.push_back(':');
    m.lit_len = (uint32_t)(lits.size() - m.lit_off);
    names.push_back(f.name);
  }
  int32_t rc = use_device(e); if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  // the literals go to a new buffer, moved in only on success: a failed call leaves the old writer and its literals intact
  DevBuf nb;
  if (!lits.empty()) {
    CUDA_TRY(e, nb.reserve(lits.size()));
    CUDA_TRY(e, cudaMemcpy(nb.p, lits.data(), lits.size(), cudaMemcpyHostToDevice));
  }
  e->writer_lits = std::move(nb);
  w.lits = (const uint8_t*)e->writer_lits.p;
  w.n = n_members;
  e->writer = w;
  e->writer_names = std::move(names);
  return SGR_OK;
}

int32_t sgr_get_batch_values(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n, uint8_t* values, uint64_t values_cap,
                             uint64_t* value_offsets, uint32_t* flags, int64_t* indices, uint64_t* values_len) {
  if (!e || !value_offsets || !flags || (!values && values_cap)) return fail(e, SGR_ERR_INVALID, "null argument");
  BatchRead b;
  int32_t rc = read_batch_front(e, "get_batch_values", true, keys, key_offsets, n, UINT64_MAX, &b); if (rc) return rc;
  if (!n) { value_offsets[0] = 0; if (values_len) *values_len = 0; return SGR_OK; }
  const uint8_t* dd = b.dd;
  // a query's id is the row's id: every found row has one
  const SvRows r{dd + b.r_rows, e->program.state_bytes - 8, (const uint32_t*)(dd + b.r_flags), (const long long*)(dd + b.r_idx), dd + b.down + b.q_ids,
                 (const uint32_t*)(dd + b.down), ~0ull, n};
  unsigned long long *d_offs = nullptr, *d_sv = nullptr;
  cudaError_t ce = e->sv_scratch.reserve(state_values_scratch_bytes(n));
  if (ce == cudaSuccess) ce = state_values_measure(e->writer, r, ~0ull, e->sv_scratch.p, &d_offs, &d_sv, e->stream);
  if (ce != cudaSuccess) return fail(e, ce == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA, "get_batch_values launch: %s", cudaGetErrorString(ce));
  CUDA_TRY(e, cudaMemcpyAsync(b.hd, dd, 8 * kCtlCut, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(b.hd + b.down, d_sv, 8 * kSvCtlWords, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  unsigned long long ctl[kCtlCut], sv[kSvCtlWords];
  memcpy(ctl, b.hd, sizeof ctl);
  memcpy(sv, b.hd + b.down, sizeof sv);
  rc = id_index_settle(e, ctl); if (rc) return rc;
  if (ctl[kCtlGatherBad]) return fail(e, SGR_ERR_INVALID, "aggregate index %llu out of range", ctl[kCtlGatherBad] - 1);
  if (sv[kSvRefused] < n) return writer_refusal(e, "get_batch_values", "batch", sv);
  const uint64_t total = sv[kSvBytes];
  if (total > values_cap) {
    if (values_len) *values_len = total;
    return fail(e, SGR_ERR_CAPACITY, "the batch's values need %llu bytes, values_cap is %llu", (unsigned long long)total, (unsigned long long)values_cap);
  }
  CUDA_TRY(e, e->sv_values.reserve(total));
  ce = state_values_write(e->writer, r, n, d_offs, (uint8_t*)e->sv_values.p, e->stream);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "get_batch_values launch: %s", cudaGetErrorString(ce));
  // pinned, from its start (the stream is idle): results | value offsets | values
  const size_t h_offs = b.down, h_vals = h_offs + round16((n + 1) * 8);
  rc = ensure_pinned(e, h_vals + total); if (rc) return rc;
  uint8_t* hd = (uint8_t*)e->gb_host.p;
  CUDA_TRY(e, cudaMemcpyAsync(hd, dd, b.r_rows, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(hd + h_offs, d_offs, (n + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
  if (total) CUDA_TRY(e, cudaMemcpyAsync(hd + h_vals, e->sv_values.p, total, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  memcpy(flags, hd + b.r_flags, n * 4);
  if (indices) memcpy(indices, hd + b.r_idx, n * 8);
  memcpy(value_offsets, hd + h_offs, (n + 1) * 8);
  if (total) memcpy(values, hd + h_vals, total);
  if (values_len) *values_len = total;
  return SGR_OK;
}

// What ing_keys_from names while the key table is the one sgr_put_batch appends to: ids the engine numbered itself, with no
// ingest dictionary behind them (a table of sgr_load_keys becomes one, unchanged, at the first put batch)
static const char kPutKeysOwner = 0;

// The apply of a put batch, before its kernels: the flags the previous operation left are cleared, the table grows to n_agg
// rows with the last-write words (pb_last) covering them, there is room for a touched list of n rows, and ev0 marks the start.
// Shared by sgr_put_batch and put_decoded_poll.
static int32_t put_apply_begin(sgr_engine* e, uint64_t n_agg, uint64_t n) {
  const size_t sb = e->program.state_bytes;
  if (e->states_valid) clear_flagged(e, false);
  if (n_agg > (e->states_valid ? e->states_n : 0)) {
    // capacity grows by at least half, so that batches adding a few ids each do not copy the table every time
    int32_t rc = grow_table(e, n_agg, e->states.cap + e->states.cap / 2); if (rc) return rc;
  }
  if (e->pb_last_n < e->states_n) {
    CUDA_TRY(e, e->pb_last.reserve(e->states.cap / sb * 4));
    CUDA_TRY(e, cudaMemsetAsync(e->pb_last.p, 0, e->pb_last.cap, e->stream));
    e->pb_last_n = e->pb_last.cap / 4;
  }
  CUDA_TRY(e, e->inc_ids.reserve(n * 4));   // this batch's touched list (the previous one is inc_prev_ids)
  CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
  return SGR_OK;
}

// ... and after them (ev1 recorded, the stream synchronised): n_live records wrote `touched` rows, which the next incremental
// fold or put batch clears; the statistics and the generation follow.
static int32_t put_apply_end(sgr_engine* e, uint64_t n_live, uint64_t touched) {
  const uint32_t sb = e->program.state_bytes;
  std::swap(e->inc_ids, e->inc_prev_ids);
  e->flagged.host_list(touched);
  e->stats.n_aggregates = touched; e->stats.n_events = n_live; e->stats.n_errors = 0; e->stats.n_long_segments = 0;
  e->stats.event_bytes = n_live * (sb - 8); e->stats.algorithmic_bytes = n_live * (sb - 8) + 2ull * sb * touched;
  e->stats.ms_h2d = 0; e->stats.ms_group = 0; e->stats.fold_launches = 2;
  CUDA_TRY(e, cudaEventElapsedTime(&e->stats.ms_fold, e->ev0, e->ev1));
  mark_dirty(e);
  return SGR_OK;
}

// sgr_put_batch once the batch's ids are resolved and known to fit (p: the batch on the device, n_new new ids taking
// new_aligned arena bytes; its positions come back at hd + r_pos and its control words at hd + r_pb). Applies it and appends the
// new ids to the host key table. On failure the caller has the id index rebuilt from the host key table, which is unchanged.
static int32_t put_batch_commit(sgr_engine* e, const PutBatch& p, uint64_t n_new, uint64_t new_aligned, const uint8_t* keys,
                                const uint32_t* key_offsets, uint8_t* hd, size_t r_pb, size_t r_pos) {
  IdIndex& x = e->id_index;
  const uint64_t n = p.n, n_keys = p.n_keys;
  int32_t rc = put_apply_begin(e, n_keys + n_new, n); if (rc) return rc;
  x.arena_used += new_aligned;
  cudaError_t ce = id_index_insert(x, n_keys + n_new, (unsigned long long*)e->gb_dev.p + kCtlDup, e->stream);
  if (ce == cudaSuccess) ce = put_batch_apply(p, (uint8_t*)e->states.p, e->dprog, (uint32_t*)e->pb_last.p, (uint32_t*)e->inc_ids.p, e->stream);
  if (ce != cudaSuccess) return fail(e, ce == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA, "put_batch: %s", cudaGetErrorString(ce));
  CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(hd, e->gb_dev.p, 8 * kCtlCut, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(hd + r_pb, p.ctl, 64, cudaMemcpyDeviceToHost, e->stream));
  if (n_new) CUDA_TRY(e, cudaMemcpyAsync(hd + r_pos, p.new_pos, n_new * 4, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  unsigned long long ctl[kCtlCut], pb[8];
  memcpy(ctl, hd, sizeof ctl);
  memcpy(pb, hd + r_pb, sizeof pb);
  rc = id_index_settle(e, ctl); if (rc) return rc;
  {
    std::lock_guard<std::mutex> lk(e->keys_mu);
    if (e->ing_keys_from != &kPutKeysOwner) {
      // the table of sgr_load_keys (or none) goes on as the put batches' table: same ids, same epoch, the index stays
      std::shared_ptr<const KeyTable> kt = std::atomic_load(&e->keys);
      const uint64_t kn = kt ? kt->size() : 0;
      e->ing_key_bytes.assign(kn ? kt->bytes() : nullptr, kn ? kt->bytes() + kt->offsets()[kn] : nullptr);
      if (kn) e->ing_key_offs.assign(kt->offsets(), kt->offsets() + kn + 1);
      else e->ing_key_offs.assign(1, 0u);
      e->ing_keys_from = &kPutKeysOwner;
    }
    const uint32_t* pos = (const uint32_t*)(hd + r_pos);
    for (uint64_t k = 0; k < n_new; ++k) {
      const uint32_t b = key_offsets[pos[k]], len = key_offsets[pos[k] + 1] - b;
      e->ing_key_bytes.insert(e->ing_key_bytes.end(), keys + b, keys + b + len);
      e->ing_key_offs.push_back(e->ing_key_offs.back() + len);
    }
    if (n_new) e->keys_stale.store(true, std::memory_order_release);
  }
  return put_apply_end(e, n, pb[kPbTouched]);
}

int32_t sgr_put_batch(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n, const void* rows, const uint8_t* present,
                      uint64_t* n_new_ids) {
  if (!e || (n && (!key_offsets || !rows || !present)) || (n && !keys && key_offsets[n] != key_offsets[0]))
    return fail(e, SGR_ERR_INVALID, "null argument");
  if (n >= (1ull << 32)) return fail(e, SGR_ERR_UNSUPPORTED, "a put batch holds fewer than 2^32 records");
  uint64_t q_aligned = 0;   // the batch's ids as arena entries
  for (uint64_t i = 0; i < n; ++i) {
    if (key_offsets[i + 1] < key_offsets[i]) return fail(e, SGR_ERR_INVALID, "key_offsets not monotone at %llu", (unsigned long long)i);
    q_aligned += ((uint64_t)(key_offsets[i + 1] - key_offsets[i]) + 7) & ~7ull;
  }
  if (n_new_ids) *n_new_ids = 0;
  if (!n) return SGR_OK;
  OpLock op_lock(e);
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  if (e->dist) return fail(e, SGR_ERR_UNSUPPORTED, "the rows of a routed engine are local slots: sgr_put_batch does not map ids to them");
  uint64_t key_bytes = 0;
  {
    std::lock_guard<std::mutex> lk(e->keys_mu);
    if (e->ing_keys_from && e->ing_keys_from != &kPutKeysOwner)
      return fail(e, SGR_ERR_STATE, "the key table mirrors an ingest's id dictionary, which numbers new ids itself");
    std::shared_ptr<const KeyTable> kt;
    if (!e->ing_key_offs.empty()) key_bytes = e->ing_key_offs.back();
    else if ((kt = std::atomic_load(&e->keys))) key_bytes = kt->size() ? kt->offsets()[kt->size()] : 0;
  }
  int32_t rc = use_device(e); if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  const uint32_t user = e->program.state_bytes - 8;
  // page-locked and device alike: offsets (from 0) | id bytes | rows | tombstone marks, one copy up; back come the index's
  // control words, the batch's (PutBatch::ctl) and the new ids' positions
  const uint64_t q0 = key_offsets[0], q_bytes = key_offsets[n] - q0;
  const size_t o_ids = round16((n + 1) * 4), o_rows = o_ids + round16(q_bytes), o_present = o_rows + round16(n * user), up = o_present + round16(n);
  const size_t r_pb = 8 * kCtlCut, r_pos = r_pb + 64, down = r_pos + round16(n * 4);
  rc = id_index_update(e, up + down, kPayloadOff + up); if (rc) return rc;
  IdIndex& x = e->id_index;
  uint8_t* hq = (uint8_t*)e->gb_host.p + (e->gb_host.cap - up - down);   // (behind the ids the index update may still be copying)
  uint8_t* hd = hq + up;
  uint32_t* qo = (uint32_t*)hq;
  for (uint64_t i = 0; i <= n; ++i) qo[i] = key_offsets[i] - (uint32_t)q0;
  if (q_bytes) memcpy(hq + o_ids, keys + q0, q_bytes);
  memcpy(hq + o_rows, rows, n * user);
  memcpy(hq + o_present, present, n);
  uint8_t* dd = (uint8_t*)e->gb_dev.p + kPayloadOff;
  CUDA_TRY(e, cudaMemcpyAsync(dd, hq, up, cudaMemcpyHostToDevice, e->stream));
  PutBatch p;
  p.offs = (const uint32_t*)dd; p.ids = dd + o_ids; p.rows = dd + o_rows; p.present = dd + o_present;
  p.n = (uint32_t)n; p.n_keys = x.n;
  CUDA_TRY(e, e->pb_scratch.reserve(put_batch_scratch_bytes(n)));
  put_batch_carve(p, e->pb_scratch.p, n);
  // every id of the batch may be new: room for their refs and bytes behind the resident ones, which do not move
  cudaError_t ce = id_index_reserve(x, x.n + n, x.arena_used + q_aligned + 8, e->stream);
  if (ce == cudaSuccess) ce = put_batch_resolve(x, x.arena_used, p, e->stream);
  if (ce != cudaSuccess) { x.valid = false; return fail(e, ce == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA, "put_batch: %s", cudaGetErrorString(ce)); }
  CUDA_TRY(e, cudaMemcpyAsync(hd, e->gb_dev.p, 8 * kCtlCut, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(hd + r_pb, p.ctl, 64, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  unsigned long long ctl[kCtlCut], pb[8];
  memcpy(ctl, hd, sizeof ctl);
  memcpy(pb, hd + r_pb, sizeof pb);
  rc = id_index_settle(e, ctl); if (rc) return rc;
  if (pb[kPbFull]) return fail(e, SGR_ERR_CUDA, "put_batch: %llu ids found no slot in the batch table", pb[kPbFull]);
  // nothing is applied yet: the limits of the key table are checked against the exact new ids
  const uint64_t n_new = pb[kPbNewIds];
  if (x.n + n_new >= 0xffffffffull)
    return fail(e, SGR_ERR_CAPACITY, "%llu ids and %llu new ones: a key table holds fewer than 2^32 - 1 ids", (unsigned long long)x.n,
                (unsigned long long)n_new);
  if (key_bytes + pb[kPbNewBytes] > 0xffffffffull)
    return fail(e, SGR_ERR_CAPACITY, "%llu id bytes and %llu new ones: a key table holds at most 4 GiB of ids", (unsigned long long)key_bytes,
                pb[kPbNewBytes]);
  rc = put_batch_commit(e, p, n_new, pb[kPbNewIds + 1], keys, key_offsets, hd, r_pb, r_pos);
  if (rc) { x.valid = false; return rc; }
  if (n_new_ids) *n_new_ids = n_new;
  return SGR_OK;
}

// The table generation and the key-table epoch a page is read against (generation >= 1 once a table exists).
static uint64_t changes_token(uint64_t generation, uint64_t keys_epoch) { return ((generation & ((1ull << 40) - 1)) << 24) | (keys_epoch & 0xffffffull); }

// The caller's arrays for one page: id_offsets and either rows or the values triple (values, values_cap, value_offsets) are
// always written, a null flags, err_idx or indices is skipped.
struct PageOut {
  void* rows; uint32_t* flags; uint32_t* err_idx; int64_t* indices; uint8_t* ids; uint32_t* id_offsets;
  uint8_t* values; uint64_t values_cap; uint64_t* value_offsets;
};

// One page of sgr_export_changes or sgr_scan, from the page cut's words (`cut`, back on the host) to the caller's arrays. The cut
// ran in nt tiles (0: none, the page is empty) over positions [lo, hi), the row at position p being map[p] (p without a map).
// Compaction, id_index_gather and changes_copy_ids fill a device block sized by the page, and one copy and one synchronisation
// bring it back. *stop: the first selected position that did not fit (hi when every one did). The stream is idle on entry.
// With out.values the page's rows become JSON values (state_values.cuh): one more read-back brings the fit, and the page ends
// before the first row whose value does not fit in values_cap. Under a map, such a page reports *stop = lo, which is below hi:
// only that comparison is read (a scan resumes from the page's last id).
static int32_t fetch_page(sgr_engine* e, const char* api, const uint32_t* map, uint32_t select, uint64_t lo, uint64_t hi, uint64_t nt,
                          const unsigned long long* cut, uint64_t ids_cap, const PageOut& out, uint64_t* n_rows, uint64_t* stop) {
  const uint64_t page = nt ? cut[kChCtlRows] : 0, bytes = nt ? cut[kChCtlBytes] : 0;
  uint64_t end = nt ? cut[kChCtlNext] : hi;
  if (!page && end < hi)
    return fail(e, SGR_ERR_CAPACITY, map ? "the id at position %llu of the order does not fit in %llu id bytes" : "the id of aggregate %llu does not fit in %llu id bytes",
                (unsigned long long)end, (unsigned long long)ids_cap);
  uint64_t rows_out = page;
  if (page) {
    const uint32_t sb = e->program.state_bytes, user = sb - 8;
    // device and page-locked alike: indices | flags | err_idx | id offsets | program bytes | ids, then (values) value offsets
    // and values
    const size_t o_fl = round16(page * 8), o_err = o_fl + round16(page * 4), o_off = o_err + round16(page * 4);
    const size_t o_rows = o_off + round16((page + 1) * 4), o_ids = o_rows + round16(page * user), total = o_ids + round16(bytes);
    CUDA_TRY(e, e->gb_dev.reserve(kPayloadOff + total));
    int32_t rc = ensure_pinned(e, total + 8 * kSvCtlWords); if (rc) return rc;
    const IdIndex& x = e->id_index;
    const uint2* key_ref = (const uint2*)x.key_ref.p;
    const uint8_t* states = (const uint8_t*)e->states.p;
    uint8_t* dd = (uint8_t*)e->gb_dev.p + kPayloadOff;
    cudaError_t ce = changes_compact(states, sb, e->states_n, map, key_ref, x.n, select, lo, hi, (const unsigned long long*)e->ch_tiles.p, nt,
                                     cut[kChCtlTiles], page, (long long*)dd, (uint32_t*)(dd + o_err), (uint32_t*)(dd + o_off), e->stream);
    // (every compacted index is below n_agg: the gather's out-of-range word stays unread)
    if (ce == cudaSuccess)
      ce = id_index_gather(states, sb, e->states_n, (const long long*)dd, page, dd + o_rows, (uint32_t*)(dd + o_fl),
                           (unsigned long long*)e->gb_dev.p + kCtlGatherBad, e->stream);
    if (ce == cudaSuccess)
      ce = changes_copy_ids((const long long*)dd, (const uint32_t*)(dd + o_off), page, key_ref, (const uint8_t*)x.arena.p, x.n, dd + o_ids, e->stream);
    if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "%s launch: %s", api, cudaGetErrorString(ce));
    const unsigned long long* d_offs = nullptr;
    uint64_t value_bytes = 0;
    if (out.value_offsets) {
      const SvRows r{dd + o_rows, user, (const uint32_t*)(dd + o_fl), (const long long*)dd, dd + o_ids, (const uint32_t*)(dd + o_off), x.n, page};
      CUDA_TRY(e, e->sv_scratch.reserve(state_values_scratch_bytes(page)));
      unsigned long long *offs = nullptr, *dctl = nullptr;
      ce = state_values_measure(e->writer, r, out.values_cap, e->sv_scratch.p, &offs, &dctl, e->stream);
      if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "%s launch: %s", api, cudaGetErrorString(ce));
      CUDA_TRY(e, cudaMemcpyAsync(e->gb_host.p, dctl, 8 * kSvCtlWords, cudaMemcpyDeviceToHost, e->stream));
      CUDA_TRY(e, cudaStreamSynchronize(e->stream));
      unsigned long long sv[kSvCtlWords];
      memcpy(sv, e->gb_host.p, sizeof sv);
      if (sv[kSvRefused] < sv[kSvRows]) return writer_refusal(e, api, "page", sv);
      if (!sv[kSvRows])
        return fail(e, SGR_ERR_CAPACITY, "%s: the value of the page's first row does not fit in %llu value bytes", api, (unsigned long long)out.values_cap);
      rows_out = sv[kSvRows];
      value_bytes = sv[kSvBytes];
      d_offs = offs;
      CUDA_TRY(e, e->sv_values.reserve(value_bytes));
      ce = state_values_write(e->writer, r, rows_out, offs, (uint8_t*)e->sv_values.p, e->stream);
      if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "%s launch: %s", api, cudaGetErrorString(ce));
      rc = ensure_pinned(e, total + round16((rows_out + 1) * 8) + value_bytes); if (rc) return rc;
    }
    const uint8_t* hd = (const uint8_t*)e->gb_host.p;
    const size_t h_voff = total, h_vals = h_voff + round16((rows_out + 1) * 8);
    CUDA_TRY(e, cudaMemcpyAsync(e->gb_host.p, dd, total, cudaMemcpyDeviceToHost, e->stream));
    if (d_offs) {
      CUDA_TRY(e, cudaMemcpyAsync((uint8_t*)e->gb_host.p + h_voff, d_offs, (rows_out + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
      if (value_bytes) CUDA_TRY(e, cudaMemcpyAsync((uint8_t*)e->gb_host.p + h_vals, e->sv_values.p, value_bytes, cudaMemcpyDeviceToHost, e->stream));
    }
    CUDA_TRY(e, cudaStreamSynchronize(e->stream));
    if (rows_out < page) end = map ? lo : (uint64_t)((const int64_t*)hd)[rows_out];
    if (out.indices) memcpy(out.indices, hd, rows_out * 8);
    if (out.flags) memcpy(out.flags, hd + o_fl, rows_out * 4);
    if (out.err_idx) memcpy(out.err_idx, hd + o_err, rows_out * 4);
    memcpy(out.id_offsets, hd + o_off, (rows_out + 1) * 4);
    const uint32_t id_bytes = ((const uint32_t*)(hd + o_off))[rows_out];
    if (out.rows) memcpy(out.rows, hd + o_rows, rows_out * user);
    if (id_bytes) memcpy(out.ids, hd + o_ids, id_bytes);
    if (d_offs) {
      memcpy(out.value_offsets, hd + h_voff, (rows_out + 1) * 8);
      if (value_bytes) memcpy(out.values, hd + h_vals, value_bytes);
    }
  } else {
    out.id_offsets[0] = 0;
    if (out.value_offsets) out.value_offsets[0] = 0;
  }
  *n_rows = rows_out;
  *stop = end;
  return SGR_OK;
}

// sgr_export_changes and sgr_export_changes_values after their argument checks (api: the name without "sgr_")
static int32_t export_changes_page(sgr_engine* e, const char* api, uint32_t select, sgr_changes_cursor* cur, uint64_t max_rows, uint64_t ids_cap,
                                   const PageOut& out, uint64_t* n_rows) {
  if (!select || (select & ~(uint32_t)(SGR_ST_CHANGED | SGR_ST_ERROR)))
    return fail(e, SGR_ERR_INVALID, "select 0x%x is not a non-empty subset of SGR_ST_CHANGED | SGR_ST_ERROR", select);
  if (!max_rows) return fail(e, SGR_ERR_INVALID, "max_rows is 0");
  // one table generation per call, and the token ties the pages of one export to it
  OpLock op_lock(e);
  int32_t rc = begin_read(e, api, out.value_offsets != nullptr); if (rc) return rc;
  const uint64_t n_agg = e->states_n, next = cur->next;
  if (next > n_agg) return fail(e, SGR_ERR_INVALID, "cursor %llu is past the table's %llu aggregates", (unsigned long long)next, (unsigned long long)n_agg);
  if (n_agg >= 0xffffffffull) return fail(e, SGR_ERR_UNSUPPORTED, "sgr_export_changes reads tables of fewer than 2^32 - 1 aggregates");
  if (cur->token) {
    uint64_t epoch;
    { std::lock_guard<std::mutex> lk(e->keys_mu); epoch = e->keys_epoch; }
    if (cur->token != changes_token(e->generation.load(std::memory_order_acquire), epoch))
      return fail(e, SGR_ERR_STATE, "the table or its key table changed since the first page of this export: start again from 0");
  }
  // the id index's and the page cut's control words: they come back behind the staged ids
  const size_t ctl_bytes = 8 * kCtlRange;
  rc = id_index_update(e, ctl_bytes, ctl_bytes); if (rc) return rc;
  const IdIndex& x = e->id_index;
  const uint64_t token = changes_token(e->generation.load(std::memory_order_acquire), x.epoch);
  const uint64_t nt = (n_agg + kChangesTile - 1) / kChangesTile - next / kChangesTile;
  if (nt) CUDA_TRY(e, e->ch_tiles.reserve(nt * 16));
  cudaError_t ce = changes_count_cut((const uint8_t*)e->states.p, e->program.state_bytes, n_agg, nullptr, (const uint2*)x.key_ref.p, x.n, select, next,
                                     n_agg, nullptr, max_rows, ids_cap, (unsigned long long*)e->ch_tiles.p, (unsigned long long*)e->gb_dev.p + kCtlCut,
                                     e->stream);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "export_changes launch: %s", cudaGetErrorString(ce));
  uint8_t* hctl = (uint8_t*)e->gb_host.p + (e->gb_host.cap - ctl_bytes);
  CUDA_TRY(e, cudaMemcpyAsync(hctl, e->gb_dev.p, ctl_bytes, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  unsigned long long ctl[kCtlRange];
  memcpy(ctl, hctl, sizeof ctl);
  rc = id_index_settle(e, ctl); if (rc) return rc;
  uint64_t stop = 0;
  rc = fetch_page(e, api, nullptr, select, next, n_agg, nt, ctl + kCtlCut, ids_cap, out, n_rows, &stop);
  if (rc) return rc;
  cur->next = stop;
  cur->token = token;
  cur->n_keys = x.n;
  return SGR_OK;
}

int32_t sgr_export_changes(sgr_engine* e, uint32_t select, sgr_changes_cursor* cur, uint64_t max_rows, void* rows, uint32_t* flags,
                           uint32_t* err_idx, int64_t* indices, uint8_t* ids, uint64_t ids_cap, uint32_t* id_offsets, uint64_t* n_rows) {
  if (!e || !cur || !rows || !flags || !err_idx || !indices || !id_offsets || !n_rows || (!ids && ids_cap)) return fail(e, SGR_ERR_INVALID, "null argument");
  return export_changes_page(e, "export_changes", select, cur, max_rows, ids_cap, {rows, flags, err_idx, indices, ids, id_offsets, nullptr, 0, nullptr},
                             n_rows);
}

int32_t sgr_export_changes_values(sgr_engine* e, uint32_t select, sgr_changes_cursor* cur, uint64_t max_rows, uint8_t* values,
                                  uint64_t values_cap, uint64_t* value_offsets, uint32_t* flags, uint32_t* err_idx, int64_t* indices,
                                  uint8_t* ids, uint64_t ids_cap, uint32_t* id_offsets, uint64_t* n_rows) {
  if (!e || !cur || !value_offsets || (!values && values_cap) || !flags || !err_idx || !indices || !id_offsets || !n_rows || (!ids && ids_cap))
    return fail(e, SGR_ERR_INVALID, "null argument");
  return export_changes_page(e, "export_changes_values", select, cur, max_rows, ids_cap,
                             {nullptr, flags, err_idx, indices, ids, id_offsets, values, values_cap, value_offsets}, n_rows);
}

// sgr_scan and sgr_scan_values after their argument checks (api: the name without "sgr_")
static int32_t scan_page(sgr_engine* e, const char* api, const uint8_t* from, uint32_t from_len, int32_t from_exclusive, const uint8_t* to,
                         uint32_t to_len, uint64_t max_rows, uint64_t ids_cap, const PageOut& out, uint64_t* n_rows, int32_t* more) {
  if (!max_rows) return fail(e, SGR_ERR_INVALID, "max_rows is 0");
  // one table generation per page; pages carry no state, so a scan resumes across folds by itself
  OpLock op_lock(e);
  int32_t rc = begin_read(e, api, out.value_offsets != nullptr); if (rc) return rc;
  const uint64_t n_agg = e->states_n;
  if (n_agg >= 0xffffffffull) return fail(e, SGR_ERR_UNSUPPORTED, "sgr_scan reads tables of fewer than 2^32 - 1 aggregates");
  // the control words come back to, and the bounds' bytes (each 16-byte aligned, at kPayloadOff in gb_dev) go up from, the
  // page-locked bytes behind the ids
  const size_t q_from = from ? round16(from_len) : 0, q_to = to ? round16(to_len) : 0, extra = kPayloadOff + q_from + q_to;
  rc = id_index_update(e, extra, extra); if (rc) return rc;
  const IdIndex& x = e->id_index;
  IdOrder& o = e->id_order;
  uint8_t* hx = (uint8_t*)e->gb_host.p + (e->gb_host.cap - extra);
  unsigned long long ctl[kPayloadOff / 8];
  if (o.builds != x.builds || o.n != x.n) {
    // the order is made from the ids the index holds: the insert must have found no duplicate first
    CUDA_TRY(e, cudaMemcpyAsync(hx, e->gb_dev.p, 8 * kCtlCut, cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(e, cudaStreamSynchronize(e->stream));
    memcpy(ctl, hx, 8 * kCtlCut);
    rc = id_index_settle(e, ctl); if (rc) return rc;
    if (o.builds != x.builds) { o.n = 0; o.builds = x.builds; }
    const cudaError_t ce = id_order_update(o, (const uint2*)x.key_ref.p, (const uint8_t*)x.arena.p, x.n, e->stream);
    if (ce != cudaSuccess) return fail(e, ce == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA, "id order: %s", cudaGetErrorString(ce));
  }
  const uint64_t n = o.n;
  const uint2* key_ref = (const uint2*)x.key_ref.p;
  const uint8_t* arena = (const uint8_t*)x.arena.p;
  const uint32_t* order = (const uint32_t*)o.order.p;
  uint8_t* dd = (uint8_t*)e->gb_dev.p;
  unsigned long long* d_ctl = (unsigned long long*)dd;
  const uint64_t nt = (n + kChangesTile - 1) / kChangesTile;
  if (n) {
    if (from_len && from) memcpy(hx + kPayloadOff, from, from_len);
    if (to_len && to) memcpy(hx + kPayloadOff + q_from, to, to_len);
    if (q_from + q_to) CUDA_TRY(e, cudaMemcpyAsync(dd + kPayloadOff, hx + kPayloadOff, q_from + q_to, cudaMemcpyHostToDevice, e->stream));
    CUDA_TRY(e, e->ch_tiles.reserve(nt * 16));
    // the range is found and the page cut on the device; one read-back brings both
    cudaError_t ce = id_order_bounds(o, key_ref, arena, from ? dd + kPayloadOff : nullptr, from_len, from_exclusive != 0,
                                     to ? dd + kPayloadOff + q_from : nullptr, to_len, d_ctl + kCtlRange, e->stream);
    if (ce == cudaSuccess)
      ce = changes_count_cut((const uint8_t*)e->states.p, e->program.state_bytes, n_agg, order, key_ref, x.n, SGR_ST_EXISTS, 0, n, d_ctl + kCtlRange,
                             max_rows, ids_cap, (unsigned long long*)e->ch_tiles.p, d_ctl + kCtlCut, e->stream);
    if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "scan launch: %s", cudaGetErrorString(ce));
  }
  CUDA_TRY(e, cudaMemcpyAsync(hx, dd, kPayloadOff, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  memcpy(ctl, hx, kPayloadOff);
  rc = id_index_settle(e, ctl); if (rc) return rc;
  const uint64_t lo = n ? ctl[kCtlRange] : 0, hi = n ? ctl[kCtlRange + 1] : 0;
  uint64_t stop = 0;
  rc = fetch_page(e, api, order, SGR_ST_EXISTS, lo, hi, nt, ctl + kCtlCut, ids_cap, out, n_rows, &stop);
  if (rc) return rc;
  *more = stop < hi ? 1 : 0;
  return SGR_OK;
}

int32_t sgr_scan(sgr_engine* e, const uint8_t* from, uint32_t from_len, int32_t from_exclusive, const uint8_t* to, uint32_t to_len,
                 uint64_t max_rows, void* rows, uint32_t* flags, int64_t* indices, uint8_t* ids, uint64_t ids_cap, uint32_t* id_offsets,
                 uint64_t* n_rows, int32_t* more) {
  if (!e || !rows || !id_offsets || !n_rows || !more || (!ids && ids_cap)) return fail(e, SGR_ERR_INVALID, "null argument");
  return scan_page(e, "scan", from, from_len, from_exclusive, to, to_len, max_rows, ids_cap,
                   {rows, flags, nullptr, indices, ids, id_offsets, nullptr, 0, nullptr}, n_rows, more);
}

int32_t sgr_scan_values(sgr_engine* e, const uint8_t* from, uint32_t from_len, int32_t from_exclusive, const uint8_t* to, uint32_t to_len,
                        uint64_t max_rows, uint8_t* values, uint64_t values_cap, uint64_t* value_offsets, uint32_t* flags, int64_t* indices,
                        uint8_t* ids, uint64_t ids_cap, uint32_t* id_offsets, uint64_t* n_rows, int32_t* more) {
  if (!e || !value_offsets || (!values && values_cap) || !flags || !id_offsets || !n_rows || !more || (!ids && ids_cap))
    return fail(e, SGR_ERR_INVALID, "null argument");
  return scan_page(e, "scan_values", from, from_len, from_exclusive, to, to_len, max_rows, ids_cap,
                   {nullptr, flags, nullptr, indices, ids, id_offsets, values, values_cap, value_offsets}, n_rows, more);
}

int32_t sgr_export_states(sgr_engine* e, void* out, uint64_t cap, uint8_t* exists_bits, uint8_t* changed_bits, uint8_t* error_bits) {
  OpLock op_lock(e);
  if (!e) return SGR_ERR_INVALID;
  if (!e->states_valid) return fail(e, SGR_ERR_STATE, "no folded state table to export");
  int32_t rc = use_device(e); if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  const uint64_t n = e->states_n; const uint32_t sb = e->program.state_bytes;
  const uint64_t need = n * sb;
  std::vector<uint8_t> tmp;
  uint8_t* host = (uint8_t*)out;
  if (out) { if (cap < need) return fail(e, SGR_ERR_CAPACITY, "export needs %llu bytes, buffer has %llu", (unsigned long long)need, (unsigned long long)cap); }
  else { tmp.resize(need); host = tmp.data(); }
  CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(host, e->states.p, need, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  CUDA_TRY(e, cudaEventElapsedTime(&e->stats.ms_d2h, e->ev0, e->ev1));
  if (exists_bits || changed_bits || error_bits) {
    const uint64_t nb = (n + 7) / 8;
    if (exists_bits) memset(exists_bits, 0, nb);
    if (changed_bits) memset(changed_bits, 0, nb);
    if (error_bits) memset(error_bits, 0, nb);
    for (uint64_t i = 0; i < n; ++i) {
      uint32_t fl; memcpy(&fl, host + i * sb + sb - 8, 4);
      if (exists_bits && (fl & SGR_ST_EXISTS)) exists_bits[i >> 3] |= (uint8_t)(1u << (i & 7));
      if (changed_bits && (fl & SGR_ST_CHANGED)) changed_bits[i >> 3] |= (uint8_t)(1u << (i & 7));
      if (error_bits && (fl & SGR_ST_ERROR)) error_bits[i >> 3] |= (uint8_t)(1u << (i & 7));
    }
  }
  return SGR_OK;
}

int32_t sgr_states_device(sgr_engine* e, void** d_states, uint64_t* n_agg, uint32_t* state_bytes) {
  OpLock op_lock(e);
  if (!e) return SGR_ERR_INVALID;
  if (!e->states_valid) return fail(e, SGR_ERR_STATE, "no folded state table");
  if (d_states) *d_states = e->states.p;
  if (n_agg) *n_agg = e->states_n;
  if (state_bytes) *state_bytes = e->program.state_bytes;
  return SGR_OK;
}

int32_t sgr_events_device(sgr_engine* e, void** d_events, uint64_t* nbytes, uint64_t** d_seg_offsets) {
  if (!e) return SGR_ERR_INVALID;
  if (!e->loaded) return fail(e, SGR_ERR_NOT_LOADED, "no event log loaded");
  if (d_events) *d_events = (void*)e->d_events;
  if (nbytes) *nbytes = e->event_bytes;
  if (d_seg_offsets) *d_seg_offsets = (uint64_t*)e->d_offsets;
  return SGR_OK;
}

int32_t sgr_get_stats(sgr_engine* e, sgr_stats* out) {
  OpLock op_lock(e);
  if (!e || !out) return SGR_ERR_INVALID;
  if (e->fold_pending) { int32_t rc = use_device(e); if (rc) return rc; rc = finish_fold(e); if (rc) return rc; }
  *out = e->stats;
  return SGR_OK;
}

static int32_t ensure_bulk_buffers(sgr_engine* e, uint64_t n_agg) {
  if (e->bulk_scratch_slots != n_agg || !e->bulk_scratch.p) {
    const size_t need = bulk_scratch_bytes(e->bulk_lay, n_agg);
    CUDA_TRY(e, e->bulk_scratch.reserve(need));
    CUDA_TRY(e, cudaMemsetAsync(e->bulk_scratch.p, 0, need, e->stream));   // the finish pass leaves it zero again
    e->bulk_scratch_slots = n_agg;
  }
  CUDA_TRY(e, e->bulk_err_ids.reserve((n_agg + 1) * 4));
  CUDA_TRY(e, e->bulk_counters.reserve(64));
  return SGR_OK;
}

// Start a fresh all-None table of n rows for a fold that rebuilds it.
static int32_t fresh_table(sgr_engine* e, uint64_t n) {
  int32_t rc = ensure_states(e, n); if (rc) return rc;
  CUDA_TRY(e, cudaMemsetAsync(e->states.p, 0, (size_t)n * e->program.state_bytes, e->stream));
  e->states_valid = true;
  e->loaded = false;
  e->flagged.forget();
  return SGR_OK;
}

// The end of a sort-free bulk fold of n_records onto n_agg rows that saw n_err throwing slots: their exact replay from
// `records` (the log, contiguous, in arrival order; read only when n_err > 0), then the statistics.
static int32_t finish_bulk_fold(sgr_engine* e, const uint8_t* records, uint64_t n_records, uint64_t n_agg, uint64_t n_err, float ms_fold,
                                uint32_t fold_launches) {
  unsigned long long throwing = 0, dropped = 0;
  if (n_err) { int32_t rc = replay_throwing_slots(e, records, n_records, n_agg, (const uint32_t*)e->bulk_err_ids.p, n_err, &throwing, &dropped); if (rc) return rc; }
  e->stats.ms_group = 0; e->stats.ms_fold = ms_fold;
  e->stats.n_aggregates = n_agg; e->stats.n_errors = throwing; e->stats.n_events = n_records - dropped;
  e->stats.event_bytes = n_records * 64; e->stats.n_long_segments = 0;
  e->stats.algorithmic_bytes = n_records * 64 + (uint64_t)(16 + 2 * e->program.state_bytes) * n_agg;
  e->stats.fold_launches = fold_launches;
  mark_dirty(e);
  return SGR_OK;
}

// sort-free fold of a large arrival-order log onto the (zeroed or prior) state table: accumulate + finish (bulk_fold.cu)
static int32_t fold_bulk(sgr_engine* e, const uint8_t* d_records, uint64_t n_records, uint64_t n_agg) {
  int32_t rc = ensure_bulk_buffers(e, n_agg); if (rc) return rc;
  unsigned long long* cnt = (unsigned long long*)e->bulk_counters.p;
  CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
  CUDA_TRY(e, cudaMemsetAsync(cnt, 0, 64, e->stream));
  BulkSrc src{};
  src.n_regions = 1; src.base[0] = d_records; src.count[0] = n_records; src.rec_bytes = 64;
  cudaError_t le = launch_bulk_accumulate(src, n_agg, e->bulk_scratch.p, e->row_prog, e->bulk_lay, cnt, e->num_sms, e->stream);
  if (le == cudaSuccess) le = launch_bulk_finish(n_agg, e->bulk_scratch.p, (uint8_t*)e->states.p, (uint32_t*)e->bulk_err_ids.p, e->bulk_lay, cnt, e->stream);
  if (le != cudaSuccess) return fail(e, SGR_ERR_CUDA, "bulk fold launch: %s", cudaGetErrorString(le));
  CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  unsigned long long h[8];
  CUDA_TRY(e, cudaMemcpyAsync(h, cnt, 64, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  float ms_fold = 0;
  CUDA_TRY(e, cudaEventElapsedTime(&ms_fold, e->ev0, e->ev1));
  if (h[4]) { e->states_valid = false; return fail(e, SGR_ERR_INVALID, "%llu records carry an aggregate index >= n_agg; nothing was applied", h[4]); }
  return finish_bulk_fold(e, d_records, n_records, n_agg, h[3], ms_fold, 2);
}

// Fold an arrival-order log (aggregates interleaved, per-aggregate order kept) from None.
// class-0 programs need no grouping at all: the records are folded with integer atomics (bulk_fold.cu / incremental.cu);
// other programs are grouped stably (K5) and folded from the CSR.
static int32_t fold_arrival_order(sgr_engine* e, const uint8_t* d_records, uint64_t n_records, uint64_t n_agg) {
  int32_t rc;
  if (folds_sort_free(e) && n_records > 0) {
    rc = fresh_table(e, n_agg); if (rc) return rc;
    if (e->bulk_ok && e->opt_bulk && n_records < (1ull << 30)) return fold_bulk(e, d_records, n_records, n_agg);
    e->flagged.nothing();   // a fresh all-None table: the micro-batch kernel has no flags to clear
    rc = fold_incremental_atomic(e, d_records, n_records);
    if (rc) return rc;
    e->stats.ms_group = 0;
    return SGR_OK;
  }
  rc = load_unsorted_impl(e, d_records, n_records, n_agg);
  if (rc) return rc;
  e->states_valid = false;
  return sgr_fold(e);
}

int32_t sgr_fold_unsorted_device(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e || (!d_records && n_records)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  if (e->program.record_kind != SGR_REC_FIXED64) return fail(e, SGR_ERR_UNSUPPORTED, "arrival-order logs take fixed 64-byte records");
  int32_t rc = before_load(e); if (rc) return rc;
  e->stats.ms_h2d = 0;
  return fold_arrival_order(e, (const uint8_t*)d_records, n_records, n_agg);
}

int32_t sgr_fold_unsorted(sgr_engine* e, const void* records, uint64_t n_records, uint64_t n_agg) {
  OpLock op_lock(e);
  if (!e || (!records && n_records)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  if (e->program.record_kind != SGR_REC_FIXED64) return fail(e, SGR_ERR_UNSUPPORTED, "arrival-order logs take fixed 64-byte records");
  int32_t rc = before_load(e); if (rc) return rc;
  CUDA_TRY(e, e->inc_records.reserve(n_records * 64));
  rc = upload_timed(e, e->ev2, e->ev3, {{e->inc_records.p, records, n_records * 64}}); if (rc) return rc;
  return fold_arrival_order(e, (const uint8_t*)e->inc_records.p, n_records, n_agg);
}

// ------------------------------------------------------------------ multi-GPU
// The return code of a dist_* call, with the reason it put into err as e's error when it failed.
static int32_t dist_result(sgr_engine* e, int rc, const std::string& err) { return rc ? fail(e, rc, "%s", err.c_str()) : SGR_OK; }

// Whether e's records go through an exchange: it is one of several ranks, or a single rank with force_route.
static bool routed(const sgr_engine* e) { return e->dist && (dist_nranks(e->dist) > 1 || e->opt_force_route); }

// The exchange statistics of the last sgr_dist_route_and_fold, after its fold; ms_pipeline and the bytes per exchanged record are
// the push path's.
static void fill_dist_stats(sgr_engine* e, float ms_pipeline, uint32_t exchange_record_bytes) {
  const DistStats* ds = dist_stats(e->dist);
  e->dstats = sgr_dist_stats{};
  e->dstats.n_sent = ds->n_sent; e->dstats.n_sent_remote = ds->n_sent_remote; e->dstats.n_recv = ds->n_recv;
  e->dstats.n_local_aggregates = dist_n_local(e->dist);
  e->dstats.ms_count = ds->ms_count; e->dstats.ms_counts_exchange = ds->ms_counts_exchange;
  e->dstats.ms_scatter = ds->ms_scatter; e->dstats.ms_exchange = ds->ms_exchange;
  e->dstats.ms_group = e->stats.ms_group; e->dstats.ms_fold = e->stats.ms_fold;
  e->dstats.ms_pipeline = ms_pipeline; e->dstats.exchange_record_bytes = exchange_record_bytes;
}

int32_t sgr_dist_unique_id(void* out128) {
  if (!out128) return SGR_ERR_INVALID;
  std::string err;
  return dist_result(nullptr, dist_unique_id(out128, &err), err);
}

int32_t sgr_dist_init(sgr_engine* e, int32_t rank, int32_t nranks, const void* unique_id128, uint64_t recv_capacity_records) {
  OpLock op_lock(e);
  if (!e) return fail(e, SGR_ERR_INVALID, "null argument");   // unique_id128 == NULL with nranks > 1: a loopback rank (sgr.h)
  int32_t rc = use_device(e); if (rc) return rc;
  e->dist.reset();
  drop_rank_keys(e);
  *e->dist.put() = dist_create();
  std::string err;
  return dist_result(e, dist_init(e->dist, rank, nranks, unique_id128, recv_capacity_records, e->stream, &err), err);
}

int32_t sgr_dist_set_partitions(sgr_engine* e, const uint32_t* partition_of_agg, uint64_t n_global_agg) {
  OpLock op_lock(e);
  if (!e || !partition_of_agg) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->dist) return fail(e, SGR_ERR_NOT_LOADED, "call sgr_dist_init first");
  int32_t rc = before_load(e); if (rc) return rc;
  drop_rank_keys(e);
  std::string err;
  return dist_result(e, dist_set_partitions(e->dist, partition_of_agg, n_global_agg, e->stream, &err), err);
}

int32_t sgr_dist_load_keys(sgr_engine* e, const uint8_t* keys, const uint32_t* key_offsets, uint64_t n_global) {
  OpLock op_lock(e);
  if (!e) return SGR_ERR_INVALID;
  if (!e->dist) return fail(e, SGR_ERR_NOT_LOADED, "call sgr_dist_init first");
  if (!dist_n_global(e->dist)) return fail(e, SGR_ERR_NOT_LOADED, "no partition table: call sgr_dist_set_partitions first");
  if (!key_offsets) return fail(e, SGR_ERR_INVALID, "null argument");
  if (n_global != dist_n_global(e->dist))
    return fail(e, SGR_ERR_INVALID, "%llu ids for a partition table of %llu aggregates", (unsigned long long)n_global,
                (unsigned long long)dist_n_global(e->dist));
  for (uint64_t g = 0; g < n_global; ++g)
    if (key_offsets[g + 1] < key_offsets[g]) return fail(e, SGR_ERR_INVALID, "key_offsets not monotone at %llu", (unsigned long long)g);
  if (!keys && key_offsets[n_global] != key_offsets[0]) return fail(e, SGR_ERR_INVALID, "null argument");
  // the owned ids in local-slot order, gathered on the host: slot i holds global aggregate global_of_local[i]
  uint64_t n_local = 0;
  int32_t rc = sgr_dist_local_aggregates(e, nullptr, 0, &n_local); if (rc) return rc;
  std::vector<uint32_t> global_of_local(n_local);
  rc = sgr_dist_local_aggregates(e, global_of_local.data(), n_local, &n_local); if (rc) return rc;
  std::vector<uint32_t> offs(n_local + 1, 0u);
  for (uint64_t i = 0; i < n_local; ++i) offs[i + 1] = offs[i] + (key_offsets[global_of_local[i] + 1] - key_offsets[global_of_local[i]]);
  std::vector<uint8_t> bytes(offs[n_local]);
  for (uint64_t i = 0; i < n_local; ++i) {
    const uint32_t g = global_of_local[i];
    if (offs[i + 1] > offs[i]) memcpy(bytes.data() + offs[i], keys + key_offsets[g], offs[i + 1] - offs[i]);
  }
  return install_keys(e, bytes.data(), offs.data(), n_local, true);
}

int32_t sgr_dist_ipc_export(sgr_engine* e, void* out64) {
  OpLock op_lock(e);
  if (!e || !out64 || !e->dist) return fail(e, SGR_ERR_INVALID, "null argument / no dist state");
  int32_t rc = use_device(e); if (rc) return rc;
  std::string err;
  return dist_result(e, dist_ipc_export(e->dist, out64, &err), err);
}

int32_t sgr_dist_ipc_import(sgr_engine* e, const void* handles64_by_rank) {
  OpLock op_lock(e);
  if (!e || !handles64_by_rank || !e->dist) return fail(e, SGR_ERR_INVALID, "null argument / no dist state");
  int32_t rc = use_device(e); if (rc) return rc;
  std::string err;
  return dist_result(e, dist_ipc_import(e->dist, handles64_by_rank, &err), err);
}

int32_t sgr_dist_route_and_fold(sgr_engine* e, const void* d_records, uint64_t n_records, int32_t fused) {
  OpLock op_lock(e);
  if (!e || (!d_records && n_records)) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  if (!e->dist) return fail(e, SGR_ERR_NOT_LOADED, "call sgr_dist_init first");
  if (e->program.record_kind != SGR_REC_FIXED64) return fail(e, SGR_ERR_UNSUPPORTED, "routing takes fixed 64-byte records");
  const bool exchange = routed(e);
  // Bytes 8..15 hold the global aggregate index when a record is fed, and each exchange rewrites them on the way to the owner
  // (local index, index within the chunk, or left alone by the projection): what a program read there would depend on the
  // exchange mode. Every rank holds the same program, so every rank refuses here alike, before anything is launched.
  if (exchange)
    for (uint32_t t = 0; t < e->dprog.n_types; ++t)
      for (uint32_t i = 0; i < e->dprog.rules[t].n_ops; ++i) {
        const uint32_t op = e->dprog.rules[t].ops[i], nwords = (op >> 4) & 63u, sw = op >> 16;
        if (sw < 4u && sw + nwords > 2u)
          return fail(e, SGR_ERR_UNSUPPORTED, "rule %u op %u reads record bytes 8..15 (the aggregate index): a routed engine "
                      "rewrites them in the exchange, so a program may not read them there", t, i);
      }
  int32_t rc = before_load(e); if (rc) return rc;
  std::string err;
  uint64_t n_recv = 0;
  e->stats.ms_h2d = 0;
  // fused >= 2: pipelined push (route + exchange + fold overlapped, route_push.cu); 3 = exchange only the words the program reads.
  // Programs outside the sort-free formulation take the scatter + group-by path below (every rank holds the same program).
  if (exchange && fused >= 2 && e->bulk_ok && e->opt_incremental != 1) {
    const uint64_t n_local = dist_n_local(e->dist);
    rc = ensure_bulk_buffers(e, n_local); if (rc) return rc;
    rc = fresh_table(e, n_local); if (rc) return rc;
    PushFoldArgs pf{};
    pf.prog = &e->row_prog; pf.lay = &e->bulk_lay; pf.scratch = e->bulk_scratch.p; pf.states = (uint8_t*)e->states.p;
    pf.err_ids = (uint32_t*)e->bulk_err_ids.p; pf.counters = (unsigned long long*)e->bulk_counters.p; pf.n_slots = n_local;
    pf.n_chunks = (uint32_t)e->opt_push_chunks; pf.compact = fused == 3; pf.num_sms = e->num_sms;
    // First attempt: CTAs place their records with atomics and the records carry their own arrival index — nothing waits for
    // anything. The exact replay of a throwing aggregate needs the records in POSITIONAL log order, so if any rank saw one,
    // every rank runs the exchange again in ordered mode (look-back) and replays from that. Throwing events are the exception.
    pf.ordered = e->opt_push_ordered != 0;
    PushFoldResult res;
    // a failed exchange leaves no table, and a bulk scratch that must be cleared again
    auto push_fold = [&]() -> int32_t {
      const int32_t r = dist_result(e, dist_push_fold(e->dist, (const uint8_t*)d_records, n_records, pf, e->stream, &res, &err), err);
      if (r) { e->states_valid = false; e->bulk_scratch_slots = 0; }
      return r;
    };
    rc = push_fold(); if (rc) return rc;
    if (!pf.ordered && res.any_err_slots) {
      if (dist_is_loopback(e->dist)) {   // loopback ranks have no collective to agree over: the caller does (sgr.h)
        e->states_valid = false;
        return fail(e, SGR_ERR_AGAIN, "throwing aggregates: every rank must repeat the call with option push_ordered = 1");
      }
      CUDA_TRY(e, cudaMemsetAsync(e->states.p, 0, (size_t)n_local * e->program.state_bytes, e->stream));
      pf.ordered = true;
      rc = push_fold(); if (rc) return rc;
    }
    const uint8_t* contiguous = nullptr;
    if (res.n_err_slots) { rc = dist_result(e, dist_gather_regions(e->dist, res, e->row_prog, e->stream, &contiguous, &err), err); if (rc) return rc; }
    // ms_fold: what the fold adds behind the last push
    rc = finish_bulk_fold(e, contiguous, res.n_recv, n_local, res.n_err_slots, res.ms_total - res.ms_push, 2 * (uint32_t)e->opt_push_chunks + 1);
    if (rc) return rc;
    fill_dist_stats(e, res.ms_total, res.out_bytes);
    return SGR_OK;
  }
  if (fused >= 2) fused = dist_nranks(e->dist) > 1 ? 1 : 0;
  if (!exchange) {
    // one rank owns everything and local index == global index: no exchange
    dist_clear_stats(e->dist, n_records);
  } else {
    rc = dist_result(e, dist_route(e->dist, (const uint8_t*)d_records, n_records, fused != 0, (unsigned long long*)e->counters.p, e->stream, &n_recv, &err), err);
    if (rc) return rc;
  }
  const uint8_t* arrived = !exchange ? (const uint8_t*)d_records : dist_recv_buffer(e->dist);
  const uint64_t n_arrived = !exchange ? n_records : n_recv;
  rc = fold_arrival_order(e, arrived, n_arrived, dist_n_local(e->dist));
  if (rc) return rc;
  fill_dist_stats(e, 0, 0);
  return SGR_OK;
}

int32_t sgr_dist_get_stats(sgr_engine* e, sgr_dist_stats* out) {
  if (!e || !out) return SGR_ERR_INVALID;
  *out = e->dstats;
  return SGR_OK;
}

int32_t sgr_dist_local_aggregates(sgr_engine* e, uint32_t* out, uint64_t cap, uint64_t* n_local) {
  OpLock op_lock(e);
  if (!e || !e->dist) return fail(e, SGR_ERR_INVALID, "no dist state");
  const uint64_t n = dist_n_local(e->dist);
  if (n_local) *n_local = n;
  if (out) {
    if (cap < n) return fail(e, SGR_ERR_CAPACITY, "need room for %llu indices", (unsigned long long)n);
    int32_t rc = use_device(e); if (rc) return rc;
    CUDA_TRY(e, cudaMemcpyAsync(out, dist_global_of_local(e->dist), n * 4, cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  }
  return SGR_OK;
}

int32_t sgr_dist_set_peers(sgr_engine* e, void* const* recv_bases_by_rank) {
  OpLock op_lock(e);
  if (!e || !recv_bases_by_rank || !e->dist) return fail(e, SGR_ERR_INVALID, "null argument / no dist state");
  std::string err;
  return dist_result(e, dist_set_peers(e->dist, recv_bases_by_rank, &err), err);
}

int32_t sgr_dist_reserve(sgr_engine* e, uint64_t max_records) {
  OpLock op_lock(e);
  if (!e || !e->dist) return fail(e, SGR_ERR_INVALID, "null argument / no dist state");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  int32_t rc = use_device(e); if (rc) return rc;
  rc = before_load(e); if (rc) return rc;
  const uint64_t n_local = dist_n_local(e->dist);
  rc = ensure_states(e, n_local); if (rc) return rc;
  if (e->bulk_ok) { rc = ensure_bulk_buffers(e, n_local); if (rc) return rc; }
  std::string err;
  rc = dist_result(e, dist_push_reserve(e->dist, max_records, (uint32_t)e->opt_push_chunks, &err), err); if (rc) return rc;
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  return SGR_OK;
}

int32_t sgr_dist_recv_base(sgr_engine* e, void** base) {
  if (!e || !base || !e->dist) return fail(e, SGR_ERR_INVALID, "null argument / no dist state");
  *base = dist_recv_base(e->dist);
  return SGR_OK;
}

int32_t sgr_states_hash(sgr_engine* e, uint64_t* out) {
  OpLock op_lock(e);
  if (!e || !out) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->states_valid) return fail(e, SGR_ERR_STATE, "no folded state table");
  int32_t rc = use_device(e); if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  CUDA_TRY(e, e->hash_out.reserve(64));
  // a routed table is hashed under its GLOBAL aggregate indices, so the sum over the ranks does not depend on their number
  const uint32_t* gids = routed(e) && dist_n_local(e->dist) == e->states_n ? dist_global_of_local(e->dist) : nullptr;
  cudaError_t ce = launch_states_hash((const uint8_t*)e->states.p, e->states_n, e->program.state_bytes, gids, (unsigned long long*)e->hash_out.p, e->stream);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "hash launch: %s", cudaGetErrorString(ce));
  unsigned long long h = 0;
  CUDA_TRY(e, cudaMemcpyAsync(&h, e->hash_out.p, 8, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  *out = h;
  return SGR_OK;
}

int32_t sgr_set_option(sgr_engine* e, const char* name, int64_t value) {
  if (!e || !name) return SGR_ERR_INVALID;
  if (!strcmp(name, "fold_variant")) { e->opt_variant = value; return SGR_OK; }
  if (!strcmp(name, "kernel")) { e->opt_kernel = value; return SGR_OK; }
  if (!strcmp(name, "incremental")) { e->opt_incremental = value; return SGR_OK; }
  if (!strcmp(name, "force_route")) { e->opt_force_route = value; return SGR_OK; }
  if (!strcmp(name, "bulk")) { e->opt_bulk = value; return SGR_OK; }
  if (!strcmp(name, "bulk_unroll")) { bulk_tuning().unroll = (int)value; return SGR_OK; }
  if (!strcmp(name, "bulk_hints")) { bulk_tuning().hints = (int)value; return SGR_OK; }
  if (!strcmp(name, "bulk_blocks_per_sm")) { bulk_tuning().blocks_per_sm = (int)value; return SGR_OK; }
  if (!strcmp(name, "push_tile")) {
    if (value != 256 && value != 512 && value != 1024) return fail(e, SGR_ERR_INVALID, "push_tile must be 256, 512 or 1024");
    push_tuning().tile = (int)value; return SGR_OK;
  }
  if (!strcmp(name, "push_fold_blocks_per_sm")) { push_tuning().fold_blocks_per_sm = (int)value; return SGR_OK; }
  if (!strcmp(name, "push_ordered")) { e->opt_push_ordered = value ? 1 : 0; return SGR_OK; }
  if (!strcmp(name, "push_staged")) { push_tuning().staged = (int)value; return SGR_OK; }
  if (!strcmp(name, "push_pull")) { push_tuning().pull = value ? 1 : 0; return SGR_OK; }
  if (!strcmp(name, "push_chunks")) {
    if (value < 1 || value > 256) return fail(e, SGR_ERR_INVALID, "push_chunks must be in [1, 256]");
    e->opt_push_chunks = value; return SGR_OK;
  }
  if (!strcmp(name, "replay_budget")) { e->opt_replay_budget = value; return SGR_OK; }
  if (!strcmp(name, "var_stage_bytes")) { e->opt_var_stage_bytes = value; return SGR_OK; }
  if (!strcmp(name, "var_stages")) { e->opt_var_stages = (value >= 1 && value <= 3) ? value : 2; return SGR_OK; }
  if (!strcmp(name, "run_variant")) {
    if (value < 0 || value >= run_variant_count()) return fail(e, SGR_ERR_INVALID, "run_variant out of range");
    e->opt_run_variant = value; return SGR_OK;
  }
  // test aid: the look-back epoch the next record-parallel fold moves on from (a value near 2^32 makes a few folds wrap it)
  if (!strcmp(name, "lookback_epoch")) { e->epoch = (uint32_t)value; return SGR_OK; }
  if (!strcmp(name, "run_chunk_bytes")) {
    if (value < 2048 || value > (1ll << 30)) return fail(e, SGR_ERR_INVALID, "run_chunk_bytes must be in [2048, 2^30]");
    e->opt_run_chunk_bytes = value; return SGR_OK;
  }
  if (!strcmp(name, "long_threshold")) { e->opt_long_threshold = value; return SGR_OK; }
  if (!strcmp(name, "max_record_bytes")) {
    if (value < 16 || value > 2048 + 16) return fail(e, SGR_ERR_INVALID, "max_record_bytes must be in [16, 2064]");
    e->opt_max_record_bytes = value; return SGR_OK;
  }
  return fail(e, SGR_ERR_INVALID, "unknown option '%s'", name);
}

int32_t sgr_stream(sgr_engine* e, void** stream) {
  if (!e || !stream) return SGR_ERR_INVALID;
  *stream = (void*)e->stream;
  return SGR_OK;
}

}  // extern "C"

int32_t sgr::fold_decoded_poll(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_live) {
  return fold_incremental_device(e, d_records, n_records, true, n_live);
}

int32_t sgr::put_decoded_poll(sgr_engine* e, const void* d_rows, const uint32_t* d_slots, const uint8_t* d_present, uint64_t n_slots, uint64_t n_live) {
  OpLock op_lock(e);
  if (!e || (n_slots && (!d_rows || !d_slots || !d_present))) return fail(e, SGR_ERR_INVALID, "null argument");
  if (!e->has_program) return fail(e, SGR_ERR_NO_PROGRAM, "register a fold program first");
  if (e->dist) return fail(e, SGR_ERR_UNSUPPORTED, "the rows of a routed engine are local slots: a state topic does not map ids to them");
  if (n_slots >= (1ull << 32)) return fail(e, SGR_ERR_UNSUPPORTED, "a poll holds fewer than 2^32 records");
  if (!e->states_valid) return fail(e, SGR_ERR_NOT_LOADED, "the device ingest grows the table before it applies a poll");
  if (!n_live) return SGR_OK;   // as a put batch of no records: nothing applied, the last fold's flags stay
  int32_t rc = use_device(e); if (rc) return rc;
  rc = finish_fold(e); if (rc) return rc;
  CUDA_TRY(e, e->pb_scratch.reserve(64));
  PutBatch p;
  p.rows = (const uint8_t*)d_rows; p.present = d_present; p.slot = const_cast<uint32_t*>(d_slots); p.n = (uint32_t)n_slots;
  p.ctl = (unsigned long long*)e->pb_scratch.p;
  rc = put_apply_begin(e, e->states_n, n_slots); if (rc) return rc;
  CUDA_TRY(e, cudaMemsetAsync(p.ctl, 0, 64, e->stream));
  const cudaError_t ce = put_batch_apply(p, (uint8_t*)e->states.p, e->dprog, (uint32_t*)e->pb_last.p, (uint32_t*)e->inc_ids.p, e->stream);
  if (ce != cudaSuccess) return fail(e, SGR_ERR_CUDA, "put_batch: %s", cudaGetErrorString(ce));
  CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  unsigned long long pb[8];
  CUDA_TRY(e, cudaMemcpyAsync(pb, p.ctl, 64, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  return put_apply_end(e, n_live, pb[kPbTouched]);
}

int32_t sgr::grow_states_for_ids(sgr_engine* e, uint64_t n_keys, uint64_t limit) {
  OpLock op_lock(e);
  if (!e) return SGR_ERR_INVALID;
  if (e->states_valid && n_keys <= e->states_n) return SGR_OK;
  // amortised doubling, like a hash table: the resize copies the table device to device
  uint64_t cap = e->states_valid ? e->states_n : 0;
  if (cap < 1024) cap = 1024;
  while (cap < n_keys) cap *= 2;
  if (cap > limit && limit >= n_keys) cap = limit;
  return sgr_grow_states(e, cap);
}

int32_t sgr::engine_program_state_bytes(sgr_engine* e, uint32_t* state_bytes, bool* routed) {
  OpLock op_lock(e);
  if (!e || !state_bytes || !routed) return SGR_ERR_INVALID;
  *state_bytes = e->has_program ? e->program.state_bytes : 0;
  *routed = e->dist != nullptr;
  return SGR_OK;
}
