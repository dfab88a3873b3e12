// fold_rows.cuh — launch interface of the record-parallel fold (K1/K3, fixed 64-byte records).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/sgr.h"
#include "sgr_device.cuh"

namespace sgr {

constexpr int kRowThreads = 256;
constexpr int kMaxSlots = 16;   // distinct record words a program may read (slot 0 = event type)
constexpr int kMaxRowWords = 14;  // widest state in transformer form: 64-byte struct
constexpr int kTabStride = 16;   // words per type in RowProgram::tab

// ---- RowProgram::tab, the only place that knows its encoding. Per type, word 0 holds the rule flags:
constexpr uint32_t kRuleValid = 1u;     // the rule does not throw (THROW rules and unknown types read as 0)
constexpr uint32_t kRuleNone = 2u;      // the result is None (TOMBSTONE)
constexpr uint32_t kRuleIfExists = 4u;  // IF_EXISTS: the ops apply only to an existing state
constexpr uint32_t kRuleNew = 8u;       // the rule builds a new state instance (Scala constructor or copy): CREATE, or any field op
// and word 1+w the spec of state word w: mode | neg << 2 | slot << 3 (mode 0 keeps the word; slot 0 reads no record word)
constexpr uint32_t kModeAdd = 1u, kModeSet = 2u;

__host__ __device__ __forceinline__ uint32_t spec_encode(uint32_t mode, uint32_t neg, uint32_t slot) { return mode | (neg << 2) | (slot << 3); }
__host__ __device__ __forceinline__ uint32_t spec_mode(uint32_t spec) { return spec & 3u; }
__host__ __device__ __forceinline__ uint32_t spec_slot(uint32_t spec) { return spec >> 3; }
// the op subtracts: the word takes -v from the record word v
__host__ __device__ __forceinline__ bool spec_neg(uint32_t spec) { return (spec & 4u) != 0u; }

// ---- transformer form shared by the fold kernels: mode word bits and the exists-op of an event
constexpr uint32_t M_ERR = 0x80000000u;   // some event in the range threw
constexpr uint32_t M_COPY = 0x40000000u;  // some applied event built a new state instance (fold_runs.cu finish_segment)
static_assert((kRuleNew << 27) == M_COPY, "rule_copy_bit moves the new-instance flag onto M_COPY");
__host__ __device__ __forceinline__ uint32_t rule_copy_bit(uint32_t flags) { return (flags & kRuleNew) << 27; }
constexpr uint32_t EX_SOME = 1u, EX_NONE = 2u;
__host__ __device__ __forceinline__ uint32_t rule_ex(uint32_t flags) { return (flags & kRuleNone) ? EX_NONE : EX_SOME; }

// Program in transformer form: per event type, how each state word is produced.
// Two closed classes of programs (build_row_program decides):
//   class 0  MATERIALISE / CREATE / TOMBSTONE / THROW rules          (Counter, IntBalance, snapshot restore)
//   class 1  IF_EXISTS / CREATE / TOMBSTONE / THROW rules            (BankAccount): an IF_EXISTS event applies iff the
//            state exists at that point, i.e. iff the input existed or a CREATE came before it — one extra
//            composition rule (a tombstoned prefix absorbs it), still associative
// A program mixing MATERIALISE and IF_EXISTS is outside both and takes the lane-sequential kernel.
struct RowProgram {
  uint32_t user_words;
  uint32_t n_slots;
  uint32_t cls;                   // 0 / 1, see above
  uint32_t f64_mask;              // bit w: state words w, w+1 form a JVM Double (numeric == for the publish rule)
  uint32_t head_only;             // every record word the program reads (slot_word) lies in words 0..7: the runs fold
                                  // may stage the head plane instead of the log
  uint32_t slot_word[kMaxSlots];  // record word index of each slot
  uint32_t tab[16 * kTabStride];  // per type: [0] kRule* flags, [1+w] spec of state word w (see above)
};

struct RowArgs {
  const uint8_t* events;        // device log; records at log_begin + 64*i
  const uint8_t* heads;         // fold_runs plane (or null): bytes 0..31 of record i at heads + 32*i (head plane), or
                                // its slot words at heads + 16*i (slot plane)
  const uint64_t* seg_offsets;  // n_seg+1 byte offsets, all == log_begin (mod 64)
  const uint32_t* seg_ids;      // optional state slot per segment
  uint64_t n_seg;
  uint64_t log_begin, log_end;  // seg_offsets[0], seg_offsets[n_seg]
  const uint8_t* states_in;     // optional prior states
  uint8_t* states_out;
  unsigned long long* counters; // [0] events applied, [1] aggregates in error, [3] segments queued for exact replay,
                                // [4] records dropped after a throw; fold_runs (16 words): [6] warps arrived,
                                // [8] ~%globaltimer at the first CTA's entry (max of the complement),
                                // [9] %globaltimer at the last warp's exit,
                                // [10] chunk ticket, [11] replay cursor
  unsigned long long* counters_next;  // fold_runs: the other counter block (16 words), zeroed for the next fold
  uint32_t* redo_ids;           // segments whose handler threw (replayed by the sequential kernel)
  uint64_t redo_cap;
  uint32_t* part_flags;         // per warp (fold_runs: per chunk): == epoch once its open transformer is published
  uint32_t* part_data;          // per warp (fold_runs: per chunk): m, v[W], ex | has_head<<2
  uint32_t epoch;
  uint64_t chunk_steps;         // fold_runs: steps per chunk of the ticketed work order (run_variant_chunk_steps)
  const uint64_t* chunk_kc;     // fold_runs from the slot plane (or null): per chunk, its first boundary (launch_build_chunk_table)
};

// false if the program is outside the transformer algebra (IF_EXISTS rules, 64-bit adds, f64 fields,
// unsupported state width): the caller then uses the lane-sequential kernel.
bool build_row_program(const DevProgram& dp, RowProgram* out);
// over the valid types: which of state words 0, 1 some type ADDs to (bit w of add) or SETs (set), and whether one makes None
struct WordModes {
  uint32_t add, set;
  bool none;
};
WordModes word_modes(const RowProgram& prog);

// The publish rule for an integer row of W state words, then the row itself (W + 2 words, 16-byte aligned): the words
// (zeroed when the result is None), exn | CHANGED, a zero err word. CHANGED when existence flips, or when the state
// exists before and after and a word differs. old/ex0: the prior state (words zero when it was None); nw/exn the new one.
template <int W>
__device__ __forceinline__ void finish_row(uint8_t* row, const uint32_t (&old)[W], uint32_t ex0, const uint32_t (&nw)[W], uint32_t exn) {
  uint32_t outw[W + 2], changed = exn != ex0;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    outw[w] = exn ? nw[w] : 0u;
    if (exn && ex0) changed |= (outw[w] != old[w]);
  }
  outw[W] = exn | (changed ? SGR_ST_CHANGED : 0u);
  outw[W + 1] = 0u;
  uint4* dp = reinterpret_cast<uint4*>(row);
#pragma unroll
  for (int q = 0; q < (W + 2) / 4; ++q) dp[q] = make_uint4(outw[4 * q], outw[4 * q + 1], outw[4 * q + 2], outw[4 * q + 3]);
}
// the same for a 16-byte row, against the row as it was read (old.x, old.y are compared only when ex0 is set)
__device__ __forceinline__ void finish_row16(uint4* row, const uint4& old, uint32_t ex0, uint32_t n0, uint32_t n1, uint32_t exn) {
  if (!exn) { n0 = 0; n1 = 0; }
  uint32_t changed = exn != ex0;
  if (exn && ex0) changed |= (n0 != old.x) | (n1 != old.y);
  *row = make_uint4(n0, n1, exn | (changed ? SGR_ST_CHANGED : 0u), 0u);
}
// one pass over the CSR offsets at load time: are all segments 64-byte aligned relative to the first, and
// where does the log begin/end (device offsets are opaque to the host otherwise)
cudaError_t inspect_offsets(const uint64_t* d_off, uint64_t n_seg, unsigned long long* d_scratch, cudaStream_t st,
                            bool* aligned64, uint64_t* log_begin, uint64_t* log_end, uint64_t* max_seg_bytes);
int row_kernel_max_grid(int num_sms, const RowProgram& prog);  // largest co-resident grid (look-back needs forward progress)
cudaError_t launch_fold_rows(const RowArgs& args, const RowProgram& prog, int grid, cudaStream_t stream);


// ---- fold_vruns.cu: variable records with a record directory
struct VarArgs {
  const uint8_t* events;
  const uint64_t* rec_offsets;   // n_rec+1 byte offsets, log order
  uint64_t n_rec;
  const uint64_t* seg_offsets;   // CSR, the source of truth (cross-checked at every segment head)
  uint64_t n_seg;
  uint8_t* states_out;           // zeroed before the launch (full rebuild: empty aggregates stay None)
  unsigned long long* counters;  // [0] records seen, [3] replay list length, [4] records of replayed segments, [7] CSR mismatches
  uint32_t* redo_ids; uint64_t redo_cap;
  uint32_t* part_flags; uint32_t* part_data; uint32_t epoch;   // part_data: 8 words per warp
  uint32_t stage_bytes;
  uint32_t max_record_bytes;      // a longer record (header included, before padding) is malformed: its segment is replayed
};
int vruns_config(int num_sms, uint32_t max_record_bytes, uint32_t stage_hint, int nstage, int* threads, size_t* smem, uint32_t* stage_bytes);  // returns max grid, 0 if impossible
cudaError_t launch_fold_vruns(const VarArgs& args, const RowProgram& prog, int nstage, int grid, int threads, size_t smem, cudaStream_t stream);

// ---- fold_runs.cu: lane-run variant (primary). Same RowArgs / RowProgram.
int run_variant_count();
const char* run_variant_name(int v);
int head_variant_count();
int proj_variant_count();
// the program may fold from the slot plane: head-only, 16-byte state, class 0, at most 4 slots
bool slot_plane_fits(const RowProgram& prog);
// plane 0: the kernel stages the log (run variant `variant`); plane 32: the head plane RowArgs::heads (head variant
// `variant`); plane 16: the slot plane RowArgs::heads (projected variant `variant`)
int run_kernel_max_grid(int num_sms, int variant, int plane, const RowProgram& prog);
int run_variant_step_bytes(int variant, int plane, const RowProgram& prog);  // log bytes per step
int run_warps_per_cta();
// steps per chunk of a log of `steps` steps folded by up to n_warps warps: at most chunk_bytes, small enough that every warp
// gets a chunk, and at least the steps the variant stages ahead
uint64_t run_variant_chunk_steps(int variant, int plane, const RowProgram& prog, uint64_t chunk_bytes, uint64_t steps, uint64_t n_warps);
// one launch, replay included; overlap: it may start while the runs fold before it on the stream drains (programmatic
// dependent launch), for a fold of the same log right behind another
cudaError_t launch_fold_runs(const RowArgs& args, const RowProgram& prog, int variant, int plane, int grid, bool overlap, cudaStream_t stream);
// the chunk table of a runs fold: table[c] = the first k in [0, n_seg] with off[k] >= log_begin + c * chunk_steps * step_bytes,
// for c in [0, n_chunks)
cudaError_t launch_build_chunk_table(const uint64_t* off, uint64_t n_seg, uint64_t log_begin, uint64_t step_bytes, uint64_t chunk_steps,
                                     uint64_t n_chunks, uint64_t* table, cudaStream_t stream);
// copy bytes 0..31 of records [rec0, rec1) of `log` (64-byte records from its first byte) to heads + 32*i
cudaError_t launch_build_heads(const uint8_t* log, uint8_t* heads, uint64_t rec0, uint64_t rec1, int num_sms, cudaStream_t stream);
// write the slot words of records [rec0, rec1) of `log` to slots + 16*i, slot s at word s, zero-padded (slot_plane_fits)
cudaError_t launch_build_slots(const uint8_t* log, uint8_t* slots, uint64_t rec0, uint64_t rec1, const RowProgram& prog, int num_sms,
                               cudaStream_t stream);

}  // namespace sgr
