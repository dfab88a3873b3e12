// put_batch.cuh — keyed state writes on the device (sgr_put_batch): launch interface of put_batch.cu.
//
// A batch is n records in arrival order, record i = (id i, row i | tombstone). Phase 1 (put_batch_resolve) gives every record
// the dense index of its id: the engine's id index answers for known ids, a batch-local table deduplicates the unknown ones
// and new ids are numbered n_keys, n_keys + 1, ... in order of first appearance, their refs and bytes written behind the
// resident ones. Phase 2 (put_batch_apply) keeps the last record per index and writes it into the live table.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "id_index.cuh"
#include "sgr_device.cuh"

namespace sgr {

// ctl words of one batch (PutBatch::ctl, 8 x u64, zeroed by put_batch_resolve)
constexpr int kPbNewBytes = 0;   // id bytes of the new ids (unaligned: what the host key table grows by)
constexpr int kPbFull = 1;       // unknown ids that found no slot in the batch table (sized so that this does not happen)
constexpr int kPbTouched = 2;    // rows written by put_batch_apply
constexpr int kPbNewIds = 3;     // new ids, and [4] their arena bytes (8-byte aligned entries); copied from the scans' ends

// One batch on the device: the staged inputs and the scratch carved from one buffer of put_batch_scratch_bytes(n) bytes.
struct PutBatch {
  const uint8_t* ids = nullptr;       // id bytes, id i = ids[offs[i] .. offs[i + 1])
  const uint32_t* offs = nullptr;     // [n + 1]
  const uint8_t* rows = nullptr;      // [n][state_bytes - 8]
  const uint8_t* present = nullptr;   // [n]; 0 = tombstone
  uint32_t n = 0;
  uint64_t n_keys = 0;                // ids of the key table before the batch (= the index's x.n)

  unsigned long long* ctl = nullptr;  // kPb*
  long long* probe = nullptr;         // [n] dense index of a known id, else -(batch table slot + 1)
  uint32_t* first = nullptr;          // [n + 1] 1 at the first appearance of a new id
  uint32_t* rank = nullptr;           // [n + 1] exclusive scan of first: rank[n] = new ids
  unsigned long long* alen = nullptr; // [n + 1] its 8-byte aligned length at a first appearance
  unsigned long long* aoff = nullptr; // [n + 1] exclusive scan of alen: its arena offset behind the resident ids
  uint32_t* slot = nullptr;           // [n] the record's dense index after the batch (~0u: a hole, skipped by put_batch_apply)
  uint32_t* new_pos = nullptr;        // [n] batch position of new id k (k < rank[n]): index order
  unsigned long long* bt_tags = nullptr;   // batch table: hash tag (0 empty)
  uint32_t* bt_owner = nullptr;            // the first claimant's position + 1 (0: still publishing)
  uint32_t* bt_min = nullptr;              // smallest batch position of the id
  uint64_t bt_mask = 0;
  void* cub_tmp = nullptr;
  size_t cub_bytes = 0;
};

// Scratch bytes of a batch of n records (see PutBatch), and the carving of `base` into it.
size_t put_batch_scratch_bytes(uint64_t n);
void put_batch_carve(PutBatch& p, void* base, uint64_t n);

// Phase 1, enqueued on `st`: probe, dedupe and number the new ids; write their refs at key_ref[n_keys + k] and their bytes at
// arena + arena_used + aoff (both grown beforehand for every id of the batch being new), and every record's dense index. The
// index `x` (ids [0, x.n), x.n == p.n_keys) is only read: the caller inserts the new ids once it knows they fit.
cudaError_t put_batch_resolve(const IdIndex& x, uint64_t arena_used, PutBatch& p, cudaStream_t st);

// Phase 2, enqueued on `st`: the last record of each touched index writes its row (program bytes and flags: EXISTS for a row,
// None for a tombstone, CHANGED against the prior state, err_idx 0) and appends the index to `touched` (count in
// ctl[kPbTouched]). last: u32 per table row, zero before and after.
cudaError_t put_batch_apply(const PutBatch& p, uint8_t* states, const DevProgram& prog, uint32_t* last, uint32_t* touched,
                            cudaStream_t st);

}  // namespace sgr
