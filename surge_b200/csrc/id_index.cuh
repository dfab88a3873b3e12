// id_index.cuh — the engine's device-resident aggregate-id index behind sgr_get_batch (launch interface of id_index.cu).
//
// It mirrors the engine's key table (sgr_load_keys, or the ids appended by an ingest) in the dictionary layout of id_dict.cuh,
// with the dense index of an id = its position in the key table. Id bytes and their (offset, length) refs stay on the device, so
// appended ids cost an upload and an insert of the new ones only, and a rehash works from what is resident.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "devbuf.h"
#include "id_dict.cuh"

namespace sgr {

struct IdIndex {
  DevBuf tags, slot_idx, key_ref, arena;
  uint64_t slots = 0;        // power of two, at least twice the ids indexed
  uint64_t n = 0;            // ids [0, n) of the key table are indexed
  uint64_t arena_used = 0;   // bytes (8-byte aligned entries)
  uint64_t epoch = 0;        // which key table the ids come from (sgr_engine::keys_epoch)
  uint64_t builds = 0;       // counts the times the index started again from id 0 (the id order, id_order.cuh, follows it)
  bool valid = false;        // false: rebuild from id 0 before the next read

  DgDict dict(unsigned long long* ctl) const {
    DgDict d{};
    d.tags = (unsigned long long*)tags.p; d.slot_idx = (uint32_t*)slot_idx.p; d.key_ref = (uint2*)key_ref.p; d.arena = (uint8_t*)arena.p;
    d.ctl = ctl; d.slots_mask = slots ? slots - 1 : 0; d.max_keys = n; d.arena_cap = arena.cap;
    return d;
  }
};

// Host bytes ids [from, to) of a key table take in the staging buffer of id_index_append (their refs and 8-byte aligned bytes).
// Sets *monotone = false (and returns 0) when the offsets decrease somewhere in that range.
uint64_t id_index_stage_bytes(const uint32_t* offs, uint64_t from, uint64_t to, bool* monotone);

// Enqueue on `st`: index ids [x.n, to) of the key table (bytes, offs), growing the resident id storage as needed, and rehash the
// whole index on the device when the load factor would pass 1/2. `stage`: page-locked memory of id_index_stage_bytes(...) bytes,
// untouched until the stream reaches this point. d_ctl: 2 device u64, zeroed; [0] counts duplicate ids, [1] full tables.
cudaError_t id_index_append(IdIndex& x, const uint8_t* bytes, const uint32_t* offs, uint64_t to, void* stage, unsigned long long* d_ctl,
                            cudaStream_t st);

// Grow the resident id storage to hold `ids` refs and `arena_bytes` id bytes, keeping what the index holds (ids [0, x.n) and
// x.arena_used bytes). Synchronises `st` when it moves them.
cudaError_t id_index_reserve(IdIndex& x, uint64_t ids, uint64_t arena_bytes, cudaStream_t st);

// Enqueue on `st`: insert ids [x.n, to), whose refs and bytes are already resident, and set x.n = to; rehashes every id from
// id 0 when the load factor would pass 1/2. d_ctl as for id_index_append.
cudaError_t id_index_insert(IdIndex& x, uint64_t to, unsigned long long* d_ctl, cudaStream_t st);

// One thread per query id: its dense index, or -1. q_offs[n + 1] index the query bytes q.
cudaError_t id_index_probe(const IdIndex& x, const uint8_t* q, const uint32_t* q_offs, uint64_t n, long long* idx, cudaStream_t st);

// Rows of the found ids: program bytes (state_bytes - 8 per row, zero for a None state or an unknown id) and SGR_ST_* flags (0 for
// an unknown id). An index at or past n_states is left out and reported as the largest such index + 1 in *bad.
cudaError_t id_index_gather(const uint8_t* states, uint32_t state_bytes, uint64_t n_states, const long long* idx, uint64_t n,
                            uint8_t* rows, uint32_t* flags, unsigned long long* bad, cudaStream_t st);

}  // namespace sgr
