// group_kernels.cuh — K5: stable group-by of arrival-ordered records into CSR form.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "devbuf.h"

namespace sgr {

struct GroupScratch {
  DevBuf keys_a, keys_b, idx_a, idx_b;  // radix-sort double buffers (u32 each)
  DevBuf cub_tmp;                       // CUB temp storage of the sort and of the compact mode's scan
  DevBuf flags;                         // segment-head flags / positions (compact mode)
  DevBuf batch_records;                 // grouped records of an incremental batch
};

// out[i] = in[0] + ... + in[i - 1] for i < n, by cub::DeviceScan::ExclusiveSum; out == in scans in place.
// tmp is CUB's temp storage, grown to the size CUB asks for.
cudaError_t exclusive_sum_u32(const uint32_t* in, uint32_t* out, uint32_t n, DevBuf& tmp, cudaStream_t stream);

// Stable group-by of n fixed 64-byte records by their aggregate index (u64 at +8, < n_agg).
// Replaces what the Kafka broker + KTable do in the reference: per-key log order is kept
// (modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:57-76).
//   full mode    (d_touched_ids == nullptr): d_out_offsets gets n_agg+1 byte offsets;
//   compact mode (d_touched_ids != nullptr): d_out_offsets gets n_touched+1 byte offsets over the
//                 aggregates that own at least one record, whose indices go to d_touched_ids
//                 (ascending); *n_touched is returned to the host.
// d_counters: >= 8 u64 of scratch. *bad_out = number of records with agg >= n_agg (nothing else is valid then).
// holes_out == nullptr: every record must carry agg < n_agg. holes_out != nullptr (the device ingest's decoded polls only):
//   records with agg == ~0 are holes. They sort behind every live record, fall outside every CSR segment, are not
//   gathered into d_out_records (which then holds n - *holes_out records) and are counted in *holes_out, not in *bad_out.
//   n_agg must be below 2^32 (n_agg itself is the holes' key).
cudaError_t group_by_agg_stable(GroupScratch& sc, const uint8_t* d_records, uint64_t n, uint64_t n_agg,
                                uint8_t* d_out_records, uint64_t* d_out_offsets, uint32_t* d_touched_ids,
                                uint64_t* n_touched, unsigned long long* d_counters, cudaStream_t stream,
                                unsigned long long* bad_out, unsigned long long* holes_out = nullptr);

// Clear the per-batch flags (CHANGED, ERROR, err_idx) of the listed state slots (ids == nullptr: all n slots).
void clear_batch_flags(uint8_t* d_states, uint32_t state_bytes, const uint32_t* d_ids, uint64_t n, cudaStream_t stream);

}  // namespace sgr
