// state_values.cuh — rows -> JSON state values on the device, behind sgr_get_batch_values, sgr_export_changes_values and
// sgr_scan_values (launch interface of state_values.cu; the value format is state_writer.h's).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "state_writer.h"

namespace sgr {

// A registered writer table (sgr_set_state_writer): members in value order, their literals (`{"name":` / `,"name":`) in lits.
struct SwWriter {
  sw::Member m[sw::kMaxMembers];
  const uint8_t* lits;   // device
  uint32_t n;            // 0: no writer
};

// What state_values_measure leaves in its control words (u64 each): the rows of the longest prefix whose values fit in `cap`,
// their value bytes, the lowest row that cannot be written (~0: none), and for that row, when it lies inside the prefix, its
// status (member << 8 | sw::Reason) and its dense index.
enum { kSvRows = 0, kSvBytes = 1, kSvRefused = 2, kSvStatus = 3, kSvIndex = 4, kSvCtlWords = 8 };

// The rows of a batch or page, as the gather left them: program bytes (user per row), SGR_ST_* flags, dense indices (negative
// for an unknown id) and ids ids[id_offs[i] .. id_offs[i + 1]). A row has an id when 0 <= idx[i] < n_keys. A row without
// SGR_ST_EXISTS has an empty value.
struct SvRows {
  const uint8_t* rows; uint32_t user;
  const uint32_t* flags; const long long* idx;
  const uint8_t* ids; const uint32_t* id_offs;
  uint64_t n_keys, n;
};

// Device scratch of a measure over n rows.
size_t state_values_scratch_bytes(uint64_t n);

// Enqueue the length pass, the exclusive scan of the lengths into offs[0 .. n] (u64, inside the scratch) and the fit step
// against cap. wrap: each value is the protobuf State around the JSON value (SGR_VALUE_PROTOBUF_JSON; a refusal of the row's id
// reports member sw::kWrapMember). *offs (out): where the offsets live; *ctl (out): the control words, kSvCtlWords u64.
cudaError_t state_values_measure(const SwWriter& w, bool wrap, const SvRows& r, uint64_t cap, void* scratch, unsigned long long** offs,
                                 unsigned long long** ctl, cudaStream_t st);

// Enqueue the write of rows [0, n_rows) at values + offs[i] (offs from state_values_measure over the same rows and wrap).
cudaError_t state_values_write(const SwWriter& w, bool wrap, const SvRows& r, uint64_t n_rows, const unsigned long long* offs, uint8_t* values,
                               cudaStream_t st);

}  // namespace sgr
