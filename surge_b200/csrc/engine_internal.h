// engine_internal.h — engine entry points for other parts of libsgr; not part of the C ABI (include/sgr.h).
#pragma once
#include <stdint.h>

#include "../../include/sgr.h"

namespace sgr {

// sgr_fold_incremental_device for a poll of the device ingest (dingest.cu), whose dropped records stay in place as holes
// (agg == ~0). Sort-free programs take the same atomic fold as sgr_fold_incremental_device, which skips holes; every other
// program groups the live records on the device (K5 in hole mode) and folds them with prior states. Holes are not events:
// they are not counted in the statistics and not in err_idx. n_live: the records that are not holes; when it is 0, a grouped
// program folds nothing (as the host decoder, which never sees dropped records) after the same checks as any other poll.
int32_t fold_decoded_poll(sgr_engine* e, const void* d_records, uint64_t n_records, uint64_t n_live);

// sgr_put_batch's apply for a poll of the device ingest in state-topic mode: slot i of the poll holds the program bytes of a row
// at d_rows + i * (state_bytes - 8), its dense index in d_slots[i] (~0u: a hole, skipped) and 0 (tombstone) / 1 in d_present[i].
// The last live slot per index decides its row; flags, the touched list, statistics and the generation follow as for a put
// batch. The table already holds every index (the ingest grew it). n_live == 0: nothing is applied, the last fold's flags stay.
int32_t put_decoded_poll(sgr_engine* e, const void* d_rows, const uint32_t* d_slots, const uint8_t* d_present, uint64_t n_slots, uint64_t n_live);

// sgr_grow_states for the n_keys ids an ingest has numbered, unless the table holds them already: the rows double from 1024
// until they do (a restore of many polls copies the table only a few times), but stop at `limit` when limit >= n_keys.
int32_t grow_states_for_ids(sgr_engine* e, uint64_t n_keys, uint64_t limit);

// The registered program's state bytes (0 without a program) and whether the engine is routed (sgr_dist_init).
int32_t engine_program_state_bytes(sgr_engine* e, uint32_t* state_bytes, bool* routed);

}  // namespace sgr
