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

}  // namespace sgr
