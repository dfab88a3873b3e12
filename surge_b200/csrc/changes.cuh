// changes.cuh — paged compaction of selected rows behind sgr_export_changes and sgr_scan (launch interface of changes.cu).
//
// A page is the rows of the live table whose flags word meets `select`, visited by position from `next` up to `end` (the row
// at position p is map[p], or p without a map), cut at a row count and at a byte budget for their ids (taken from the engine's
// id index, id_index.cuh). The export visits dense indices from its cursor to n_agg; the scan visits the id order. Rows are counted in tiles of
// kChangesTile; a tile's count and id bytes travel packed in one u64: selected rows << 32 | id bytes (a key table holds fewer
// than 2^32 id bytes, and the table fewer than 2^32 rows, so neither half carries into the other).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgr {

constexpr uint32_t kChangesTile = 1024;   // rows per tile: one CTA of the count, cut and compaction kernels

// What changes_count_cut leaves in ctl[0..4): rows in the page, id bytes in the page, the position of the first selected row that
// did not fit (end when everything fit), and the number of tiles from next's tile that hold rows of the page.
enum { kChCtlRows = 0, kChCtlBytes = 1, kChCtlNext = 2, kChCtlTiles = 3 };

// Enqueue the count pass over tiles [next / kChangesTile, ceil(end / kChangesTile)) and the page cut. `tiles`: 2 u64 per tile
// from next's tile (totals, then exclusive bases). Positions outside [next, end), and rows at or past n_agg, are not selected.
// map: null, or u32[end] rows by position. range: null, or 2 device u64 read in place of next and end by the kernels, which must
// lie inside the host's [next, end). key_ref[i].y is id i's length for i < n_keys; rows at or past n_keys have a zero-length id.
cudaError_t changes_count_cut(const uint8_t* states, uint32_t state_bytes, uint64_t n_agg, const uint32_t* map, const uint2* key_ref,
                              uint64_t n_keys, uint32_t select, uint64_t next, uint64_t end, const unsigned long long* range, uint64_t max_rows,
                              uint64_t ids_cap, unsigned long long* tiles, unsigned long long* ctl, cudaStream_t st);

// Enqueue the compaction of the page that changes_count_cut cut (its ctl, read back by the host: n_rows, n_tiles), with the
// next and end the kernels read: the dense index, err_idx and id offset of every row of the page, in position order, and
// id_offs[n_rows] = the page's id bytes. n_tiles_total: the tiles changes_count_cut was launched over.
cudaError_t changes_compact(const uint8_t* states, uint32_t state_bytes, uint64_t n_agg, const uint32_t* map, const uint2* key_ref,
                            uint64_t n_keys, uint32_t select, uint64_t next, uint64_t end, const unsigned long long* tiles, uint64_t n_tiles_total,
                            uint64_t n_tiles, uint64_t n_rows, long long* idx, uint32_t* err_idx, uint32_t* id_offs, cudaStream_t st);

// Enqueue the copy of the page's ids from the index arena to ids + id_offs[i] (nothing for rows at or past n_keys).
cudaError_t changes_copy_ids(const long long* idx, const uint32_t* id_offs, uint64_t n_rows, const uint2* key_ref, const uint8_t* arena,
                             uint64_t n_keys, uint8_t* ids, cudaStream_t st);

}  // namespace sgr
