// changes.cu — paged compaction of selected rows: the changed-state export (sgr_export_changes) and the ordered scan
// (sgr_scan) share these count, cut, compaction and id-copy kernels.
//
// Rows are visited by position p in [next, end): the row at p is p itself (the export: positions are dense indices) or map[p]
// (the scan: map is the id order of id_order.cuh). A row is selected when its flags word meets `select`.
//   count    one CTA per tile of kChangesTile positions from next's tile, a thread per position: the row's 8-byte flags | err_idx
//            word; the tile's selected rows and their id bytes (key_ref[row].y) as one packed u64
//   cut      one CTA: an exclusive scan of the tile totals, kChangesTile tiles per step, writes each tile's base and stops at the
//            first tile that does not fit whole (rows or id bytes); that tile's rows are scanned again and the cut falls on its
//            first selected row that does not fit. ctl: rows and id bytes of the page, the position after it, the tiles it spans
//   compact  one CTA per tile of the page: a block scan puts each selected row at base + rank, with err_idx and its id offset
//   ids      16 adjacent threads per row copy its id bytes from the index arena (8-byte aligned) to their offset in the page
// count and cut can take [next, end) from device memory (`range`, written by an earlier launch): the grid then covers the
// widest range and the tiles outside the one read are empty.
// The program bytes and flags of the page's rows are gathered by id_index_gather (id_index.cu) over the compacted indices.
#include "../../include/sgr.h"
#include "changes.cuh"

namespace sgr {
namespace {

constexpr unsigned long long kLow32 = 0xffffffffull;
constexpr int kIdLanes = 16;
constexpr int kIdThreads = 256;

// Position p as packed (selected << 32 | id length), its row and the row's flags | err_idx word. Positions [next, end) are in
// range; the row at position p is map[p], or p itself without a map.
__device__ __forceinline__ unsigned long long row_word(const uint8_t* __restrict__ states, uint32_t state_bytes, uint64_t n_agg,
                                                       const uint32_t* __restrict__ map, const uint2* __restrict__ key_ref, uint64_t n_keys,
                                                       uint32_t select, uint64_t next, uint64_t end, uint64_t p, uint64_t* row, uint2* word) {
  *word = make_uint2(0, 0);
  *row = p;
  if (p < next || p >= end) return 0;
  const uint64_t r = map ? __ldg(map + p) : p;
  *row = r;
  if (r >= n_agg) return 0;
  *word = __ldg(reinterpret_cast<const uint2*>(states + r * state_bytes + state_bytes - 8));
  if (!(word->x & select)) return 0;
  return (1ull << 32) | (r < n_keys ? __ldg(key_ref + r).y : 0u);
}

// Exclusive scan of v over the CTA (kChangesTile threads = 32 warps); *total = the sum. sm: 32 u64 of shared memory.
__device__ __forceinline__ unsigned long long block_excl_scan(unsigned long long v, unsigned long long* sm, unsigned long long* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sm[w] = x;
  __syncthreads();
  if (w == 0) {
    unsigned long long s = sm[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    sm[lane] = s;
  }
  __syncthreads();
  const unsigned long long ex = x - v + (w ? sm[w - 1] : 0ull);
  *total = sm[31];
  __syncthreads();   // sm is free again for the next scan
  return ex;
}

__global__ void __launch_bounds__(kChangesTile) ch_count_kernel(const uint8_t* __restrict__ states, uint32_t state_bytes, uint64_t n_agg,
                                                                const uint32_t* __restrict__ map, const uint2* __restrict__ key_ref, uint64_t n_keys,
                                                                uint32_t select, uint64_t next, uint64_t end, const unsigned long long* __restrict__ range,
                                                                unsigned long long* __restrict__ tot) {
  __shared__ unsigned long long sm[32];
  if (range) { next = range[0]; end = range[1]; }
  const uint64_t t0 = next / kChangesTile;
  if ((t0 + blockIdx.x) * kChangesTile >= end) {   // a tile past a range read from the device
    if (threadIdx.x == 0) tot[blockIdx.x] = 0;
    return;
  }
  uint64_t r;
  uint2 w;
  const unsigned long long v = row_word(states, state_bytes, n_agg, map, key_ref, n_keys, select, next, end,
                                        (t0 + blockIdx.x) * kChangesTile + threadIdx.x, &r, &w);
  unsigned long long sum;
  block_excl_scan(v, sm, &sum);
  if (threadIdx.x == 0) tot[blockIdx.x] = sum;
}

__global__ void __launch_bounds__(kChangesTile) ch_cut_kernel(const uint8_t* __restrict__ states, uint32_t state_bytes, uint64_t n_agg,
                                                              const uint32_t* __restrict__ map, const uint2* __restrict__ key_ref, uint64_t n_keys,
                                                              uint32_t select, uint64_t next, uint64_t end, const unsigned long long* __restrict__ range,
                                                              uint64_t max_rows, uint64_t ids_cap, uint64_t nt, unsigned long long* tiles,
                                                              unsigned long long* __restrict__ ctl) {
  __shared__ unsigned long long sm[32];
  __shared__ unsigned long long s_cut, s_end, s_next;
  const unsigned long long* tot = tiles;
  unsigned long long* base = tiles + nt;
  if (range) { next = range[0]; end = range[1]; }
  const uint64_t span = (end + kChangesTile - 1) / kChangesTile - next / kChangesTile;   // the tiles [next, end) touches
  const uint64_t nr = span < nt ? span : nt;
  if (threadIdx.x == 0) s_cut = nr;
  __syncthreads();
  unsigned long long carry = 0;
  for (uint64_t c0 = 0; c0 < nr; c0 += kChangesTile) {
    const uint64_t t = c0 + threadIdx.x;
    const unsigned long long v = t < nr ? tot[t] : 0ull;
    unsigned long long step;
    const unsigned long long ex = carry + block_excl_scan(v, sm, &step);
    const unsigned long long in = ex + v;
    if (t < nr) {
      base[t] = ex;
      if ((in >> 32) > max_rows || (in & kLow32) > ids_cap) atomicMin(&s_cut, (unsigned long long)t);
    }
    __syncthreads();
    if (s_cut < nr) break;   // the same value in every thread
    carry += step;
  }
  const uint64_t cut = s_cut;
  if (cut == nr) {           // everything selected from the cursor on fits
    if (threadIdx.x == 0) { ctl[kChCtlRows] = carry >> 32; ctl[kChCtlBytes] = carry & kLow32; ctl[kChCtlNext] = end; ctl[kChCtlTiles] = nr; }
    return;
  }
  // the cut falls inside tile `cut`: its selected rows fit up to the first one past either budget
  const unsigned long long b = base[cut];   // (written above by another thread of this CTA; visible after the barrier)
  if (threadIdx.x == 0) { s_end = b; s_next = end; }
  __syncthreads();
  const uint64_t p = (next / kChangesTile + cut) * kChangesTile + threadIdx.x;
  uint64_t r;
  uint2 w;
  const unsigned long long v = row_word(states, state_bytes, n_agg, map, key_ref, n_keys, select, next, end, p, &r, &w);
  unsigned long long sum;
  const unsigned long long in = b + block_excl_scan(v, sm, &sum) + v;
  if (v >> 32) {
    if ((in >> 32) <= max_rows && (in & kLow32) <= ids_cap) atomicMax(&s_end, in);
    else atomicMin(&s_next, (unsigned long long)p);
  }
  __syncthreads();
  if (threadIdx.x == 0) { ctl[kChCtlRows] = s_end >> 32; ctl[kChCtlBytes] = s_end & kLow32; ctl[kChCtlNext] = s_next; ctl[kChCtlTiles] = cut + 1; }
}

__global__ void __launch_bounds__(kChangesTile) ch_compact_kernel(const uint8_t* __restrict__ states, uint32_t state_bytes, uint64_t n_agg,
                                                                  const uint32_t* __restrict__ map, const uint2* __restrict__ key_ref, uint64_t n_keys,
                                                                  uint32_t select, uint64_t next, uint64_t end,
                                                                  const unsigned long long* __restrict__ base, uint64_t n_rows,
                                                                  long long* __restrict__ idx, uint32_t* __restrict__ err_idx,
                                                                  uint32_t* __restrict__ id_offs) {
  __shared__ unsigned long long sm[32];
  const uint64_t p = (next / kChangesTile + blockIdx.x) * kChangesTile + threadIdx.x;
  uint64_t r;
  uint2 w;
  const unsigned long long v = row_word(states, state_bytes, n_agg, map, key_ref, n_keys, select, next, end, p, &r, &w);
  unsigned long long sum;
  const unsigned long long ex = __ldg(base + blockIdx.x) + block_excl_scan(v, sm, &sum);
  const uint64_t pos = ex >> 32;
  if ((v >> 32) && pos < n_rows) {   // the page's rows are the first n_rows selected ones
    idx[pos] = (long long)r;
    err_idx[pos] = w.y;
    id_offs[pos] = (uint32_t)(ex & kLow32);
    if (pos + 1 == n_rows) id_offs[n_rows] = (uint32_t)((ex + v) & kLow32);
  }
}

__global__ void __launch_bounds__(kIdThreads) ch_copy_ids_kernel(const long long* __restrict__ idx, const uint32_t* __restrict__ id_offs,
                                                                 uint64_t n_rows, const uint2* __restrict__ key_ref,
                                                                 const uint8_t* __restrict__ arena, uint64_t n_keys, uint8_t* __restrict__ ids) {
  const uint64_t t = (uint64_t)blockIdx.x * kIdThreads + threadIdx.x;
  const uint64_t i = t / kIdLanes;
  const uint32_t lane = (uint32_t)(t % kIdLanes);
  if (i >= n_rows) return;
  const long long a = idx[i];
  if ((uint64_t)a >= n_keys) return;
  const uint2 ref = __ldg(key_ref + a);
  const uint8_t* src = arena + ((unsigned long long)ref.x << 3);
  uint8_t* dst = ids + id_offs[i];
  for (uint32_t k = lane; k < ref.y; k += kIdLanes) dst[k] = __ldg(src + k);
}

}  // namespace

cudaError_t changes_count_cut(const uint8_t* states, uint32_t state_bytes, uint64_t n_agg, const uint32_t* map, const uint2* key_ref,
                              uint64_t n_keys, uint32_t select, uint64_t next, uint64_t end, const unsigned long long* range, uint64_t max_rows,
                              uint64_t ids_cap, unsigned long long* tiles, unsigned long long* ctl, cudaStream_t st) {
  const uint64_t nt = (end + kChangesTile - 1) / kChangesTile - next / kChangesTile;
  if (!nt) return cudaSuccess;
  ch_count_kernel<<<(unsigned)nt, kChangesTile, 0, st>>>(states, state_bytes, n_agg, map, key_ref, n_keys, select, next, end, range, tiles);
  ch_cut_kernel<<<1, kChangesTile, 0, st>>>(states, state_bytes, n_agg, map, key_ref, n_keys, select, next, end, range, max_rows, ids_cap, nt,
                                            tiles, ctl);
  return cudaGetLastError();
}

cudaError_t changes_compact(const uint8_t* states, uint32_t state_bytes, uint64_t n_agg, const uint32_t* map, const uint2* key_ref,
                            uint64_t n_keys, uint32_t select, uint64_t next, uint64_t end, const unsigned long long* tiles, uint64_t n_tiles_total,
                            uint64_t n_tiles, uint64_t n_rows, long long* idx, uint32_t* err_idx, uint32_t* id_offs, cudaStream_t st) {
  if (!n_rows || !n_tiles) return cudaSuccess;
  ch_compact_kernel<<<(unsigned)n_tiles, kChangesTile, 0, st>>>(states, state_bytes, n_agg, map, key_ref, n_keys, select, next, end,
                                                                 tiles + n_tiles_total, n_rows, idx, err_idx, id_offs);
  return cudaGetLastError();
}

cudaError_t changes_copy_ids(const long long* idx, const uint32_t* id_offs, uint64_t n_rows, const uint2* key_ref, const uint8_t* arena,
                             uint64_t n_keys, uint8_t* ids, cudaStream_t st) {
  if (!n_rows || !n_keys) return cudaSuccess;
  const uint64_t threads = n_rows * kIdLanes;
  ch_copy_ids_kernel<<<(unsigned)((threads + kIdThreads - 1) / kIdThreads), kIdThreads, 0, st>>>(idx, id_offs, n_rows, key_ref, arena, n_keys, ids);
  return cudaGetLastError();
}

}  // namespace sgr
