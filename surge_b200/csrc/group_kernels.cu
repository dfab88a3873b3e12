// group_kernels.cu — K5: stable group-by of arrival-ordered 64-byte records into CSR form (sm_90a).
//
// A Kafka partition log interleaves aggregates; the fold wants each aggregate's events
// contiguous and in log order. The reference gets that from the broker + KTable keyed store
// (modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:57-76);
// here it is a stable radix sort of (aggregate index, arrival index) pairs — 8 bytes per
// record instead of 64 — followed by ONE gather of the 64-byte records into CSR order:
//   extract keys -> cub::DeviceRadixSort::SortPairs over bits [0, bits) -> offsets -> gather
// The sort's stability keeps per-aggregate arrival order, which is the only order the
// fold depends on. All kernels are plain HBM-bound integer kernels (no tensor cores).
#include "group_kernels.cuh"

#include <stdio.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/sgr.h"

namespace sgr {
namespace {

// ---------------------------------------------------------------- keys
// kHoles: a hole (agg == ~0, a record the device decode dropped) gets the key n_agg, one past the table, so that every hole
// sorts behind every live record; holes are counted in bad[2] (one atomic per warp), apart from the bad records in bad[0].
// idx[i] = i: the sort's values are the arrival indices.
template <bool kHoles>
__global__ void extract_keys_kernel(const uint8_t* __restrict__ rec, uint32_t n, uint64_t n_agg,
                                    uint32_t* __restrict__ keys, uint32_t* __restrict__ idx, unsigned long long* __restrict__ bad) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long agg = *reinterpret_cast<const unsigned long long*>(rec + (size_t)i * 64 + 8);
  if (kHoles) {
    const bool hole = agg == ~0ull;
    const uint32_t m = __ballot_sync(__activemask(), hole);
    if (hole) {
      if ((threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(bad + 2, (unsigned long long)__popc(m));
      agg = n_agg;
    } else if (agg >= n_agg) {
      atomicAdd(bad, 1ull);
    }
  } else if (agg >= n_agg) {
    atomicAdd(bad, 1ull);
  }
  keys[i] = (uint32_t)agg;
  idx[i] = i;
}

// ---------------------------------------------------------------- CSR offsets from sorted keys
// full mode: offsets[a] = 64 * lower_bound(sorted, a) for a in [0, n_agg]
__global__ void offsets_full_kernel(const uint32_t* __restrict__ sorted, uint32_t n, uint64_t n_agg, uint64_t* __restrict__ offsets) {
  const uint64_t a = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (a > n_agg) return;
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if ((uint64_t)sorted[mid] < a) lo = mid + 1; else hi = mid;
  }
  offsets[a] = (uint64_t)lo * 64;
}

// compact mode: heads[j] = 1 where a new aggregate starts in the sorted order
__global__ void heads_kernel(const uint32_t* __restrict__ sorted, uint32_t n, uint32_t* __restrict__ heads) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  heads[j] = (j == 0 || sorted[j] != sorted[j - 1]) ? 1u : 0u;
}
// kHoles: the n_holes holes sort last and are left out; a poll of holes only leaves n_touched == 0 (zeroed with the counters)
template <bool kHoles>
__global__ void compact_kernel(const uint32_t* __restrict__ sorted, uint32_t n, const uint32_t* __restrict__ heads,
                               const uint32_t* __restrict__ pos, uint32_t* __restrict__ ids, uint64_t* __restrict__ offsets,
                               unsigned long long* __restrict__ n_touched, const unsigned long long* __restrict__ n_holes) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (kHoles) {
    n -= (uint32_t)*n_holes;
    if (n == 0 && j == 0) offsets[0] = 0;
  }
  if (j >= n) return;
  if (heads[j]) { ids[pos[j]] = sorted[j]; offsets[pos[j]] = (uint64_t)j * 64; }
  if (j == n - 1) {
    const uint32_t t = pos[j] + heads[j];
    offsets[t] = (uint64_t)n * 64;
    *n_touched = t;
  }
}

// ---------------------------------------------------------------- gather: out[j] = rec[idx[j]], 4 lanes x 16 bytes per record
// kHoles: only the n - n_holes live records move (the holes sort last)
template <bool kHoles>
__global__ void gather_records_kernel(const uint8_t* __restrict__ rec, const uint32_t* __restrict__ idx, uint32_t n, uint8_t* __restrict__ out,
                                      const unsigned long long* __restrict__ n_holes) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (kHoles) n -= (uint32_t)*n_holes;
  const uint64_t j = t >> 2;
  if (j >= n) return;
  const uint32_t part = (uint32_t)t & 3u;
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(rec + (size_t)idx[j] * 64) + part);
  reinterpret_cast<uint4*>(out + j * 64)[part] = v;
}

__global__ void clear_flags_kernel(uint8_t* __restrict__ states, uint32_t state_bytes, const uint32_t* __restrict__ ids, uint64_t n) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t slot = ids ? (uint64_t)ids[i] : i;
  uint2* p = reinterpret_cast<uint2*>(states + slot * state_bytes + state_bytes - 8);
  uint2 v = *p;
  v.x &= SGR_ST_EXISTS; v.y = 0;
  *p = v;
}

inline uint32_t cdiv(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }

}  // namespace

cudaError_t exclusive_sum_u32(const uint32_t* in, uint32_t* out, uint32_t n, DevBuf& tmp, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  size_t bytes = 0;
  cudaError_t e;
  if ((e = cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, st)) != cudaSuccess || (e = tmp.reserve(bytes)) != cudaSuccess) return e;
  return cub::DeviceScan::ExclusiveSum(tmp.p, bytes, in, out, n, st);
}

void clear_batch_flags(uint8_t* d_states, uint32_t state_bytes, const uint32_t* d_ids, uint64_t n, cudaStream_t stream) {
  if (!n) return;
  clear_flags_kernel<<<cdiv(n, 256), 256, 0, stream>>>(d_states, state_bytes, d_ids, n);
}

cudaError_t group_by_agg_stable(GroupScratch& sc, const uint8_t* d_records, uint64_t n64, uint64_t n_agg,
                                uint8_t* d_out_records, uint64_t* d_out_offsets, uint32_t* d_touched_ids,
                                uint64_t* n_touched, unsigned long long* d_counters, cudaStream_t st,
                                unsigned long long* bad_out, unsigned long long* holes_out) {
  const uint32_t n = (uint32_t)n64;
  cudaError_t e;
  *bad_out = 0;
  if (n_touched) *n_touched = 0;
  if (holes_out) *holes_out = 0;
  if (n == 0) {
    // empty batch: every aggregate has an empty segment
    if (!d_touched_ids) {
      if ((e = cudaMemsetAsync(d_out_offsets, 0, (n_agg + 1) * 8, st)) != cudaSuccess) return e;
    } else if ((e = cudaMemsetAsync(d_out_offsets, 0, 8, st)) != cudaSuccess) return e;
    return cudaStreamSynchronize(st);
  }
  if ((e = sc.keys_a.reserve((size_t)n * 4)) != cudaSuccess || (e = sc.keys_b.reserve((size_t)n * 4)) != cudaSuccess ||
      (e = sc.idx_a.reserve((size_t)n * 4)) != cudaSuccess || (e = sc.idx_b.reserve((size_t)n * 4)) != cudaSuccess)
    return e;
  cub::DoubleBuffer<uint32_t> keys((uint32_t*)sc.keys_a.p, (uint32_t*)sc.keys_b.p), idx((uint32_t*)sc.idx_a.p, (uint32_t*)sc.idx_b.p);
  // the keys run up to n_agg - 1, or up to n_agg with holes
  const uint64_t key_end = holes_out ? n_agg + 1 : n_agg;
  int bits = 1;
  while (bits < 32 && (1ull << bits) < key_end) ++bits;
  size_t sort_bytes = 0;
  if ((e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, idx, n, 0, bits, st)) != cudaSuccess ||
      (e = sc.cub_tmp.reserve(sort_bytes)) != cudaSuccess)
    return e;

  if ((e = cudaMemsetAsync(d_counters, 0, 64, st)) != cudaSuccess) return e;
  if (holes_out) extract_keys_kernel<true><<<cdiv(n, 256), 256, 0, st>>>(d_records, n, n_agg, keys.Current(), idx.Current(), d_counters + 4);
  else extract_keys_kernel<false><<<cdiv(n, 256), 256, 0, st>>>(d_records, n, n_agg, keys.Current(), idx.Current(), d_counters + 4);
  if ((e = cub::DeviceRadixSort::SortPairs(sc.cub_tmp.p, sort_bytes, keys, idx, n, 0, bits, st)) != cudaSuccess) return e;
  // sorted keys and the arrival indices in CSR order, holes last (the full-mode lower bound of n_agg is the first hole, so
  // offsets[n_agg] ends the CSR before them)
  const uint32_t* sorted = keys.Current();
  const uint32_t* order = idx.Current();
  const unsigned long long* d_holes = d_counters + 6;
  if (!d_touched_ids) {
    offsets_full_kernel<<<cdiv(n_agg + 1, 256), 256, 0, st>>>(sorted, n, n_agg, d_out_offsets);
  } else {
    if ((e = sc.flags.reserve((size_t)n * 8)) != cudaSuccess) return e;
    uint32_t* heads = (uint32_t*)sc.flags.p;
    uint32_t* pos = heads + n;
    heads_kernel<<<cdiv(n, 256), 256, 0, st>>>(sorted, n, heads);
    if ((e = exclusive_sum_u32(heads, pos, n, sc.cub_tmp, st)) != cudaSuccess) return e;
    if (holes_out) compact_kernel<true><<<cdiv(n, 256), 256, 0, st>>>(sorted, n, heads, pos, d_touched_ids, d_out_offsets, d_counters + 5, d_holes);
    else compact_kernel<false><<<cdiv(n, 256), 256, 0, st>>>(sorted, n, heads, pos, d_touched_ids, d_out_offsets, d_counters + 5, nullptr);
  }
  if (holes_out) gather_records_kernel<true><<<cdiv((uint64_t)n * 4, 256), 256, 0, st>>>(d_records, order, n, d_out_records, d_holes);
  else gather_records_kernel<false><<<cdiv((uint64_t)n * 4, 256), 256, 0, st>>>(d_records, order, n, d_out_records, nullptr);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  unsigned long long h[3];
  if ((e = cudaMemcpyAsync(h, d_counters + 4, holes_out ? 24 : 16, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
  *bad_out = h[0];
  if (n_touched) *n_touched = h[1];
  if (holes_out) *holes_out = h[2];
  return cudaSuccess;
}

}  // namespace sgr
