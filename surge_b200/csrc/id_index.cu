// id_index.cu — batched recovery reads on the device (sgr_get_batch): insert, rehash, probe and gather kernels over the
// engine's id index (id_index.cuh), all in the dictionary layout of id_dict.cuh.
//
//   insert  one thread per new id: insert_at(its dense index); a rehash is the same launch over every resident id into cleared
//           slots, so ids are uploaded once
//   probe   one thread per query id: hash, probe, write the dense index or -1
//   gather  state_bytes / 16 threads per query row, each one 16-byte load of the found row (a row's threads are adjacent, so its
//           loads coalesce): program bytes out as 8-byte stores (rows are state_bytes - 8 long), the flags word by the row's last
//           thread
#include <string.h>

#include "../../include/sgr.h"
#include "id_index.cuh"

namespace sgr {
namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) gb_insert_kernel(const DgDict d, uint64_t from, uint64_t to) {
  const uint64_t i = from + (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i < to) insert_at(d, (uint32_t)i);
}

__global__ void __launch_bounds__(kThreads) gb_probe_kernel(const DgDict d, const uint8_t* __restrict__ q, const uint32_t* __restrict__ q_offs,
                                                            uint64_t n, long long* __restrict__ idx) {
  const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const uint32_t b = q_offs[i];
  idx[i] = find(d, q + b, q_offs[i + 1] - b);
}

__global__ void __launch_bounds__(kThreads) gb_gather_kernel(const uint8_t* __restrict__ states, uint32_t state_bytes, uint64_t n_states,
                                                             const long long* __restrict__ idx, uint64_t n, uint8_t* __restrict__ rows,
                                                             uint32_t* __restrict__ flags, unsigned long long* __restrict__ bad) {
  const uint32_t w = state_bytes >> 4;
  const uint64_t t = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  const uint64_t i = t / w;
  const uint32_t c = (uint32_t)(t - i * w);
  if (i >= n) return;
  const long long a = idx[i];
  uint4 v = make_uint4(0, 0, 0, 0);
  uint32_t fl = 0;
  if (a >= 0 && (uint64_t)a < n_states) {
    const uint8_t* row = states + (uint64_t)a * state_bytes;
    fl = __ldg(reinterpret_cast<const uint32_t*>(row + state_bytes - 8));
    if (fl & SGR_ST_EXISTS) v = __ldg(reinterpret_cast<const uint4*>(row) + c);
  } else if (a >= 0 && c == 0) {
    atomicMax(bad, (unsigned long long)a + 1ull);
  }
  uint2* o = reinterpret_cast<uint2*>(rows + i * (state_bytes - 8) + 16ull * c);
  o[0] = make_uint2(v.x, v.y);
  if (c + 1 < w) o[1] = make_uint2(v.z, v.w);
  else flags[i] = fl;
}

uint32_t blocks_for(uint64_t n) { return (uint32_t)((n + kThreads - 1) / kThreads); }

// grow a device buffer to at least `need` bytes, doubling from 4096, keeping its first `keep` bytes
cudaError_t grow_doubling(DevBuf& b, size_t need, size_t keep, cudaStream_t st) {
  if (need <= b.cap) return cudaSuccess;
  size_t cap = b.cap ? b.cap : 4096;
  while (cap < need) cap *= 2;
  return b.grow_keep(cap, keep, st);
}

}  // namespace

uint64_t id_index_stage_bytes(const uint32_t* offs, uint64_t from, uint64_t to, bool* monotone) {
  *monotone = true;
  uint64_t bytes = (to - from) * sizeof(uint2);
  for (uint64_t i = from; i < to; ++i) {
    if (offs[i + 1] < offs[i]) { *monotone = false; return 0; }
    bytes += ((uint64_t)(offs[i + 1] - offs[i]) + 7) & ~7ull;
  }
  return bytes;
}

cudaError_t id_index_append(IdIndex& x, const uint8_t* bytes, const uint32_t* offs, uint64_t to, void* stage, unsigned long long* d_ctl,
                            cudaStream_t st) {
  const uint64_t from = x.n;
  if (to <= from) return cudaSuccess;
  const uint64_t n_new = to - from;
  // refs then bytes, in the layout they take on the device
  uint2* refs = (uint2*)stage;
  uint8_t* arena = (uint8_t*)stage + n_new * sizeof(uint2);
  uint64_t pos = 0;
  for (uint64_t i = 0; i < n_new; ++i) {
    const uint32_t len = offs[from + i + 1] - offs[from + i];
    memcpy(arena + pos, bytes + offs[from + i], len);
    refs[i] = make_uint2((uint32_t)((x.arena_used + pos) >> 3), len);
    pos += ((uint64_t)len + 7) & ~7ull;
  }
  cudaError_t e;
  if ((e = id_index_reserve(x, to, x.arena_used + pos + 8, st)) != cudaSuccess) return e;
  if ((e = cudaMemcpyAsync((uint2*)x.key_ref.p + from, refs, n_new * sizeof(uint2), cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  if (pos && (e = cudaMemcpyAsync((uint8_t*)x.arena.p + x.arena_used, arena, pos, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  x.arena_used += pos;
  return id_index_insert(x, to, d_ctl, st);
}

cudaError_t id_index_reserve(IdIndex& x, uint64_t ids, uint64_t arena_bytes, cudaStream_t st) {
  cudaError_t e = grow_doubling(x.key_ref, ids * sizeof(uint2), x.n * sizeof(uint2), st);
  return e != cudaSuccess ? e : grow_doubling(x.arena, arena_bytes, x.arena_used, st);
}

cudaError_t id_index_insert(IdIndex& x, uint64_t to, unsigned long long* d_ctl, cudaStream_t st) {
  if (to <= x.n) return cudaSuccess;
  cudaError_t e;
  uint64_t insert_from = x.n;
  if (2 * to > x.slots) {
    // load factor past 1/2: a table of at least twice the ids, every resident id inserted again (nothing is uploaded twice)
    uint64_t slots = 1024;
    while (slots < 2 * to) slots *= 2;
    if ((e = x.tags.reserve(slots * 8)) != cudaSuccess) return e;
    if ((e = x.slot_idx.reserve(slots * 4)) != cudaSuccess) return e;
    x.slots = slots;
    insert_from = 0;
  }
  if (insert_from == 0) {
    if ((e = cudaMemsetAsync(x.tags.p, 0, x.slots * 8, st)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(x.slot_idx.p, 0, x.slots * 4, st)) != cudaSuccess) return e;
  }
  x.n = to;
  gb_insert_kernel<<<blocks_for(to - insert_from), kThreads, 0, st>>>(x.dict(d_ctl), insert_from, to);
  return cudaGetLastError();
}

cudaError_t id_index_probe(const IdIndex& x, const uint8_t* q, const uint32_t* q_offs, uint64_t n, long long* idx, cudaStream_t st) {
  if (!n) return cudaSuccess;
  if (!x.n) return cudaMemsetAsync(idx, 0xff, n * sizeof(long long), st);   // no key table: every id is unknown
  gb_probe_kernel<<<blocks_for(n), kThreads, 0, st>>>(x.dict(nullptr), q, q_offs, n, idx);
  return cudaGetLastError();
}

cudaError_t id_index_gather(const uint8_t* states, uint32_t state_bytes, uint64_t n_states, const long long* idx, uint64_t n,
                            uint8_t* rows, uint32_t* flags, unsigned long long* bad, cudaStream_t st) {
  if (!n) return cudaSuccess;
  gb_gather_kernel<<<blocks_for(n * (state_bytes / 16)), kThreads, 0, st>>>(states, state_bytes, n_states, idx, n, rows, flags, bad);
  return cudaGetLastError();
}

}  // namespace sgr
