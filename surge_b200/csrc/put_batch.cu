// put_batch.cu — keyed state writes on the device (sgr_put_batch): a batch of (id, row | tombstone) records in arrival order
// becomes the last write per id in the live table, the KTable a state topic restores (SurgeStateStoreConsumer.scala:57-76).
//
//   probe    one thread per record: find() in the engine's id index; an unknown id claims a slot of a batch-local table
//            (open addressing on the same 64-bit hash, ids compared byte for byte against the slot's first claimant) and
//            atomicMin's its batch position there, so the table ends up holding each new id's first appearance
//   first    one thread per record: 1 at a new id's first appearance, with the id's 8-byte aligned length; the new ids' unaligned
//            bytes are summed per warp into one counter (the host key table's size check)
//   scans    cub::DeviceScan::ExclusiveSum over both: new id k (first-appearance order) gets dense index n_keys + k and arena
//            offset aoff
//   resolve  one thread per record: its dense index; a first appearance also writes its key_ref, its bytes into the arena and
//            its batch position into new_pos[k] (what the host appends to its key table: no id bytes come back)
//   last     one thread per record: atomicMax(last[slot], position + 1)
//            (last and write skip a slot of ~0u: the holes of a device-ingest poll of a state topic, put_decoded_poll)
//   write    one thread per record: the record whose position + 1 is last[slot] zeroes last[slot], compares its row with the
//            prior state (program_words_differ: the publish rule the fold kernels use) and writes the row, its flags and
//            err_idx 0; the written indices are appended to `touched` by one atomic per warp
//
// Why an atomic max and not a sort of (slot, position) pairs: each record needs only one 4-byte atomic on its slot's word, the
// word stays zero between batches (the winner clears it), and the batch is never reordered, so the scratch is 4 bytes per
// table row instead of a sort's two key and value buffers per record plus its temporary storage. Repeated ids contend on one
// word each, which costs nothing measurable next to the row writes.
#include <cub/cub.cuh>

#include "../../include/sgr.h"
#include "put_batch.cuh"

namespace sgr {
namespace {

constexpr int kThreads = 256;

uint32_t blocks_for(uint64_t n) { return (uint32_t)((n + kThreads - 1) / kThreads); }
size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

uint64_t bt_slots(uint64_t n) {
  uint64_t s = 1024;
  while (s < 2 * n) s *= 2;
  return s;
}

size_t cub_scan_bytes(uint64_t n) {
  size_t a = 0, b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, a, (const uint32_t*)nullptr, (uint32_t*)nullptr, (uint64_t)(n + 1));
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (uint64_t)(n + 1));
  return a > b ? a : b;
}

// The slot of record i's (unknown) id in the batch table; ~0u when the table is full.
__device__ __forceinline__ uint32_t bt_claim(const PutBatch& p, uint32_t i, const uint8_t* id, uint32_t len) {
  const unsigned long long h = hash_id(id, len);
  uint64_t pos = h & p.bt_mask;
  for (uint64_t probes = 0; probes <= p.bt_mask; ++probes, pos = (pos + 1) & p.bt_mask) {
    unsigned long long tag = __ldcg(p.bt_tags + pos);
    if (tag == 0ull) {
      tag = atomicCAS(p.bt_tags + pos, 0ull, h);
      if (tag == 0ull) {   // this record owns the slot: its bytes (staged before the launch) stand for the id
        atomicExch(p.bt_owner + pos, i + 1u);
        atomicMin(p.bt_min + pos, i);
        return (uint32_t)pos;
      }
    }
    if (tag != h) continue;
    uint32_t v;
    while ((v = ld_volatile_u32(p.bt_owner + pos)) == 0u) __nanosleep(40);   // the owner is still publishing its position
    const uint32_t b = p.offs[v - 1u];
    if (p.offs[v] - b != len) continue;
    const uint8_t* have = p.ids + b;
    bool same = true;
    for (uint32_t k = 0; k < len && same; ++k) same = have[k] == id[k];
    if (same) { atomicMin(p.bt_min + pos, i); return (uint32_t)pos; }
  }
  atomicAdd(p.ctl + kPbFull, 1ull);
  return ~0u;
}

__global__ void __launch_bounds__(kThreads) pb_probe_kernel(const DgDict d, bool have_index, const PutBatch p) {
  const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i >= p.n) return;
  const uint32_t b = p.offs[i], len = p.offs[i + 1] - b;
  const long long f = have_index ? find(d, p.ids + b, len) : -1;
  if (f >= 0) { p.probe[i] = f; return; }
  const uint32_t s = bt_claim(p, (uint32_t)i, p.ids + b, len);
  p.probe[i] = s == ~0u ? -1 : -(long long)s - 1;   // (a full table fails the batch)
}

__global__ void __launch_bounds__(kThreads) pb_first_kernel(const PutBatch p) {
  const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  uint32_t new_bytes = 0;
  if (i < p.n) {
    const long long s = p.probe[i];
    const uint32_t len = p.offs[i + 1] - p.offs[i];
    const bool fi = s < 0 && p.bt_min[-(s + 1)] == (uint32_t)i;
    p.first[i] = fi ? 1u : 0u;
    p.alen[i] = fi ? ((unsigned long long)len + 7) & ~7ull : 0ull;
    new_bytes = fi ? len : 0u;
  } else if (i == p.n) {
    p.first[i] = 0u;
    p.alen[i] = 0ull;
  }
  new_bytes = __reduce_add_sync(0xffffffffu, new_bytes);   // (a batch's id bytes are fewer than 2^32)
  if ((threadIdx.x & 31) == 0 && new_bytes) atomicAdd(p.ctl + kPbNewBytes, (unsigned long long)new_bytes);
}

__global__ void __launch_bounds__(kThreads) pb_resolve_kernel(const PutBatch p, uint2* __restrict__ key_ref, uint8_t* __restrict__ arena,
                                                              uint64_t arena_used) {
  const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i == 0) { p.ctl[kPbNewIds] = p.rank[p.n]; p.ctl[kPbNewIds + 1] = p.aoff[p.n]; }
  if (i >= p.n) return;
  const long long s = p.probe[i];
  if (s >= 0) { p.slot[i] = (uint32_t)s; return; }
  const uint32_t m = p.bt_min[-(s + 1)];
  const uint32_t k = p.rank[m];
  p.slot[i] = (uint32_t)(p.n_keys + k);
  if (m != (uint32_t)i) return;
  const uint32_t b = p.offs[i], len = p.offs[i + 1] - b;
  const uint64_t off = arena_used + p.aoff[i];
  p.new_pos[k] = (uint32_t)i;
  key_ref[p.n_keys + k] = make_uint2((uint32_t)(off >> 3), len);
  for (uint32_t c = 0; c < len; ++c) arena[off + c] = p.ids[b + c];
}

__global__ void __launch_bounds__(kThreads) pb_last_kernel(const PutBatch p, uint32_t* __restrict__ last) {
  const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  if (i < p.n && p.slot[i] != ~0u) atomicMax(last + p.slot[i], (uint32_t)i + 1u);   // (~0u: a hole of a device-ingest poll)
}

__global__ void __launch_bounds__(kThreads) pb_write_kernel(const PutBatch p, uint8_t* __restrict__ states, const __grid_constant__ DevProgram prog,
                                                            uint32_t* __restrict__ last, uint32_t* __restrict__ touched) {
  const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  const uint32_t uw = prog.user_words;
  uint32_t sl = 0;
  bool win = false;
  if (i < p.n) {
    sl = p.slot[i];
    win = sl != ~0u && last[sl] == (uint32_t)i + 1u;   // (the winner zeroes the word: no other record of the slot ever reads its own position)
  }
  if (win) {
    last[sl] = 0u;
    uint32_t* st = reinterpret_cast<uint32_t*>(states + (uint64_t)sl * (4ull * (uw + 2)));
    const uint32_t ex0 = st[uw] & SGR_ST_EXISTS;
    uint32_t flags;
    if (p.present[i]) {
      // a snapshot is a new instance: CREATE + SET of every program byte
      const uint32_t* row = reinterpret_cast<const uint32_t*>(p.rows + i * (4ull * uw));
      const bool changed = !ex0 || program_words_differ(prog, uw, [&](uint32_t w) { return row[w]; }, [&](uint32_t w) { return st[w]; }, 1u);
      for (uint32_t w = 0; w < uw; ++w) st[w] = row[w];
      flags = SGR_ST_EXISTS | (changed ? SGR_ST_CHANGED : 0u);
    } else {
      for (uint32_t w = 0; w < uw; ++w) st[w] = 0u;
      flags = ex0 ? SGR_ST_CHANGED : 0u;
    }
    *reinterpret_cast<uint2*>(st + uw) = make_uint2(flags, 0u);
  }
  const uint32_t m = __ballot_sync(0xffffffffu, win);
  const int lane = threadIdx.x & 31, leader = m ? __ffs(m) - 1 : 0;
  unsigned long long base = 0;
  if (m && lane == leader) base = atomicAdd(p.ctl + kPbTouched, (unsigned long long)__popc(m));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (win) touched[base + __popc(m & ((1u << lane) - 1u))] = sl;
}

}  // namespace

size_t put_batch_scratch_bytes(uint64_t n) {
  const uint64_t m = n + 1, bs = bt_slots(n);
  return 64 + align16(8 * n) + 2 * align16(4 * m) + 2 * align16(8 * m) + 2 * align16(4 * n) + align16(8 * bs) + 2 * align16(4 * bs) +
         align16(cub_scan_bytes(n));
}

void put_batch_carve(PutBatch& p, void* base, uint64_t n) {
  const uint64_t m = n + 1, bs = bt_slots(n);
  uint8_t* c = (uint8_t*)base;
  auto take = [&](size_t bytes) { uint8_t* r = c; c += align16(bytes); return r; };
  p.ctl = (unsigned long long*)take(64);
  p.probe = (long long*)take(8 * n);
  p.first = (uint32_t*)take(4 * m);
  p.rank = (uint32_t*)take(4 * m);
  p.alen = (unsigned long long*)take(8 * m);
  p.aoff = (unsigned long long*)take(8 * m);
  p.slot = (uint32_t*)take(4 * n);
  p.new_pos = (uint32_t*)take(4 * n);
  p.bt_tags = (unsigned long long*)take(8 * bs);
  p.bt_owner = (uint32_t*)take(4 * bs);
  p.bt_min = (uint32_t*)take(4 * bs);
  p.bt_mask = bs - 1;
  p.cub_bytes = cub_scan_bytes(n);
  p.cub_tmp = take(p.cub_bytes);
}

cudaError_t put_batch_resolve(const IdIndex& x, uint64_t arena_used, PutBatch& p, cudaStream_t st) {
  if (!p.n) return cudaSuccess;
  const uint64_t bs = p.bt_mask + 1;
  cudaError_t e;
  if ((e = cudaMemsetAsync(p.ctl, 0, 64, st)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(p.bt_tags, 0, 8 * bs, st)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(p.bt_owner, 0, 4 * bs, st)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(p.bt_min, 0xff, 4 * bs, st)) != cudaSuccess) return e;
  pb_probe_kernel<<<blocks_for(p.n), kThreads, 0, st>>>(x.dict(nullptr), x.n > 0, p);
  pb_first_kernel<<<blocks_for((uint64_t)p.n + 1), kThreads, 0, st>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  size_t tb = p.cub_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(p.cub_tmp, tb, p.first, p.rank, (uint64_t)p.n + 1, st)) != cudaSuccess) return e;
  tb = p.cub_bytes;
  if ((e = cub::DeviceScan::ExclusiveSum(p.cub_tmp, tb, p.alen, p.aoff, (uint64_t)p.n + 1, st)) != cudaSuccess) return e;
  pb_resolve_kernel<<<blocks_for(p.n), kThreads, 0, st>>>(p, (uint2*)x.key_ref.p, (uint8_t*)x.arena.p, arena_used);
  return cudaGetLastError();
}

cudaError_t put_batch_apply(const PutBatch& p, uint8_t* states, const DevProgram& prog, uint32_t* last, uint32_t* touched,
                            cudaStream_t st) {
  if (!p.n) return cudaSuccess;
  pb_last_kernel<<<blocks_for(p.n), kThreads, 0, st>>>(p, last);
  pb_write_kernel<<<blocks_for(p.n), kThreads, 0, st>>>(p, states, prog, last, touched);
  return cudaGetLastError();
}

}  // namespace sgr
