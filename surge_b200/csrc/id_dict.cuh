// id_dict.cuh — the device aggregate-id dictionary: open addressing on a 64-bit hash, ids compared byte for byte.
//
// Two owners use this one layout and probe: the device ingest interns ids as it parses records (intern: the dense index comes
// from an atomic counter, csrc/dingest_kernels.cu), and the engine's id index (csrc/id_index.cu) inserts ids whose dense index
// is their position in the key table (insert_at) and answers batched recovery reads (find). The id order of the ordered scan
// (csrc/id_order.cu) compares ids in Bytes order with cmp_ids.
//
// tests/fuzz/id_dict_main.cpp builds this header for the host (SGR_ID_DICT_HOST, with single-threaded stand-ins for the atomics
// and cache-hinted loads) and checks intern, insert_at and find against a Python dict on ids built to share one tag.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sgr {

struct DgDict {           // device id dictionary: open addressing on a 64-bit hash, ids compared byte for byte
  unsigned long long* tags;   // [slots] 0 = empty, else the id's hash (never 0)
  uint32_t* slot_idx;         // [slots] dense index + 1 once the owner has published the id (0 = not yet)
  uint2* key_ref;             // [max_keys] (arena offset in 8-byte units, length) of dense index i
  uint8_t* arena;             // id bytes, 8-byte aligned entries
  unsigned long long* ctl;    // [0] n_keys [1] arena bytes used [2] records dropped as markers [3] null values [4] duplicates
                              // [5] dictionary overflow (keys or arena) [6] packed records written (non-holes)
                              // [8] [9] [10] decode arena: bytes claimed, capacity, overflow flag (dg_launch_crc_size_fast)
                              // (the engine's id index uses [0] duplicate ids, [1] overflow)
  uint64_t slots_mask;        // slots - 1 (power of two)
  uint64_t max_keys, arena_cap;
};

#if defined(__CUDACC__) || defined(SGR_ID_DICT_HOST)
namespace {

__device__ __forceinline__ unsigned long long hash_id(const uint8_t* k, uint32_t len) {
  unsigned long long h = 0x9e3779b97f4a7c15ull ^ ((unsigned long long)len * 0xff51afd7ed558ccdull);
  while (len >= 8) {
    unsigned long long w = 0;
    for (int q = 7; q >= 0; --q) w = (w << 8) | k[q];
    h = (h ^ w) * 0x9fb21c651e98df25ull; h ^= h >> 32; k += 8; len -= 8;
  }
  if (len) {
    unsigned long long w = 0;
    for (int q = (int)len - 1; q >= 0; --q) w = (w << 8) | k[q];
    h = (h ^ w) * 0x9fb21c651e98df25ull; h ^= h >> 32;
  }
  h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 29;
  return h ? h : 1ull;
}

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
#ifdef __CUDA_ARCH__
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
#else
  return *(const volatile uint32_t*)p;
#endif
}

// id -> dense index. Returns 0xffffffff when the dictionary is full (the call then fails as a whole).
//
// A new id takes its arena bytes first and a dense index only if the bytes fit, so every index below max_keys is written and
// none is lost to a claim refused on bytes. ctl[0] and ctl[1] still count refused claims: readers clamp them to max_keys and
// arena_cap. A refused claim leaves its slot dead (slot_idx 0xffffffff): probes step over it, so an admitted id further along
// the same chain is still found, and the refused id, arriving again, claims a new slot and is refused again.
__device__ uint32_t intern(const DgDict& d, const uint8_t* id, uint32_t len) {
  const unsigned long long h = hash_id(id, len);
  uint64_t pos = h & d.slots_mask;
  for (uint64_t probes = 0; probes <= d.slots_mask; ++probes, pos = (pos + 1) & d.slots_mask) {
    unsigned long long tag = __ldcg(d.tags + pos);
    if (tag == 0ull) {
      tag = atomicCAS(d.tags + pos, 0ull, h);
      if (tag == 0ull) {   // this thread owns the slot: the id is new
        const unsigned long long need = ((unsigned long long)len + 7) & ~7ull;
        const unsigned long long off = atomicAdd(d.ctl + 1, need);
        const unsigned long long idx = off + need <= d.arena_cap ? atomicAdd(d.ctl + 0, 1ull) : ~0ull;
        if (idx >= d.max_keys) {
          atomicAdd(d.ctl + 5, 1ull);
          __threadfence();
          atomicExch(d.slot_idx + pos, 0xffffffffu);
          return 0xffffffffu;
        }
        for (uint32_t k = 0; k < len; ++k) d.arena[off + k] = id[k];
        d.key_ref[idx] = make_uint2((uint32_t)(off >> 3), len);
        __threadfence();
        atomicExch(d.slot_idx + pos, (uint32_t)idx + 1u);
        return (uint32_t)idx;
      }
    }
    if (tag != h) continue;
    uint32_t v;
    while ((v = ld_volatile_u32(d.slot_idx + pos)) == 0u) __nanosleep(40);   // the owner is still writing the id
    if (v == 0xffffffffu) continue;                                           // a dead slot
    __threadfence();
    // (L2 loads: an L1 line fetched before the owner wrote its part would be stale)
    const uint2 ref = __ldcg(d.key_ref + (v - 1u));
    if (ref.y != len) continue;                                               // same 64-bit hash, another id: keep probing
    const uint8_t* have = d.arena + ((unsigned long long)ref.x << 3);
    bool same = true;
    for (uint32_t k = 0; k < len && same; ++k) same = __ldcg(have + k) == id[k];
    if (same) return v - 1u;
  }
  atomicAdd(d.ctl + 5, 1ull);
  return 0xffffffffu;
}

// Dense index `idx` -> a slot, for a dictionary whose key_ref[idx] and id bytes are already in place (written before the
// launch). Ids inserted by one launch are distinct slots unless two of them are equal: the second one to probe then finds the
// first published under the same tag with the same bytes, and the id is counted in ctl[0] (a duplicate id). ctl[1] counts
// probes that found no free slot (the table is sized so that this does not happen).
__device__ __forceinline__ void insert_at(const DgDict& d, uint32_t idx) {
  const uint2 mine = d.key_ref[idx];
  const uint8_t* id = d.arena + ((unsigned long long)mine.x << 3);
  const uint32_t len = mine.y;
  const unsigned long long h = hash_id(id, len);
  uint64_t pos = h & d.slots_mask;
  for (uint64_t probes = 0; probes <= d.slots_mask; ++probes, pos = (pos + 1) & d.slots_mask) {
    unsigned long long tag = __ldcg(d.tags + pos);
    if (tag == 0ull) {
      tag = atomicCAS(d.tags + pos, 0ull, h);
      if (tag == 0ull) { atomicExch(d.slot_idx + pos, idx + 1u); return; }
    }
    if (tag != h) continue;
    uint32_t v;
    while ((v = ld_volatile_u32(d.slot_idx + pos)) == 0u) __nanosleep(40);   // the owner is still publishing its index
    const uint2 ref = d.key_ref[v - 1u];
    if (ref.y != len) continue;
    const uint8_t* have = d.arena + ((unsigned long long)ref.x << 3);
    bool same = true;
    for (uint32_t k = 0; k < len && same; ++k) same = have[k] == id[k];
    if (same) { atomicAdd(d.ctl + 0, 1ull); return; }
  }
  atomicAdd(d.ctl + 1, 1ull);
}

// Lookup only, on a dictionary no kernel is writing: the dense index of the id, or -1.
__device__ __forceinline__ long long find(const DgDict& d, const uint8_t* id, uint32_t len) {
  const unsigned long long h = hash_id(id, len);
  uint64_t pos = h & d.slots_mask;
  for (uint64_t probes = 0; probes <= d.slots_mask; ++probes, pos = (pos + 1) & d.slots_mask) {
    const unsigned long long tag = d.tags[pos];
    if (tag == 0ull) return -1;
    if (tag != h) continue;
    const uint32_t v = d.slot_idx[pos];
    const uint2 ref = d.key_ref[v - 1u];
    if (ref.y != len) continue;
    const uint8_t* have = d.arena + ((unsigned long long)ref.x << 3);
    bool same = true;
    for (uint32_t k = 0; k < len && same; ++k) same = have[k] == id[k];
    if (same) return (long long)(v - 1u);
  }
  return -1;
}

// The 8 bytes at p (8-byte aligned) as a big-endian word: p[0] is the most significant byte.
__device__ __forceinline__ unsigned long long be_word(const uint8_t* p) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  return ((unsigned long long)__byte_perm(v.x, 0, 0x0123) << 32) | __byte_perm(v.y, 0, 0x0123);
}

// Bytes order of two ids (unsigned lexicographic, a prefix before any longer id): < 0, 0 or > 0 as a sorts before, equal to or
// after b. Both start 8-byte aligned and are readable in whole words up to their length rounded up to 8 (arena entries, or a
// staged query); bytes past an id's length are masked off, whatever they hold.
__device__ __forceinline__ int cmp_ids(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  const uint32_t n = la < lb ? la : lb;
  for (uint32_t k = 0; k < n; k += 8) {
    unsigned long long wa = be_word(a + k), wb = be_word(b + k);
    if (n - k < 8) {
      const unsigned long long keep = ~0ull << (64 - 8 * (n - k));
      wa &= keep; wb &= keep;
    }
    if (wa != wb) return wa < wb ? -1 : 1;
  }
  return la < lb ? -1 : (la > lb ? 1 : 0);
}

}  // namespace
#endif

}  // namespace sgr
