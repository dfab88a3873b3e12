// route_push.cu — pipelined route + exchange + fold over peer memory (sm_90a, NVLink 4 / NVSwitch).
//
// The reference shards by key and lets the BROKER shuffle: aggregateId -> partitionForKey
// (modules/common/src/main/scala/surge/kafka/KafkaPartitioner.scala:7-9) -> owner node
// (KafkaProducerHelperCommon.getPartitionFor, modules/common/src/main/scala/surge/kafka/KafkaProducer.scala:45-57).
// Here every rank holds the records of its source partitions in arrival order and ONE pass does route + all-to-all:
//
//   source log, cut into C chunks in log order
//     push kernel (one launch per chunk, 1024 records per CTA):
//        cp.async the CTA's records into shared memory (64 KiB), look up owner | local index of every record,
//        counting-sort the CTA's records by owner in shared memory (stable), obtain the CTA's offset inside each owner's
//        region by a decoupled look-back over the earlier CTAs of the chunk (ordered by a ticket), then write every owner's
//        run CONTIGUOUSLY into region (me, chunk) of that owner's receive buffer through the peer mapping: 512 contiguous
//        bytes per warp store, records rewritten to the owner's local aggregate index. One read of the log, one write, no
//        send buffer, no count pass, no host synchronisation.
//     flag kernel: (epoch << 32 | count + 1) into every owner's header -> region (me, chunk) is complete
//   second stream, per chunk: wait for the flags of all sources, then the sort-free accumulate (bulk_fold.cu) over the
//     chunk's regions; after the last chunk the finish pass by slot. The fold of chunk c overlaps the push of chunk c+1.
//
// Per-aggregate order: all events of an aggregate come from ONE source (one key -> one partition); chunks are in log order,
// the partition inside a CTA is stable, CTAs are ordered by the look-back, and the arrival index the fold uses is
// chunk * region_capacity + position: monotone along the aggregate's own order. Nothing else matters to the fold.
//
// Receive layout on every rank: header | regions [source][chunk] of region_capacity records. Fixed-capacity regions are
// what makes the single pass possible; a region that would overflow drops nothing silently: the sender marks the flag,
// every rank learns it (error gather) and the call fails with SGR_ERR_CAPACITY on ALL ranks before any state is published.
//
// compact != 0: only what the fold program reads crosses NVLink (projection): u32 local index + the program's slot words,
// 16 bytes per record for the Counter model instead of 64.
#include "route_push.cuh"

#include <stdio.h>
#include <string.h>

#include "../../include/sgr.h"
#include "dist_state.h"

namespace sgr {
namespace {

constexpr int kPushThreads = 256;
constexpr int kPushWarps = kPushThreads / 32;           // 8
constexpr unsigned long long kSpinLimit = 1ull << 26;   // ~ seconds: a lost peer must not hang the GPU

struct PushArgs {
  const uint8_t* rec;            // first record of this chunk
  uint32_t n;                    // records in this chunk
  uint32_t nranks;
  uint64_t n_global;
  const uint32_t* route_of;      // owner << 28 | local index
  uint8_t* dst[kMaxRanks];       // region (me, chunk) in every owner's receive buffer
  uint32_t cap_region;           // records
  uint32_t out_bytes;            // 64, or the compact stride
  unsigned long long* lb;        // look-back cells of this chunk: [owner][cta], flag << 62 | count (1 local, 2 inclusive)
  uint32_t n_ctas;               // CTAs (tiles) per chunk: the row length of lb
  uint32_t* ticket;              // CTA order of this chunk
  uint32_t* totals;              // [kMaxRanks]: records sent to each owner by this chunk
  unsigned long long* status;    // [0] records with a global index out of range [1] records that did not fit their region
                                 // [2] spin time-outs [3] error flags received
  uint32_t n_proj;               // compact: number of projected record words
  uint32_t proj_word[7];
  uint32_t ordered;              // 1: CTAs take their place inside the regions in log order (look-back): position == arrival order.
                                 // 0: a CTA takes its place with one atomicAdd per owner; the order travels INSIDE the records
                                 //    (record index within the chunk), which is all the sort-free fold needs
};

// Every routed record carries its index within the source's chunk: full records in the (now free) upper half of the agg field,
// projected records next to the event type: word 1 = min(type, 16) << 27 | index (chunks hold fewer than 2^27 records).
constexpr uint32_t kIdxBits = 27;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_na_v4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// Decoupled look-back of one warp for one owner: the exclusive prefix, over the earlier CTAs of the chunk, of the per-CTA record
// counts for that owner. Every CTA first publishes its own count (flag 1), then sums predecessors back to the nearest one that
// already knows its inclusive prefix (flag 2), 32 predecessors per step (cells are [owner][cta]: a window is one coalesced read),
// and publishes its own inclusive prefix. All lanes return the prefix.
__device__ __forceinline__ uint32_t look_back(unsigned long long* cells, uint32_t bid, uint32_t local, int lane, unsigned long long* status) {
  uint32_t ex = 0;
  if (bid == 0) {
    if (lane == 0) st_relaxed_u64(cells, (2ull << 62) | local);
    return 0;
  }
  if (lane == 0) st_relaxed_u64(cells + bid, (1ull << 62) | local);
  uint32_t hi = bid;                    // predecessors hi-1, hi-2, ... are still to be summed
  unsigned long long spins = 0;
  for (;;) {
    const bool in = (uint32_t)lane < hi;
    const unsigned long long v = in ? ld_relaxed_u64(cells + (hi - 1 - lane)) : (2ull << 62);   // before CTA 0: inclusive 0
    const uint32_t fl = (uint32_t)(v >> 62);
    const uint32_t inc = __ballot_sync(0xffffffffu, fl == 2u);
    const uint32_t need = inc ? ((2u << (__ffs(inc) - 1)) - 1u) : 0xffffffffu;   // lanes up to the nearest inclusive prefix
    if (__ballot_sync(0xffffffffu, fl == 0u) & need) {
      if (++spins > kSpinLimit) { if (lane == 0) atomicAdd(status + 2, 1ull); break; }
      __nanosleep(20);
      continue;
    }
    uint32_t part = ((need >> lane) & 1u) ? (uint32_t)v : 0u;
#pragma unroll
    for (int of = 16; of; of >>= 1) part += __shfl_xor_sync(0xffffffffu, part, of);
    ex += part;
    if (inc) break;
    hi -= 32;
  }
  if (lane == 0) st_relaxed_u64(cells + bid, (2ull << 62) | (ex + local));
  return ex;
}

extern __shared__ __align__(16) uint8_t push_smem[];

// One CTA = one tile of RECS consecutive records of the chunk (RECS = 256 * ROUNDS). Smaller tiles put more CTAs on an SM, so
// that tiles in their load, sort and store phases overlap (the store phase is where NVLink back-pressure lands).
template <int ROUNDS>
__global__ void __launch_bounds__(kPushThreads) route_push_kernel(const __grid_constant__ PushArgs a) {
  constexpr int RECS = ROUNDS * kPushThreads;
  uint8_t* srec = push_smem;                                           // [RECS][64]
  uint32_t* loc = reinterpret_cast<uint32_t*>(push_smem + RECS * 64);  // [RECS] local index, by record
  uint16_t* perm = reinterpret_cast<uint16_t*>(loc + RECS);            // [RECS] sorted position -> record
  uint8_t* own_s = reinterpret_cast<uint8_t*>(perm + RECS);            // [RECS] owner, by sorted position
  __shared__ uint32_t wcnt[ROUNDS][kPushWarps][kMaxRanks];
  __shared__ uint32_t start[kMaxRanks + 1], excl[kMaxRanks], cnt[kMaxRanks];
  __shared__ uint32_t s_bid, s_ok;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t R = a.nranks;
  if (t == 0) { s_bid = atomicAdd(a.ticket, 1u); s_ok = 0xffffffffu; }
  __syncthreads();
  const uint32_t bid = s_bid;
  const uint32_t base = bid * RECS;
  const uint32_t nrec = a.n - base < (uint32_t)RECS ? a.n - base : (uint32_t)RECS;
  const uint8_t* src = a.rec + (uint64_t)base * 64;
  // ---- the CTA's records -> shared memory (asynchronous; the owner lookups below run meanwhile)
#pragma unroll
  for (int it = 0; it < 4 * ROUNDS; ++it) {
    const uint32_t q = it * kPushThreads + t;
    if (q < nrec * 4) cp_async16(srec + (size_t)q * 16, src + (size_t)q * 16);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  // ---- owner | local index of this thread's records (record r = round * 256 + t: lanes hold consecutive records)
  unsigned long long g[ROUNDS];
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    const uint32_t r = j * kPushThreads + t;
    g[j] = r < nrec ? *reinterpret_cast<const unsigned long long*>(src + (size_t)r * 64 + 8) : ~0ull;
  }
  uint32_t o[ROUNDS], rk[ROUNDS];
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    const uint32_t r = j * kPushThreads + t;
    o[j] = 0xffu; rk[j] = 0;
    if (r < nrec) {
      if (g[j] < a.n_global) { const uint32_t ro = __ldg(a.route_of + g[j]); o[j] = ro >> 28; loc[r] = ro & 0x0fffffffu; }
      else atomicAdd(a.status + 0, 1ull);
    }
  }
  // ---- stable rank inside the warp, per owner
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    for (uint32_t rr = 0; rr < R; ++rr) {
      const uint32_t m = __ballot_sync(0xffffffffu, o[j] == rr);
      if (o[j] == rr) rk[j] = __popc(m & ((1u << lane) - 1u));
      if (lane == 0) wcnt[j][warp][rr] = __popc(m);
    }
  }
  __syncthreads();
  // ---- exclusive scan over (round, warp) per owner
  if (t < (int)R) {
    uint32_t run = 0;
#pragma unroll
    for (int j = 0; j < ROUNDS; ++j)
#pragma unroll
      for (int w = 0; w < kPushWarps; ++w) { const uint32_t c = wcnt[j][w][t]; wcnt[j][w][t] = run; run += c; }
    cnt[t] = run;
  }
  __syncthreads();
  if (t == 0) {
    uint32_t s = 0;
    for (uint32_t rr = 0; rr < R; ++rr) { start[rr] = s; s += cnt[rr]; }
    start[R] = s;
  }
  // ---- decoupled look-back: this CTA's offset inside each owner's region of the chunk. One warp per owner; the 32 lanes
  //      examine a window of 32 predecessors at once (cells are [owner][cta], a window is one coalesced read).
  for (uint32_t rr = warp; rr < R; rr += kPushWarps) {
    const uint32_t local = cnt[rr];
    const uint32_t ex = look_back(a.lb + (size_t)rr * a.n_ctas, bid, local, lane, a.status);
    if (lane == 0) {
      excl[rr] = ex;
      if ((unsigned long long)ex + local > a.cap_region) {   // would overflow the region: nothing of this CTA goes to that owner
        atomicAnd(&s_ok, ~(1u << rr));
        atomicAdd(a.status + 1, (unsigned long long)local);
      }
      if (base + nrec >= a.n) a.totals[rr] = ex + local;     // the chunk's last CTA: its inclusive prefix is the chunk total
    }
  }
  __syncthreads();
  // ---- sorted position of every record
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    if (o[j] != 0xffu) {
      const uint32_t p = start[o[j]] + wcnt[j][warp][o[j]] + rk[j];
      perm[p] = (uint16_t)(j * kPushThreads + t);
      own_s[p] = (uint8_t)o[j];
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
  const uint32_t nvalid = start[R];
  const uint32_t ok = s_ok;
  if (a.out_bytes == 64u) {
    // ---- every owner's run, contiguous: thread -> (sorted position, 16-byte piece)
#pragma unroll 4
    for (int it = 0; it < 4 * ROUNDS; ++it) {
      const uint32_t q = it * kPushThreads + t;
      const uint32_t p = q >> 2, k = q & 3u;
      if (p < nvalid) {
        const uint32_t r = perm[p], ow = own_s[p];
        if ((ok >> ow) & 1u) {
          uint4 v = *reinterpret_cast<const uint4*>(srec + (size_t)r * 64 + k * 16);
          if (k == 0) { v.z = loc[r]; v.w = base + r; }   // agg := the owner's LOCAL aggregate index | index within the chunk
          st_na_v4(a.dst[ow] + (size_t)(excl[ow] + p - start[ow]) * 64 + k * 16, v);
        }
      }
    }
  } else {
    // ---- projection: u32 local index, then the program's slot words (slot 0 = event type)
    const uint32_t ow4 = a.out_bytes >> 2;
#pragma unroll
    for (int j = 0; j < ROUNDS; ++j) {
      const uint32_t p = j * kPushThreads + t;
      if (p < nvalid) {
        const uint32_t r = perm[p], ow = own_s[p];
        if ((ok >> ow) & 1u) {
          const uint32_t* rw = reinterpret_cast<const uint32_t*>(srec + (size_t)r * 64);
          uint32_t out[8];
          out[0] = loc[r];
          { const uint32_t ty = rw[a.proj_word[0]]; out[1] = ((ty < 16u ? ty : 16u) << kIdxBits) | (base + r); }
#pragma unroll
          for (uint32_t k = 1; k < 7; ++k) out[1 + k] = k < a.n_proj ? rw[a.proj_word[k]] : 0u;
          uint8_t* dp = a.dst[ow] + (size_t)(excl[ow] + p - start[ow]) * a.out_bytes;
          st_na_v4(dp, make_uint4(out[0], out[1], out[2], out[3]));
          if (ow4 > 4) st_na_v4(dp + 16, make_uint4(out[4], out[5], out[6], out[7]));
        }
      }
    }
  }
}

// The same partition WITHOUT staging the records in shared memory: every thread keeps ITS records in registers.
//   load    4 x LDG.128 per record, all issued up front (each 32-byte sector as two adjacent halves)
//   place   owner | local index from the record's aggregate index, stable rank by ballots, per-owner counts, look-back
//   store   4 x STG.128 per record at its position in the owner's region (agg rewritten to the owner's local index)
// One read of every byte, one write, 3 barriers, a few hundred bytes of shared memory: eight CTAs per SM, and the DRAM latency
// of the records overlaps the latency chain of the placement (route lookup -> counts -> look-back). Consecutive records of one
// owner land on consecutive positions, so L2 merges the 64-byte writes into full lines. This is the kernel of the PULL mode,
// where every region is in this rank's own HBM; contiguous per-owner runs (route_push_kernel) only pay for stores over NVLink.
// 32 bytes as two 16-byte accesses: 128 bits is the widest global load / store sm_90 has
__device__ __forceinline__ void ldg256(const void* p, uint4& a, uint4& b) {
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p));
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(static_cast<const uint8_t*>(p) + 16));
}
__device__ __forceinline__ void stg256(void* p, const uint4& a, const uint4& b) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w) : "memory");
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(static_cast<uint8_t*>(p) + 16), "r"(b.x), "r"(b.y), "r"(b.z), "r"(b.w) : "memory");
}
__device__ __forceinline__ uint32_t word_of(const uint4& a, const uint4& b, const uint4& c, const uint4& d, uint32_t w) {
  // value selects only: taking a reference to one of the four would push the records to local memory
  const uint32_t x = (w & 8u) ? ((w & 4u) ? d.x : c.x) : ((w & 4u) ? b.x : a.x);
  const uint32_t y = (w & 8u) ? ((w & 4u) ? d.y : c.y) : ((w & 4u) ? b.y : a.y);
  const uint32_t z = (w & 8u) ? ((w & 4u) ? d.z : c.z) : ((w & 4u) ? b.z : a.z);
  const uint32_t v = (w & 8u) ? ((w & 4u) ? d.w : c.w) : ((w & 4u) ? b.w : a.w);
  return (w & 2u) ? ((w & 1u) ? v : z) : ((w & 1u) ? y : x);
}

template <int ROUNDS>
__global__ void __launch_bounds__(kPushThreads) route_part_kernel(const __grid_constant__ PushArgs a) {
  constexpr int RECS = ROUNDS * kPushThreads;
  __shared__ uint32_t wcnt[ROUNDS][kPushWarps][kMaxRanks];
  __shared__ uint32_t excl[kMaxRanks], cnt[kMaxRanks];
  __shared__ uint32_t s_bid, s_ok;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const uint32_t R = a.nranks;
  uint32_t bid = blockIdx.x;
  if (t == 0) s_ok = 0xffffffffu;
  if (a.ordered) {   // the look-back needs every earlier tile to be running already: tiles are taken in ticket order
    if (t == 0) s_bid = atomicAdd(a.ticket, 1u);
    __syncthreads();
    bid = s_bid;
  }
  const uint32_t base = bid * RECS;
  const uint32_t nrec = a.n - base < (uint32_t)RECS ? a.n - base : (uint32_t)RECS;
  const uint8_t* src = a.rec + (uint64_t)base * 64;
  const bool full = a.out_bytes == 64u;
  bool second = full;   // the second half of the record is needed for a full copy, or when the projection reaches into it
  for (uint32_t k = 0; k < a.n_proj; ++k) second |= a.proj_word[k] >= 8u;
  uint4 d0[ROUNDS], d1[ROUNDS], d2[ROUNDS], d3[ROUNDS];
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    const uint32_t r = j * kPushThreads + t;
    d0[j] = d1[j] = d2[j] = d3[j] = make_uint4(0, 0, 0, 0);
    if (r < nrec) {
      ldg256(src + (size_t)r * 64, d0[j], d1[j]);
      if (second) ldg256(src + (size_t)r * 64 + 32, d2[j], d3[j]);
    }
  }
  uint32_t o[ROUNDS], rk[ROUNDS], loc[ROUNDS];
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    const uint32_t r = j * kPushThreads + t;
    o[j] = 0xffu; rk[j] = 0; loc[j] = 0;
    if (r < nrec) {
      const unsigned long long g = ((unsigned long long)d0[j].w << 32) | d0[j].z;
      if (g < a.n_global) { const uint32_t ro = __ldg(a.route_of + g); o[j] = ro >> 28; loc[j] = ro & 0x0fffffffu; }
      else atomicAdd(a.status + 0, 1ull);
    }
  }
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    for (uint32_t rr = 0; rr < R; ++rr) {
      const uint32_t m = __ballot_sync(0xffffffffu, o[j] == rr);
      if (o[j] == rr) rk[j] = __popc(m & ((1u << lane) - 1u));
      if (lane == 0) wcnt[j][warp][rr] = __popc(m);
    }
  }
  __syncthreads();
  if (t < (int)R) {
    uint32_t run = 0;
#pragma unroll
    for (int j = 0; j < ROUNDS; ++j)
#pragma unroll
      for (int w = 0; w < kPushWarps; ++w) { const uint32_t c = wcnt[j][w][t]; wcnt[j][w][t] = run; run += c; }
    cnt[t] = run;
  }
  __syncthreads();
  if (a.ordered) {
    for (uint32_t rr = warp; rr < R; rr += kPushWarps) {
      const uint32_t local = cnt[rr];
      const uint32_t ex = look_back(a.lb + (size_t)rr * a.n_ctas, bid, local, lane, a.status);
      if (lane == 0) {
        excl[rr] = ex;
        if ((unsigned long long)ex + local > a.cap_region) {   // would overflow the region: nothing of this CTA goes to that owner
          atomicAnd(&s_ok, ~(1u << rr));
          atomicAdd(a.status + 1, (unsigned long long)local);
        }
        if (base + nrec >= a.n) a.totals[rr] = ex + local;     // the chunk's last CTA: its inclusive prefix is the chunk total
      }
    }
  } else if (t < (int)R) {
    // no CTA waits for another: the chunk totals double as allocation cursors (they end up as the totals the flag kernel sends)
    const uint32_t local = cnt[t];
    const uint32_t ex = local ? atomicAdd(a.totals + t, local) : 0u;
    excl[t] = ex;
    if ((unsigned long long)ex + local > a.cap_region) { atomicAnd(&s_ok, ~(1u << t)); atomicAdd(a.status + 1, (unsigned long long)local); }
  }
  __syncthreads();
  const uint32_t ok = s_ok;
#pragma unroll
  for (int j = 0; j < ROUNDS; ++j) {
    if (o[j] == 0xffu || !((ok >> o[j]) & 1u)) continue;
    const uint32_t pos = excl[o[j]] + wcnt[j][warp][o[j]] + rk[j];
    if (full) {
      uint8_t* dp = a.dst[o[j]] + (size_t)pos * 64;
      d0[j].z = loc[j]; d0[j].w = base + j * kPushThreads + t;   // agg := the owner's LOCAL aggregate index | index within the chunk
      stg256(dp, d0[j], d1[j]);
      stg256(dp + 32, d2[j], d3[j]);
    } else {
      uint32_t out[8];
      out[0] = loc[j];
      { const uint32_t ty = word_of(d0[j], d1[j], d2[j], d3[j], a.proj_word[0]); out[1] = ((ty < 16u ? ty : 16u) << kIdxBits) | (base + j * kPushThreads + t); }
#pragma unroll
      for (uint32_t k = 1; k < 7; ++k) out[1 + k] = k < a.n_proj ? word_of(d0[j], d1[j], d2[j], d3[j], a.proj_word[k]) : 0u;
      uint8_t* dp = a.dst[o[j]] + (size_t)pos * a.out_bytes;
      if (a.out_bytes == 16u) *reinterpret_cast<uint4*>(dp) = make_uint4(out[0], out[1], out[2], out[3]);
      else stg256(dp, make_uint4(out[0], out[1], out[2], out[3]), make_uint4(out[4], out[5], out[6], out[7]));
    }
  }
}

template <int ROUNDS>
constexpr size_t push_smem_bytes() { return (size_t)ROUNDS * kPushThreads * (64 + 4 + 2 + 1); }

struct FlagArgs {
  unsigned long long* peer_flag[kMaxRanks];   // &header(owner).flags[me][chunk]
  const uint32_t* totals;
  const unsigned long long* status;
  uint32_t nranks, epoch;
};
// after the chunk's push kernel (stream order): every store of the chunk is performed, publish the counts
__global__ void push_flag_kernel(const __grid_constant__ FlagArgs f) {
  const uint32_t lane = threadIdx.x;
  if (lane < f.nranks) {
    const bool bad = f.status[1] != 0 || f.status[2] != 0;
    const unsigned long long v = ((unsigned long long)f.epoch << 32) | (bad ? 0xffffffffull : (unsigned long long)(f.totals[lane] + 1u));
    __threadfence_system();
    st_release_sys(f.peer_flag[lane], v);
  }
}
// receiver: region (s, chunk) of every source is complete (or a source reported an error)
__global__ void push_wait_kernel(const unsigned long long* flags, uint32_t chunk, uint32_t nranks, uint32_t epoch, unsigned long long* status) {
  const uint32_t lane = threadIdx.x;
  if (lane < nranks) {
    const unsigned long long* p = flags + (size_t)lane * kMaxChunks + chunk;
    unsigned long long spins = 0;
    for (;;) {
      const unsigned long long v = ld_acquire_sys(p);
      if ((uint32_t)(v >> 32) == epoch) { if ((uint32_t)v == 0xffffffffu) atomicAdd(status + 3, 1ull); break; }
      if (++spins > kSpinLimit) { atomicAdd(status + 2, 1ull); break; }
      __nanosleep(100);
    }
  }
}

// replay support: region -> contiguous 64-byte records (compact records are expanded: the program reads nothing else)
__global__ void gather_region_kernel(const uint8_t* __restrict__ src, uint32_t n, uint32_t in_bytes, uint8_t* __restrict__ dst,
                                     uint32_t n_proj, const uint32_t* __restrict__ proj_word) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint4* d4 = reinterpret_cast<uint4*>(dst + i * 64);
  if (in_bytes == 64u) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src + i * 64);
    for (int k = 0; k < 4; ++k) d4[k] = s4[k];
    reinterpret_cast<uint32_t*>(d4)[3] = 0u;   // the upper half of the agg field carried the index within the chunk
    return;
  }
  uint32_t w[16];
  for (int k = 0; k < 16; ++k) w[k] = 0;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(src + i * in_bytes);
  for (uint32_t k = 0; k < n_proj; ++k) {
    const uint32_t pw = proj_word[k];
    const uint32_t val = k == 0 ? s[1] >> kIdxBits : s[1 + k];   // word 1 = type << 27 | index within the chunk
    for (int q = 0; q < 16; ++q) if ((uint32_t)q == pw) w[q] = val;
  }
  w[2] = s[0]; w[3] = 0;
  for (int k = 0; k < 4; ++k) d4[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
}

}  // namespace

// every allocation the push path makes for logs of up to n records, up front: a cudaMalloc inside the call can wait for a
// peer's spinning wait kernel when several ranks share one device (loopback)
PushTuning& push_tuning() { static PushTuning t; return t; }

static int tile_recs() { const int t = push_tuning().tile; return t == 256 || t == 1024 ? t : 512; }
// chunks are whole multiples of 1024 records (the largest tile), so the chunk boundaries do not depend on the tile size
// (surge_b200/dist.py chunk_records is the Python twin)
static uint64_t chunk_records(uint64_t n, uint32_t n_chunks) {
  const uint64_t c = (n + n_chunks - 1) / n_chunks;
  return (c + 1023) / 1024 * 1024;
}

// One arrival-flag word, (epoch << 32) | count + 1: false when it is not this epoch's or the source failed (count 0xffffffff).
static bool arrived_count(unsigned long long v, uint32_t epoch, uint32_t* count) {
  if ((uint32_t)(v >> 32) != epoch || (uint32_t)v == 0xffffffffu) return false;
  *count = (uint32_t)v - 1u;
  return true;
}

// CUDA loads a kernel lazily at its first launch, and that load can wait for the kernels already running on the device — such as
// another loopback rank's spinning wait kernel, which in turn waits for THIS rank's flags. Touch every kernel of the path once.
static cudaError_t preload_kernels() {
  cudaFuncAttributes fa;
  cudaError_t e;
#define SGR_TOUCH(k) if ((e = cudaFuncGetAttributes(&fa, k)) != cudaSuccess) return e;
  SGR_TOUCH(route_push_kernel<1>) SGR_TOUCH(route_push_kernel<2>) SGR_TOUCH(route_push_kernel<4>)
  SGR_TOUCH(route_part_kernel<1>) SGR_TOUCH(route_part_kernel<2>) SGR_TOUCH(route_part_kernel<4>)
  SGR_TOUCH(push_flag_kernel) SGR_TOUCH(push_wait_kernel) SGR_TOUCH(gather_region_kernel)
#undef SGR_TOUCH
  return bulk_preload_kernels();
}

int dist_push_reserve(DistState* d, uint64_t n, uint32_t n_chunks, std::string* err) {
  if (n_chunks < 1 || n_chunks > (uint32_t)kMaxChunks) { *err = "push_chunks out of range"; return SGR_ERR_INVALID; }
  { cudaError_t pe = preload_kernels(); if (pe != cudaSuccess) { *err = std::string("kernel preload: ") + cudaGetErrorString(pe); return SGR_ERR_CUDA; } }
  const uint64_t chunk_recs = chunk_records(n, n_chunks);
  const uint64_t ctas_per_chunk = chunk_recs / 256;   // sized for the smallest tile
  cudaError_t ce;
  if (!d->h_pinned && (ce = cudaHostAlloc(&d->h_pinned, 128 + (size_t)kMaxRanks * kMaxChunks * 8 + 256, cudaHostAllocDefault)) != cudaSuccess) {
    *err = std::string("page-locked read-back buffer: ") + cudaGetErrorString(ce);
    return SGR_ERR_OOM;
  }
  if ((ce = d->push_ctl.reserve((size_t)kMaxChunks * 4 + (size_t)kMaxChunks * kMaxRanks * 4 + 64 + 64)) != cudaSuccess ||
      (ce = d->lb.reserve((size_t)n_chunks * ctas_per_chunk * kMaxRanks * 8 + 256)) != cudaSuccess ||
      (ce = d->counts_all.reserve((size_t)kMaxRanks * kMaxRanks * 8 + 64)) != cudaSuccess ||
      (ce = cudaFuncSetAttribute(route_push_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)push_smem_bytes<1>())) != cudaSuccess ||
      (ce = cudaFuncSetAttribute(route_push_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)push_smem_bytes<2>())) != cudaSuccess ||
      (ce = cudaFuncSetAttribute(route_push_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)push_smem_bytes<4>())) != cudaSuccess) {
    *err = std::string("push buffers: ") + cudaGetErrorString(ce);
    return ce == cudaErrorMemoryAllocation ? SGR_ERR_OOM : SGR_ERR_CUDA;
  }
  return SGR_OK;
}

int dist_push_fold(DistState* d, const uint8_t* d_records, uint64_t n, const PushFoldArgs& pf, cudaStream_t st, PushFoldResult* out,
                   std::string* err) {
  cudaError_t ce;
  const int R = d->nranks;
  if (!d->n_global) { *err = "no partition table: call sgr_dist_set_partitions first"; return SGR_ERR_NOT_LOADED; }
  if (R > 1 && !d->peers_mapped) { *err = "the push path needs the peers' receive buffers (sgr_dist_ipc_import / sgr_dist_set_peers)"; return SGR_ERR_NOT_LOADED; }
  if (d->n_global > (1ull << 28)) { *err = "push path: at most 2^28 global aggregates"; return SGR_ERR_UNSUPPORTED; }
  const uint32_t C = pf.n_chunks;
  if (C < 1 || C > (uint32_t)kMaxChunks) { *err = "push_chunks out of range"; return SGR_ERR_INVALID; }
  const uint64_t cap_region = d->recv_capacity / ((uint64_t)R * C);
  if (!cap_region) { *err = "receive buffer too small for R x chunks regions"; return SGR_ERR_CAPACITY; }
  if (n >= (1ull << 30)) { *err = "push path: at most 2^30 records per rank per call"; return SGR_ERR_UNSUPPORTED; }
  // chunk size: whole CTAs, the same number of chunks on every rank (the flags are indexed by chunk)
  const uint64_t chunk_recs = chunk_records(n, C);
  const int tile = tile_recs();
  const uint64_t idx_stride = ((1ull << 30) - 2) / C;   // the same on every rank: arrival index = chunk * idx_stride + index within the chunk < 2^30
  if (chunk_recs >= (1ull << kIdxBits) || chunk_recs > idx_stride) { *err = "push path: chunk too large, raise push_chunks"; return SGR_ERR_UNSUPPORTED; }
  const uint32_t out_bytes = pf.compact ? ((1 + pf.prog->n_slots) * 4 <= 16 ? 16u : 32u) : 64u;
  if (pf.compact && pf.prog->n_slots > 7) { *err = "compact exchange: program reads more than 7 record words"; return SGR_ERR_UNSUPPORTED; }
  const uint64_t ctas_per_chunk = chunk_recs / tile;
  // control block: tickets[C] | totals[C][kMaxRanks] | status[8] u64 | proj words
  const size_t off_tot = (size_t)kMaxChunks * 4, off_status = off_tot + (size_t)kMaxChunks * kMaxRanks * 4, off_proj = off_status + 64;
  { int rr = dist_push_reserve(d, n, C, err); if (rr) return rr; }
  uint32_t* tickets = (uint32_t*)d->push_ctl.p;
  uint32_t* totals = (uint32_t*)((uint8_t*)d->push_ctl.p + off_tot);
  unsigned long long* status = (unsigned long long*)((uint8_t*)d->push_ctl.p + off_status);
  const bool pull = push_tuning().pull != 0;
  const uint32_t epoch = ++d->epoch;
  // st: the engine's stream (brackets the call); sp: partition + flag kernels, HIGH priority; s1: wait + fold kernels, LOW
  // priority with one tile per CTA — the fold fills whatever the partition leaves free and takes the whole GPU once it is done
  cudaStream_t s0 = st, sp = d->stream_hi, s1 = d->stream2;
  DTRY(cudaMemsetAsync(d->push_ctl.p, 0, off_proj + 64, s0));
  DTRY(cudaMemsetAsync(d->lb.p, 0, (size_t)C * ctas_per_chunk * kMaxRanks * 8, s0));
  DTRY(cudaMemsetAsync(pf.counters, 0, 64, s0));
  // everybody has finished the previous call (its folds read the regions this call overwrites)
  if (R > 1 && !d->loopback) NTRY(nccl_api().AllGather((uint8_t*)d->push_ctl.p + off_proj, d->counts_all.p, 1, ncclUint32, d->comm, s0));
  DTRY(cudaEventRecord(d->pev[0], s0));
  DTRY(cudaStreamWaitEvent(s1, d->pev[0], 0));
  DTRY(cudaStreamWaitEvent(sp, d->pev[0], 0));
  unsigned long long* my_flags = (unsigned long long*)d->peer_base[d->rank];
  // region (source s, owner q, chunk c): push, the source stores it into the owner's buffer at [s][c]; pull, the source keeps
  // it in its own buffer at [q][c] and the owner's fold reads it over NVLink
  auto region = [&](int s, int q, uint32_t c) -> uint8_t* {
    return pull ? d->peer_recv[s] + ((uint64_t)q * C + c) * cap_region * out_bytes
                : d->peer_recv[q] + ((uint64_t)s * C + c) * cap_region * out_bytes;
  };
  // receiver side of chunk c: wait for the flags of every source, then the sort-free accumulate over the chunk's regions
  auto fold_chunk = [&](uint32_t c) -> cudaError_t {
    push_wait_kernel<<<1, 32, 0, s1>>>(my_flags, c, (uint32_t)R, epoch, status);
    BulkSrc bs{};
    bs.n_regions = (uint32_t)R; bs.compact = pf.compact ? 1u : 0u; bs.rec_bytes = out_bytes; bs.rotate = (uint32_t)d->rank; bs.carried = 1;
    bs.blocks_per_sm = push_tuning().fold_blocks_per_sm > 0 ? (uint32_t)push_tuning().fold_blocks_per_sm : 0xffffffffu;
    for (int s = 0; s < R; ++s) {
      bs.base[s] = region(s, d->rank, c);
      bs.count_flag[s] = my_flags + (size_t)s * kMaxChunks + c;
      bs.count[s] = cap_region;
      // + the index the record carries within ITS SOURCE's chunk c. The sources cut their logs into chunks of different lengths
      // (each from its own record count), so the base must not depend on any rank's chunk length: a fixed stride that bounds
      // them all keeps the arrival index monotone along every aggregate's log
      bs.idx_base[s] = (uint32_t)((uint64_t)c * idx_stride);
    }
    return launch_bulk_accumulate(bs, pf.n_slots, pf.scratch, *pf.prog, *pf.lay, pf.counters, pf.num_sms, s1);
  };
  for (uint32_t c = 0; c < C; ++c) {
    const uint64_t begin = (uint64_t)c * chunk_recs;
    const uint64_t cn = begin >= n ? 0 : (n - begin < chunk_recs ? n - begin : chunk_recs);
    if (cn) {
      PushArgs a{};
      a.rec = d_records + begin * 64; a.n = (uint32_t)cn; a.nranks = (uint32_t)R; a.n_global = d->n_global;
      a.route_of = (const uint32_t*)d->route_of.p;
      for (int q = 0; q < R; ++q) a.dst[q] = region(d->rank, q, c);
      a.cap_region = (uint32_t)cap_region; a.out_bytes = out_bytes;
      a.lb = (unsigned long long*)d->lb.p + (size_t)c * ctas_per_chunk * kMaxRanks; a.n_ctas = (uint32_t)ctas_per_chunk;
      a.ticket = tickets + c; a.totals = totals + (size_t)c * kMaxRanks; a.status = status;
      a.ordered = pf.ordered ? 1u : 0u;
      if (pf.compact) { a.n_proj = pf.prog->n_slots; for (uint32_t k = 0; k < a.n_proj; ++k) a.proj_word[k] = pf.prog->slot_word[k]; }
      const uint32_t grid = (uint32_t)((cn + tile - 1) / tile);
      // contiguous per-owner runs only pay across NVLink; the staged kernel is always ordered
      const bool staged = pf.ordered && (push_tuning().staged >= 0 ? push_tuning().staged != 0 : !pull);
      if (staged) {
        if (tile == 256) route_push_kernel<1><<<grid, kPushThreads, push_smem_bytes<1>(), sp>>>(a);
        else if (tile == 512) route_push_kernel<2><<<grid, kPushThreads, push_smem_bytes<2>(), sp>>>(a);
        else route_push_kernel<4><<<grid, kPushThreads, push_smem_bytes<4>(), sp>>>(a);
      } else {
        if (tile == 256) route_part_kernel<1><<<grid, kPushThreads, 0, sp>>>(a);
        else if (tile == 512) route_part_kernel<2><<<grid, kPushThreads, 0, sp>>>(a);
        else route_part_kernel<4><<<grid, kPushThreads, 0, sp>>>(a);
      }
    }
    FlagArgs f{};
    for (int q = 0; q < R; ++q) f.peer_flag[q] = (unsigned long long*)d->peer_base[q] + (size_t)d->rank * kMaxChunks + c;
    f.totals = totals + (size_t)c * kMaxRanks; f.status = status; f.nranks = (uint32_t)R; f.epoch = epoch;
    push_flag_kernel<<<1, 32, 0, sp>>>(f);
    if (!d->group) DTRY(fold_chunk(c));
  }
  if (d->group) {   // loopback ranks: every rank's partition and flag kernels are queued before any rank queues a wait
    DTRY(cudaGetLastError());
    if (!d->group->arrive_and_wait(60)) { *err = "time-out waiting for the other loopback ranks to enter the exchange"; return SGR_ERR_DIST; }
    for (uint32_t c = 0; c < C; ++c) DTRY(fold_chunk(c));
  }
  DTRY(cudaGetLastError());
  DTRY(cudaEventRecord(d->pev[1], sp));    // all partition kernels done and flagged
  DTRY(cudaStreamWaitEvent(s0, d->pev[1], 0));
  DTRY(launch_bulk_finish(pf.n_slots, pf.scratch, pf.states, pf.err_ids, *pf.lay, pf.counters, s1));
  DTRY(cudaEventRecord(d->pev[2], s1));
  DTRY(cudaStreamWaitEvent(s0, d->pev[2], 0));
  DTRY(cudaEventRecord(d->pev[3], s0));
  // ---- results
  // page-locked landing area: a copy into pageable memory blocks inside the driver, which stalls the launches of the other
  // ranks of a loopback job (one process, one context) and with them the flags this rank is waiting for
  unsigned long long* h_status = (unsigned long long*)d->h_pinned;
  unsigned long long* h_cnt = h_status + 8;
  unsigned long long* h_flags = h_status + 16;
  DTRY(cudaMemcpyAsync(h_status, status, 64, cudaMemcpyDeviceToHost, s0));
  DTRY(cudaMemcpyAsync(h_cnt, pf.counters, 64, cudaMemcpyDeviceToHost, s0));
  DTRY(cudaMemcpyAsync(h_flags, my_flags, (size_t)kMaxRanks * kMaxChunks * 8, cudaMemcpyDeviceToHost, s0));
  DTRY(cudaStreamSynchronize(s0));
  float ms_push = 0, ms_total = 0;
  cudaEventElapsedTime(&ms_push, d->pev[0], d->pev[1]);
  cudaEventElapsedTime(&ms_total, d->pev[0], d->pev[3]);
  // what arrived, and what stayed local: region (me, *)
  uint64_t n_recv = 0, kept = 0; bool remote_err = false;
  out->regions.clear();
  for (int s = 0; s < R; ++s)
    for (uint32_t c = 0; c < C; ++c) {
      uint32_t cnt;
      if (!arrived_count(h_flags[(size_t)s * kMaxChunks + c], epoch, &cnt)) { remote_err = true; continue; }
      n_recv += cnt;
      if (s == d->rank) kept += cnt;
      out->regions.push_back({region(s, d->rank, c), cnt});
    }
  int my_err = SGR_OK;
  if (h_status[0]) { *err = std::to_string(h_status[0]) + " records carry a global aggregate index >= n_global"; my_err = SGR_ERR_INVALID; }
  else if (h_status[2]) { *err = "time-out waiting for a peer / an earlier CTA (push path)"; my_err = SGR_ERR_DIST; }
  else if (h_status[1]) { *err = std::to_string(h_status[1]) + " records did not fit their receive region (capacity " + std::to_string(cap_region) + " records per source and chunk)"; my_err = SGR_ERR_CAPACITY; }
  else if (remote_err || h_status[3]) { *err = "a source rank reported a full receive region"; my_err = SGR_ERR_CAPACITY; }
  else if (h_cnt[4]) { *err = std::to_string(h_cnt[4]) + " arrived records carry a local index out of range"; my_err = SGR_ERR_INVALID; }
  // every rank fails or nobody does: gather the verdicts (the fold of a failed call is discarded by the caller), and whether
  // ANY rank saw a throwing slot (then every rank repeats the call in ordered mode, see engine.cu)
  out->any_err_slots = h_cnt[3] != 0;
  if (R > 1 && !d->loopback) {
    uint32_t* all = (uint32_t*)((uint8_t*)d->h_pinned + 128 + (size_t)kMaxRanks * kMaxChunks * 8);
    uint32_t* mine = all + 2 * kMaxRanks;   // behind the gathered verdicts
    mine[0] = my_err ? 1u : 0u; mine[1] = h_cnt[3] ? 1u : 0u;
    DTRY(cudaMemcpyAsync((uint8_t*)d->push_ctl.p + off_proj, mine, 8, cudaMemcpyHostToDevice, s0));
    NTRY(nccl_api().AllGather((uint8_t*)d->push_ctl.p + off_proj, d->counts_all.p, 2, ncclUint32, d->comm, s0));
    DTRY(cudaMemcpyAsync(all, d->counts_all.p, (size_t)R * 8, cudaMemcpyDeviceToHost, s0));
    DTRY(cudaStreamSynchronize(s0));
    for (int q = 0; q < R; ++q) {
      if (!my_err && all[2 * q]) { *err = "rank " + std::to_string(q) + " failed the exchange"; my_err = SGR_ERR_DIST; }
      if (all[2 * q + 1]) out->any_err_slots = true;
    }
  }
  out->n_recv = n_recv; out->n_err_slots = h_cnt[3]; out->ms_push = ms_push; out->ms_total = ms_total; out->out_bytes = out_bytes;
  d->stats = DistStats{};
  d->stats.n_sent = n; d->stats.n_recv = n_recv;
  d->stats.ms_scatter = ms_push; d->stats.ms_exchange = 0;
  d->stats.n_sent_remote = n >= kept ? n - kept : 0;
  return my_err;
}

// contiguous 64-byte copy of everything that arrived, regions in (source, chunk) order: an aggregate's events keep their order
int dist_gather_regions(DistState* d, const PushFoldResult& res, const RowProgram& prog, cudaStream_t st, const uint8_t** out, std::string* err) {
  cudaError_t ce = d->gather_buf.reserve(res.n_recv * 64 + 256);
  if (ce != cudaSuccess) { *err = std::string("gather buffer: ") + cudaGetErrorString(ce); return SGR_ERR_OOM; }
  uint32_t* d_proj = nullptr;
  if (res.out_bytes != 64u) {
    d_proj = (uint32_t*)((uint8_t*)d->gather_buf.p + res.n_recv * 64);
    if ((ce = cudaMemcpyAsync(d_proj, prog.slot_word, 7 * 4, cudaMemcpyHostToDevice, st)) != cudaSuccess) { *err = cudaGetErrorString(ce); return SGR_ERR_CUDA; }
  }
  uint64_t off = 0;
  for (const auto& rg : res.regions) {
    if (!rg.count) continue;
    gather_region_kernel<<<(rg.count + 255) / 256, 256, 0, st>>>(rg.base, rg.count, res.out_bytes, (uint8_t*)d->gather_buf.p + off * 64, prog.n_slots, d_proj);
    off += rg.count;
  }
  if ((ce = cudaGetLastError()) != cudaSuccess) { *err = cudaGetErrorString(ce); return SGR_ERR_CUDA; }
  *out = (const uint8_t*)d->gather_buf.p;
  return SGR_OK;
}

}  // namespace sgr
