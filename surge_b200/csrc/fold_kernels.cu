// fold_kernels.cu — K1/K2: CSR segmented left fold of packed event records (sm_90a).
//
// Replaces, for every aggregate at once, the per-actor
//   events.foldLeft(state)((stateAccum, evt) => handleEvent(stateAccum, evt))
// of the reference (modules/command-engine/scaladsl/src/main/scala/surge/scaladsl/command/
// CommandModels.scala:25-28) plus the actor's error/publish rules
// (modules/command-engine/core/src/main/scala/surge/internal/persistence/PersistentActor.scala:245-264).
//
// Shape of the kernel (HBM-bound byte parse + segmented scan; no tensor cores):
//   * persistent grid, one CTA per SM; every LANE owns one aggregate's segment at a time and
//     folds it strictly left to right — exact for arbitrary (non-commutative) handlers;
//   * each lane stages its own segment into shared memory with 1-D TMA bulk copies
//     (cp.async.bulk, CH bytes per copy, 16-byte aligned by the format) into a per-lane ring
//     of NST chunks; completion is counted in bytes on one mbarrier per (warp, stage);
//     no register staging, NST-1-LAG chunks per lane in flight while one is folded;
//   * lane rings are skewed by 16 bytes so that the 128-bit header reads of 32 lanes walking
//     equal-length segments hit 8 distinct bank groups per quarter-warp (conflict free);
//   * the lane's state lives in shared memory, transposed ([word][thread]) — conflict free,
//     dynamically indexable by the op table; flags/err_idx live in registers;
//   * segments are dealt to lanes round-robin (lane l of warp w takes segment base+l), so
//     neighbouring lanes read neighbouring segments and write neighbouring 16-byte states.
#include "fold_kernels.cuh"

#include <stdio.h>

#include "../../include/sgr.h"

namespace sgr {

namespace {

constexpr uint32_t DESC_LAST = 0x80000000u;
constexpr uint32_t DESC_BYTES = 0x3fffffffu;

template <int THREADS, int CH, int NST, int LAG, int KIND>
struct Cfg {
  static constexpr int kThreads = THREADS;
  static constexpr int kChunk = CH;
  static constexpr int kStages = NST;
  static constexpr int kLag = LAG;
  static constexpr int kKind = KIND;
  static constexpr int kRing = CH * NST;         // ring bytes per lane
  static constexpr int kLaneStride = CH * NST + 16;  // 16-byte skew per lane
  static constexpr int kWarps = THREADS / 32;
  static_assert(CH % 64 == 0 && THREADS % 32 == 0 && NST > LAG + 1, "bad fold config");
};

template <class C>
__host__ __device__ constexpr size_t smem_bytes(uint32_t user_words) {
  return (size_t)C::kThreads * C::kLaneStride      // rings
         + (((size_t)C::kWarps * C::kStages * 8 + 15) & ~(size_t)15)  // mbarriers
         + sizeof(DevProgram)                      // program copy
         + (size_t)C::kThreads * C::kStages * 4    // chunk descriptors
         + (size_t)2 * user_words * C::kThreads * 4;  // state + initial state, transposed
}

template <class C>
__global__ void __launch_bounds__(C::kThreads, 1)
fold_stream_kernel(const __grid_constant__ FoldArgs a, const __grid_constant__ DevProgram prog_in) {
  constexpr int THREADS = C::kThreads, CH = C::kChunk, NST = C::kStages, LAG = C::kLag, KIND = C::kKind;
  constexpr int RB = C::kRing;
  extern __shared__ __align__(128) uint8_t smem[];

  const int tid = threadIdx.x;
  const int warp = tid >> 5;

  uint8_t* p = smem;
  const uint32_t ring = smem_u32(p) + (uint32_t)tid * C::kLaneStride;
  p += (size_t)THREADS * C::kLaneStride;
  const uint32_t bars = smem_u32(p) + (uint32_t)warp * NST * 8;
  uint64_t* bar_ptr = reinterpret_cast<uint64_t*>(p);
  p += ((size_t)C::kWarps * NST * 8 + 15) & ~(size_t)15;
  DevProgram* prog = reinterpret_cast<DevProgram*>(p);
  p += sizeof(DevProgram);
  uint32_t* desc = reinterpret_cast<uint32_t*>(p) + tid;  // desc[s * THREADS]
  p += (size_t)THREADS * NST * 4;
  uint32_t* st = reinterpret_cast<uint32_t*>(p) + tid;  // st[w * THREADS]: working state
  const uint32_t user_words = prog_in.user_words;
  uint32_t* st0 = st + (size_t)user_words * THREADS;    // st0[w * THREADS]: state before the batch

  // ---- one-time setup: program into smem, mbarriers
  {
    const uint4* src = reinterpret_cast<const uint4*>(&prog_in);
    uint4* dst = reinterpret_cast<uint4*>(prog);
    for (int i = tid; i < (int)(sizeof(DevProgram) / 16); i += THREADS) dst[i] = src[i];
    if (tid < C::kWarps * NST) mbar_init(smem_u32(bar_ptr + tid), 32);
    fence_mbar_init();
    fence_proxy_async();
    __syncthreads();
  }

  const uint64_t policy = l2_policy_evict_first();
  const uint32_t state_words = prog->state_words;
  const uint32_t n_types = prog->n_types;
  uint64_t n_seg = a.n_seg;
  if (a.n_seg_dev) { const unsigned long long d = *a.n_seg_dev; n_seg = d < n_seg ? d : n_seg; }
  const uint64_t stride = (uint64_t)gridDim.x * THREADS;
  const uint64_t first = (uint64_t)blockIdx.x * THREADS + tid;

  // ---- producer cursor (the lane's TMA side)
  uint64_t p_seg = first, p_pos = 0, p_end = 0, nxt_b = 0, nxt_e = 0;
  bool p_has = p_seg < n_seg;
  auto seg_of = [&](uint64_t i) -> uint64_t { return a.seg_list ? (uint64_t)a.seg_list[i] : i; };
  if (p_has) {
    const uint64_t sg = seg_of(p_seg);
    p_pos = a.seg_offsets[sg];
    p_end = a.seg_offsets[sg + 1];
    if (p_seg + stride < n_seg) {
      const uint64_t sn = seg_of(p_seg + stride);
      nxt_b = a.seg_offsets[sn];
      nxt_e = a.seg_offsets[sn + 1];
    }
  }

  auto produce = [&](int s) {
    const uint32_t bar = bars + s * 8;
    uint32_t d = 0;
    if (p_has) {
      const uint64_t rem = p_end - p_pos;
      const uint32_t bytes = rem < (uint64_t)CH ? (uint32_t)rem : (uint32_t)CH;
      if (bytes) {
        mbar_arrive_expect_tx(bar, bytes);
        bulk_g2s(ring + s * CH, a.events + p_pos, bytes, bar, policy);
      } else {
        mbar_arrive(bar);
      }
      p_pos += bytes;
      d |= bytes;
      if (p_pos == p_end) {
        d |= DESC_LAST;
        p_seg += stride;
        p_has = p_seg < n_seg;
        p_pos = nxt_b;
        p_end = nxt_e;
        if (p_seg + stride < n_seg) {
          const uint64_t sn = seg_of(p_seg + stride);
          nxt_b = a.seg_offsets[sn];
          nxt_e = a.seg_offsets[sn + 1];
        }
      }
    } else {
      mbar_arrive(bar);
    }
    desc[s * THREADS] = d;
  };

  // ---- consumer state (the lane's fold side)
  uint64_t c_seg = first;
  bool c_has = c_seg < n_seg;
  bool c_fresh = true;
  uint32_t rp = 0, avail = 0, k = 0, exists = 0, exists0 = 0, err = 0, err_idx = 0;
  uint32_t copied = 0;  // some event of this segment produced a NEW state instance (Scala copy / constructor), see end_segment
  unsigned long long n_applied = 0, n_err = 0, n_dropped = 0;
  uint32_t c_total = 0;  // bytes of the current segment received so far

  auto zero_state = [&]() {
    for (uint32_t w = 0; w < user_words; ++w) st[w * THREADS] = 0u;
  };

  // apply one record located at ring offset rp; hdr = its first 16 bytes
  auto apply = [&](const uint4 hdr, uint32_t rec_bytes) {
    const uint32_t type = hdr.x;
    if (type >= n_types) { err = 1; err_idx = k; return; }
    const DevRule* r = &prog->rules[type];
    const uint4 r0 = *reinterpret_cast<const uint4*>(r);  // exists_rule, n_ops, min_len, pad
    if (r0.z > rec_bytes) { err = 1; err_idx = k; return; }  // record too short for this event class
    switch (r0.x) {
      case SGR_IF_EXISTS:
        if (!exists) { ++k; ++n_applied; return; }
        break;
      case SGR_MATERIALISE:
        if (!exists) { zero_state(); exists = 1; copied = 1; }
        break;
      case SGR_CREATE:
        zero_state(); exists = 1; copied = 1;
        break;
      case SGR_TOMBSTONE:
        zero_state(); exists = 0; ++k; ++n_applied; return;
      default:
        err = 1; err_idx = k; return;
    }
    if (r0.y) copied = 1;   // field ops = `current.copy(...)`; a rule without ops hands the same instance back
    for (uint32_t i = 0; i < r0.y; ++i) {
      const uint32_t op = r->ops[i];
      const uint32_t opcode = op & 15u, nwords = (op >> 4) & 63u, dw = (op >> 10) & 63u, sw = op >> 16;
      uint32_t off = rp + sw * 4;
      if (off >= (uint32_t)RB) off -= RB;
      if (opcode == SGR_OP_SET) {
        for (uint32_t w = 0; w < nwords; ++w) {
          st[(dw + w) * THREADS] = lds32(ring + off);
          off += 4; if (off >= (uint32_t)RB) off -= RB;
        }
      } else if (opcode <= SGR_OP_SUB_I32) {
        const uint32_t v = lds32(ring + off);
        const uint32_t old = st[dw * THREADS];
        st[dw * THREADS] = (opcode == SGR_OP_ADD_I32) ? old + v : old - v;
      } else {
        const uint32_t vlo = lds32(ring + off);
        uint32_t off2 = off + 4; if (off2 >= (uint32_t)RB) off2 -= RB;
        const uint32_t vhi = lds32(ring + off2);
        const unsigned long long v = ((unsigned long long)vhi << 32) | vlo;
        const unsigned long long old = ((unsigned long long)st[(dw + 1) * THREADS] << 32) | st[dw * THREADS];
        const unsigned long long nw = (opcode == SGR_OP_ADD_I64) ? old + v : old - v;
        st[dw * THREADS] = (uint32_t)nw;
        st[(dw + 1) * THREADS] = (uint32_t)(nw >> 32);
      }
    }
    ++k; ++n_applied;
  };

  auto begin_segment = [&](int s) {
    rp = (uint32_t)s * CH; avail = 0; k = 0; err = 0; err_idx = 0; exists = 0; exists0 = 0; c_total = 0; copied = 0;
    if (a.states_in) {
      const uint64_t sg = seg_of(c_seg);
      const uint64_t slot = a.seg_ids ? (uint64_t)a.seg_ids[sg] : sg;
      const uint4* src = reinterpret_cast<const uint4*>(a.states_in + slot * (uint64_t)state_words * 4);
      for (uint32_t q = 0; q < state_words / 4; ++q) {
        const uint4 v = __ldg(src + q);
        const uint32_t w = q * 4;
        if (w + 0 < user_words) st[(w + 0) * THREADS] = st0[(w + 0) * THREADS] = v.x;
        if (w + 1 < user_words) st[(w + 1) * THREADS] = st0[(w + 1) * THREADS] = v.y;
        if (w + 2 < user_words) st[(w + 2) * THREADS] = st0[(w + 2) * THREADS] = v.z; else if (w + 2 == user_words) exists0 = v.z & SGR_ST_EXISTS;
        if (w + 3 < user_words) st[(w + 3) * THREADS] = st0[(w + 3) * THREADS] = v.w;
      }
      exists = exists0;
      if (!exists0) { for (uint32_t w = 0; w < user_words; ++w) st[w * THREADS] = st0[w * THREADS] = 0u; }
    } else {
      for (uint32_t w = 0; w < user_words; ++w) st[w * THREADS] = st0[w * THREADS] = 0u;
    }
  };

  auto end_segment = [&]() {
    const uint64_t sg = seg_of(c_seg);
    const uint64_t slot = a.seg_ids ? (uint64_t)a.seg_ids[sg] : sg;
    uint4* dst = reinterpret_cast<uint4*>(a.states_out + slot * (uint64_t)state_words * 4);
    uint32_t flags;
    const uint32_t* src = st;
    if (err) {
      // .recover { case e => ACKError(e) }: the actor keeps its previous state
      flags = exists0 | SGR_ST_ERROR; src = st0; ++n_err;
      if (KIND == (int)SGR_REC_FIXED64) n_dropped += (c_total >> 6) - k;  // records of this segment that were not applied
    } else {
      // shouldPublish = state.stateOpt != context.state
      uint32_t changed = exists != exists0;
      if (exists && exists0)
        changed |= program_words_differ(*prog, user_words, [=](uint32_t w) { return st[w * THREADS]; },
                                        [=](uint32_t w) { return st0[w * THREADS]; }, copied);
      flags = exists | (changed ? SGR_ST_CHANGED : 0u);
    }
    const bool live = (flags & SGR_ST_EXISTS) != 0;
    for (uint32_t q = 0; q < state_words / 4; ++q) {
      const uint32_t w = q * 4;
      uint32_t v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t ww = w + j;
        if (ww < user_words) v[j] = live ? src[ww * THREADS] : 0u;
        else if (ww == user_words) v[j] = flags;
        else v[j] = err ? err_idx : 0u;
      }
      dst[q] = make_uint4(v[0], v[1], v[2], v[3]);
    }
  };

  auto consume = [&](int s, uint32_t parity) {
    mbar_wait(bars + s * 8, parity);
    const uint32_t d = desc[s * THREADS];
    if (!c_has) return;
    if (c_fresh) { begin_segment(s); c_fresh = false; }
    avail += d & DESC_BYTES;
    c_total += d & DESC_BYTES;
    if (err) avail = 0;  // drain: nothing more is applied once the handler threw
    while (true) {
      uint32_t rec_len, rec_bytes;
      uint4 hdr;
      if (KIND == (int)SGR_REC_FIXED64) {
        if (avail < 64) break;
        hdr = lds128(ring + rp);
        rec_len = 64; rec_bytes = 64;
      } else {
        if (avail < 16) break;
        hdr = lds128(ring + rp);
        rec_bytes = 16 + (hdr.z > 0x10000u ? 0x10000u : hdr.z);  // clamp: anything this long is rejected below
        rec_len = (rec_bytes + 15u) & ~15u;
        if (rec_bytes > a.max_record_bytes || rec_len > (uint32_t)(LAG * CH + 16)) {
          // longer than the format allows, or than the ring can hold behind the refill point: a malformed event,
          // never mis-parsed (the launch keeps max_record_bytes within the ring, the second test is a guard)
          err = 1; err_idx = k; avail = 0;
          break;
        }
        if (rec_len > avail) {
          // not all here yet; if the segment is over, the record is malformed
          if (d & DESC_LAST) { err = 1; err_idx = k; avail = 0; }
          break;
        }
      }
      apply(hdr, rec_bytes);
      if (err) { avail = 0; break; }
      rp += rec_len; if (rp >= (uint32_t)RB) rp -= RB;
      avail -= rec_len;
    }
    if (d & DESC_LAST) {
      if (avail != 0 && !err) { err = 1; err_idx = k; }  // trailing partial record
      end_segment();
      c_seg += stride;
      c_has = c_seg < n_seg;
      c_fresh = true;
    }
  };

  // ---- pipeline: prologue fills NST-LAG slots, then consume slot s / refill slot s-LAG
#pragma unroll 1
  for (int s = 0; s < NST - LAG; ++s) produce(s);

  int s = 0;
  uint32_t parity = 0;
#pragma unroll 1
  while (true) {
    consume(s, parity);
    int rs = s - LAG; if (rs < 0) rs += NST;
    // generic-proxy reads of slot rs are done; order them before the async-proxy refill
    fence_proxy_async();
    produce(rs);
    if (__all_sync(0xffffffffu, !c_has)) break;
    if (++s == NST) { s = 0; parity ^= 1u; }
  }

  // ---- stats
  for (int o = 16; o > 0; o >>= 1) {
    n_applied += __shfl_xor_sync(0xffffffffu, n_applied, o);
    n_err += __shfl_xor_sync(0xffffffffu, n_err, o);
    n_dropped += __shfl_xor_sync(0xffffffffu, n_dropped, o);
  }
  if ((tid & 31) == 0 && a.counters) {
    // replay mode (n_seg_dev set): the record-parallel kernel already counted every record as applied
    if (n_applied) atomicAdd(a.counters + (a.n_seg_dev ? 5 : 0), n_applied);
    if (n_dropped) atomicAdd(a.counters + 4, n_dropped);
    if (n_err) atomicAdd(a.counters + 1, n_err);
  }
}

// ---------------------------------------------------------------- config table
using F0 = Cfg<128, 512, 3, 0, SGR_REC_FIXED64>;
using F1 = Cfg<256, 256, 3, 0, SGR_REC_FIXED64>;
using F2 = Cfg<192, 256, 4, 0, SGR_REC_FIXED64>;
using F3 = Cfg<128, 256, 4, 0, SGR_REC_FIXED64>;
using F4 = Cfg<64, 1024, 3, 0, SGR_REC_FIXED64>;
using F5 = Cfg<256, 128, 6, 0, SGR_REC_FIXED64>;
using V0 = Cfg<96, 512, 4, 1, SGR_REC_VAR16>;
using V1 = Cfg<64, 1024, 3, 1, SGR_REC_VAR16>;
using V2 = Cfg<32, 2048, 3, 1, SGR_REC_VAR16>;

struct VariantDesc {
  const char* name;
  int kind, threads, chunk, stages, lag;
};
const VariantDesc kVariants[] = {
    {"fixed64 t128 ch512 st3", SGR_REC_FIXED64, 128, 512, 3, 0},  {"fixed64 t256 ch256 st3", SGR_REC_FIXED64, 256, 256, 3, 0},
    {"fixed64 t192 ch256 st4", SGR_REC_FIXED64, 192, 256, 4, 0},  {"fixed64 t128 ch256 st4", SGR_REC_FIXED64, 128, 256, 4, 0},
    {"fixed64 t64 ch1024 st3", SGR_REC_FIXED64, 64, 1024, 3, 0},  {"fixed64 t256 ch128 st6", SGR_REC_FIXED64, 256, 128, 6, 0},
    {"var16 t96 ch512 st4 lag1", SGR_REC_VAR16, 96, 512, 4, 1},   {"var16 t64 ch1024 st3 lag1", SGR_REC_VAR16, 64, 1024, 3, 1},
    {"var16 t32 ch2048 st3 lag1", SGR_REC_VAR16, 32, 2048, 3, 1},
};
constexpr int kNumVariants = sizeof(kVariants) / sizeof(kVariants[0]);

template <class C>
cudaError_t launch_cfg(const FoldArgs& args, const DevProgram& prog, int num_sms, cudaStream_t stream,
                       FoldLaunchInfo* info, int variant) {
  const size_t smem = smem_bytes<C>(prog.user_words);
  if (smem > 227 * 1024) return cudaErrorInvalidConfiguration;
  cudaError_t e = cudaFuncSetAttribute(fold_stream_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  uint64_t want = (args.n_seg + C::kThreads - 1) / C::kThreads;
  int grid = (int)(want < (uint64_t)num_sms ? (want ? want : 1) : (uint64_t)num_sms);
  fold_stream_kernel<C><<<grid, C::kThreads, smem, stream>>>(args, prog);
  if (info) {
    info->variant = variant; info->threads = C::kThreads; info->chunk = C::kChunk; info->stages = C::kStages;
    info->grid = grid; info->smem = smem;
  }
  return cudaGetLastError();
}

}  // namespace

int fold_variant_count() { return kNumVariants; }
const char* fold_variant_name(int v) { return (v >= 0 && v < kNumVariants) ? kVariants[v].name : "?"; }

static cudaError_t launch_variant(int variant, const FoldArgs& args, const DevProgram& prog, int num_sms, cudaStream_t stream, FoldLaunchInfo* info) {
  switch (variant) {
    case 0: return launch_cfg<F0>(args, prog, num_sms, stream, info, variant);
    case 1: return launch_cfg<F1>(args, prog, num_sms, stream, info, variant);
    case 2: return launch_cfg<F2>(args, prog, num_sms, stream, info, variant);
    case 3: return launch_cfg<F3>(args, prog, num_sms, stream, info, variant);
    case 4: return launch_cfg<F4>(args, prog, num_sms, stream, info, variant);
    case 5: return launch_cfg<F5>(args, prog, num_sms, stream, info, variant);
    case 6: return launch_cfg<V0>(args, prog, num_sms, stream, info, variant);
    case 7: return launch_cfg<V1>(args, prog, num_sms, stream, info, variant);
    case 8: return launch_cfg<V2>(args, prog, num_sms, stream, info, variant);
  }
  return cudaErrorInvalidValue;
}

cudaError_t launch_fold_stream(const FoldArgs& fold_args, const DevProgram& prog, int variant, int num_sms,
                               uint32_t max_record_bytes, cudaStream_t stream, FoldLaunchInfo* info) {
  FoldArgs args = fold_args;
  args.max_record_bytes = max_record_bytes;
  const bool explicit_variant = variant >= 0 && variant < kNumVariants && kVariants[variant].kind == (int)prog.record_kind;
  if (prog.record_kind == SGR_REC_VAR16) {
    if (!explicit_variant) variant = max_record_bytes <= 512 + 16 ? 6 : (max_record_bytes <= 1024 + 16 ? 7 : 8);
    // a variable record must fit in LAG*CH+16 bytes of ring behind the slot being refilled
    if (max_record_bytes > (uint32_t)kVariants[variant].chunk * kVariants[variant].lag + 16) return cudaErrorNotSupported;
    return launch_variant(variant, args, prog, num_sms, stream, info);
  }
  if (explicit_variant) return launch_variant(variant, args, prog, num_sms, stream, info);
  // fixed records: more warps per SM hide more of the memory latency; take the widest configuration whose rings + state
  // tables fit in shared memory
  const int order[] = {1, 2, 0, 3};
  cudaError_t e = cudaErrorInvalidConfiguration;
  for (int v : order) {
    e = launch_variant(v, args, prog, num_sms, stream, info);
    if (e != cudaErrorInvalidConfiguration) return e;
  }
  return e;
}

}  // namespace sgr
