// fold_rows.cu — K1/K3: record-parallel segmented fold of fixed 64-byte records (sm_90a).
//
// Same contract as fold_kernels.cu (events.foldLeft(state)(handleEvent) per aggregate,
// modules/command-engine/scaladsl/src/main/scala/surge/scaladsl/command/CommandModels.scala:25-28),
// different shape: instead of one lane walking one segment, every lane takes ONE record and
// the left-to-right order is restored by composing *state transformers* with warp shuffles.
//
//   event  e  ->  T_e = per state word (KEEP | ADD v | SET v) + exists-op      (exact: i32 wrap add, bit copy)
//   T_b . T_a  (a before b)   word: b SET ? b : (a.mode|b.mode, a.v + b.v)     associative, NOT commutative
//   state' = (T_n . ... . T_1)(state)                                           == the sequential fold
//
// This is exact for every program whose rules are MATERIALISE / CREATE / TOMBSTONE / THROW with
// SET / ADD_I32 / SUB_I32 ops (Counter, IntBalance, ...). Programs with IF_EXISTS rules or 64-bit
// adds take the lane-sequential kernel in fold_kernels.cu.
//
// Data movement (HBM-bound, no tensor cores, no shared-memory staging):
//   * the log is cut into byte-balanced spans, one per warp (skew-proof: a hot aggregate is
//     spread over many warps); a warp walks its span in steps of 32 records = 4 rows of 512 B;
//   * each row is ONE fully coalesced 128-bit-per-lane load (4 x 128-B lines per instruction);
//     the next step's rows are in flight while the current step is folded;
//   * lane i needs words of record i: a word of chunk c sits in lane 4*(i&7) + ((c - (i>>3)) & 3)
//     because row r is loaded with the quad rotated by r — one shuffle per needed word, no
//     bank conflicts, no smem;
//   * segment heads come from the CSR offsets (coalesced 8-byte loads, one window per step);
//     a 5-step segmented inclusive scan composes the transformers in log order; the lane that
//     holds a segment's END offset fetches the scan value at the tail record, applies it to the
//     prior state and writes the 16-byte state — consecutive segments => coalesced stores;
//   * a segment that crosses a span boundary is finished by the warp that sees its end, after a
//     decoupled look-back over the predecessors' published partial transformers.
#include "fold_rows.cuh"

#include <stdio.h>

#include "../../include/sgr.h"

namespace sgr {
namespace {

template <int W>
struct Xf {
  uint32_t m;      // bits [2w+1:2w]: mode of word w (bit0 ADD, bit1 SET; OR-composable), bit31 error
  uint32_t v[W];   // KEEP => 0
};

// later . earlier  (apply `a` first, then `b`)
template <int W>
__device__ __forceinline__ Xf<W> compose(const Xf<W>& a, const Xf<W>& b) {
  Xf<W> r;
  r.m = a.m | b.m;
#pragma unroll
  for (int w = 0; w < W; ++w) r.v[w] = (b.m & (2u << (2 * w))) ? b.v[w] : a.v[w] + b.v[w];
  return r;
}

template <int W>
__device__ __forceinline__ Xf<W> shfl_xf(const Xf<W>& t, int src) {
  Xf<W> r;
  r.m = __shfl_sync(0xffffffffu, t.m, src);
#pragma unroll
  for (int w = 0; w < W; ++w) r.v[w] = __shfl_sync(0xffffffffu, t.v[w], src);
  return r;
}

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

// select one of four registers by a 2-bit lane-dependent index (3 SEL)
__device__ __forceinline__ uint32_t sel4(uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, int i) {
  const uint32_t lo = (i & 1) ? a1 : a0, hi = (i & 1) ? a3 : a2;
  return (i & 2) ? hi : lo;
}

// Finish one segment: apply the composed transformer to the prior state and write the state struct.
template <int W>
__device__ __forceinline__ void finish_segment(const RowArgs& a, uint64_t seg, bool nonempty, const Xf<W>& ts, uint32_t tex) {
  const uint64_t slot = a.seg_ids ? (uint64_t)a.seg_ids[seg] : seg;
  uint32_t old[W], ex0 = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) old[w] = 0;
  if (a.states_in) {
    const uint4* sp = reinterpret_cast<const uint4*>(a.states_in + slot * (uint64_t)(W + 2) * 4);
    uint32_t raw[W + 2];
#pragma unroll
    for (int q = 0; q < (W + 2) / 4; ++q) { const uint4 v4 = __ldg(sp + q); raw[4 * q] = v4.x; raw[4 * q + 1] = v4.y; raw[4 * q + 2] = v4.z; raw[4 * q + 3] = v4.w; }
    ex0 = raw[W] & SGR_ST_EXISTS;
#pragma unroll
    for (int w = 0; w < W; ++w) old[w] = ex0 ? raw[w] : 0u;
  }
  uint32_t nw[W], exn = ex0;
#pragma unroll
  for (int w = 0; w < W; ++w) nw[w] = old[w];
  if (nonempty) {
    exn = (tex == EX_NONE) ? 0u : SGR_ST_EXISTS;
#pragma unroll
    for (int w = 0; w < W; ++w) nw[w] = (ts.m & (2u << (2 * w))) ? ts.v[w] : old[w] + ts.v[w];
  }
  finish_row<W>(a.states_out + slot * (uint64_t)(W + 2) * 4, old, ex0, nw, exn);
}

template <int W, int NS>
__global__ void __launch_bounds__(kRowThreads, 3) fold_rows_kernel(const __grid_constant__ RowArgs a, const __grid_constant__ RowProgram pg) {
  // per type, one uint4-aligned entry of RowProgram::tab
  __shared__ __align__(16) uint32_t tab[16 * kTabStride];
  for (int i = threadIdx.x; i < 16 * kTabStride; i += kRowThreads) tab[i] = pg.tab[i];
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const uint64_t gw = (uint64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);  // global warp id
  const uint64_t n_warps = (uint64_t)gridDim.x * (kRowThreads / 32);
  const uint64_t n_seg = a.n_seg;
  const uint64_t base = a.log_begin;
  const uint64_t total_bytes = a.log_end - base;
  const uint64_t total_steps = (total_bytes + 2047) / 2048;
  if (total_steps == 0) {  // every segment is empty: no warp has a span, so the grid writes each state (prior or None) itself
    Xf<W> none; none.m = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) none.v[w] = 0;
    for (uint64_t s = (uint64_t)blockIdx.x * kRowThreads + threadIdx.x; s < n_seg; s += (uint64_t)gridDim.x * kRowThreads)
      finish_segment<W>(a, s, false, none, 0u);
    return;
  }
  const uint64_t spw = (total_steps + n_warps - 1) / n_warps;  // steps per warp
  uint64_t step = gw * spw;
  const uint64_t step_end = step + spw < total_steps ? step + spw : total_steps;
  const bool has_span = step < step_end;
  const uint64_t wb = base + step * 2048;

  // ---- first boundary of the span: kc = first k in [1, n_seg] with off[k] > wb (32-ary search);
  //      warp 0 starts at k = 1 so that leading empty segments are written too.
  uint64_t kc = 1;
  if (has_span && gw != 0) {
    uint64_t lo = 1, hi = n_seg + 1;  // answer in [lo, hi]; hi == n_seg+1 means "no such boundary"
    while (lo < hi) {
      const uint64_t chunk = (hi - lo + 31) / 32;
      const uint64_t p = lo + (uint64_t)lane * chunk;  // probes lo, lo+chunk, ...
      const bool valid = p < hi;
      const bool gt = !valid || a.seg_offsets[p] > wb;  // monotone in lane
      const uint32_t bal = __ballot_sync(0xffffffffu, gt);
      if (bal == 0) { lo = lo + 31 * chunk + 1; continue; }
      const int f = __ffs(bal) - 1;
      if (f == 0) { hi = lo; break; }
      const uint64_t pf = lo + (uint64_t)f * chunk;
      lo = lo + (uint64_t)(f - 1) * chunk + 1;
      hi = pf < hi ? pf : hi;
    }
    kc = lo;
  }
  // offset of the last boundary already consumed (== start of the segment open at the span start)
  uint64_t prev_last = has_span ? a.seg_offsets[kc - 1] : 0;
  bool head_pending = has_span && (gw == 0 || prev_last == wb);  // the span starts on a segment head
  bool span_has_head = head_pending;

  // pending finalisation of the inherited first segment (uniform across the warp)
  bool inh_pending = false;
  uint64_t inh_seg = 0, inh_len = 0;
  Xf<W> inh_t; inh_t.m = 0;
  uint32_t inh_ex = 0;
  Xf<W> carry; carry.m = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) { inh_t.v[w] = 0; carry.v[w] = 0; }
  uint32_t carry_ex = 0;
  unsigned long long n_applied = 0;

  // ---- row loads: row r of a step is 512 B; lane l reads chunk ((l&3)+r)&3 of quad l>>2
  uint32_t ro[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) ro[r] = (uint32_t)r * 512u + (uint32_t)(((lane & 3) + r) & 3) * 16u;
  const uint32_t quad_off = (uint32_t)(lane >> 2) * 64u;
  const uint8_t* lane_base = a.events + base + quad_off;
  uint4 cur[4], nxt[4];
  auto load_step = [&](uint64_t s, uint4* dst) {
    const uint8_t* p = lane_base + s * 2048;
    if ((s + 1) * 2048 <= total_bytes) {  // uniform: whole step inside the log
#pragma unroll
      for (int r = 0; r < 4; ++r) dst[r] = ldg_stream(reinterpret_cast<const uint4*>(p + ro[r]));
    } else {
#pragma unroll
      for (int r = 0; r < 4; ++r)
        dst[r] = (s * 2048 + (uint64_t)r * 512 + quad_off < total_bytes) ? ldg_stream(reinterpret_cast<const uint4*>(p + ro[r]))
                                                                        : make_uint4(0xffffffffu, 0, 0, 0);
    }
  };
  if (has_span) load_step(step, nxt);

  // lane i fetches chunk c of record i from lane 4*(i&7) + ((c - (i>>3)) & 3); that lane holds chunk c in row (c - (l&3)) & 3
  const int src_quad = (lane & 7) << 2, my_row = lane >> 3, lane3 = lane & 3;

  for (; step < step_end; ++step) {
#pragma unroll
    for (int r = 0; r < 4; ++r) cur[r] = nxt[r];
    if (step + 1 < step_end) load_step(step + 1, nxt);

    const uint64_t sb = base + step * 2048;
    const uint64_t rem = a.log_end - sb;
    const uint32_t span = rem < 2048 ? (uint32_t)rem : 2048u;  // bytes of this step
    const int nvalid = (int)(span >> 6);

    // ---- the needed words of record `lane`, in record order ---------------------------------------
    uint32_t sv[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const int c = (int)(pg.slot_word[s] >> 2), k = (int)(pg.slot_word[s] & 3);  // warp-uniform
      const int rs = (c - lane3) & 3;
      uint32_t x;
      switch (k) {  // uniform branch
        case 0: x = sel4(cur[0].x, cur[1].x, cur[2].x, cur[3].x, rs); break;
        case 1: x = sel4(cur[0].y, cur[1].y, cur[2].y, cur[3].y, rs); break;
        case 2: x = sel4(cur[0].z, cur[1].z, cur[2].z, cur[3].z, rs); break;
        default: x = sel4(cur[0].w, cur[1].w, cur[2].w, cur[3].w, rs); break;
      }
      sv[s] = __shfl_sync(0xffffffffu, x, src_quad + ((c - my_row) & 3));
    }
    // ---- event -> transformer (slot 0 is the event type) --------------------------------------------
    Xf<W> t; t.m = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) t.v[w] = 0;
    uint32_t ex = 0;
    if (lane < nvalid) {
      const uint32_t type = sv[0];
      uint4 e0 = make_uint4(0, 0, 0, 0);
      if (type < 16u) e0 = *reinterpret_cast<const uint4*>(tab + type * kTabStride);
      if (!(e0.x & kRuleValid)) {
        t.m = M_ERR;  // THROW rule or scala.MatchError: replayed exactly by the sequential kernel
      } else {
        ex = rule_ex(e0.x);
        uint32_t spec[W];
        spec[0] = e0.y;
        if (W > 1) spec[1] = e0.z;
        if (W > 2) spec[2] = e0.w;
#pragma unroll
        for (int w = 3; w < W; ++w) spec[w] = tab[type * kTabStride + 1 + w];
#pragma unroll
        for (int w = 0; w < W; ++w) {
          uint32_t val = 0;
#pragma unroll
          for (int s = 1; s < NS; ++s) val = ((int)spec_slot(spec[w]) == s) ? sv[s] : val;
          if (spec_neg(spec[w])) val = 0u - val;
          const uint32_t mode = spec_mode(spec[w]);
          t.v[w] = mode ? val : 0u;
          t.m |= mode << (2 * w);
        }
      }
    }

    // ---- segment boundaries inside (sb, sb+span], from the CSR offsets -------------------------------
    // lane j of a window holds boundary k = kb+j: segment k-1 ends there and segment k begins.
    uint32_t heads = head_pending ? 1u : 0u;
    head_pending = false;
    uint64_t kb = kc;
    uint32_t rel0 = 0xffffffffu;  // window 0, kept for the output pass
    int cnt0 = 0;
    while (true) {
      const uint64_t k = kb + lane;
      const uint64_t b = k <= n_seg ? a.seg_offsets[k] : ~0ull;
      const uint64_t d = b - sb;                        // > 0 for every unconsumed boundary
      const uint32_t rel = d <= (uint64_t)span ? (uint32_t)d : 0xffffffffu;
      const bool in = rel != 0xffffffffu;
      heads |= __reduce_or_sync(0xffffffffu, (in && rel < span) ? (1u << (rel >> 6)) : 0u);
      if (__any_sync(0xffffffffu, in && rel == span)) head_pending = true;
      const int cnt = __popc(__ballot_sync(0xffffffffu, in));
      if (kb == kc) { rel0 = rel; cnt0 = cnt; }
      kb += cnt;
      if (cnt < 32) break;
    }
    if (heads) span_has_head = true;

    // ---- carry-in, then segmented inclusive scan in record order -------------------------------------
    if (lane == 0 && !(heads & 1u)) t = compose(carry, t);
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const Xf<W> o = shfl_xf(t, lane - dd);  // wraps for lane < dd; masked below
      const int sh = lane >= dd ? lane - dd + 1 : 0;
      const uint32_t window = (heads >> sh) & ((1u << dd) - 1u);  // a head in records (lane-dd, lane]?
      if (lane >= dd && window == 0) t = compose(o, t);
    }
    carry = shfl_xf(t, nvalid - 1);
    {
      const uint32_t e_last = __shfl_sync(0xffffffffu, ex, nvalid - 1);
      carry_ex = e_last ? e_last : carry_ex;  // a throwing tail keeps the previous exists-op (segment is replayed anyway)
    }

    // ---- outputs: the lane holding boundary k finishes segment k-1 -----------------------------------
    if (cnt0 | (int)(kb != kc)) {
      uint64_t kw = kc;
      uint32_t rel = rel0;
      int cnt = cnt0;
      while (true) {
        if (kw != kc) {
          const uint64_t k = kw + lane;
          const uint64_t b = k <= n_seg ? a.seg_offsets[k] : ~0ull;
          const uint64_t d = b - sb;
          rel = d <= (uint64_t)span ? (uint32_t)d : 0xffffffffu;
          cnt = __popc(__ballot_sync(0xffffffffu, rel != 0xffffffffu));
        }
        const bool in = rel != 0xffffffffu;
        // start of segment k-1, relative to sb (negative => before this step)
        uint32_t relp = __shfl_up_sync(0xffffffffu, rel, 1);
        const int64_t prev_rel0 = (int64_t)(prev_last - sb);
        const bool prev_before = (lane == 0) && prev_rel0 < 0;
        if (lane == 0) relp = prev_before ? 0u : (uint32_t)prev_rel0;
        const bool empty = in && !prev_before && relp == rel;
        const bool mine = in && !empty;
        const int tpos = mine ? (int)((rel - 64u) >> 6) : 0;
        const Xf<W> ts = shfl_xf(t, tpos);
        const uint32_t tex = __shfl_sync(0xffffffffu, ex, tpos);
        const bool inherited = mine && prev_before && prev_last < wb;
        if (__any_sync(0xffffffffu, inherited)) {  // only lane 0 of the first window of a span can be
          inh_t = shfl_xf(ts, 0);
          inh_ex = __shfl_sync(0xffffffffu, tex, 0);
          inh_seg = kw - 1;
          inh_len = (sb + (uint64_t)__shfl_sync(0xffffffffu, rel, 0) - prev_last) >> 6;
          inh_pending = true;
        }
        if (in && !inherited) {
          const uint64_t seg = kw + lane - 1;
          if (mine && (ts.m & M_ERR)) {
            const unsigned long long pos = atomicAdd(a.counters + 3, 1ull);  // exact replay by the sequential kernel
            if (pos < a.redo_cap) a.redo_ids[pos] = (uint32_t)seg;
          } else {
            finish_segment<W>(a, seg, mine, ts, tex);
            if (mine) n_applied += prev_before ? ((sb + rel - prev_last) >> 6) : (uint64_t)((rel - relp) >> 6);
          }
        }
        if (cnt) prev_last = sb + (uint64_t)__shfl_sync(0xffffffffu, rel, cnt - 1);
        kw += cnt;
        if (cnt < 32) break;
      }
      kc = kb;
    }
  }

  // ---- publish this span's open transformer, then finish the inherited segment -----------------
  if (has_span) {
    uint32_t* part_data = a.part_data + gw * (W + 2);
    if (lane == 0) {
      part_data[0] = carry.m;
#pragma unroll
      for (int w = 0; w < W; ++w) part_data[1 + w] = carry.v[w];
      part_data[W + 1] = carry_ex | (span_has_head ? 4u : 0u);
      __threadfence();
      st_volatile_u32(a.part_flags + gw, a.epoch);
    }
    if (inh_pending && lane == 0) {
      // decoupled look-back: compose predecessors' open transformers until one that contains a head
      Xf<W> acc = inh_t;
      uint64_t p = gw;
      while (p > 0) {
        --p;
        const uint32_t* pf = a.part_flags + p;
        while (ld_volatile_u32(pf) != a.epoch) { __nanosleep(64); }
        __threadfence();
        const uint32_t* pd = a.part_data + p * (W + 2);
        Xf<W> e;
        e.m = ld_volatile_u32(pd);
#pragma unroll
        for (int w = 0; w < W; ++w) e.v[w] = ld_volatile_u32(pd + 1 + w);
        const uint32_t tailw = ld_volatile_u32(pd + W + 1);
        acc = compose(e, acc);
        if (tailw & 4u) break;
      }
      if (acc.m & M_ERR) {
        const unsigned long long pos = atomicAdd(a.counters + 3, 1ull);
        if (pos < a.redo_cap) a.redo_ids[pos] = (uint32_t)inh_seg;
      } else {
        finish_segment<W>(a, inh_seg, true, acc, inh_ex);
        n_applied += inh_len;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) n_applied += __shfl_xor_sync(0xffffffffu, n_applied, o);
  if (lane == 0 && n_applied) atomicAdd(a.counters + 0, n_applied);
}

// misaligned[0] += segments whose offset is not log_begin (mod 64) or not monotone; bounds = off[0], off[n]
__global__ void inspect_offsets_kernel(const uint64_t* __restrict__ off, uint64_t n_seg, unsigned long long* __restrict__ out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_seg) return;
  const uint64_t b0 = off[0], b = off[i];
  if (i == 0) out[1] = b0;
  if (i == n_seg) out[2] = b;
  bool bad = ((b - b0) & 63ull) != 0 || b < b0;
  if (i > 0 && off[i - 1] > b) bad = true;
  if (bad) atomicAdd(out, 1ull);
  if (i > 0 && b >= off[i - 1]) atomicMax(out + 3, (unsigned long long)(b - off[i - 1]));  // longest segment, bytes
}

}  // namespace

cudaError_t inspect_offsets(const uint64_t* d_off, uint64_t n_seg, unsigned long long* d_scratch, cudaStream_t st,
                            bool* aligned64, uint64_t* log_begin, uint64_t* log_end, uint64_t* max_seg_bytes) {
  cudaError_t e = cudaMemsetAsync(d_scratch, 0, 32, st);
  if (e != cudaSuccess) return e;
  inspect_offsets_kernel<<<(unsigned)((n_seg + 256) / 256), 256, 0, st>>>(d_off, n_seg, d_scratch);
  unsigned long long h[4];
  if ((e = cudaMemcpyAsync(h, d_scratch, 32, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
  if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
  *aligned64 = h[0] == 0;
  *log_begin = h[1];
  *log_end = h[2];
  *max_seg_bytes = h[3];
  return cudaSuccess;
}

namespace {
}  // namespace

bool build_row_program(const DevProgram& dp, RowProgram* out) {
  memset(out, 0, sizeof *out);
  if (dp.user_words != 2 && dp.user_words != 6 && dp.user_words != 14) return false;  // 16 / 32 / 64-byte states
  out->user_words = dp.user_words;
  out->n_slots = 1;
  out->slot_word[0] = 0;  // the event type
  for (uint32_t f = 0; f < dp.n_f64; ++f) out->f64_mask |= 1u << dp.f64_word[f];
  bool any_mat = false, any_ifx = false;
  for (uint32_t t = 0; t < dp.n_types; ++t) {
    any_mat |= dp.rules[t].exists_rule == SGR_MATERIALISE;
    any_ifx |= dp.rules[t].exists_rule == SGR_IF_EXISTS;
  }
  if (any_mat && any_ifx) return false;  // outside both closed classes
  out->cls = any_ifx ? 1u : 0u;
  for (uint32_t t = 0; t < dp.n_types; ++t) {
    const DevRule& r = dp.rules[t];
    uint32_t* e = out->tab + t * kTabStride;
    if (r.exists_rule == SGR_THROW) { e[0] = 0; continue; }
    uint32_t mode[kMaxRowWords] = {0}, slot[kMaxRowWords] = {0}, neg[kMaxRowWords] = {0};
    const bool reset = r.exists_rule == SGR_CREATE || r.exists_rule == SGR_TOMBSTONE;
    if (reset) for (uint32_t w = 0; w < dp.user_words; ++w) mode[w] = kModeSet;  // SET 0
    for (uint32_t i = 0; i < r.n_ops; ++i) {
      const uint32_t op = r.ops[i];
      const uint32_t opcode = op & 15u, nwords = (op >> 4) & 63u, dw = (op >> 10) & 63u, sw = op >> 16;
      if (opcode > SGR_OP_SUB_I32) return false;  // 64-bit adds carry between words: not a per-word map
      for (uint32_t j = 0; j < nwords; ++j) {
        const uint32_t w = dw + j, src = sw + j;
        if (w >= dp.user_words || src >= (dp.record_kind == SGR_REC_FIXED64 ? 16u : 136u)) return false;
        // one source per state word per event: a word written twice by the same rule is not a single (mode, value)
        if (mode[w] != 0 && !(reset && slot[w] == 0)) return false;
        uint32_t s = 0;
        for (uint32_t q = 1; q < out->n_slots; ++q) if (out->slot_word[q] == src) s = q;
        if (!s) {
          if (out->n_slots >= (uint32_t)kMaxSlots) return false;
          s = out->n_slots++;
          out->slot_word[s] = src;
        }
        slot[w] = s;
        neg[w] = opcode == SGR_OP_SUB_I32;
        mode[w] = (opcode == SGR_OP_SET || reset) ? kModeSet : kModeAdd;  // over a reset state ADD v == SET v and SUB v == SET -v
      }
    }
    e[0] = kRuleValid | (r.exists_rule == SGR_TOMBSTONE ? kRuleNone : 0u) | (r.exists_rule == SGR_IF_EXISTS ? kRuleIfExists : 0u) |
           ((r.exists_rule == SGR_CREATE || r.n_ops > 0) ? kRuleNew : 0u);
    for (uint32_t w = 0; w < dp.user_words; ++w) e[1 + w] = spec_encode(mode[w], neg[w], slot[w]);
  }
  // slot 0 is the type word; the fold, its look-back and its replay read no record word but the slots
  out->head_only = 1;
  for (uint32_t q = 0; q < out->n_slots; ++q) if (out->slot_word[q] >= 8) out->head_only = 0;
  return true;
}

WordModes word_modes(const RowProgram& prog) {
  WordModes m{0u, 0u, false};
  for (int t = 0; t < 16; ++t) {
    const uint32_t fl = prog.tab[t * kTabStride];
    if (!(fl & kRuleValid)) continue;
    if (fl & kRuleNone) m.none = true;
    for (int w = 0; w < 2; ++w) {
      const uint32_t mode = spec_mode(prog.tab[t * kTabStride + 1 + w]);
      if (mode == kModeAdd) m.add |= 1u << w;
      if (mode == kModeSet) m.set |= 1u << w;
    }
  }
  return m;
}

namespace {
constexpr int kV1Slots = 6;
typedef void (*RowKernel)(const RowArgs, const RowProgram);
RowKernel pick_kernel(const RowProgram& prog) {
  if (prog.user_words != 2 || prog.cls != 0 || prog.n_slots > (uint32_t)kV1Slots) return nullptr;
  if (prog.n_slots <= 2) return fold_rows_kernel<2, 2>;
  if (prog.n_slots <= 3) return fold_rows_kernel<2, 3>;
  if (prog.n_slots <= 4) return fold_rows_kernel<2, 4>;
  return fold_rows_kernel<2, kV1Slots>;
}
}  // namespace

int row_kernel_max_grid(int num_sms, const RowProgram& prog) {
  int per_sm = 0;
  RowKernel k = pick_kernel(prog);
  if (!k || cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kRowThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * num_sms;
}

cudaError_t launch_fold_rows(const RowArgs& args, const RowProgram& prog, int grid, cudaStream_t stream) {
  RowKernel k = pick_kernel(prog);
  if (!k) return cudaErrorInvalidValue;
  k<<<grid, kRowThreads, 0, stream>>>(args, prog);
  return cudaGetLastError();
}

}  // namespace sgr
