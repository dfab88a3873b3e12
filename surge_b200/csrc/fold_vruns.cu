// fold_vruns.cu — K2/K3 for VARIABLE records with a record directory (configs[3]: Zipf keys, 32-512 B payloads).
//
// Same contract and the same transformer algebra as fold_runs.cu; what changes is how records are found.
// A variable-length log cannot be cut in the middle without knowing where records start, so the packer emits a
// record directory next to the CSR: u64 rec_offsets[n_rec+1]. With it the log splits into record-balanced spans,
// one per warp — a hot aggregate (11 % of all events on the top Zipf key) is spread over thousands of warps
// instead of serialising one lane (SURVEY.md hard part #2, kernel K3).
//
//   * a step is 32 consecutive records = one contiguous byte range [rec_off[j], rec_off[j+32]) of at most
//     32 * max_record_bytes; it is staged into shared memory with coalesced 16-byte cp.async copies, NSTAGE deep —
//     every payload byte is read from HBM exactly once, whether or not the fold program looks at it;
//   * lane i parses record j+i from smem (header + the program's needed words), validates its length against the
//     directory, and turns it into a transformer;
//   * segment heads: a record whose header aggregate index differs from its predecessor's. At every head the CSR is
//     cross-checked (rec_off[j] == seg_offsets[agg], previous segment ends there); any disagreement raises a flag
//     and the engine re-runs the whole fold on the sequential kernel, so the CSR stays the source of truth;
//   * 5-step segmented warp-shuffle scan in log order; the head lane finishes the segment ending before it;
//     spans are joined by the same decoupled look-back as fold_runs.cu; throwing / malformed segments are queued
//     for exact sequential replay.
#include <stdio.h>

#include "../../include/sgr.h"
#include "fold_rows.cuh"

namespace sgr {
namespace {

constexpr int W = 2;

struct Xv {
  uint32_t m, ex, cnt;  // cnt: records composed (for the event statistics of replayed segments)
  uint32_t v[W];
};
__device__ __forceinline__ Xv xv_identity() { Xv r; r.m = 0; r.ex = 0; r.cnt = 0; r.v[0] = 0; r.v[1] = 0; return r; }
__device__ __forceinline__ Xv xv_compose(const Xv& a, const Xv& b) {  // a first, then b
  Xv r;
  r.m = a.m | b.m; r.ex = b.ex ? b.ex : a.ex; r.cnt = a.cnt + b.cnt;
#pragma unroll
  for (int w = 0; w < W; ++w) r.v[w] = (b.m & (2u << (2 * w))) ? b.v[w] : a.v[w] + b.v[w];
  return r;
}
__device__ __forceinline__ Xv xv_shfl(const Xv& t, int src) {
  Xv r;
  r.m = __shfl_sync(0xffffffffu, t.m, src); r.ex = __shfl_sync(0xffffffffu, t.ex, src); r.cnt = __shfl_sync(0xffffffffu, t.cnt, src);
  r.v[0] = __shfl_sync(0xffffffffu, t.v[0], src); r.v[1] = __shfl_sync(0xffffffffu, t.v[1], src);
  return r;
}

// full rebuild only: prior state is None (the table is zeroed before the launch, empty aggregates stay None)
__device__ __forceinline__ void finish_var(const VarArgs& a, uint32_t seg, const Xv& ts) {
  if (ts.m & M_ERR) {
    const unsigned long long pos = atomicAdd(a.counters + 3, 1ull);
    if (pos < a.redo_cap) a.redo_ids[pos] = seg;
    atomicAdd(a.counters + 4, (unsigned long long)ts.cnt);  // all of its records are taken back; the replay re-adds the applied ones
    return;
  }
  if (!ts.ex) return;
  const uint32_t exn = (ts.ex == EX_NONE) ? 0u : SGR_ST_EXISTS;
  // old state is zero: SET v -> v, ADD v -> 0 + v
  finish_row16(reinterpret_cast<uint4*>(a.states_out + (uint64_t)seg * 16), make_uint4(0, 0, 0, 0), 0u, ts.v[0], ts.v[1], exn);
}

template <int NSTAGE>
__global__ void __launch_bounds__(512) fold_vruns_kernel(const __grid_constant__ VarArgs a, const __grid_constant__ RowProgram pg) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ __align__(16) uint32_t tab[16 * kTabStride];
  for (int i = threadIdx.x; i < 16 * kTabStride; i += blockDim.x) tab[i] = pg.tab[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;
  const uint32_t stage_bytes = a.stage_bytes;
  const uint32_t stage0 = smem_u32(smem_raw) + (uint32_t)warp * NSTAGE * stage_bytes;

  const uint64_t gw = (uint64_t)blockIdx.x * wpc + warp, n_warps = (uint64_t)gridDim.x * wpc;
  const uint64_t n_rec = a.n_rec;
  const uint64_t total_steps = (n_rec + 31) / 32;
  const uint64_t spw = (total_steps + n_warps - 1) / n_warps;
  const uint64_t step0 = gw * spw;
  const uint64_t step_end = step0 + spw < total_steps ? step0 + spw : total_steps;
  const bool has_span = step0 < step_end;
  const bool owns_end = has_span && step_end == total_steps;

  bool span_has_head = false, inh_pending = false;
  uint32_t inh_seg = 0;
  Xv inh_t = xv_identity(), carry = xv_identity();
  uint32_t carry_agg = 0xffffffffu;  // aggregate of the record before the current step (0xffffffff: none)
  if (has_span && step0 > 0) carry_agg = *reinterpret_cast<const uint32_t*>(a.events + a.rec_offsets[step0 * 32 - 1] + 12);

  // directory window of a step: lane l holds rec_off[j0+l] and rec_off[j0+l+1]
  auto load_dir = [&](uint64_t s, uint64_t* lo, uint64_t* hi) {
    const uint64_t j = s * 32 + lane;
    *lo = j <= n_rec ? a.rec_offsets[j] : a.rec_offsets[n_rec];
    *hi = j + 1 <= n_rec ? a.rec_offsets[j + 1] : a.rec_offsets[n_rec];
  };
  auto issue_step = [&](uint64_t s, int stage) {
    // the byte range of the step, known from the directory entries of lane 0 and of the last lane
    const uint64_t j0 = s * 32, j1 = j0 + 32 < n_rec ? j0 + 32 : n_rec;
    const uint64_t rb = a.rec_offsets[j0], re = a.rec_offsets[j1];
    const uint32_t bytes = (uint32_t)(re - rb) <= stage_bytes ? (uint32_t)(re - rb) : stage_bytes;  // longer: flagged when parsed
    const uint32_t dst = stage0 + (uint32_t)stage * stage_bytes;
    const uint8_t* src = a.events + rb;
    for (uint32_t o = (uint32_t)lane * 16; o < bytes; o += 512) cp_async16(dst + o, src + o);
  };
  if (has_span) {
#pragma unroll
    for (int s = 0; s < NSTAGE - 1; ++s) { if (step0 + s < step_end) issue_step(step0 + s, s); cp_async_commit(); }
  }
  uint64_t d_lo = 0, d_hi = 0;
  if (has_span) load_dir(step0, &d_lo, &d_hi);

  int stage = 0;
  for (uint64_t step = step0; step < step_end; ++step) {
    {
      const uint64_t ahead = step + (NSTAGE - 1);
      int st = stage + (NSTAGE - 1); if (st >= NSTAGE) st -= NSTAGE;
      if (ahead < step_end) issue_step(ahead, st);
      cp_async_commit();
    }
    const uint64_t lo = d_lo, hi = d_hi;
    if (step + 1 < step_end) load_dir(step + 1, &d_lo, &d_hi);  // next step's directory, one step ahead
    const uint64_t j = step * 32 + lane;
    const bool valid = j < n_rec;
    const uint64_t rb = __shfl_sync(0xffffffffu, lo, 0);
    cp_async_wait<NSTAGE - 1>();
    __syncwarp();

    // ---- parse record `lane` -> transformer
    Xv t = xv_identity();
    uint32_t agg = 0xffffffffu;
    if (valid) {
      const uint32_t off = (uint32_t)(lo - rb), len = (uint32_t)(hi - lo);
      t.cnt = 1;
      bool ok = len >= 16 && (len & 15u) == 0;
      // the stage is sized for the AVERAGE step (32 records of mean length); a record of an unusually long step that
      // did not fit is parsed straight from HBM instead (rare: the sum of 32 lengths concentrates around its mean)
      const bool in_stage = off + len <= stage_bytes;
      const uint32_t base = stage0 + (uint32_t)stage * stage_bytes + off;
      const uint8_t* grec = a.events + lo;
      uint4 hdr = make_uint4(0xffffffffu, 0, 0, 0xffffffffu);
      if (len >= 16) hdr = in_stage ? lds128(base) : *reinterpret_cast<const uint4*>(grec);
      agg = hdr.w;
      const uint32_t rec_bytes = 16 + hdr.z;
      ok = ok && hdr.z <= 0x10000u && ((rec_bytes + 15u) & ~15u) == len;          // directory and header agree on the length
      ok = ok && rec_bytes <= a.max_record_bytes;                                  // longer than the format allows: malformed
      uint32_t fl = 0;
      if (ok && hdr.x < 16u) fl = tab[hdr.x * kTabStride];
      if (!(fl & kRuleValid)) ok = false;
      if (ok) {
        uint32_t mode[W], val[W];
#pragma unroll
        for (int w = 0; w < W; ++w) {
          const uint32_t spec = tab[hdr.x * kTabStride + 1 + w];
          mode[w] = spec_mode(spec);
          uint32_t v = 0;
          if (spec_slot(spec)) {
            const uint32_t wo = pg.slot_word[spec_slot(spec)] * 4;
            if (wo + 4 > rec_bytes) ok = false;                                          // the event class needs a word the record does not have
            else v = in_stage ? lds32(base + wo) : *reinterpret_cast<const uint32_t*>(grec + wo);
          }
          if (spec_neg(spec)) v = 0u - v;
          val[w] = mode[w] ? v : 0u;
        }
        if (ok) {
          t.ex = rule_ex(fl);
          t.m = mode[0] | (mode[1] << 2);
          t.v[0] = val[0]; t.v[1] = val[1];
        }
      }
      if (!ok) t.m = M_ERR;  // throws, or is malformed: exact replay by the sequential kernel
    }
    // ---- heads: the aggregate index changes
    uint32_t prev_agg = __shfl_up_sync(0xffffffffu, agg, 1);
    if (lane == 0) prev_agg = carry_agg;
    const bool head = valid && agg != prev_agg;
    const uint32_t heads = __ballot_sync(0xffffffffu, head);
    if (head) {
      // the CSR is the source of truth: the directory/header view must agree with it at every segment boundary
      bool bad = agg >= a.n_seg || (prev_agg != 0xffffffffu && agg < prev_agg);
      if (!bad) bad = a.seg_offsets[agg] != lo || (prev_agg != 0xffffffffu && a.seg_offsets[(uint64_t)prev_agg + 1] != lo);
      if (bad) atomicAdd(a.counters + 7, 1ull);
    }
    // ---- segmented inclusive scan in record order
    Xv sc = t;
    if (lane == 0 && !head) sc = xv_compose(carry, sc);
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const Xv o = xv_shfl(sc, lane - dd);
      const int sh = lane >= dd ? lane - dd + 1 : 0;
      const uint32_t window = (heads >> sh) & ((1u << dd) - 1u);
      if (lane >= dd && window == 0) sc = xv_compose(o, sc);
    }
    Xv cin = xv_shfl(sc, lane - 1);
    if (lane == 0) cin = carry;
    // ---- a head finishes the segment that ended just before it
    if (head && prev_agg != 0xffffffffu) {
      const bool is_span_first = !span_has_head && (heads & ((1u << lane) - 1u)) == 0;
      if (is_span_first && gw != 0) { inh_t = cin; inh_seg = prev_agg; inh_pending = true; }
      else finish_var(a, prev_agg, cin);
    }
    if (heads) {
      if (!span_has_head) {
        const int src = __ffs(heads) - 1;
        inh_t = xv_shfl(inh_t, src);
        inh_seg = __shfl_sync(0xffffffffu, inh_seg, src);
        inh_pending = __shfl_sync(0xffffffffu, (int)inh_pending, src) != 0;
      }
      span_has_head = true;
    }
    const int last = (int)((n_rec - step * 32 < 32 ? n_rec - step * 32 : 32) - 1);
    carry = xv_shfl(sc, last);
    carry_agg = __shfl_sync(0xffffffffu, agg, last);
    __syncwarp();
    if (++stage == NSTAGE) stage = 0;
  }
  cp_async_wait<0>();

  bool end_needs_lookback = false;
  if (owns_end) {
    // the log must end where the CSR says the last non-empty segment ends
    if (lane == 0 && carry_agg != 0xffffffffu && (carry_agg >= a.n_seg || a.seg_offsets[(uint64_t)carry_agg + 1] != a.rec_offsets[n_rec])) atomicAdd(a.counters + 7, 1ull);
    if (span_has_head || gw == 0) { if (lane == 0 && carry_agg != 0xffffffffu && carry_agg < a.n_seg) finish_var(a, carry_agg, carry); }
    else end_needs_lookback = true;
  }
  if (has_span) {
    uint32_t* pd = a.part_data + gw * 8;
    if (lane == 0) {
      pd[0] = carry.m; pd[1] = carry.v[0]; pd[2] = carry.v[1]; pd[3] = carry.ex | (span_has_head ? 4u : 0u); pd[4] = carry.cnt;
      __threadfence();
      st_volatile_u32(a.part_flags + gw, a.epoch);
    }
    if (lane == 0 && (inh_pending || end_needs_lookback)) {
      Xv pre = xv_identity();
      uint64_t p = gw;
      while (p > 0) {
        --p;
        while (ld_volatile_u32(a.part_flags + p) != a.epoch) { __nanosleep(64); }
        __threadfence();
        const uint32_t* q = a.part_data + p * 8;
        Xv e;
        e.m = ld_volatile_u32(q); e.v[0] = ld_volatile_u32(q + 1); e.v[1] = ld_volatile_u32(q + 2);
        const uint32_t tw = ld_volatile_u32(q + 3);
        e.ex = tw & 3u; e.cnt = ld_volatile_u32(q + 4);
        pre = xv_compose(e, pre);
        if (tw & 4u) break;
      }
      if (inh_pending) finish_var(a, inh_seg, xv_compose(pre, inh_t));
      if (end_needs_lookback && carry_agg < a.n_seg) finish_var(a, carry_agg, xv_compose(pre, carry));
    }
  }
  if (lane == 0 && has_span) {
    const uint64_t r0 = step0 * 32, r1 = step_end * 32 < n_rec ? step_end * 32 : n_rec;
    atomicAdd(a.counters + 0, (unsigned long long)(r1 - r0));
  }
}

}  // namespace

typedef void (*VKernel)(const VarArgs, const RowProgram);
static VKernel vkernel(int nstage) { return nstage == 1 ? fold_vruns_kernel<1> : (nstage == 2 ? fold_vruns_kernel<2> : fold_vruns_kernel<3>); }

int vruns_config(int num_sms, uint32_t max_record_bytes, uint32_t stage_hint, int nstage, int* threads, size_t* smem, uint32_t* stage_bytes) {
  if (nstage < 1 || nstage > 3) nstage = 2;
  const int NSTAGE = nstage;
  uint32_t stage = ((32u * max_record_bytes) + 127u) & ~127u;   // worst case: every record of a step at the maximum
  if (stage_hint && stage_hint < stage) stage = (stage_hint + 127u) & ~127u;
  const size_t per_warp = (size_t)NSTAGE * stage;
  int warps = (int)((220u * 1024u) / per_warp);
  if (warps < 1) return 0;
  if (warps > 16) warps = 16;
  *threads = warps * 32; *smem = per_warp * warps; *stage_bytes = stage;
  cudaFuncSetAttribute(vkernel(nstage), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, vkernel(nstage), *threads, *smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * num_sms;
}

cudaError_t launch_fold_vruns(const VarArgs& args, const RowProgram& prog, int nstage, int grid, int threads, size_t smem, cudaStream_t stream) {
  vkernel(nstage)<<<grid, threads, smem, stream>>>(args, prog);
  return cudaGetLastError();
}

}  // namespace sgr
