// fold_runs.cu — K1/K3 (primary): segmented fold of fixed 64-byte records, lane-runs + warp scan (sm_90a).
//
// Contract: for every aggregate, events.foldLeft(state)(handleEvent)
// (modules/command-engine/scaladsl/src/main/scala/surge/scaladsl/command/CommandModels.scala:25-28) with the
// actor's publish rule (modules/command-engine/core/src/main/scala/surge/internal/persistence/
// PersistentActor.scala:252-257). Exactness comes from the transformer algebra of fold_rows.cuh:
// an event is a per-word (KEEP | ADD v | SET v) map, composition is associative, so any
// bracketing of the log-ordered product equals the sequential fold bit for bit.
//
// Shape (HBM-bound byte parse + segmented scan; no tensor cores):
//   * the log is cut into byte-balanced chunks, handed out to warps in log order (work order
//     below) — a hot aggregate (Zipf skew) is spread over many warps instead of serialising one lane;
//   * a warp walks a chunk in steps of 32*R records. The step's 2048*R bytes are staged into
//     shared memory with coalesced 16-byte cp.async copies (512 contiguous bytes per warp
//     instruction), NSTAGE steps deep, no register staging;
//   * the staging layout XOR-swizzles each record's 16-byte chunks with (record/R)&7, so that
//     lane i reading its run of R consecutive records [R*i, R*i+R) is bank-conflict free;
//   * lane i folds its R records left to right into a running transformer (the only per-record
//     work: 1 table read + the needed record words); segments that start and end inside the
//     run are finished on the spot;
//   * once per step the 32 lane-transformers are combined by a 5-step segmented warp-shuffle
//     scan in log order; the lane holding the first segment head of its run finishes the segment
//     that flows into it; the scan's tail is the carry into the next step;
//   * segment heads come from the CSR offsets: a window of 32 boundaries is read with coalesced
//     8-byte loads and scattered into a per-step head bitmap + segment-id table in smem;
//   * a segment that crosses a chunk boundary is finished by the warp that sees its end, after a
//     decoupled look-back over the preceding chunks' published open transformers.
//
// Work order: the log is cut into chunks of a few steps (RowArgs::chunk_steps). Warp g takes chunk g first, then further
// chunks in log order by an atomic ticket (counters[10]), the single-pass-scan pattern: a warp that finishes early takes
// more, so the fold ends when HBM runs dry rather than when the slowest of fixed spans ends. A chunk only ever waits on
// chunks handed out before it. There is no grid barrier either: a warp leaves when its last chunk is done, unless a
// segment threw, in which case the warps still there replay the list once every warp has arrived (replay_segments).
// A fold queued right behind a fold of the same log is launched with programmatic dependent launch: before
// griddepcontrol.wait it reads only the program, the log and its offsets (table load, first boundary search, first steps
// in flight), which the fold before it only reads too, so it overlaps that fold's tail; states, look-back buffers,
// counters, the replay list and the ticket come after the wait. Behind any other work (a kernel that writes the log, a
// copy) it is launched plainly and the wait is a no-op. The chunk size shrinks on small logs so that every resident warp
// gets a chunk (run_variant_chunk_steps). From the slot plane a chunk's first boundary comes from the engine's chunk table
// (RowArgs::chunk_kc) instead of the search, and the next chunk's entry and boundary window are loaded a step or two
// before the switch.
#include <stdio.h>

#include "../../include/sgr.h"
#include "fold_rows.cuh"

namespace sgr {
namespace {

constexpr int kRunThreads = 128;
constexpr int kRunWarps = kRunThreads / 32;

template <int W>
struct Xf {
  uint32_t m;     // bits [2w+1:2w]: mode of word w (bit0 ADD, bit1 SET; OR-composable), bit30 copy, bit31 error
  uint32_t ex;    // exists-op of the LAST event in the range: 0 = no event, EX_SOME, EX_NONE
  uint32_t v[W];  // KEEP => 0
};

template <int W>
__device__ __forceinline__ Xf<W> identity() {
  Xf<W> r;
  r.m = 0; r.ex = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) r.v[w] = 0;
  return r;
}
// later . earlier  (apply `a` first, then `b`)
template <int W, int CLS = 1>
__device__ __forceinline__ Xf<W> compose(const Xf<W>& a, const Xf<W>& b) {
  // class 1: b.ex == 0 means b holds only IF_EXISTS events (or nothing); they apply iff the state exists after a — a
  // tombstoned prefix absorbs them — but not a throw among them: a throwing event sets no exists-op, and the segment must
  // still be replayed. (In class 0, b.ex == 0 only for the identity or a range of throwing events, where the plain rule
  // gives a with b's error bit too.)
  Xf<W> r;
  if (CLS == 1 && b.ex == 0u && a.ex == EX_NONE) { r = a; r.m |= b.m & M_ERR; return r; }
  r.m = a.m | b.m;
  r.ex = b.ex ? b.ex : a.ex;
#pragma unroll
  for (int w = 0; w < W; ++w) r.v[w] = (b.m & (2u << (2 * w))) ? b.v[w] : a.v[w] + b.v[w];
  return r;
}
template <int W>
__device__ __forceinline__ Xf<W> shfl_xf(const Xf<W>& t, int src) {
  Xf<W> r;
  r.m = __shfl_sync(0xffffffffu, t.m, src);
  r.ex = __shfl_sync(0xffffffffu, t.ex, src);
#pragma unroll
  for (int w = 0; w < W; ++w) r.v[w] = __shfl_sync(0xffffffffu, t.v[w], src);
  return r;
}

// programmatic dependent launch: no-ops when the grid was launched without the attribute
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Finish one segment: apply the composed transformer to the prior state, write the state struct.
template <int W>
__device__ __forceinline__ void finish_segment(const RowArgs& a, uint32_t f64_mask, uint32_t seg, const Xf<W>& ts) {
  if (ts.m & M_ERR) {
    // the handler threw somewhere in the segment: exact replay by the sequential phase
    const unsigned long long pos = atomicAdd(a.counters + 3, 1ull);
    if (pos < a.redo_cap) a.redo_ids[pos] = seg;
    return;
  }
  const uint64_t slot = a.seg_ids ? (uint64_t)a.seg_ids[seg] : (uint64_t)seg;
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
  // ts.ex: SOME / NONE = exists-op of the last CREATE/MATERIALISE/TOMBSTONE-class event; 0 = only IF_EXISTS events
  // (or none at all): the words apply iff the prior state exists
  const uint32_t exn = ts.ex == EX_NONE ? 0u : (ts.ex == EX_SOME ? (uint32_t)SGR_ST_EXISTS : ex0);
  uint32_t nw[W];
#pragma unroll
  for (int w = 0; w < W; ++w) {
    nw[w] = (ts.m & (2u << (2 * w))) ? ts.v[w] : old[w] + ts.v[w];
    if (!exn) nw[w] = 0u;
  }
  uint32_t changed = exn != ex0;
  if (exn && ex0) {
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const bool f_lo = (f64_mask >> w) & 1u, f_hi = w > 0 && ((f64_mask >> (w - 1)) & 1u);
      if (f_lo) {
        // JVM Double ==: numeric (0.0 == -0.0, NaN != NaN), as Scala case-class equality does — after its `this eq that`
        // shortcut: if no applied event built a new instance the state is the old object, equal to itself even with a NaN
        const uint32_t xh = nw[w + 1 < W ? w + 1 : w], yh = old[w + 1 < W ? w + 1 : w];
        const double x = __hiloint2double((int)xh, (int)nw[w]);
        const double y = __hiloint2double((int)yh, (int)old[w]);
        changed |= !(x == y) && ((ts.m & M_COPY) != 0u || nw[w] != old[w] || xh != yh);
      } else if (!f_hi) {
        changed |= (nw[w] != old[w]);
      }
    }
  }
  uint32_t outw[W + 2];
#pragma unroll
  for (int w = 0; w < W; ++w) outw[w] = nw[w];
  outw[W] = exn | (changed ? SGR_ST_CHANGED : 0u);
  outw[W + 1] = 0u;
  uint4* dp = reinterpret_cast<uint4*>(a.states_out + slot * (uint64_t)(W + 2) * 4);
#pragma unroll
  for (int q = 0; q < (W + 2) / 4; ++q) dp[q] = make_uint4(outw[4 * q], outw[4 * q + 1], outw[4 * q + 2], outw[4 * q + 3]);
}

// state of an aggregate that received no event in this batch: unchanged, per-batch flags cleared
template <int W>
__device__ __forceinline__ void finish_empty(const RowArgs& a, uint32_t seg) {
  const uint64_t slot = a.seg_ids ? (uint64_t)a.seg_ids[seg] : (uint64_t)seg;
  uint4* dp = reinterpret_cast<uint4*>(a.states_out + slot * (uint64_t)(W + 2) * 4);
  if (a.states_in) {
    const uint4* sp = reinterpret_cast<const uint4*>(a.states_in + slot * (uint64_t)(W + 2) * 4);
#pragma unroll
    for (int q = 0; q < (W + 2) / 4; ++q) {
      uint4 v4 = __ldg(sp + q);
      if (q == (W + 2) / 4 - 1) { v4.z &= SGR_ST_EXISTS; v4.w = 0u; }
      dp[q] = v4;
    }
  } else {
#pragma unroll
    for (int q = 0; q < (W + 2) / 4; ++q) dp[q] = make_uint4(0, 0, 0, 0);
  }
}

// REC: bytes staged per record, 64 (the log itself), 32 (the head plane: each record's bytes 0..31) or 16 (the slot plane:
// the program's slot words, slot s at word s)
template <int R, int NSTAGE, int REC = 64>
__host__ __device__ constexpr int warp_smem_bytes() {
  return NSTAGE * 32 * REC * R  // staged steps
         + 2 * 32 * R * 4    // segment ids at head positions: starting segment, ending segment
         + 32 * 4;           // head bitmap (R words used) + pad
}

template <int W>
__device__ __noinline__ void replay_segments(const RowArgs& a, const RowProgram& pg, const uint32_t* tab, int lane, unsigned long long n_redo);

// The slot-plane fold publishes a chunk's open transformer as one 16-byte row of part_flags: m | ex << 4 | has_head << 6,
// v[0], v[1], epoch. One aligned 16-byte access carries the row and its flag together, so neither side needs a fence
// between them. Word 3 of a row lies where every other fold writes only epochs (a u32 flag per part), so a stale row never
// shows the current epoch.
__device__ __forceinline__ uint4 ld_volatile_v4(const uint32_t* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_volatile_v4(uint32_t* p, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
constexpr uint32_t kRowEx = 4, kRowHead = 64u, kRowFields = 0x70u;  // fields of a packed row's word 0 (m bits 4..29 are free at W = 2)

// Decoupled look-back (lane 0): compose the open transformers of the chunks before chunk c until one that contains a head.
// They were all handed out before c, to warps that are running, and a chunk publishes without waiting on anyone.
// PACKED: the rows of the slot-plane fold (above).
template <int W, int CLS, bool PACKED = false>
__device__ __forceinline__ Xf<W> look_back_chunks(const RowArgs& a, uint64_t c) {
  Xf<W> pre = identity<W>();
  while (c > 0) {
    --c;
    if constexpr (PACKED) {
      static_assert(W == 2, "a packed row holds two state words");
      uint4 r = ld_volatile_v4(a.part_flags + 4 * c);
      while (r.w != a.epoch) { __nanosleep(64); r = ld_volatile_v4(a.part_flags + 4 * c); }
      Xf<W> e;
      e.m = r.x & ~kRowFields; e.ex = (r.x >> kRowEx) & 3u; e.v[0] = r.y; e.v[1] = r.z;
      pre = compose<W, CLS>(e, pre);
      if (r.x & kRowHead) break;
      continue;
    }
    const uint32_t* pf = a.part_flags + c;
    while (ld_volatile_u32(pf) != a.epoch) { __nanosleep(64); }
    __threadfence();
    const uint32_t* pd = a.part_data + c * (W + 2);
    Xf<W> e;
    e.m = ld_volatile_u32(pd);
#pragma unroll
    for (int w = 0; w < W; ++w) e.v[w] = ld_volatile_u32(pd + 1 + w);
    const uint32_t tailw = ld_volatile_u32(pd + W + 1);
    e.ex = tailw & 3u;
    pre = compose<W, CLS>(e, pre);
    if (tailw & 4u) break;
  }
  return pre;
}

// DIRECT: programs with many source words read each state word's source straight from the staged record instead of
// pre-fetching NS slots and selecting (NS is then unused)
// REC == 32: the records are staged from the head plane (RowArgs::heads) rather than the log; offsets still count log bytes.
// REC == 16: from the slot plane (RowArgs::heads): a lane reads a whole record with one 16-byte load, its slot words in slot
// order (NS == 4: all four words are read, whatever the program's slot count).
template <int W, int R, int NSTAGE, int NS, int MINB, bool DIRECT, int CLS, int REC = 64>
__global__ void __launch_bounds__(kRunThreads, MINB) fold_runs_kernel(const __grid_constant__ RowArgs a, const __grid_constant__ RowProgram pg) {
  static_assert(R % 2 == 0 && 8 % R == 0, "R in {2,4,8}");
  static_assert(REC == 64 || REC == 32 || REC == 16, "the log, the head plane or the slot plane");
  static_assert(R * REC >= 128, "a lane's run starts on a 128-byte line: R >= 128 / REC");
  static_assert(REC != 16 || (!DIRECT && NS == 4), "the slot plane holds four slot words, not record words");
  constexpr int STEP_BYTES = 2048 * R;          // log bytes per step
  constexpr int STEP_RECS = 32 * R;
  constexpr int STAGE_BYTES = STEP_RECS * REC;  // staged bytes per step
  constexpr int RPL = 128 / REC;                // records per 128-byte shared-memory line
  constexpr int CPR = REC / 16;                 // 16-byte chunks per record
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ __align__(16) uint32_t tab[16 * kTabStride];
  // the next fold may be scheduled now: it waits for this grid to complete before it touches anything this one writes
  grid_dep_launch();
  const unsigned long long t_entry = global_ns();
  for (int i = threadIdx.x; i < 16 * kTabStride; i += kRunThreads) tab[i] = pg.tab[i];
  const uint32_t f64_mask = pg.f64_mask;
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* wsm = smem_raw + (size_t)warp * warp_smem_bytes<R, NSTAGE, REC>();
  const uint32_t stage0 = smem_u32(wsm);
  uint32_t* hs_start = reinterpret_cast<uint32_t*>(wsm + NSTAGE * STAGE_BYTES);  // segment starting at a head
  uint32_t* hs_end = hs_start + STEP_RECS;                                       // segment ending at a head (0xffffffff: none)
  uint32_t* hmask = hs_end + STEP_RECS;                                          // head bitmap, R words

  const uint64_t gw = (uint64_t)blockIdx.x * kRunWarps + warp;  // global warp id
  const uint64_t n_warps = (uint64_t)gridDim.x * kRunWarps;
  const uint64_t n_seg = a.n_seg;
  const uint64_t base = a.log_begin;
  const uint64_t total_bytes = a.log_end - base;
  const uint64_t total_steps = (total_bytes + STEP_BYTES - 1) / STEP_BYTES;
  // >= NSTAGE-1 (and >= 1): the steps staged ahead never reach past the next chunk, whose ticket is drawn when the
  // current chunk starts
  const uint64_t cs = a.chunk_steps;
  const uint64_t n_chunks = (total_steps + cs - 1) / cs;
  constexpr uint64_t kNone = ~0ull;

  // ---- first boundary at or after byte wb: the first k in [0, n_seg] with off[k] >= wb (32-ary search)
  auto first_boundary = [&](uint64_t wb) -> uint64_t {
    uint64_t lo = 0, hi = n_seg + 1;  // answer in [lo, hi]; hi == n_seg+1: no such boundary
    while (lo < hi) {
      const uint64_t part = (hi - lo + 31) / 32;
      const uint64_t p = lo + (uint64_t)lane * part;
      const bool valid = p < hi;
      const bool ge = !valid || a.seg_offsets[p] >= wb;  // monotone in lane
      const uint32_t bal = __ballot_sync(0xffffffffu, ge);
      if (bal == 0) { lo = lo + 31 * part + 1; continue; }
      const int f = __ffs(bal) - 1;
      if (f == 0) { hi = lo; break; }
      const uint64_t pf = lo + (uint64_t)f * part;
      lo = lo + (uint64_t)(f - 1) * part + 1;
      hi = pf < hi ? pf : hi;
    }
    return lo;
  };

  // ---- staging: lane l, copy q of a step moves the 16-byte chunk g = q*32 + l (source order) to its
  //      swizzled place: record j = g/CPR, chunk c = g%CPR -> line j/RPL, position (CPR*(j%RPL)+c) ^ ((j/R)&7).
  //      A 512-byte copy holds whole lines, so CPR*(j%RPL)+c == l&7 and the line is q*4 + l/8.
  constexpr int QPS = STAGE_BYTES / 512;  // copies per step
  const uint8_t* src_lane = (REC == 64 ? a.events + base : a.heads) + (uint64_t)lane * 16;
  const uint64_t total_staged = total_bytes / 64 * REC;
  const uint32_t lane_jr = (uint32_t)(lane / CPR) / R;
  uint32_t dst_q[QPS];  // smem offset (within a stage) of copy q
#pragma unroll
  for (int q = 0; q < QPS; ++q)
    dst_q[q] = (uint32_t)q * 512u + (uint32_t)(lane >> 3) * 128u + (((uint32_t)(lane & 7) ^ (((uint32_t)(q * (512 / REC)) / R + lane_jr) & 7u)) << 4);
  auto issue_step = [&](uint64_t s, int stage) {
    const uint64_t sbyte = s * (uint64_t)STAGE_BYTES;
    const uint8_t* src = src_lane + sbyte;
    const uint32_t dst = stage0 + (uint32_t)stage * STAGE_BYTES;
    if (sbyte + STAGE_BYTES <= total_staged) {  // uniform: the whole step lies inside the log
#pragma unroll
      for (int q = 0; q < QPS; ++q) cp_async16(dst + dst_q[q], src + q * 512);
    } else {
#pragma unroll
      for (int q = 0; q < QPS; ++q)
        if (sbyte + (uint64_t)q * 512 + (uint64_t)lane * 16 < total_staged) cp_async16(dst + dst_q[q], src + q * 512);
    }
  };
  // ---- issue side: steps are staged in the warp's own order, the current chunk's and then the next one's, so the pipeline
  //      runs on across chunk boundaries. iss: the next step to stage, iss_end: the end of its chunk iss_chunk.
  uint64_t chunk = gw < n_chunks ? gw : kNone;  // the chunk being folded: the first one fixed, later ones by ticket
  uint64_t iss_chunk = chunk, iss = 0, iss_end = 0;
  if (chunk != kNone) { iss = chunk * cs; iss_end = iss + cs < total_steps ? iss + cs : total_steps; }
  uint64_t nxt = kNone;             // the chunk after the current one, once the ticket is read
  bool nxt_pending = false;         // lane 0 holds a ticket not yet read
  unsigned long long tk = 0;
  auto resolve_next = [&]() {
    if (!nxt_pending) return;
    const unsigned long long t = __shfl_sync(0xffffffffu, tk, 0);
    nxt = n_warps + t < n_chunks ? n_warps + t : kNone;
    nxt_pending = false;
  };
  int ist = 0;
  auto issue_next = [&]() {
    if (iss == iss_end && iss_chunk != kNone) {
      resolve_next();
      if (nxt != kNone && nxt != iss_chunk) {
        iss_chunk = nxt; iss = nxt * cs; iss_end = iss + cs < total_steps ? iss + cs : total_steps;
      }
    }
    if (iss < iss_end) {
      issue_step(iss, ist);
      ++iss;
      if (++ist == NSTAGE) ist = 0;
    }
  };

  // ---- before the wait: the first chunk's first steps in flight, its first boundary and boundary window
#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    issue_next();
    cp_async_commit();
  }
  uint64_t kc = 0;
  if (chunk != kNone && chunk != 0) {
    if constexpr (REC == 16) kc = a.chunk_kc ? a.chunk_kc[chunk] : first_boundary(base + chunk * cs * STEP_BYTES);
    else kc = first_boundary(base + chunk * cs * STEP_BYTES);
  }

  // where lane i finds word (c,k) of the record at place rl of its line: byte (((CPR*rl + c) ^ (i&7)) << 4) + 4k of the line
  // (rl == t % RPL for the t-th record of the run: a run starts on a line). The slot plane needs no table: record rl of
  // the line is the chunk rl ^ (i&7).
  constexpr int NSOFF = DIRECT ? 1 : NS;
  constexpr int SOFF_RPL = REC == 16 ? 1 : RPL;
  uint32_t soff[SOFF_RPL][NSOFF];
  if constexpr (REC != 16) {
#pragma unroll
    for (int s = 0; s < NSOFF; ++s) {
      const uint32_t c = pg.slot_word[s] >> 2, k = pg.slot_word[s] & 3u;
#pragma unroll
      for (int rl = 0; rl < RPL; ++rl) soff[rl][s] = ((((uint32_t)(CPR * rl) + c) ^ (uint32_t)(lane & 7)) << 4) + (k << 2);
    }
  }
  // boundary window: lane j holds off[kc+j] and off[kc+j+1]; reloaded right after boundaries are consumed,
  // so the values a step needs were requested one step earlier
  uint64_t win_b = ~0ull, win_bn = ~0ull;
  auto load_window = [&]() {
    const uint64_t k = kc + lane;
    win_b = k <= n_seg ? a.seg_offsets[k] : ~0ull;
    win_bn = k < n_seg ? a.seg_offsets[k + 1] : ~0ull;
  };
  if (chunk != kNone) load_window();
  // the slot plane with a chunk table: the next chunk's first boundary (pf_kc, ~0u until loaded; n_seg < 2^32) and its
  // boundary window (pf_b, pf_bn once pf_win) are loaded while this chunk is folded, so the switch only swaps registers
  // instead of a search and a window load that no step hid
  uint32_t pf_kc = ~0u;
  uint64_t pf_b = ~0ull, pf_bn = ~0ull;
  bool pf_win = false;

  // ---- after the wait: the previous fold (and its replay) has completed; its states, counters and buffers are free
  grid_dep_wait();
  if (threadIdx.x == 0) atomicMax(a.counters + 8, ~t_entry);  // the earliest CTA entry, complemented (stats ms_fold)
  if (gw == 0 && lane < 16) a.counters_next[lane] = 0ull;    // the next fold starts from clean counters without a memset
  auto look_back = [&](uint64_t c) -> Xf<W> { return look_back_chunks<W, CLS, REC == 16>(a, c); };
  // lane 0: a chunk's first segment, begun in an earlier chunk, is finished after the warp's next chunk (or at its exit),
  // so the warp does not wait on a predecessor that is still being folded
  bool dfr = false;
  uint64_t dfr_chunk = 0;
  uint32_t dfr_seg = 0;
  Xf<W> dfr_t = identity<W>();

  unsigned long long n_applied = 0;  // records of this warp's chunks
  int stage = 0;
  uint64_t prev_chunk = kNone;
  while (chunk != kNone) {
    const uint64_t step0 = chunk * cs;
    const uint64_t step_end = step0 + cs < total_steps ? step0 + cs : total_steps;
    const uint64_t wb = base + step0 * STEP_BYTES;
    if (iss_chunk != chunk) { iss_chunk = chunk; iss = step0; iss_end = step_end; }  // one stage: nothing was staged ahead
    if (lane == 0) tk = atomicAdd(a.counters + 10, 1ull);  // the chunk after this one; read when the issue side reaches it
    nxt_pending = true;
    if (prev_chunk != kNone && chunk != prev_chunk + 1) {
      // a chunk right after the previous one starts at the boundary where that one stopped
      bool have_win = false;
      if constexpr (REC == 16) {
        if (!a.chunk_kc) kc = first_boundary(wb);
        else if (pf_win) { kc = pf_kc; win_b = pf_b; win_bn = pf_bn; have_win = true; }
        else kc = pf_kc != ~0u ? pf_kc : a.chunk_kc[chunk];
      } else {
        kc = chunk != 0 ? first_boundary(wb) : 0;
      }
      if (!have_win) load_window();
    }
    pf_kc = ~0u; pf_win = false;

    bool span_has_head = false;          // a segment head was seen in this chunk
    bool inh_pending = false;            // the segment flowing into the chunk awaits the look-back (held by lane 0)
    uint32_t inh_seg = 0;
    Xf<W> inh_t = identity<W>();
    Xf<W> carry = identity<W>();         // open transformer at the end of the previous step

    for (uint64_t step = step0; step < step_end; ++step) {
      // keep NSTAGE-1 steps in flight
      issue_next();
      cp_async_commit();
      const uint64_t sb = base + step * (uint64_t)STEP_BYTES;
      const uint64_t rem = a.log_end - sb;
      const uint32_t span = rem < (uint64_t)STEP_BYTES ? (uint32_t)rem : (uint32_t)STEP_BYTES;
      const int nvalid = (int)(span >> 6);

      // ---- segment heads of this step: boundaries k with off[k] in [sb, sb+span) ----------------------
#pragma unroll
      for (int i = 0; i < R; ++i) { hs_end[i * 32 + lane] = 0xffffffffu; hs_start[i * 32 + lane] = 0u; }
      if (lane < R) hmask[lane] = 0u;
      __syncwarp();
      while (true) {
        const uint64_t k = kc + lane;
        const uint64_t b = win_b, bn = win_bn;  // window at kc, loaded one step ahead
        const uint64_t d = b - sb;  // >= 0 for every unconsumed boundary
        const bool in = d < (uint64_t)span;
        if (in) {
          const uint32_t pos = (uint32_t)d >> 6;
          atomicOr(&hmask[pos >> 5], 1u << (pos & 31));
          atomicMax(&hs_start[pos], (uint32_t)k);                       // the last boundary at this offset starts the live segment
          if (k > 0) atomicMin(&hs_end[pos], (uint32_t)k - 1u);         // the first one ends the previous segment
          if (bn == b) finish_empty<W>(a, (uint32_t)k);                 // segment k is empty
        }
        const int cnt = __popc(__ballot_sync(0xffffffffu, in));
        kc += cnt;
        if (cnt) load_window();
        if (cnt < 32) break;
      }
      __syncwarp();

      // ---- wait for this step's bytes --------------------------------------------------------------------
      cp_async_wait<NSTAGE - 1>();
      __syncwarp();

      // ---- lane run: R consecutive records, left to right -------------------------------------------------
      const uint32_t sbase = stage0 + (uint32_t)stage * STAGE_BYTES;
      uint32_t hbits;
      if (R >= 32) hbits = hmask[lane];
      else hbits = (hmask[(lane * R) >> 5] >> ((lane * R) & 31)) & ((R >= 32) ? 0xffffffffu : ((1u << R) - 1u));
      Xf<W> cur = identity<W>();
      Xf<W> first = identity<W>();
      uint32_t first_seg = 0xffffffffu;
      bool have_first = false;
#pragma unroll
      for (int t = 0; t < R; ++t) {
        const int p = lane * R + t;
        if (hbits & (1u << t)) {
          const uint32_t eseg = hs_end[p];
          if (!have_first) { first = cur; first_seg = eseg; have_first = true; }
          else if (eseg != 0xffffffffu) finish_segment<W>(a, f64_mask, eseg, cur);  // began and ended inside this run
          cur = identity<W>();
        }
        if (p < nvalid) {
          const uint32_t rec = sbase + (uint32_t)(p / RPL) * 128u;
          const uint32_t lane7 = (uint32_t)(lane & 7), parc = (uint32_t)(t % RPL) * CPR;  // p%RPL == t%RPL: RPL divides R
          uint32_t sv[DIRECT ? 1 : NS];
          if constexpr (REC == 16) {
            const uint4 r4 = lds128(rec + ((((uint32_t)(t % RPL)) ^ lane7) << 4));
            sv[0] = r4.x; sv[1] = r4.y; sv[2] = r4.z; sv[3] = r4.w;
          } else if (DIRECT) {
            sv[0] = lds32(rec + soff[t % RPL][0]);
          } else {
#pragma unroll
            for (int s = 0; s < NS; ++s) sv[s] = lds32(rec + soff[t % RPL][s]);
          }
          const uint32_t type = sv[0];
          uint4 e0 = make_uint4(0, 0, 0, 0);
          if (type < 16u) e0 = *reinterpret_cast<const uint4*>(tab + type * kTabStride);
          if (!(e0.x & kRuleValid)) {
            cur.m |= M_ERR;  // THROW rule or scala.MatchError
          } else if (CLS == 1 && (e0.x & kRuleIfExists) && cur.ex == EX_NONE) {
            // IF_EXISTS event after a tombstone in this run: the state does not exist, the event is a no-op
          } else {
            if (CLS == 0 || !(e0.x & kRuleIfExists)) cur.ex = rule_ex(e0.x);  // an IF_EXISTS event leaves the exists-op as it is
            uint32_t spec[W];
            spec[0] = e0.y;
            if (W > 1) spec[1] = e0.z;
            if (W > 2) spec[2] = e0.w;
#pragma unroll
            for (int w = 3; w < W; ++w) spec[w] = tab[type * kTabStride + 1 + w];
#pragma unroll
            for (int w = 0; w < W; ++w) {
              uint32_t val = 0;
              if (DIRECT) {
                const uint32_t sl = spec_slot(spec[w]);
                if (sl) { const uint32_t sw = pg.slot_word[sl]; val = lds32(rec + ((((parc + (sw >> 2)) ^ lane7) << 4) | ((sw & 3u) << 2))); }
              } else {
#pragma unroll
                for (int s = 1; s < NS; ++s) val = (spec_slot(spec[w]) == (uint32_t)s) ? sv[s] : val;
              }
              if (spec_neg(spec[w])) val = 0u - val;
              const uint32_t mode = spec_mode(spec[w]);
              if (mode == kModeSet) cur.v[w] = val;
              else if (mode == kModeAdd) cur.v[w] += val;
              cur.m |= mode << (2 * w);
            }
            cur.m |= rule_copy_bit(e0.x);
          }
        }
      }
      // cur = transformer of the records after the run's last head (the whole run if it has none)

      // ---- once per step: segmented inclusive scan of the 32 lane transformers, in log order -------------
      const uint32_t lane_heads = __ballot_sync(0xffffffffu, have_first);
      Xf<W> sc = cur;
      if (lane == 0 && !have_first) sc = compose<W, CLS>(carry, sc);
#pragma unroll
      for (int dd = 1; dd < 32; dd <<= 1) {
        const Xf<W> o = shfl_xf(sc, lane - dd);  // wraps for lane < dd; masked below
        const int sh = lane >= dd ? lane - dd + 1 : 0;
        const uint32_t window = (lane_heads >> sh) & ((1u << dd) - 1u);  // a head in lanes (lane-dd, lane]?
        if (lane >= dd && window == 0) sc = compose<W, CLS>(o, sc);
      }
      // what flows INTO each lane's run: the scan value of the previous lane (lane 0: the carry)
      Xf<W> cin = shfl_xf(sc, lane - 1);
      if (lane == 0) cin = carry;
      carry = shfl_xf(sc, 31);

      // ---- the segment that ends at a run's first head needs what flowed in ----------------------------------
      if (have_first && first_seg != 0xffffffffu) {
        const Xf<W> tot = compose<W, CLS>(cin, first);
        // the very first head of the chunk ends a segment that began in an earlier chunk: look-back needed
        const bool is_span_first = !span_has_head && (lane_heads & ((1u << lane) - 1u)) == 0;
        if (is_span_first && chunk != 0) { inh_t = tot; inh_seg = first_seg; inh_pending = true; }
        else finish_segment<W>(a, f64_mask, first_seg, tot);
      }
      if (lane_heads) {
        // the pending look-back lives in the lane that saw the chunk's first head: move it to lane 0
        if (!span_has_head) {
          const int src = __ffs(lane_heads) - 1;
          inh_t = shfl_xf(inh_t, src);
          inh_seg = __shfl_sync(0xffffffffu, inh_seg, src);
          inh_pending = __shfl_sync(0xffffffffu, (int)inh_pending, src) != 0;
        }
        span_has_head = true;
      }
      __syncwarp();
      if constexpr (REC == 16) {
        // one load per step, so each has a step's time to arrive: the ticket drawn at the chunk's start, then its table entry,
        // then its window
        if (a.chunk_kc && pf_kc == ~0u) {
          resolve_next();
          if (nxt != kNone && nxt != chunk + 1) pf_kc = (uint32_t)a.chunk_kc[nxt];
        } else if (a.chunk_kc && !pf_win) {
          const uint64_t k = (uint64_t)pf_kc + lane;
          pf_b = k <= n_seg ? a.seg_offsets[k] : ~0ull;
          pf_bn = k < n_seg ? a.seg_offsets[k + 1] : ~0ull;
          pf_win = true;
        }
      }
      if (++stage == NSTAGE) stage = 0;
    }

    // ---- end of the log: the open segment and any trailing empty segments --------------------------------
    // boundaries with off[k] == log_end were never a head inside a step; kc is the first of them.
    bool end_needs_lookback = false;
    if (step_end == total_steps) {
      for (uint64_t k = kc + lane; k < n_seg; k += 32) finish_empty<W>(a, (uint32_t)k);  // segments kc..n_seg-1 are empty
      if (kc >= 1) {
        // segment kc-1 is the last non-empty one; its transformer is the carry
        if (span_has_head || chunk == 0) { if (lane == 0) finish_segment<W>(a, f64_mask, (uint32_t)(kc - 1), carry); }
        else end_needs_lookback = true;  // the whole chunk lies inside that segment
      }
    }

    // ---- publish this chunk's open transformer, then finish what needs the preceding chunks -----------------
    {
      if constexpr (REC == 16) {
        if (lane == 0)
          st_volatile_v4(a.part_flags + 4 * chunk, carry.m | (carry.ex << kRowEx) | (span_has_head ? kRowHead : 0u), carry.v[0], carry.v[1],
                         a.epoch);
      } else if (lane == 0) {
        uint32_t* part_data = a.part_data + chunk * (W + 2);
        part_data[0] = carry.m;
#pragma unroll
        for (int w = 0; w < W; ++w) part_data[1 + w] = carry.v[w];
        part_data[W + 1] = carry.ex | (span_has_head ? 4u : 0u);
        __threadfence();
        st_volatile_u32(a.part_flags + chunk, a.epoch);
      }
      if (lane == 0) {
        // the previous chunk's look-back, left until now: its predecessors were folded while this chunk was
        if (dfr) { finish_segment<W>(a, f64_mask, dfr_seg, compose<W, CLS>(look_back(dfr_chunk), dfr_t)); dfr = false; }
        if (inh_pending) { dfr = true; dfr_chunk = chunk; dfr_seg = inh_seg; dfr_t = inh_t; }
        // (a chunk without a head has no pending segment; the one that ends the log finishes the open one now)
        if (end_needs_lookback) finish_segment<W>(a, f64_mask, (uint32_t)(kc - 1), compose<W, CLS>(look_back(chunk), carry));
      }
      __syncwarp();
    }
    // every record of the chunk was applied; records of throwing segments are taken back by the replay below
    {
      const uint64_t we = base + step_end * (uint64_t)STEP_BYTES < a.log_end ? base + step_end * (uint64_t)STEP_BYTES : a.log_end;
      n_applied += (we - wb) >> 6;
    }
    prev_chunk = chunk;
    resolve_next();
    chunk = nxt;
  }  // chunks
  cp_async_wait<0>();
  if (lane == 0 && dfr) finish_segment<W>(a, f64_mask, dfr_seg, compose<W, CLS>(look_back(dfr_chunk), dfr_t));

  // an empty log (every segment empty): warp 0 writes every state
  if (n_chunks == 0 && gw == 0)
    for (uint64_t k = lane; k < n_seg; k += 32) finish_empty<W>(a, (uint32_t)k);

  // ---- arrival, then the exact replay of the throwing segments, without a grid barrier ----------------------------
  // A warp that arrives while no segment is queued for replay leaves at once (its SM slot goes to the next fold). One that
  // arrives after a throw waits for the others and helps with the replay; the last warp to arrive always does, so the
  // replay list is complete whoever replays it.
  unsigned long long arrived = 0, n_redo = 0;
  if (lane == 0) {
    if (n_applied) atomicAdd(a.counters + 0, n_applied);
    __threadfence();
    arrived = atomicAdd(a.counters + 6, 1ull) + 1;
    __threadfence();
    n_redo = ld_volatile_u64(a.counters + 3);
    if (arrived < n_warps && n_redo != 0) {
      while (ld_volatile_u64(a.counters + 6) < n_warps) { __nanosleep(128); }
      __threadfence();
      n_redo = ld_volatile_u64(a.counters + 3);
    }
    if (n_redo == 0) atomicMax(a.counters + 9, global_ns());
  }
  n_redo = __shfl_sync(0xffffffffu, n_redo, 0);
  if (n_redo == 0) return;
  replay_segments<W>(a, pg, tab, lane, n_redo);
}

// ---- exact replay of the throwing segments the fold listed (counters[3] of them) -------------------------------------
// A segment whose handler threw keeps its pre-batch state and reports the index of the throwing event
// (PersistentActor.scala:260-263); that needs the strictly sequential walk, done here one lane per segment. The warps that
// replay take 32 list entries at a time from a cursor (counters[11]).
template <int W>
__device__ __noinline__ void replay_segments(const RowArgs& a, const RowProgram& pg, const uint32_t* tab, int lane, unsigned long long n_redo) {
  if (n_redo > a.redo_cap) n_redo = a.redo_cap;  // overflow: the host re-runs the whole fold sequentially
  unsigned long long n_err = 0, n_dropped = 0;
  while (true) {
    unsigned long long i0 = 0;
    if (lane == 0) i0 = atomicAdd(a.counters + 11, 32ull);
    i0 = __shfl_sync(0xffffffffu, i0, 0);
    if (i0 >= n_redo) break;
    const unsigned long long i = i0 + lane;
    if (i >= n_redo) continue;
    const uint32_t seg = a.redo_ids[i];
    const uint64_t b = a.seg_offsets[seg], e = a.seg_offsets[(uint64_t)seg + 1];
    const uint64_t slot = a.seg_ids ? (uint64_t)a.seg_ids[seg] : (uint64_t)seg;
    uint32_t st[W], ex0 = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) st[w] = 0;
    if (a.states_in) {
      const uint32_t* sp = reinterpret_cast<const uint32_t*>(a.states_in + slot * (uint64_t)(W + 2) * 4);
      ex0 = sp[W] & SGR_ST_EXISTS;
#pragma unroll
      for (int w = 0; w < W; ++w) st[w] = ex0 ? sp[w] : 0u;
    }
    uint32_t old[W];
#pragma unroll
    for (int w = 0; w < W; ++w) old[w] = st[w];
    uint32_t exn = ex0, k = 0;
    bool threw = false;
    for (uint64_t pos = b; pos < e; pos += 64, ++k) {
      const uint32_t* rec = reinterpret_cast<const uint32_t*>(a.events + pos);
      const uint32_t type = rec[pg.slot_word[0]];
      const uint32_t fl = type < 16u ? tab[type * kTabStride] : 0u;
      if (!(fl & kRuleValid)) { threw = true; break; }
      if (fl & kRuleNone) { exn = 0u; for (int w = 0; w < W; ++w) st[w] = 0u; continue; }  // tombstone
      if ((fl & kRuleIfExists) && !exn) continue;                                          // IF_EXISTS on None: no-op
#pragma unroll
      for (int w = 0; w < W; ++w) {
        const uint32_t spec = tab[type * kTabStride + 1 + w];
        const uint32_t mode = spec_mode(spec);
        uint32_t val = spec_slot(spec) ? rec[pg.slot_word[spec_slot(spec)]] : 0u;
        if (spec_neg(spec)) val = 0u - val;
        if (mode == kModeSet) st[w] = val; else if (mode == kModeAdd) st[w] = (exn ? st[w] : 0u) + val;
        else if (!exn) st[w] = 0u;
      }
      exn = SGR_ST_EXISTS;
    }
    uint8_t* row = a.states_out + slot * (uint64_t)(W + 2) * 4;
    if (threw) {
      uint32_t* dp = reinterpret_cast<uint32_t*>(row);
#pragma unroll
      for (int w = 0; w < W; ++w) dp[w] = old[w];
      dp[W] = ex0 | SGR_ST_ERROR;
      dp[W + 1] = k;
      ++n_err;
      n_dropped += ((e - b) >> 6) - k;
    } else {
      finish_row<W>(row, old, ex0, st, exn);  // (a replayed segment that did not throw cannot occur)
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    n_err += __shfl_xor_sync(0xffffffffu, n_err, o);
    n_dropped += __shfl_xor_sync(0xffffffffu, n_dropped, o);
  }
  if (lane == 0) {
    if (n_err) atomicAdd(a.counters + 1, n_err);
    if (n_dropped) atomicAdd(a.counters + 4, n_dropped);
    __threadfence();
    atomicMax(a.counters + 9, global_ns());
  }
}

typedef void (*RunKernel)(const RowArgs, const RowProgram);
struct RunVariant { RunKernel k[3]; int r, nstage; const char* name; };  // 16-byte states; k[i]: NS = 2, 3, 6 (slot plane: k[0])
#define RUN_VARIANT(R, ST, MINB) {{fold_runs_kernel<2, R, ST, 2, MINB, false, 0>, fold_runs_kernel<2, R, ST, 3, MINB, false, 0>, fold_runs_kernel<2, R, ST, 6, MINB, false, 0>}, R, ST, "runs W2 R" #R " st" #ST}
const RunVariant kRunVariants[] = {
    RUN_VARIANT(4, 2, 3), RUN_VARIANT(4, 1, 5), RUN_VARIANT(2, 2, 5), RUN_VARIANT(2, 1, 5), RUN_VARIANT(4, 3, 2), RUN_VARIANT(8, 1, 3), RUN_VARIANT(2, 3, 4),
};
constexpr int kNumRunVariants = sizeof(kRunVariants) / sizeof(kRunVariants[0]);
// the same staging from the head plane (32 bytes per record): a step stages half the bytes, so deeper pipelines fit. The
// first is the default: the fastest on the configs[1] log (scripts/fold_ceiling.py --head-variants, DESIGN.md section 4)
#define HEAD_VARIANT(R, ST, MINB) {{fold_runs_kernel<2, R, ST, 2, MINB, false, 0, 32>, fold_runs_kernel<2, R, ST, 3, MINB, false, 0, 32>, fold_runs_kernel<2, R, ST, 6, MINB, false, 0, 32>}, R, ST, "heads W2 R" #R " st" #ST}
const RunVariant kHeadVariants[] = {
    HEAD_VARIANT(8, 2, 3), HEAD_VARIANT(4, 3, 4), HEAD_VARIANT(4, 2, 4), HEAD_VARIANT(4, 4, 3), HEAD_VARIANT(8, 3, 2),
};
constexpr int kNumHeadVariants = sizeof(kHeadVariants) / sizeof(kHeadVariants[0]);
// the slot plane (16 bytes per record, slot s at word s): a 128-byte line holds 8 records, so a run is R = 8 records, one
// line, and one kernel serves every slot count. The first is the default (scripts/fold_ceiling.py --proj-variants,
// DESIGN.md section 4)
#define PROJ_VARIANT(ST, MINB) {{fold_runs_kernel<2, 8, ST, 4, MINB, false, 0, 16>, nullptr, nullptr}, 8, ST, "slots W2 R8 st" #ST}
const RunVariant kProjVariants[] = {
    PROJ_VARIANT(2, 5), PROJ_VARIANT(3, 3), PROJ_VARIANT(4, 2), PROJ_VARIANT(6, 2),
};
constexpr int kNumProjVariants = sizeof(kProjVariants) / sizeof(kProjVariants[0]);
// wider states / many source words: one configuration each (R = 4, 2 stages, direct word reads)
constexpr int kWideR = 4, kWideStages = 2;

bool is_wide(const RowProgram& prog) { return prog.user_words != 2 || prog.n_slots > 6 || prog.cls != 0; }
// plane 0: the log, run variant v; 32: the head plane, head variant v; 16: the slot plane, projected variant v
const RunVariant& pick_variant(int v, int plane) {
  if (plane == 16) return kProjVariants[(v >= 0 && v < kNumProjVariants) ? v : 0];
  if (plane == 32) return kHeadVariants[(v >= 0 && v < kNumHeadVariants) ? v : 0];
  return kRunVariants[(v >= 0 && v < kNumRunVariants) ? v : 0];
}
int variant_r(int v, int plane, const RowProgram& prog) { return plane != 16 && is_wide(prog) ? kWideR : pick_variant(v, plane).r; }
int variant_nstage(int v, int plane, const RowProgram& prog) { return plane != 16 && is_wide(prog) ? kWideStages : pick_variant(v, plane).nstage; }
size_t variant_smem(int v, int plane, const RowProgram& prog) {
  const size_t r = (size_t)variant_r(v, plane, prog), ns = (size_t)variant_nstage(v, plane, prog), rec = plane ? (size_t)plane : 64;
  return (size_t)kRunWarps * (ns * 32 * rec * r + 2 * 32 * r * 4 + 32 * 4);
}
RunKernel variant_kernel(int v, int plane, const RowProgram& prog) {
  if (plane == 16) return pick_variant(v, plane).k[0];
  if (plane == 32) {
    if (prog.user_words == 14) return fold_runs_kernel<14, kWideR, kWideStages, 1, 1, true, 1, 32>;
    if (prog.user_words == 6) return fold_runs_kernel<6, kWideR, kWideStages, 1, 2, true, 1, 32>;
    if (is_wide(prog)) return fold_runs_kernel<2, kWideR, kWideStages, 1, 3, true, 1, 32>;
  } else {
    if (prog.user_words == 14) return fold_runs_kernel<14, kWideR, kWideStages, 1, 1, true, 1>;
    if (prog.user_words == 6) return fold_runs_kernel<6, kWideR, kWideStages, 1, 2, true, 1>;
    if (is_wide(prog)) return fold_runs_kernel<2, kWideR, kWideStages, 1, 3, true, 1>;
  }
  return pick_variant(v, plane).k[prog.n_slots <= 2 ? 0 : (prog.n_slots <= 3 ? 1 : 2)];
}

}  // namespace

int run_variant_count() { return kNumRunVariants; }
const char* run_variant_name(int v) { return (v >= 0 && v < kNumRunVariants) ? kRunVariants[v].name : "?"; }
int head_variant_count() { return kNumHeadVariants; }
int proj_variant_count() { return kNumProjVariants; }
bool slot_plane_fits(const RowProgram& prog) {
  return prog.head_only && prog.user_words == 2 && prog.cls == 0 && prog.n_slots <= 4;
}

int run_kernel_max_grid(int num_sms, int variant, int plane, const RowProgram& prog) {
  const size_t smem = variant_smem(variant, plane, prog);
  RunKernel k = variant_kernel(variant, plane, prog);
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kRunThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * num_sms;
}

int run_variant_step_bytes(int variant, int plane, const RowProgram& prog) { return 2048 * variant_r(variant, plane, prog); }
int run_warps_per_cta() { return kRunWarps; }

uint64_t run_variant_chunk_steps(int variant, int plane, const RowProgram& prog, uint64_t chunk_bytes, uint64_t steps, uint64_t n_warps) {
  const uint64_t ns = (uint64_t)variant_nstage(variant, plane, prog);
  const uint64_t lo = ns > 1 ? ns - 1 : 1;  // what is staged ahead stays inside the next chunk
  uint64_t hi = chunk_bytes / (uint64_t)run_variant_step_bytes(variant, plane, prog);
  if (hi < lo) hi = lo;
  const uint64_t fair = n_warps ? steps / n_warps : hi;  // a chunk for every warp on a small log
  return fair < lo ? lo : (fair > hi ? hi : fair);
}

cudaError_t launch_fold_runs(const RowArgs& args, const RowProgram& prog, int variant, int plane, int grid, bool overlap, cudaStream_t stream) {
  const size_t smem = variant_smem(variant, plane, prog);
  RunKernel k = variant_kernel(variant, plane, prog);  // its smem attribute was set by run_kernel_max_grid
  // overlap: the launch may begin while the fold before it drains (programmatic dependent launch); the kernel waits on the
  // device for its predecessor before it touches anything that predecessor writes
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(kRunThreads); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = overlap ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, k, args, prog);
}

// ---- the head plane: bytes 0..31 of every record of the log, densely --------------------------------------------------
// One warp moves 16 records per pass: lane l reads the 16-byte chunk l&1 of record l/2, so a warp's reads are the 32-byte
// halves of 16 consecutive records (sixteen 64-byte blocks, the first of each read) and its 512-byte write is contiguous.
__global__ void __launch_bounds__(256) build_heads_kernel(const uint8_t* log, uint8_t* heads, uint64_t rec0, uint64_t rec1) {
  const uint64_t n_chunks = (rec1 - rec0) * 2;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_chunks; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r = rec0 + (g >> 1), c = g & 1;
    const uint4 v = __ldcs(reinterpret_cast<const uint4*>(log + r * 64) + c);
    reinterpret_cast<uint4*>(heads + r * 32)[c] = v;
  }
}

cudaError_t launch_build_heads(const uint8_t* log, uint8_t* heads, uint64_t rec0, uint64_t rec1, int num_sms, cudaStream_t stream) {
  if (rec1 <= rec0) return cudaSuccess;
  const uint64_t want = ((rec1 - rec0) * 2 + 255) / 256;
  const uint64_t cap = (uint64_t)num_sms * 16;
  build_heads_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, stream>>>(log, heads, rec0, rec1);
  return cudaGetLastError();
}

// ---- the slot plane: the program's slot words of every record, 16 bytes per record, slot s at word s --------------------
// One thread per record: it reads the record's head (the second 16 bytes only when a slot word lies there) and keeps the
// slot words, so a warp writes 32 records' slots as one contiguous 512-byte block. sel: slot word s in bits [4s, 4s+4).
__global__ void __launch_bounds__(256) build_slots_kernel(const uint8_t* log, uint8_t* slots, uint64_t rec0, uint64_t rec1, uint32_t sel,
                                                          uint32_t n_slots, bool upper) {
  for (uint64_t r = rec0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rec1; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint4* rp = reinterpret_cast<const uint4*>(log + r * 64);
    const uint4 lo = __ldcs(rp), hi = upper ? __ldcs(rp + 1) : make_uint4(0, 0, 0, 0);
    const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    uint32_t o[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const uint32_t sw = (sel >> (4 * s)) & 7u;
      uint32_t v = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) v = sw == (uint32_t)k ? w[k] : v;  // a select chain: no local-memory indexing
      o[s] = (uint32_t)s < n_slots ? v : 0u;
    }
    reinterpret_cast<uint4*>(slots)[r] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

cudaError_t launch_build_slots(const uint8_t* log, uint8_t* slots, uint64_t rec0, uint64_t rec1, const RowProgram& prog, int num_sms,
                               cudaStream_t stream) {
  if (rec1 <= rec0) return cudaSuccess;
  if (!slot_plane_fits(prog)) return cudaErrorInvalidValue;
  uint32_t sel = 0;
  bool upper = false;
  for (uint32_t s = 0; s < prog.n_slots; ++s) { sel |= prog.slot_word[s] << (4 * s); upper |= prog.slot_word[s] >= 4; }
  const uint64_t want = (rec1 - rec0 + 255) / 256;
  const uint64_t cap = (uint64_t)num_sms * 16;
  build_slots_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, stream>>>(log, slots, rec0, rec1, sel, prog.n_slots, upper);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256) build_chunk_table_kernel(const uint64_t* off, uint64_t n_seg, uint64_t log_begin, uint64_t chunk_bytes,
                                                               uint64_t n_chunks, uint64_t* table) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const uint64_t wb = log_begin + c * chunk_bytes;
  uint64_t lo = 0, hi = n_seg + 1;  // the first k in [0, n_seg] with off[k] >= wb, as fold_runs_kernel's first_boundary
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (off[mid] >= wb) hi = mid; else lo = mid + 1;
  }
  table[c] = lo;
}

cudaError_t launch_build_chunk_table(const uint64_t* off, uint64_t n_seg, uint64_t log_begin, uint64_t step_bytes, uint64_t chunk_steps,
                                     uint64_t n_chunks, uint64_t* table, cudaStream_t stream) {
  if (!n_chunks) return cudaSuccess;
  build_chunk_table_kernel<<<(unsigned)((n_chunks + 255) / 256), 256, 0, stream>>>(off, n_seg, log_begin, step_bytes * chunk_steps, n_chunks, table);
  return cudaGetLastError();
}

namespace {
// ---- read-ceiling probe (scripts/fold_ceiling.py) ----------------------------------------------------------------------
// The default variant's staging alone — the same CTAs, warps and shared memory, 16-byte cp.async copies of 8 KiB steps,
// two stages — over a buffer, with no fold work: the practical read ceiling of the fold on this card. Warps take fixed
// spans (1/n of the buffer each) or chunks of chunk_steps steps by ticket (ctl[0], zero before the launch).
template <bool TICKET>
__global__ void __launch_bounds__(kRunThreads, 3) read_probe_kernel(const uint8_t* buf, uint64_t bytes, uint64_t chunk_steps, unsigned long long* ctl) {
  constexpr int R = 4, NSTAGE = 2, STEP_BYTES = 2048 * R;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t stage0 = smem_u32(smem_raw + (size_t)warp * warp_smem_bytes<R, NSTAGE>());
  const uint64_t gw = (uint64_t)blockIdx.x * kRunWarps + warp, n_warps = (uint64_t)gridDim.x * kRunWarps;
  const uint64_t total_steps = (bytes + STEP_BYTES - 1) / STEP_BYTES;
  auto issue = [&](uint64_t s, int stage) {
    const uint64_t sbyte = s * (uint64_t)STEP_BYTES;
    const uint32_t dst = stage0 + (uint32_t)stage * STEP_BYTES + (uint32_t)lane * 16u;
#pragma unroll
    for (int q = 0; q < 4 * R; ++q)
      if (sbyte + (uint64_t)q * 512 + (uint64_t)lane * 16 < bytes) cp_async16(dst + q * 512, buf + sbyte + q * 512 + lane * 16);
  };
  uint32_t acc = 0;
  auto run = [&](uint64_t s0, uint64_t s1) {
    if (s0 < s1) issue(s0, 0);
    cp_async_commit();
    int stage = 0;
    for (uint64_t s = s0; s < s1; ++s) {
      if (s + 1 < s1) issue(s + 1, stage ^ 1);
      cp_async_commit();
      cp_async_wait<NSTAGE - 1>();
      __syncwarp();
      acc ^= lds32(stage0 + (uint32_t)stage * STEP_BYTES + (uint32_t)lane * 4u);
      __syncwarp();
      stage ^= 1;
    }
    cp_async_wait<0>();
  };
  if (!TICKET) {
    const uint64_t spw = (total_steps + n_warps - 1) / n_warps, s0 = gw * spw;
    run(s0, s0 + spw < total_steps ? s0 + spw : total_steps);
  } else {
    const uint64_t n_chunks = (total_steps + chunk_steps - 1) / chunk_steps;
    for (uint64_t c = gw; c < n_chunks;) {
      const uint64_t s0 = c * chunk_steps;
      run(s0, s0 + chunk_steps < total_steps ? s0 + chunk_steps : total_steps);
      unsigned long long t = 0;
      if (lane == 0) t = atomicAdd(ctl, 1ull);
      c = n_warps + __shfl_sync(0xffffffffu, t, 0);
    }
  }
  if (acc == 0x9e3779b9u) ctl[1] = acc;  // keeps the shared-memory reads
}
}  // namespace

}  // namespace sgr

extern "C" int32_t sgr_probe_read(const void* buf, uint64_t bytes, int32_t ticketed, uint64_t chunk_bytes, void* ctl, void* stream) {
  using namespace sgr;
  int dev = 0, n_sm = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return SGR_ERR_CUDA;
  auto k = ticketed ? read_probe_kernel<true> : read_probe_kernel<false>;
  const size_t smem = (size_t)kRunWarps * warp_smem_bytes<4, 2>();
  if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kRunThreads, smem) != cudaSuccess || per_sm < 1)
    return SGR_ERR_CUDA;
  const uint64_t steps = chunk_bytes / 8192 > 2 ? chunk_bytes / 8192 : 2;
  k<<<per_sm * n_sm, kRunThreads, smem, (cudaStream_t)stream>>>((const uint8_t*)buf, bytes, steps, (unsigned long long*)ctl);
  return cudaGetLastError() == cudaSuccess ? SGR_OK : SGR_ERR_CUDA;
}
