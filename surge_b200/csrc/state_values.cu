// state_values.cu — rows -> JSON state values (state_writer.h) on the device, for the value-returning reads of engine.cu.
// Under the protobuf wrapping (kWrap: sgr_set_state_writer_framing) each value is the multilanguage State around the JSON value:
// the length pass adds the wrapper to the JSON length, and the write pass recovers the JSON length from the value's span.
//
//   length   one thread per row: the value's bytes, or 0 for a None row and for a row that cannot be written (whose status it
//            records, the lowest such row by atomicMin)
//   scan     cub::DeviceScan::ExclusiveSum over the n + 1 lengths: every value's offset, offs[n] the total
//   fit      one thread: the longest prefix whose values fit in the caller's capacity (binary search over the offsets), and
//            the status and dense index of the lowest refused row when it lies inside that prefix
//   write    one thread per row of the prefix writes its value at its offset
// The host reads the control words back between fit and write. A row's value is written by one thread, members in order, the id
// member with a loop over its bytes: ids are short in practice, and the rare long one (up to 2^24 bytes, 6x that escaped) costs
// that thread a long loop but never registers or local memory.
#include <cub/device/device_scan.cuh>

#include "../../include/sgr.h"
#include "state_values.cuh"

namespace sgr {
namespace {

constexpr int kThreads = 256;

unsigned blocks_for(uint64_t n) {
  const uint64_t b = (n + kThreads - 1) / kThreads;
  return (unsigned)(b < 65535ull * 16 ? (b ? b : 1) : 65535ull * 16);
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// scratch: control words | lengths (n + 1) | offsets (n + 1) | statuses (n) | cub temporary storage
struct Carve { unsigned long long *ctl, *lens, *offs; uint32_t* status; void* tmp; size_t tmp_bytes, total; };

Carve carve(void* base, uint64_t n) {
  Carve c{};
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (uint64_t)(n + 1));
  uint8_t* p = (uint8_t*)base;
  size_t at = 0;
  c.ctl = (unsigned long long*)(p + at); at += align256(8 * kSvCtlWords);
  c.lens = (unsigned long long*)(p + at); at += align256((n + 1) * 8);
  c.offs = (unsigned long long*)(p + at); at += align256((n + 1) * 8);
  c.status = (uint32_t*)(p + at); at += align256(n * 4 + 4);
  c.tmp = p + at; c.tmp_bytes = tb; at += align256(tb);
  c.total = at;
  return c;
}

__device__ __forceinline__ void row_id(const SvRows& r, uint64_t i, const uint8_t** id, uint64_t* len, bool* has) {
  const long long d = r.idx[i];
  *has = d >= 0 && (unsigned long long)d < r.n_keys;
  *id = r.ids + r.id_offs[i];
  *len = *has ? r.id_offs[i + 1] - r.id_offs[i] : 0;
}

template <bool kWrap>
__global__ void __launch_bounds__(kThreads) sv_len_kernel(const SwWriter w, const SvRows r, unsigned long long* lens, uint32_t* status,
                                                          unsigned long long* ctl) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= r.n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (i == r.n) { lens[i] = 0; continue; }
    uint64_t len = 0;
    if (r.flags[i] & SGR_ST_EXISTS) {
      const uint8_t* id; uint64_t id_len; bool has_id;
      row_id(r, i, &id, &id_len, &has_id);
      const uint8_t* row = r.rows + i * r.user;
      len = 1;   // '}'
      uint32_t why = sw::OK, k = 0;
      for (; k < w.n; ++k) {
        len += sw::member_len(w.m[k], row, id, id_len, has_id, &why);
        if (why) break;
      }
      if constexpr (kWrap) {   // the State around it: the id must be one the ID member could write
        if (!why) {
          if (!has_id) { why = sw::NO_ID; k = sw::kWrapMember; }
          else if (!sw::utf8_ok(id, id_len)) { why = sw::ID_UTF8; k = sw::kWrapMember; }
          else len = sw::wrap_len(id_len, len);
        }
      }
      if (why) {
        len = 0;
        status[i] = k << 8 | why;
        atomicMin(ctl + kSvRefused, (unsigned long long)i);
      }
    }
    lens[i] = len;
  }
}

__global__ void sv_fit_kernel(const unsigned long long* offs, uint64_t n, unsigned long long cap, const uint32_t* status, const long long* idx,
                              unsigned long long* ctl) {
  uint64_t lo = 0, hi = n;   // offs[0] == 0 always fits
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo + 1) / 2;
    if (offs[mid] <= cap) lo = mid; else hi = mid - 1;
  }
  ctl[kSvRows] = lo;
  ctl[kSvBytes] = offs[lo];
  const unsigned long long bad = ctl[kSvRefused];
  if (bad < lo) { ctl[kSvStatus] = status[bad]; ctl[kSvIndex] = (unsigned long long)idx[bad]; }
}

template <bool kWrap>
__global__ void __launch_bounds__(kThreads) sv_write_kernel(const SwWriter w, const SvRows r, uint64_t n_rows, const unsigned long long* offs,
                                                            uint8_t* values) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_rows; i += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long b = offs[i];
    if (offs[i + 1] == b) continue;   // a None row
    const uint8_t* id; uint64_t id_len; bool has_id;
    row_id(r, i, &id, &id_len, &has_id);
    const uint8_t* row = r.rows + i * r.user;
    uint8_t* o = values + b;
    if constexpr (kWrap) o = sw::wrap_head_write(o, id, id_len, sw::wrap_json_len(id_len, offs[i + 1] - b));
    for (uint32_t k = 0; k < w.n; ++k) o = sw::member_write(o, w.m[k], w.lits, row, id, id_len);
    *o = '}';
  }
}

}  // namespace

size_t state_values_scratch_bytes(uint64_t n) { return carve(nullptr, n).total; }

cudaError_t state_values_measure(const SwWriter& w, bool wrap, const SvRows& r, uint64_t cap, void* scratch, unsigned long long** offs,
                                 unsigned long long** ctl, cudaStream_t st) {
  Carve c = carve(scratch, r.n);
  *offs = c.offs; *ctl = c.ctl;
  cudaError_t e;
  if ((e = cudaMemsetAsync(c.ctl, 0xff, 8 * kSvCtlWords, st)) != cudaSuccess) return e;
  if (wrap) sv_len_kernel<true><<<blocks_for(r.n + 1), kThreads, 0, st>>>(w, r, c.lens, c.status, c.ctl);
  else sv_len_kernel<false><<<blocks_for(r.n + 1), kThreads, 0, st>>>(w, r, c.lens, c.status, c.ctl);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  if ((e = cub::DeviceScan::ExclusiveSum(c.tmp, c.tmp_bytes, c.lens, c.offs, (uint64_t)(r.n + 1), st)) != cudaSuccess) return e;
  sv_fit_kernel<<<1, 1, 0, st>>>(c.offs, r.n, cap, c.status, r.idx, c.ctl);
  return cudaGetLastError();
}

cudaError_t state_values_write(const SwWriter& w, bool wrap, const SvRows& r, uint64_t n_rows, const unsigned long long* offs, uint8_t* values,
                               cudaStream_t st) {
  if (!n_rows) return cudaSuccess;
  if (wrap) sv_write_kernel<true><<<blocks_for(n_rows), kThreads, 0, st>>>(w, r, n_rows, offs, values);
  else sv_write_kernel<false><<<blocks_for(n_rows), kThreads, 0, st>>>(w, r, n_rows, offs, values);
  return cudaGetLastError();
}

}  // namespace sgr
