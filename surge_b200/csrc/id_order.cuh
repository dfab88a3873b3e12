// id_order.cuh — the Bytes order of the engine's aggregate ids behind sgr_scan (launch interface of id_order.cu).
//
// The order is a permutation of the ids [0, n) that the id index (id_index.cuh) holds: order[p] is the dense index of the id at
// position p in Bytes order (unsigned lexicographic over the UTF-8 bytes, a prefix before any longer id). It reads the ids
// where the index keeps them (key_ref + arena), so it costs 4 bytes per id on the device. It follows the index: appended ids
// are sorted among themselves and merged in; a rebuilt index (new key table) is ordered again from id 0; a rehash, which
// moves neither key_ref nor the arena, leaves it alone.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "devbuf.h"

namespace sgr {

struct IdOrder {
  DevBuf order;                // u32[n]
  uint64_t n = 0;              // ids [0, n) of the index are ordered
  uint64_t builds = ~0ull;     // the IdIndex::builds the order was made for (another value: order again from id 0)
};

// Bring the order up to ids [0, to) of the index: from id 0 when o.n == 0, else sort ids [o.n, to) and merge them with the
// ordered ones. Synchronises `st` once per sort round. Scratch is allocated for the call and freed before it returns.
cudaError_t id_order_update(IdOrder& o, const uint2* key_ref, const uint8_t* arena, uint64_t to, cudaStream_t st);

// One small launch: range[0] = the first position whose id is >= from (> from when from_exclusive; 0 when from is null),
// range[1] = the first position whose id is > to (n when to is null), raised to range[0] when from > to. from / to: device
// bytes, 8-byte aligned and readable up to their length rounded up to 8.
cudaError_t id_order_bounds(const IdOrder& o, const uint2* key_ref, const uint8_t* arena, const uint8_t* from, uint32_t from_len,
                            bool from_exclusive, const uint8_t* to, uint32_t to_len, unsigned long long* range, cudaStream_t st);

}  // namespace sgr
