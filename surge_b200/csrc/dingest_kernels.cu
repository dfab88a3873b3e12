// dingest_kernels.cu — Kafka RecordBatch v2 decode ON THE DEVICE (sm_90a): the step right before the fold (SURVEY §8 f1).
//
// What feeds the store today is a read_committed consumer of a topic whose producer compresses with lz4
// (modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:38; modules/common/src/main/resources/
// reference.conf:124). Round 1 decoded those bytes on the host (csrc/ingest.cpp) and copied 64-byte packed records over PCIe —
// the copy was 95 % of the end-to-end step. Here the WIRE bytes cross PCIe (about 25 B per event instead of 64) and everything
// per-batch and per-record happens on the GPU; the host keeps only the walk over the 61-byte batch headers and the
// read_committed bookkeeping (csrc/dingest.cu). csrc/ingest.cpp stays as the byte-equal checker (tests/test_gpu_dingest.py).
//
// One chain of three launches per group of batches, with no host round trip in between (csrc/dingest.cu runs such chains on
// several streams behind the H2D copies):
//   crc_size    one THREAD per batch: CRC-32C of the batch (slicing-by-8, tables in shared memory) against the header's field;
//               every lz4 batch claims an arena slot of 3x its compressed size with an atomicAdd. (When the claims overflow, the
//               poll is repeated without them: this pass then walks each lz4 frame adding up sequence lengths -> the exact
//               decompressed size, and the host lays the arena out.)
//   decode_walk one thread per batch: lz4 sequences decoded into the batch's arena slot (lz4_fast.h), then the record-boundary
//               walk — a chain of varints — writes every record's offset
//   parse       one thread per RECORD: varint fields, key -> aggregate id (up to ':', KafkaPartitioner.scala:38-42), value ->
//               packed 64-byte record at the record's own slot (arrival order kept), id -> dense index through a device hash
//               table (64-bit hash tag claimed by CAS, id bytes compared, index from an atomic counter)
// Records a read_committed consumer would not deliver (flush markers, duplicates below the partition position, dropped null
// values) become HOLES (agg == ~0) that the fold kernels skip; nothing is compacted.
//
// Thread-per-batch is deliberate: a 16 KiB producer batch is ~2 k lz4 sequences and ~500 varint-delimited records, strictly
// serial inside; the parallelism is the tens of thousands of batches of a restore poll. All of it is HBM/latency-bound
// byte work — no tensor cores anywhere. The two thread-per-batch kernels read their input through a per-thread cp.async ring in
// shared memory (RingIn) and keep memory current behind an 8-byte output accumulator (lz4_fast.h): one dependent memory access
// per lz4 sequence, where bytes walked straight from global memory cost ~10, and in a warp of 32 independent batches some lane
// misses at every step.
#include "dingest_kernels.cuh"
#include "group_kernels.cuh"
#include "lz4_fast.h"

namespace sgr {
namespace {

constexpr int kThreads = 128;
__device__ uint32_t g_crc_tab[8][256];

struct CrcInit {
  uint32_t t[8][256];
  CrcInit() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0x82F63B78u & (0u - (c & 1u)));
      t[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; ++i)
      for (int k = 1; k < 8; ++k) t[k][i] = (t[k - 1][i] >> 8) ^ t[0][t[k - 1][i] & 0xff];
  }
};

cudaError_t ensure_crc_tables() {
  static bool done = false;
  if (done) return cudaSuccess;
  static const CrcInit init;
  cudaError_t e = cudaMemcpyToSymbol(g_crc_tab, init.t, sizeof init.t);
  if (e == cudaSuccess) done = true;
  return e;
}

// A lone thread walking a byte stream pays one global access (hundreds of ns) per byte it looks at: a decode kernel that does
// so takes the same time whatever the number of batches — it is the serial latency of ONE batch. ByteWin keeps the aligned 16-byte chunk around the cursor in registers: one load per 16 bytes of
// tokens, lengths, offsets and varints instead of one per byte. (Buffers are padded so the chunk load never leaves them.)
struct ByteWin {
  const uint8_t* chunk;
  uint4 w;
  __device__ ByteWin() : chunk(nullptr), w(make_uint4(0, 0, 0, 0)) {}
  __device__ __forceinline__ uint32_t at(const uint8_t* p) {
    const uint8_t* c = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)15);
    if (c != chunk) { chunk = c; w = *reinterpret_cast<const uint4*>(c); }
    const uint32_t i = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 15);
    const uint32_t word = (i & 8u) ? ((i & 4u) ? w.w : w.z) : ((i & 4u) ? w.y : w.x);
    return (word >> ((i & 3u) * 8u)) & 0xffu;
  }
};

__device__ __forceinline__ uint32_t rd32le(const uint8_t* p) { return p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

struct Cur {   // zig-zag varints of org.apache.kafka.common.utils.ByteUtils over a byte range
  const uint8_t* p; uint64_t n, pos; bool ok;
  ByteWin win;
  __device__ Cur(const uint8_t* p_, uint64_t n_) : p(p_), n(n_), pos(0), ok(true) {}
  __device__ int64_t varlong() {
    unsigned long long v = 0; int shift = 0;
    for (int i = 0; i < 10; ++i) {
      if (pos >= n) { ok = false; return 0; }
      const uint8_t b = (uint8_t)win.at(p + pos++);
      v |= (unsigned long long)(b & 0x7f) << shift;
      if (!(b & 0x80)) return (int64_t)(v >> 1) ^ -(int64_t)(v & 1);
      shift += 7;
    }
    ok = false; return 0;
  }
  __device__ int32_t varint() {
    uint32_t v = 0; int shift = 0;
    for (int i = 0; i < 5; ++i) {
      if (pos >= n) { ok = false; return 0; }
      const uint8_t b = (uint8_t)win.at(p + pos++);
      v |= (uint32_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return (int32_t)(v >> 1) ^ -(int32_t)(v & 1);
      shift += 7;
    }
    ok = false; return 0;
  }
  __device__ const uint8_t* bytes(uint64_t k) {
    if (k > n - pos) { ok = false; return nullptr; }
    const uint8_t* r = p + pos; pos += k; return r;
  }
};

// ---------------------------------------------------------------------------------------------- CRC + size, decode + walk
constexpr int kFastThreads = 64;   // thread-per-batch kernels: small CTAs spread a group of a few thousand batches over all SMs
constexpr int kRingChunks = 8;     // 16-byte chunks per thread in the input ring

// Input policy of lz4_fast.h on the device: a private ring of eight 16-byte chunks per thread in shared memory, kept six
// chunks ahead of the read position by cp.async. An asynchronous copy has no destination register, so nobody stalls on it
// (a register prefetch does not survive SIMT: the scoreboard of a load's destination is per warp, and in a warp of 32 independent
// streams some lane touches that register name at every step). Streams are read front to back; buffers are padded by 256 bytes.
struct RingIn {
  uint32_t cell;            // shared-space address of this thread's 16 bytes in ring row 0
  const uint8_t* base;      // 16-byte aligned address of the chunk that holds the read position
  static constexpr uint32_t kRow = kFastThreads * 16;
  __device__ __forceinline__ void init(const uint4* ring_row0) {
    cell = (uint32_t)__cvta_generic_to_shared(ring_row0 + threadIdx.x);
    base = nullptr;
  }
  static __device__ __forceinline__ uint32_t slot_at(uint32_t cell, const uint8_t* chunk) { return cell + (((uint32_t)reinterpret_cast<uintptr_t>(chunk) >> 4) & (kRingChunks - 1)) * kRow; }
  __device__ __forceinline__ uint32_t slot_of(const uint8_t* chunk) const { return slot_at(cell, chunk); }
  static __device__ __forceinline__ void issue_at(uint32_t cell, const uint8_t* chunk) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n\tcp.async.commit_group;" ::"r"(slot_at(cell, chunk)), "l"(chunk) : "memory");
  }
  __device__ __forceinline__ void issue(const uint8_t* chunk) { issue_at(cell, chunk); }
  // (out of line and by value: the ring's state stays in registers, the eight requests are not replicated at every call site)
  static __device__ __noinline__ const uint8_t* seek_at(uint32_t cell, const uint8_t* p) {
    asm volatile("cp.async.wait_all;" ::: "memory");   // nothing of the previous stream may still land in the ring
    const uint8_t* b = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)15);
#pragma unroll
    for (int k = 0; k < kRingChunks; ++k) issue_at(cell, b + 16 * k);
    asm volatile("cp.async.wait_group %0;" ::"n"(kRingChunks - 2) : "memory");   // this chunk and the next have landed
    return b;
  }
  __device__ __forceinline__ void seek(const uint8_t* p) { base = seek_at(cell, p); }
  __device__ __forceinline__ void advance(const uint8_t* p) {   // afterwards base <= p < base + 16 and chunks base, base + 16 are readable
    if (p >= base + 16) {
      if (p >= base + 16 * kRingChunks) { seek(p); return; }
      // One chunk at a time, each followed by its wait: a request goes into the slot of the OLDEST chunk, and that slot's
      // previous request must have landed first — copies in flight complete in any order, and two of them aimed at one slot
      // would leave whichever arrives last. (Issuing k requests and waiting once was wrong for k >= 3: the third reuses a slot
      // whose copy may still be among the six allowed to be pending. Found on records of about 40 bytes; pinned by
      // test_forty_byte_records_walk_through_the_ring and modelled in tests/test_ring_protocol_model.py.)
      do {
        issue(base + 16 * kRingChunks); base += 16;
        asm volatile("cp.async.wait_group %0;" ::"n"(kRingChunks - 2) : "memory");
      } while (p >= base + 16);
    }
  }
  __device__ __forceinline__ unsigned long long word_at(const uint8_t* a8) const {   // a8 is 8-byte aligned, inside chunks base / base + 16
    unsigned long long v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(slot_of(a8) + ((uint32_t)reinterpret_cast<uintptr_t>(a8) & 8u)) : "memory");
    return v;
  }
  __device__ __forceinline__ uint64_t get64(const uint8_t* p) const {   // bytes p .. p+7, base <= p < base + 16
    const uint8_t* a = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)7);
    return lzf::funnel(word_at(a), word_at(a + 8), (uint32_t)reinterpret_cast<uintptr_t>(p) & 7u);
  }
};

// CRC-32C over a byte range read through the ring
__device__ uint32_t crc32c_ring(const uint32_t (*tab)[256], RingIn& in, const uint8_t* p, uint64_t n) {
  uint32_t crc = 0xffffffffu;
  if (!n) return ~crc;
  in.seek(p);
  while (n && ((uintptr_t)p & 7)) { crc = (crc >> 8) ^ tab[0][(crc ^ (uint32_t)in.get64(p)) & 0xff]; ++p; --n; in.advance(p); }
  while (n >= 8) {
    const unsigned long long w = in.get64(p);
    const uint32_t lo = (uint32_t)w ^ crc, hi = (uint32_t)(w >> 32);
    crc = tab[7][lo & 0xff] ^ tab[6][(lo >> 8) & 0xff] ^ tab[5][(lo >> 16) & 0xff] ^ tab[4][lo >> 24] ^
          tab[3][hi & 0xff] ^ tab[2][(hi >> 8) & 0xff] ^ tab[1][(hi >> 16) & 0xff] ^ tab[0][hi >> 24];
    p += 8; n -= 8;
    in.advance(p);
  }
  while (n) { crc = (crc >> 8) ^ tab[0][(crc ^ (uint32_t)in.get64(p)) & 0xff]; ++p; --n; in.advance(p); }
  return ~crc;
}

// arena_ctl (optional): [0] bytes claimed so far, [1] capacity, [2] set when a claim (or, later, a batch in its slot) did not fit.
// With it: CRC only, and every lz4 batch leaves the kernel with an arena slot of claim_mult x its compressed size. Without it: CRC
// and the exact decoded size (an lz4 walk that only adds up lengths); the host then lays the arena out.
__device__ __forceinline__ void crc_size_one(const uint32_t (*tab)[256], RingIn& in, const uint8_t* __restrict__ wire, DgBatch* __restrict__ batches, uint32_t i,
                                             unsigned long long* __restrict__ arena_ctl, uint32_t claim_mult) {
  const DgBatch bt = batches[i];
  const uint8_t* b = wire + bt.src_off;
  uint32_t err = DG_OK, dsize = bt.total_len - 61u;
  unsigned long long arena_off = 0;
  if (crc32c_ring(tab, in, b + 21, (uint64_t)bt.total_len - 21) != bt.stored_crc) err = DG_CRC;
  else if (bt.codec == 3) {
    if (arena_ctl) {
      // claim mode: no size walk. The slot is claim_mult x the compressed bytes (what the arena is sized for as a whole); a batch
      // that decodes to more reports DG_ARENA_FULL from the decode kernel and the poll is repeated from exact sizes.
      const unsigned long long cap = min((unsigned long long)claim_mult * (bt.total_len - 61u) + 64ull, 0xfffffff0ull);
      const unsigned long long need = (cap + 15ull) & ~15ull;
      dsize = (uint32_t)cap;   // (the slot's capacity until the decode kernel replaces it by the decoded size)
      arena_off = atomicAdd(arena_ctl + 0, need);
      if (arena_off + need > arena_ctl[1]) { arena_ctl[2] = 1ull; err = DG_ARENA_FULL; }
    } else {
      uint64_t len = 0;
      err = lzf::frame<false>(in, b + 61, (uint64_t)bt.total_len - 61, nullptr, 0, &len);
      if (!err && len > 0xffffffffull) err = DG_LZ4_TOO_LARGE;
      dsize = (uint32_t)len;
    }
  }
  if (!err && !(bt.codec == 3 && arena_ctl) && (uint64_t)bt.n_records > (uint64_t)dsize / 7 + 1) err = DG_RECORD_COUNT;   // every record is at least 7 bytes on the wire
  batches[i].dsize = dsize;
  if (arena_ctl) batches[i].arena_off = arena_off;
  batches[i].err = (uint16_t)err;
}

__global__ void __launch_bounds__(kFastThreads) dg_crc_size_fast_kernel(const uint8_t* __restrict__ wire, DgBatch* __restrict__ batches, uint32_t n,
                                                                        unsigned long long* __restrict__ arena_ctl, uint32_t claim_mult) {
  __shared__ uint32_t tab[8][256];
  __shared__ uint4 ring[kRingChunks][kFastThreads];
  for (int i = threadIdx.x; i < 8 * 256; i += kFastThreads) (&tab[0][0])[i] = (&g_crc_tab[0][0])[i];
  __syncthreads();
  const uint32_t i = blockIdx.x * kFastThreads + threadIdx.x;
  if (i >= n) return;
  RingIn in;
  in.init(&ring[0][0]);
  crc_size_one(tab, in, wire, batches, i, arena_ctl, claim_mult);
  asm volatile("cp.async.wait_all;" ::: "memory");   // chunks requested ahead of the last byte land before the CTA's memory goes
}

// one thread per batch: lz4 into the batch's arena slot, then the record-boundary walk (a chain of varints) over the decoded
// bytes, read back through the same ring three records ahead
__device__ __forceinline__ void decode_walk_one(RingIn& in, const uint8_t* __restrict__ wire, uint8_t* arena, DgBatch* __restrict__ batches, uint32_t i, uint32_t index_base,
                                                uint32_t* __restrict__ rec_off, uint32_t* __restrict__ rec_batch, unsigned long long* __restrict__ arena_ctl) {
  const DgBatch bt = batches[i];
  batches[i].rec_err = kNoRecErr;
  if (bt.err) return;
  const uint8_t* sect = wire + bt.src_off + 61;
  uint64_t sect_len = (uint64_t)bt.total_len - 61;
  if (bt.codec == 3) {
    uint64_t len = 0;
    const uint32_t e = lzf::frame<true>(in, sect, sect_len, arena + bt.arena_off, bt.dsize, &len);
    if (arena_ctl) {   // bt.dsize was the capacity of a claimed slot
      if (e == DG_LZ4_TOO_LARGE) { arena_ctl[2] = 1ull; batches[i].err = DG_ARENA_FULL; return; }   // (or a block past its maximum: the exact pass tells)
      if (e) { batches[i].err = (uint16_t)e; return; }
      if ((uint64_t)bt.n_records > len / 7 + 1) { batches[i].err = DG_RECORD_COUNT; return; }
      batches[i].dsize = (uint32_t)len;
    } else if (e || len != bt.dsize) { batches[i].err = (uint16_t)(e ? e : DG_LZ4_BLOCK); return; }
    sect = arena + bt.arena_off; sect_len = len;
  }
  in.seek(sect);
  uint64_t pos = 0;
  for (uint32_t r = 0; r < bt.n_records; ++r) {
    bool ok = pos < sect_len;
    uint32_t raw = 0, used = 0;
    if (ok) {
      in.advance(sect + pos);
      const unsigned long long v = in.get64(sect + pos);
      ok = false;
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const uint32_t byte = (uint32_t)(v >> (8 * k)) & 0xffu;
        raw |= (byte & 0x7fu) << (7 * k);
        if (!(byte & 0x80u)) { used = k + 1; ok = true; break; }
      }
      ok = ok && pos + used <= sect_len;
    }
    const int32_t len = (int32_t)(raw >> 1) ^ -(int32_t)(raw & 1u);
    if (!ok || len < 0 || (uint64_t)len > sect_len - (pos + used)) { batches[i].err = DG_RECORD_LENGTH; batches[i].rec_err = ((unsigned long long)r << 32) | DG_RECORD_LENGTH; return; }
    rec_off[bt.rec_base + r] = (uint32_t)pos; rec_batch[bt.rec_base + r] = index_base + i;
    pos += used + (uint64_t)len;
  }
  if (pos != sect_len) { batches[i].err = DG_STRAY_BYTES; batches[i].rec_err = ((unsigned long long)bt.n_records << 32) | DG_STRAY_BYTES; }
}

__global__ void __launch_bounds__(kFastThreads) dg_decode_walk_fast_kernel(const uint8_t* __restrict__ wire, uint8_t* arena, DgBatch* __restrict__ batches,
                                                                           uint32_t n, uint32_t index_base, uint32_t* __restrict__ rec_off, uint32_t* __restrict__ rec_batch,
                                                                           unsigned long long* __restrict__ arena_ctl) {
  __shared__ uint4 ring[kRingChunks][kFastThreads];
  const uint32_t i = blockIdx.x * kFastThreads + threadIdx.x;
  if (i >= n) return;
  RingIn in;
  in.init(&ring[0][0]);
  decode_walk_one(in, wire, arena, batches, i, index_base, rec_off, rec_batch, arena_ctl);
  asm volatile("cp.async.wait_all;" ::: "memory");
}

// ---- new ids -> contiguous bytes in dense-index order, for the host key table (lengths, [scan outside], copy)
__global__ void dg_key_lens_kernel(const uint2* __restrict__ key_ref, uint64_t from, uint32_t n, uint32_t* __restrict__ lens) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n) lens[i] = i < n ? key_ref[from + i].y : 0u;
}
__global__ void dg_key_copy_kernel(const uint2* __restrict__ key_ref, const uint8_t* __restrict__ arena, uint64_t from, uint32_t n,
                                   const uint32_t* __restrict__ offs, uint8_t* __restrict__ out) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 3, part = threadIdx.x & 7;   // 8 lanes per id
  if (i >= n) return;
  const uint2 ref = key_ref[from + i];
  const uint8_t* src = arena + ((unsigned long long)ref.x << 3);
  uint8_t* dst = out + offs[i];
  for (uint32_t k = part; k < ref.y; k += 8) dst[k] = src[k];
}

// A refused record leaves (index << 32) | reason in the batch's rec_err; the lowest index wins, whichever thread gets there
// first, as the host decoder reports the first bad record of a batch.
__device__ __forceinline__ void refuse_record(DgBatch& bt, uint32_t r, uint32_t code) {
  atomicMin(&bt.rec_err, ((unsigned long long)r << 32) | code);
}

// One live record of a compacted state topic at slot i: the id is the whole key (no cut at ':'), a null value is a tombstone,
// any other value (after its framing) is 0 .. row_bytes program bytes, zero-padded to the row. Counted as a record either way.
template <int32_t kFraming>
__device__ __forceinline__ void state_row(const DgParse& p, DgBatch& bt, uint32_t i, uint32_t r, const uint8_t* key, uint32_t key_len,
                                          const uint8_t* val, int32_t val_len) {
  uint8_t converted[vf::kStateRowMax];
  if constexpr (kFraming != vf::PACKED) {
    if (val_len >= 0) {
      uint32_t n = 0;
      const uint32_t why = vf::convert<vf::STATE>(kFraming, p.json, val, (uint32_t)val_len, converted, &val, &n);
      if (why) { refuse_record(bt, r, (uint32_t)DG_VALUE_FRAMING | (why << 8)); return; }
      val_len = kFraming == vf::PROTOBUF_EVENT ? (int32_t)n : (int32_t)p.row_bytes;   // (the member table was checked against the row)
    }
  }
  if (val_len > (int32_t)p.row_bytes) { refuse_record(bt, r, (uint32_t)DG_STATE_LENGTH | ((uint32_t)min(val_len, 0xffffff) << 8)); return; }
  if (key_len >= (1u << 24)) { refuse_record(bt, r, DG_ID_LENGTH); return; }
  const uint32_t idx = intern(p.dict, key, key_len);
  if (idx == 0xffffffffu) return;   // dictionary full: counted in ctl[5], the whole call fails
  if (val_len < 0) {
    p.present[i] = 0;
    atomicAdd(p.dict.ctl + 3, 1ull);
  } else {
    uint32_t* row = reinterpret_cast<uint32_t*>(p.out + (size_t)i * p.row_bytes);   // (row_bytes is a multiple of 4)
    for (uint32_t w = 0; w < p.row_bytes / 4; ++w) {
      uint32_t x = 0;
      for (uint32_t b = 0; b < 4; ++b) if (4 * w + b < (uint32_t)val_len) x |= (uint32_t)val[4 * w + b] << (8 * b);
      row[w] = x;
    }
    p.present[i] = 1;
  }
  p.idx[i] = idx;
  const uint32_t grp = __activemask();
  if ((threadIdx.x & 31) == (uint32_t)(__ffs(grp) - 1)) atomicAdd(p.dict.ctl + 6, (unsigned long long)__popc(grp));
}

// kFraming (SGR_VALUE_*): the packed instantiation copies the value as it is; the others convert it first (value_framing.h),
// after the null-value check and before the 8..56 length check, in the host decoder's order.
// kState (a compacted state topic, DgParse::state_topic): the record becomes a row of the program bytes, its dense index and a
// present byte instead of a packed event (state_row); the events instantiations compile as they did without it.
template <int32_t kFraming, bool kState>
__global__ void __launch_bounds__(kThreads) dg_parse_kernel(const __grid_constant__ DgParse p) {
  const uint32_t i = p.rec_begin + blockIdx.x * kThreads + threadIdx.x;
  if (i >= p.n_records) return;
  uint4* out = reinterpret_cast<uint4*>(p.out + (size_t)i * 64);
  if constexpr (kState) {
    p.idx[i] = ~0u;   // a hole until the record proves live
  } else {
    const uint4 zero = make_uint4(0, 0, 0, 0), hole = make_uint4(0, 0, 0xffffffffu, 0xffffffffu);
    out[1] = zero; out[2] = zero; out[3] = zero;
    out[0] = hole;
  }
  const uint32_t bi = p.rec_batch[i];
  if (bi >= p.n_batches) return;    // a slot the walk never reached (its batch failed earlier)
  DgBatch& bt = p.batches[bi];
  if (bt.err) return;
  const uint8_t* sect = bt.codec == 3 ? p.arena + bt.arena_off : p.wire + bt.src_off + 61;
  const uint32_t r = i - bt.rec_base;
  Cur c(sect + p.rec_off[i], (uint64_t)bt.dsize - p.rec_off[i]);
  const int32_t rec_len = c.varint();
  Cur q(sect + p.rec_off[i] + c.pos, (uint64_t)rec_len);   // the walk validated the length
  q.bytes(1);                 // record attributes (unused in v2)
  q.varlong();                // timestampDelta
  const int32_t offset_delta = q.varint();
  const int32_t key_len = q.varint();
  const uint8_t* key = key_len > 0 ? q.bytes((uint64_t)key_len) : nullptr;
  int32_t val_len = q.varint();
  const uint8_t* val = val_len > 0 ? q.bytes((uint64_t)val_len) : nullptr;
  const int32_t n_headers = q.varint();
  for (int32_t h = 0; q.ok && h < n_headers; ++h) {
    const int32_t hk = q.varint(); if (hk < 0) { q.ok = false; break; } q.bytes((uint64_t)hk);
    const int32_t hv = q.varint(); if (hv > 0) q.bytes((uint64_t)hv);
  }
  if (!q.ok || q.pos != q.n || n_headers < 0) { refuse_record(bt, r, DG_RECORD_MALFORMED); return; }
  if (bt.base_offset + offset_delta < bt.min_offset) { atomicAdd(p.dict.ctl + 4, 1ull); return; }      // refetch after a restart
  if (key_len <= 0) { atomicAdd(p.dict.ctl + 2, 1ull); return; }                                        // the producer's flush record
  if constexpr (kState) {
    state_row<kFraming>(p, bt, i, r, key, (uint32_t)key_len, val, val_len);
    return;
  }
  if (val_len < 0 && p.null_value_type < 0) { atomicAdd(p.dict.ctl + 3, 1ull); return; }
  uint8_t converted[56];
  if constexpr (kFraming != vf::PACKED) {
    if (val_len >= 0) {
      uint32_t n = 0;
      const uint32_t why = vf::convert(kFraming, p.json, val, (uint32_t)val_len, converted, &val, &n);
      if (why) { refuse_record(bt, r, (uint32_t)DG_VALUE_FRAMING | (why << 8)); return; }
      val_len = (int32_t)n;   // (a protobuf payload lies inside the value: at most 2^31 - 1 bytes)
    }
  }
  if (val_len >= 0 && (val_len < 8 || val_len > 56)) { refuse_record(bt, r, DG_VALUE_LENGTH); return; }
  uint32_t id_len = (uint32_t)key_len;
  for (uint32_t k = 0; k < (uint32_t)key_len; ++k) if (key[k] == ':') { id_len = k; break; }          // PartitionStringUpToColon
  if (id_len >= (1u << 24)) { refuse_record(bt, r, DG_ID_LENGTH); return; }
  const uint32_t idx = intern(p.dict, key, id_len);
  if (idx == 0xffffffffu) return;   // dictionary full: counted in ctl[5], the whole call fails
  uint32_t w[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) w[k] = 0;
  if (val_len < 0) { w[0] = (uint32_t)p.null_value_type; atomicAdd(p.dict.ctl + 3, 1ull); }
  else {
    w[0] = rd32le(val); w[1] = rd32le(val + 4);
    uint8_t* pay = reinterpret_cast<uint8_t*>(w + 4);
    for (int32_t k = 8; k < val_len; ++k) pay[k - 8] = val[k];
  }
  w[2] = idx; w[3] = 0;
  out[0] = make_uint4(w[0], w[1], w[2], w[3]); out[1] = make_uint4(w[4], w[5], w[6], w[7]);
  out[2] = make_uint4(w[8], w[9], w[10], w[11]); out[3] = make_uint4(w[12], w[13], w[14], w[15]);
  // one atomic per converged group of lanes, not per record: 3e7 atomics on one address serialise in the L2
  const uint32_t grp = __activemask();
  if ((threadIdx.x & 31) == (uint32_t)(__ffs(grp) - 1)) atomicAdd(p.dict.ctl + 6, (unsigned long long)__popc(grp));
}

}  // namespace

// descriptors host -> device by the SMs (zero-copy read of page-locked memory): the copy engine's queue is full of the poll's
// fetches, and a cudaMemcpyAsync for 512 KiB of descriptors would wait behind ALL of them
__global__ void dg_copy16_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, uint64_t n16) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (uint64_t)gridDim.x * blockDim.x) dst[i] = src[i];
}

cudaError_t dg_copy_from_mapped_host(const void* host_mapped, void* dst, uint64_t nbytes, cudaStream_t st) {
  if (!nbytes) return cudaSuccess;
  const uint64_t n16 = (nbytes + 15) / 16;
  const uint32_t blocks = (uint32_t)((n16 + 255) / 256 < 528 ? (n16 + 255) / 256 : 528);   // 4 CTAs on each of H100's 132 SMs
  dg_copy16_kernel<<<blocks, 256, 0, st>>>((const uint4*)host_mapped, (uint4*)dst, n16);
  return cudaGetLastError();
}

cudaError_t dg_prepare() { return ensure_crc_tables(); }

cudaError_t dg_launch_crc_size_fast(const uint8_t* wire, DgBatch* batches, uint32_t n, unsigned long long* arena_ctl, uint32_t claim_mult, cudaStream_t st) {
  cudaError_t e = ensure_crc_tables();
  if (e != cudaSuccess || !n) return e;
  dg_crc_size_fast_kernel<<<(n + kFastThreads - 1) / kFastThreads, kFastThreads, 0, st>>>(wire, batches, n, arena_ctl, claim_mult);
  return cudaGetLastError();
}

cudaError_t dg_launch_decode_walk_fast(const uint8_t* wire, uint8_t* arena, DgBatch* batches, uint32_t n, uint32_t index_base, uint32_t* rec_off, uint32_t* rec_batch,
                                       unsigned long long* arena_ctl, cudaStream_t st) {
  if (!n) return cudaSuccess;
  dg_decode_walk_fast_kernel<<<(n + kFastThreads - 1) / kFastThreads, kFastThreads, 0, st>>>(wire, arena, batches, n, index_base, rec_off, rec_batch, arena_ctl);
  return cudaGetLastError();
}

// ids [from, from + n) of the dictionary as contiguous bytes in dense-index order: d_offs[n + 1] (exclusive prefix of the lengths),
// d_bytes. scan_tmp: the scan's temp storage.
cudaError_t dg_gather_keys(const DgDict& d, uint64_t from, uint32_t n, uint32_t* d_offs, uint8_t* d_bytes, DevBuf& scan_tmp, cudaStream_t st) {
  if (!n) return cudaSuccess;
  dg_key_lens_kernel<<<(n + 1 + 255) / 256, 256, 0, st>>>(d.key_ref, from, n, d_offs);
  cudaError_t e = exclusive_sum_u32(d_offs, d_offs, n + 1, scan_tmp, st);
  if (e != cudaSuccess) return e;
  dg_key_copy_kernel<<<(uint32_t)(((uint64_t)n * 8 + 255) / 256), 256, 0, st>>>(d.key_ref, d.arena, from, n, d_offs, d_bytes);
  return cudaGetLastError();
}

cudaError_t dg_launch_parse(const DgParse& p, cudaStream_t st) {
  if (p.n_records <= p.rec_begin) return cudaSuccess;
  const uint32_t blocks = (p.n_records - p.rec_begin + kThreads - 1) / kThreads;
  // (framing, topic mode) -> one instantiation: the framing in bits 0..1, the state-topic mode in bit 2
  switch (p.value_framing | (p.state_topic ? 4 : 0)) {
    case vf::PACKED: dg_parse_kernel<vf::PACKED, false><<<blocks, kThreads, 0, st>>>(p); break;
    case vf::PROTOBUF_EVENT: dg_parse_kernel<vf::PROTOBUF_EVENT, false><<<blocks, kThreads, 0, st>>>(p); break;
    case vf::JSON: dg_parse_kernel<vf::JSON, false><<<blocks, kThreads, 0, st>>>(p); break;
    case vf::PROTOBUF_JSON: dg_parse_kernel<vf::PROTOBUF_JSON, false><<<blocks, kThreads, 0, st>>>(p); break;
    case 4 | vf::PACKED: dg_parse_kernel<vf::PACKED, true><<<blocks, kThreads, 0, st>>>(p); break;
    case 4 | vf::PROTOBUF_EVENT: dg_parse_kernel<vf::PROTOBUF_EVENT, true><<<blocks, kThreads, 0, st>>>(p); break;
    case 4 | vf::JSON: dg_parse_kernel<vf::JSON, true><<<blocks, kThreads, 0, st>>>(p); break;
    case 4 | vf::PROTOBUF_JSON: dg_parse_kernel<vf::PROTOBUF_JSON, true><<<blocks, kThreads, 0, st>>>(p); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace sgr
