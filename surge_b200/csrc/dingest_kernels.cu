// dingest_kernels.cu — Kafka RecordBatch v2 decode ON THE DEVICE (sm_90a): the step right before the fold (SURVEY §8 f1).
//
// What feeds the store today is a read_committed consumer of a topic whose producer compresses with lz4
// (modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:38; modules/common/src/main/resources/
// reference.conf:124). Round 1 decoded those bytes on the host (csrc/ingest.cpp) and copied 64-byte packed records over PCIe —
// the copy was 95 % of the end-to-end step. Here the WIRE bytes cross PCIe (about 25 B per event instead of 64) and everything
// per-batch and per-record happens on the GPU; the host keeps only the walk over the 61-byte batch headers and the
// read_committed bookkeeping (csrc/dingest.cu). csrc/ingest.cpp stays as the byte-equal checker (tests/test_gpu_dingest.py).
//
//   crc_size    one THREAD per batch: CRC-32C of the batch (slicing-by-8, tables in shared memory) against the header's field;
//               lz4 frames: header + block walk that only ADDS UP sequence lengths -> decompressed size (the arena is then laid
//               out by an exclusive scan on the host: 4 bytes per batch come back)
//   decode_walk one thread per batch: lz4 sequences copied into the batch's arena slot (byte-serial by nature: matches may
//               overlap their own output), then the record-boundary walk — a chain of varints — writes every record's offset
//   parse       one thread per RECORD: varint fields, key -> aggregate id (up to ':', KafkaPartitioner.scala:38-42), value ->
//               packed 64-byte record at the record's own slot (arrival order kept), id -> dense index through a device hash
//               table (64-bit hash tag claimed by CAS, id bytes compared, index from an atomic counter)
// Records a read_committed consumer would not deliver (flush markers, duplicates below the partition position, dropped null
// values) become HOLES (agg == ~0) that the fold kernels skip; nothing is compacted.
//
// Thread-per-batch is deliberate: a 16 KiB producer batch is ~2 k lz4 sequences and ~500 varint-delimited records, strictly
// serial inside; the parallelism is the tens of thousands of batches of a restore poll. All of it is HBM/latency-bound
// byte work — no tensor cores anywhere.
//
// Two generations live here. The first (dg_crc_size_kernel, dg_decode_walk_kernel; SGR_DINGEST_V1=1 selects it) walks the bytes
// through global memory and spends the same time on the decode of ANY number of batches: ~10 dependent memory round trips per lz4
// sequence, and in a warp of 32 independent batches some lane misses at every step. The second (the *_fast kernels, default)
// reads its input through a per-thread cp.async ring in shared memory and keeps memory current behind an 8-byte output
// accumulator (lz4_fast.h) — one dependent access per sequence — and claims each batch's arena slot with an atomicAdd in the size pass, so that CRC -> decode -> parse of a group of batches is one chain of launches with
// no host round trip in between (csrc/dingest.cu runs such chains on several streams behind the H2D copies).
#include "dingest_kernels.cuh"
#include "lz4_fast.h"

#include <stdlib.h>
#include <string.h>

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

__device__ uint32_t crc32c_dev(const uint32_t (*tab)[256], const uint8_t* p, uint64_t n) {
  uint32_t crc = 0xffffffffu;
  while (n && ((uintptr_t)p & 7)) { crc = (crc >> 8) ^ tab[0][(crc ^ *p++) & 0xff]; --n; }
  while (n >= 8) {
    const unsigned long long w = *reinterpret_cast<const unsigned long long*>(p);
    const uint32_t lo = (uint32_t)w ^ crc, hi = (uint32_t)(w >> 32);
    crc = tab[7][lo & 0xff] ^ tab[6][(lo >> 8) & 0xff] ^ tab[5][(lo >> 16) & 0xff] ^ tab[4][lo >> 24] ^
          tab[3][hi & 0xff] ^ tab[2][(hi >> 8) & 0xff] ^ tab[1][(hi >> 16) & 0xff] ^ tab[0][hi >> 24];
    p += 8; n -= 8;
  }
  while (n--) crc = (crc >> 8) ^ tab[0][(crc ^ *p++) & 0xff];
  return ~crc;
}

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__device__ uint32_t xxh32_dev(const uint8_t* p, uint64_t len, uint32_t seed) {
  const uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
  const uint8_t* end = p + len;
  uint32_t h;
  if (len >= 16) {
    const uint8_t* limit = end - 16;
    uint32_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
    do {
      v1 = rotl32(v1 + rd32le(p) * P2, 13) * P1; p += 4;
      v2 = rotl32(v2 + rd32le(p) * P2, 13) * P1; p += 4;
      v3 = rotl32(v3 + rd32le(p) * P2, 13) * P1; p += 4;
      v4 = rotl32(v4 + rd32le(p) * P2, 13) * P1; p += 4;
    } while (p <= limit);
    h = rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18);
  } else {
    h = seed + P5;
  }
  h += (uint32_t)len;
  while (p + 4 <= end) { h = rotl32(h + rd32le(p) * P3, 17) * P4; p += 4; }
  while (p < end) { h = rotl32(h + (*p++) * P5, 11) * P1; }
  h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
  return h;
}

// dst[0..n) = src[0..n) for one thread, 4 bytes per memory instruction: aligned word stores, aligned word loads funnel-shifted
// to the source's misalignment (a GPU has no unaligned accesses). The regions must not overlap within 8 bytes (the caller sends
// close overlapping matches down the byte path). Byte-wise copies were the bulk of the decode: every byte access of every thread
// is an L1 wavefront of its own.
__device__ __forceinline__ void copy_words(uint8_t* dst, const uint8_t* src, uint64_t n) {
  uint64_t k = 0;
  while (k < n && ((uintptr_t)(dst + k) & 3)) { dst[k] = src[k]; ++k; }
  if (n - k >= 4) {
    const uint8_t* s = src + k;
    const uint32_t mis = (uint32_t)((uintptr_t)s & 3);
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(s - mis);
    uint32_t* dw = reinterpret_cast<uint32_t*>(dst + k);
    const uint64_t words = (n - k) >> 2;
    if (mis == 0) {
      for (uint64_t w = 0; w < words; ++w) dw[w] = sw[w];
    } else {
      uint32_t lo = sw[0];
      for (uint64_t w = 0; w < words; ++w) { const uint32_t hi = sw[w + 1]; dw[w] = __funnelshift_r(lo, hi, mis * 8); lo = hi; }
    }
    k += words << 2;
  }
  while (k < n) { dst[k] = src[k]; ++k; }
}

// LZ4 frame walk. out == nullptr: only the decoded size is computed (and everything validated except the content checksum).
// Mirrors lz4_frame_decode of csrc/ingest.cpp decision for decision (same accept / reject behaviour).
// `lane`/`lanes`: every participating thread runs the SAME control flow over the same compressed bytes (broadcast loads) and copies
// its share of every literal run and match (bytes lane, lane + lanes, ...): one thread (0, 1) for the size pass, a whole warp
// (lane, 32) for the decode — 32 consecutive bytes per step, coalesced. An overlapping match (offset < length) repeats its last
// `offset` bytes, so byte k of the match is byte (k mod offset) of that period: independent per byte, no serial dependency.
__device__ uint32_t lz4_frame(const uint8_t* src, uint64_t n, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint32_t lane = 0, uint32_t lanes = 1) {
  if (n < 7) return DG_LZ4_HEADER;
  if (rd32le(src) != 0x184D2204u) return DG_LZ4_HEADER;
  const uint8_t flg = src[4], bd = src[5];
  if ((flg >> 6) != 1 || (flg & 0x02)) return DG_LZ4_HEADER;
  const bool block_checksum = flg & 0x10, content_size = flg & 0x08, content_checksum = flg & 0x04, dict_id = flg & 0x01;
  const uint32_t bs_code = (bd >> 4) & 7;
  if (bs_code < 4 || (bd & 0x8F)) return DG_LZ4_HEADER;
  const uint64_t max_block = 1ull << (8 + 2 * bs_code);
  const uint64_t desc_len = 2 + (content_size ? 8 : 0) + (dict_id ? 4 : 0);
  if (n < 4 + desc_len + 1) return DG_LZ4_HEADER;
  uint64_t declared = 0;
  if (content_size) for (int k = 7; k >= 0; --k) declared = (declared << 8) | src[6 + k];
  if (((xxh32_dev(src + 4, desc_len, 0) >> 8) & 0xff) != src[4 + desc_len]) return DG_LZ4_HEADER;
  uint64_t pos = 4 + desc_len + 1, op = 0;
  for (;;) {
    if (pos + 4 > n) return DG_LZ4_BLOCK;
    const uint32_t word = rd32le(src + pos); pos += 4;
    if (word == 0) break;
    const bool stored = word & 0x80000000u;
    const uint64_t bsz = word & 0x7FFFFFFFu;
    if (bsz > max_block) return DG_LZ4_BLOCK;
    if (pos + bsz + (block_checksum ? 4 : 0) > n) return DG_LZ4_BLOCK;
    const uint8_t* b = src + pos;
    if (block_checksum && xxh32_dev(b, bsz, 0) != rd32le(b + bsz)) return DG_LZ4_CHECKSUM;
    if (stored) {
      if (out) {
        if (op + bsz > out_cap) return DG_LZ4_TOO_LARGE;
        if (lanes == 1) copy_words(out + op, b, bsz);
        else { for (uint64_t k = lane; k < bsz; k += lanes) out[op + k] = b[k]; __syncwarp(); }
      }
      op += bsz;
    } else {
      const uint64_t block_start = op;
      uint64_t ip = 0;
      ByteWin win;
      for (;;) {
        if (ip >= bsz) return DG_LZ4_SEQUENCE;
        const uint8_t token = (uint8_t)win.at(b + ip++);
        uint64_t lit = token >> 4;
        if (lit == 15) {
          uint8_t s;
          do { if (ip >= bsz) return DG_LZ4_SEQUENCE; s = (uint8_t)win.at(b + ip++); lit += s; } while (s == 255);
        }
        if (lit > bsz - ip) return DG_LZ4_SEQUENCE;
        if (op - block_start + lit > max_block) return DG_LZ4_TOO_LARGE;
        if (out) {
          if (op + lit > out_cap) return DG_LZ4_TOO_LARGE;
          if (lanes == 1) copy_words(out + op, b + ip, lit);
          else for (uint64_t k = lane; k < lit; k += lanes) out[op + k] = b[ip + k];
        }
        op += lit; ip += lit;
        if (ip == bsz) break;   // the last sequence carries literals only
        if (ip + 2 > bsz) return DG_LZ4_SEQUENCE;
        const uint32_t off = win.at(b + ip) | (win.at(b + ip + 1) << 8); ip += 2;
        uint64_t mlen = token & 15;
        if (mlen == 15) {
          uint8_t s;
          do { if (ip >= bsz) return DG_LZ4_SEQUENCE; s = (uint8_t)win.at(b + ip++); mlen += s; } while (s == 255);
        }
        mlen += 4;
        if (off == 0 || off > op) return DG_LZ4_SEQUENCE;   // matches may reach back across blocks, never before the frame
        if (op - block_start + mlen > max_block) return DG_LZ4_TOO_LARGE;
        if (out) {
          if (op + mlen > out_cap) return DG_LZ4_TOO_LARGE;
          if (lanes > 1) __syncwarp();                                  // the literals (and earlier matches) this match may read
          const uint8_t* period = out + op - off;
          if (lanes == 1 && off >= 8) {
            // a far match never reads a word it has not finished writing when copied in pieces of at most `off` bytes
            for (uint64_t done = 0; done < mlen; done += off) copy_words(out + op + done, period + done, mlen - done < off ? mlen - done : off);
          } else {
            for (uint64_t k = lane; k < mlen; k += lanes) out[op + k] = period[off >= mlen ? k : k % off];
          }
          if (lanes > 1) __syncwarp();
        }
        op += mlen;
      }
    }
    pos += bsz + (block_checksum ? 4 : 0);
  }
  if (content_checksum) {
    if (pos + 4 > n) return DG_LZ4_BLOCK;
    if (out && lanes > 1) __syncwarp();
    if (out && xxh32_dev(out, op, 0) != rd32le(src + pos)) return DG_LZ4_CHECKSUM;
    pos += 4;
  }
  if (content_size && declared != op) return DG_LZ4_BLOCK;
  *out_len = op;
  return DG_OK;
}

__global__ void __launch_bounds__(kThreads) dg_crc_size_kernel(const uint8_t* __restrict__ wire, DgBatch* __restrict__ batches, uint32_t n) {
  __shared__ uint32_t tab[8][256];
  for (int i = threadIdx.x; i < 8 * 256; i += kThreads) (&tab[0][0])[i] = (&g_crc_tab[0][0])[i];
  __syncthreads();
  const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  DgBatch bt = batches[i];
  const uint8_t* b = wire + bt.src_off;
  uint32_t err = DG_OK, dsize = bt.total_len - 61u;
  if (crc32c_dev(tab, b + 21, (uint64_t)bt.total_len - 21) != bt.stored_crc) err = DG_CRC;
  else if (bt.codec == 3) {
    uint64_t len = 0;
    err = lz4_frame(b + 61, (uint64_t)bt.total_len - 61, nullptr, 0, &len);
    if (!err && len > 0xffffffffull) err = DG_LZ4_TOO_LARGE;
    dsize = (uint32_t)len;
  }
  if (!err && (uint64_t)bt.n_records > (uint64_t)dsize / 7 + 1) err = DG_RECORD_COUNT;   // every record is at least 7 bytes on the wire
  batches[i].dsize = dsize;
  batches[i].err = err;
  batches[i].err_record = 0;
}

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

// one WARP per batch: cooperative lz4 copies, then the (serial) record-boundary walk run redundantly by all lanes — same loads,
// broadcast — with the writes spread over the lanes
template <int WARP>
__global__ void __launch_bounds__(kThreads) dg_decode_walk_kernel(const uint8_t* __restrict__ wire, uint8_t* __restrict__ arena, DgBatch* __restrict__ batches,
                                                                  uint32_t n, uint32_t index_base, uint32_t* __restrict__ rec_off, uint32_t* __restrict__ rec_batch) {
  // WARP == 1: one warp per batch (cooperative copies); 0: one thread per batch (word-wise copies, 32x more batches in flight —
  // for 16 KiB producer batches, where the token chain, not the copy width, is the latency)
  const uint32_t i = WARP ? (blockIdx.x * kThreads + threadIdx.x) >> 5 : blockIdx.x * kThreads + threadIdx.x;
  const uint32_t lane = WARP ? threadIdx.x & 31 : 0;
  if (i >= n) return;
  DgBatch bt = batches[i];
  if (bt.err) return;
  const uint8_t* sect = wire + bt.src_off + 61;
  uint64_t sect_len = (uint64_t)bt.total_len - 61;
  if (bt.codec == 3) {
    uint64_t len = 0;
    const uint32_t e = lz4_frame(sect, sect_len, arena + bt.arena_off, bt.dsize, &len, lane, WARP ? 32 : 1);
    if (WARP) __syncwarp();
    if (e || len != bt.dsize) { if (lane == 0) batches[i].err = e ? e : DG_LZ4_BLOCK; return; }
    sect = arena + bt.arena_off; sect_len = len;
  }
  Cur c(sect, sect_len);
  for (uint32_t r = 0; r < bt.n_records; ++r) {
    const uint64_t at = c.pos;
    const int32_t len = c.varint();
    if (!c.ok || len < 0 || (uint64_t)len > sect_len - c.pos) { if (lane == 0) { batches[i].err = DG_RECORD_LENGTH; batches[i].err_record = r; } return; }
    if (!WARP || lane == (r & 31u)) { rec_off[bt.rec_base + r] = (uint32_t)at; rec_batch[bt.rec_base + r] = index_base + i; }
    c.pos += (uint64_t)len;
  }
  if (c.pos != sect_len && lane == 0) { batches[i].err = DG_STRAY_BYTES; batches[i].err_record = bt.n_records; }
}

// ---------------------------------------------------------------------------------------------- second generation
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
      // whose copy may still be among the six allowed to be pending. Found by the 40-byte records of scripts/dingest_race.py.)
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

// The same interface over plain global loads (two aligned 8-byte words per read): the A/B partner of the ring
// (SGR_DINGEST_DEBUG bit 1: record walk, bit 2: CRC + lz4 input) — every read is a dependent round trip.
struct DirectIn {
  __device__ __forceinline__ void seek(const uint8_t*) {}
  __device__ __forceinline__ void advance(const uint8_t*) {}
  __device__ __forceinline__ uint64_t get64(const uint8_t* p) const {
    const uint8_t* a = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)7);
    return lzf::funnel(__ldcg(reinterpret_cast<const unsigned long long*>(a)), __ldcg(reinterpret_cast<const unsigned long long*>(a + 8)), (uint32_t)reinterpret_cast<uintptr_t>(p) & 7u);
  }
};

__device__ uint32_t g_dbg_flags = 0;   // SGR_DINGEST_DEBUG: 1 walk without the ring, 2 CRC + lz4 input without the ring, 4 match sources bypass L1, 8 fence before the walk

// CRC-32C over a byte range read through the ring
template <class IN>
__device__ uint32_t crc32c_ring(const uint32_t (*tab)[256], IN& in, const uint8_t* p, uint64_t n) {
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
// With it: CRC only, and every lz4 batch leaves the kernel with an arena slot of 3x its compressed size. Without it: CRC and the
// exact decoded size (an lz4 walk that only adds up lengths); the host then lays the arena out.
template <class IN>
__device__ __forceinline__ void crc_size_one(const uint32_t (*tab)[256], IN& in, const uint8_t* __restrict__ wire, DgBatch* __restrict__ batches, uint32_t i,
                                             unsigned long long* __restrict__ arena_ctl) {
  const DgBatch bt = batches[i];
  const uint8_t* b = wire + bt.src_off;
  uint32_t err = DG_OK, dsize = bt.total_len - 61u;
  unsigned long long arena_off = 0;
  if (crc32c_ring(tab, in, b + 21, (uint64_t)bt.total_len - 21) != bt.stored_crc) err = DG_CRC;
  else if (bt.codec == 3) {
    if (arena_ctl) {
      // claim mode: no size walk. The slot is 3x the compressed bytes (what the arena is sized for as a whole); a batch that
      // decodes to more reports DG_ARENA_FULL from the decode kernel and the poll is repeated from exact sizes.
      const unsigned long long cap = min(3ull * (bt.total_len - 61u) + 64ull, 0xfffffff0ull);
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
  batches[i].err = err;
  batches[i].err_record = 0;
}

__global__ void __launch_bounds__(kFastThreads) dg_crc_size_fast_kernel(const uint8_t* __restrict__ wire, DgBatch* __restrict__ batches, uint32_t n,
                                                                        unsigned long long* __restrict__ arena_ctl) {
  __shared__ uint32_t tab[8][256];
  __shared__ uint4 ring[kRingChunks][kFastThreads];
  for (int i = threadIdx.x; i < 8 * 256; i += kFastThreads) (&tab[0][0])[i] = (&g_crc_tab[0][0])[i];
  __syncthreads();
  const uint32_t i = blockIdx.x * kFastThreads + threadIdx.x;
  if (i >= n) return;
  RingIn in;
  in.init(&ring[0][0]);
  if (g_dbg_flags & 2u) { DirectIn din; crc_size_one(tab, din, wire, batches, i, arena_ctl); }
  else crc_size_one(tab, in, wire, batches, i, arena_ctl);
  asm volatile("cp.async.wait_all;" ::: "memory");   // chunks requested ahead of the last byte land before the CTA's memory goes
}

// one thread per batch: lz4 into the batch's arena slot, then the record-boundary walk (a chain of varints) over the decoded
// bytes, read back through the same ring three records ahead
template <class IN, class WIN>
__device__ __forceinline__ void decode_walk_one(IN& lzin, WIN& in, const uint8_t* __restrict__ wire, uint8_t* arena, DgBatch* __restrict__ batches, uint32_t i, uint32_t index_base,
                                                uint32_t* __restrict__ rec_off, uint32_t* __restrict__ rec_batch, unsigned long long* __restrict__ arena_ctl) {
  const DgBatch bt = batches[i];
  if (bt.err) return;
  const uint8_t* sect = wire + bt.src_off + 61;
  uint64_t sect_len = (uint64_t)bt.total_len - 61;
  if (bt.codec == 3) {
    uint64_t len = 0;
    const uint32_t e = lzf::frame<true>(lzin, sect, sect_len, arena + bt.arena_off, bt.dsize, &len, (g_dbg_flags & 4u) != 0);
    if (g_dbg_flags & 8u) __threadfence();
    if (arena_ctl) {   // bt.dsize was the capacity of a claimed slot
      if (e == DG_LZ4_TOO_LARGE) { arena_ctl[2] = 1ull; batches[i].err = DG_ARENA_FULL; return; }   // (or a block past its maximum: the exact pass tells)
      if (e) { batches[i].err = e; return; }
      if ((uint64_t)bt.n_records > len / 7 + 1) { batches[i].err = DG_RECORD_COUNT; return; }
      batches[i].dsize = (uint32_t)len;
    } else if (e || len != bt.dsize) { batches[i].err = e ? e : DG_LZ4_BLOCK; return; }
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
    if (!ok || len < 0 || (uint64_t)len > sect_len - (pos + used)) {
      uint32_t diag = 0;
      if (g_dbg_flags & 16u) {   // diagnosis: does the same walk over plain L2 loads succeed? (bit 31: yes -> the ring served stale bytes)
        DirectIn d; uint64_t q = 0; bool fine = true;
        for (uint32_t r2 = 0; r2 < bt.n_records && fine; ++r2) {
          if (q >= sect_len) { fine = false; break; }
          const unsigned long long v2 = d.get64(sect + q);
          uint32_t raw2 = 0, used2 = 0; bool t = false;
          for (int k = 0; k < 5; ++k) { const uint32_t byte = (uint32_t)(v2 >> (8 * k)) & 0xffu; raw2 |= (byte & 0x7fu) << (7 * k); if (!(byte & 0x80u)) { used2 = k + 1; t = true; break; } }
          const int32_t l2 = (int32_t)(raw2 >> 1) ^ -(int32_t)(raw2 & 1u);
          if (!t || l2 < 0 || q + used2 > sect_len || (uint64_t)l2 > sect_len - (q + used2)) fine = false; else q += used2 + (uint64_t)l2;
        }
        if (fine && q == sect_len) diag = 0x80000000u;
        diag |= ((uint32_t)pos & 0xfffffu) << 8;
      }
      batches[i].err = DG_RECORD_LENGTH; batches[i].err_record = r | diag; return;
    }
    rec_off[bt.rec_base + r] = (uint32_t)pos; rec_batch[bt.rec_base + r] = index_base + i;
    pos += used + (uint64_t)len;
  }
  if (pos != sect_len) { batches[i].err = DG_STRAY_BYTES; batches[i].err_record = bt.n_records; }
}

__global__ void __launch_bounds__(kFastThreads) dg_decode_walk_fast_kernel(const uint8_t* __restrict__ wire, uint8_t* arena, DgBatch* __restrict__ batches,
                                                                           uint32_t n, uint32_t index_base, uint32_t* __restrict__ rec_off, uint32_t* __restrict__ rec_batch,
                                                                           unsigned long long* __restrict__ arena_ctl) {
  __shared__ uint4 ring[kRingChunks][kFastThreads];
  const uint32_t i = blockIdx.x * kFastThreads + threadIdx.x;
  if (i >= n) return;
  RingIn in;
  in.init(&ring[0][0]);
  const uint32_t dbg = g_dbg_flags;
  DirectIn din;
  if ((dbg & 3u) == 0u) decode_walk_one(in, in, wire, arena, batches, i, index_base, rec_off, rec_batch, arena_ctl);
  else if ((dbg & 3u) == 1u) decode_walk_one(in, din, wire, arena, batches, i, index_base, rec_off, rec_batch, arena_ctl);
  else if ((dbg & 3u) == 2u) decode_walk_one(din, in, wire, arena, batches, i, index_base, rec_off, rec_batch, arena_ctl);
  else decode_walk_one(din, din, wire, arena, batches, i, index_base, rec_off, rec_batch, arena_ctl);
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
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

// id -> dense index. Returns 0xffffffff when the dictionary is full (the call then fails as a whole).
__device__ uint32_t intern(const DgDict& d, const uint8_t* id, uint32_t len) {
  const unsigned long long h = hash_id(id, len);
  uint64_t pos = h & d.slots_mask;
  for (uint64_t probes = 0; probes <= d.slots_mask; ++probes, pos = (pos + 1) & d.slots_mask) {
    unsigned long long tag = __ldcg(d.tags + pos);
    if (tag == 0ull) {
      tag = atomicCAS(d.tags + pos, 0ull, h);
      if (tag == 0ull) {   // this thread owns the slot: the id is new
        const unsigned long long idx = atomicAdd(d.ctl + 0, 1ull);
        const unsigned long long need = ((unsigned long long)len + 7) & ~7ull;
        const unsigned long long off = atomicAdd(d.ctl + 1, need);
        if (idx >= d.max_keys || off + need > d.arena_cap) {
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
    if (v == 0xffffffffu) return 0xffffffffu;
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

__global__ void __launch_bounds__(kThreads) dg_parse_kernel(const __grid_constant__ DgParse p) {
  const uint32_t i = p.rec_begin + blockIdx.x * kThreads + threadIdx.x;
  if (i >= p.n_records) return;
  uint4* out = reinterpret_cast<uint4*>(p.out + (size_t)i * 64);
  const uint4 zero = make_uint4(0, 0, 0, 0), hole = make_uint4(0, 0, 0xffffffffu, 0xffffffffu);
  out[1] = zero; out[2] = zero; out[3] = zero;
  out[0] = hole;
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
  const int32_t val_len = q.varint();
  const uint8_t* val = val_len > 0 ? q.bytes((uint64_t)val_len) : nullptr;
  const int32_t n_headers = q.varint();
  for (int32_t h = 0; q.ok && h < n_headers; ++h) {
    const int32_t hk = q.varint(); if (hk < 0) { q.ok = false; break; } q.bytes((uint64_t)hk);
    const int32_t hv = q.varint(); if (hv > 0) q.bytes((uint64_t)hv);
  }
  if (!q.ok || q.pos != q.n || n_headers < 0) { if (atomicCAS(&bt.err, 0u, (uint32_t)DG_RECORD_MALFORMED) == 0u) bt.err_record = r; return; }
  if (bt.base_offset + offset_delta < bt.min_offset) { atomicAdd(p.dict.ctl + 4, 1ull); return; }      // refetch after a restart
  if (key_len <= 0) { atomicAdd(p.dict.ctl + 2, 1ull); return; }                                        // the producer's flush record
  if (val_len < 0 && p.null_value_type < 0) { atomicAdd(p.dict.ctl + 3, 1ull); return; }
  if (val_len >= 0 && (val_len < 8 || val_len > 56)) { if (atomicCAS(&bt.err, 0u, (uint32_t)DG_VALUE_LENGTH) == 0u) bt.err_record = r; return; }
  uint32_t id_len = (uint32_t)key_len;
  for (uint32_t k = 0; k < (uint32_t)key_len; ++k) if (key[k] == ':') { id_len = k; break; }          // PartitionStringUpToColon
  if (id_len >= (1u << 24)) { if (atomicCAS(&bt.err, 0u, (uint32_t)DG_ID_LENGTH) == 0u) bt.err_record = r; return; }
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

uint32_t dg_crc32c_host_reference_polynomial() { return 0x82F63B78u; }

cudaError_t dg_launch_crc_size(const uint8_t* wire, DgBatch* batches, uint32_t n, cudaStream_t st) {
  cudaError_t e = ensure_crc_tables();
  if (e != cudaSuccess || !n) return e;
  dg_crc_size_kernel<<<(n + kThreads - 1) / kThreads, kThreads, 0, st>>>(wire, batches, n);
  return cudaGetLastError();
}

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

cudaError_t dg_prepare() {
  cudaError_t e = ensure_crc_tables();
  if (e != cudaSuccess) return e;
  const char* d = getenv("SGR_DINGEST_DEBUG");
  const uint32_t flags = d ? (uint32_t)atoi(d) : 0u;
  return cudaMemcpyToSymbol(g_dbg_flags, &flags, sizeof flags);
}

cudaError_t dg_launch_crc_size_fast(const uint8_t* wire, DgBatch* batches, uint32_t n, unsigned long long* arena_ctl, cudaStream_t st) {
  cudaError_t e = ensure_crc_tables();
  if (e != cudaSuccess || !n) return e;
  dg_crc_size_fast_kernel<<<(n + kFastThreads - 1) / kFastThreads, kFastThreads, 0, st>>>(wire, batches, n, arena_ctl);
  return cudaGetLastError();
}

cudaError_t dg_launch_decode_walk_fast(const uint8_t* wire, uint8_t* arena, DgBatch* batches, uint32_t n, uint32_t index_base, uint32_t* rec_off, uint32_t* rec_batch,
                                       unsigned long long* arena_ctl, cudaStream_t st) {
  if (!n) return cudaSuccess;
  dg_decode_walk_fast_kernel<<<(n + kFastThreads - 1) / kFastThreads, kFastThreads, 0, st>>>(wire, arena, batches, n, index_base, rec_off, rec_batch, arena_ctl);
  return cudaGetLastError();
}

cudaError_t dg_launch_decode_walk(const uint8_t* wire, uint8_t* arena, DgBatch* batches, uint32_t n, uint32_t index_base, uint32_t* rec_off, uint32_t* rec_batch, cudaStream_t st) {
  if (!n) return cudaSuccess;
  static const bool warp_mode = getenv("SGR_DINGEST_WARP_DECODE") != nullptr;
  if (warp_mode) {
    const uint32_t warps_per_block = kThreads / 32;
    dg_decode_walk_kernel<1><<<(n + warps_per_block - 1) / warps_per_block, kThreads, 0, st>>>(wire, arena, batches, n, index_base, rec_off, rec_batch);
  } else {
    dg_decode_walk_kernel<0><<<(n + kThreads - 1) / kThreads, kThreads, 0, st>>>(wire, arena, batches, n, index_base, rec_off, rec_batch);
  }
  return cudaGetLastError();
}

cudaError_t exclusive_scan_u32_public(const uint32_t* in, uint32_t* out, uint32_t n, uint32_t* tmp, cudaStream_t st);

// ids [from, from + n) of the dictionary as contiguous bytes in dense-index order: d_offs[n + 1] (exclusive prefix of the lengths),
// d_bytes. d_tmp: scratch of at least 2 * (n / 4096 + 2) + 4 * 4096 u32.
cudaError_t dg_gather_keys(const DgDict& d, uint64_t from, uint32_t n, uint32_t* d_offs, uint8_t* d_bytes, uint32_t* d_tmp, cudaStream_t st) {
  if (!n) return cudaSuccess;
  dg_key_lens_kernel<<<(n + 1 + 255) / 256, 256, 0, st>>>(d.key_ref, from, n, d_offs);
  cudaError_t e = exclusive_scan_u32_public(d_offs, d_offs, n + 1, d_tmp, st);
  if (e != cudaSuccess) return e;
  dg_key_copy_kernel<<<(uint32_t)(((uint64_t)n * 8 + 255) / 256), 256, 0, st>>>(d.key_ref, d.arena, from, n, d_offs, d_bytes);
  return cudaGetLastError();
}

cudaError_t dg_launch_parse(const DgParse& p, cudaStream_t st) {
  if (p.n_records <= p.rec_begin) return cudaSuccess;
  dg_parse_kernel<<<(p.n_records - p.rec_begin + kThreads - 1) / kThreads, kThreads, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace sgr
