// ingest.cpp — Kafka RecordBatch (magic 2) -> packed 64-byte event records  (SURVEY §8 row f1), and the per-partition
// offset bookkeeping the KTable lag gate needs (row f2).
//
// What this replaces on the reference side: the consumer that feeds the state store reads the topic with
// isolation.level = read_committed (modules/common/src/main/scala/surge/kafka/streams/SurgeStateStoreConsumer.scala:38),
// the publisher compresses with LZ4 by default (modules/common/src/main/resources/reference.conf:124), events are
// published inside Kafka transactions and every new producer first writes an empty-key flush record
// (modules/command-engine/core/src/main/scala/surge/internal/kafka/KafkaProducerActorImpl.scala:321-329). The byte format
// itself lives in a third-party dependency that is not under the reference checkout: org.apache.kafka:kafka-clients:3.2.3
// (project/Dependencies.scala:42) — DefaultRecordBatch / DefaultRecord / KafkaLZ4BlockInputStream. No test of the
// reference holds broker bytes, so byte-level parity of the RecordBatch framing is UNPINNED; it is restated from the
// published format (KIP-98 message format v2) and checked against an independent encoder/decoder in oracle/kafka_batch.py.
// The layers below it are pinned against real implementations: lz4 frames by liblz4 (via pyarrow), xxHash32 by the xxhash
// package, CRC-32C by the RFC 3720 vectors, the multilanguage protobuf framing by the protobuf runtime (tests/test_ingest_cpu.py).
//
// Host-only C++: the decode is byte parsing with data-dependent control flow on a few MB per poll; the fold it
// feeds is the GPU path. Nothing here touches CUDA.
#include <errno.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <queue>
#include <chrono>
#include <thread>
#include <map>
#include <string>
#include <vector>

#include "../../include/sgr.h"
#include "record_batch.h"

using namespace sgr;

namespace {

// ------------------------------------------------------------------ CRC-32C (Castagnoli, reflected 0x82F63B78)
struct Crc32cTables {
  uint32_t t[8][256];
  Crc32cTables() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      t[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; ++i)
      for (int s = 1; s < 8; ++s) t[s][i] = (t[s - 1][i] >> 8) ^ t[0][t[s - 1][i] & 0xff];
  }
};
const Crc32cTables g_crc;

uint32_t crc32c_sw(const uint8_t* p, uint64_t n, uint32_t crc) {
  crc = ~crc;
  while (n && ((uintptr_t)p & 7)) { crc = g_crc.t[0][(crc ^ *p++) & 0xff] ^ (crc >> 8); --n; }
  while (n >= 8) {
    uint64_t w; memcpy(&w, p, 8);
    w ^= crc;
    crc = g_crc.t[7][w & 0xff] ^ g_crc.t[6][(w >> 8) & 0xff] ^ g_crc.t[5][(w >> 16) & 0xff] ^ g_crc.t[4][(w >> 24) & 0xff] ^
          g_crc.t[3][(w >> 32) & 0xff] ^ g_crc.t[2][(w >> 40) & 0xff] ^ g_crc.t[1][(w >> 48) & 0xff] ^ g_crc.t[0][(w >> 56) & 0xff];
    p += 8; n -= 8;
  }
  while (n--) crc = g_crc.t[0][(crc ^ *p++) & 0xff] ^ (crc >> 8);
  return ~crc;
}

#if defined(__x86_64__)
__attribute__((target("sse4.2"))) uint32_t crc32c_hw(const uint8_t* p, uint64_t n, uint32_t crc) {
  uint64_t c = (uint32_t)~crc;
  while (n && ((uintptr_t)p & 7)) { c = __builtin_ia32_crc32qi((uint32_t)c, *p++); --n; }
  while (n >= 8) { uint64_t w; memcpy(&w, p, 8); c = __builtin_ia32_crc32di(c, w); p += 8; n -= 8; }
  while (n--) c = __builtin_ia32_crc32qi((uint32_t)c, *p++);
  return ~(uint32_t)c;
}
bool have_sse42() { static const bool v = __builtin_cpu_supports("sse4.2"); return v; }
#endif

uint32_t crc32c(const uint8_t* p, uint64_t n) {
#if defined(__x86_64__)
  if (have_sse42()) return crc32c_hw(p, n, 0);
#endif
  return crc32c_sw(p, n, 0);
}

// ------------------------------------------------------------------ xxHash32 (LZ4 frame checksums)
inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
inline uint32_t rd32le(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

uint32_t xxh32(const uint8_t* p, uint64_t len, uint32_t seed) {
  const uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
  const uint8_t* const end = p + len;
  uint32_t h;
  if (len >= 16) {
    uint32_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
    const uint8_t* const limit = end - 16;
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

// ------------------------------------------------------------------ LZ4 frame -> bytes
// Returns an empty string on success, else what was wrong. Output is appended to `out`; matches may reach back across
// block boundaries (block-dependent frames), never before the start of this frame's output.
std::string lz4_frame_decode(const uint8_t* src, uint64_t n, std::vector<uint8_t>* out) {
  const uint64_t out_base = out->size();
  uint64_t pos = 0;
  if (n < 7) return "LZ4 frame shorter than its header";
  if (rd32le(src) != 0x184D2204u) return "bad LZ4 frame magic";
  const uint8_t flg = src[4], bd = src[5];
  if ((flg >> 6) != 1) return "unsupported LZ4 frame version";
  if (flg & 0x02) return "reserved LZ4 FLG bit set";
  const bool block_checksum = flg & 0x10, content_size = flg & 0x08, content_checksum = flg & 0x04, dict_id = flg & 0x01;
  const uint32_t bs_code = (bd >> 4) & 7;
  if (bs_code < 4 || (bd & 0x8F)) return "bad LZ4 block-size descriptor";
  const uint64_t max_block = 1ull << (8 + 2 * bs_code);  // 4 -> 64 KiB ... 7 -> 4 MiB
  uint64_t desc_len = 2 + (content_size ? 8 : 0) + (dict_id ? 4 : 0);
  if (n < 4 + desc_len + 1) return "LZ4 frame header truncated";
  uint64_t declared = 0;
  if (content_size) memcpy(&declared, src + 6, 8);
  const uint8_t hc = src[4 + desc_len];
  if (((xxh32(src + 4, desc_len, 0) >> 8) & 0xff) != hc) return "LZ4 frame header checksum mismatch";
  pos = 4 + desc_len + 1;
  for (;;) {
    if (pos + 4 > n) return "LZ4 frame truncated (no end mark)";
    const uint32_t word = rd32le(src + pos); pos += 4;
    if (word == 0) break;
    const bool stored = word & 0x80000000u;
    const uint64_t bsz = word & 0x7FFFFFFFu;
    if (bsz > max_block) return "LZ4 block larger than the frame's maximum";
    if (pos + bsz + (block_checksum ? 4 : 0) > n) return "LZ4 block truncated";
    const uint8_t* b = src + pos;
    if (block_checksum && xxh32(b, bsz, 0) != rd32le(b + bsz)) return "LZ4 block checksum mismatch";
    if (stored) {
      out->insert(out->end(), b, b + bsz);
    } else {
      // decode through raw pointers into a window of max_block (+ slack for 8-byte copies) bytes, then trim
      const uint64_t block_out_start = out->size();
      out->resize(block_out_start + max_block + 16);
      uint8_t* const win = out->data() + block_out_start;
      uint8_t* const frame_begin = out->data() + out_base;
      uint8_t* op = win;
      uint8_t* const op_limit = win + max_block;
      uint64_t ip = 0;
      const char* bad = nullptr;
      for (;;) {
        if (ip >= bsz) { bad = "LZ4 block ends inside a sequence"; break; }
        const uint8_t token = b[ip++];
        uint64_t lit = token >> 4;
        if (lit == 15) {
          uint8_t s;
          do { if (ip >= bsz) { bad = "LZ4 literal length truncated"; break; } s = b[ip++]; lit += s; } while (s == 255);
          if (bad) break;
        }
        if (lit > bsz - ip) { bad = "LZ4 literals run past the block"; break; }
        if (lit > (uint64_t)(op_limit - op)) { bad = "LZ4 block decodes past the frame's maximum block size"; break; }
        memcpy(op, b + ip, lit);
        op += lit; ip += lit;
        if (ip == bsz) break;  // the last sequence carries literals only
        if (ip + 2 > bsz) { bad = "LZ4 match offset truncated"; break; }
        const uint32_t off = b[ip] | ((uint32_t)b[ip + 1] << 8); ip += 2;
        uint64_t mlen = (token & 15);
        if (mlen == 15) {
          uint8_t s;
          do { if (ip >= bsz) { bad = "LZ4 match length truncated"; break; } s = b[ip++]; mlen += s; } while (s == 255);
          if (bad) break;
        }
        mlen += 4;
        if (off == 0 || off > (uint64_t)(op - frame_begin)) { bad = "LZ4 match offset outside the decoded data"; break; }
        if (mlen > (uint64_t)(op_limit - op)) { bad = "LZ4 block decodes past the frame's maximum block size"; break; }
        const uint8_t* from = op - off;
        if (off >= 8) {   // 8 bytes at a time; may write up to 7 bytes past the match, inside the slack
          for (uint64_t k = 0; k < mlen; k += 8) memcpy(op + k, from + k, 8);
        } else {
          for (uint64_t k = 0; k < mlen; ++k) op[k] = from[k];   // overlapping match: replicates the last `off` bytes
        }
        op += mlen;
      }
      out->resize(block_out_start + (uint64_t)(op - win));
      if (bad) return bad;
    }
    pos += bsz + (block_checksum ? 4 : 0);
  }
  if (content_checksum) {
    if (pos + 4 > n) return "LZ4 content checksum truncated";
    if (xxh32(out->data() + out_base, out->size() - out_base, 0) != rd32le(src + pos)) return "LZ4 content checksum mismatch";
    pos += 4;
  }
  if (content_size && declared != out->size() - out_base) return "LZ4 content size mismatch";
  return std::string();
}

uint64_t uvarint(Cursor& c) {   // protobuf base-128 varint (no zig-zag), at most 10 bytes
  uint64_t v = 0; int shift = 0;
  for (int i = 0; i < 10; ++i) {
    if (c.pos >= c.n) { c.ok = false; return 0; }
    const uint8_t b = c.p[c.pos++];
    v |= (uint64_t)(b & 0x7f) << shift;
    if (!(b & 0x80)) return v;
    shift += 7;
  }
  c.ok = false; return 0;
}

// ------------------------------------------------------------------ growable aggregate-id dictionary (first-seen order = dense index)
inline uint64_t hash_bytes(const uint8_t* k, uint32_t len) {   // 8 bytes at a time, multiply-xorshift mixing
  uint64_t h = 0x9e3779b97f4a7c15ull ^ ((uint64_t)len * 0xff51afd7ed558ccdull);
  while (len >= 8) { uint64_t w; memcpy(&w, k, 8); h = (h ^ w) * 0x9fb21c651e98df25ull; h ^= h >> 32; k += 8; len -= 8; }
  if (len) { uint64_t w = 0; memcpy(&w, k, len); h = (h ^ w) * 0x9fb21c651e98df25ull; h ^= h >> 32; }
  h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 29;
  return h;
}

// 64 independent open-addressing tables (shard = top 6 hash bits) over ONE append-only id arena. A decode call probes the
// shards in parallel (each shard belongs to one worker), new ids get a provisional slot, and dense indices are then handed
// out serially in arrival order — so the index of an id is its first-seen rank no matter how many threads decoded.
class ShardedDict {
 public:
  static constexpr int kShards = 64;
  static constexpr uint32_t kEmpty = 0xFFFFFFFFu;
  static constexpr uint32_t kProv = 0x80000000u;   // idx bit 31: provisional, low bits = position in the owner's NewKey list
  struct Slot { uint32_t tag; uint32_t idx; uint64_t off_len; };   // tag = low 32 hash bits (also the home position, so growing
                                                                   // never re-reads keys); off_len = arena offset << 24 | length
  struct NewKey { uint32_t fetch, rec; const uint8_t* bytes; uint32_t len, shard, slot_pos, final_idx; };
  ShardedDict() { offs_.push_back(0); }
  static int shard_of(uint64_t h) { return (int)(h >> 58); }

  void reserve_shard(int s, uint64_t extra) { while ((count_[s].n + extra + 1) * 2 > slots_[s].size()) grow(s); }
  void prefetch_slot(uint64_t h) const { const auto& t = slots_[shard_of(h)]; if (!t.empty()) __builtin_prefetch(&t[(uint32_t)h & (t.size() - 1)]); }
  void prefetch_key(uint64_t h) const {   // the slot is expected in cache by now: pull the candidate's id bytes
    const auto& t = slots_[shard_of(h)];
    if (t.empty()) return;
    const Slot& sl = t[(uint32_t)h & (t.size() - 1)];
    if (sl.idx != kEmpty && !(sl.idx & kProv)) __builtin_prefetch(bytes_.data() + (sl.off_len >> 24));
  }
  // Owner thread of the shard only; reserve_shard() first. Returns the dense index, or kProv | position in `news`.
  uint32_t probe(const uint8_t* k, uint32_t len, uint64_t h, uint32_t fetch, uint32_t rec, std::vector<NewKey>* news) {
    const int s = shard_of(h);
    std::vector<Slot>& t = slots_[s];
    const uint64_t mask = t.size() - 1;
    const uint32_t tag = (uint32_t)h;
    uint64_t at = tag & mask;
    for (;;) {
      Slot& sl = t[at];
      if (sl.idx == kEmpty) {
        sl.tag = tag; sl.idx = kProv | (uint32_t)news->size(); sl.off_len = 0;
        news->push_back(NewKey{fetch, rec, k, len, (uint32_t)s, (uint32_t)at, 0u});
        ++count_[s].n;
        return sl.idx;
      }
      if (sl.tag == tag) {
        if (sl.idx & kProv) {
          const NewKey& nk = (*news)[sl.idx & ~kProv];
          if (nk.len == len && (len == 0 || memcmp(nk.bytes, k, len) == 0)) return sl.idx;
        } else if ((uint32_t)(sl.off_len & 0xFFFFFF) == len && (len == 0 || memcmp(bytes_.data() + (sl.off_len >> 24), k, len) == 0)) {
          return sl.idx;
        }
      }
      at = (at + 1) & mask;
    }
  }
  // serial, in arrival order: the id gets the next dense index and its bytes move into the arena
  void admit(NewKey* nk) {
    nk->final_idx = (uint32_t)n_++;
    bytes_.insert(bytes_.end(), nk->bytes, nk->bytes + nk->len);
    offs_.push_back((uint32_t)bytes_.size());
  }
  // owner thread of the shard: the provisional slot becomes a final one
  void publish(const NewKey& nk) {
    Slot& sl = slots_[nk.shard][nk.slot_pos];
    sl.idx = nk.final_idx;
    sl.off_len = ((uint64_t)offs_[nk.final_idx] << 24) | nk.len;
  }
  uint64_t size() const { return n_; }
  uint64_t arena_bytes() const { return bytes_.size(); }
  const uint8_t* bytes() const { return bytes_.data(); }
  const uint32_t* offsets() const { return offs_.data(); }

 private:
  void grow(int sh) {
    std::vector<Slot>& t = slots_[sh];
    const uint64_t cap = t.empty() ? 256 : t.size() * 2;
    std::vector<Slot> s(cap, Slot{0, kEmpty, 0});
    for (const Slot& sl : t) {
      if (sl.idx == kEmpty) continue;
      uint64_t at = sl.tag & (cap - 1);
      while (s[at].idx != kEmpty) at = (at + 1) & (cap - 1);
      s[at] = sl;
    }
    t.swap(s);
  }
  std::vector<uint8_t> bytes_;
  std::vector<uint32_t> offs_;
  std::vector<Slot> slots_[kShards];
  struct alignas(64) Count { uint64_t n = 0; };   // one cache line per shard: each is bumped by a different worker
  Count count_[kShards];
  uint64_t n_ = 0;
};

// a few long-lived workers: a poll is decoded in ~10 ms, spawning threads for each of its three parallel phases would show
class WorkerPool {
 public:
  ~WorkerPool() { stop(); }
  template <typename F>
  void run(uint32_t n_tasks, uint32_t n_thr, F&& task) {
    if (n_thr > n_tasks) n_thr = n_tasks;
    if (n_thr <= 1) { for (uint32_t i = 0; i < n_tasks; ++i) task(i); return; }
    ensure(n_thr - 1);
    std::function<void(uint32_t)> fn = std::ref(task);
    {
      std::lock_guard<std::mutex> lk(mu_);
      fn_ = &fn; n_tasks_ = n_tasks; next_.store(0); active_ = n_thr - 1; want_ = n_thr - 1; ++epoch_;
    }
    cv_.notify_all();
    for (uint32_t c; (c = next_.fetch_add(1)) < n_tasks;) task(c);      // the caller works too
    std::unique_lock<std::mutex> lk(mu_);
    done_cv_.wait(lk, [&] { return active_ == 0; });
    fn_ = nullptr;
  }

 private:
  void ensure(uint32_t n) {
    while (threads_.size() < n) {
      const uint32_t id = (uint32_t)threads_.size();
      threads_.emplace_back([this, id] { loop(id); });
    }
  }
  void loop(uint32_t id) {
    uint64_t seen = 0;
    for (;;) {
      std::function<void(uint32_t)>* fn;
      uint32_t n_tasks;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return quit_ || (epoch_ != seen && id < want_); });
        if (quit_) return;
        seen = epoch_; fn = fn_; n_tasks = n_tasks_;
      }
      for (uint32_t c; (c = next_.fetch_add(1)) < n_tasks;) (*fn)(c);
      std::lock_guard<std::mutex> lk(mu_);
      if (--active_ == 0) done_cv_.notify_one();
    }
  }
  void stop() {
    { std::lock_guard<std::mutex> lk(mu_); quit_ = true; }
    cv_.notify_all();
    for (auto& t : threads_) t.join();
    threads_.clear();
  }
  std::mutex mu_;
  std::condition_variable cv_, done_cv_;
  std::vector<std::thread> threads_;
  std::function<void(uint32_t)>* fn_ = nullptr;
  std::atomic<uint32_t> next_{0};
  uint32_t n_tasks_ = 0, active_ = 0, want_ = 0;
  uint64_t epoch_ = 0;
  bool quit_ = false;
};

// append-only byte buffer that grows without zero-filling (the pending log is written exactly once per byte)
struct RawBuf {
  uint8_t* p = nullptr; size_t n = 0, cap = 0;
  void* (*alloc_fn)(size_t) = malloc;     // the engine swaps in page-locked memory so the H2D copy of a poll runs at DMA speed
  void (*free_fn)(void*) = free;
  ~RawBuf() { if (p) free_fn(p); }
  bool grow_to(size_t need) {
    if (need <= cap) return true;
    size_t c = cap ? cap : (1u << 16);
    while (c < need) c *= 2;
    return move_to(c, alloc_fn, free_fn);
  }
  bool move_to(size_t c, void* (*a)(size_t), void (*f)(void*)) {
    uint8_t* q = (uint8_t*)a(c);
    if (!q) return false;
    if (n) memcpy(q, p, n);
    if (p) free_fn(p);
    p = q; cap = c; alloc_fn = a; free_fn = f;
    return true;
  }
};

// ------------------------------------------------------------------ flat JSON event -> packed event (SGR_VALUE_JSON)
// The reference's sample models write their events as play-json objects, e.g. (core TestBoundedContext.scala:44-56,153-161)
//   {"_type":"...CountIncremented","aggregateId":"a","incrementBy":1,"sequenceNumber":4}
// A model registers which member is the class discriminator, which event type index each class name maps to, and which
// numeric members land at which byte of the packed record. Members are looked up by name: order and extra members do not matter.
struct JsonFieldSpec { std::string name; uint8_t kind; uint16_t dst_off; uint32_t len; };
struct JsonEventSpec { std::string type_name; uint32_t event_type; std::vector<JsonFieldSpec> fields; };
struct JsonPacker {
  std::string discriminator;
  std::vector<JsonEventSpec> events;
  int32_t unknown_type = -1;          // >= 0: an unknown class name becomes this event type (a scala.MatchError in the handler)
};

struct JsonMember { const uint8_t* key; uint32_t key_len; bool key_escaped; const uint8_t* val; uint32_t val_len; char kind; };  // kind: s n o a t f z

struct JsonScan {
  const uint8_t* p; const uint8_t* end; const char* err = nullptr;
  void ws() { while (p < end && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) ++p; }
  // p at the opening quote; leaves p after the closing quote; [*b, *b + *n) is the raw content between the quotes
  bool string(const uint8_t** b, uint32_t* n, bool* escaped) {
    if (p >= end || *p != '"') { err = "expected a string"; return false; }
    ++p; *b = p; *escaped = false;
    while (p < end && *p != '"') {
      if (*p < 0x20) { err = "control character inside a string"; return false; }
      if (*p == '\\') { *escaped = true; ++p; if (p >= end) break; }
      ++p;
    }
    if (p >= end) { err = "unterminated string"; return false; }
    *n = (uint32_t)(p - *b); ++p;
    return true;
  }
  bool value(JsonMember* m, int depth) {
    ws();
    if (p >= end) { err = "value expected"; return false; }
    m->val = p;
    const uint8_t c = *p;
    if (c == '"') {
      const uint8_t* b; uint32_t n; bool esc;
      if (!string(&b, &n, &esc)) return false;
      m->kind = 's'; m->val = b; m->val_len = n;
      if (esc) m->kind = 'S';   // string with escapes: compared after unescaping
      return true;
    }
    if (c == '{' || c == '[') {
      if (depth > 32) { err = "nesting too deep"; return false; }
      const uint8_t close = c == '{' ? '}' : ']';
      ++p; ws();
      if (p < end && *p == close) { ++p; m->kind = c == '{' ? 'o' : 'a'; m->val_len = (uint32_t)(p - m->val); return true; }
      for (;;) {
        if (c == '{') {
          ws();
          const uint8_t* b; uint32_t n; bool esc;
          if (!string(&b, &n, &esc)) return false;
          ws();
          if (p >= end || *p != ':') { err = "':' expected"; return false; }
          ++p;
        }
        JsonMember inner{};
        if (!value(&inner, depth + 1)) return false;
        ws();
        if (p < end && *p == ',') { ++p; continue; }
        if (p < end && *p == close) { ++p; break; }
        err = "',' or a closing bracket expected"; return false;
      }
      m->kind = c == '{' ? 'o' : 'a'; m->val_len = (uint32_t)(p - m->val);
      return true;
    }
    if (c == '-' || (c >= '0' && c <= '9')) {
      const uint8_t* q = p;
      if (*q == '-') ++q;
      if (q >= end || *q < '0' || *q > '9') { err = "malformed number"; return false; }
      if (*q == '0') ++q; else while (q < end && *q >= '0' && *q <= '9') ++q;
      if (q < end && *q == '.') { ++q; if (q >= end || *q < '0' || *q > '9') { err = "malformed number"; return false; } while (q < end && *q >= '0' && *q <= '9') ++q; }
      if (q < end && (*q == 'e' || *q == 'E')) {
        ++q; if (q < end && (*q == '+' || *q == '-')) ++q;
        if (q >= end || *q < '0' || *q > '9') { err = "malformed number"; return false; }
        while (q < end && *q >= '0' && *q <= '9') ++q;
      }
      m->kind = 'n'; m->val_len = (uint32_t)(q - p); p = q;
      return true;
    }
    auto lit = [&](const char* w, char k) { const size_t n = strlen(w); if ((size_t)(end - p) >= n && memcmp(p, w, n) == 0) { p += n; m->kind = k; m->val_len = (uint32_t)n; return true; } return false; };
    if (lit("true", 't') || lit("false", 'f') || lit("null", 'z')) return true;
    err = "unexpected character";
    return false;
  }
};

// JSON string content (between the quotes) -> bytes; \uXXXX incl. surrogate pairs -> UTF-8
bool json_unescape(const uint8_t* b, uint32_t n, std::string* out) {
  out->clear();
  auto hex4 = [&](uint32_t i, uint32_t* v) { if (i + 4 > n) return false; *v = 0; for (int k = 0; k < 4; ++k) { const uint8_t c = b[i + k]; uint32_t d; if (c >= '0' && c <= '9') d = c - '0'; else if (c >= 'a' && c <= 'f') d = c - 'a' + 10; else if (c >= 'A' && c <= 'F') d = c - 'A' + 10; else return false; *v = *v * 16 + d; } return true; };
  for (uint32_t i = 0; i < n; ++i) {
    if (b[i] != '\\') { out->push_back((char)b[i]); continue; }
    if (++i >= n) return false;
    switch (b[i]) {
      case '"': out->push_back('"'); break;   case '\\': out->push_back('\\'); break; case '/': out->push_back('/'); break;
      case 'b': out->push_back('\b'); break;  case 'f': out->push_back('\f'); break;  case 'n': out->push_back('\n'); break;
      case 'r': out->push_back('\r'); break;  case 't': out->push_back('\t'); break;
      case 'u': {
        uint32_t cp;
        if (!hex4(i + 1, &cp)) return false;
        i += 4;
        if (cp >= 0xD800 && cp < 0xDC00 && i + 6 < n + 0u && b[i + 1] == '\\' && b[i + 2] == 'u') {
          uint32_t lo;
          if (hex4(i + 3, &lo) && lo >= 0xDC00 && lo < 0xE000) { cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00); i += 6; }
        }
        if (cp < 0x80) out->push_back((char)cp);
        else if (cp < 0x800) { out->push_back((char)(0xC0 | (cp >> 6))); out->push_back((char)(0x80 | (cp & 0x3F))); }
        else if (cp < 0x10000) { out->push_back((char)(0xE0 | (cp >> 12))); out->push_back((char)(0x80 | ((cp >> 6) & 0x3F))); out->push_back((char)(0x80 | (cp & 0x3F))); }
        else { out->push_back((char)(0xF0 | (cp >> 18))); out->push_back((char)(0x80 | ((cp >> 12) & 0x3F))); out->push_back((char)(0x80 | ((cp >> 6) & 0x3F))); out->push_back((char)(0x80 | (cp & 0x3F))); }
        break;
      }
      default: return false;
    }
  }
  return true;
}

bool json_name_is(const uint8_t* b, uint32_t n, bool escaped, const std::string& want, std::string* tmp) {
  if (!escaped) return n == want.size() && memcmp(b, want.data(), n) == 0;
  return json_unescape(b, n, tmp) && *tmp == want;
}

// value bytes -> the 56 bytes the record parser copies into the packed record (type, seq, payload). Returns nullptr on success.
const char* json_pack(const JsonPacker& jp, const uint8_t* val, uint32_t val_len, uint8_t out[56], std::string* tmp) {
  JsonScan sc{val, val + val_len};
  JsonMember members[48];
  uint32_t n_members = 0;
  sc.ws();
  if (sc.p >= sc.end || *sc.p != '{') return "the value is not a JSON object";
  ++sc.p; sc.ws();
  if (sc.p < sc.end && *sc.p == '}') { ++sc.p; }
  else {
    for (;;) {
      sc.ws();
      JsonMember m{};
      if (!sc.string(&m.key, &m.key_len, &m.key_escaped)) return sc.err;
      sc.ws();
      if (sc.p >= sc.end || *sc.p != ':') return "':' expected";
      ++sc.p;
      if (!sc.value(&m, 1)) return sc.err;
      if (n_members >= 48) return "more than 48 members";
      members[n_members++] = m;
      sc.ws();
      if (sc.p < sc.end && *sc.p == ',') { ++sc.p; continue; }
      if (sc.p < sc.end && *sc.p == '}') { ++sc.p; break; }
      return "',' or '}' expected";
    }
  }
  sc.ws();
  if (sc.p != sc.end) return "bytes after the JSON object";
  // later duplicates of a member win, as in play-json's JsObject
  auto find = [&](const std::string& name) -> const JsonMember* {
    const JsonMember* hit = nullptr;
    for (uint32_t i = 0; i < n_members; ++i) if (json_name_is(members[i].key, members[i].key_len, members[i].key_escaped, name, tmp)) hit = &members[i];
    return hit;
  };
  const JsonEventSpec* ev = nullptr;
  if (jp.discriminator.empty()) {
    ev = &jp.events[0];       // one class only (a state topic: Json.toJson(agg) carries no discriminator)
  } else {
    const JsonMember* d = find(jp.discriminator);
    if (!d || (d->kind != 's' && d->kind != 'S')) return "the class discriminator member is missing or not a string";
    std::string cls;
    for (const JsonEventSpec& e : jp.events) if (json_name_is(d->val, d->val_len, d->kind == 'S', e.type_name, &cls)) { ev = &e; break; }
  }
  memset(out, 0, 56);
  if (!ev) {
    if (jp.unknown_type < 0) return "unknown event class";
    const uint32_t ty = (uint32_t)jp.unknown_type;
    memcpy(out, &ty, 4);
    return nullptr;
  }
  memcpy(out, &ev->event_type, 4);
  for (const JsonFieldSpec& f : ev->fields) {
    const JsonMember* m = find(f.name);
    uint8_t* dst = out + (f.dst_off < 8 ? f.dst_off : f.dst_off - 8);   // record offsets 0..7 = type, seq; 16.. = payload (value bytes 8..)
    if (f.kind == SGR_JSON_UUID || f.kind == SGR_JSON_PSTR) {
      if (!m || (m->kind != 's' && m->kind != 'S')) return "a string member of the event is missing or not a string";
      const uint8_t* sb = m->val; uint32_t sn = m->val_len;
      if (m->kind == 'S') { if (!json_unescape(m->val, m->val_len, tmp)) return "bad escape in a string member"; sb = (const uint8_t*)tmp->data(); sn = (uint32_t)tmp->size(); }
      if (f.kind == SGR_JSON_UUID) {
        // java.util.UUID.toString: 8-4-4-4-12 hex digits; stored as the 16 bytes most significant first
        if (sn != 36 || sb[8] != '-' || sb[13] != '-' || sb[18] != '-' || sb[23] != '-') return "a UUID member is not in 8-4-4-4-12 form";
        uint32_t k = 0;
        for (uint32_t i = 0; i < 36; ++i) {
          if (i == 8 || i == 13 || i == 18 || i == 23) continue;
          const uint8_t c = sb[i];
          uint32_t d;
          if (c >= '0' && c <= '9') d = c - '0'; else if (c >= 'a' && c <= 'f') d = c - 'a' + 10; else if (c >= 'A' && c <= 'F') d = c - 'A' + 10; else return "a UUID member holds a non-hex digit";
          if (k & 1) dst[k >> 1] |= (uint8_t)d; else dst[k >> 1] = (uint8_t)(d << 4);
          ++k;
        }
      } else {
        // length byte + UTF-8 bytes, zero padded to the slot (surge_b200/formats.py _pstr)
        if (sn > f.len - 1 || sn > 255) return "a string member does not fit its slot";
        dst[0] = (uint8_t)sn;
        memcpy(dst + 1, sb, sn);
      }
      continue;
    }
    if (!m || m->kind != 'n') return "a numeric member of the event is missing or not a number";
    char num[64];
    if (m->val_len >= sizeof num) return "number too long";
    memcpy(num, m->val, m->val_len); num[m->val_len] = 0;
    if (f.kind == 2) {
      const double v = strtod(num, nullptr);      // correctly rounded, like java.lang.Double.parseDouble
      memcpy(dst, &v, 8);
    } else {
      bool integral = true;
      for (uint32_t i = 0; i < m->val_len; ++i) if (num[i] == '.' || num[i] == 'e' || num[i] == 'E') integral = false;
      if (!integral) return "an integer member holds a fraction or an exponent";
      errno = 0;
      char* endp = nullptr;
      const long long v = strtoll(num, &endp, 10);
      if (errno || *endp) return "integer out of range";
      if (f.kind == 0) { if (v < INT32_MIN || v > INT32_MAX) return "integer does not fit an Int"; const int32_t w = (int32_t)v; memcpy(dst, &w, 4); }
      else memcpy(dst, &v, 8);
    }
  }
  return nullptr;
}

struct ProbeOut {                 // one worker's probe results: (record position, dense index or provisional) per fetch
  std::vector<uint32_t> pos, val;
  std::vector<size_t> off;        // n_fetches + 1
};

struct KeyRef { uint32_t off, len; uint64_t hash; };
struct Staged {
  std::vector<uint8_t> recs;      // 64-byte records, agg field still zero
  std::vector<KeyRef> keys;       // one per record, into `arena`
  std::vector<uint8_t> arena;     // aggregate-id bytes (copied: the decompression scratch is reused per batch)
  std::vector<uint8_t> shard;     // dictionary shard of each record's id
  uint32_t shard_count[ShardedDict::kShards];
  std::vector<uint8_t> scratch;
  PartitionState ps;              // the partition's state after this fetch (committed in phase 2)
  sgr_ingest_stats st{};
  int32_t rc = SGR_OK;
  int32_t null_value_type = -1;
  int32_t value_framing = 0;
  const JsonPacker* json = nullptr;
  std::string json_tmp;
  std::string err;
  void reset() { recs.clear(); keys.clear(); arena.clear(); shard.clear(); memset(shard_count, 0, sizeof shard_count); scratch.clear(); st = sgr_ingest_stats{}; rc = SGR_OK; err.clear(); }
};

}  // namespace

struct sgr_ingest {
  std::string last_error;
  ShardedDict dict;
  WorkerPool workers;
  std::vector<std::vector<ShardedDict::NewKey>> news;   // per worker, reused across calls
  std::vector<ProbeOut> probed;                          // per worker, reused across calls
  RawBuf pending;                   // packed 64-byte records, arrival order
  std::vector<uint8_t> scratch;     // decompressed records section of the batch being decoded
  std::map<int32_t, PartitionState> parts;
  sgr_ingest_stats total{};
  uint64_t keys_at_mark = 0;
  uint64_t max_ids = 1ull << 31, max_id_bytes = 1ull << 32;   // what the 32-bit dictionary fields can address
  int32_t value_framing = 0;        // SGR_VALUE_PACKED | SGR_VALUE_PROTOBUF_EVENT | SGR_VALUE_JSON | SGR_VALUE_PROTOBUF_JSON
  JsonPacker json;
  int32_t null_value_type = -1;     // >= 0: a keyed record with a null value becomes an event of this type (state-topic tombstones)
  std::vector<Staged> pool;         // staging buffers, reused across calls (a restore loop polls similar sizes)
};

namespace {
template <class... A> int32_t ifail(sgr_ingest* g, int32_t code, const char* fmt, A... a) { return g ? set_error(&g->last_error, code, fmt, a...) : code; }

const char* codec_name(int c) {
  switch (c) { case 1: return "gzip"; case 2: return "snappy"; case 4: return "zstd"; default: return "unknown"; }
}

}  // namespace

extern "C" {

uint32_t sgr_crc32c(const void* data, uint64_t nbytes) { return crc32c((const uint8_t*)data, nbytes); }
uint32_t sgr_crc32c_portable(const void* data, uint64_t nbytes) { return crc32c_sw((const uint8_t*)data, nbytes, 0); }
uint32_t sgr_xxh32(const void* data, uint64_t nbytes, uint32_t seed) { return xxh32((const uint8_t*)data, nbytes, seed); }

int32_t sgr_lz4_frame_decode(const void* src, uint64_t nbytes, void* out, uint64_t cap, uint64_t* out_len) {
  if ((!src && nbytes) || !out_len) return SGR_ERR_INVALID;
  std::vector<uint8_t> v;
  const std::string err = lz4_frame_decode((const uint8_t*)src, nbytes, &v);
  if (!err.empty()) return SGR_ERR_INVALID;
  *out_len = v.size();
  if (v.size() > cap) return SGR_ERR_CAPACITY;
  if (!v.empty()) memcpy(out, v.data(), v.size());
  return SGR_OK;
}

int32_t sgr_ingest_create(sgr_ingest** out) {
  if (!out) return SGR_ERR_INVALID;
  *out = new (std::nothrow) sgr_ingest();
  return *out ? SGR_OK : SGR_ERR_OOM;
}

int32_t sgr_ingest_destroy(sgr_ingest* g) { delete g; return SGR_OK; }

const char* sgr_ingest_last_error(const sgr_ingest* g) { return g ? g->last_error.c_str() : "null ingest handle"; }

int32_t sgr_ingest_set_json_packer(sgr_ingest* g, const char* discriminator, const sgr_json_event* events, uint32_t n_events, int32_t unknown_type) {
  if (!g || !discriminator || (n_events && !events)) return ifail(g, SGR_ERR_INVALID, "null argument");
  if (unknown_type >= (int32_t)SGR_MAX_TYPES) return ifail(g, SGR_ERR_INVALID, "unknown_type out of range");
  if (!*discriminator && n_events != 1) return ifail(g, SGR_ERR_INVALID, "without a discriminator member exactly one class can be registered");
  JsonPacker jp;
  jp.discriminator = discriminator;
  jp.unknown_type = unknown_type < 0 ? -1 : unknown_type;
  for (uint32_t i = 0; i < n_events; ++i) {
    const sgr_json_event& e = events[i];
    if (!e.type_name || e.event_type >= SGR_MAX_TYPES || e.n_fields > SGR_JSON_MAX_FIELDS) return ifail(g, SGR_ERR_INVALID, "JSON event %u: bad type name, type index or field count", i);
    JsonEventSpec es{e.type_name, e.event_type, {}};
    for (uint32_t f = 0; f < e.n_fields; ++f) {
      const sgr_json_field& jf = e.fields[f];
      const uint32_t size = json_member_size(jf);
      if (!size || !json_event_slot_ok(jf, size)) return ifail(g, SGR_ERR_INVALID, "JSON event %u field %u: bad name, kind, length or record offset", i, f);
      es.fields.push_back(JsonFieldSpec{jf.name, jf.kind, jf.dst_off, size});
    }
    jp.events.push_back(es);
  }
  g->json = jp;
  return SGR_OK;
}

int32_t sgr_ingest_set_value_framing(sgr_ingest* g, int32_t framing) {
  if (!g || framing < SGR_VALUE_PACKED || framing > SGR_VALUE_PROTOBUF_JSON) return ifail(g, SGR_ERR_INVALID, "unknown value framing %d", framing);
  if ((framing == SGR_VALUE_JSON || framing == SGR_VALUE_PROTOBUF_JSON) && g->json.events.empty()) return ifail(g, SGR_ERR_INVALID, "register a JSON packer first (sgr_ingest_set_json_packer)");
  g->value_framing = framing;
  return SGR_OK;
}

int32_t sgr_ingest_set_null_value_type(sgr_ingest* g, int32_t event_type) {
  if (!g || event_type >= (int32_t)SGR_MAX_TYPES) return ifail(g, SGR_ERR_INVALID, "event type out of range");
  g->null_value_type = event_type < 0 ? -1 : event_type;
  return SGR_OK;
}

int32_t sgr_ingest_set_dictionary_limits(sgr_ingest* g, uint64_t max_ids, uint64_t max_id_bytes) {
  if (!g || max_ids == 0 || max_ids > (1ull << 31) || max_id_bytes == 0 || max_id_bytes > (1ull << 32))
    return ifail(g, SGR_ERR_INVALID, "limits must be in (0, 2^31] ids and (0, 2^32] bytes");
  g->max_ids = max_ids; g->max_id_bytes = max_id_bytes;
  return SGR_OK;
}

int32_t sgr_ingest_set_aborted(sgr_ingest* g, int32_t partition, const int64_t* producer_ids, const int64_t* first_offsets, uint64_t n) {
  if (!g || (n && (!producer_ids || !first_offsets))) return ifail(g, SGR_ERR_INVALID, "null argument");
  g->parts[partition].announce_aborted(producer_ids, first_offsets, n);
  return SGR_OK;
}

}  // extern "C"

// ---- phase 1 (any thread, touches nothing shared): one fetch -> staged records + key references
namespace {
int32_t decode_fetch(int32_t partition, const uint8_t* buf, uint64_t nbytes, Staged* o) {
  PartitionState& ps = o->ps;
  sgr_ingest_stats& st = o->st;
  o->recs.reserve(nbytes + nbytes / 4);
  uint64_t pos = 0;
  for (BatchHeader h;; pos += h.total) {
    if (const int32_t rc = frame_batch(partition, buf, nbytes, pos, &h, &o->err)) return rc;
    if (!h.total) break;
    const uint32_t got = crc32c(h.b + 21, h.total - 21);
    if (h.stored_crc != got) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: CRC-32C mismatch (stored %08x, computed %08x)", partition, (long long)h.base_offset, h.stored_crc, got);
    if (const int32_t rc = read_batch_fields(partition, &h, &o->err)) return rc;
    ++st.n_batches;

    // A batch of an aborted transaction is skipped after its CRC and before anything else, as Kafka's consumer skips it: its
    // codec is not looked at and it is not decompressed.
    const bool aborted_batch = ps.reach(h);
    const uint8_t* recs = h.b + kBatchHeader;
    uint64_t recs_len = h.total - kBatchHeader;
    if (h.codec != 0 && !aborted_batch) {
      if (h.codec != 3) return set_error(&o->err, SGR_ERR_UNSUPPORTED, "partition %d offset %lld: %s-compressed batch (none and lz4 are decoded)", partition, (long long)h.base_offset, codec_name(h.codec));
      o->scratch.clear();
      const std::string err = lz4_frame_decode(recs, recs_len, &o->scratch);
      if (!err.empty()) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: %s", partition, (long long)h.base_offset, err.c_str());
      recs = o->scratch.data(); recs_len = o->scratch.size();
      st.n_compressed_bytes += h.total - kBatchHeader; st.n_decompressed_bytes += recs_len;
    }

    if (h.control) {
      ++st.n_control_batches;
      ps.apply_control(h, recs, recs_len);
    } else if (aborted_batch) {
      ++st.n_aborted_batches; st.n_aborted_records += (uint64_t)h.records_count;
    } else {
      Cursor c(recs, recs_len);
      // every record is at least 7 bytes on the wire, so the count cannot lie by much; size the outputs once per batch
      if ((uint64_t)h.records_count > recs_len / 7 + 1) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: recordsCount %d does not fit %llu bytes", partition, (long long)h.base_offset, h.records_count, (unsigned long long)recs_len);
      const size_t recs_at0 = o->recs.size(), arena_at0 = o->arena.size();
      o->recs.resize(recs_at0 + 64 * (size_t)h.records_count);
      o->arena.resize(arena_at0 + recs_len);
      const size_t keys_at0 = o->keys.size();
      o->keys.resize(keys_at0 + (size_t)h.records_count);
      o->shard.resize(keys_at0 + (size_t)h.records_count);
      KeyRef* kr = o->keys.data() + keys_at0;
      uint8_t* shp = o->shard.data() + keys_at0;
      uint8_t* rec = o->recs.data() + recs_at0;
      uint8_t* ar = o->arena.data() + arena_at0;
      for (int32_t r = 0; r < h.records_count; ++r) {
        const int32_t rec_len = c.varint();
        if (!c.ok || rec_len < 0 || (uint64_t)rec_len > recs_len - c.pos) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: record %d length runs past the batch", partition, (long long)h.base_offset, r);
        Cursor q(recs + c.pos, (uint64_t)rec_len);
        c.pos += (uint64_t)rec_len;
        q.bytes(1);             // record attributes (unused in v2)
        q.varlong();            // timestampDelta
        const int32_t offset_delta = q.varint();
        const int32_t key_len = q.varint();
        const uint8_t* key = key_len > 0 ? q.bytes((uint64_t)key_len) : nullptr;
        const int32_t wire_val_len = q.varint();
        const uint8_t* val = wire_val_len > 0 ? q.bytes((uint64_t)wire_val_len) : nullptr;
        const int32_t n_headers = q.varint();
        for (int32_t h = 0; q.ok && h < n_headers; ++h) {
          const int32_t hk = q.varint(); if (hk < 0) { q.ok = false; break; } q.bytes((uint64_t)hk);
          const int32_t hv = q.varint(); if (hv > 0) q.bytes((uint64_t)hv);
        }
        if (!q.ok || q.pos != q.n || n_headers < 0) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: record %d is malformed", partition, (long long)h.base_offset, r);
        const int64_t offset = h.base_offset + offset_delta;
        if (ps.seen && offset < ps.decoded_next) { ++st.n_duplicates; continue; }  // refetch after a restart: already decoded
        if (key_len <= 0) { ++st.n_markers; continue; }                              // the producer's empty-key flush record
        if (wire_val_len < 0 && o->null_value_type < 0) { ++st.n_null_values; continue; }
        int32_t val_len = wire_val_len;
        if (val_len >= 0 && (o->value_framing == SGR_VALUE_PROTOBUF_EVENT || o->value_framing == SGR_VALUE_PROTOBUF_JSON)) {
          // multilanguage topics: the value is protobuf Event { string aggregateId = 1; bytes payload = 2; }
          // (multilanguage-protocol.proto:17-20, written by GenericSurgeCommandBusinessLogic.scala:30-33); the payload is the packed
          // event (SGR_VALUE_PROTOBUF_EVENT) or the business app's JSON (SGR_VALUE_PROTOBUF_JSON, packed next)
          Cursor pb(val, (uint64_t)val_len);
          const uint8_t* payload = nullptr; uint64_t payload_len = 0;
          while (pb.ok && pb.pos < pb.n) {
            const uint64_t tag = uvarint(pb);
            if (!pb.ok) break;
            switch (tag & 7) {
              case 0: uvarint(pb); break;
              case 1: pb.bytes(8); break;
              case 5: pb.bytes(4); break;
              case 2: {
                const uint64_t ln = uvarint(pb);
                const uint8_t* b = pb.ok ? pb.bytes(ln) : nullptr;
                if (pb.ok && (tag >> 3) == 2) { payload = b; payload_len = ln; }
                break;
              }
              default: pb.ok = false;
            }
          }
          if (!pb.ok) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: value is not a protobuf Event", partition, (long long)offset);
          val = payload; val_len = (int32_t)(payload_len > 0x7fffffff ? 0x7fffffff : payload_len);
        }
        uint8_t json_out[56];
        if (val_len >= 0 && (o->value_framing == SGR_VALUE_JSON || o->value_framing == SGR_VALUE_PROTOBUF_JSON)) {
          const char* why = json_pack(*o->json, val, (uint32_t)val_len, json_out, &o->json_tmp);
          if (why) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: JSON event: %s", partition, (long long)offset, why);
          val = json_out; val_len = 56;
        }
        if (val_len >= 0 && (val_len < 8 || val_len > 56)) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: packed event value of %d bytes (expected 8..56: u32 type, u32 seq, payload)", partition, (long long)offset, val_len);
        uint32_t id_len = 0;
        {   // PartitionStringUpToColon (KafkaPartitioner.scala:38-42)
          const void* colon = memchr(key, ':', (size_t)key_len);
          id_len = colon ? (uint32_t)((const uint8_t*)colon - key) : (uint32_t)key_len;
        }
        if (id_len >= (1u << 24)) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: aggregate id of %u bytes", partition, (long long)offset, id_len);
        const uint64_t kh = hash_bytes(key, id_len);
        *kr++ = KeyRef{(uint32_t)(ar - o->arena.data()), id_len, kh};
        *shp++ = (uint8_t)ShardedDict::shard_of(kh);
        ++o->shard_count[ShardedDict::shard_of(kh)];
        memcpy(ar, key, id_len); ar += id_len;
        if (val_len < 0) {                      // null value on a compacted state topic = delete the key (SurgeModel.scala:62-64)
          const uint32_t ty = (uint32_t)o->null_value_type;
          memcpy(rec, &ty, 4);
          ++st.n_null_values;
        } else {
          memcpy(rec, val, 8);                  // u32 type, u32 seq (little endian, as the packer wrote them)
          memcpy(rec + 16, val + 8, (size_t)val_len - 8);   // the rest of the slot is zero from resize(): agg, payload tail
        }
        rec += 64;
        ++st.n_records;
      }
      o->recs.resize((size_t)(rec - o->recs.data()));
      o->arena.resize((size_t)(ar - o->arena.data()));
      o->keys.resize((size_t)(kr - o->keys.data()));
      o->shard.resize((size_t)(shp - o->shard.data()));
      if (c.pos != recs_len) return set_error(&o->err, SGR_ERR_INVALID, "partition %d offset %lld: %llu stray bytes after the last record", partition, (long long)h.base_offset, (unsigned long long)(recs_len - c.pos));
    }
    ps.close(h);
  }
  st.n_trailing_bytes = nbytes - pos;
  st.n_bytes = pos;
  if (o->arena.size() >= (1ull << 32)) return set_error(&o->err, SGR_ERR_INVALID, "partition %d: more than 4 GiB of aggregate ids in one fetch", partition);
  return SGR_OK;
}

// ---- phase 2a (worker t of n_workers; owns the shards s with s % n_workers == t): probe every id of those shards, in
// arrival order. Known ids get their dense index at once; new ones a provisional slot and an entry in the worker's list.
void probe_shards(sgr_ingest* g, std::vector<Staged>& staged, uint32_t n, uint32_t t, uint32_t n_workers) {
  std::vector<ShardedDict::NewKey>& news = g->news[t];
  news.clear();
  // Results stay in the worker's own arrays (record position, index), fetch by fetch: neighbouring records belong to
  // different workers, and writing into one shared per-record array would bounce its cache lines between all of them.
  ProbeOut& out = g->probed[t];
  out.pos.clear(); out.val.clear(); out.off.assign(1, 0);
  uint8_t owner[ShardedDict::kShards];
  for (int s = 0; s < ShardedDict::kShards; ++s) owner[s] = (uint8_t)(s % (int)n_workers);
  for (int s = (int)t; s < ShardedDict::kShards; s += (int)n_workers) {
    uint64_t extra = 0;
    for (uint32_t i = 0; i < n; ++i) extra += staged[i].shard_count[s];
    g->dict.reserve_shard(s, extra);
  }
  for (uint32_t i = 0; i < n; ++i) {
    const Staged& o = staged[i];
    const size_t cnt = o.keys.size();
    const uint8_t* sh = o.shard.data();
    const size_t base = out.pos.size();
    if (n_workers == 1) { out.pos.resize(base + cnt); for (size_t r = 0; r < cnt; ++r) out.pos[base + r] = (uint32_t)r; }
    else for (size_t r = 0; r < cnt; ++r) if (owner[sh[r]] == t) out.pos.push_back((uint32_t)r);
    const size_t m = out.pos.size() - base;
    out.val.resize(base + m);
    const uint32_t* mine = out.pos.data() + base;
    uint32_t* val = out.val.data() + base;
    const uint8_t* arena = o.arena.data();
    // the dictionary of a big topic does not fit any cache: run the probe as a software pipeline — slot prefetched 16
    // ids ahead, the candidate's id bytes 8 ahead — so that the misses of neighbouring records overlap
    constexpr size_t kSlotAhead = 16, kKeyAhead = 8;
    for (size_t j = 0; j < std::min(m, kSlotAhead); ++j) g->dict.prefetch_slot(o.keys[mine[j]].hash);
    for (size_t j = 0; j < m; ++j) {
      if (j + kSlotAhead < m) g->dict.prefetch_slot(o.keys[mine[j + kSlotAhead]].hash);
      if (j + kKeyAhead < m) g->dict.prefetch_key(o.keys[mine[j + kKeyAhead]].hash);
      const uint32_t r = mine[j];
      const KeyRef& k = o.keys[r];
      val[j] = g->dict.probe(arena + k.off, k.len, k.hash, i, r, &news);
    }
    out.off.push_back(out.pos.size());
  }
}

// ---- phase 2b (caller's thread): the new ids of all workers, merged back into arrival order, get the next dense indices
void admit_new_keys(sgr_ingest* g, std::vector<Staged>& staged, uint32_t n_workers) {
  typedef std::pair<uint64_t, uint32_t> Head;   // (fetch << 32 | rec, worker)
  std::priority_queue<Head, std::vector<Head>, std::greater<Head>> heap;
  std::vector<size_t> pos(n_workers, 0);
  auto key_of = [](const ShardedDict::NewKey& k) { return ((uint64_t)k.fetch << 32) | k.rec; };
  for (uint32_t t = 0; t < n_workers; ++t) if (!g->news[t].empty()) heap.push(Head(key_of(g->news[t][0]), t));
  while (!heap.empty()) {
    const uint32_t t = heap.top().second;
    heap.pop();
    ShardedDict::NewKey& nk = g->news[t][pos[t]++];
    g->dict.admit(&nk);
    ++staged[nk.fetch].st.n_new_keys;
    if (pos[t] < g->news[t].size()) heap.push(Head(key_of(g->news[t][pos[t]]), t));
  }
}

// ---- phase 2d (any thread; one task per fetch = the only writer of that part of the pending log): staged records to
// their place, aggregate indices gathered from the workers' result lists
void place_fetch(const sgr_ingest* g, uint8_t* dst, const Staged* o, uint32_t fetch, uint32_t n_workers) {
  memcpy(dst, o->recs.data(), o->recs.size());
  for (uint32_t t = 0; t < n_workers; ++t) {
    const ProbeOut& out = g->probed[t];
    const std::vector<ShardedDict::NewKey>& news = g->news[t];
    for (size_t j = out.off[fetch]; j < out.off[fetch + 1]; ++j) {
      uint32_t v = out.val[j];
      if (v & ShardedDict::kProv) v = news[v & ~ShardedDict::kProv].final_idx;
      const uint64_t agg = v;
      memcpy(dst + (size_t)out.pos[j] * 64 + 8, &agg, 8);
    }
  }
}

// ---- phase 2c (caller's thread): the partition's position and the totals
void commit_fetch(sgr_ingest* g, int32_t partition, Staged* o) {
  PartitionState& live = g->parts[partition];
  const int64_t folded = live.folded_next;
  live = std::move(o->ps);
  live.folded_next = folded;
  add_stats(&g->total, o->st);
}

}  // namespace

extern "C" {

// Decodes n fetches in one call: parsing, CRC and decompression run on up to `threads` host threads (fetches of one
// partition stay on one thread, in call order); ids are interned and records appended afterwards, in call order, so
// the result is identical to n single calls. All or nothing: if any fetch is malformed nothing is applied.
int32_t sgr_ingest_record_batches_mt(sgr_ingest* g, uint32_t n, const int32_t* partitions, const void* const* datas, const uint64_t* nbytes,
                                     uint32_t threads, sgr_ingest_stats* stats /* n entries or NULL */) {
  if (!g || (n && (!partitions || !datas || !nbytes))) return ifail(g, SGR_ERR_INVALID, "null argument");
  for (uint32_t i = 0; i < n; ++i) if (!datas[i] && nbytes[i]) return ifail(g, SGR_ERR_INVALID, "null data for fetch %u", i);
  if (g->pool.size() < n) g->pool.resize(n);
  std::vector<Staged>& staged = g->pool;
  for (uint32_t i = 0; i < n; ++i) staged[i].reset();
  // chain the fetches of one partition: fetch i starts from the state fetch prev[i] left (or the live state)
  std::map<int32_t, std::vector<uint32_t>> by_part;
  for (uint32_t i = 0; i < n; ++i) by_part[partitions[i]].push_back(i);
  std::vector<const std::vector<uint32_t>*> chains;
  for (auto& kv : by_part) chains.push_back(&kv.second);
  for (auto& kv : by_part) g->parts[kv.first];   // create the entries now: phase 1 only reads the map
  auto run_chain = [&](const std::vector<uint32_t>& chain) {
    const PartitionState* from = &g->parts.find(partitions[chain[0]])->second;
    for (uint32_t i : chain) {
      staged[i].ps = *from;
      staged[i].null_value_type = g->null_value_type;
      staged[i].value_framing = g->value_framing;
      staged[i].json = &g->json;
      if ((staged[i].rc = decode_fetch(partitions[i], (const uint8_t*)datas[i], nbytes[i], &staged[i])) != SGR_OK) return;
      from = &staged[i].ps;
    }
  };
  const bool timing = getenv("SGR_INGEST_TIMING") != nullptr;
  const auto t0 = std::chrono::steady_clock::now();
  const uint32_t n_thr = std::max(1u, std::min<uint32_t>(threads ? threads : 1, (uint32_t)chains.size()));
  g->workers.run((uint32_t)chains.size(), n_thr, [&](uint32_t c) { run_chain(*chains[c]); });
  for (uint32_t i = 0; i < n; ++i)
    if (staged[i].rc != SGR_OK) { g->last_error = staged[i].err; return staged[i].rc; }
  const auto t1 = std::chrono::steady_clock::now();
  size_t add = 0, n_rec_total = 0;
  for (uint32_t i = 0; i < n; ++i) { add += staged[i].recs.size(); n_rec_total += staged[i].keys.size(); }
  if (!g->pending.grow_to(g->pending.n + add)) return ifail(g, SGR_ERR_OOM, "pending log of %zu bytes", g->pending.n + add);
  // The dictionary addresses its id arena with 32-bit offsets and keeps bit 31 of an index for provisional slots: refuse, BEFORE
  // anything is probed or admitted, a call that could carry it past either bound (conservative: every id of the call counted as
  // new). Without this a restore of more than 4 GiB of id bytes or 2^31 ids would wrap silently and fold events into the wrong
  // aggregates (ADVICE r1).
  {
    uint64_t id_bytes = 0;
    for (uint32_t i = 0; i < n; ++i) for (const KeyRef& k : staged[i].keys) id_bytes += k.len;
    if (g->dict.arena_bytes() + id_bytes >= g->max_id_bytes || g->dict.size() + n_rec_total >= g->max_ids)
      return ifail(g, SGR_ERR_CAPACITY, "id dictionary full: %llu ids / %llu id bytes held, this call may add %zu / %llu (limits 2^31 ids, 4 GiB)",
                   (unsigned long long)g->dict.size(), (unsigned long long)g->dict.arena_bytes(), n_rec_total, (unsigned long long)id_bytes);
  }
  // ids -> dense indices: shards probed in parallel, new ids admitted serially in arrival order, slots published in parallel
  const uint32_t n_workers = std::max(1u, std::min<uint32_t>(std::min<uint32_t>(threads ? threads : 1, (uint32_t)ShardedDict::kShards),
                                                             (uint32_t)(n_rec_total / 1024 + 1)));   // a worker per ~1k ids at least
  if (g->news.size() < n_workers) g->news.resize(n_workers);
  if (g->probed.size() < n_workers) g->probed.resize(n_workers);
  g->workers.run(n_workers, n_workers, [&](uint32_t t) { probe_shards(g, staged, n, t, n_workers); });
  admit_new_keys(g, staged, n_workers);
  g->workers.run(n_workers, n_workers, [&](uint32_t t) { for (const auto& nk : g->news[t]) g->dict.publish(nk); });
  std::vector<size_t> at(n);
  for (uint32_t i = 0; i < n; ++i) { at[i] = g->pending.n; g->pending.n += staged[i].recs.size(); }
  g->workers.run(n, std::max(1u, threads), [&](uint32_t i) { place_fetch(g, g->pending.p + at[i], &staged[i], i, n_workers); });
  for (uint32_t i = 0; i < n; ++i) {
    commit_fetch(g, partitions[i], &staged[i]);
    if (stats) stats[i] = staged[i].st;
  }
  if (timing) {
    const auto t2 = std::chrono::steady_clock::now();
    fprintf(stderr, "[sgr_ingest] %u fetches on %u threads: decode %.3f ms, intern+append %.3f ms\n", n, n_thr,
            std::chrono::duration<double, std::milli>(t1 - t0).count(), std::chrono::duration<double, std::milli>(t2 - t1).count());
  }
  return SGR_OK;
}

int32_t sgr_ingest_record_batches(sgr_ingest* g, int32_t partition, const void* data, uint64_t nbytes, sgr_ingest_stats* stats) {
  if (!g || (!data && nbytes)) return ifail(g, SGR_ERR_INVALID, "null argument");
  const void* d[1] = {data};
  return sgr_ingest_record_batches_mt(g, 1, &partition, d, &nbytes, 1, stats);
}

int32_t sgr_ingest_set_allocator(sgr_ingest* g, void* (*alloc_fn)(size_t), void (*free_fn)(void*)) {
  if (!g || !alloc_fn || !free_fn) return ifail(g, SGR_ERR_INVALID, "null argument");
  if (g->pending.alloc_fn == alloc_fn && g->pending.free_fn == free_fn) return SGR_OK;
  const size_t c = g->pending.cap ? g->pending.cap : (1u << 16);
  if (!g->pending.move_to(c, alloc_fn, free_fn)) return ifail(g, SGR_ERR_OOM, "pending log of %zu bytes", c);
  return SGR_OK;
}

int32_t sgr_ingest_pending(sgr_ingest* g, const void** records, uint64_t* n_records) {
  if (!g || !records || !n_records) return ifail(g, SGR_ERR_INVALID, "null argument");
  *records = g->pending.n ? g->pending.p : nullptr;
  *n_records = g->pending.n / 64;
  return SGR_OK;
}

int32_t sgr_ingest_keys(sgr_ingest* g, const uint8_t** keys, const uint32_t** key_offsets, uint64_t* n_keys) {
  if (!g || !keys || !key_offsets || !n_keys) return ifail(g, SGR_ERR_INVALID, "null argument");
  *keys = g->dict.bytes(); *key_offsets = g->dict.offsets(); *n_keys = g->dict.size();
  return SGR_OK;
}

int32_t sgr_ingest_mark_folded(sgr_ingest* g) {
  if (!g) return SGR_ERR_INVALID;
  g->pending.n = 0;
  for (auto& kv : g->parts) kv.second.folded_next = kv.second.decoded_next;
  g->keys_at_mark = g->dict.size();
  return SGR_OK;
}

int32_t sgr_ingest_offsets(sgr_ingest* g, int32_t partition, int64_t* decoded_next, int64_t* folded_next) {
  return g ? partition_offsets(g->parts, partition, decoded_next, folded_next) : SGR_ERR_INVALID;
}

int32_t sgr_ingest_get_stats(sgr_ingest* g, sgr_ingest_stats* out) {
  if (!g || !out) return ifail(g, SGR_ERR_INVALID, "null argument");
  *out = g->total;
  return SGR_OK;
}

}  // extern "C"
