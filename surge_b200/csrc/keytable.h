// keytable.h — host-side aggregate-id -> dense index table behind sgr_get.
// The fold never reads keys; this serves the recovery read
// AggregateStateStoreKafkaStreams.getAggregateBytes(aggregateId)
// (modules/common/src/main/scala/surge/kafka/streams/AggregateStateStoreKafkaStreams.scala:83-85),
// which the reference calls from a 32-thread pool: find() is read-only and lock free once built.
#pragma once
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

namespace sgr {

class KeyTable {
 public:
  bool build(const uint8_t* keys, const uint32_t* offs, uint64_t n, std::string* err) {
    std::vector<uint8_t> bytes(keys, keys + (n ? offs[n] : 0));
    std::vector<uint32_t> o(offs, offs + n + 1);
    uint64_t cap = 16;
    while (cap < n * 2 + 1) cap <<= 1;
    std::vector<int64_t> slots(cap, -1);
    for (uint64_t i = 0; i < n; ++i) {
      if (o[i + 1] < o[i]) { if (err) *err = "key_offsets not monotone"; return false; }
      const uint8_t* k = bytes.data() + o[i];
      const uint32_t len = o[i + 1] - o[i];
      uint64_t h = hash(k, len) & (cap - 1);
      while (slots[h] >= 0) {
        const uint64_t j = (uint64_t)slots[h];
        if (o[j + 1] - o[j] == len && memcmp(bytes.data() + o[j], k, len) == 0) {
          if (err) *err = "duplicate aggregate id in key table"; return false;
        }
        h = (h + 1) & (cap - 1);
      }
      slots[h] = (int64_t)i;
    }
    bytes_.swap(bytes); offs_.swap(o); slots_.swap(slots); n_ = n;
    return true;
  }
  // returns the dense index of the key, or -1
  int64_t find(const uint8_t* k, uint32_t len) const {
    if (slots_.empty()) return -1;
    const uint64_t cap = slots_.size();
    uint64_t h = hash(k, len) & (cap - 1);
    while (slots_[h] >= 0) {
      const uint64_t j = (uint64_t)slots_[h];
      if (offs_[j + 1] - offs_[j] == len && memcmp(bytes_.data() + offs_[j], k, len) == 0) return (int64_t)j;
      h = (h + 1) & (cap - 1);
    }
    return -1;
  }
  uint64_t size() const { return n_; }
  // the table's ids back to back: key i = bytes()[offsets()[i] .. offsets()[i + 1])
  const uint8_t* bytes() const { return bytes_.data(); }
  const uint32_t* offsets() const { return offs_.data(); }
  // key i as (pointer, length)
  const uint8_t* key(uint64_t i, uint32_t* len) const { *len = offs_[i + 1] - offs_[i]; return bytes_.data() + offs_[i]; }

 private:
  static uint64_t hash(const uint8_t* k, uint32_t len) {  // FNV-1a 64 with a final mix
    uint64_t h = 1469598103934665603ull;
    for (uint32_t i = 0; i < len; ++i) { h ^= k[i]; h *= 1099511628211ull; }
    h ^= h >> 32; h *= 0x9e3779b97f4a7c15ull; h ^= h >> 29;
    return h;
  }
  std::vector<uint8_t> bytes_;
  std::vector<uint32_t> offs_;
  std::vector<int64_t> slots_;
  uint64_t n_ = 0;
};

}  // namespace sgr
