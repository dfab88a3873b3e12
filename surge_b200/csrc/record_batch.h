// record_batch.h — the RecordBatch v2 header walk (KIP-98) and the read_committed bookkeeping of org.apache.kafka consumers, one
// host-only copy for the host decoder (ingest.cpp) and the device ingest (dingest.cu): same refusals, same partition positions.
#pragma once
#include <stdarg.h>
#include <stdio.h>
#include <algorithm>
#include <map>
#include <string>
#include <unordered_set>
#include <vector>
#include "../../include/sgr.h"

namespace sgr {

inline uint16_t be16(const uint8_t* p) { return (uint16_t)((p[0] << 8) | p[1]); }
inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
inline uint64_t be64(const uint8_t* p) { return ((uint64_t)be32(p) << 32) | be32(p + 4); }
constexpr uint64_t kBatchHeader = 61;  // baseOffset .. recordsCount

struct Cursor {
  const uint8_t* p; uint64_t n; uint64_t pos = 0; bool ok = true;
  Cursor(const uint8_t* p_, uint64_t n_) : p(p_), n(n_) {}
  int64_t varlong() {  // ByteUtils.readVarlong: zig-zag, at most 10 bytes
    if (pos < n && !(p[pos] & 0x80)) { const uint64_t b = p[pos++]; return (int64_t)(b >> 1) ^ -(int64_t)(b & 1); }
    uint64_t v = 0; int shift = 0;
    for (int i = 0; i < 10; ++i) {
      if (pos >= n) { ok = false; return 0; }
      const uint8_t b = p[pos++];
      v |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return (int64_t)(v >> 1) ^ -(int64_t)(v & 1);
      shift += 7;
    }
    ok = false; return 0;
  }
  int32_t varint() {  // ByteUtils.readVarint: zig-zag, at most 5 bytes
    if (pos < n && !(p[pos] & 0x80)) { const uint32_t b = p[pos++]; return (int32_t)(b >> 1) ^ -(int32_t)(b & 1); }
    uint32_t v = 0; int shift = 0;
    for (int i = 0; i < 5; ++i) {
      if (pos >= n) { ok = false; return 0; }
      const uint8_t b = p[pos++];
      v |= (uint32_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return (int32_t)(v >> 1) ^ -(int32_t)(v & 1);
      shift += 7;
    }
    ok = false; return 0;
  }
  const uint8_t* bytes(uint64_t k) {
    if (k > n - pos) { ok = false; return nullptr; }
    const uint8_t* r = p + pos; pos += k; return r;
  }
};

struct BatchHeader {            // frame_batch fills b, total, base_offset and stored_crc; read_batch_fields the rest
  const uint8_t* b = nullptr;
  uint64_t total = 0;           // 12 + batchLength; 0 when no whole batch is left in the fetch
  int64_t base_offset = 0, last_offset = 0, producer_id = 0;
  int32_t records_count = 0, codec = 0;
  uint32_t stored_crc = 0;      // of attributes .. the batch's end
  bool transactional = false, control = false;
};

inline int32_t set_error(std::string* err, int32_t code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  *err = buf;
  return code;
}

// The batch at buf + pos, its length and magic checked. SGR_OK with h->total == 0 when no whole batch is left: a fetch response
// may end with a partial batch, which is not an error, the next fetch repeats it.
inline int32_t frame_batch(int32_t partition, const uint8_t* buf, uint64_t nbytes, uint64_t pos, BatchHeader* h, std::string* err) {
  h->total = 0;
  if (nbytes - pos < 12) return SGR_OK;
  h->b = buf + pos;
  h->base_offset = (int64_t)be64(h->b);
  const int32_t batch_length = (int32_t)be32(h->b + 8);
  if (batch_length < (int32_t)(kBatchHeader - 12)) return set_error(err, SGR_ERR_INVALID, "partition %d offset %lld: batch length %d is smaller than a v2 header", partition, (long long)h->base_offset, batch_length);
  if (nbytes - pos < 12ull + (uint32_t)batch_length) return SGR_OK;
  const int8_t magic = (int8_t)h->b[16];
  if (magic != 2) return set_error(err, SGR_ERR_UNSUPPORTED, "partition %d offset %lld: message format v%d (only RecordBatch magic 2 is decoded)", partition, (long long)h->base_offset, (int)magic);
  h->total = 12ull + (uint32_t)batch_length;
  h->stored_crc = be32(h->b + 17);
  return SGR_OK;
}

// The rest of a framed header; the host decoder checks the CRC before it.
inline int32_t read_batch_fields(int32_t partition, BatchHeader* h, std::string* err) {
  const uint16_t attrs = be16(h->b + 21);
  const int32_t last_offset_delta = (int32_t)be32(h->b + 23);
  h->producer_id = (int64_t)be64(h->b + 43);
  h->records_count = (int32_t)be32(h->b + 57);
  if (last_offset_delta < 0 || h->records_count < 0) return set_error(err, SGR_ERR_INVALID, "partition %d offset %lld: negative lastOffsetDelta / recordsCount", partition, (long long)h->base_offset);
  h->last_offset = h->base_offset + last_offset_delta;
  h->codec = attrs & 7;
  h->transactional = attrs & 0x10; h->control = attrs & 0x20;
  return SGR_OK;
}

struct PartitionState {
  int64_t decoded_next = 0;   // next offset this partition expects (last decoded batch's lastOffset + 1)
  int64_t folded_next = 0;    // everything below this offset is inside the state table
  bool seen = false;
  std::vector<std::pair<int64_t, int64_t>> aborted;  // (first_offset, producer_id), ascending first_offset, not yet reached
  std::unordered_set<int64_t> aborting;              // producer ids inside an aborted transaction right now

  // the aborted transactions a fetch response announces
  void announce_aborted(const int64_t* producer_ids, const int64_t* first_offsets, uint64_t n) {
    for (uint64_t i = 0; i < n; ++i) aborted.emplace_back(first_offsets[i], producer_ids[i]);
    std::sort(aborted.begin(), aborted.end());
  }
  // an announced aborted transaction starts when the log reaches its first offset; true: a data batch the consumer skips
  bool reach(const BatchHeader& h) {
    while (!aborted.empty() && aborted.front().first <= h.last_offset) { aborting.insert(aborted.front().second); aborted.erase(aborted.begin()); }
    return !h.control && h.transactional && aborting.count(h.producer_id);
  }
  // a control batch's records, decompressed: an ABORT marker (key int16 version, int16 type 0) ends the producer's transaction
  void apply_control(const BatchHeader& h, const uint8_t* recs, uint64_t n) {
    Cursor c(recs, n);
    c.varint(); c.bytes(1); c.varlong(); c.varint();   // length, attributes, timestampDelta, offsetDelta
    const int32_t kl = c.varint();
    const uint8_t* k = (c.ok && kl >= 4) ? c.bytes((uint64_t)kl) : nullptr;
    if (k && c.ok && be16(k + 2) == 0) aborting.erase(h.producer_id);
  }
  void close(const BatchHeader& h) {
    if (!seen || h.last_offset + 1 > decoded_next) decoded_next = h.last_offset + 1;
    seen = true;
  }
};

inline int32_t partition_offsets(const std::map<int32_t, PartitionState>& parts, int32_t partition, int64_t* decoded_next, int64_t* folded_next) {
  auto it = parts.find(partition);
  if (decoded_next) *decoded_next = it == parts.end() ? 0 : it->second.decoded_next;
  if (folded_next) *folded_next = it == parts.end() ? 0 : it->second.folded_next;
  return SGR_OK;
}

// every counter but n_trailing_bytes, which describes one call only
inline void add_stats(sgr_ingest_stats* t, const sgr_ingest_stats& s) {
  t->n_bytes += s.n_bytes; t->n_batches += s.n_batches; t->n_records += s.n_records; t->n_markers += s.n_markers; t->n_null_values += s.n_null_values;
  t->n_control_batches += s.n_control_batches; t->n_aborted_batches += s.n_aborted_batches; t->n_aborted_records += s.n_aborted_records;
  t->n_duplicates += s.n_duplicates; t->n_new_keys += s.n_new_keys; t->n_compressed_bytes += s.n_compressed_bytes; t->n_decompressed_bytes += s.n_decompressed_bytes;
}

// The bytes a JSON packer's member fills, by kind; 0 when it has no name, an unknown kind, or is not whole 4-byte words.
inline uint32_t json_member_size(const sgr_json_field& jf) {
  const uint32_t size = jf.kind == SGR_JSON_I32 ? 4u : jf.kind == SGR_JSON_UUID ? 16u : jf.kind == SGR_JSON_PSTR ? jf.len : 8u;
  return jf.name && jf.kind <= SGR_JSON_PSTR && jf.dst_off % 4 == 0 && size >= 4 && size % 4 == 0 ? size : 0u;
}
// an event's member may land on the sequence number (+4, Int only) or anywhere in the payload (+16 .. +64); never on type or agg
inline bool json_event_slot_ok(const sgr_json_field& jf, uint32_t size) {
  return (jf.dst_off == 4 && jf.kind == SGR_JSON_I32) || (jf.dst_off >= 16 && jf.dst_off + size <= 64);
}

}  // namespace sgr
