// Differential harness for protobuf-wrapped JSON values (SGR_VALUE_PROTOBUF_JSON) through the device ingest's conversion
// (surge_b200/csrc/value_framing.h), built for the HOST by tests/test_multilanguage_framing_cpu.py with
// g++ -fsanitize=address,undefined together with surge_b200/csrc/ingest.cpp.
//
//   pbjson_framing_main CORPUS   every value goes through the host decoder (one single-record batch through
//                                sgr_ingest_record_batches, framing 3 after sgr_ingest_set_json_packer) and through
//                                vf::convert(PROTOBUF_JSON) + the 8..56 length check. Both must refuse with the same text or
//                                accept with the same 56 bytes.
// CORPUS (little endian): u32 len + discriminator, i32 unknown_type, u32 n_events, per event u32 len + class name,
// u32 event_type, u32 n_fields, per field u32 len + name, u32 kind, u32 dst_off, u32 len; then u32 n_values, per value
// u32 len + bytes. Each value sits alone in a heap block of exactly its size, so a read past it is an ASan report.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/sgr.h"
#include "../../surge_b200/csrc/value_framing.h"

namespace {
struct Reader {
  FILE* f;
  uint32_t u32() { uint32_t v = 0; if (fread(&v, 4, 1, f) != 1) { fprintf(stderr, "short corpus\n"); exit(2); } return v; }
  std::string str() { const uint32_t n = u32(); std::string s(n, '\0'); if (n && fread(&s[0], 1, n, f) != n) { fprintf(stderr, "short corpus\n"); exit(2); } return s; }
};

void put_be(std::vector<uint8_t>& b, uint64_t v, int n) { for (int k = n - 1; k >= 0; --k) b.push_back((uint8_t)(v >> (8 * k))); }
void put_varint(std::vector<uint8_t>& b, int64_t v) {   // zig-zag, as org.apache.kafka.common.utils.ByteUtils
  uint64_t z = ((uint64_t)v << 1) ^ (uint64_t)(v >> 63);
  while (z >= 0x80) { b.push_back((uint8_t)(z | 0x80)); z >>= 7; }
  b.push_back((uint8_t)z);
}

// one RecordBatch v2, no compression, one record with key "k" and the value
std::vector<uint8_t> batch_of(int64_t base_offset, const std::string& value) {
  std::vector<uint8_t> rec;
  rec.push_back(0);
  put_varint(rec, 0);
  put_varint(rec, 0);
  put_varint(rec, 1); rec.push_back('k');
  put_varint(rec, (int64_t)value.size()); rec.insert(rec.end(), value.begin(), value.end());
  put_varint(rec, 0);
  std::vector<uint8_t> recs;
  put_varint(recs, (int64_t)rec.size());
  recs.insert(recs.end(), rec.begin(), rec.end());
  std::vector<uint8_t> b;
  put_be(b, (uint64_t)base_offset, 8);
  put_be(b, 49 + recs.size(), 4);    // batchLength
  put_be(b, 0, 4);                   // partitionLeaderEpoch
  b.push_back(2);                    // magic
  put_be(b, 0, 4);                   // crc (below)
  put_be(b, 0, 2);                   // attributes
  put_be(b, 0, 4);                   // lastOffsetDelta
  put_be(b, 0, 8); put_be(b, 0, 8);  // timestamps
  put_be(b, ~0ull, 8); put_be(b, 0xffff, 2); put_be(b, 0xffffffffu, 4);
  put_be(b, 1, 4);                   // recordsCount
  b.insert(b.end(), recs.begin(), recs.end());
  const uint32_t crc = sgr_crc32c(b.data() + 21, b.size() - 21);
  for (int k = 0; k < 4; ++k) b[17 + k] = (uint8_t)(crc >> (8 * (3 - k)));
  return b;
}
}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  Reader rd{f};
  const std::string disc = rd.str();
  const int32_t unknown_type = (int32_t)rd.u32();
  const uint32_t n_events = rd.u32();
  std::vector<std::string> names;   // keeps the C strings of the host table alive
  names.reserve(1 + n_events * (1 + SGR_JSON_MAX_FIELDS));
  std::vector<sgr_json_event> events(n_events);
  std::string arena = disc;
  std::vector<sgr::vf::Class> classes;
  std::vector<sgr::vf::Field> fields;
  for (uint32_t i = 0; i < n_events; ++i) {
    sgr_json_event& e = events[i];
    memset(&e, 0, sizeof e);
    names.push_back(rd.str());
    e.type_name = names.back().c_str();
    e.event_type = rd.u32();
    e.n_fields = rd.u32();
    classes.push_back(sgr::vf::Class{(uint32_t)arena.size(), (uint32_t)names.back().size(), e.event_type, (uint32_t)fields.size(), e.n_fields});
    arena += names.back();
    for (uint32_t j = 0; j < e.n_fields; ++j) {
      names.push_back(rd.str());
      e.fields[j].name = names.back().c_str();
      e.fields[j].kind = (uint8_t)rd.u32();
      e.fields[j].dst_off = (uint16_t)rd.u32();
      e.fields[j].len = rd.u32();
      const uint32_t size = e.fields[j].kind == SGR_JSON_I32 ? 4u : e.fields[j].kind == SGR_JSON_UUID ? 16u : e.fields[j].kind == SGR_JSON_PSTR ? e.fields[j].len : 8u;
      fields.push_back(sgr::vf::Field{(uint32_t)arena.size(), (uint32_t)names.back().size(), e.fields[j].kind, e.fields[j].dst_off, size});
      arena += names.back();
    }
  }
  sgr_ingest* g = nullptr;
  if (sgr_ingest_create(&g) != SGR_OK) return 2;
  if (sgr_ingest_set_json_packer(g, disc.c_str(), events.data(), n_events, unknown_type) != SGR_OK ||
      sgr_ingest_set_value_framing(g, SGR_VALUE_PROTOBUF_JSON) != SGR_OK) {
    fprintf(stderr, "host set-up refused: %s\n", sgr_ingest_last_error(g));
    return 2;
  }
  const sgr::vf::Table t{(const uint8_t*)arena.data(), classes.data(), fields.data(), (uint32_t)classes.size(), 0, (uint32_t)disc.size(),
                         unknown_type < 0 ? -1 : unknown_type};

  const uint32_t n_values = rd.u32();
  uint64_t accepted = 0, refused = 0, bad = 0;
  for (uint32_t i = 0; i < n_values; ++i) {
    const std::string value = rd.str();
    const std::vector<uint8_t> b = batch_of((int64_t)i, value);
    std::string host_err;
    uint8_t host_out[56] = {0};
    if (sgr_ingest_record_batches(g, 0, b.data(), b.size(), nullptr) == SGR_OK) {
      const void* recs = nullptr; uint64_t n = 0;
      if (sgr_ingest_pending(g, &recs, &n) != SGR_OK || n != 1) { fprintf(stderr, "case %u: %llu pending records\n", i, (unsigned long long)n); return 2; }
      memcpy(host_out, recs, 8);
      memcpy(host_out + 8, (const uint8_t*)recs + 16, 48);
      sgr_ingest_mark_folded(g);
    } else {
      host_err = sgr_ingest_last_error(g);
      const size_t colon = host_err.find(": ");   // "partition 0 offset N: <reason>"
      host_err = colon == std::string::npos ? host_err : host_err.substr(colon + 2);
    }
    uint8_t* v = value.empty() ? nullptr : (uint8_t*)malloc(value.size());
    if (v) memcpy(v, value.data(), value.size());
    uint8_t out[56];
    const uint8_t* pv = nullptr; uint32_t plen = 0;
    const uint32_t why = sgr::vf::convert(sgr::vf::PROTOBUF_JSON, t, v, (uint32_t)value.size(), out, &pv, &plen);
    std::string dev_err;
    uint8_t dev_out[56] = {0};
    if (why) dev_err = std::string(why == sgr::vf::NOT_PROTOBUF ? "" : "JSON event: ") + sgr::vf::reason_text(why);
    else if (plen != 56) dev_err = "a JSON event packs to 56 bytes";
    else memcpy(dev_out, pv, plen);
    free(v);
    if (host_err != dev_err || (host_err.empty() && memcmp(host_out, dev_out, 56) != 0)) {
      if (bad < 20) printf("MISMATCH case %u (%zu bytes): host [%s] header [%s]\n", i, value.size(), host_err.c_str(), dev_err.c_str());
      ++bad;
    }
    if (host_err.empty()) ++accepted; else ++refused;
  }
  sgr_ingest_destroy(g);
  fclose(f);
  printf("cases %u accepted %llu refused %llu mismatches %llu\n", n_values, (unsigned long long)accepted, (unsigned long long)refused, (unsigned long long)bad);
  return 0;
}
