// Host harness for the state writer's protobuf wrapping (surge_b200/csrc/state_writer.h, wrap_*), built for the HOST by
// tests/test_multilanguage_framing_cpu.py with g++ -fsanitize=address,undefined.
//
//   state_wrap_main IN OUT   IN (little endian): u32 n, per case u32 len + id bytes, u32 len + JSON bytes. For each case the
//                            wrapped value is laid out as the device's two passes lay it out: wrap_len gives its size (a heap
//                            block of exactly that size, so a write past it is an ASan report), wrap_json_len must give the JSON
//                            length back from that size, wrap_head_write writes the wrapper and the JSON follows. OUT: per case
//                            u32 len + the wrapped bytes.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>

#include "../../surge_b200/csrc/state_writer.h"

namespace {
bool rd_u32(FILE* f, uint32_t* v) { return fread(v, 4, 1, f) == 1; }
bool rd_str(FILE* f, std::string* s) {
  uint32_t n = 0;
  if (!rd_u32(f, &n)) return false;
  s->assign(n, '\0');
  return !n || fread(&(*s)[0], 1, n, f) == n;
}
}  // namespace

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) return 2;
  uint32_t n = 0;
  if (!rd_u32(in, &n)) return 2;
  uint32_t bad = 0;
  for (uint32_t i = 0; i < n; ++i) {
    std::string id, json;
    if (!rd_str(in, &id) || !rd_str(in, &json)) return 2;
    const uint64_t total = sgr::sw::wrap_len(id.size(), json.size());
    if (sgr::sw::wrap_json_len(id.size(), total) != json.size()) {
      printf("MISMATCH case %u: wrap_json_len(%zu, %llu) != %zu\n", i, id.size(), (unsigned long long)total, json.size());
      ++bad;
    }
    uint8_t* v = (uint8_t*)malloc(total);
    uint8_t* o = sgr::sw::wrap_head_write(v, (const uint8_t*)id.data(), id.size(), json.size());
    if ((uint64_t)(o - v) + json.size() != total) { printf("MISMATCH case %u: header of %lld bytes\n", i, (long long)(o - v)); ++bad; }
    else memcpy(o, json.data(), json.size());
    const uint32_t len = (uint32_t)total;
    fwrite(&len, 4, 1, out);
    fwrite(v, 1, total, out);
    free(v);
  }
  fclose(in);
  fclose(out);
  printf("cases %u mismatches %u\n", n, bad);
  return 0;
}
