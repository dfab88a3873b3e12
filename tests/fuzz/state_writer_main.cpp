// Host harness for the JSON state writer (surge_b200/csrc/state_writer.h), built by tests/test_state_writer_cpu.py with
// g++ -fsanitize=address,undefined. The test compares what it writes with oracle/state_json.py byte for byte.
//
//   state_writer_main f64 IN OUT      IN: u64 n, n x u64 double bits. OUT per double: u32 len (0xffffffff: refused as not finite)
//                                     + the F64 member's text.
//   state_writer_main values IN OUT   IN: u32 user, u32 n_members, per member u32 len + name, u32 kind, u32 off, u32 len; u32 n_rows,
//                                     per row u32 has_id, u32 len + id, user program bytes. OUT per row: u32 status (0, or
//                                     member << 8 | reason), u32 len + the value. Every value is parsed back by the device
//                                     restore's parser (vf::json_pack<STATE>, the writer's table without its ID member) and must
//                                     give the row again (doubles by ==); stdout's last line counts the rows that did not.
// Each id, row and value sits alone in a heap block of exactly its size, so a read or write past it is an ASan report.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../surge_b200/csrc/state_writer.h"
#include "../../surge_b200/csrc/value_framing.h"

using namespace sgr;

namespace {
struct Reader {
  FILE* f;
  uint32_t u32() { uint32_t v = 0; if (fread(&v, 4, 1, f) != 1) { fprintf(stderr, "short input\n"); exit(2); } return v; }
  uint64_t u64() { uint64_t v = 0; if (fread(&v, 8, 1, f) != 1) { fprintf(stderr, "short input\n"); exit(2); } return v; }
  std::string str() { const uint32_t n = u32(); std::string s(n, '\0'); if (n && fread(&s[0], 1, n, f) != n) { fprintf(stderr, "short input\n"); exit(2); } return s; }
};

void put32(FILE* o, uint32_t v) { fwrite(&v, 4, 1, o); }

int run_f64(Reader& r, FILE* o) {
  const uint64_t n = r.u64();
  for (uint64_t i = 0; i < n; ++i) {
    const uint64_t bits = r.u64();
    if (!sw::f64_finite(bits)) { put32(o, 0xffffffffu); continue; }
    const uint32_t len = sw::f64_len(bits);
    uint8_t* buf = (uint8_t*)malloc(len);
    uint8_t* end = sw::f64_write(buf, bits);
    if ((uint32_t)(end - buf) != len) { fprintf(stderr, "f64 %016llx: length %u, wrote %ld\n", (unsigned long long)bits, len, (long)(end - buf)); exit(3); }
    put32(o, len);
    fwrite(buf, 1, len, o);
    free(buf);
  }
  printf("f64 %llu\n", (unsigned long long)n);
  return 0;
}

int run_values(Reader& r, FILE* o) {
  const uint32_t user = r.u32(), nm = r.u32();
  std::vector<sw::Member> mem;
  std::vector<uint8_t> lits;
  std::string names;
  std::vector<vf::Field> fields;   // the restore's table: the writer's without its ID member
  for (uint32_t i = 0; i < nm; ++i) {
    const std::string name = r.str();
    sw::Member m{};
    m.kind = (uint8_t)r.u32(); m.off = (uint16_t)r.u32(); m.len = r.u32();
    m.lit_off = (uint32_t)lits.size();
    lits.push_back(i ? ',' : '{');
    std::vector<uint8_t> q(sw::str_len((const uint8_t*)name.data(), name.size()));
    sw::str_write(q.data(), (const uint8_t*)name.data(), name.size());
    lits.insert(lits.end(), q.begin(), q.end());
    lits.push_back(':');
    m.lit_len = (uint32_t)lits.size() - m.lit_off;
    mem.push_back(m);
    if (m.kind != sw::K_ID) {
      const uint32_t size = m.kind == sw::K_I32 ? 4u : m.kind == sw::K_UUID ? 16u : m.kind == sw::K_PSTR ? m.len : 8u;
      fields.push_back(vf::Field{(uint32_t)names.size(), (uint32_t)name.size(), m.kind, m.off, size});
      names += name;
    }
  }
  const vf::Class cls{0, 0, 0, 0, (uint32_t)fields.size()};
  const vf::Table table{(const uint8_t*)names.data(), &cls, fields.data(), 1, 0, 0, -1};
  const uint32_t n = r.u32();
  uint64_t bad = 0, written = 0, refused = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const bool has_id = r.u32() != 0;
    const std::string id_s = r.str();
    uint8_t* id = (uint8_t*)malloc(id_s.size() ? id_s.size() : 1);
    memcpy(id, id_s.data(), id_s.size());
    uint8_t* row = (uint8_t*)malloc(user);
    if (fread(row, 1, user, r.f) != user) { fprintf(stderr, "short input\n"); exit(2); }
    uint64_t len = 1;   // "}"
    uint32_t status = 0;
    for (uint32_t k = 0; k < nm && !status; ++k) {
      uint32_t why = sw::OK;
      len += sw::member_len(mem[k], row, id, id_s.size(), has_id, &why);
      if (why) status = k << 8 | why;
    }
    if (status) {
      put32(o, status); put32(o, 0);
      ++refused;
    } else {
      uint8_t* val = (uint8_t*)malloc(len);
      uint8_t* p = val;
      for (uint32_t k = 0; k < nm; ++k) p = sw::member_write(p, mem[k], lits.data(), row, id, id_s.size());
      *p++ = '}';
      if ((uint64_t)(p - val) != len) { fprintf(stderr, "row %u: length %llu, wrote %ld\n", i, (unsigned long long)len, (long)(p - val)); exit(3); }
      put32(o, 0); put32(o, (uint32_t)len);
      fwrite(val, 1, len, o);
      ++written;
      // parse back
      uint8_t back[vf::kStateRowMax];
      const uint32_t e = vf::json_pack<vf::STATE>(table, val, (uint32_t)len, back);
      bool same = e == vf::OK;
      for (uint32_t k = 0; k < nm && same; ++k) {
        const sw::Member& m = mem[k];
        if (m.kind == sw::K_ID) continue;
        if (m.kind == sw::K_F64) {
          double a, b;
          memcpy(&a, row + m.off, 8); memcpy(&b, back + m.off, 8);
          same = a == b;
        } else if (m.kind == sw::K_PSTR) {
          same = memcmp(row + m.off, back + m.off, 1u + row[m.off]) == 0;
        } else {
          same = memcmp(row + m.off, back + m.off, m.kind == sw::K_I32 ? 4 : m.kind == sw::K_UUID ? 16 : 8) == 0;
        }
      }
      if (!same) {
        if (bad < 10) fprintf(stderr, "row %u: parse-back differs (reason %u): %.*s\n", i, e, (int)len, (const char*)val);
        ++bad;
      }
      free(val);
    }
    free(row);
    free(id);
  }
  printf("values %u written %llu refused %llu parse_back_mismatches %llu\n", n, (unsigned long long)written, (unsigned long long)refused,
         (unsigned long long)bad);
  return 0;
}
}  // namespace

int main(int argc, char** argv) {
  if (argc != 4) { fprintf(stderr, "usage: %s f64|values IN OUT\n", argv[0]); return 2; }
  FILE* f = fopen(argv[2], "rb");
  FILE* o = fopen(argv[3], "wb");
  if (!f || !o) { fprintf(stderr, "cannot open files\n"); return 2; }
  Reader r{f};
  const int rc = strcmp(argv[1], "f64") == 0 ? run_f64(r, o) : run_values(r, o);
  fclose(f);
  fclose(o);
  return rc;
}
