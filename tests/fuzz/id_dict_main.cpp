// Host harness for the device id dictionary (surge_b200/csrc/id_dict.cuh), built by tests/test_id_dict_cpu.py with
// g++ -fsanitize=address,undefined. The header's device functions run here single-threaded, with plain stand-ins for the atomics
// and the cache-hinted loads; the test compares what they return with a Python dict.
//
//   id_dict_main hash IN OUT     IN: u32 n, n x (u32 len + bytes). OUT: u64 hash_id per id.
//   id_dict_main intern IN OUT   IN: u64 slots, u64 max_keys, u64 arena_cap, u32 n_ops, per op u32 kind + u32 len + id bytes.
//                                kind 0: intern(id), OUT u32 (dense index or 0xffffffff). kind 1: leave the slot a claim of id
//                                refused by a full dictionary would leave (tagged, slot_idx 0xffffffff) at the first free slot of
//                                its chain, as a concurrent claim that lost the race for the last index does; OUT u32 slot.
//                                Then OUT u64 ctl[0], ctl[1], ctl[5] and, for each dense index below min(ctl[0], max_keys),
//                                u32 len + the bytes key_ref names (len 0xffffffff for an entry never written).
//   id_dict_main index IN OUT    IN: u64 slots, u32 n + ids (dense index = position), u32 q + query ids. insert_at for every
//                                index in order, then find for every query. OUT: u64 ctl[0] (duplicates), ctl[1] (no free
//                                slot), then i64 per query.
// The tables, key_ref and the arena are heap blocks of exactly their size, so a probe or copy past them is an ASan report.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include <cuda_runtime.h>

// single-threaded stand-ins for the device intrinsics the header uses
static unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  const unsigned long long o = *p;
  if (o == cmp) *p = v;
  return o;
}
static unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; *p += v; return o; }
static unsigned int atomicExch(unsigned int* p, unsigned int v) { const unsigned int o = *p; *p = v; return o; }
template <class T> static T __ldcg(const T* p) { return *p; }
static void __threadfence() {}
static void __nanosleep(unsigned int) {}
static unsigned int __byte_perm(unsigned int x, unsigned int y, unsigned int s) {
  const uint64_t v = (uint64_t)y << 32 | x;
  unsigned int r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned int)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
  return r;
}

#define SGR_ID_DICT_HOST
#include "../../surge_b200/csrc/id_dict.cuh"

using namespace sgr;

namespace {
struct Reader {
  FILE* f;
  uint32_t u32() { uint32_t v = 0; if (fread(&v, 4, 1, f) != 1) { fprintf(stderr, "short input\n"); exit(2); } return v; }
  uint64_t u64() { uint64_t v = 0; if (fread(&v, 8, 1, f) != 1) { fprintf(stderr, "short input\n"); exit(2); } return v; }
  std::string str() { const uint32_t n = u32(); std::string s(n, '\0'); if (n && fread(&s[0], 1, n, f) != n) { fprintf(stderr, "short input\n"); exit(2); } return s; }
};

void put32(FILE* o, uint32_t v) { fwrite(&v, 4, 1, o); }
void put64(FILE* o, uint64_t v) { fwrite(&v, 8, 1, o); }

// an id alone in a heap block of exactly its length
struct Id {
  uint8_t* p; uint32_t n;
  explicit Id(const std::string& s) : p((uint8_t*)malloc(s.size() ? s.size() : 1)), n((uint32_t)s.size()) { memcpy(p, s.data(), s.size()); }
  ~Id() { free(p); }
};

struct Dict {
  DgDict d{};
  explicit Dict(uint64_t slots, uint64_t max_keys, uint64_t arena_cap) {
    d.tags = (unsigned long long*)calloc(slots, 8);
    d.slot_idx = (uint32_t*)calloc(slots, 4);
    d.key_ref = (uint2*)malloc(max_keys ? max_keys * 8 : 1);
    memset(d.key_ref, 0xff, max_keys * 8);
    d.arena = (uint8_t*)malloc(arena_cap ? arena_cap : 1);
    d.ctl = (unsigned long long*)calloc(16, 8);
    d.slots_mask = slots - 1; d.max_keys = max_keys; d.arena_cap = arena_cap;
  }
  ~Dict() { free(d.tags); free(d.slot_idx); free(d.key_ref); free(d.arena); free(d.ctl); }
};

int run_hash(Reader& r, FILE* o) {
  const uint32_t n = r.u32();
  for (uint32_t i = 0; i < n; ++i) { Id id(r.str()); put64(o, hash_id(id.p, id.n)); }
  printf("hash %u\n", n);
  return 0;
}

int run_intern(Reader& r, FILE* o) {
  const uint64_t slots = r.u64(), max_keys = r.u64(), arena_cap = r.u64();
  Dict x(slots, max_keys, arena_cap);
  const uint32_t n = r.u32();
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t kind = r.u32();
    Id id(r.str());
    if (kind == 0) { put32(o, intern(x.d, id.p, id.n)); continue; }
    const unsigned long long h = hash_id(id.p, id.n);
    uint64_t pos = h & x.d.slots_mask;
    while (x.d.tags[pos]) pos = (pos + 1) & x.d.slots_mask;
    x.d.tags[pos] = h; x.d.slot_idx[pos] = 0xffffffffu; ++x.d.ctl[5];
    put32(o, (uint32_t)pos);
  }
  put64(o, x.d.ctl[0]); put64(o, x.d.ctl[1]); put64(o, x.d.ctl[5]);
  const uint64_t nk = x.d.ctl[0] < max_keys ? x.d.ctl[0] : max_keys;
  for (uint64_t k = 0; k < nk; ++k) {
    const uint2 ref = x.d.key_ref[k];
    if (ref.x == 0xffffffffu && ref.y == 0xffffffffu) { put32(o, 0xffffffffu); continue; }
    if (((uint64_t)ref.x << 3) + ref.y > arena_cap) { fprintf(stderr, "key_ref[%llu] past the arena\n", (unsigned long long)k); return 3; }
    put32(o, ref.y);
    fwrite(x.d.arena + ((uint64_t)ref.x << 3), 1, ref.y, o);
  }
  printf("intern %u\n", n);
  return 0;
}

int run_index(Reader& r, FILE* o) {
  const uint64_t slots = r.u64();
  const uint32_t n = r.u32();
  std::vector<std::string> ids(n);
  uint64_t bytes = 0;
  for (auto& s : ids) { s = r.str(); bytes += (s.size() + 7) & ~(size_t)7; }
  Dict x(slots, n, bytes);
  for (uint32_t i = 0, off = 0; i < n; ++i) {
    memcpy(x.d.arena + off, ids[i].data(), ids[i].size());
    x.d.key_ref[i] = make_uint2(off >> 3, (uint32_t)ids[i].size());
    off += (uint32_t)((ids[i].size() + 7) & ~(size_t)7);
  }
  for (uint32_t i = 0; i < n; ++i) insert_at(x.d, i);
  put64(o, x.d.ctl[0]); put64(o, x.d.ctl[1]);
  const uint32_t q = r.u32();
  for (uint32_t i = 0; i < q; ++i) {
    Id id(r.str());
    const long long f = find(x.d, id.p, id.n);
    fwrite(&f, 8, 1, o);
  }
  printf("index %u %u\n", n, q);
  return 0;
}
}  // namespace

int main(int argc, char** argv) {
  if (argc != 4) { fprintf(stderr, "usage: %s hash|intern|index IN OUT\n", argv[0]); return 2; }
  FILE* in = fopen(argv[2], "rb");
  FILE* out = fopen(argv[3], "wb");
  if (!in || !out) { fprintf(stderr, "cannot open files\n"); return 2; }
  Reader r{in};
  const std::string mode = argv[1];
  const int rc = mode == "hash" ? run_hash(r, out) : mode == "intern" ? run_intern(r, out) : mode == "index" ? run_index(r, out) : 2;
  fclose(in);
  fclose(out);
  return rc;
}
