// value_framing.h — record value -> the 56 bytes of a packed event (u32 type, u32 seq, payload[48]), for protobuf-wrapped,
// play-json and protobuf-wrapped play-json values. One source for the device ingest's parse kernel (dingest_kernels.cu) and the CPU tests.
//
// The host decoder (ingest.cpp: the protobuf unwrap of decode_fetch, JsonScan, json_unescape and json_pack) defines the
// behaviour; this file gives the same result on every input, accepted or refused, with the same refusal text. What differs is
// the shape, so that it runs as one GPU thread per record: no allocation, no recursion (nesting is a bit stack), no libc
// (strtoll and strtod are replaced by exact integer code), and escaped strings are compared and copied as they are unescaped.
// tests/test_value_framing_cpu.py runs both on one corpus under ASan + UBSan.
//
// Doubles are correctly rounded, as strtod and java.lang.Double.parseDouble are. A number text is under 64 characters, so an
// exact method has fixed bounds: Clinger's fast path (at most 15 significant digits, |exponent| <= 22: one rounded multiply or
// divide of two exact doubles), else big integers of at most 44 32-bit words (f64_slow).
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define VF_HD __host__ __device__ __forceinline__
#define VF_HDN inline __host__ __device__ __noinline__   // (inline: one definition across translation units)
#else
#define VF_HD inline
#define VF_HDN inline
#endif

namespace sgr {
namespace vf {

// framings (include/sgr.h SGR_VALUE_*)
enum : int32_t { PACKED = 0, PROTOBUF_EVENT = 1, JSON = 2, PROTOBUF_JSON = 3 };
// member kinds (include/sgr.h SGR_JSON_*)
enum : uint8_t { K_I32 = 0, K_I64 = 1, K_F64 = 2, K_UUID = 3, K_PSTR = 4 };

enum Reason : uint32_t {
  OK = 0,
  NOT_PROTOBUF,
  NOT_OBJECT, EXPECTED_STRING, CONTROL_CHAR, UNTERMINATED, VALUE_EXPECTED, NESTING, COLON, COMMA_OR_BRACKET, BAD_NUMBER,
  UNEXPECTED_CHAR, TOO_MANY_MEMBERS, COMMA_OR_BRACE, TRAILING_BYTES, NO_DISCRIMINATOR, UNKNOWN_CLASS, STRING_MISSING,
  BAD_ESCAPE, UUID_FORM, UUID_DIGIT, PSTR_FIT, NUMBER_MISSING, NUMBER_TOO_LONG, INT_FRACTION, INT_RANGE, INT_NOT_INT,
  N_REASONS
};

// the host decoder's texts (JSON reasons follow "JSON event: " in its messages)
inline const char* reason_text(uint32_t r) {
  switch (r) {
    case NOT_PROTOBUF: return "value is not a protobuf Event";
    case NOT_OBJECT: return "the value is not a JSON object";
    case EXPECTED_STRING: return "expected a string";
    case CONTROL_CHAR: return "control character inside a string";
    case UNTERMINATED: return "unterminated string";
    case VALUE_EXPECTED: return "value expected";
    case NESTING: return "nesting too deep";
    case COLON: return "':' expected";
    case COMMA_OR_BRACKET: return "',' or a closing bracket expected";
    case BAD_NUMBER: return "malformed number";
    case UNEXPECTED_CHAR: return "unexpected character";
    case TOO_MANY_MEMBERS: return "more than 48 members";
    case COMMA_OR_BRACE: return "',' or '}' expected";
    case TRAILING_BYTES: return "bytes after the JSON object";
    case NO_DISCRIMINATOR: return "the class discriminator member is missing or not a string";
    case UNKNOWN_CLASS: return "unknown event class";
    case STRING_MISSING: return "a string member of the event is missing or not a string";
    case BAD_ESCAPE: return "bad escape in a string member";
    case UUID_FORM: return "a UUID member is not in 8-4-4-4-12 form";
    case UUID_DIGIT: return "a UUID member holds a non-hex digit";
    case PSTR_FIT: return "a string member does not fit its slot";
    case NUMBER_MISSING: return "a numeric member of the event is missing or not a number";
    case NUMBER_TOO_LONG: return "number too long";
    case INT_FRACTION: return "an integer member holds a fraction or an exponent";
    case INT_RANGE: return "integer out of range";
    case INT_NOT_INT: return "integer does not fit an Int";
  }
  return "";
}

// The registered member table (sgr_*_set_json_packer): every name is a byte range of `names`.
struct Field { uint32_t name_off, name_len; uint32_t kind; uint32_t dst_off; uint32_t len; };   // dst_off: record offset (4 or 16..63)
struct Class { uint32_t name_off, name_len; uint32_t event_type; uint32_t field_begin, n_fields; };
struct Table {
  const uint8_t* names;
  const Class* classes;
  const Field* fields;
  uint32_t n_classes;
  uint32_t disc_off, disc_len;   // disc_len == 0: no discriminator, every value is class 0
  int32_t unknown_type;          // >= 0: an unknown class name becomes this event type
};

constexpr uint32_t kMaxMembers = 48;
constexpr int kMaxDepth = 32;

VF_HD bool is_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
VF_HD bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
VF_HD int hex_val(uint8_t c) {
  if (c >= '0' && c <= '9') return c - '0';
  if (c >= 'a' && c <= 'f') return c - 'a' + 10;
  if (c >= 'A' && c <= 'F') return c - 'A' + 10;
  return -1;
}

// ------------------------------------------------------------------------------------------------------------ unescaping
// The bytes json_unescape makes of a string's raw content, one code point's UTF-8 at a time. next() gives a byte, -1 at the end
// or -2 where json_unescape fails.
struct Unesc {
  const uint8_t* b; uint32_t n, i;
  uint8_t pend[4]; uint32_t np, pi;
  VF_HD Unesc(const uint8_t* b_, uint32_t n_) : b(b_), n(n_), i(0), np(0), pi(0) {}
  VF_HD bool hex4(uint32_t at, uint32_t* v) const {
    if (at + 4 > n) return false;
    uint32_t x = 0;
    for (int k = 0; k < 4; ++k) { const int d = hex_val(b[at + k]); if (d < 0) return false; x = x * 16 + (uint32_t)d; }
    *v = x; return true;
  }
  VF_HD int next() {
    if (pi < np) return pend[pi++];
    if (i >= n) return -1;
    const uint8_t c = b[i++];
    if (c != '\\') return c;
    if (i >= n) return -2;
    switch (b[i++]) {
      case '"': return '"';  case '\\': return '\\'; case '/': return '/';
      case 'b': return '\b'; case 'f': return '\f';  case 'n': return '\n';
      case 'r': return '\r'; case 't': return '\t';
      case 'u': {
        uint32_t cp, lo;
        if (!hex4(i, &cp)) return -2;
        i += 4;   // (json_unescape's index then sits on the last hex digit: i - 1 here)
        if (cp >= 0xD800 && cp < 0xDC00 && i + 5 < n && b[i] == '\\' && b[i + 1] == 'u' && hex4(i + 2, &lo) && lo >= 0xDC00 && lo < 0xE000) {
          cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00); i += 6;
        }
        if (cp < 0x80) return (int)cp;
        np = 0; pi = 0;
        if (cp < 0x800) { pend[np++] = (uint8_t)(0xC0 | (cp >> 6)); pend[np++] = (uint8_t)(0x80 | (cp & 0x3F)); }
        else if (cp < 0x10000) { pend[np++] = (uint8_t)(0xE0 | (cp >> 12)); pend[np++] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F)); pend[np++] = (uint8_t)(0x80 | (cp & 0x3F)); }
        else { pend[np++] = (uint8_t)(0xF0 | (cp >> 18)); pend[np++] = (uint8_t)(0x80 | ((cp >> 12) & 0x3F)); pend[np++] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F)); pend[np++] = (uint8_t)(0x80 | (cp & 0x3F)); }
        return pend[pi++];
      }
      default: return -2;
    }
  }
};

// json_name_is: raw string content (escaped or not) equal to want[0, wn)? A bad escape is "not equal".
VF_HD bool name_is(const uint8_t* b, uint32_t n, bool escaped, const uint8_t* want, uint32_t wn) {
  if (!escaped) {
    if (n != wn) return false;
    for (uint32_t k = 0; k < n; ++k) if (b[k] != want[k]) return false;
    return true;
  }
  Unesc u(b, n);
  uint32_t k = 0;
  for (;;) {
    const int c = u.next();
    if (c == -2) return false;
    if (c == -1) return k == wn;
    if (k >= wn || (uint8_t)c != want[k]) return false;   // (whether the rest unescapes or not: not equal either way)
    ++k;
  }
}

// --------------------------------------------------------------------------------------------------------------- scanning
struct Member {
  uint32_t key_off, key_len, val_off, val_len;   // offsets into the value
  uint8_t key_escaped, kind;                     // kind: 's' string, 'S' string with escapes, 'n' number, anything else
};

struct Scan {
  const uint8_t* v; uint32_t n, p;
  VF_HD void ws() { while (p < n && is_ws(v[p])) ++p; }
  // v[p] should be the opening quote; leaves p after the closing quote
  VF_HD uint32_t string(uint32_t* b, uint32_t* len, bool* escaped) {
    if (p >= n || v[p] != '"') return EXPECTED_STRING;
    ++p; *b = p; *escaped = false;
    while (p < n && v[p] != '"') {
      if (v[p] < 0x20) return CONTROL_CHAR;
      if (v[p] == '\\') { *escaped = true; ++p; if (p >= n) break; }
      ++p;
    }
    if (p >= n) return UNTERMINATED;
    *len = p - *b; ++p;
    return OK;
  }
  VF_HD uint32_t number() {   // -?(0|[1-9][0-9]*)(.[0-9]+)?([eE][+-]?[0-9]+)?
    uint32_t q = p;
    if (v[q] == '-') ++q;
    if (q >= n || !is_digit(v[q])) return BAD_NUMBER;
    if (v[q] == '0') ++q; else while (q < n && is_digit(v[q])) ++q;
    if (q < n && v[q] == '.') { ++q; if (q >= n || !is_digit(v[q])) return BAD_NUMBER; while (q < n && is_digit(v[q])) ++q; }
    if (q < n && (v[q] == 'e' || v[q] == 'E')) {
      ++q; if (q < n && (v[q] == '+' || v[q] == '-')) ++q;
      if (q >= n || !is_digit(v[q])) return BAD_NUMBER;
      while (q < n && is_digit(v[q])) ++q;
    }
    p = q;
    return OK;
  }
  VF_HD bool literal(const char* w, uint32_t len) {
    if (n - p < len) return false;
    for (uint32_t k = 0; k < len; ++k) if (v[p + k] != (uint8_t)w[k]) return false;
    p += len; return true;
  }
  // One member value (JsonScan::value at depth 1), nested containers walked with a bit stack instead of recursion.
  VF_HD uint32_t value(Member* m) {
    ws();
    if (p >= n) return VALUE_EXPECTED;
    m->val_off = p;
    const uint8_t c0 = v[p];
    if (c0 == '"') {
      uint32_t b, len; bool esc;
      const uint32_t e = string(&b, &len, &esc);
      if (e) return e;
      m->kind = esc ? 'S' : 's'; m->val_off = b; m->val_len = len;
      return OK;
    }
    if (c0 != '{' && c0 != '[') {
      if (c0 == '-' || is_digit(c0)) { const uint32_t e = number(); if (e) return e; m->kind = 'n'; m->val_len = p - m->val_off; return OK; }
      if (literal("true", 4) || literal("false", 5) || literal("null", 4)) { m->kind = 'z'; m->val_len = p - m->val_off; return OK; }
      return UNEXPECTED_CHAR;
    }
    uint64_t objects = 0;   // bit d - 1: the container at depth d is an object
    int depth = 0;
    uint8_t c = c0;
    for (;;) {
      // c (at v[p]) opens a container at depth + 1
      if (depth + 1 > kMaxDepth) return NESTING;
      ++depth;
      const bool obj = c == '{';
      if (obj) objects |= 1ull << (depth - 1); else objects &= ~(1ull << (depth - 1));
      ++p; ws();
      bool closed = p < n && v[p] == (obj ? '}' : ']');
      if (closed) { ++p; --depth; }
      // members / elements until a container opens (continue the outer loop) or the first one closes completely (return)
      for (;;) {
        if (closed) {
          if (depth == 0) { m->kind = c0 == '{' ? 'o' : 'a'; m->val_len = p - m->val_off; return OK; }
          // after a value inside the container at `depth`
          const bool in_obj = (objects >> (depth - 1)) & 1;
          ws();
          if (p < n && v[p] == ',') { ++p; closed = false; }
          else if (p < n && v[p] == (in_obj ? '}' : ']')) { ++p; --depth; continue; }
          else return COMMA_OR_BRACKET;
        }
        // the next member / element of the container at `depth`
        if ((objects >> (depth - 1)) & 1) {
          ws();
          uint32_t b, len; bool esc;
          const uint32_t e = string(&b, &len, &esc);
          if (e) return e;
          ws();
          if (p >= n || v[p] != ':') return COLON;
          ++p;
        }
        ws();
        if (p >= n) return VALUE_EXPECTED;
        c = v[p];
        if (c == '{' || c == '[') break;   // a nested container opens
        if (c == '"') { uint32_t b, len; bool esc; const uint32_t e = string(&b, &len, &esc); if (e) return e; }
        else if (c == '-' || is_digit(c)) { const uint32_t e = number(); if (e) return e; }
        else if (!(literal("true", 4) || literal("false", 5) || literal("null", 4))) return UNEXPECTED_CHAR;
        closed = true;   // (a scalar: continue after it)
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------------------------- numbers
// strtoll over a text the number grammar accepted, without '.', 'e' or 'E': -2^63 .. 2^63 - 1, else INT_RANGE
VF_HD uint32_t parse_i64(const uint8_t* s, uint32_t len, int64_t* out) {
  const bool neg = s[0] == '-';
  uint64_t v = 0;
  const uint64_t lim = neg ? (1ull << 63) : (1ull << 63) - 1;
  for (uint32_t k = neg; k < len; ++k) {
    const uint64_t d = (uint64_t)(s[k] - '0');
    if (v > (lim - d) / 10) return INT_RANGE;
    v = v * 10 + d;
  }
  *out = neg ? (int64_t)(0ull - v) : (int64_t)v;
  return OK;
}

// Big unsigned integers, little-endian 32-bit words.
constexpr int kWords = 44;   // 10^387 * 2^55 < 2^1341 (the largest operand of f64_slow) fits 42 words
struct Big {
  uint32_t w[kWords]; int n;   // n: words in use (w[n..] are 0)
  VF_HD void set(uint64_t x) { for (int k = 0; k < kWords; ++k) w[k] = 0; w[0] = (uint32_t)x; w[1] = (uint32_t)(x >> 32); n = w[1] ? 2 : (w[0] ? 1 : 0); }
  VF_HD void mul_small(uint32_t m) {
    uint64_t carry = 0;
    for (int k = 0; k < n; ++k) { const uint64_t t = (uint64_t)w[k] * m + carry; w[k] = (uint32_t)t; carry = t >> 32; }
    if (carry) w[n++] = (uint32_t)carry;
  }
  VF_HD void add_small(uint32_t a) {
    uint64_t carry = a;
    for (int k = 0; carry; ++k) {
      if (k == n) w[n++] = 0;
      const uint64_t t = (uint64_t)w[k] + carry; w[k] = (uint32_t)t; carry = t >> 32;
    }
  }
  VF_HD void mul_pow10(uint32_t e) {
    const uint32_t p9 = 1000000000u;
    while (e >= 9) { mul_small(p9); e -= 9; }
    uint32_t r = 1;
    while (e--) r *= 10;
    if (r > 1) mul_small(r);
  }
  VF_HD int bits() const {
    if (!n) return 0;
    uint32_t top = w[n - 1]; int b = 0;
    while (top) { ++b; top >>= 1; }
    return (n - 1) * 32 + b;
  }
  VF_HD void shl(int s) {   // s >= 0, the result fits
    const int ws = s / 32, bs = s % 32;
    if (!n) return;
    int top = n - 1 + ws + 1;
    for (int k = top; k >= 0; --k) {
      const int src = k - ws;
      const uint32_t hi = (src >= 0 && src < n) ? w[src] : 0u;
      const uint32_t lo = (bs && src - 1 >= 0 && src - 1 < n) ? w[src - 1] : 0u;
      w[k] = bs ? (hi << bs) | (lo >> (32 - bs)) : hi;
    }
    n = top + 1;
    while (n && !w[n - 1]) --n;
  }
  VF_HD void shr1() {
    for (int k = 0; k < n; ++k) w[k] = (w[k] >> 1) | (k + 1 < n ? w[k + 1] << 31 : 0u);
    while (n && !w[n - 1]) --n;
  }
  VF_HD bool ge(const Big& o) const {
    if (n != o.n) return n > o.n;
    for (int k = n - 1; k >= 0; --k) if (w[k] != o.w[k]) return w[k] > o.w[k];
    return true;
  }
  VF_HD void sub(const Big& o) {   // *this >= o
    int64_t borrow = 0;
    for (int k = 0; k < n; ++k) {
      const int64_t t = (int64_t)w[k] - (k < o.n ? (int64_t)o.w[k] : 0) - borrow;
      w[k] = (uint32_t)t; borrow = t < 0;
    }
    while (n && !w[n - 1]) --n;
  }
  VF_HD bool bit_below(int b) const {   // any bit below position b set?
    for (int k = 0; k < n && k * 32 < b; ++k) {
      const int lo = b - k * 32;
      const uint32_t mask = lo >= 32 ? 0xffffffffu : ((1u << lo) - 1u);
      if (w[k] & mask) return true;
    }
    return false;
  }
  VF_HD uint64_t bits_at(int b) const {   // the 64 bits starting at bit b
    uint64_t r = 0;
    for (int k = 0; k < 64; k += 32) {
      const int pos = b + k, wi = pos / 32, bi = pos % 32;
      uint64_t part = wi < n ? w[wi] >> bi : 0;
      if (bi && wi + 1 < n) part |= (uint64_t)w[wi + 1] << (32 - bi);
      r |= (part & 0xffffffffull) << k;
    }
    return r;
  }
};

// (q + a fraction, nonzero when sticky) * 2^e2, 0 < q < 2^63 -> the nearest double, ties to even; subnormals round at their
// reduced precision; beyond DBL_MAX: infinity
VF_HD uint64_t round_bits(uint64_t q, bool sticky, int e2) {
  int L = 0;
  for (uint64_t t = q; t; t >>= 1) ++L;
  int drop = L - 53;
  if (e2 + drop < -1074) drop = -1074 - e2;   // below the normal range: the lowest kept bit is 2^-1074
  uint64_t kept = q;
  if (drop > 0) {
    if (drop > 63) return 0;
    kept = q >> drop;
    const uint64_t rem = q & ((1ull << drop) - 1), half = 1ull << (drop - 1);
    if (rem > half || (rem == half && (sticky || (kept & 1)))) ++kept;
  } else if (drop < 0) {
    kept = q << -drop;   // (exact: fewer than 53 significant bits)
  }
  int e = e2 + drop;
  if (kept < (1ull << 52)) return kept;   // subnormal (e == -1074), or zero
  if (kept == (1ull << 53)) { kept >>= 1; ++e; }
  const int biased = e + 1075;
  if (biased >= 2047) return 0x7ff0000000000000ull;
  return ((uint64_t)biased << 52) | (kept & ((1ull << 52) - 1));
}

// D * 10^e10, D of nd <= 63 decimal digits (a 63-character integer text: D < 2^210), -324 < nd + e10 <= 309, so 10^-e10 < 10^387:
// exact big-integer arithmetic
VF_HDN uint64_t f64_slow(const uint8_t* digits, const uint32_t* at, uint32_t nd, int e10) {
  Big num;
  num.set(0);
  for (uint32_t k = 0; k < nd; ++k) { num.mul_small(10); num.add_small(digits[at[k]] - '0'); }
  if (e10 >= 0) {
    num.mul_pow10((uint32_t)e10);
    const int L = num.bits();
    if (L <= 63) return round_bits(num.bits_at(0), false, 0);
    return round_bits(num.bits_at(L - 63), num.bit_below(L - 63), L - 63);
  }
  Big den;
  den.set(1);
  den.mul_pow10((uint32_t)-e10);
  const int s = den.bits() - num.bits() + 55;   // num * 2^s / den lies in [2^54, 2^56)
  if (s >= 0) num.shl(s); else den.shl(-s);
  Big t = den;
  t.shl(55);
  uint64_t q = 0;
  for (int b = 55; b >= 0; --b) {
    if (num.ge(t)) { num.sub(t); q |= 1ull << b; }
    t.shr1();
  }
  return round_bits(q, num.n != 0, -s);
}

// strtod over a text the number grammar accepted (fewer than 64 characters)
VF_HD double parse_f64(const uint8_t* s, uint32_t len) {
  const bool neg = s[0] == '-';
  uint32_t k = neg, at[64], nd = 0, frac = 0;
  bool seen_dot = false;
  for (; k < len && s[k] != 'e' && s[k] != 'E'; ++k) {
    if (s[k] == '.') { seen_dot = true; continue; }
    if (seen_dot) ++frac;
    if (nd == 0 && s[k] == '0') continue;   // leading zeros
    at[nd++] = k;
  }
  int64_t ex = 0;
  if (k < len) {
    ++k;
    const bool eneg = s[k] == '-';
    if (s[k] == '+' || s[k] == '-') ++k;
    for (; k < len; ++k) if (ex < 100000) ex = ex * 10 + (s[k] - '0');   // (any exponent beyond that saturates the result)
    if (eneg) ex = -ex;
  }
  while (nd && s[at[nd - 1]] == '0') { --nd; ++ex; }
  int64_t e10 = ex - (int64_t)frac;
  uint64_t bits;
  if (!nd) bits = 0;
  else if ((int64_t)nd + e10 > 309) bits = 0x7ff0000000000000ull;
  else if ((int64_t)nd + e10 <= -324) bits = 0;
  else if (nd <= 15 && e10 >= -22 && e10 <= 22) {
    const double p10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
    uint64_t d = 0;
    for (uint32_t j = 0; j < nd; ++j) d = d * 10 + (uint64_t)(s[at[j]] - '0');
    double r;
#if defined(__CUDA_ARCH__)
    r = e10 >= 0 ? __dmul_rn((double)d, p10[e10]) : __ddiv_rn((double)d, p10[-e10]);
#else
    r = e10 >= 0 ? (double)d * p10[e10] : (double)d / p10[-e10];
#endif
    if (neg) r = -r;
    return r;
  } else bits = f64_slow(s, at, nd, (int)e10);
  if (neg) bits |= 1ull << 63;
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)bits);
#else
  double r;
  memcpy(&r, &bits, 8);
  return r;
#endif
}

// ------------------------------------------------------------------------------------------------------------ conversions
// protobuf Event { string aggregateId = 1; bytes payload = 2; }: the last field 2 of wire type 2 is the packed event
// (a missing one gives 0 bytes, which the caller's 8..56 length check refuses)
VF_HD uint32_t protobuf_payload(const uint8_t* v, uint32_t n, uint32_t* off, uint32_t* len) {
  uint64_t pos = 0;
  *off = 0; *len = 0;
  auto uvarint = [&](bool* ok) -> uint64_t {
    uint64_t x = 0; int shift = 0;
    for (int i = 0; i < 10; ++i) {
      if (pos >= n) { *ok = false; return 0; }
      const uint8_t b = v[pos++];
      x |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return x;
      shift += 7;
    }
    *ok = false; return 0;
  };
  bool ok = true;
  while (pos < n) {
    const uint64_t tag = uvarint(&ok);
    if (!ok) return NOT_PROTOBUF;
    switch (tag & 7) {
      case 0: uvarint(&ok); break;
      case 1: if (8 > n - pos) ok = false; else pos += 8; break;
      case 5: if (4 > n - pos) ok = false; else pos += 4; break;
      case 2: {
        const uint64_t ln = uvarint(&ok);
        if (ok && ln > n - pos) ok = false;
        if (ok && (tag >> 3) == 2) { *off = (uint32_t)pos; *len = (uint32_t)ln; }
        if (ok) pos += ln;
        break;
      }
      default: ok = false;
    }
    if (!ok) return NOT_PROTOBUF;
  }
  return OK;
}

// Where json_pack puts a member. RECORD: Field::dst_off is a record offset and out[56] holds record bytes 0..7, then 16..63 (the
// class's event type goes to bytes 0..3), as the host decoder's json_pack does. STATE: Field::dst_off is a program byte offset
// and out[kStateRowMax] holds the program bytes of a state row (state-topic values carry no event type).
enum Layout : int { RECORD = 0, STATE = 1 };
constexpr uint32_t kStateRowMax = 120;   // program bytes of the widest state (128 bytes)

// a flat JSON object -> out, in layout kLayout
template <int kLayout = RECORD>
VF_HD uint32_t json_pack(const Table& t, const uint8_t* v, uint32_t n, uint8_t* out) {
  constexpr int kOutBytes = kLayout == RECORD ? 56 : (int)kStateRowMax;
  Member mem[kMaxMembers];
  uint32_t n_members = 0;
  Scan sc{v, n, 0};
  sc.ws();
  if (sc.p >= n || v[sc.p] != '{') return NOT_OBJECT;
  ++sc.p; sc.ws();
  if (sc.p < n && v[sc.p] == '}') ++sc.p;
  else {
    for (;;) {
      sc.ws();
      Member m;
      bool esc;
      uint32_t e = sc.string(&m.key_off, &m.key_len, &esc);
      if (e) return e;
      m.key_escaped = esc;
      sc.ws();
      if (sc.p >= n || v[sc.p] != ':') return COLON;
      ++sc.p;
      if ((e = sc.value(&m))) return e;
      if (n_members >= kMaxMembers) return TOO_MANY_MEMBERS;
      mem[n_members++] = m;
      sc.ws();
      if (sc.p < n && v[sc.p] == ',') { ++sc.p; continue; }
      if (sc.p < n && v[sc.p] == '}') { ++sc.p; break; }
      return COMMA_OR_BRACE;
    }
  }
  sc.ws();
  if (sc.p != n) return TRAILING_BYTES;
  auto find = [&](uint32_t off, uint32_t len) -> const Member* {   // later duplicates win, as in play-json's JsObject
    const Member* hit = nullptr;
    for (uint32_t i = 0; i < n_members; ++i) if (name_is(v + mem[i].key_off, mem[i].key_len, mem[i].key_escaped, t.names + off, len)) hit = &mem[i];
    return hit;
  };
  const Class* ev = nullptr;
  if (!t.disc_len) ev = &t.classes[0];
  else {
    const Member* d = find(t.disc_off, t.disc_len);
    if (!d || (d->kind != 's' && d->kind != 'S')) return NO_DISCRIMINATOR;
    for (uint32_t c = 0; c < t.n_classes && !ev; ++c)
      if (name_is(v + d->val_off, d->val_len, d->kind == 'S', t.names + t.classes[c].name_off, t.classes[c].name_len)) ev = &t.classes[c];
  }
  for (int k = 0; k < kOutBytes; ++k) out[k] = 0;
  const uint32_t ty = ev ? ev->event_type : (uint32_t)t.unknown_type;
  if (!ev && t.unknown_type < 0) return UNKNOWN_CLASS;
  if constexpr (kLayout == RECORD) { out[0] = (uint8_t)ty; out[1] = (uint8_t)(ty >> 8); out[2] = (uint8_t)(ty >> 16); out[3] = (uint8_t)(ty >> 24); }
  if (!ev) return OK;
  for (uint32_t fi = 0; fi < ev->n_fields; ++fi) {
    const Field& f = t.fields[ev->field_begin + fi];
    const Member* m = find(f.name_off, f.name_len);
    uint8_t* dst = out + (kLayout == STATE ? f.dst_off : f.dst_off < 8 ? f.dst_off : f.dst_off - 8);
    if (f.kind == K_UUID || f.kind == K_PSTR) {
      if (!m || (m->kind != 's' && m->kind != 'S')) return STRING_MISSING;
      uint32_t sn = 0;
      {   // the unescaped length (and whether the escapes are good)
        Unesc u(v + m->val_off, m->val_len);
        for (int c; (c = u.next()) != -1; ++sn) if (c == -2) return BAD_ESCAPE;
      }
      Unesc u(v + m->val_off, m->val_len);
      if (f.kind == K_UUID) {
        // java.util.UUID.toString: 8-4-4-4-12 hex digits, stored as the 16 bytes most significant first
        uint8_t s[36];
        if (sn == 36) for (int i = 0; i < 36; ++i) s[i] = (uint8_t)u.next();
        if (sn != 36 || s[8] != '-' || s[13] != '-' || s[18] != '-' || s[23] != '-') return UUID_FORM;
        uint32_t k = 0;
        for (int i = 0; i < 36; ++i) {
          if (i == 8 || i == 13 || i == 18 || i == 23) continue;
          const int d = hex_val(s[i]);
          if (d < 0) return UUID_DIGIT;
          if (k & 1) dst[k >> 1] |= (uint8_t)d; else dst[k >> 1] = (uint8_t)(d << 4);
          ++k;
        }
      } else {
        // length byte + UTF-8 bytes, zero padded to the slot
        if (sn > f.len - 1 || sn > 255) return PSTR_FIT;
        dst[0] = (uint8_t)sn;
        for (uint32_t k = 0; k < sn; ++k) dst[1 + k] = (uint8_t)u.next();
      }
      continue;
    }
    if (!m || m->kind != 'n') return NUMBER_MISSING;
    if (m->val_len >= 64) return NUMBER_TOO_LONG;
    const uint8_t* s = v + m->val_off;
    if (f.kind == K_F64) {
      const double d = parse_f64(s, m->val_len);
#if defined(__CUDA_ARCH__)
      const uint64_t bits = (uint64_t)__double_as_longlong(d);
#else
      uint64_t bits;
      memcpy(&bits, &d, 8);
#endif
      for (int k = 0; k < 8; ++k) dst[k] = (uint8_t)(bits >> (8 * k));
      continue;
    }
    for (uint32_t k = 0; k < m->val_len; ++k) if (s[k] == '.' || s[k] == 'e' || s[k] == 'E') return INT_FRACTION;
    int64_t x;
    if (parse_i64(s, m->val_len, &x)) return INT_RANGE;
    if (f.kind == K_I32) {
      if (x < INT32_MIN || x > INT32_MAX) return INT_NOT_INT;
      for (int k = 0; k < 4; ++k) dst[k] = (uint8_t)((uint64_t)x >> (8 * k));
    } else {
      for (int k = 0; k < 8; ++k) dst[k] = (uint8_t)((uint64_t)x >> (8 * k));
    }
  }
  return OK;
}

// A non-null record value under `framing` (PROTOBUF_EVENT, JSON or PROTOBUF_JSON) -> the packed event value: on OK, *len bytes
// of it are at *val (a part of the value itself, or out[56]). The caller applies the 8..56 length check, as the host decoder
// does next. Under the STATE layout the value is a state-topic value (the protobuf State message has Event's field numbers) and
// a JSON object fills out[kStateRowMax]; the caller checks the length against its program bytes.
// PROTOBUF_JSON is the multilanguage gateway's wrapping of a JSON business-app payload: the payload of the protobuf message (the
// unwrap of PROTOBUF_EVENT; a message without field 2 has an empty payload) goes through json_pack. Field 1, the aggregate id,
// is not read: the record key is the id, as under PROTOBUF_EVENT.
template <int kLayout = RECORD>
VF_HD uint32_t convert(int32_t framing, const Table& t, const uint8_t* v, uint32_t n, uint8_t* out, const uint8_t** val, uint32_t* len) {
  if (framing == PROTOBUF_EVENT || framing == PROTOBUF_JSON) {
    uint32_t off;
    const uint32_t e = protobuf_payload(v, n, &off, len);
    *val = v + off;
    if (e || framing == PROTOBUF_EVENT) return e;
    v += off; n = *len;
  }
  *val = out; *len = kLayout == RECORD ? 56 : kStateRowMax;
  return json_pack<kLayout>(t, v, n, out);
}

}  // namespace vf
}  // namespace sgr
