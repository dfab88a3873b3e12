// state_writer.h — a state row's program bytes -> the model's JSON state value, as Json.toJson(state) writes it for a case class
// of flat members. One source for the device kernels (state_values.cu) and the CPU tests (tests/fuzz/state_writer_main.cpp,
// built under ASan + UBSan and compared byte for byte with oracle/state_json.py).
//
// A value is `{"name":value,...}`: members in table order, no whitespace. Each member is written in two passes over the same
// code, its length first (so a batch's values can be laid out by a scan), then its bytes. Members:
//   I32 / I64  plain decimal;
//   UUID       36 lowercase hex digits 8-4-4-4-12, the 16 bytes most significant first (java.util.UUID.toString);
//   PSTR       a JSON string of the slot's first length-byte bytes, which must be well-formed UTF-8;
//   F64        the shortest decimal that rounds back to the double (Ryu-style, 128-bit powers of five from f64_tables.h), laid
//              out as play-json writes a BigDecimal: trailing zeros stripped, plain for 1e-10 <= |v| <= 1e20, else
//              BigDecimal.toString's scientific form (1.5E+21, 1E-11); 0.0 and -0.0 are 0; NaN and infinities are refused;
//   ID         the row's aggregate id as a JSON string (well-formed UTF-8).
// Strings escape '"' and '\' as \" and \\, \b \t \n \f \r by their short forms, other control characters below U+0020 as \u00XX
// with uppercase hex (as Jackson writes them), and keep every other character, U+007F and non-ASCII included, as its UTF-8 bytes.
#pragma once
#include <stdint.h>
#include <string.h>

#include "f64_tables.h"

#if defined(__CUDACC__)
#define SW_HD __host__ __device__ __forceinline__
#else
#define SW_HD inline
#endif

namespace sgr {
namespace sw {

// member kinds (include/sgr.h SGR_JSON_*)
enum : uint8_t { K_I32 = 0, K_I64 = 1, K_F64 = 2, K_UUID = 3, K_PSTR = 4, K_ID = 5 };

// why a row cannot be written
enum Reason : uint32_t { OK = 0, F64_NOT_FINITE, PSTR_LENGTH, PSTR_UTF8, ID_UTF8, NO_ID };

inline const char* reason_text(uint32_t r) {
  switch (r) {
    case F64_NOT_FINITE: return "a Double member holds NaN or an infinity, which a JSON number cannot hold";
    case PSTR_LENGTH: return "a string member's length byte is larger than its slot";
    case PSTR_UTF8: return "a string member is not well-formed UTF-8";
    case ID_UTF8: return "the aggregate id is not well-formed UTF-8";
    case NO_ID: return "the row has no aggregate id in the key table";
  }
  return "";
}

// One member of a writer table. lit: the bytes written before the member's value, `{"name":` for the first and `,"name":` for
// the others, the name escaped; the value ends with `}`.
struct Member { uint8_t kind; uint8_t reserved; uint16_t off; uint32_t len; uint32_t lit_off, lit_len; };
constexpr uint32_t kMaxMembers = 32;

// ------------------------------------------------------------------------------------------------------------------- strings
// RFC 3629: no overlong forms, no surrogates, nothing above U+10FFFF, no truncated sequence
SW_HD bool utf8_ok(const uint8_t* s, uint64_t n) {
  uint64_t i = 0;
  while (i < n) {
    const uint8_t c = s[i];
    if (c < 0x80) { ++i; continue; }
    uint32_t need; uint8_t lo = 0x80, hi = 0xBF;
    if (c >= 0xC2 && c <= 0xDF) need = 1;
    else if (c >= 0xE0 && c <= 0xEF) { need = 2; if (c == 0xE0) lo = 0xA0; else if (c == 0xED) hi = 0x9F; }
    else if (c >= 0xF0 && c <= 0xF4) { need = 3; if (c == 0xF0) lo = 0x90; else if (c == 0xF4) hi = 0x8F; }
    else return false;
    if (n - i - 1 < need) return false;
    if (s[i + 1] < lo || s[i + 1] > hi) return false;
    for (uint32_t k = 2; k <= need; ++k) if (s[i + k] < 0x80 || s[i + k] > 0xBF) return false;
    i += need + 1;
  }
  return true;
}

SW_HD uint32_t esc_char_len(uint8_t c) {
  if (c == '"' || c == '\\' || c == '\b' || c == '\t' || c == '\n' || c == '\f' || c == '\r') return 2;
  return c < 0x20 ? 6 : 1;
}

SW_HD uint8_t* esc_char_write(uint8_t* o, uint8_t c) {
  const char* hex = "0123456789ABCDEF";
  switch (c) {
    case '"': *o++ = '\\'; *o++ = '"'; return o;
    case '\\': *o++ = '\\'; *o++ = '\\'; return o;
    case '\b': *o++ = '\\'; *o++ = 'b'; return o;
    case '\t': *o++ = '\\'; *o++ = 't'; return o;
    case '\n': *o++ = '\\'; *o++ = 'n'; return o;
    case '\f': *o++ = '\\'; *o++ = 'f'; return o;
    case '\r': *o++ = '\\'; *o++ = 'r'; return o;
  }
  if (c < 0x20) { *o++ = '\\'; *o++ = 'u'; *o++ = '0'; *o++ = '0'; *o++ = (uint8_t)hex[c >> 4]; *o++ = (uint8_t)hex[c & 15]; return o; }
  *o++ = c;
  return o;
}

// a JSON string of s[0, n), quotes included
SW_HD uint64_t str_len(const uint8_t* s, uint64_t n) {
  uint64_t l = 2;
  for (uint64_t i = 0; i < n; ++i) l += esc_char_len(s[i]);
  return l;
}

SW_HD uint8_t* str_write(uint8_t* o, const uint8_t* s, uint64_t n) {
  *o++ = '"';
  for (uint64_t i = 0; i < n; ++i) o = esc_char_write(o, s[i]);
  *o++ = '"';
  return o;
}

// ------------------------------------------------------------------------------------------------------------------ integers
SW_HD uint32_t u64_digits(uint64_t v) {
  uint32_t d = 1;
  while (v >= 10) { v /= 10; ++d; }
  return d;
}

SW_HD uint8_t* u64_write(uint8_t* o, uint64_t v, uint32_t nd) {
  for (uint32_t k = nd; k-- > 0;) { o[k] = (uint8_t)('0' + v % 10); v /= 10; }
  return o + nd;
}

SW_HD uint32_t i64_len(int64_t v) {
  const uint64_t m = v < 0 ? 0ull - (uint64_t)v : (uint64_t)v;
  return (v < 0) + u64_digits(m);
}

SW_HD uint8_t* i64_write(uint8_t* o, int64_t v) {
  const uint64_t m = v < 0 ? 0ull - (uint64_t)v : (uint64_t)v;
  if (v < 0) *o++ = '-';
  return u64_write(o, m, u64_digits(m));
}

// --------------------------------------------------------------------------------------------------------------------- UUID
constexpr uint32_t kUuidLen = 38;   // quotes included

SW_HD uint8_t* uuid_write(uint8_t* o, const uint8_t* b) {
  const char* hex = "0123456789abcdef";
  *o++ = '"';
  for (int i = 0; i < 16; ++i) {
    if (i == 4 || i == 6 || i == 8 || i == 10) *o++ = '-';
    *o++ = (uint8_t)hex[b[i] >> 4]; *o++ = (uint8_t)hex[b[i] & 15];
  }
  *o++ = '"';
  return o;
}

// -------------------------------------------------------------------------------------------------------------------- doubles
// The shortest decimal m * 10^e in the rounding interval of a finite, non-zero double (the interval's ends belong to it when
// the mantissa is even); among the shortest, the one nearest the double, ties to even. This is Ulf Adams' Ryu: the interval's
// ends and middle are multiplied by a 125-bit power of five (f64_tables.h) and digits are dropped while the ends still differ.
#if defined(__CUDACC__)
static __device__ const uint64_t d_pow5[SGR_F64_N_POW5][2] = SGR_F64_POW5_SPLIT;
static __device__ const uint64_t d_pow5_inv[SGR_F64_N_POW5_INV][2] = SGR_F64_POW5_INV_SPLIT;
#endif
static const uint64_t h_pow5[SGR_F64_N_POW5][2] = SGR_F64_POW5_SPLIT;
static const uint64_t h_pow5_inv[SGR_F64_N_POW5_INV][2] = SGR_F64_POW5_INV_SPLIT;

SW_HD const uint64_t* pow5_split(uint32_t i) {
#if defined(__CUDA_ARCH__)
  return d_pow5[i];
#else
  return h_pow5[i];
#endif
}

SW_HD const uint64_t* pow5_inv_split(uint32_t i) {
#if defined(__CUDA_ARCH__)
  return d_pow5_inv[i];
#else
  return h_pow5_inv[i];
#endif
}

SW_HD uint64_t umulh(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

SW_HD int32_t pow5bits(int32_t e) { return (int32_t)(((uint32_t)e * 1217359u) >> 19) + 1; }   // ceil(log2(5^e)), 1 for e = 0
SW_HD uint32_t log10_pow2(int32_t e) { return ((uint32_t)e * 78913u) >> 18; }              // floor(log10(2^e))
SW_HD uint32_t log10_pow5(int32_t e) { return ((uint32_t)e * 732923u) >> 20; }             // floor(log10(5^e))

SW_HD uint32_t pow5_factor(uint64_t v) {
  uint32_t c = 0;
  while (v % 5 == 0) { v /= 5; ++c; }
  return c;
}

// (m * mul) >> j for the 128-bit mul, 64 < j < 128
SW_HD uint64_t mul_shift(uint64_t m, const uint64_t* mul, int32_t j) {
  const uint64_t hi0 = umulh(m, mul[0]);
  const uint64_t lo1 = m * mul[1];
  uint64_t hi1 = umulh(m, mul[1]);
  const uint64_t sum = hi0 + lo1;
  if (sum < hi0) ++hi1;
  const int32_t d = j - 64;
  return (hi1 << (64 - d)) | (sum >> d);
}

struct Dec { uint64_t m; int32_t e; };

SW_HD Dec f64_shortest(uint64_t bits) {
  const uint64_t mant = bits & ((1ull << 52) - 1);
  const uint32_t bexp = (uint32_t)((bits >> 52) & 0x7ff);
  int32_t e2; uint64_t m2;
  if (bexp == 0) { e2 = 1 - 1023 - 52 - 2; m2 = mant; }
  else { e2 = (int32_t)bexp - 1023 - 52 - 2; m2 = (1ull << 52) | mant; }
  const bool accept = (m2 & 1) == 0;
  const uint64_t mv = 4 * m2;
  const uint32_t mm_shift = mant != 0 || bexp <= 1;   // the lower end is closer when the double is a power of two
  uint64_t vr, vp, vm;
  int32_t e10;
  bool vm_tz = false, vr_tz = false;
  if (e2 >= 0) {
    const uint32_t q = log10_pow2(e2) - (e2 > 3);
    e10 = (int32_t)q;
    const int32_t k = SGR_F64_POW5_BITS + pow5bits((int32_t)q) - 1;
    const int32_t i = -e2 + (int32_t)q + k;
    const uint64_t* mul = pow5_inv_split(q);
    vr = mul_shift(4 * m2, mul, i);
    vp = mul_shift(4 * m2 + 2, mul, i);
    vm = mul_shift(4 * m2 - 1 - mm_shift, mul, i);
    if (q <= 21) {
      if (mv % 5 == 0) vr_tz = pow5_factor(mv) >= q;
      else if (accept) vm_tz = pow5_factor(mv - 1 - mm_shift) >= q;
      else vp -= pow5_factor(mv + 2) >= q;
    }
  } else {
    const uint32_t q = log10_pow5(-e2) - (-e2 > 1);
    e10 = (int32_t)q + e2;
    const int32_t i = -e2 - (int32_t)q;
    const int32_t k = pow5bits(i) - SGR_F64_POW5_BITS;
    const int32_t j = (int32_t)q - k;
    const uint64_t* mul = pow5_split((uint32_t)i);
    vr = mul_shift(4 * m2, mul, j);
    vp = mul_shift(4 * m2 + 2, mul, j);
    vm = mul_shift(4 * m2 - 1 - mm_shift, mul, j);
    if (q <= 1) {
      vr_tz = true;
      if (accept) vm_tz = mm_shift == 1;
      else --vp;
    } else if (q < 63) {
      vr_tz = (mv & ((1ull << q) - 1)) == 0;
    }
  }
  int32_t removed = 0;
  uint32_t last = 0;
  uint64_t out;
  if (vm_tz || vr_tz) {
    for (;;) {
      const uint64_t vp10 = vp / 10, vm10 = vm / 10;
      if (vp10 <= vm10) break;
      const uint64_t vr10 = vr / 10;
      vm_tz &= vm % 10 == 0;
      vr_tz &= last == 0;
      last = (uint32_t)(vr % 10);
      vr = vr10; vp = vp10; vm = vm10; ++removed;
    }
    if (vm_tz) {
      while (vm % 10 == 0) {
        const uint64_t vr10 = vr / 10;
        vr_tz &= last == 0;
        last = (uint32_t)(vr % 10);
        vr = vr10; vp /= 10; vm /= 10; ++removed;
      }
    }
    if (vr_tz && last == 5 && vr % 2 == 0) last = 4;   // exactly halfway: round to even
    out = vr + ((vr == vm && (!accept || !vm_tz)) || last >= 5);
  } else {
    bool up = false;
    if (vp / 100 > vm / 100) {
      up = vr % 100 >= 50;
      vr /= 100; vp /= 100; vm /= 100; removed += 2;
    }
    for (;;) {
      const uint64_t vp10 = vp / 10, vm10 = vm / 10;
      if (vp10 <= vm10) break;
      up = vr % 10 >= 5;
      vr /= 10; vp = vp10; vm = vm10; ++removed;
    }
    out = vr + (vr == vm || up);
  }
  Dec d{out, e10 + removed};
  while (d.m % 10 == 0) { d.m /= 10; ++d.e; }   // (a round-up can end in a zero)
  return d;
}

SW_HD bool f64_finite(uint64_t bits) { return ((bits >> 52) & 0x7ff) != 0x7ff; }

// The layout of a finite double's digits. sci: E < -10, or v > 1e20 (E > 20, or E == 20 with more than the digit 1).
struct F64Text { Dec d; uint32_t nd; int32_t E; bool neg, zero, sci; };

SW_HD F64Text f64_text(uint64_t bits) {
  F64Text t{};
  t.neg = bits >> 63;
  t.zero = (bits << 1) == 0;
  if (t.zero) return t;
  t.d = f64_shortest(bits);
  t.nd = u64_digits(t.d.m);
  t.E = (int32_t)t.nd - 1 + t.d.e;
  t.sci = t.E < -10 || t.E > 20 || (t.E == 20 && t.d.m != 1);
  return t;
}

SW_HD uint32_t f64_len(uint64_t bits) {
  const F64Text t = f64_text(bits);
  if (t.zero) return 1;
  uint32_t l = t.neg + t.nd;
  if (t.sci) {
    const int32_t ae = t.E < 0 ? -t.E : t.E;
    return l + (t.nd > 1) + 2 + u64_digits((uint64_t)ae);   // "." if more digits, "E", the sign, the exponent
  }
  if (t.d.e >= 0) return l + (uint32_t)t.d.e;               // trailing zeros
  if (t.E >= 0) return l + 1;                                // a point inside the digits
  return l + 2 + (uint32_t)(-t.E - 1);                       // "0." and leading zeros
}

SW_HD uint8_t* f64_write(uint8_t* o, uint64_t bits) {
  const F64Text t = f64_text(bits);
  if (t.zero) { *o++ = '0'; return o; }
  if (t.neg) *o++ = '-';
  uint8_t dig[20];
  u64_write(dig, t.d.m, t.nd);
  if (t.sci) {
    *o++ = dig[0];
    if (t.nd > 1) { *o++ = '.'; for (uint32_t k = 1; k < t.nd; ++k) *o++ = dig[k]; }
    *o++ = 'E';
    *o++ = t.E < 0 ? '-' : '+';
    const int32_t ae = t.E < 0 ? -t.E : t.E;
    return u64_write(o, (uint64_t)ae, u64_digits((uint64_t)ae));
  }
  if (t.d.e >= 0) {
    for (uint32_t k = 0; k < t.nd; ++k) *o++ = dig[k];
    for (int32_t k = 0; k < t.d.e; ++k) *o++ = '0';
  } else if (t.E >= 0) {
    for (uint32_t k = 0; k < t.nd; ++k) { if ((int32_t)k == t.E + 1) *o++ = '.'; *o++ = dig[k]; }
  } else {
    *o++ = '0'; *o++ = '.';
    for (int32_t k = 0; k < -t.E - 1; ++k) *o++ = '0';
    for (uint32_t k = 0; k < t.nd; ++k) *o++ = dig[k];
  }
  return o;
}

// ---------------------------------------------------------------------------------------------------------------------- rows
SW_HD uint32_t ld32(const uint8_t* p) { uint32_t v = 0; for (int k = 0; k < 4; ++k) v |= (uint32_t)p[k] << (8 * k); return v; }
SW_HD uint64_t ld64(const uint8_t* p) { return (uint64_t)ld32(p) | (uint64_t)ld32(p + 4) << 32; }

// The bytes member m takes in the value of a row (program bytes `row`, id[0, id_len) when has_id), its literal included; a row
// it cannot write gives *why != OK.
SW_HD uint64_t member_len(const Member& m, const uint8_t* row, const uint8_t* id, uint64_t id_len, bool has_id, uint32_t* why) {
  const uint8_t* p = row + m.off;
  uint64_t l = m.lit_len;
  switch (m.kind) {
    case K_I32: return l + i64_len((int32_t)ld32(p));
    case K_I64: return l + i64_len((int64_t)ld64(p));
    case K_UUID: return l + kUuidLen;
    case K_F64: {
      const uint64_t b = ld64(p);
      if (!f64_finite(b)) { *why = F64_NOT_FINITE; return 0; }
      return l + f64_len(b);
    }
    case K_PSTR: {
      if (p[0] > m.len - 1) { *why = PSTR_LENGTH; return 0; }
      if (!utf8_ok(p + 1, p[0])) { *why = PSTR_UTF8; return 0; }
      return l + str_len(p + 1, p[0]);
    }
    default: {   // K_ID
      if (!has_id) { *why = NO_ID; return 0; }
      if (!utf8_ok(id, id_len)) { *why = ID_UTF8; return 0; }
      return l + str_len(id, id_len);
    }
  }
}

// member m of a row that member_len accepted, its literal included
SW_HD uint8_t* member_write(uint8_t* o, const Member& m, const uint8_t* lits, const uint8_t* row, const uint8_t* id, uint64_t id_len) {
  for (uint32_t k = 0; k < m.lit_len; ++k) *o++ = lits[m.lit_off + k];
  const uint8_t* p = row + m.off;
  switch (m.kind) {
    case K_I32: return i64_write(o, (int32_t)ld32(p));
    case K_I64: return i64_write(o, (int64_t)ld64(p));
    case K_UUID: return uuid_write(o, p);
    case K_F64: return f64_write(o, ld64(p));
    case K_PSTR: return str_write(o, p + 1, p[0]);
    default: return str_write(o, id, id_len);
  }
}

// --------------------------------------------------------------------------------------------- protobuf State wrapping
// SGR_VALUE_PROTOBUF_JSON (sgr_set_state_writer_framing): the value is the multilanguage State { string aggregateId = 1; bytes
// payload = 2; } around the JSON value, as ScalaPB's toByteArray writes it: field 1 (left out for an empty id, as proto3 leaves
// out a default string), then field 2.
constexpr uint32_t kWrapMember = kMaxMembers;   // the member index of a row refused for the wrapper's id (State.aggregateId)

SW_HD uint32_t varint_len(uint64_t v) { uint32_t n = 1; while (v >= 0x80) { v >>= 7; ++n; } return n; }

SW_HD uint8_t* varint_write(uint8_t* o, uint64_t v) {
  while (v >= 0x80) { *o++ = (uint8_t)(v | 0x80); v >>= 7; }
  *o++ = (uint8_t)v;
  return o;
}

SW_HD uint64_t wrap_id_len(uint64_t id_len) { return id_len ? 1 + varint_len(id_len) + id_len : 0; }

// the wrapped value of an id and a JSON value of json_len bytes
SW_HD uint64_t wrap_len(uint64_t id_len, uint64_t json_len) { return wrap_id_len(id_len) + 1 + varint_len(json_len) + json_len; }

// the JSON bytes inside a wrapped value of `total` bytes (json_len + varint_len(json_len) grows strictly: one answer)
SW_HD uint64_t wrap_json_len(uint64_t id_len, uint64_t total) {
  const uint64_t rest = total - wrap_id_len(id_len) - 1;
  for (uint32_t k = 1; k < 10; ++k) if (varint_len(rest - k) == k) return rest - k;
  return 0;
}

// the wrapper's bytes in front of the JSON value
SW_HD uint8_t* wrap_head_write(uint8_t* o, const uint8_t* id, uint64_t id_len, uint64_t json_len) {
  if (id_len) {
    *o++ = 0x0A;
    o = varint_write(o, id_len);
    for (uint64_t k = 0; k < id_len; ++k) *o++ = id[k];
  }
  *o++ = 0x12;
  return varint_write(o, json_len);
}

}  // namespace sw
}  // namespace sgr
