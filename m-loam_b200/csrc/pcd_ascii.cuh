// pcd_ascii.cuh — one token of an ASCII PCD body -> the float pcl::io::loadPCDFile<pcl::PointXYZ> stores for it (PCL 1.8
// copyStringValue<float>: "nan" is quiet_NaN, else std::istringstream(tok) >> f in the classic locale, and (float)atof(tok) when that
// fails).  In libstdc++ the stream read is strtof, correctly rounded with ties to even, subnormals included, and it fails exactly when
// strtof overflows to +-inf, where (float)atof gives +-inf again.  So the value is the correctly rounded float of the decimal, +-inf
// beyond FLT_MAX's rounding boundary.  Written once for the host and the device (csrc/pcd.cu, the CPU tests' host build).
//
// Tokens taken: [+-]?(d+(.d*)?|.d+)([eE][+-]?d+)?, nan, inf, +inf, -inf — every form %.8g (PCL's writer) and %.17g emit.  Refused
// (PCD_BAD_TOKEN): anything else, for which PCL stores a prefix parse or atof's reading.  Refused (PCD_TOO_LONG): more than 19
// significant digits (the digit string without its leading and trailing zeros), so that the digits are one 64-bit integer w.
//
// The value w * 10^q: an Eisel-Lemire step multiplies w by the 128-bit power of five of pcd_pow5.h (tools/gen_pcd_pow5.py), which gives
// the product's top 128 bits to within 2 units of their last bit.  That decides the rounding unless the bits below the float's last bit
// lie within those 2 units of the halfway point; then an exact comparison of w * 10^q with the halfway point, on 256-bit integers,
// decides (every exact tie, e.g. 16777217 or 2345678.25, goes there and rounds to even).
#pragma once
#include <cstdint>

#include "pcd_pow5.h"

#if defined(__CUDACC__)
#define PCD_HD __host__ __device__ inline
#else
#define PCD_HD inline
#endif

namespace pcd {

enum { PCD_OK = 0, PCD_BAD_TOKEN = 1, PCD_TOO_LONG = 2 };  // parse_float
// Why a body is refused, as bits (a token's status t is bit t << 1): a line with fewer tokens than the header's, a token outside the
// grammar, a token over 19 significant digits, fewer lines than POINTS
enum { PCD_E_SHORT_LINE = 1, PCD_E_BAD_TOKEN = 2, PCD_E_TOO_LONG = 4, PCD_E_FEW_LINES = 8 };

// the separators of a line's tokens (boost::split with is_any_of("\t\r "), token_compress_on)
PCD_HD bool is_sep(unsigned char ch) { return ch == ' ' || ch == '\t' || ch == '\r'; }

#if defined(__CUDACC__)
static __device__ const uint64_t kPow5T_dev[] = PCD_POW5_T_DATA;
static __device__ const short kPow5E_dev[] = PCD_POW5_E_DATA;
#endif
static const uint64_t kPow5T_host[] = PCD_POW5_T_DATA;
static const short kPow5E_host[] = PCD_POW5_E_DATA;

PCD_HD uint64_t pow5_t(int i) {
#if defined(__CUDA_ARCH__)
  return kPow5T_dev[i];
#else
  return kPow5T_host[i];
#endif
}
PCD_HD int pow5_e(int i) {
#if defined(__CUDA_ARCH__)
  return kPow5E_dev[i];
#else
  return kPow5E_host[i];
#endif
}

PCD_HD uint64_t mulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

PCD_HD int clz64(uint64_t x) {
#if defined(__CUDA_ARCH__)
  return __clzll((long long)x);
#else
  return __builtin_clzll(x);
#endif
}

// ---- the exact comparison: unsigned integers of 8 x 32 bits, little-endian limbs
struct Big {
  uint32_t d[8];
};
PCD_HD void big_set(Big &b, uint64_t v) {
  for (int k = 0; k < 8; k++) b.d[k] = 0;
  b.d[0] = (uint32_t)v, b.d[1] = (uint32_t)(v >> 32);
}
PCD_HD void big_mul(Big &b, uint32_t m) {
  uint64_t carry = 0;
  for (int k = 0; k < 8; k++) {
    const uint64_t t = (uint64_t)b.d[k] * m + carry;
    b.d[k] = (uint32_t)t, carry = t >> 32;
  }
}
PCD_HD void big_mul_pow5(Big &b, int k) {
  for (; k >= 13; k -= 13) big_mul(b, 1220703125u);  // 5^13
  uint32_t m = 1;
  for (; k > 0; k--) m *= 5;
  big_mul(b, m);
}
PCD_HD void big_shl(Big &b, int s) {
  const int w = s >> 5, r = s & 31;
  for (int k = 7; k >= 0; k--) {
    const uint32_t hi = k - w >= 0 ? b.d[k - w] : 0u, lo = k - w - 1 >= 0 ? b.d[k - w - 1] : 0u;
    b.d[k] = r ? (hi << r) | (lo >> (32 - r)) : hi;
  }
}
PCD_HD int big_cmp(const Big &a, const Big &b) {
  for (int k = 7; k >= 0; k--)
    if (a.d[k] != b.d[k]) return a.d[k] < b.d[k] ? -1 : 1;
  return 0;
}
// sign of w * 10^q - b * 2^e, for callers whose aligned sides stay below 2^256
PCD_HD int cmp_dec_bin(uint64_t w, int q, uint64_t b, int e) {
  Big x, y;
  big_set(x, w), big_set(y, b);
  if (q >= 0) big_mul_pow5(x, q);
  else big_mul_pow5(y, -q);
  const int s = q - e;  // x * 2^q vs y * 2^e
  if (s >= 0) big_shl(x, s);
  else big_shl(y, -s);
  return big_cmp(x, y);
}
// sign of w * 10^q - (2m + 1) * 2^e.  Both sides stay below 2^180 for the w, q, m and e decimal_to_float passes.
PCD_HD int cmp_halfway(uint64_t w, int q, uint32_t m, int e) { return cmp_dec_bin(w, q, 2ull * m + 1ull, e); }

// The float bits nearest to w * 10^q (ties to even), +inf past FLT_MAX's rounding boundary; w > 0, w < 10^19
PCD_HD uint32_t decimal_to_float(uint64_t w, int q) {
  if (q > PCD_POW5_QMAX) return 0x7f800000u;  // >= 10^39
  if (q < PCD_POW5_QMIN) return 0u;           // < 10^19 * 10^-66: below half the smallest subnormal
  const int i = q - PCD_POW5_QMIN;
  const int lz = clz64(w);
  const uint64_t wn = w << lz, th = pow5_t(2 * i), tl = pow5_t(2 * i + 1);
  // P = floor(wn * T / 2^64), exact; the true wn * 5^q, scaled alike, lies in [P, P + 2)
  const uint64_t lo_hi = mulhi64(wn, tl), hi_lo = wn * th, hi_hi = mulhi64(wn, th);
  const uint64_t p1 = hi_lo + lo_hi, p2 = hi_hi + (p1 < hi_lo ? 1u : 0u);
  const int top = (int)(p2 >> 63);
  const int L = 126 + top + 64 + pow5_e(i) + q - lz;  // w * 10^q in [2^L, 2^(L+1)), up to a carry that rounding absorbs
  if (L >= 128) return 0x7f800000u;
  if (L <= -152) return 0u;
  const int nb = L + 150 < 24 ? L + 150 : 24;  // bits the float keeps: 24, fewer for a subnormal
  if (nb <= 0) return cmp_halfway(w, q, 0u, -150) > 0 ? 1u : 0u;  // 0 or the smallest subnormal: against 2^-150
  const int d = 127 + top - nb;                                   // bits of P below the kept ones: 103 .. 127
  uint32_t m = (uint32_t)(p2 >> (d - 64));
  const uint64_t r_hi = p2 & ((1ull << (d - 64)) - 1ull), r_lo = p1, half_hi = 1ull << (d - 65);
  bool up;
  if (r_hi > half_hi || (r_hi == half_hi && r_lo > 0)) {
    up = true;  // above halfway whatever the product's last 2 units
  } else if (r_hi + 1 < half_hi || (r_hi + 1 == half_hi && r_lo != ~0ull)) {
    up = false;  // P + 2 still at or below halfway
  } else {
    const int c = cmp_halfway(w, q, m, L - nb);
    up = c > 0 || (c == 0 && (m & 1u));
  }
  m += up ? 1u : 0u;
  if (nb < 24) return m;  // subnormal; 2^23 after the carry is the smallest normal's bits
  const uint32_t bits = ((uint32_t)(L + 126) << 23) + m;
  return bits >= 0x7f800000u ? 0x7f800000u : bits;
}

PCD_HD bool is_digit(unsigned char ch) { return ch >= '0' && ch <= '9'; }

// Token s[0, n) -> *bits.  PCD_OK, PCD_BAD_TOKEN or PCD_TOO_LONG (then *bits is 0).
PCD_HD int parse_float(const unsigned char *s, long long n, uint32_t *bits) {
  *bits = 0;
  if (n == 3 && s[0] == 'n' && s[1] == 'a' && s[2] == 'n') {
    *bits = 0x7fc00000u;
    return PCD_OK;
  }
  long long k = 0;
  uint32_t sign = 0;
  if (n > 0 && (s[0] == '+' || s[0] == '-')) sign = s[0] == '-' ? 0x80000000u : 0u, k = 1;
  if (n - k == 3 && s[k] == 'i' && s[k + 1] == 'n' && s[k + 2] == 'f') {
    *bits = sign | 0x7f800000u;
    return PCD_OK;
  }
  // digits: w holds the significant ones seen so far, `zeros` the zeros after them not yet known to be followed by another digit
  uint64_t w = 0;
  int nd = 0;
  long long zeros = 0, frac = 0, n_int = 0, n_frac = 0;
  constexpr long long SAT = 1ll << 40;  // counts saturate here: far past any exponent that reaches a float
  // one digit of the mantissa; false: a 20th significant digit
  auto take = [&](int dg) {
    if (dg == 0) {
      if (nd > 0 && zeros < SAT) zeros++;
      return true;
    }
    if (nd + zeros + 1 > 19) return false;
    for (; zeros > 0; zeros--) w *= 10u, nd++;
    w = w * 10u + (uint64_t)dg, nd++;
    return true;
  };
  for (; k < n && is_digit(s[k]); k++, n_int++)
    if (!take(s[k] - '0')) return PCD_TOO_LONG;
  if (k < n && s[k] == '.') {
    for (k++; k < n && is_digit(s[k]); k++, n_frac++) {
      if (!take(s[k] - '0')) return PCD_TOO_LONG;
      if (frac < SAT) frac++;
    }
  }
  if (n_int + n_frac == 0) return PCD_BAD_TOKEN;
  long long e = 0;
  if (k < n && (s[k] == 'e' || s[k] == 'E')) {
    k++;
    bool eneg = false;
    if (k < n && (s[k] == '+' || s[k] == '-')) eneg = s[k] == '-', k++;
    if (k >= n || !is_digit(s[k])) return PCD_BAD_TOKEN;
    for (; k < n && is_digit(s[k]); k++)
      if (e < SAT) e = e * 10 + (s[k] - '0');
    if (eneg) e = -e;
  }
  if (k != n) return PCD_BAD_TOKEN;
  if (w == 0) {
    *bits = sign;
    return PCD_OK;
  }
  long long q = e + zeros - frac;
  if (q > 100000) q = 100000;
  if (q < -100000) q = -100000;
  *bits = sign | decimal_to_float(w, (int)q);
  return PCD_OK;
}

}  // namespace pcd
