// pcd_format.cuh — one float -> the characters pcl::PCDWriter::writeASCII (PCL 1.8.0, precision 8) prints for it: `stream << value` in
// the classic locale at precision 8, which is printf's %.8g of the float widened to double, except that every NaN is "nan" (PCL tests
// pcl_isnan before formatting; printf prints "-nan" for a negative one).  +-inf are "inf" / "-inf", -0.0f is "-0".  Written once for the
// host and the device (csrc/pcd_write.cu, host/mloam_io.hpp's tests, the CPU tests' host build).
//
// %.8g: the value rounded to 8 significant digits, d * 10^(X - 7) with 10^7 <= d < 10^8, ties to even on the exact binary value; then
// %f style with 7 - X decimals when -4 <= X < 8, else %e style d.ddddddde+-XX (at least two exponent digits); trailing zeros of the
// fraction and a bare '.' removed.
//
// The digits: X is estimated from the binary exponent (floor(e2 log10 2), too small by at most one) and the quotient v / 10^(X - 7) is
// formed in double from exact powers of ten, at most three roundings, so within 4e-8 of the true quotient (< 10^8 + 1).  That decides
// the rounding unless the quotient's fraction lies within 1e-6 of one half; then the exact comparison of 2v with (2d + 1) * 10^(X - 7)
// (pcd_ascii.cuh cmp_dec_bin; both sides below 2^150 once aligned) decides, and an exact tie goes to the even d.  A d that rounds up to
// 10^8 becomes 10^7 with X + 1, which may switch %f to %e (99999999.5 -> 1e+08).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "pcd_ascii.cuh"

namespace pcd {

constexpr int PCD_FMT_MAX = 14;  // the longest token: "-1.2345678e-38" or "-0.00012345678"

#define PCD_POW10_DATA \
  { 1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22 }
#if defined(__CUDACC__)
static __device__ const double kPow10_dev[] = PCD_POW10_DATA;
#endif
static const double kPow10_host[] = PCD_POW10_DATA;

// 10^i, 0 <= i <= 22: exact in double
PCD_HD double pow10_exact(int i) {
#if defined(__CUDA_ARCH__)
  return kPow10_dev[i];
#else
  return kPow10_host[i];
#endif
}

PCD_HD int clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __clz((int)x);
#else
  return __builtin_clz(x);
#endif
}

PCD_HD float bits_float(uint32_t bits) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(bits);
#else
  float f;
  std::memcpy(&f, &bits, 4);
  return f;
#endif
}

// v / 10^s for v > 0 and -52 <= s <= 31, by exact powers of ten: at most three roundings
PCD_HD double div_pow10(double v, int s) {
  if (s >= 0) return s <= 22 ? v / pow10_exact(s) : v / pow10_exact(22) / pow10_exact(s - 22);
  int t = -s;
  for (; t > 22; t -= 22) v *= pow10_exact(22);
  return v * pow10_exact(t);
}

// The %.8g characters of the float with these bits into out (PCD_FMT_MAX bytes at most, no terminator); returns their count
PCD_HD int format_float(uint32_t bits, char *out) {
  const uint32_t a = bits & 0x7fffffffu;
  if (a > 0x7f800000u) {
    out[0] = 'n', out[1] = 'a', out[2] = 'n';
    return 3;
  }
  int n = 0;
  if (bits >> 31) out[n++] = '-';
  if (a == 0x7f800000u) {
    out[n] = 'i', out[n + 1] = 'n', out[n + 2] = 'f';
    return n + 3;
  }
  if (a == 0) {
    out[n] = '0';
    return n + 1;
  }
  // v = M * 2^E exactly
  const int e8 = (int)(a >> 23);
  const uint32_t M = e8 ? (a & 0x7fffffu) | 0x800000u : a;
  const int E = e8 ? e8 - 150 : -149;
  const int e2 = E + 31 - clz32(M);  // floor(log2 v)
  int X = (e2 * 78913) >> 18;        // floor(e2 log10 2): 10^X <= v < 10^(X + 2)
  const double v = (double)bits_float(a);
  double q = div_pow10(v, X - 7);
  if (q >= 1e8) X++, q = div_pow10(v, X - 7);
  const double fl = floor(q), r = q - fl;
  uint32_t d = (uint32_t)fl;
  if (r > 0.5 - 1e-6 && r < 0.5 + 1e-6) {
    // sign of 2v - (2d + 1) 10^(X - 7)
    const int c = -cmp_dec_bin(2ull * d + 1ull, X - 7, M, E + 1);
    d += (c > 0 || (c == 0 && (d & 1u))) ? 1u : 0u;
  } else {
    d += r > 0.5 ? 1u : 0u;
  }
  if (d >= 100000000u) d = 10000000u, X++;
  char dg[8];
  for (int k = 7; k >= 0; k--) dg[k] = (char)('0' + d % 10u), d /= 10u;
  int last = 7;  // the last significant digit kept: dg[0] is never '0'
  while (dg[last] == '0') last--;
  if (X < -4 || X >= 8) {
    out[n++] = dg[0];
    if (last > 0) {
      out[n++] = '.';
      for (int k = 1; k <= last; k++) out[n++] = dg[k];
    }
    out[n++] = 'e';
    out[n++] = X < 0 ? '-' : '+';
    const int ax = X < 0 ? -X : X;  // <= 45: two digits
    out[n++] = (char)('0' + ax / 10), out[n++] = (char)('0' + ax % 10);
  } else if (X >= 0) {
    for (int k = 0; k <= X; k++) out[n++] = dg[k];
    if (last > X) {
      out[n++] = '.';
      for (int k = X + 1; k <= last; k++) out[n++] = dg[k];
    }
  } else {
    out[n++] = '0', out[n++] = '.';
    for (int k = 0; k < -X - 1; k++) out[n++] = '0';
    for (int k = 0; k <= last; k++) out[n++] = dg[k];
  }
  return n;
}

}  // namespace pcd
