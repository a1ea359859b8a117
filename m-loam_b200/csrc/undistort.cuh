// TransformToEnd (utility.h:54-100) of the DISTORTION step (Estimator::undistortMeasurements, estimator.cpp:376-408), on the host and on the
// device with the same bits.  Per point, with pose = (q, t) the LiDAR's pose_undist and s the point's fraction of the sweep:
//   s    = (double)((p.i - (float)int(p.i)) / scan_period)                      float subtract and divide (intensity = ring + rel_time)
//   q_s  = Identity.slerp(s, q)                                                  Eigen 3.3's slerp, d = q.w, NOT renormalised
//   un   = (float)(q_s * p + s t)                                                TransformToStart stores to float
//   end  = (float)(q^-1 * ((double)un - t)),  q^-1 = conj(q) / |q|^2           Eigen's Quaternion::inverse
// The pose alone decides acos(|w|) and its sine: they are computed once on the host with the C library, as Eigen calls them, and staged
// (undist_pose_make).  The two sines that depend on the point run where the point is: sin_fd restates fdlibm's sin (k_sin.c, k_cos.c and
// the medium-size reduction of e_rem_pio2.c, Sun Microsystems' freely distributable libm) from + - x / only, which every translation unit
// of the project evaluates once-rounded (-fmad=false on the device, -ffp-contract=off on the host), so the device equals the host build.
// fdlibm's sin is within 1 ulp of glibc's; what must agree is the float point, and tests/test_undistort_cpu.py checks over millions of
// points that the header's transform with sin_fd gives the same floats as with the C library's sin.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define UD_HD __host__ __device__ inline
#else
#define UD_HD inline
#endif

namespace ud {

// The staged pose of one LiDAR: pose_undist as given (q_ is normalised by the Pose that holds it) and what the host derived from it
struct UndistPose {
  double q[4];      // x y z w
  double t[3];
  double qi[4];     // q.inverse(): conj(q) / squaredNorm(q), x y z w
  double theta;     // acos(|w|) (slerp's angle); unused when fast
  double sin_theta; // sin(theta)
  int fast;         // |w| >= 1 - DBL_EPSILON: slerp's linear weights 1 - s, s
  int pad;
};

// squaredNorm summed x, y, z, w in order, as the project restates Eigen's Quaternion::normalize (common.cuh qnormalized)
inline void undist_pose_make(const double *pose7, UndistPose *P) {
  std::memset(P, 0, sizeof(*P));
  for (int k = 0; k < 3; k++) P->t[k] = pose7[k];
  for (int k = 0; k < 4; k++) P->q[k] = pose7[3 + k];
  const double n2 = P->q[0] * P->q[0] + P->q[1] * P->q[1] + P->q[2] * P->q[2] + P->q[3] * P->q[3];
  if (n2 > 0.0) P->qi[0] = -P->q[0] / n2, P->qi[1] = -P->q[1] / n2, P->qi[2] = -P->q[2] / n2, P->qi[3] = P->q[3] / n2;
  const double d = P->q[3], absD = std::fabs(d), one = 1.0 - DBL_EPSILON;  // slerp from Identity: d = Identity . q = w
  P->fast = absD >= one ? 1 : 0;
  if (!P->fast) P->theta = std::acos(absD), P->sin_theta = std::sin(P->theta);
}

UD_HD int32_t hi_word(double x) {
#if defined(__CUDA_ARCH__)
  return __double2hiint(x);
#else
  uint64_t b;
  std::memcpy(&b, &x, 8);
  return (int32_t)(b >> 32);
#endif
}
UD_HD double from_words(int32_t hi, uint32_t lo) {
#if defined(__CUDA_ARCH__)
  return __hiloint2double(hi, (int)lo);
#else
  const uint64_t b = ((uint64_t)(uint32_t)hi << 32) | lo;
  double x;
  std::memcpy(&x, &b, 8);
  return x;
#endif
}

// fdlibm __kernel_sin(x, y, iy) on [-pi/4, pi/4], y the tail of x
UD_HD double kernel_sin(double x, double y, int iy) {
  const double half = 5.00000000000000000000e-01, S1 = -1.66666666666666324348e-01, S2 = 8.33333333332248946124e-03,
               S3 = -1.98412698298579493134e-04, S4 = 2.75573137070700676789e-06, S5 = -2.50507602534068634195e-08,
               S6 = 1.58969099521155010221e-10;
  const int32_t ix = hi_word(x) & 0x7fffffff;
  if (ix < 0x3e400000 && (int)x == 0) return x;  // |x| < 2^-27
  const double z = x * x, v = z * x, r = S2 + z * (S3 + z * (S4 + z * (S5 + z * S6)));
  if (iy == 0) return x + v * (S1 + z * r);
  return x - ((z * (half * y - v * r) - y) - v * S1);
}

// fdlibm __kernel_cos(x, y) on [-pi/4, pi/4]
UD_HD double kernel_cos(double x, double y) {
  const double one = 1.0, C1 = 4.16666666666666019037e-02, C2 = -1.38888888888741095749e-03, C3 = 2.48015872894767294178e-05,
               C4 = -2.75573143513906633035e-07, C5 = 2.08757232129817482790e-09, C6 = -1.13596475577881948265e-11;
  const int32_t ix = hi_word(x) & 0x7fffffff;
  if (ix < 0x3e400000 && (int)x == 0) return one;
  const double z = x * x, r = z * (C1 + z * (C2 + z * (C3 + z * (C4 + z * (C5 + z * C6)))));
  if (ix < 0x3fd33333) return one - (0.5 * z - (z * r - x * y));  // |x| < 0.3
  const double qx = ix > 0x3fe90000 ? 0.28125 : from_words(ix - 0x00200000, 0u);
  const double hz = 0.5 * z - qx, a = one - qx;
  return a - (hz - (z * r - x * y));
}

// fdlibm sin.  The argument reduction is e_rem_pio2's medium-size one (three-part pi/2, good to 151 bits), exact for |x| <= 2^19 pi/2;
// slerp's arguments are (1 - s) theta and s theta with theta <= pi/2 and s a fraction of the sweep.
UD_HD double sin_fd(double x) {
  const int32_t hx = hi_word(x), ix = hx & 0x7fffffff;
  if (ix <= 0x3fe921fb) return kernel_sin(x, 0.0, 0);  // |x| ~< pi/4
  if (ix >= 0x7ff00000) return x - x;                   // inf, NaN
  const double invpio2 = 6.36619772367581382433e-01, pio2_1 = 1.57079632673412561417e+00, pio2_1t = 6.07710050650619224932e-11,
               pio2_2 = 6.07710050630396597660e-11, pio2_2t = 2.02226624879595063154e-21, pio2_3 = 2.02226624871116645580e-21,
               pio2_3t = 8.47842766036889956997e-32;
  double t = fabs(x);
  const int n = (int)(t * invpio2 + 0.5);
  const double fn = (double)n;
  double r = t - fn * pio2_1, w = fn * pio2_1t;
  double y0 = r - w;
  const int j = ix >> 20;
  int i = j - ((hi_word(y0) >> 20) & 0x7ff);
  if (i > 16) {  // second iteration, good to 118 bits
    t = r;
    w = fn * pio2_2;
    r = t - w;
    w = fn * pio2_2t - ((t - r) - w);
    y0 = r - w;
    i = j - ((hi_word(y0) >> 20) & 0x7ff);
    if (i > 49) {  // third iteration, 151 bits
      t = r;
      w = fn * pio2_3;
      r = t - w;
      w = fn * pio2_3t - ((t - r) - w);
      y0 = r - w;
    }
  }
  double y1 = (r - y0) - w;
  int q = n;
  if (hx < 0) y0 = -y0, y1 = -y1, q = -n;
  switch (q & 3) {
    case 0: return kernel_sin(y0, y1, 1);
    case 1: return kernel_cos(y0, y1);
    case 2: return -kernel_sin(y0, y1, 1);
    default: return -kernel_cos(y0, y1);
  }
}

// q * v as Eigen's _transformVector evaluates it: v + w (2 u x v) + u x (2 u x v)  (common.cuh qrot)
UD_HD void qrot(const double q[4], const double v[3], double out[3]) {
  double uv[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
  uv[0] = uv[0] + uv[0], uv[1] = uv[1] + uv[1], uv[2] = uv[2] + uv[2];
  const double c[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
  for (int k = 0; k < 3; k++) out[k] = v[k] + q[3] * uv[k] + c[k];
}

// TransformToEnd(p, p, pose, true, scan_period) of one point (x y z intensity in p, in place); Sin: sin_fd, or the C library's sin
template <class Sin>
UD_HD void transform_to_end(const UndistPose &P, float scan_period, float p[4], Sin sn) {
  const float fr = p[3] - (float)(int)p[3];
  const double s = (double)(fr / scan_period);
  double s0, s1;
  if (P.fast) {
    s0 = 1.0 - s, s1 = s;
  } else {
    s0 = sn((1.0 - s) * P.theta) / P.sin_theta;
    s1 = sn(s * P.theta) / P.sin_theta;
  }
  if (P.q[3] < 0.0) s1 = -s1;
  // scale0 * Identity.coeffs() + scale1 * q.coeffs(), element by element
  const double qs[4] = {s0 * 0.0 + s1 * P.q[0], s0 * 0.0 + s1 * P.q[1], s0 * 0.0 + s1 * P.q[2], s0 * 1.0 + s1 * P.q[3]};
  const double v[3] = {(double)p[0], (double)p[1], (double)p[2]};
  double un[3];
  qrot(qs, v, un);
  const float uf[3] = {(float)(un[0] + s * P.t[0]), (float)(un[1] + s * P.t[1]), (float)(un[2] + s * P.t[2])};
  const double d[3] = {(double)uf[0] - P.t[0], (double)uf[1] - P.t[1], (double)uf[2] - P.t[2]};
  double e[3];
  qrot(P.qi, d, e);
  p[0] = (float)e[0], p[1] = (float)e[1], p[2] = (float)e[2];
}

}  // namespace ud
