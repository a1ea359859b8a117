// Host builds for tests/test_front_end_cpu.py and tests/test_front_end.py (g++ -ffp-contract=off, no CUDA; built by tests/front_end_lib.py
// into a temporary directory that is removed when the test process exits):
//   ref_cal_timestamp   pcl::removeNaNFromPointCloud + FeatureExtract::calTimestamp (feature_extract.cpp:25-114) restated as the reference
//                       writes it — one sequential loop, libm atan2 on floats (parameters.h:43 `using namespace std`)
//   host_cal_timestamp  csrc/cal_timestamp.cuh — what the kernels evaluate: first / last finite point and the flip index as index
//                       reductions, then every point on its own
// Both write the finite points in input order with intensity = relative time and return their count.
#include <cmath>
#include <cstdint>

#include "cal_timestamp.cuh"

using namespace std;

namespace {
struct P4 {
  float x, y, z, intensity;
};
bool finite3(const P4 &p) { return std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z); }
}  // namespace

extern "C" int ref_cal_timestamp(const float *cloud_in, int n_in, int time_field, float SCAN_PERIOD, float *cloud_out) {
  const P4 *in = reinterpret_cast<const P4 *>(cloud_in);
  P4 *out = reinterpret_cast<P4 *>(cloud_out);
  int n = 0;
  for (int i = 0; i < n_in; i++)  // removeNaNFromPointCloud
    if (finite3(in[i])) out[n++] = in[i];
  if (time_field) {  // calTimestamp(PointITimeCloud): the timestamp rides in the intensity lane
    for (int i = 0; i < n; i++) out[i].intensity = out[i].intensity * 1e-6;
    return n;
  }
  if (n == 0) return 0;
  // findStartEndAngle
  float start_ori = -atan2(out[0].y, out[0].x);
  float end_ori = -atan2(out[n - 1].y, out[n - 1].x) + 2 * M_PI;
  if (end_ori - start_ori > 3 * M_PI) end_ori -= 2 * M_PI;
  else if (end_ori - start_ori < M_PI) end_ori += 2 * M_PI;
  bool half_passed = false;
  for (int i = 0; i < n; i++) {
    float ori = -atan2(out[i].y, out[i].x);
    if (!half_passed) {
      if (ori < start_ori - M_PI / 2) ori += 2 * M_PI;
      else if (ori > start_ori + M_PI * 3 / 2) ori -= 2 * M_PI;
      if (ori - start_ori > M_PI) half_passed = true;
    } else {
      ori += 2 * M_PI;
      if (ori < end_ori - M_PI * 3 / 2) ori += 2 * M_PI;
      else if (ori > end_ori + M_PI / 2) ori -= 2 * M_PI;
    }
    float rel_time = (ori - start_ori) / (end_ori - start_ori) * SCAN_PERIOD;
    out[i].intensity = rel_time;
  }
  return n;
}

extern "C" int host_cal_timestamp(const float *cloud_in, int n_in, int time_field, float scan_period, float *cloud_out) {
  const float4 *in = reinterpret_cast<const float4 *>(cloud_in);
  float4 *out = reinterpret_cast<float4 *>(cloud_out);
  int first = INT32_MAX, last = -1, flip = INT32_MAX;
  for (int i = 0; i < n_in; i++)
    if (ts_finite(in[i])) first = first < i ? first : i, last = last > i ? last : i;
  float start_ori = 0.f, end_ori = 0.f;  // once per sweep, as k_front_flip does
  if (!time_field && last >= 0) {
    ts_start_end(in[first], in[last], &start_ori, &end_ori);
    for (int i = 0; i < n_in; i++) {
      if (!ts_finite(in[i])) continue;
      bool flips;
      ts_ori_first_half(in[i], start_ori, &flips);
      if (flips && i < flip) flip = i;
    }
  }
  int n = 0;
  for (int i = 0; i < n_in; i++) {
    if (!ts_finite(in[i])) continue;
    const float t = ts_point_time_at(in[i], i, start_ori, end_ori, flip, time_field, scan_period);
    out[n++] = float4{in[i].x, in[i].y, in[i].z, t};
  }
  return n;
}
