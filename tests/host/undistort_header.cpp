// TEST HARNESS — m-loam_b200/csrc/undistort.cuh compiled for the host (as the project's device code, once-rounded: -ffp-contract=off):
// TransformToEnd of a batch of points with the header's restated sine or with the C library's, and how many double sines differed.
#include "../../m-loam_b200/csrc/undistort.cuh"

extern "C" {

// pts / out: n x (x y z intensity); pose7: n_poses x [t q], point i takes pose i % n_poses.  use_libm: std::sin instead of ud::sin_fd.
// *sin_diff (nullable): the double sines that differ between the two, over the sines this batch evaluated.
void ud_transform(const float *pts, int n, const double *pose7, int n_poses, float scan_period, int use_libm, float *out, long long *sin_diff) {
  long long diff = 0;
  for (int i = 0; i < n; i++) {
    ud::UndistPose P;
    ud::undist_pose_make(pose7 + 7 * (i % n_poses), &P);
    float p[4] = {pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3]};
    auto libm = [&](double x) {
      const double a = std::sin(x);
      if (a != ud::sin_fd(x)) diff++;
      return a;
    };
    if (use_libm) ud::transform_to_end(P, scan_period, p, libm);
    else ud::transform_to_end(P, scan_period, p, ud::sin_fd);
    for (int k = 0; k < 4; k++) out[4 * i + k] = p[k];
  }
  if (sin_diff) *sin_diff = diff;
}

}  // extern "C"
