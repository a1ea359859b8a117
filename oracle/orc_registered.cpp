// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// C entry point of liborc_registered.so (registered.mk): pubPointCloud (lidar_mapper_keyframe.cpp:690-714) of one frame at a GIVEN pose, from
// the frame's inputs as orc_frame_ua takes them.  Built from the pieces of orc_capi.hpp: the rig partition of prepare_multi, extract_cloud,
// transform_point_to_end, FloatTransform and associate.  Never linked into the product library.
//   laser_cloud_full_res  per LiDAR l in order its part of the ring-ordered sweep (feature_extract.cpp:281's laser_cloud), every point:
//                         [TransformToEnd with poses7[l], estimator.cpp:405] -> FloatTransform(ext7[l]) with intensity = l (transformCloudFeature,
//                         visualization.cpp:40-52), or without the rig merge pointAssociateToMap with single_ext7 (nullable) -> `+=` LiDAR by
//                         LiDAR (:98); with `outlier`, laser_cloud_outlier appended (:693-694): per LiDAR whose part is not empty its first point
//                         (image_segmenter.hpp:390), FloatTransform of its extrinsic (single_ext7 or identity without the merge), intensity = l
//   laser_cloud_surf_last / laser_cloud_corner_last   surf_points_less_flat / corner_points_less_sharp after the undistortion and the merge
//                         (or the single extrinsic), before downsampleCurrentScan's filters
// then pointAssociateToMap(., pose7) on every point (:695-713).
#include "orc_capi.hpp"

using namespace orc;

namespace {
const double kIdentity7[7] = {0, 0, 0, 0, 0, 0, 1};

void put(const Cloud &c, const Pose &T, float *out, int *n_out) {
  for (size_t i = 0; i < c.size(); i++) {
    const PointI p = associate(c[i], T);
    std::memcpy(out + 4 * i, &p, sizeof(PointI));
  }
  *n_out = (int)c.size();
}
}  // namespace

extern "C" {

// ext7 (n_lidars x 7): the rig merge; nullptr: the whole sweep is one LiDAR's (n_lidars ignored), moved with single_ext7 (nullable).
// poses7 (nullable, one per LiDAR): the undistortion.  Capacities: full_out n + n_lidars points, surf_out and corner_out n points.
void orc_frame_registered(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                          const double *single_ext7, const double *poses7, float scan_period, int outlier, const double *pose7, float *full_out,
                          int *n_full, float *surf_out, int *n_surf, float *corner_out, int *n_corner) {
  const int L = ext7 ? n_lidars : 1, R = n_scans / L;
  Cloud full, outl, surf, corner;
  for (int l = 0; l < L; l++) {
    // LiDAR l's part as prepare_multi cuts it: [scan_start[l R] - 5, scan_start[(l + 1) R] - 5), the last one ending at n
    const int lo = ext7 ? scan_start[l * R] - 5 : 0, hi = (ext7 && l + 1 < L) ? scan_start[(l + 1) * R] - 5 : n;
    const Cloud part = hi > lo ? to_cloud(cloud + 4 * (size_t)lo, hi - lo) : Cloud();
    ScanInfo si;
    for (int r = 0; r < R; r++) si.scan_start_ind.push_back(scan_start[l * R + r] - lo), si.scan_end_ind.push_back(scan_end[l * R + r] - lo);
    CloudFeature f;
    extract_cloud(part, si, R, f);
    Cloud pc = part;
    if (poses7) {
      undistort_cloud(pc, poses7 + 7 * l, scan_period);
      undistort_cloud(f.corner_points_less_sharp, poses7 + 7 * l, scan_period);
      undistort_cloud(f.surf_points_less_flat, poses7 + 7 * l, scan_period);
    }
    const FloatTransform xf(ext7 ? ext7 + 7 * l : (single_ext7 ? single_ext7 : kIdentity7));
    auto to_base = [&](const Cloud &in, Cloud &out) {
      for (const PointI &p : in) out.push_back(ext7 ? xf(p, (float)l) : (single_ext7 ? associate(p, to_pose(single_ext7)) : p));
    };
    to_base(pc, full);
    to_base(f.surf_points_less_flat, surf);
    to_base(f.corner_points_less_sharp, corner);
    if (outlier && lo < hi && lo >= 0 && lo < n) outl.push_back(xf(to_cloud(cloud + 4 * (size_t)lo, 1)[0], (float)l));
  }
  full.insert(full.end(), outl.begin(), outl.end());
  const Pose T = to_pose(pose7);
  put(full, T, full_out, n_full);
  put(surf, T, surf_out, n_surf);
  put(corner, T, corner_out, n_corner);
}

}  // extern "C"
