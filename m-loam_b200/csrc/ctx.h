// ctx.h — host-side context behind the C ABI (include/mloam_b200.h) and the kernel launchers.
#pragma once
#include <cuda_runtime.h>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/mloam_b200.h"
#include "common.cuh"
#include "layout.h"
#include "undistort.cuh"

namespace mloam {

// Bumped whenever a device buffer is (re)allocated: captured CUDA graphs hold raw pointers and are re-captured
// when the epoch they were recorded in is over.
inline unsigned long long &alloc_epoch() {
  static unsigned long long e = 0;
  return e;
}

// Input / output of the per-feature line / plane fit (match_fit.cuh)
struct FitSet {
  const float4 *sorted;  // MapView::sorted of the set's map
  const float4 *pts;
  int n;
  const int *d_n;
  const int *pos;        // n * K from k_match_knn
  int half;              // double-buffered lists (SpecState): features per half, half 1 starts at pos + half * K; 0: one buffer
  unsigned char *valid;  // out
  float *coeff;          // out: n * 6
  int *nn;               // out (nullable): n * K original map indices
  int is_plane;
  const unsigned char *changed;  // nullable: 0 -> same neighbours as the previous iteration, valid/coeff already hold the fit
};
constexpr int KNN_TRACE_SLOTS = 16;  // MLOAM_KNN_TRACE=1: traced k_match_knn launches per solve (Ctx::knn_trace)

// Launch of a kernel of the single-GPU scan2map GN chain.  pdl: programmatic dependent launch (programmatic stream serialisation; a
// programmatic edge in a captured graph) — the kernel's CTAs are placed and run their prologue while the kernel before it on the stream
// finishes.  Every kernel launched so executes cudaGridDependencySynchronize before its first read of anything the kernels before it
// write, and none triggers its dependents before that wait, so everything two or more launches back is complete when a kernel starts.
// !pdl: an ordinary launch (stage profiling, multi-GPU, MLOAM_PDL=0).
template <typename... P, typename... A>
cudaError_t launch_chain(bool pdl, void (*kernel)(P...), unsigned grid, unsigned block, cudaStream_t st, A &&...args) {
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid), cfg.blockDim = dim3(block), cfg.dynamicSmemBytes = 0, cfg.stream = st;
  cfg.attrs = &attr, cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<A &&>(args)...);
}

// Speculative re-association (plain scan2map, max_inner == 1, one GPU): the matcher of GN iteration i + 1 searches at the
// candidate pose of iteration i while that candidate is evaluated.  The neighbour lists and anchors are double-buffered; the
// matcher reads half `sel` and writes the other one.  The next evaluation at x decides on the device which half is valid:
// the lists matched at xc are the right ones iff x == xc bitwise (the step was taken); otherwise x did not move, the lists of
// half `sel` still hold, and so do valid / coeff.  Written by the k_linearize tail only, read by k_match_knn / k_linearize.
struct SpecState {
  double xc[7];  // pose the next matcher searches at: the candidate of the last mode-1 tail (x at the start of a solve)
  int sel;       // half of the lists / anchors valid at LMState::x (before the evaluation at x commits the speculation); 0 at solve start
  int pad;
};
// A fit whose launch the matcher left to the first evaluation of the solve (k_linearize pass 0)
struct PendingFit {
  FitSet set[2];
  int K = 0;  // 0: nothing pending
  float min_plane_dis = 0.f;
  int check_fov = 0;
};
// Settings of one linearize_device call
struct LinOpts {
  double eig_thre;                  // evalDegenracy threshold (params.eig_thre; the tracker disables it with 0)
  int want_eig = 1;                 // k_lm mode 1: always run the 6x6 eigen-solver (1) or only when degenerate (0)
  bool collective = false;          // the collective solve (scan2map on every rank in lock-step): sum over the ranks
  bool two_pass = false;            // both evaluations of the LM iteration in one launch, if the launch can (lm_mode 1, fused tail)
  SpecState *spec = nullptr;        // speculative schedule (lm_mode 1): commit the speculation ...
  bool spec_publish = false;        // ... and publish the new candidate for the next matcher
  const PendingFit *fit = nullptr;  // the fit the matcher deferred to this evaluation (lm_mode 1)
  bool pdl = false;                 // launch_chain: programmatic dependent launch (single-GPU scan2map chain)
};

// Grow-only device buffer (cudaMalloc only when capacity is exceeded; steady-state frames allocate nothing).
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  bool in_graphs = true;  // false: no frame graph references the buffer, so its reallocation leaves the captured graphs valid
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    size_t want = bytes + bytes / 4 + 256;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    if (in_graphs) alloc_epoch()++;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <typename T>
  T *as() const {
    return reinterpret_cast<T *>(p);
  }
};

// Reserve `b` for the regions `layout` (a callable on a Carve &) takes, then point them into it: a layout lists its regions once.
template <typename Layout>
cudaError_t carve(DevBuf &b, Layout &&layout) {
  Carve sizing;
  layout(sizing);
  const cudaError_t e = b.reserve(sizing.size);
  if (e != cudaSuccess) return e;
  Carve cv(b.p);
  layout(cv);
  return cudaSuccess;
}

#define MLOAM_MAX_RINGS 1024  // rings of one (possibly multi-LiDAR) extraction
#define MLOAM_MAX_LIDARS 16

// A rig's raw sweeps concatenated LiDAR-major: LiDAR l owns points [off[l], off[l + 1]).  Zero-initialised past n_lidars (hashed whole).
struct RigLayout {
  int n_lidars;
  int off[MLOAM_MAX_LIDARS + 1];
};
// The front end of raw frames (mloam_set_front_end): removeNaNFromPointCloud + FeatureExtract::calTimestamp + the range-image projection
// of segment_cloud: 0, per LiDAR (estimator.cpp:249-261).  No padding: hashed whole into the frame graph key.
struct FrontEnd {
  int vertical_scans, horizon_scans;
  double roi_range;
  float scan_period;
  int time_field;  // 0: time from the azimuth; 1: from the point's timestamp [us] in the w lane (PointITimeCloud overload)
};
static_assert(sizeof(FrontEnd) == 24 && sizeof(RigLayout) == 4 * (MLOAM_MAX_LIDARS + 2), "hashed whole: no padding");
// A rig's PointCloud2 messages (mloam_frame_msg*): per LiDAR the caller's message and the layout it was checked against; zero past the
// rig's LiDARs.  Compared whole by the look-ahead and hashed whole into the frame graph key.
struct WireMsgs {
  mloam_pc2_msg_t msg[MLOAM_MAX_LIDARS];
  mloam_pc2_layout_t layout[MLOAM_MAX_LIDARS];
};
// The rig's ASCII PCD bodies of a PCD sweep (mloam_frame_pcd*), one per LiDAR
struct PcdFiles {
  mloam_pcd_t body[MLOAM_MAX_LIDARS];
};
static_assert(sizeof(mloam_pcd_t) == 40 && sizeof(PcdFiles) % 8 == 0, "compared whole: no padding");
static_assert(sizeof(mloam_pc2_msg_t) == 32 && sizeof(mloam_pc2_layout_t) == 40 && sizeof(WireMsgs) % 8 == 0, "hashed whole: no padding");

// The frame path's configuration as the mloam_set_* calls leave it.  The frame graph key (pipeline.cu frame_key) and the staged inputs
// (pipeline.cu stage_frame_inputs) derive from it; a value that is staged (the with_ua covariances and threshold, the outlier leaf, the
// scan period, MAP_DEG_THRE) never enters the key.
struct FrameCfg {
  int n_lidars = 1;                         // mloam_set_lidars: LiDARs batched into one frame
  bool lidar_merge = false;                 // ... was given extrinsics: features go through the rig merge (also for one LiDAR)
  double lidar_ext[MLOAM_MAX_LIDARS][7];    // ... their sensor -> base extrinsics
  bool has_ext = false;                     // mloam_set_extrinsic: the sensor -> base extrinsic applied to extracted features
  double ext[7] = {0, 0, 0, 0, 0, 0, 1};
  FrontEnd front{};                         // mloam_set_front_end: the front end of raw frames
  bool front_set = false;
  int n_layouts = 0;                        // mloam_set_front_end_layout: the PointCloud2 layouts of the rig's LiDARs (0: none given)
  mloam_pc2_layout_t layouts[MLOAM_MAX_LIDARS];
  int with_ua = 0;                          // mloam_set_uncertainty
  double ua_ext_cov[MLOAM_MAX_LIDARS][36];  // per LiDAR: pose_ext[l].cov_, row-major [translation | rotation]
  double ua_cov_meas[9];                    // COV_MEASUREMENT
  double ua_trace_threshold = 0.0;          // TRACE_THRESHOLD_MAPPING
  bool outlier_on = false;                  // mloam_set_outlier, with MAP_OUTLIER_RES
  float outlier_leaf = 0.f;
  bool undist_on = false;                   // mloam_set_distortion, with SCAN_PERIOD
  float undist_scan_period = 0.1f;
  bool reg_on = false;                      // mloam_set_registered
  bool gf_float_on = false;                 // mloam_set_gf_float, with MAP_DEG_THRE
  float gf_float_thre = 0.f;

  // The rig decision: with the merge the frame has n_lidars parts and part l goes to the base frame with lidar_ext[l]; without it, one
  // part with ext (the identity without mloam_set_extrinsic).  part_ext(0) begins the n_parts() poses, 7 doubles each.
  bool rig_merge() const { return n_lidars > 1 || lidar_merge; }
  int n_parts() const { return rig_merge() ? n_lidars : 1; }
  const double *part_ext(int l) const { return rig_merge() ? lidar_ext[l] : ext; }
};

// What the caller hands a frame: a ring-ordered cloud with its ScanInfo (mloam_frame*), or the rig's raw sweeps, which the front end
// turns into one (mloam_frame_raw*) — given as such, as PointCloud2 messages (mloam_frame_msg*, wire.cu) or as ASCII PCD bodies
// (mloam_frame_pcd*, pcd.cu)
enum class SweepKind : int { ring, raw, msg, pcd };

// One sweep of a frame (mloam_frame*) or announced for the next one (mloam_frame_set_next*).  What its kind does not use stays zero:
// the look-ahead compares the payloads (L, wire, pcdf) whole and the frame graph key hashes them whole.
struct Sweep {
  SweepKind kind = SweepKind::ring;
  const void *key = nullptr;             // the caller's pointer (host or device; the first message's or body's data): the look-ahead matches on it
  bool host = false;                     // key is a host pointer
  int n = 0, n_scans = 0;                // points (a raw-like sweep: in all of the rig's raw sweeps) and rings
  const float4 *cloud = nullptr;         // ring, raw: the sweep on the device (a host sweep: where its copy goes)
  const int *scan_start = nullptr, *scan_end = nullptr;      // ring: its ScanInfo on the device
  const int *h_scan_start = nullptr, *h_scan_end = nullptr;  // ring, host: its ScanInfo in host memory
  RigLayout L{};                         // raw, msg, pcd: where each LiDAR's points lie in the raw sweep
  WireMsgs wire{};                       // msg: the messages and the layouts they were checked against
  PcdFiles pcdf{};                       // pcd: the bodies
  const unsigned char *bytes = nullptr;  // msg, pcd from host memory: where the bytes are copied (wire_stage_offset / pcd_stage per LiDAR)
  bool raw_like() const { return kind != SweepKind::ring; }  // the front end runs before extraction
};

// the per-point association with uncertainty (uct.h): per LiDAR of the rig, and per run
struct UctLaser {
  double ext_inv[7];   // pose_ext[n].inverse()
  double compound[7];  // pose_global * pose_ext[n]
  double cov[36];      // its covariance (compoundPoseWithCov)
};
struct UctFrame {
  double pose_global[7];
  double cov_meas[9];
  double trace_threshold;
  int with_ua, n_lasers;
  int scan_frame;  // 1: the scan of a with_ua frame (downsampleCurrentScan, lidar_mapper_keyframe.cpp:376-387): no pose_global transform
};
static_assert(sizeof(UctFrame) <= 256, "UctFrame is staged in 256 B");
// the configuration of a frame's with_ua stage, copied to the device as one block (submap.cu ua_scan_stage)
struct UaStage {
  UctFrame frame;
  alignas(256) UctLaser lasers[MLOAM_MAX_LIDARS];
};
static_assert(sizeof(UaStage) == 256 + sizeof(UctLaser) * MLOAM_MAX_LIDARS, "with_ua stage layout");
// the configuration of a frame's outlier stage (mloam_set_outlier; submap.cu outlier_stage), copied to the device as one block
struct OutlierStage {
  float leaf;                        // MAP_OUTLIER_RES
  int n_lasers;                      // LiDARs of the frame (first points recorded by the extraction)
  int pad[2];
  float mat[MLOAM_MAX_LIDARS][12];   // per LiDAR the float 3x4 extrinsic of pubPointCloud's transformPointCloud (identity without one)
};
// The per-LiDAR pose_undist of one sweep as the caller gave it (mloam_frame_undistort, mloam_frame_set_next_undistort); n == 0: none
struct UndistPoses {
  int n = 0;
  double pose7[MLOAM_MAX_LIDARS][7];
  bool same_bits(const UndistPoses &o) const { return n == o.n && std::memcmp(pose7, o.pose7, sizeof(double) * 7 * (size_t)n) == 0; }
};
// the configuration of a sweep's undistortion (mloam_set_distortion / mloam_frame_undistort; undistort.cu), copied to the device as one block
// per half of the feature double buffer
struct UndistStage {
  float scan_period;                       // SCAN_PERIOD
  int n_lidars;                            // staged poses (the frame's LiDARs; 1 in the single-LiDAR path)
  int pad[2];
  ud::UndistPose pose[MLOAM_MAX_LIDARS];   // per LiDAR the pose TransformToEnd moves its features with
};

// Ctx::registered carved for one frame (registered.cu registered_layout): the clouds [MLOAM_REGISTERED_FULL_RES | _SURF | _CORNER] with
// their capacities and the kernel's device counts
struct RegOut {
  float4 *cloud[3];
  int *counts;
  int cap[3];
};

// gd_float (mloam_set_gf_float; gf_kernels.cu k_gf_full_hessian): what the mapper carries from frame to frame, on the device.
// k_gf_select reads ratio_cur there, so the host never sees the ratio on a frame's path.
struct GfFloatState {
  double ratio_cur;    // gf_ratio_cur (lidar_mapper_keyframe.cpp:1248, :474-492)
  double deg_factor;   // gf_deg_factor of the last evaluation (:470)
  int total_feat_num;  // matched surf + corner features of the last evaluation
  int evaluations;     // evaluations since the mode was turned on
};
// Ctx::gf_float: the state, then the device end of PinnedBlock::gf_float_cfg
struct GfFloatDev {
  GfFloatState st;
  double cfg[2];
};

// The byte sizes of the ASCII PCD bodies a decode reads (pcd.cu), and where a host body lies in the staging: read on the device, so that
// the launches depend on the bodies' point counts only
struct PcdStage {
  long long size[MLOAM_MAX_LIDARS];
  long long off[MLOAM_MAX_LIDARS];
};

// The context's pinned host block (Ctx::pinned): staging of small host-to-device copies and landing of small read-backs, so that
// they are truly asynchronous.
struct PinnedBlock {
  // Read by captured copies: a frame graph copies these to the device at execution time.  pipeline.cu stage_frame_inputs writes them
  // from FrameCfg before a frame is enqueued and before every replay; the stages below only copy them.
  double pose[7];                   // lm_init_state: the initial pose of a solve
  double ext[7];                    // features_enqueue: the single sensor -> base extrinsic
  float rig[MLOAM_MAX_LIDARS][12];  // features_enqueue: the rig's float 3x4 extrinsics of the merge
  UaStage ua;                       // ua_scan_stage: the with_ua configuration
  OutlierStage outlier;             // outlier_stage: the outlier cloud's configuration
  UndistStage undist[2];            // undistort_stage: per half of the feature double buffer, the poses of the sweep in that half
  // Written by captured copies (landing of a frame's results) and by the host-buffer entry points, one call at a time
  LMState lm;                       // LMState mirror
  int counts[192];                  // count read-backs; mloam_project_cloud: [0] count, [64..] scan starts, [128..] scan ends
  double pose_cov[36];              // H^-1 of the last solve (with_ua)
  GridHdr map_hdr[MLOAM_NUM_MAPS];  // map_build_device: the GridHdr head of each slot's last build (auto cell)
  int done;                         // LM done-flag poll of the solves with max_inner > 1
  double upload_pose[7];            // upload_pose
  double odom_x[21];                // odometry / good-feature poses: pivot | pose_i | ext (DevCtl::odom_x)
  alignas(16) unsigned char odom[4096];  // OdomState mirror (odom_kernels.cu)
  double normal_eq[30];             // mloam_normal_equations read-back
  double pose_plus[64];             // mloam_pose_plus: x | delta | V in, result at [56]
  double gf_float_cfg[2];           // scan2map_enqueue (gd_float): MAP_DEG_THRE | gf_ratio_ini, read by a captured copy like pose
  GfFloatState gf_float;            // GfFloatState mirror, landed with LMState
  int scan_info[2][MLOAM_MAX_RINGS];       // mloam_frame: ScanInfo of the sweep (start | end)
  int scan_info_next[2][MLOAM_MAX_RINGS];  // ... and of the announced next sweep, copied on Ctx::br_ahead
  PcdStage pcd;                            // pcd.cu: the ASCII bodies' sizes and staging offsets, copied to the device by the decode
  unsigned pcd_status;                     // ... and the PCD_E_* bits of the bodies it refused
  PcdStage pcd_half[2];                    // PCD frames: per half of the feature double buffer, the staged bodies of the sweep decoded into it
  unsigned pcd_half_status[2];             // ... and their refusal bits, landed with the frame's results
};

// Matcher counters of k_match_knn with stage profiling on (mloam_profile_get "knn_*"); zeroed at creation and by mloam_profile_reset
struct KnnPathStats {
  unsigned queries[4];           // per search path: 0 keep (matched), 1 keep (rejected), 2 ball, 3 blind
  unsigned max_query_cycles;
  unsigned over_32k, over_64k;   // queries over 32k / 64k cycles
  unsigned pad0;
  unsigned long long cycles[4];  // SM cycles per path
  unsigned long long slowest;    // cycles << 32 | path << 30 | set << 29 | feature index
  unsigned long long pad1[3];
  unsigned long long blind[8];   // blind searches: 0, cycles of ring 1 / ball, ring-1 points, ball points / steps / rows, queries with a ball
  long long slow_rec[10];        // one blind query over 90k cycles
  long long pad2[2];
};
static_assert(sizeof(KnnPathStats) == 256 && offsetof(KnnPathStats, cycles) == 32 && offsetof(KnnPathStats, blind) == 96 &&
                  offsetof(KnnPathStats, slow_rec) == 160,
              "k_match_knn addresses the counters by these offsets");

// Device control words (Ctx::ctl): the device ends of the pinned staging and small fixed-size results
struct DevCtl {
  double pose[8];                       // PinnedBlock::pose
  double upload_pose[8];                // PinnedBlock::upload_pose
  double ext[8];                        // PinnedBlock::ext
  double odom_x[24];                    // PinnedBlock::odom_x
  double normal_eq[32];                 // mloam_normal_equations
  double pose_plus[64];                 // mloam_pose_plus
  float rig[MLOAM_MAX_LIDARS][12];      // PinnedBlock::rig
  KnnPathStats knn_stats;
};

struct MapStorage {
  DevBuf sorted, orig, cells, rank_of, tile_sums, hdr;
  unsigned capacity = 0;  // cells the dense grid may use (4 B each)
  int m = 0;
  float cell = 0.f;       // requested cell edge of the last build (the device may have coarsened it: GridHdr::level)
  float auto_cell = 0.25f;  // map_cell <= 0: cell edge picked from the occupancy statistics of the previous build
  bool built = false;
  MapView view() const {
    MapView v;
    v.sorted = sorted.as<float4>();
    v.orig = orig.as<float4>();
    v.cell_start = cells.as<unsigned>();
    v.hdr = hdr.as<GridHdr>();
    v.m = m;
    return v;
  }
  // Sticky auto cell: a cell edge that gives a few points per occupied cell lets the 3x3x3 neighbourhood of a query
  // hold its K neighbours (knn.cuh ring 1).  Decided from the header the previous build of this slot copied to pinned
  // memory (possibly one build stale — it only steers speed, never results).  Power-of-two edges only.
  float auto_cell_pick(const PinnedBlock *pinned, int slot) {
    if (built && pinned) {
      const GridHdr *h = &pinned->map_hdr[slot];
      if (h->n_occupied > 0 && h->n_sorted > 0 && h->cell > 0.f) {
        const float avg = (float)h->n_sorted / (float)h->n_occupied;
        float cur = h->cell;
        if (avg < 2.5f && cur < 1.0f) cur *= 2.0f;
        else if (avg > 40.0f && cur > 0.125f) cur *= 0.5f;
        auto_cell = cur;
      }
    }
    return auto_cell;
  }
};

struct ProfSlot {
  double ms = 0;
  long long launches = 0;
};

// Parameters the kernels need, flattened from mloam_params_t.
struct MatchCfg {
  float min_match_sq_dis, min_plane_dis;
  int n_neigh, check_fov;
};

struct KeyframeStore;

// A side stream with the events of its fork from and its join into Ctx::stream (pipeline.cu on_branch)
struct Branch {
  cudaStream_t stream = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
};

struct Ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  Branch br_maps;                        // submap upload + build, concurrently with extraction
  Branch br_scan;                        // corner-scan voxel filter next to the surf-scan one; corner good-feature selection; speculative matcher
  Branch br_ahead, br_ahead_scan;        // look-ahead extraction and its corner-voxel fork
  cudaEvent_t ev_maps = nullptr;         // recorded on br_maps after the host API's submap H2D copies
  bool maps_pending = false;             // the map-build branch must wait on ev_maps (external to a captured graph)
  mloam_params_t params;
  std::string err;
  long long launches = 0;

  MapStorage maps[MLOAM_NUM_MAPS];

  // scan features (device copies when the caller passes host buffers)
  DevBuf scan_pts[2];             // [0] corner, [1] surf
  DevBuf feat_valid[2];           // unsigned char per query
  DevBuf feat_coeff[2];           // float[6] per query
  DevBuf feat_nn[2];              // int[n_neigh] per query (optional)
  DevBuf knn_pos[2];              // int[n_neigh] per query: neighbour positions handed from k_match_knn to k_match_fit
  DevBuf knn_changed[2];          // unsigned char per query: neighbour list differs from the previous iteration's
  DevBuf knn_anchor[2];           // float4 per query: position of its last real search + tolerated displacement
  DevBuf knn_spec;                // SpecState of the speculative scan2map schedule
  DevBuf gf_work[2];              // good-feature selection scratch per set (Jacobian rows, pool tree, mask, ...)
  DevBuf knn_heavy[2];            // 2 x unsigned char per query: "needed a real search" verdicts of the last two launches
  DevBuf knn_heavy_list;          // 3 rotating counters + 2 lists of feature indices that needed a real search (match_kernels.cu HeavyQ)
  int knn_rot = 0;                // launch ordinal inside the current solve (rotation of the heavy lists / counters)
  int knn_parity = 0;             // which half of knn_heavy the next seeded launch reads
  int knn_half[2] = {0, 0};       // per set: features per half of knn_pos / knn_anchor in its last launch (0: one half)
  int knn_k = 0;                  // neighbours per feature of the last launch
  MapView knn_map[2] = {};        // per set: the map its last launch searched (mloam_debug_knn_lists)
  DevBuf partials;                // per-block packed normal equations
  DevBuf lm_state;                // LMState
  void *ticket_zeroed_for = nullptr;  // partials allocation whose last-block ticket has been zeroed
  // Work buffers, named by their role in a frame.  The host-buffer entry points, each one synchronous call, stage through them too.
  DevBuf sweep_in;                // mloam_frame: the sweep + its ScanInfo.  Host entry points: their input
  DevBuf map_in[2];               // mloam_frame: the surf / corner submap uploads on br_maps.  Host entry points: [0] their output
  DevBuf extract_work;            // extract_device (extract_work_layout); the look-ahead branch reuses it after the current extraction
  DevBuf voxel_work;              // voxel filters of the host entry points and of the keyframe submap
  DevBuf voxel_corner, voxel_surf;  // the frame's two scan filters, on two streams at once; the look-ahead branch forks after them
  DevBuf host_work;               // host entry points: work and output staging (good features, kNN, factors, scan2map_ua, ...)
  DevBuf odom_work;               // OdomState + partials of mloam_odom_solve
  DevBuf rig_work;                // mloam_calib_rig / mloam_calib_frame: the rig's features, their matches and fits, RigState, partials (calib_rig.cu)
  // association work (uct.h uct_bufs) of the keyframe submap and the host entry points: never inside a frame, so it shares the
  // corner submap upload's allocation
  DevBuf &assoc_work() { return map_in[1]; }
  DevBuf ctl;                     // DevCtl
  PinnedBlock *pinned = nullptr;

  // profiling with CUDA events on `stream`
  bool prof_on = false;
  std::map<std::string, ProfSlot> prof;
  struct PendingEvt {
    std::string name;
    cudaEvent_t a, b;
  };
  std::vector<PendingEvt> pending;
  std::vector<cudaEvent_t> evt_pool;

  // NCCL (multi-GPU); opaque here
  void *d_ring_stage = nullptr;     // RingStage[n_scans] of the last extraction (extract_kernels.cu)
  int *d_ring_cnt = nullptr;        // per-ring less-flat centroid counts of the last extraction
  int *d_extract_status = nullptr;  // device flag of the last extraction (1: ring window overflow / bad ScanInfo)
  // CUDA-graph cache of whole frames (pipeline.cu frame_run)
  struct ScanRef {
    const float4 *surf;
    int n_surf;            // count or upper bound
    const int *d_n_surf;   // nullable device-side count
    const float4 *corner;
    int n_corner;
    const int *d_n_corner;
    const double *sinfo_surf, *sinfo_corner;  // nullable per-feature sqrt_info (uncertainty-aware mapping)
    const float *cov6_surf, *cov6_corner;     // nullable PointIWithCov::cov_vec per feature (with_ua frame: gated scans)
    // the raw first point of each LiDAR's part of the ring-ordered sweep (first_ok[l] = 0: the part is empty), recorded by the
    // extraction into the sweep's half of the feature double buffer (ExtractOut::first)
    const float4 *first;
    const int *first_ok;
    // laser_cloud_outlier_cov of the frame (mloam_set_outlier; null when the outlier stage did not run): points, cov_vec, device count
    const float4 *outlier;
    const float *cov6_outlier;
    const int *d_n_outlier;
  };
  // Sweep look-ahead (mloam_frame_set_next*): while frame k is matched and solved, the features of sweep k+1 are extracted and
  // down-sampled on a side stream into the other half of a double buffer — the reference runs the two stages in different nodes
  // (estimator -> lidar_mapper), so they overlap there too.  `Features` describes one half.
  struct Features {
    bool valid = false;
    int parity = 0;
    Sweep sw;                   // the sweep they were extracted from
    ScanRef S{};
    bool extract_only = false;  // the undistortion was on: the half holds the extraction only (undistortion, merge and the scan
                                // filters run at the frame call, which knows the sweep's pose)
    bool registered = false;    // the registered clouds were on: the half also holds the sweep itself (FrameBufs::reg_sweep)
    UndistPoses undist;         // n > 0: the undistortion was on and the look-ahead ran it too, with these poses (the sweep's announced
                                // ones); a call takes the half only with the same bits
  };
  struct NextSweep {
    bool set = false;
    Sweep sw;                   // a host sweep's device buffers are set when its copy is enqueued (pipeline.cu stage_next_sweep)
    bool undist_open = false;   // mloam_frame_set_next_undistort may still give its poses: no setter has withdrawn them since
    UndistPoses undist;         // ... and the poses it gave
  };
  // The sweep announced with the last mloam_frame* call and its poses (mloam_frame_set_next_undistort): the call that takes that sweep
  // undistorts it with them unless it gives its own (mloam_frame_undistort).  Consumed by the next mloam_frame* call.
  struct AnnouncedPoses {
    Sweep sw;
    UndistPoses undist;
  };
  // A frame's results on the host, applied by pipeline.cu frame_commit on the stream, capture and replay paths alike
  struct FrameOutcome {
    ScanRef S{};                   // the scan the solve took (Ctx::last_scan)
    int ran = 0;                   // the map gate passed and the solve ran
    Features next{};               // the announced sweep's features, valid when the frame ran the look-ahead (Ctx::prefetched)
    RegOut reg{};                  // where the registered clouds went (Ctx::reg_last)
    bool gf_evaluated = false;     // gd_float evaluated the full Hessian (Ctx::gf_float_evaluated)
  };
  FrameCfg cfg;                    // what the mloam_set_* calls configured for the frame path
  // raw frames (mloam_set_front_end, mloam_frame_raw*): the front end runs inside features_enqueue, on the main stream and in the look-ahead
  // branch.  Its work (winner images, sort) and output (projected cloud + ScanInfo) have buffers of their own: the look-ahead reuses them
  // after the main stream's front end, while the main stream runs the with_ua stage and the solve.
  DevBuf front_work, front_out;
  DevBuf wire_out;                 // message frames (mloam_frame_msg*): the unpacked raw sweep the front end reads, on either stream like front_out
  // mloam_cloud_msgs* (wire.cu): the packed PointCloud2 bytes of the last call, each message 256-byte aligned, then the widths.  No frame
  // graph references it, so its growth re-captures nothing.
  DevBuf cloud_msgs{nullptr, 0, false};
  // mloam_cloud_pcd* / mloam_pcd_encode (pcd_write.cu): the files of the last call, each 256-byte aligned, then their sizes; the points
  // uploaded for it (caller clouds, keyframe positions); the tile ticket counter and the look-back's tile words.  No frame graph
  // references them.  The ticket counter is never reset: pcd_tickets is its value, and each call's tile words carry pcd_epoch.
  DevBuf pcd_files{nullptr, 0, false}, pcd_src{nullptr, 0, false}, pcd_tiles{nullptr, 0, false};
  unsigned long long pcd_tickets = 0;
  unsigned pcd_epoch = 0;
  // mloam_pcd_decode* / mloam_front_end_pcd (pcd.cu): the host bodies' staging, and the PcdStage, per-CTA line counts and status word
  DevBuf pcd_in{nullptr, 0, false}, pcd_work{nullptr, 0, false};
  // PCD frames (pcd.cu pcd_decode_half): per half of the feature double buffer, the PcdStage, status word and per-CTA line counts
  DevBuf pcd_frame;
  Features prefetched;             // features of the sweep announced with the previous frame, ready when that frame returned
  NextSweep next;                  // announced for the frame being enqueued (consumed by it)
  bool next_pending = false;       // its H2D copy was enqueued on br_ahead outside of any capture (ev_next)
  int frame_parity = 0;
  int use_lookahead = 1;           // MLOAM_LOOKAHEAD=0: announcements are ignored
  bool stamp_mute = false;
  DevBuf frame_main, frame_alt, next_in;  // the two halves of the frame feature double buffer; the announced sweep's staging
  cudaEvent_t ev_next = nullptr;
  struct GraphEntry {
    unsigned long long key = 0, epoch = 0;
    cudaGraphExec_t exec = nullptr;
    int launches = 0, seen = 0;
    FrameOutcome out{};            // what every replay of the graph leaves
  };
  std::vector<GraphEntry> graphs;
  bool smem_opt_in_gf = false;     // k_gf_select's 200 KB pool
  bool smem_opt_in[3] = {false, false, false};  // >48 KB dynamic shared memory enabled for k_voxel_small / k_ring_pick / k_ring_voxel
  long long graph_captures = 0;          // frame graphs captured and instantiated (mloam_profile_get "graph_captures")
  long long graph_capture_failures = 0;  // frames that fell back to the stream path because their capture failed (mloam_profile_get "graph_capture_failures")
  int use_graphs = 1;
  unsigned knn_tma_min = 8;        // kNN staging: runs of >= this many points use TMA bulk copies, shorter ones 16 B loads (MLOAM_KNN_TMA_MIN)
  // MLOAM_KNN_TRACE=1 (diagnosis, tools/knn_micro.py, tools/trace_replay.py --phases): per k_match_knn launch of the last solve
  // (KNN_TRACE_SLOTS slots of knn_trace_slot bytes) 4 words per query, then the per-warp [enter, exit] %globaltimer timeline
  DevBuf knn_trace;
  bool knn_trace_on = false;
  int knn_trace_n = 0;             // slots written since the last solve began
  size_t knn_trace_slot = 0, knn_trace_timeline = 0;  // bytes per slot; where in a slot the timeline begins
  // MLOAM_LIN_TRACE=1 (diagnosis, tools/trace_replay.py --phases): %globaltimer / clock64 stamps at the phase boundaries of
  // k_linearize's pass 0, one slot per evaluation at x of the last solve (LIN_TRACE_SLOTS slots of LIN_TRACE_WORDS words)
  DevBuf lin_trace;
  bool lin_trace_on = false;
  int lin_trace_n = 0;
  // MLOAM_STAMP=1 (diagnosis, tools/stamp_frame.py): one-thread kernels that write %globaltimer between the stages of a frame, so that
  // the stage times of a GRAPH REPLAY can be read (the event scopes of mloam_profile_enable force the stream path and add launch gaps)
  bool stamp_on = false;
  DevBuf stamps;
  int stamp_n = 0;
  std::vector<std::string> stamp_labels;
  int knn_min_blocks = 3;          // k_match_knn instance: resident CTAs per SM it is compiled for (MLOAM_KNN_MB = 2 | 3, match_kernels.cu)
  // MLOAM_KNN_SCHEDULE=0: k_match_knn as before the shortened queries — every ball and blind search listed for the next launch
  // (HeavyQ) and the selection unpruned by the search bound (scan_runs).  Same results; kept to compare the two
  bool knn_all_searches = false;
  int use_seeds = 1;               // seed the kNN of re-association iterations > 0 with the previous neighbour lists
  int fuse_iter = 1;               // scan2map: fit inside the first evaluation + both evaluations of an LM iteration in ONE launch
                                   // (grid barrier between them); MLOAM_FUSE_ITER=0 restores the three launches
  int lm_tail_serial = 0;          // the LM step on one thread of the tail block (MLOAM_LM_TAIL=serial) instead of one warp; bit-identical
  int use_pdl = 1;                 // scan2map's GN chain with programmatic dependent launch (launch_chain); MLOAM_PDL=0: ordinary launches,
                                   // the reference the tests compare against
  int graph_pdl_edges = 0;         // programmatic edges of the last instantiated frame graph (mloam_debug_pdl)
  bool frame_from_graph = false;   // the last frame ran from a frame graph
  void *nccl_comm = nullptr;
  int nranks = 1, rank = 0;
  // peer-memory exchange of the packed normal equations (comm.cu, solve_kernels.cu lm_tail): every rank's exchange
  // buffer is mapped into every other rank through CUDA IPC; p2p_on replaces the NCCL all-reduce + two extra launches
  // by stores / polls over NVLink inside the k_linearize tail
  void *p2p_local = nullptr;
  void *p2p_peer[MLOAM_P2P_MAX_RANKS] = {nullptr};
  void *p2p_view = nullptr;        // device copy of the P2PView the kernels read
  bool p2p_on = false;
  // uncertainty-aware mapping in the frame path (FrameCfg::with_ua): the per-point uncertainty + trace gate of downsampleCurrentScan
  // (lidar_mapper_keyframe.cpp:356-421) between the scan filters and the solve, and the pose covariance H^-1 at the returned pose (:600-610)
  DevBuf ua_scan;                  // gated scans of the last with_ua frame (points, cov6, sqrt_info, counts) + its staged configuration
  DevBuf pose_cov;                 // 36 doubles: H^-1 of the last solve (k_pose_cov), copied back with LMState
  // the outlier cloud of segment_cloud: 0 (FrameCfg::outlier_on): per LiDAR the first point of its ring-ordered sweep -> base frame ->
  // VoxelGridCovarianceMLOAM<PointI>(MAP_OUTLIER_RES) -> the with_ua gate (lidar_mapper_keyframe.cpp:366-418), one launch next to the
  // with_ua stage
  DevBuf outlier;                  // the staged configuration, the frame's outlier cloud (points, cov_vec) and its count
  // DISTORTION (FrameCfg::undist_on): TransformToEnd of each LiDAR's less-sharp and less-flat features with the pose of
  // mloam_frame_undistort (estimator.cpp:545-590, :376-408), one launch before the rig merge.  The poses are staged like the scan period
  // (PinnedBlock::undist), so a captured frame replays with new ones.  A pose is consumed by one mloam_frame* call.
  bool undist_set = false;         // a pose was given for the next mloam_frame* call
  int undist_n = 0;
  double undist_pose7[MLOAM_MAX_LIDARS][7];
  DevBuf undist;                   // the staged configuration, one UndistStage per half of the feature double buffer
  AnnouncedPoses undist_announced;  // the poses announced with the sweep of the last call's look-ahead, for the call that takes it
  long long undist_ahead_taken = 0;  // sweeps undistorted by the look-ahead and taken by their frame call (mloam_profile_get "undistort_ahead")
  // gd_float (FrameCfg::gf_float_on): every 10th solve call that passes the map gate evaluates the full information matrix of the scan
  // (evalFullHessian) from the Jacobian rows of outer iteration 0 and sets the ratio k_gf_select reads from GfFloatDev.  Allocated once,
  // outside alloc_epoch(): turning the mode on re-captures nothing.  MAP_DEG_THRE and gf_ratio_ini are staged (PinnedBlock::gf_float_cfg).
  long long gf_float_frames = 0;   // frame_cnt (:1059): solve calls since the mode was turned on
  bool gf_float_eval = false;      // this call's frame_cnt % 10 == 0
  bool gf_float_evaluated = false; // ... and it passed the map gate: the last call evaluated
  bool gf_float_reported = false;  // a solve call has run since the mode was turned on
  DevBuf gf_float;                 // GfFloatDev
  GfFloatState gf_float_host{};    // the state as the last solve call left it (mloam_gf_float_report)
  // pubPointCloud (FrameCfg::reg_on; registered.cu): the full-resolution sweep with its outlier points, surf_last and corner_last in
  // the map frame, written by one launch at the end of every mloam_frame* call.  The extraction keeps the ring-ordered sweep in the
  // sweep's half of the feature double buffer, because the sweep's own buffers are reused before the frame that registers it ends.
  bool reg_valid = false;          // Ctx::registered holds the clouds of the last mloam_frame* call
  DevBuf registered;               // the three clouds and their device counts (registered_layout)
  RegOut reg_last{};               // where the last frame's clouds are
  double pose_cov36[36] = {0};     // pose_wmap_curr.cov_ of the last mloam_frame* / mloam_scan2map* call
  bool last_scan_valid = false;    // last_scan describes the scan of the last mloam_frame* call (mloam_frame_scan)
  ScanRef last_scan{};
  // keyframe store (keyframe.cu, mloam_keyframes_init): saveKeyframe / extractSurroundingKeyFrames on device-resident keyframes
  KeyframeStore *kf = nullptr;
  double last_pose7[7] = {0, 0, 0, 0, 0, 0, 1};  // pose_wmap_curr returned by the last mloam_frame* call
  bool frame_since_save = false;   // an mloam_frame* call has run since the last mloam_keyframe_save / mloam_keyframes_init
};

// RAII-less helper: bracket a kernel (or a few) with events when profiling is on.
struct ProfScope {
  Ctx *c;
  cudaEvent_t a = nullptr, b = nullptr;
  const char *name;
  ProfScope(Ctx *ctx, const char *nm);
  ~ProfScope();
};
void prof_collect(Ctx *c);

// A communicator or a peer-memory exchange is attached: the single-GPU features (with_ua frames, outlier, ..., keyframe store) refuse it
inline bool multi_gpu(const Ctx *c) { return c->nccl_comm != nullptr || c->p2p_on; }

#define MLOAM_CUDA_OK(ctx, expr)                                                                      \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) {                                                                          \
      (ctx)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                                \
      return MLOAM_E_CUDA;                                                                            \
    }                                                                                                 \
  } while (0)

// ---------------------------------------------------------------- launchers (one per .cu)
// map_kernels.cu
int map_build_device(Ctx *c, int slot, const float4 *d_pts, int m, float cell);
int knn_device(Ctx *c, int slot, const float4 *d_q, int nq, const double *d_pose7_or_null, int k, float max_sqdist,
               int *d_idx, float *d_sqd);
// type 'c' / 's'.  d_pose7 device pointer to 7 doubles.  Outputs: valid[n], coeff[n*6] float, nn[n*n_neigh] (nullable)
// d_n (nullable): device-side feature count, n is then the launch upper bound.
int match_from_map_device(Ctx *c, int slot, int type, const float4 *d_pts, int n, const int *d_n, const double *d_pose7,
                          const MatchCfg &cfg, unsigned char *d_valid, float *d_coeff, int *d_nn);

// match_kernels.cu: one kNN launch + one fit launch over up to two feature sets
struct MatchJob {
  int slot;                 // map slot
  int type;                 // 'c' (line fit) | 's' (plane fit)
  const float4 *pts;        // sensor-frame features
  int n;                    // count / upper bound
  const int *d_n;           // nullable device-side count
  unsigned char *valid;     // out
  float *coeff;             // out, n * 6
  int *nn;                  // out, nullable, n * n_neigh original indices
  int seeded;               // 1: same features against the same map as the previous call with this job index — its neighbour
                            // lists (Ctx::knn_pos) seed the search and unchanged lists keep their fit
};
// defer (nullable): skip the fit launch and write the fit into *defer for the caller's next linearize_device(lm_mode 1) (LinOpts::fit);
// defer->K == 0 when the fit was launched here (a job wants neighbour indices) or nothing was matched.  nullptr: fit now.
// d_sel (speculative schedule, with defer): double-buffered lists, read half *d_sel and write the other (SpecState::sel)
// pdl: the kNN launch is a link of scan2map's GN chain (launch_chain)
int match_pair_device(Ctx *c, const MatchJob *jobs, int n_jobs, const double *d_pose7, const MatchCfg &cfg, PendingFit *defer = nullptr,
                      const int *d_sel = nullptr, bool pdl = false);
// the k_match_knn instance this context launches for K (non-instrumented): resident CTAs per SM by the occupancy calculator, registers
int knn_residency(const Ctx *c, int K, int *ctas_per_sm, int *regs);

// track_kernels.cu
int match_from_scan_device(Ctx *c, int slot, int type, const float4 *d_pts, int n, const double *d_pose7, unsigned char *d_valid,
                           float *d_coeff, int *d_nn3);
int track_cloud_device(Ctx *c, const float4 *d_prev_less_sharp, int n_pls, const float4 *d_prev_less_flat, int n_plf,
                       const float4 *d_cur_sharp, int n_cs, const float4 *d_cur_flat, int n_cf, const double *pose_ini7,
                       double *pose_out7, mloam_solve_stats_t *stats);

// solve_kernels.cu
struct FeatSet {
  const float4 *pts;           // sensor-frame points
  const unsigned char *valid;
  const float *coeff;          // float[6]
  int n;                       // count, or launch upper bound when d_n is set
  int is_plane;                // 1: LidarMapPlaneNormFactor, 0: LidarMapEdgeFactor
  const int *d_n;              // nullable device-side count
  const double *sinfo;         // nullable per-feature sqrt_info (with_ua: lidar_map_factor.hpp:34,41 on the point's covariance)
  const unsigned char *mask;   // nullable: only features with mask[i] != 0 enter (good-feature selection)
};
// Accumulate loss-corrected normal equations of both feature sets at pose *d_pose7 (or LMState x / xc when
// use_state != 0: 1 -> x, 2 -> xc) into c->partials, then run the LM state machine step (`lm_mode`):
//   0: none (partials only, reduced into d_out28 if non-null)   1: begin Solve   2: iterate
// two_pass_done (nullable): whether the launch ran both evaluations of the LM iteration (LinOpts::two_pass honoured)
int linearize_device(Ctx *c, const FeatSet *sets, int n_sets, double sqrt_info, double huber_a, const double *d_pose7,
                     int use_state, int lm_mode, double *d_out29, const LinOpts &o, bool *two_pass_done = nullptr);
// Evaluation at LMState::xc + the acceptance step (mode 2) of a solve with max_inner == 1, as the second pass of
// k_linearize computes it, but accumulating only g, cost and row counts (H at xc is never read with one LM iteration).
// Small blocks with a register cap, so that it runs beside the speculative matcher of the next GN iteration.
int eval_candidate_device(Ctx *c, const FeatSet *sets, int n_sets, double sqrt_info, double huber_a, double eig_thre, bool pdl);
// min_corr: minimum matched features for a Solve (tracker: 10); spec (nullable): also start SpecState::xc at the initial pose;
// pdl: launch_chain
int lm_init_state(Ctx *c, const double *pose7_host, int max_inner, int min_corr, SpecState *spec = nullptr, bool pdl = false);
void eig_report_host(const double *H36, double *w6);  // ascending eigenvalues of a symmetric 6x6 (host side)
int factor_evaluate_device(Ctx *c, int kind, int n, const double *d_points, const double *d_coeffs, const double *d_sqrt_info,
                           const double *d_params, double *d_res, double *d_jac);

// in place: p <- T * p for the first min(n, *d_n) points (pointAssociateToMap, utility.h:103-117); d_pose7 on device
int transform_points_device(Ctx *c, float4 *d_pts, int n, const int *d_n, const double *d_pose7);

// gf_kernels.cu: good-feature selection of one matched feature set on the device (goodFeatureMatching inside
// scan2MapOptimization): Jacobian rows + selection, result as a 0/1 mask over the features (set index t: 0 corner, 1 surf)
// d_ratio (nullable): the ratio on the device (GfFloatState::ratio_cur), read in place of gf_ratio.  phase: 3 rows + selection,
// 1 the Jacobian rows only, 2 the selection over the rows phase 1 left (an evaluation frame puts gf_full_hessian_device between them)
int gf_select_set_device(Ctx *c, int t, const FeatSet &fs, const double *d_pose7, double default_sinfo, int method, double gf_ratio,
                         unsigned long long seed, unsigned char **d_mask_out, const double *d_ratio = nullptr, int phase = 3);
// evalFullHessian + the gd_float policy over the rows phase 1 left in Ctx::gf_work for sets[1] (surf) then sets[0] (corner): one launch
int gf_full_hessian_device(Ctx *c, const FeatSet *sets);
void stage_gf_float(Ctx *c);  // writes PinnedBlock::gf_float_cfg

// uct_kernels.cu: per-point sqrt_info from PointIWithCov::cov_vec (float[6] per point)
int sqrt_info_device(Ctx *c, const float *d_cov6, int n, double *d_sinfo);
// submap.cu: the with_ua stage of a frame (downsampleCurrentScan, lidar_mapper_keyframe.cpp:356-421) on c->stream.  The scans of *S
// (device counts) -> per point ext^-1 -> evalPointUncertainty under pose_ext -> trace gate -> stable compaction into Ctx::ua_scan with
// cov6 and sqrt_info; *S then points at the gated scans.  ua_stage_host stages its configuration (PinnedBlock::ua).
// d_cfg (nullable): where the staged configuration lies on the device (the outlier stage reads its with_ua part)
int ua_scan_stage(Ctx *c, Ctx::ScanRef *S, const UaStage **d_cfg = nullptr);
void ua_stage_host(Ctx *c);
// submap.cu: the outlier stage of a frame (downsampleCurrentScan, lidar_mapper_keyframe.cpp:366-418) on c->stream, after ua_scan_stage:
// the first points S->first of the LiDARs' parts of the sweep -> float extrinsic, intensity = laser id -> VoxelGridCovarianceMLOAM<PointI>
// (MAP_OUTLIER_RES) -> with d_ua (the with_ua stage's configuration) the trace gate, else zero cov_vec -> Ctx::outlier, *S's outlier
// fields.  One single-CTA launch.  stage_outlier stages its configuration (PinnedBlock::outlier).
int outlier_stage(Ctx *c, Ctx::ScanRef *S, const UaStage *d_ua);
void stage_outlier(Ctx *c);
// registered.cu: pubPointCloud (lidar_mapper_keyframe.cpp:690-714) of a frame, one launch on c->stream after the solve.  Per point of the
// three clouds: [TransformToEnd] -> [the float rig matrix, intensity = laser id | pointAssociateToMap with the single extrinsic] for the sweep
// (the less-* features and the outlier points arrive in the base frame already) -> pointAssociateToMap with *pose.
struct RegArgs {
  const float4 *sweep;              // the ring-ordered sweep in the sensor frame(s), LiDAR-major
  int n_sweep;                      // its size, or the bound when d_n_sweep is set
  const int *d_n_sweep;             // nullable: its size on the device (the projection count of a raw sweep)
  const int *scan_start;            // its ScanInfo starts: LiDAR l's part begins at scan_start[l * rings_per_lidar] - 5
  int rings_per_lidar, n_parts;     // n_parts LiDARs (1 without the rig merge)
  int to_base;                      // 0 none, 1 the rig's float matrices (rig, intensity = l), 2 pointAssociateToMap with ext
  const float *rig;                 // DevCtl::rig
  const double *ext;                // DevCtl::ext
  const UndistStage *undist;        // nullable: the frame's staged undistortion
  const float4 *first;              // nullable: the outlier cloud's input, the LiDARs' first points (ExtractOut::first) ...
  const int *first_ok;              // ... and their flags
  const OutlierStage *outlier;      // ... and their float matrices
  const float4 *less_flat, *less_sharp;  // in the base frame, after the undistortion and the merge; before the scan filters
  int cap_flat, cap_sharp;
  const int *n_flat, *n_sharp;      // device counts (ExtractOut::counts + 3, + 1)
  const double *pose;               // pose_wmap_curr on the device: LMState::x, or the staged initial pose of a map-gated frame
};
// Ctx::registered for a frame of n_sweep sweep points and the given feature capacities
int registered_layout(Ctx *c, int n_sweep, int cap_flat, int cap_sharp, RegOut *out);
int registered_stage(Ctx *c, const RegArgs &a, const RegOut &out);
// pipeline.cu: PinnedBlock::pose <- the initial pose of a solve
void stage_pose(Ctx *c, const double *pose7);
// solve_kernels.cu: Ctx::pose_cov <- LMState::H^-1 (partial-pivot LU), zeros when the last evaluation had no residual rows
int pose_cov_device(Ctx *c, bool pdl);
// keyframe.cu: frees the keyframe store (mloam_ctx_destroy)
void keyframes_release(Ctx *c);
// One run of points a PointCloud2 message is packed from (wire.cu k_wire_pack): points, and for the 48-byte layout cov_vec and
// cov_trace; n points, or min(n, *d_n) when the count lives on the device
struct PackSeg {
  const float4 *pts;
  const float *cov6, *trace;
  const int *d_n;
  int n;
  int cloud;  // the message it belongs to (set by the packer)
};
// keyframe.cu: the segments of source MLOAM_MSG_SURROUND (the filtered surf map, then the filtered corner map) or MLOAM_MSG_GLOBAL_MAP0 / 1
// into seg[0..]; returns their count (1 or 2).  The caller has checked that the store exists.
int keyframe_msg_segments(const Ctx *c, int source, PackSeg *seg);
// keyframe.cu: pose_keyframes_3d in id order, x / y / z the keyframe's float position and w its id.  The caller has checked that the store
// exists.
void keyframe_positions(const Ctx *c, std::vector<float4> &pos);

// comm.cu: in-place sum over ranks on the context stream (no-op without a communicator)
int comm_allreduce_doubles(Ctx *c, double *d_buf, int count);

// extract_kernels.cu
struct ExtractOut {
  float4 *sharp, *less_sharp, *flat, *less_flat;  // device buffers, capacity n each
  int *counts;                                     // device int[4]
  // nullable: the first point of each LiDAR's part of the sweep (rings l * first_rings .. (l + 1) * first_rings - 1), first_ok[l] = 0
  // when the part is empty (image_segmenter.hpp:390's laser_cloud_out.points[0], the outlier cloud of segment_cloud: 0)
  float4 *first = nullptr;
  int *first_ok = nullptr;
  int first_rings = 0;
};
int extract_device(Ctx *c, const float4 *d_cloud, int n, const int *d_scan_start, const int *d_scan_end, int n_scans,
                   ExtractOut out, float *d_curv_or_null, int *d_label_or_null);
// undistort.cu: TransformToEnd in place of the extraction's less-sharp (capacity cap_less, count out.counts[1]) and less-flat (cap_flat,
// out.counts[3]) features on c->stream, LiDAR l's with the staged pose l; d_off (nullable, the rig's per-LiDAR offsets of the two clouds,
// 2 x (n_lidars + 1)) finds a point's LiDAR, without it every point is LiDAR 0's.  One launch.  stage_undistort stages its configuration.
// parity: the half of the feature double buffer the features are in; its UndistStage is copied and read.
int undistort_stage(Ctx *c, int parity, ExtractOut out, int cap_less, int cap_flat, const int *d_off, int n_lidars);
// PinnedBlock::undist[parity] <- the poses of this call (Ctx::undist_pose7); with `ahead`, undist[parity ^ 1] <- the announced sweep's
void stage_undistort(Ctx *c, int parity, const UndistPoses *ahead);
// mloam_set_lidars / _params / _front_end / _distortion: the announced sweep's poses are withdrawn, and so are the features the
// look-ahead undistorted with them
void undist_withdraw(Ctx *c);
// extract_device's work in Ctx::extract_work for n points in n_scans rings
struct RingStage;
struct ExtractWork {
  float *curv;
  int *label;
  unsigned char *gap;
  RingStage *stage;
  int *ring_cnt;  // per-ring less-flat centroid counts
  int *status;
  float4 *less_flat;  // staged less-flat centroids
};
void extract_work_layout(Carve &cv, int n, int n_scans, ExtractWork *W);
// in place: segment l of d_pts (points [d_off[l], d_off[l + 1])) <- float 3x4 matrix l times the point, intensity kept
void stamp(Ctx *c, const char *label);  // api.cu
// Range-image projection of the LiDARs of layout L (each with a vertical_scans x horizon_scans image of its own): output LiDAR-major,
// ring-major, input order within a ring, packed; ScanInfo of L.n_lidars x vertical_scans rings (+5 / -6).  fe (nullable): removeNaN +
// calTimestamp of every LiDAR first, and the output's tail past the projected count zeroed.  Work in `work`.
int project_cloud_device(Ctx *c, const float4 *d_in, const RigLayout &L, int vertical_scans, int horizon_scans, double roi_range,
                         const FrontEnd *fe, float4 *d_out, int *d_scan_start, int *d_scan_end, int *d_n_out, DevBuf &work);
// removeNaN + calTimestamp of the LiDARs of L, compacted: d_out receives the finite points in input order with w = relative time,
// *d_n_out their count.
int front_times_device(Ctx *c, const float4 *d_in, const RigLayout &L, int time_field, float scan_period, float4 *d_out, int *d_n_out,
                       DevBuf &work);
// wire.cu: the PointCloud2 messages of message sweep sw -> the float4 raw sweep out (sw.L's offsets), one launch on c->stream
int wire_unpack_device(Ctx *c, const Sweep &sw, float4 *out);
// Host message / PCD sweep *sw: point sw->bytes into B, which grows to hold each LiDAR's bytes, and with `upload` copy them there on st.
// The PCD staging keeps room for bodies half as large again, so that a replay of other files rarely grows it (a growth re-captures the
// frame graphs).
int wire_upload(Ctx *c, DevBuf &B, Sweep *sw, bool upload, cudaStream_t st);
int pcd_upload(Ctx *c, DevBuf &B, Sweep *sw, bool upload, cudaStream_t st);
// The n ASCII PCD bodies (host bytes: staged through Ctx::pcd_in) -> their points, file after file, at out on c->stream; waits for the
// stream and returns MLOAM_E_INVALID for a refused body
int pcd_decode_device(Ctx *c, int n, const mloam_pcd_t *pcds, bool host, float4 *out);
// The checks of n ASCII PCD bodies every PCD entry point makes (MLOAM_E_INVALID), and the message of refusal bits (MLOAM_OK for none)
int pcd_check(Ctx *c, int n, const mloam_pcd_t *pcds);
int pcd_refusal(Ctx *c, unsigned bits);
// The decode of PCD sweep sw in a frame, on c->stream (also while capturing): its PcdStage copied from PinnedBlock::pcd_half[half]
// (staged by the frame), the refusal bits into the half's status word, the points to out
int pcd_decode_half(Ctx *c, const Sweep &sw, int half, float4 *out);
// What a frame does for sweep sw that only a PCD sweep needs (nothing for the other kinds).  stage: its bodies' byte sizes (and staging
// offsets) into PinnedBlock::pcd_half[half], before the frame is enqueued and before every replay — they change from file to file and the
// captured decode reads them at execution time.  land: the refusal bits of both halves into PinnedBlock::pcd_half_status, on c->stream at
// the frame's end.  refusal: after the frame, MLOAM_E_INVALID for a body the decode in half `half` refused (waits for the stream).
void pcd_frame_stage(Ctx *c, const Sweep &sw, int half);
int pcd_frame_land(Ctx *c, const Sweep &sw);
int pcd_frame_refusal(Ctx *c, const Sweep &sw, int half);
int transform_segments_device(Ctx *c, float4 *d_pts, int n, const int *d_off, int n_seg, const float *d_mat12);
// VoxelGridCovarianceMLOAM<PointIWithCov>::filter: covariance-weighted merge per voxel (cov6 + trace per point in and out)
int voxel_downsample_cov_device(Ctx *c, const float4 *d_in, const float *d_cov6, const float *d_trace, int n, const int *d_n_in, float leaf,
                                float trace_threshold, float4 *d_out, float *d_cov6_out, float *d_trace_out, int *d_n_out, DevBuf &work);
// exclusive scan of ints on the context stream (extract_kernels.cu); tmp holds ceil(n / 2048) ints
void scan_exclusive(Ctx *c, const int *d_in, int *d_out, int n, int *d_tmp, int *d_total);
// After a batched extraction over the concatenated sweeps of n_lidars LiDARs: move the less-sharp / less-flat features of LiDAR l into
// the base frame with its float 3x4 extrinsic d_ext12[l] and set intensity = l (transformCloudFeature, visualization.cpp:40-52).
// d_off: the per-LiDAR offsets lidar_offsets_device wrote for this extraction.
int merge_lidars_device(Ctx *c, ExtractOut out, int n_cap_less, int n_cap_lflat, int n_lidars, const float *d_ext12, const int *d_off);
// Right after that batched extraction (it reads the extraction's per-ring counts in Ctx::extract_work): where each LiDAR's less-sharp
// and less-flat features begin, d_off[0 .. n_lidars] and d_off[n_lidars + 1 .. 2 n_lidars + 1].  One launch.
int lidar_offsets_device(Ctx *c, int n_lidars, int rings_per_lidar, int *d_off);
// d_n_in (nullable): device-side input count (n is then the upper bound the kernels are sized for).
int voxel_downsample_device(Ctx *c, const float4 *d_in, int n, const int *d_n_in, float leaf, int intensity_last, float4 *d_out,
                            int *d_n_out, DevBuf &work);

}  // namespace mloam

struct mloam_ctx {
  mloam::Ctx c;
};
