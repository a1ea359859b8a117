// ctx.h — host-side context behind the C ABI (include/mloam_b200.h) and the kernel launchers.
#pragma once
#include <cuda_runtime.h>
#include <map>
#include <string>
#include <vector>

#include "../../include/mloam_b200.h"
#include "common.cuh"
#include "layout.h"

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
};

// Grow-only device buffer (cudaMalloc only when capacity is exceeded; steady-state frames allocate nothing).
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    size_t want = bytes + bytes / 4 + 256;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    alloc_epoch()++;
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

// One sweep of a frame (mloam_frame*) or announced for the next one (mloam_frame_set_next*)
struct Sweep {
  const void *key = nullptr;             // the caller's cloud pointer (host or device): the look-ahead matches on it
  const float4 *cloud = nullptr;         // the sweep on the device (a host sweep: where its copy goes)
  const int *scan_start = nullptr, *scan_end = nullptr;      // its ScanInfo on the device; none for a raw sweep (the front end makes it)
  const int *h_scan_start = nullptr, *h_scan_end = nullptr;  // a host sweep's ScanInfo in host memory
  int n = 0, n_scans = 0;
  bool host = false;                     // key is a host pointer
  bool raw = false;                      // the rig's raw sweeps with layout L: the front end runs before extraction
  RigLayout L{};
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

// The context's pinned host block (Ctx::pinned): staging of small host-to-device copies and landing of small read-backs, so that
// they are truly asynchronous.
struct PinnedBlock {
  // Read by captured copies: a frame graph copies these to the device at execution time, so every replay writes them again first
  // (pipeline.cu stage_frame_inputs).
  double pose[7];                   // lm_init_state: the initial pose of a solve
  double ext[7];                    // features_enqueue: the single sensor -> base extrinsic
  float rig[MLOAM_MAX_LIDARS][12];  // features_enqueue: the rig's float 3x4 extrinsics of the merge
  UaStage ua;                       // ua_scan_stage: the with_ua configuration
  // Written by captured copies (landing of a frame's results) and by the host-buffer entry points, one call at a time
  LMState lm;                       // LMState mirror
  int counts[192];                  // count read-backs; mloam_project_cloud: [0] count, [64..] scan starts, [128..] scan ends
  double pose_cov[36];              // H^-1 of the last solve (with_ua)
  GridHdr map_hdr[MLOAM_NUM_MAPS];  // map_build_device: the GridHdr head of each slot's last build (auto cell)
  int done;                         // LM done-flag poll of the solves with max_inner > 1
  double upload_pose[7];            // upload_pose
  double odom_x[28];                // odometry / calibration / good-feature poses (DevCtl::odom_x)
  alignas(16) unsigned char odom[4096];  // OdomState mirror (odom_kernels.cu)
  double normal_eq[30];             // mloam_normal_equations read-back
  double pose_plus[64];             // mloam_pose_plus: x | delta | V in, result at [56]
  int scan_info[2][MLOAM_MAX_RINGS];       // mloam_frame: ScanInfo of the sweep (start | end)
  int scan_info_next[2][MLOAM_MAX_RINGS];  // ... and of the announced next sweep, copied on Ctx::br_ahead
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
  double odom_x[32];                    // PinnedBlock::odom_x: 21 (odometry, good features) or 28 (calibration) doubles
  double match_pose[2][8];              // calibration: the poses its two feature groups are matched at
  double normal_eq[32];                 // mloam_normal_equations
  double pose_plus[64];                 // mloam_pose_plus
  float rig[MLOAM_MAX_LIDARS][12];      // PinnedBlock::rig
  int merge_off[2 * (MLOAM_MAX_LIDARS + 1)];  // merge_lidars_device: per-LiDAR feature offsets
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
  DevBuf scan_pts[4];             // [0] corner, [1] surf
  DevBuf feat_valid[4];           // unsigned char per query
  DevBuf feat_coeff[4];           // float[6] per query
  DevBuf feat_nn[4];              // int[n_neigh] per query (optional)
  DevBuf knn_pos[4];              // int[n_neigh] per query: neighbour positions handed from k_match_knn to k_match_fit
  DevBuf knn_changed[4];          // unsigned char per query: neighbour list differs from the previous iteration's
  DevBuf knn_anchor[4];           // float4 per query: position of its last real search + tolerated displacement
  DevBuf knn_spec;                // SpecState of the speculative scan2map schedule
  DevBuf gf_work[2];              // good-feature selection scratch per set (Jacobian rows, pool tree, mask, ...)
  DevBuf knn_heavy[4];            // 2 x unsigned char per query: "needed a real search" verdicts of the last two launches
  DevBuf knn_heavy_list;          // 3 rotating counters + 2 lists of feature indices that needed a real search (match_kernels.cu HeavyQ)
  int knn_rot = 0;                // launch ordinal inside the current solve (rotation of the heavy lists / counters)
  int knn_parity = 0;             // which half of knn_heavy the next seeded launch reads
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
  DevBuf odom_work;               // OdomState + partials of mloam_odom_solve / mloam_calib_frame
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
  };
  // Sweep look-ahead (mloam_frame_set_next*): while frame k is matched and solved, the features of sweep k+1 are extracted and
  // down-sampled on a side stream into the other half of a double buffer — the reference runs the two stages in different nodes
  // (estimator -> lidar_mapper), so they overlap there too.  `Features` describes one half.
  struct Features {
    bool valid = false;
    int parity = 0;
    Sweep sw;                   // the sweep they were extracted from
    ScanRef S{};
  };
  struct NextSweep {
    bool set = false;
    Sweep sw;                   // a host sweep's device buffers are set when its copy is enqueued (pipeline.cu stage_next_sweep)
  };
  // raw frames (mloam_set_front_end, mloam_frame_raw*): the front end runs inside features_enqueue, on the main stream and in the look-ahead
  // branch.  Its work (winner images, sort) and output (projected cloud + ScanInfo) have buffers of their own: the look-ahead reuses them
  // after the main stream's front end, while the main stream runs the with_ua stage and the solve.
  FrontEnd front{};
  bool front_set = false;
  DevBuf front_work, front_out;
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
    int launches = 0, seen = 0, s2m_ran = 0;
    ScanRef S{};
    Features prefetched_out{};     // what the frame leaves in Ctx::prefetched
  };
  std::vector<GraphEntry> graphs;
  bool smem_opt_in_gf = false;     // k_gf_select's 200 KB pool
  bool smem_opt_in[3] = {false, false, false};  // >48 KB dynamic shared memory enabled for k_voxel_small / k_ring_pick / k_ring_voxel
  long long graph_capture_failures = 0;  // frames that fell back to the stream path because their capture failed (mloam_profile_get "graph_capture_failures")
  int use_graphs = 1;
  unsigned knn_tma_min = 8;        // kNN staging: runs of >= this many points use TMA bulk copies, shorter ones 16 B loads (MLOAM_KNN_TMA_MIN)
  DevBuf knn_trace;                // MLOAM_KNN_TRACE=1: 4 words per query of the last k_match_knn launch (diagnosis, tools/knn_micro.py)
  bool knn_trace_on = false;
  // MLOAM_STAMP=1 (diagnosis, tools/stamp_frame.py): one-thread kernels that write %globaltimer between the stages of a frame, so that
  // the stage times of a GRAPH REPLAY can be read (the event scopes of mloam_profile_enable force the stream path and add launch gaps)
  bool stamp_on = false;
  DevBuf stamps;
  int stamp_n = 0;
  std::vector<std::string> stamp_labels;
  int knn_min_blocks = 2;          // k_match_knn variant: resident CTAs per SM it is compiled for (MLOAM_KNN_MB = 2 | 3 | 4); 2 is fastest on the H100
  int use_seeds = 1;               // seed the kNN of re-association iterations > 0 with the previous neighbour lists
  int fuse_iter = 1;               // scan2map: fit inside the first evaluation + both evaluations of an LM iteration in ONE launch
                                   // (grid barrier between them); MLOAM_FUSE_ITER=0 restores the three launches
  int lm_tail_serial = 0;          // the LM step on one thread of the tail block (MLOAM_LM_TAIL=serial) instead of one warp; bit-identical
  bool lidar_merge = false;        // mloam_set_lidars was given extrinsics: features go through the rig merge (also for one LiDAR)
  int n_lidars = 1;                // LiDARs batched into one frame of this context (mloam_set_lidars)
  double lidar_ext[MLOAM_MAX_LIDARS][7];  // their sensor -> base extrinsics
  bool has_ext = false;            // sensor -> base extrinsic applied to extracted features (frame path)
  double ext[7] = {0, 0, 0, 0, 0, 0, 1};
  void *nccl_comm = nullptr;
  int nranks = 1, rank = 0;
  // peer-memory exchange of the packed normal equations (comm.cu, solve_kernels.cu lm_tail): every rank's exchange
  // buffer is mapped into every other rank through CUDA IPC; p2p_on replaces the NCCL all-reduce + two extra launches
  // by stores / polls over NVLink inside the k_linearize tail
  void *p2p_local = nullptr;
  void *p2p_peer[MLOAM_P2P_MAX_RANKS] = {nullptr};
  void *p2p_view = nullptr;        // device copy of the P2PView the kernels read
  bool p2p_on = false;
  // uncertainty-aware mapping in the frame path (mloam_set_uncertainty): the per-point uncertainty + trace gate of
  // downsampleCurrentScan (lidar_mapper_keyframe.cpp:356-421) between the scan filters and the solve, and the pose covariance
  // H^-1 at the returned pose (:600-610).  The covariances reach the device through the pinned block (PinnedBlock::ua), so a
  // captured frame replays with new values.
  int with_ua = 0;
  double ua_ext_cov[MLOAM_MAX_LIDARS][36];  // per LiDAR: pose_ext[l].cov_, row-major [translation | rotation]
  double ua_cov_meas[9];                    // COV_MEASUREMENT
  double ua_trace_threshold = 0.0;          // TRACE_THRESHOLD_MAPPING
  DevBuf ua_scan;                  // gated scans of the last with_ua frame (points, cov6, sqrt_info, counts) + its staged configuration
  DevBuf pose_cov;                 // 36 doubles: H^-1 of the last solve (k_pose_cov), copied back with LMState
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
// buf_base: which pair of the context's per-set buffers (knn_pos / knn_anchor / ...) the jobs use: 0 (sets 0, 1) or 2 (sets 2, 3)
// defer (nullable): skip the fit launch and write the fit into *defer for the caller's next linearize_device(lm_mode 1) (LinOpts::fit);
// defer->K == 0 when the fit was launched here (a job wants neighbour indices) or nothing was matched.  nullptr: fit now.
// d_sel (speculative schedule, with defer): double-buffered lists, read half *d_sel and write the other (SpecState::sel)
int match_pair_device(Ctx *c, const MatchJob *jobs, int n_jobs, const double *d_pose7, const MatchCfg &cfg, int buf_base = 0,
                      PendingFit *defer = nullptr, const int *d_sel = nullptr);

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
int eval_candidate_device(Ctx *c, const FeatSet *sets, int n_sets, double sqrt_info, double huber_a, double eig_thre);
// min_corr: minimum matched features for a Solve (tracker: 10); spec (nullable): also start SpecState::xc at the initial pose
int lm_init_state(Ctx *c, const double *pose7_host, int max_inner, int min_corr, SpecState *spec = nullptr);
void eig_report_host(const double *H36, double *w6);  // ascending eigenvalues of a symmetric 6x6 (host side)
int factor_evaluate_device(Ctx *c, int kind, int n, const double *d_points, const double *d_coeffs, const double *d_sqrt_info,
                           const double *d_params, double *d_res, double *d_jac);

// in place: p <- T * p for the first min(n, *d_n) points (pointAssociateToMap, utility.h:103-117); d_pose7 on device
int transform_points_device(Ctx *c, float4 *d_pts, int n, const int *d_n, const double *d_pose7);

// gf_kernels.cu: good-feature selection of one matched feature set on the device (goodFeatureMatching inside
// scan2MapOptimization): Jacobian rows + selection, result as a 0/1 mask over the features (set index t: 0 corner, 1 surf)
int gf_select_set_device(Ctx *c, int t, const FeatSet &fs, const double *d_pose7, double default_sinfo, int method, double gf_ratio,
                         unsigned long long seed, unsigned char **d_mask_out);

// uct_kernels.cu: per-point sqrt_info from PointIWithCov::cov_vec (float[6] per point)
int sqrt_info_device(Ctx *c, const float *d_cov6, int n, double *d_sinfo);
// submap.cu: the with_ua stage of a frame (downsampleCurrentScan, lidar_mapper_keyframe.cpp:356-421) on c->stream.  The scans of *S
// (device counts) -> per point ext^-1 -> evalPointUncertainty under pose_ext -> trace gate -> stable compaction into Ctx::ua_scan with
// cov6 and sqrt_info; *S then points at the gated scans.  ua_stage_host writes the staged configuration (PinnedBlock::ua).
int ua_scan_stage(Ctx *c, Ctx::ScanRef *S);
void ua_stage_host(Ctx *c);
// pipeline.cu: writers of the pinned fields a captured frame graph reads (PinnedBlock), shared by the enqueue and the replay paths
void stage_pose(Ctx *c, const double *pose7);
void stage_ext(Ctx *c);
void stage_rig(Ctx *c);
// solve_kernels.cu: Ctx::pose_cov <- LMState::H^-1 (partial-pivot LU), zeros when the last evaluation had no residual rows
int pose_cov_device(Ctx *c);
// keyframe.cu: frees the keyframe store (mloam_ctx_destroy)
void keyframes_release(Ctx *c);

// comm.cu: in-place sum over ranks on the context stream (no-op without a communicator)
int comm_allreduce_doubles(Ctx *c, double *d_buf, int count);

// extract_kernels.cu
struct ExtractOut {
  float4 *sharp, *less_sharp, *flat, *less_flat;  // device buffers, capacity n each
  int *counts;                                     // device int[4]
};
int extract_device(Ctx *c, const float4 *d_cloud, int n, const int *d_scan_start, const int *d_scan_end, int n_scans,
                   ExtractOut out, float *d_curv_or_null, int *d_label_or_null);
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
int transform_segments_device(Ctx *c, float4 *d_pts, int n, const int *d_off, int n_seg, const float *d_mat12);
// VoxelGridCovarianceMLOAM<PointIWithCov>::filter: covariance-weighted merge per voxel (cov6 + trace per point in and out)
int voxel_downsample_cov_device(Ctx *c, const float4 *d_in, const float *d_cov6, const float *d_trace, int n, const int *d_n_in, float leaf,
                                float trace_threshold, float4 *d_out, float *d_cov6_out, float *d_trace_out, int *d_n_out, DevBuf &work);
// exclusive scan of ints on the context stream (extract_kernels.cu); tmp holds ceil(n / 2048) ints
void scan_exclusive(Ctx *c, const int *d_in, int *d_out, int n, int *d_tmp, int *d_total);
// After a batched extraction over the concatenated sweeps of n_lidars LiDARs: move the less-sharp / less-flat features of LiDAR l into
// the base frame with its float 3x4 extrinsic d_ext12[l] and set intensity = l (transformCloudFeature, visualization.cpp:40-52).
// d_off: scratch for 2 x (n_lidars + 1) ints.
int merge_lidars_device(Ctx *c, ExtractOut out, int n_cap_less, int n_cap_lflat, int n_lidars, int rings_per_lidar, const float *d_ext12,
                        int *d_off);
// d_n_in (nullable): device-side input count (n is then the upper bound the kernels are sized for).
int voxel_downsample_device(Ctx *c, const float4 *d_in, int n, const int *d_n_in, float leaf, int intensity_last, float4 *d_out,
                            int *d_n_out, DevBuf &work);

}  // namespace mloam

struct mloam_ctx {
  mloam::Ctx c;
};
