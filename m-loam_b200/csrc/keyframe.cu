// keyframe.cu — the mapper's keyframe state machine with the keyframes kept on the device (lidar_mapper_keyframe.cpp):
//   mloam_keyframes_init   an empty store: no keyframes, empty surrounding set, empty map slots (the first frame fails the map gate, :429)
//   mloam_keyframe_save    saveKeyframe (:641-683): distance / angle test, the last frame's gated scans and outlier cloud appended device
//                          to device to a grow-only arena; a save marks the submap stale (clearCloud, :921-927, called at :1101)
//   mloam_keyframe_submap  extractSurroundingKeyFrames (:254-354): radius search over the keyframe positions, the surrounding-set
//                          bookkeeping (:274-323) with a device cache of the associated clouds (cloudUCTAssociateToMap once per entering
//                          keyframe), the keyframe-position filter (:325-338), `+=` of the chosen cached clouds (k_gather_*), the two
//                          covariance filters (:344-347) and the map build into MLOAM_MAP_SURF / MLOAM_MAP_CORNER
//   mloam_keyframe_query / mloam_keyframe_scan / mloam_keyframe_outlier   what a caller that publishes keyframes needs
//   mloam_global_map       pubGlobalMap (:780-851) / saveGlobalMap (:853-919): radius search or every keyframe, the keyframe-position
//                          filter, one batched cloudUCTAssociateToMap over every cloud of the chosen keyframes (k_uct_associate_seg,
//                          submap.cu) and the covariance filter, into buffers of its own; _read / _chosen return the result
// No point of a keyframe crosses PCIe: only poses, counts and the ids of the surrounding set do.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "ctx.h"
#include "host_util.h"
#include "uct.h"

namespace mloam {

namespace {

// Grow-only device memory outside alloc_epoch(): frame graphs never reference the store, so its growth must not make them re-capture.
struct RawBuf {
  char *p = nullptr;
  size_t cap = 0;
  void release() {
    if (p) cudaFree(p);
    p = nullptr, cap = 0;
  }
};
// Grow to at least `bytes`, keeping the first `keep` bytes (copy on grow).  The old allocation is freed after the copy has run.
cudaError_t raw_grow(RawBuf &b, size_t bytes, size_t keep, cudaStream_t st) {
  if (bytes <= b.cap) return cudaSuccess;
  // doubling with a 4 MiB floor: every growth costs a cudaMalloc and a cudaFree (which waits for the device), and the merged clouds and
  // the cache grow with the surrounding set, keyframe after keyframe
  const size_t want = std::max(2 * bytes, bytes + ((size_t)4 << 20));
  char *np = nullptr;
  cudaError_t e = cudaMalloc(&np, want);
  if (e != cudaSuccess) return e;
  if (b.p && keep) e = cudaMemcpyAsync(np, b.p, keep, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess && b.p) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    cudaFree(np);
    return e;
  }
  if (b.p) cudaFree(b.p);
  b.p = np, b.cap = want;
  return cudaSuccess;
}

// One cached entry of the surrounding set: [int count[2] | 256 B] then per cloud t (0 surf, 1 corner) points, cov_vec, cov_trace, each
// sized for the keyframe's stored (ungated) count; count[t] is the gated count the association left on the device.
struct EntLayout {
  size_t pts[2], cov6[2], trace[2], bytes;
};
__host__ __device__ inline EntLayout ent_layout(int n_surf, int n_corner) {
  EntLayout L;
  size_t o = 256;
  const int n[2] = {n_surf, n_corner};
  for (int t = 0; t < 2; t++) {
    const size_t m = (size_t)n[t];
    L.pts[t] = o, o += align256(16 * m);
    L.cov6[t] = o, o += align256(24 * m);
    L.trace[t] = o, o += align256(4 * m);
  }
  L.bytes = o;
  return L;
}

// A keyframe's record in the arena (laser_cloud_{surf,corner,outlier}_cov of saveKeyframe): per cloud t (0 surf, 1 corner, 2 outlier) its
// points, then its cov_vec, sized for the stored counts n[t]
struct KfRecord {
  float4 *pts[3];
  float *cov6[3];
  size_t bytes;
};
inline KfRecord kf_record(char *base, const int n[3]) {
  KfRecord R;
  Carve cv(base);
  for (int t = 0; t < 3; t++) R.pts[t] = cv.take<float4>(n[t]), R.cov6[t] = cv.take<float>(6 * (size_t)n[t]);
  R.bytes = cv.size + 256;
  return R;
}

struct GatherEnt {
  long long off;  // byte offset of the entry in the cache
  int n[2];       // the keyframe's stored counts (the entry's capacities)
};

// laser_cloud_{surf,corner}_from_map_cov += *surrounding_*_cloud_keyframes[j] for the position filter's output in order (:336-341):
// an exclusive scan of the chosen entries' gated sizes, appended after what the merged clouds already hold (they are only emptied by
// clearCloud).  One thread: the surrounding set holds tens to hundreds of keyframes.
__global__ void k_gather_scan(const float4 *__restrict__ chosen, const int *__restrict__ d_n_chosen, const GatherEnt *__restrict__ tab,
                              const char *__restrict__ cache, int *__restrict__ merged_n, int *__restrict__ dst) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int n = *d_n_chosen;
  int tot[2] = {merged_n[0], merged_n[1]};
  for (int i = 0; i < n; i++) {
    const int *cnt = reinterpret_cast<const int *>(cache + tab[(int)chosen[i].w].off);
    for (int t = 0; t < 2; t++) dst[2 * i + t] = tot[t], tot[t] += cnt[t];
  }
  merged_n[0] = tot[0], merged_n[1] = tot[1];
}

struct MergedOut {
  float4 *pts[2];
  float *cov6[2], *trace[2];
};
// grid (entries of the set, y, 2 clouds): block (i, ., t) copies chosen entry i's cloud t to its scanned offset
__global__ void k_gather_copy(const float4 *__restrict__ chosen, const int *__restrict__ d_n_chosen, const GatherEnt *__restrict__ tab,
                              const char *__restrict__ cache, const int *__restrict__ dst, MergedOut out) {
  const int i = blockIdx.x, t = blockIdx.z;
  if (i >= *d_n_chosen) return;
  const GatherEnt e = tab[(int)chosen[i].w];
  const char *base = cache + e.off;
  const EntLayout L = ent_layout(e.n[0], e.n[1]);
  const int n = reinterpret_cast<const int *>(base)[t];
  const float4 *p = reinterpret_cast<const float4 *>(base + L.pts[t]);
  const float *c6 = reinterpret_cast<const float *>(base + L.cov6[t]);
  const float *tr = reinterpret_cast<const float *>(base + L.trace[t]);
  const size_t d = (size_t)dst[2 * i + t];
  for (int k = blockIdx.y * blockDim.x + threadIdx.x; k < n; k += gridDim.y * blockDim.x) {
    out.pts[t][d + k] = p[k];
#pragma unroll
    for (int q = 0; q < 6; q++) out.cov6[t][(d + k) * 6 + q] = c6[(size_t)k * 6 + q];
    out.trace[t][d + k] = tr[k];
  }
}

}  // namespace

struct KeyframeStore {
  double dist_kf = 0.0, orient_kf_deg = 0.0, radius = 0.0, trace_thr = 0.0;  // DISTANCE_KEYFRAMES, ORIENTATION_KEYFRAMES, ..., TRACE_THRESHOLD_MAPPING
  float sur_kf_res = 1.f;                                                    // MAP_SUR_KF_RES
  // saveKeyframe: pose_point_prev (a PointI, float) and q_ori_prev
  float prev_pt[3] = {0.f, 0.f, 0.f};
  double prev_q[4] = {0, 0, 0, 1};
  struct Kf {
    double pose[7], cov[36];  // pose_keyframes_6d
    float pos[3];             // pose_keyframes_3d (intensity = id)
    int chunk;
    size_t off;               // in its chunk: surf points | surf cov_vec | corner points | corner cov_vec | outlier points | outlier cov_vec
    int n[3];                 // stored points: [0] surf, [1] corner, [2] outlier (0 when the frame ran without the outlier cloud)
  };
  std::vector<Kf> kfs;
  std::vector<RawBuf> chunks;  // keyframe arena; a keyframe lies in one chunk and chunks never move, so growth keeps every keyframe valid
  size_t chunk_used = 0;       // bytes used in the last chunk
  // extractSurroundingKeyFrames
  std::vector<int> sur;         // surrounding_existing_keyframes_id
  std::vector<size_t> ent_off;  // its cached clouds (surrounding_*_cloud_keyframes): byte offset in cache[cur]
  RawBuf cache[2];              // ping-pong: ids that leave the set are compacted out into the other buffer
  int cur = 0;
  size_t cache_used = 0;
  std::vector<int> chosen;      // keyframe ids the position filter chose in the last rebuild, in filter order
  int map_n[2] = {0, 0};        // laser_cloud_{surf,corner}_from_map_cov_ds sizes (0 after clearCloud)
  size_t merged_ub[2] = {0, 0}; // upper bound of laser_cloud_*_from_map_cov's device-side size
  RawBuf merged_pts[2], merged_cov6[2], merged_trace[2];  // laser_cloud_*_from_map_cov, kept until clearCloud
  RawBuf filt[2];               // laser_cloud_*_from_map_cov_ds (filt_layout)
  RawBuf ctl;                   // ints: [0..1] merged sizes, [2..3] filtered sizes, [4] position-filter count, [8..] staged counts
  RawBuf tab;                   // per rebuild: positions in | filter out | GatherEnt table | dst offsets | UctLaser of the entering keyframes
  std::vector<float4> h_pos;
  std::vector<GatherEnt> h_tab;
  std::vector<UctLaser> h_lasers;
  std::vector<float4> h_chosen;
  float cur_pt[3] = {0.f, 0.f, 0.f};  // pose_point_cur: the position the last mloam_keyframe_save call tested (:643-645)
  // the last mloam_global_map: its own work and result buffers (no frame graph references them, and the mapper's submap state is never
  // touched), sized by its input
  struct GlobalMap {
    DevBuf tab{nullptr, 0, false};        // positions in | position filter out | count | segments | keyframe poses | UctLaser blocks
    DevBuf assoc{nullptr, 0, false};      // UctBufs of the larger map input
    DevBuf merged{nullptr, 0, false};     // the associated, gated cloud of one map: points | cov_vec | trace
    DevBuf voxel{nullptr, 0, false};      // the filters' work
    DevBuf out[2] = {{nullptr, 0, false}, {nullptr, 0, false}};  // filtered map t: points | cov_vec | trace | count
    int n[2] = {0, 0};                    // filtered sizes
    const float4 *pts[2] = {nullptr, nullptr};
    const float *cov6[2] = {nullptr, nullptr};
    const float *trace[2] = {nullptr, nullptr};  // cov_trace as the filter stored it (mloam_cloud_msgs)
    std::vector<int> chosen;              // keyframe ids the position filter chose, in filter order
  } gm;
  void release() {
    for (auto &b : chunks) b.release();
    chunks.clear();
    for (int t = 0; t < 2; t++) cache[t].release(), merged_pts[t].release(), merged_cov6[t].release(), merged_trace[t].release(), filt[t].release();
    ctl.release(), tab.release();
    for (DevBuf *b : {&gm.tab, &gm.assoc, &gm.merged, &gm.voxel, &gm.out[0], &gm.out[1]}) b->release();
  }
  size_t filt_cap(int t) const { return merged_ub[t] + 16; }
  // filtered map t: points | cov_vec | cov_trace, sized for filt_cap(t) points
  struct Filt {
    float4 *pts;
    float *cov6, *trace;
    size_t bytes;
  };
  Filt filt_layout(int t) const {
    const size_t m = filt_cap(t);
    Filt F;
    Carve cv(filt[t].p);
    F.pts = cv.take<float4>(m), F.cov6 = cv.take<float>(6 * m), F.trace = cv.take<float>(m);
    F.bytes = cv.size;
    return F;
  }
};

void keyframes_release(Ctx *c) {
  if (!c->kf) return;
  c->kf->release();
  delete c->kf;
  c->kf = nullptr;
}

int keyframe_msg_segments(const Ctx *c, int source, PackSeg *seg) {
  const KeyframeStore &S = *c->kf;
  if (source == MLOAM_MSG_SURROUND) {  // laser_cloud_surf_from_map_cov_ds + laser_cloud_corner_from_map_cov_ds (:789)
    for (int t = 0; t < 2; t++) {
      const int m = S.map_n[t];
      const KeyframeStore::Filt F = m > 0 ? S.filt_layout(t) : KeyframeStore::Filt{nullptr, nullptr, nullptr, 0};
      seg[t] = PackSeg{F.pts, F.cov6, F.trace, nullptr, m, 0};
    }
    return 2;
  }
  const int m = source - MLOAM_MSG_GLOBAL_MAP0, n = S.gm.n[m];
  seg[0] = n > 0 ? PackSeg{S.gm.pts[m], S.gm.cov6[m], S.gm.trace[m], nullptr, n, 0} : PackSeg{nullptr, nullptr, nullptr, nullptr, 0, 0};
  return 1;
}

void keyframe_positions(const Ctx *c, std::vector<float4> &pos) {
  const KeyframeStore &S = *c->kf;
  pos.resize(S.kfs.size());
  for (size_t i = 0; i < S.kfs.size(); i++) pos[i] = make_float4(S.kfs[i].pos[0], S.kfs[i].pos[1], S.kfs[i].pos[2], (float)i);
}

namespace {

// saveKeyframe's test (:649-653): the float distance of the PointI positions, and Eigen's
// angularDistance(q_cur, q_prev) = 2 atan2(|(q_cur q_prev^-1).vec|, |(q_cur q_prev^-1).w|) in degrees
bool keyframe_due(const KeyframeStore &S, const double *pose7) {
  if (S.kfs.empty()) return true;
  const float cur[3] = {(float)pose7[0], (float)pose7[1], (float)pose7[2]};
  const float dx = cur[0] - S.prev_pt[0], dy = cur[1] - S.prev_pt[1], dz = cur[2] - S.prev_pt[2];
  const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
  if ((double)dist > S.dist_kf) return true;
  const double ax = pose7[3], ay = pose7[4], az = pose7[5], aw = pose7[6];
  const double bx = -S.prev_q[0], by = -S.prev_q[1], bz = -S.prev_q[2], bw = S.prev_q[3];
  const double x = aw * bx + ax * bw + ay * bz - az * by, y = aw * by + ay * bw + az * bx - ax * bz;
  const double z = aw * bz + az * bw + ax * by - ay * bx, w = aw * bw - ax * bx - ay * by - az * bz;
  const double ang = 2.0 * std::atan2(std::sqrt(x * x + y * y + z * z), std::fabs(w));
  return ang / 3.14159265358979323846 * 180.0 > S.orient_kf_deg;  // / M_PI * 180
}

// pcl::KdTreeFLANN::radiusSearch over pose_keyframes_3d around the float PointI q (L2_Simple in float): the keyframes with
// d2 < (float)(radius^2) (FLANN's RadiusResultSet), ascending (d2, id)
std::vector<std::pair<float, int>> radius_hits(const KeyframeStore &S, const float q[3], double radius) {
  const float r2 = (float)(radius * radius);
  std::vector<std::pair<float, int>> hits;
  for (int k = 0; k < (int)S.kfs.size(); k++) {
    const float dx = S.kfs[k].pos[0] - q[0], dy = S.kfs[k].pos[1] - q[1], dz = S.kfs[k].pos[2] - q[2];
    float d2 = 0.f;
    d2 += dx * dx, d2 += dy * dy, d2 += dz * dz;
    if (d2 < r2) hits.push_back({d2, k});
  }
  std::sort(hits.begin(), hits.end());
  return hits;
}

}  // namespace
}  // namespace mloam

using namespace mloam;

extern "C" {

int mloam_keyframes_init(mloam_ctx_t *h, double distance_keyframes, double orientation_keyframes_deg, double surrounding_kf_radius,
                         double map_sur_kf_res, double trace_threshold) {
  if (!h || !(distance_keyframes >= 0.0) || !(orientation_keyframes_deg >= 0.0) || !(surrounding_kf_radius > 0.0) || !(map_sur_kf_res > 0.0))
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "keyframes: the keyframe store is single-GPU only; detach the communicator");
  cudaSetDevice(c->device);
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  keyframes_release(c);
  c->kf = new KeyframeStore();
  KeyframeStore &S = *c->kf;
  S.dist_kf = distance_keyframes, S.orient_kf_deg = orientation_keyframes_deg, S.radius = surrounding_kf_radius;
  S.sur_kf_res = (float)map_sur_kf_res, S.trace_thr = trace_threshold;
  MLOAM_CUDA_OK(c, raw_grow(S.ctl, 4096, 0, c->stream));
  MLOAM_CUDA_OK(c, cudaMemsetAsync(S.ctl.p, 0, 4096, c->stream));
  c->frame_since_save = false;
  // the reference's map clouds start empty: the first frames fail the map gate (:429) until a keyframe has been saved and extracted
  int rc = map_build_device(c, MLOAM_MAP_SURF, nullptr, 0, pick_cell(c, 0.f));
  if (rc == MLOAM_OK) rc = map_build_device(c, MLOAM_MAP_CORNER, nullptr, 0, pick_cell(c, 0.f));
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}

int mloam_keyframe_save(mloam_ctx_t *h, const double *pose7, const double *cov36, int *saved) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (saved) *saved = 0;
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "keyframe_save: the keyframe store is single-GPU only; detach the communicator");
  if (!c->kf) return fail(c, MLOAM_E_STATE, "keyframe_save: call mloam_keyframes_init first");
  if (!c->frame_since_save || !c->last_scan_valid)
    return fail(c, MLOAM_E_STATE, "keyframe_save: no mloam_frame / mloam_frame_device call has run since the last save or init");
  cudaSetDevice(c->device);
  KeyframeStore &S = *c->kf;
  c->frame_since_save = false;  // one decision per frame
  const double *pose = pose7 ? pose7 : c->last_pose7;
  for (int q = 0; q < 3; q++) S.cur_pt[q] = (float)pose[q];
  if (!keyframe_due(S, pose)) return MLOAM_OK;
  KeyframeStore::Kf k;
  memcpy(k.pose, pose, sizeof(k.pose));
  if (cov36) memcpy(k.cov, cov36, sizeof(k.cov));
  else if (S.kfs.size() <= 10) memset(k.cov, 0, sizeof(k.cov));  // cov_mapping.setZero() while <= 10 keyframes (:607-608), as the solve saw it
  else memcpy(k.cov, c->pose_cov36, sizeof(k.cov));
  k.pos[0] = (float)pose[0], k.pos[1] = (float)pose[1], k.pos[2] = (float)pose[2];
  // the last frame's gated scans (laser_cloud_{surf,corner}_cov, :675-676): their device-side counts decide the copy sizes
  const Ctx::ScanRef &R = c->last_scan;
  cudaStream_t st = c->stream;
  int *hc = c->pinned->counts;
  hc[0] = R.n_surf, hc[1] = R.n_corner;
  if (R.d_n_surf) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, R.d_n_surf, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (R.d_n_corner) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc + 1, R.d_n_corner, sizeof(int), cudaMemcpyDeviceToHost, st));
  hc[2] = 0;  // laser_cloud_outlier_cov (:677): empty when the frame ran without the outlier cloud
  if (R.d_n_outlier) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc + 2, R.d_n_outlier, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  k.n[0] = std::max(0, std::min(hc[0], R.n_surf)), k.n[1] = std::max(0, std::min(hc[1], R.n_corner));
  k.n[2] = std::max(0, std::min(hc[2], MLOAM_MAX_LIDARS));
  const size_t need = kf_record(nullptr, k.n).bytes;
  if (S.chunks.empty() || S.chunk_used + need > S.chunks.back().cap) {  // a new chunk, twice the last one: O(log K) allocations
    RawBuf b;
    MLOAM_CUDA_OK(c, raw_grow(b, std::max(need, S.chunks.empty() ? (size_t)0 : 2 * S.chunks.back().cap), 0, st));
    S.chunks.push_back(b);
    S.chunk_used = 0;
  }
  k.chunk = (int)S.chunks.size() - 1, k.off = S.chunk_used;
  S.chunk_used += need;
  const KfRecord rec = kf_record(S.chunks[k.chunk].p + k.off, k.n);
  const float4 *src[3] = {R.surf, R.corner, R.outlier};
  const float *srcc[3] = {R.cov6_surf, R.cov6_corner, R.cov6_outlier};
  for (int t = 0; t < 3; t++) {
    const size_t m = (size_t)k.n[t];
    if (m) MLOAM_CUDA_OK(c, cudaMemcpyAsync(rec.pts[t], src[t], 16 * m, cudaMemcpyDeviceToDevice, st));
    if (m && srcc[t]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(rec.cov6[t], srcc[t], 24 * m, cudaMemcpyDeviceToDevice, st));
    else if (m) MLOAM_CUDA_OK(c, cudaMemsetAsync(rec.cov6[t], 0, 24 * m, st));  // with_ua = false: PointIWithCov(point, Zero) (:378-386)
  }
  S.kfs.push_back(k);
  S.prev_pt[0] = k.pos[0], S.prev_pt[1] = k.pos[1], S.prev_pt[2] = k.pos[2];
  for (int q = 0; q < 4; q++) S.prev_q[q] = pose[3 + q];
  // clearCloud (:921-927, :1101): the next mloam_keyframe_submap rebuilds
  S.map_n[0] = S.map_n[1] = 0, S.merged_ub[0] = S.merged_ub[1] = 0;
  MLOAM_CUDA_OK(c, cudaMemsetAsync(S.ctl.p, 0, 4 * sizeof(int), st));
  if (saved) *saved = 1;
  return MLOAM_OK;
}

int mloam_keyframe_submap(mloam_ctx_t *h, const double *pose_pred7, int *rebuilt, mloam_point_t *h_surf, float *h_surf_cov6, int cap_surf,
                          int *n_surf, mloam_point_t *h_corner, float *h_corner_cov6, int cap_corner, int *n_corner) {
  if (!h || !pose_pred7) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (rebuilt) *rebuilt = 0;
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "keyframe_submap: the keyframe store is single-GPU only; detach the communicator");
  if (!c->kf) return fail(c, MLOAM_E_STATE, "keyframe_submap: call mloam_keyframes_init first");
  cudaSetDevice(c->device);
  KeyframeStore &S = *c->kf;
  cudaStream_t st = c->stream;
  int rc = MLOAM_OK;
  // :256-261.  `(!a->size() == 0) && (!b->size() == 0)`: nothing to do while both filtered maps hold points
  if (!S.kfs.empty() && !(S.map_n[0] > 0 && S.map_n[1] > 0)) {
    // :263-272 radius search over pose_keyframes_3d with the float PointI of the prediction (pcl::KdTreeFLANN, L2_Simple in float):
    // d2 < radius^2 (FLANN's RadiusResultSet), ascending (d2, id)
    const float q[3] = {(float)pose_pred7[0], (float)pose_pred7[1], (float)pose_pred7[2]};
    const std::vector<std::pair<float, int>> hits = radius_hits(S, q, S.radius);
    std::vector<char> in_radius(S.kfs.size(), 0), in_set(S.kfs.size(), 0);
    for (const auto &x : hits) in_radius[x.second] = 1;
    // :274-292 drop the ids that left, survivors keep their order; :294-323 append the new ids in radius order
    std::vector<int> sur;
    std::vector<size_t> surv_off;
    for (size_t i = 0; i < S.sur.size(); i++)
      if (in_radius[S.sur[i]]) sur.push_back(S.sur[i]), surv_off.push_back(S.ent_off[i]), in_set[S.sur[i]] = 1;
    const size_t n_surv = sur.size();
    const bool compact = n_surv < S.sur.size();
    for (const auto &x : hits)
      if (!in_set[x.second]) sur.push_back(x.second), in_set[x.second] = 1;
    // the cache: survivors stay where they are unless an id left (then they are compacted into the other buffer), new ids appended
    size_t surv_bytes = 0, new_bytes = 0;
    for (size_t i = 0; i < sur.size(); i++) {
      const KeyframeStore::Kf &k = S.kfs[sur[i]];
      (i < n_surv ? surv_bytes : new_bytes) += ent_layout(k.n[0], k.n[1]).bytes;
    }
    std::vector<size_t> ent_off(sur.size());
    if (compact) {
      RawBuf &dst = S.cache[S.cur ^ 1];
      MLOAM_CUDA_OK(c, raw_grow(dst, surv_bytes + new_bytes, 0, st));
      size_t o = 0;
      for (size_t i = 0; i < n_surv; i++) {
        const KeyframeStore::Kf &k = S.kfs[sur[i]];
        const size_t b = ent_layout(k.n[0], k.n[1]).bytes;
        MLOAM_CUDA_OK(c, cudaMemcpyAsync(dst.p + o, S.cache[S.cur].p + surv_off[i], b, cudaMemcpyDeviceToDevice, st));
        ent_off[i] = o, o += b;
      }
      S.cur ^= 1, S.cache_used = o;
    } else {
      MLOAM_CUDA_OK(c, raw_grow(S.cache[S.cur], S.cache_used + new_bytes, S.cache_used, st));
      for (size_t i = 0; i < n_surv; i++) ent_off[i] = surv_off[i];
    }
    // per-rebuild device tables: positions in | filter out | GatherEnt | dst offsets | UctLaser of the entering keyframes
    const int n_set = (int)sur.size();
    const int n_lasers = c->cfg.n_parts();
    const size_t n_new = sur.size() - n_surv;
    float4 *d_pos, *d_chosen;
    GatherEnt *d_tab;
    int *d_dst;
    UctLaser *d_las;
    auto tab_layout = [&](Carve &cv) {
      const size_t m = (size_t)(n_set + 1);
      d_pos = cv.take<float4>(m), d_chosen = cv.take<float4>(m), d_tab = cv.take<GatherEnt>(m), d_dst = cv.take<int>(2 * m);
      d_las = cv.take<UctLaser>(MLOAM_MAX_LIDARS * (n_new + 1));
    };
    Carve tab_size;
    tab_layout(tab_size);
    MLOAM_CUDA_OK(c, raw_grow(S.tab, tab_size.size, 0, st));
    Carve tab_cv(S.tab.p);
    tab_layout(tab_cv);
    // :311-322 cloudUCTAssociateToMap of each entering keyframe with its pose + covariance and the context's current extrinsics and
    // covariances (mloam_set_lidars / mloam_set_uncertainty; the with_ua = false branch without uncertainty)
    S.h_lasers.clear();
    std::vector<double> pc(7 * (size_t)n_lasers), cc(36 * (size_t)n_lasers);
    const double zero36[36] = {0}, *ext7 = c->cfg.part_ext(0);  // the n_lasers extrinsics
    for (size_t i = n_surv; i < sur.size(); i++) {
      const KeyframeStore::Kf &k = S.kfs[sur[i]];
      for (int l = 0; l < n_lasers; l++)
        mloam_compound_pose_cov(k.pose, k.cov, ext7 + 7 * l, c->cfg.with_ua ? c->cfg.ua_ext_cov[l] : zero36, &pc[7 * l], &cc[36 * l]);
      std::vector<UctLaser> one;
      fill_lasers(n_lasers, ext7, pc.data(), cc.data(), one);
      S.h_lasers.insert(S.h_lasers.end(), one.begin(), one.end());
    }
    if (!S.h_lasers.empty())
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_las, S.h_lasers.data(), sizeof(UctLaser) * S.h_lasers.size(), cudaMemcpyHostToDevice, st));
    int n_max = 1;
    for (size_t i = n_surv; i < sur.size(); i++) n_max = std::max(n_max, std::max(S.kfs[sur[i]].n[0], S.kfs[sur[i]].n[1]));
    UctBufs B;
    rc = uct_bufs(c, n_max, &B);
    if (rc) return rc;
    size_t o = S.cache_used;
    for (size_t i = n_surv; i < sur.size(); i++) {
      const KeyframeStore::Kf &k = S.kfs[sur[i]];
      const EntLayout L = ent_layout(k.n[0], k.n[1]);
      ent_off[i] = o;
      char *e = S.cache[S.cur].p + o;
      MLOAM_CUDA_OK(c, cudaMemsetAsync(e, 0, 2 * sizeof(int), st));
      UctFrame f;
      memcpy(f.pose_global, k.pose, sizeof(f.pose_global)), memcpy(f.cov_meas, c->cfg.ua_cov_meas, sizeof(f.cov_meas));
      f.trace_threshold = S.trace_thr, f.with_ua = c->cfg.with_ua ? 1 : 0, f.n_lasers = n_lasers, f.scan_frame = 0;
      const KfRecord rec = kf_record(S.chunks[k.chunk].p + k.off, k.n);
      for (int t = 0; t < 2; t++) {
        rc = uct_associate_append(c, rec.pts[t], k.n[t], f, d_las + (i - n_surv) * n_lasers, B, reinterpret_cast<float4 *>(e + L.pts[t]),
                                  reinterpret_cast<float *>(e + L.cov6[t]), reinterpret_cast<float *>(e + L.trace[t]), reinterpret_cast<int *>(e) + t);
        if (rc) return rc;
      }
      o += L.bytes;
    }
    S.cache_used = o;
    S.sur = sur, S.ent_off = ent_off;
    // :325-335 VoxelGridCovarianceMLOAM<PointI> over the set's positions, intensity = position in the set, the last one per voxel
    S.h_pos.resize(n_set), S.h_tab.resize(n_set);
    for (int i = 0; i < n_set; i++) {
      const KeyframeStore::Kf &k = S.kfs[sur[i]];
      S.h_pos[i] = make_float4(k.pos[0], k.pos[1], k.pos[2], (float)i);
      S.h_tab[i].off = (long long)ent_off[i], S.h_tab[i].n[0] = k.n[0], S.h_tab[i].n[1] = k.n[1];
    }
    int *ctl = reinterpret_cast<int *>(S.ctl.p);
    if (n_set > 0) {
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_pos, S.h_pos.data(), sizeof(float4) * n_set, cudaMemcpyHostToDevice, st));
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_tab, S.h_tab.data(), sizeof(GatherEnt) * n_set, cudaMemcpyHostToDevice, st));
      rc = voxel_downsample_device(c, d_pos, n_set, nullptr, S.sur_kf_res, 1, d_chosen, ctl + 4, c->voxel_work);
      if (rc) return rc;
    } else {  // no keyframe within the radius: nothing is chosen, nothing appended (the reference's filters then see what the
              // merged clouds already hold — empty after a save — and the frame fails the map gate)
      MLOAM_CUDA_OK(c, cudaMemsetAsync(ctl + 4, 0, sizeof(int), st));
    }
    // :336-341 `+=` of the chosen cached clouds, in filter order, on the device
    size_t ub[2] = {S.merged_ub[0], S.merged_ub[1]};
    for (int i = 0; i < n_set; i++) ub[0] += (size_t)S.h_tab[i].n[0], ub[1] += (size_t)S.h_tab[i].n[1];
    if (ub[0] > 0x7fffff00ull || ub[1] > 0x7fffff00ull) return fail(c, MLOAM_E_INVALID, "keyframe_submap: more than 2^31 map points");
    MergedOut mo;
    for (int t = 0; t < 2; t++) {
      const size_t keep = S.merged_ub[t] + 16, want = ub[t] + 16;
      MLOAM_CUDA_OK(c, raw_grow(S.merged_pts[t], 16 * want, 16 * keep, st));
      MLOAM_CUDA_OK(c, raw_grow(S.merged_cov6[t], 24 * want, 24 * keep, st));
      MLOAM_CUDA_OK(c, raw_grow(S.merged_trace[t], 4 * want, 4 * keep, st));
      mo.pts[t] = reinterpret_cast<float4 *>(S.merged_pts[t].p), mo.cov6[t] = reinterpret_cast<float *>(S.merged_cov6[t].p);
      mo.trace[t] = reinterpret_cast<float *>(S.merged_trace[t].p);
      S.merged_ub[t] = ub[t];
    }
    if (n_set > 0) {  // a grid dimension of 0 is not a launch
      k_gather_scan<<<1, 32, 0, st>>>(d_chosen, ctl + 4, d_tab, S.cache[S.cur].p, ctl, d_dst);
      int ymax = 1;
      for (int i = 0; i < n_set; i++) ymax = std::max(ymax, std::max(S.h_tab[i].n[0], S.h_tab[i].n[1]));
      const int gy = std::min(16, (ymax + 1023) / 1024);
      k_gather_copy<<<dim3(n_set, gy, 2), 256, 0, st>>>(d_chosen, ctl + 4, d_tab, S.cache[S.cur].p, d_dst, mo);
      c->launches += 2;
      MLOAM_CUDA_OK(c, cudaGetLastError());
    }
    // :343-347 the two VoxelGridCovarianceMLOAM<PointIWithCov> filters (MAP_SURF_RES / MAP_CORNER_RES, TRACE_THRESHOLD_MAPPING), sized
    // by the host-side bound and reading the merged sizes from the device
    const float leaf[2] = {c->params.surf_leaf, c->params.corner_leaf};
    for (int t = 0; t < 2; t++) {
      MLOAM_CUDA_OK(c, raw_grow(S.filt[t], S.filt_layout(t).bytes, 0, st));
      if (ub[t] == 0) {
        MLOAM_CUDA_OK(c, cudaMemsetAsync(ctl + 2 + t, 0, sizeof(int), st));
        continue;
      }
      const KeyframeStore::Filt F = S.filt_layout(t);
      rc = voxel_downsample_cov_device(c, mo.pts[t], mo.cov6[t], mo.trace[t], (int)ub[t], ctl + t, leaf[t], (float)S.trace_thr, F.pts, F.cov6,
                                       F.trace, ctl + 2 + t, c->voxel_work);
      if (rc) return rc;
    }
    // the one host round trip of a rebuild: the map build is sized by the filtered counts; the chosen ids ride along
    int *hc = c->pinned->counts;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, ctl, 8 * sizeof(int), cudaMemcpyDeviceToHost, st));
    S.h_chosen.resize(n_set);
    if (n_set > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(S.h_chosen.data(), d_chosen, sizeof(float4) * n_set, cudaMemcpyDeviceToHost, st));
    MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
    S.map_n[0] = hc[2], S.map_n[1] = hc[3];
    S.chosen.clear();
    for (int i = 0; i < hc[4]; i++) S.chosen.push_back(sur[(int)S.h_chosen[i].w]);
    // kdtree_{surf,corner}_from_map->setInputCloud (:433-434)
    rc = map_build_device(c, MLOAM_MAP_SURF, reinterpret_cast<const float4 *>(S.filt[0].p), S.map_n[0], pick_cell(c, 0.f));
    if (rc == MLOAM_OK) rc = map_build_device(c, MLOAM_MAP_CORNER, reinterpret_cast<const float4 *>(S.filt[1].p), S.map_n[1], pick_cell(c, 0.f));
    if (rc) return rc;
    if (rebuilt) *rebuilt = 1;
  }
  if (n_surf) *n_surf = S.map_n[0];
  if (n_corner) *n_corner = S.map_n[1];
  mloam_point_t *hp[2] = {h_surf, h_corner};
  float *hcv[2] = {h_surf_cov6, h_corner_cov6};
  const int cap[2] = {cap_surf, cap_corner};
  bool copied = false;
  for (int t = 0; t < 2; t++) {
    const int m = S.map_n[t];
    if (!(hp[t] || hcv[t]) || m == 0) continue;
    if (m > cap[t]) return fail(c, MLOAM_E_INVALID, "keyframe_submap: output capacity too small");
    const KeyframeStore::Filt F = S.filt_layout(t);
    if (hp[t]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hp[t], F.pts, sizeof(float4) * (size_t)m, cudaMemcpyDeviceToHost, st));
    if (hcv[t]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hcv[t], F.cov6, sizeof(float) * 6 * (size_t)m, cudaMemcpyDeviceToHost, st));
    copied = true;
  }
  if (copied) MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));  // the map build itself stays queued ahead of the next frame on the stream
  return MLOAM_OK;
}

int mloam_keyframe_query(mloam_ctx_t *h, int *n_keyframes, int *h_surrounding, int cap_surrounding, int *n_surrounding, int *h_chosen,
                         int cap_chosen, int *n_chosen) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->kf) return fail(c, MLOAM_E_STATE, "keyframe_query: call mloam_keyframes_init first");
  const KeyframeStore &S = *c->kf;
  if (n_keyframes) *n_keyframes = (int)S.kfs.size();
  if (n_surrounding) *n_surrounding = (int)S.sur.size();
  if (n_chosen) *n_chosen = (int)S.chosen.size();
  if (h_surrounding) {
    if ((int)S.sur.size() > cap_surrounding) return fail(c, MLOAM_E_INVALID, "keyframe_query: surrounding capacity too small");
    std::copy(S.sur.begin(), S.sur.end(), h_surrounding);
  }
  if (h_chosen) {
    if ((int)S.chosen.size() > cap_chosen) return fail(c, MLOAM_E_INVALID, "keyframe_query: chosen capacity too small");
    std::copy(S.chosen.begin(), S.chosen.end(), h_chosen);
  }
  return MLOAM_OK;
}

int mloam_keyframe_scan(mloam_ctx_t *h, int id, double *pose7, double *cov36, mloam_point_t *h_surf, float *h_surf_cov6, int cap_surf,
                        int *n_surf, mloam_point_t *h_corner, float *h_corner_cov6, int cap_corner, int *n_corner) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->kf) return fail(c, MLOAM_E_STATE, "keyframe_scan: call mloam_keyframes_init first");
  const KeyframeStore &S = *c->kf;
  if (id < 0 || id >= (int)S.kfs.size()) return fail(c, MLOAM_E_INVALID, "keyframe_scan: no such keyframe");
  cudaSetDevice(c->device);
  const KeyframeStore::Kf &k = S.kfs[id];
  if (pose7) memcpy(pose7, k.pose, sizeof(k.pose));
  if (cov36) memcpy(cov36, k.cov, sizeof(k.cov));
  if (n_surf) *n_surf = k.n[0];
  if (n_corner) *n_corner = k.n[1];
  mloam_point_t *hp[2] = {h_surf, h_corner};
  float *hcv[2] = {h_surf_cov6, h_corner_cov6};
  const int cap[2] = {cap_surf, cap_corner};
  cudaStream_t st = c->stream;
  const KfRecord rec = kf_record(S.chunks[k.chunk].p + k.off, k.n);
  for (int t = 0; t < 2; t++) {
    const size_t m = (size_t)k.n[t];
    if ((hp[t] || hcv[t]) && k.n[t] > cap[t]) return fail(c, MLOAM_E_INVALID, "keyframe_scan: capacity too small");
    if (m && hp[t]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hp[t], rec.pts[t], 16 * m, cudaMemcpyDeviceToHost, st));
    if (m && hcv[t]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hcv[t], rec.cov6[t], 24 * m, cudaMemcpyDeviceToHost, st));
  }
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

int mloam_keyframe_outlier(mloam_ctx_t *h, int id, mloam_point_t *h_pts, float *h_cov6, int cap, int *n) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (n) *n = 0;
  if (!c->kf) return fail(c, MLOAM_E_STATE, "keyframe_outlier: call mloam_keyframes_init first");
  const KeyframeStore &S = *c->kf;
  if (id < 0 || id >= (int)S.kfs.size()) return fail(c, MLOAM_E_INVALID, "keyframe_outlier: no such keyframe");
  const KeyframeStore::Kf &k = S.kfs[id];
  const int m = k.n[2];
  if (n) *n = m;
  if (!(h_pts || h_cov6) || m == 0) return MLOAM_OK;
  if (m > cap) return fail(c, MLOAM_E_INVALID, "keyframe_outlier: capacity too small (*n holds the cloud's size)");
  cudaSetDevice(c->device);
  cudaStream_t st = c->stream;
  const KfRecord rec = kf_record(S.chunks[k.chunk].p + k.off, k.n);
  if (h_pts) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_pts, rec.pts[2], 16 * (size_t)m, cudaMemcpyDeviceToHost, st));
  if (h_cov6) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cov6, rec.cov6[2], 24 * (size_t)m, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

int mloam_global_map(mloam_ctx_t *h, int mode, const double *center7, double radius, double kf_leaf, float leaf, int *n_chosen, int *n_map0,
                     int *n_map1) {
  if (n_chosen) *n_chosen = 0;
  if (n_map0) *n_map0 = 0;
  if (n_map1) *n_map1 = 0;
  if (!h || (mode != MLOAM_GLOBAL_MAP_SURROUND && mode != MLOAM_GLOBAL_MAP_SAVE) || !(kf_leaf > 0.0) || !(leaf > 0.f) ||
      (mode == MLOAM_GLOBAL_MAP_SURROUND && !(radius > 0.0)))
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "global_map: the keyframe store is single-GPU only; detach the communicator");
  if (!c->kf) return fail(c, MLOAM_E_STATE, "global_map: call mloam_keyframes_init first");
  cudaSetDevice(c->device);
  KeyframeStore &S = *c->kf;
  KeyframeStore::GlobalMap &G = S.gm;
  // the result is committed at the end: a call that fails leaves an empty result, never a part of one
  G.n[0] = G.n[1] = 0;
  G.chosen.clear();
  std::vector<int> chosen;
  // the keyframes offered to the position filter, in order: pubGlobalMap's radius search around pose_point_cur (:804-808), or
  // saveGlobalMap's every keyframe in id order (:862-863; global_map_keyframes taken as empty before, as when the publisher never ran)
  std::vector<int> cand;
  if (mode == MLOAM_GLOBAL_MAP_SURROUND) {
    const float q[3] = {center7 ? (float)center7[0] : S.cur_pt[0], center7 ? (float)center7[1] : S.cur_pt[1], center7 ? (float)center7[2] : S.cur_pt[2]};
    for (const auto &x : radius_hits(S, q, radius)) cand.push_back(x.second);
  } else {
    for (int k = 0; k < (int)S.kfs.size(); k++) cand.push_back(k);
  }
  if (cand.empty()) return MLOAM_OK;
  cudaStream_t st = c->stream;
  const int n_cand = (int)cand.size();
  const int n_lasers = c->cfg.n_parts();
  // the position filter (down_size_filter_global_map_keyframes, VoxelGridCovarianceMLOAM<PointI>(kf_leaf), :809-810): intensity = id,
  // the last id of a voxel wins; its choice goes to the host, which lays out the association
  float4 *d_pos, *d_ds;
  int *d_cnt;
  MLOAM_CUDA_OK(c, carve(G.tab, [&](Carve &cv) {
    d_pos = cv.take<float4>(n_cand), d_ds = cv.take<float4>(n_cand + 16), d_cnt = cv.take<int>(16);
  }));
  std::vector<float4> h_pos(n_cand);
  for (int i = 0; i < n_cand; i++) {
    const KeyframeStore::Kf &k = S.kfs[cand[i]];
    h_pos[i] = make_float4(k.pos[0], k.pos[1], k.pos[2], (float)cand[i]);
  }
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_pos, h_pos.data(), sizeof(float4) * n_cand, cudaMemcpyHostToDevice, st));
  int rc = voxel_downsample_device(c, d_pos, n_cand, nullptr, (float)kf_leaf, 1, d_ds, d_cnt, G.voxel);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  std::vector<float4> h_ds(n_cand);
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_ds.data(), d_ds, sizeof(float4) * n_cand, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  const int n_ch = std::max(0, std::min(hc[0], n_cand));
  for (int i = 0; i < n_ch; i++) chosen.push_back((int)h_ds[i].w);
  // per chosen keyframe in filter order (:814-828 / :866-881): cloudUCTAssociateToMap of each cloud with the keyframe's pose and
  // covariance and the context's current extrinsics and covariances (as mloam_keyframe_submap).  pubGlobalMap appends surf, corner
  // and outlier to one map (:818-827); saveGlobalMap appends surf then outlier to the surf map and corner to the corner map
  // (:873-882).  A keyframe saved without the outlier cloud has an empty one and adds no segment.
  const int n_maps = mode == MLOAM_GLOBAL_MAP_SURROUND ? 1 : 2;
  static const int order_surround[3] = {0, 1, 2}, order_save[2][2] = {{0, 2}, {1, -1}};
  std::vector<UctSeg> segs;
  int seg_n[2] = {0, 0};
  size_t tot[2] = {0, 0};
  for (int m = 0; m < n_maps; m++)
    for (int i = 0; i < n_ch; i++) {
      const KeyframeStore::Kf &k = S.kfs[chosen[i]];
      const KfRecord rec = kf_record(S.chunks[k.chunk].p + k.off, k.n);
      const int *order = n_maps == 1 ? order_surround : order_save[m];
      const int n_order = n_maps == 1 ? 3 : 2;
      for (int j = 0; j < n_order; j++) {
        const int t = order[j];
        if (t < 0 || k.n[t] == 0) continue;
        if (tot[m] + (size_t)k.n[t] > 0x7fffff00ull) return fail(c, MLOAM_E_INVALID, "global_map: more than 2^31 map points");
        segs.push_back(UctSeg{rec.pts[t], (int)tot[m], k.n[t], i});
        tot[m] += (size_t)k.n[t], seg_n[m]++;
      }
    }
  std::vector<double> h_kpose(7 * (size_t)n_ch);
  std::vector<UctLaser> h_las;
  std::vector<double> pc(7 * (size_t)n_lasers), cc(36 * (size_t)n_lasers);
  const double zero36[36] = {0}, *ext7 = c->cfg.part_ext(0);  // the n_lasers extrinsics
  for (int i = 0; i < n_ch; i++) {
    const KeyframeStore::Kf &k = S.kfs[chosen[i]];
    memcpy(&h_kpose[7 * (size_t)i], k.pose, sizeof(k.pose));
    for (int l = 0; l < n_lasers; l++)
      mloam_compound_pose_cov(k.pose, k.cov, ext7 + 7 * l, c->cfg.with_ua ? c->cfg.ua_ext_cov[l] : zero36, &pc[7 * l], &cc[36 * l]);
    std::vector<UctLaser> one;
    fill_lasers(n_lasers, ext7, pc.data(), cc.data(), one);
    h_las.insert(h_las.end(), one.begin(), one.end());
  }
  UctSeg *d_seg;
  double *d_kpose;
  UctLaser *d_las;
  MLOAM_CUDA_OK(c, carve(G.tab, [&](Carve &cv) {
    d_pos = cv.take<float4>(n_cand), d_ds = cv.take<float4>(n_cand + 16), d_cnt = cv.take<int>(16);
    d_seg = cv.take<UctSeg>(segs.size() + 1), d_kpose = cv.take<double>(h_kpose.size() + 7), d_las = cv.take<UctLaser>(h_las.size() + 1);
  }));
  if (!segs.empty()) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_seg, segs.data(), sizeof(UctSeg) * segs.size(), cudaMemcpyHostToDevice, st));
  if (n_ch) {
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_kpose, h_kpose.data(), sizeof(double) * h_kpose.size(), cudaMemcpyHostToDevice, st));
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_las, h_las.data(), sizeof(UctLaser) * h_las.size(), cudaMemcpyHostToDevice, st));
  }
  // one batched association per map, then VoxelGridCovarianceMLOAM<PointIWithCov>(leaf, TRACE_THRESHOLD_MAPPING) (:840-843 / :894-899),
  // every buffer sized by this map's input
  const int n_max = (int)std::max(tot[0], tot[1]);
  const size_t N1 = (size_t)n_max + 16;
  UctBufs B;
  float4 *mp;
  float *mc6, *mtr;
  MLOAM_CUDA_OK(c, carve(G.assoc, [&](Carve &cv) { uct_bufs_layout(cv, n_max, &B); }));
  MLOAM_CUDA_OK(c, carve(G.merged, [&](Carve &cv) { mp = cv.take<float4>(N1), mc6 = cv.take<float>(6 * N1), mtr = cv.take<float>(N1); }));
  UctFrame f;
  memset(&f, 0, sizeof(f));
  memcpy(f.cov_meas, c->cfg.ua_cov_meas, sizeof(f.cov_meas));
  f.trace_threshold = S.trace_thr, f.with_ua = c->cfg.with_ua ? 1 : 0, f.n_lasers = n_lasers, f.scan_frame = 0;
  int *d_out_n[2] = {nullptr, nullptr};
  int seg0 = 0;
  for (int m = 0; m < n_maps; m++) {
    const size_t M1 = tot[m] + 16;
    float4 *op;
    float *oc6, *otr;
    MLOAM_CUDA_OK(c, carve(G.out[m], [&](Carve &cv) {
      op = cv.take<float4>(M1), oc6 = cv.take<float>(6 * M1), otr = cv.take<float>(M1), d_out_n[m] = cv.take<int>(16);
    }));
    G.pts[m] = op, G.cov6[m] = oc6, G.trace[m] = otr;
    if (tot[m] == 0) {
      MLOAM_CUDA_OK(c, cudaMemsetAsync(d_out_n[m], 0, sizeof(int), st));
    } else {
      rc = uct_associate_segments(c, d_seg + seg0, seg_n[m], (int)tot[m], f, d_kpose, d_las, B, mp, mc6, mtr);
      if (rc) return rc;
      rc = voxel_downsample_cov_device(c, mp, mc6, mtr, (int)tot[m], B.count, leaf, (float)S.trace_thr, op, oc6, otr, d_out_n[m], G.voxel);
      if (rc) return rc;
    }
    seg0 += seg_n[m];
  }
  for (int m = 0; m < n_maps; m++) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc + m, d_out_n[m], sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));  // also: the host tables above have been consumed
  for (int m = 0; m < n_maps; m++) G.n[m] = hc[m];
  G.chosen.swap(chosen);
  if (n_chosen) *n_chosen = (int)G.chosen.size();
  if (n_map0) *n_map0 = G.n[0];
  if (n_map1) *n_map1 = G.n[1];
  return MLOAM_OK;
}

int mloam_global_map_read(mloam_ctx_t *h, int which, mloam_point_t *h_pts, float *h_cov6, int cap, int *n) {
  if (!h || which < 0 || which > 1) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->kf) return fail(c, MLOAM_E_STATE, "global_map_read: call mloam_keyframes_init first");
  const KeyframeStore::GlobalMap &G = c->kf->gm;
  const int m = G.n[which];
  if (n) *n = m;
  if (!(h_pts || h_cov6) || m == 0) return MLOAM_OK;
  if (m > cap) return fail(c, MLOAM_E_INVALID, "global_map_read: capacity too small (*n holds the map's size)");
  cudaSetDevice(c->device);
  cudaStream_t st = c->stream;
  if (h_pts) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_pts, G.pts[which], sizeof(float4) * (size_t)m, cudaMemcpyDeviceToHost, st));
  if (h_cov6) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cov6, G.cov6[which], sizeof(float) * 6 * (size_t)m, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

int mloam_global_map_chosen(mloam_ctx_t *h, int *h_ids, int cap, int *n) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->kf) return fail(c, MLOAM_E_STATE, "global_map_chosen: call mloam_keyframes_init first");
  const std::vector<int> &ch = c->kf->gm.chosen;
  if (n) *n = (int)ch.size();
  if (!h_ids) return MLOAM_OK;
  if ((int)ch.size() > cap) return fail(c, MLOAM_E_INVALID, "global_map_chosen: capacity too small (*n holds the count)");
  std::copy(ch.begin(), ch.end(), h_ids);
  return MLOAM_OK;
}

}  // extern "C"
