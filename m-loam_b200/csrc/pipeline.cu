// pipeline.cu — the orchestrators of the hot path as kernel sequences on the context stream:
//   scan2MapOptimization  (lidar_mapper_keyframe.cpp:423-639, gf_method wo_gf)
//   the per-sweep frame   (extractCloud -> downsampleCurrentScan -> scan2MapOptimization)
// plus the host-buffer entry points of extraction and the voxel filters.
//
// Feature counts produced on the device (extraction, voxel filters) are consumed on the device: kernels are
// sized for the host-known upper bound and read the true count from HBM, so a frame with max_inner == 1 runs
// without a single host round trip until the final pose read-back.
#include <cstdio>
#include <cstring>

#include "ctx.h"
#include "host_util.h"

using namespace mloam;

namespace {

typedef Ctx::ScanRef ScanRef;

// Run body on branch b — forked from c->stream, which is b's stream meanwhile — and record b's join; or run it on c->stream when the
// branch must not fork.  The caller waits on b.join where it needs the branch's results.
template <typename Body>
int on_branch(Ctx *c, const Branch &b, bool fork, Body &&body) {
  if (!fork) return body();
  MLOAM_CUDA_OK(c, cudaEventRecord(b.fork, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamWaitEvent(b.stream, b.fork, 0));
  cudaStream_t main_stream = c->stream;
  c->stream = b.stream;
  const int rc = body();
  c->stream = main_stream;
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaEventRecord(b.join, b.stream));
  return MLOAM_OK;
}

// Enqueue the whole solve on the context stream (no host synchronisation when max_inner == 1, so the sequence can be
// captured into a CUDA graph); scan2map_finish() waits and unpacks.  *ran: the map-size gate passed and the solve is enqueued.
// want_cov: also H^-1 at the returned pose (with_ua frame, mloam_scan2map_ua).
int scan2map_enqueue(Ctx *c, const ScanRef &S, const double *pose_init7, bool want_cov, int *ran) {
  const mloam_params_t &P = c->params;
  *ran = 0;
  const MapStorage &MS = c->maps[MLOAM_MAP_SURF], &MC = c->maps[MLOAM_MAP_CORNER];
  if (!MS.built || !MC.built) return fail(c, MLOAM_E_STATE, "scan2map: build MLOAM_MAP_SURF and MLOAM_MAP_CORNER first");
  if (!((MS.m > 50) && (MC.m > 10))) return MLOAM_OK;  // lidar_mapper_keyframe.cpp:429 ("Map surf num is not enough")
  *ran = 1;
  // Collective participation: the gate above depends on the replicated maps only, so every rank takes the same branch; from here
  // on every rank enqueues the same number of LM evaluations (max_outer x (1 + max_inner) with max_inner == 1; with max_inner > 1
  // the done flag all ranks poll is the identical, summed state).  Per-rank solves (tracker, odometry) are never collective.
  LinOpts first{P.eig_thre}, iter{P.eig_thre};  // the evaluation at x that begins a Solve, and the LM iterations
  first.collective = iter.collective = true;
  first.want_eig = 0;
  int rc = reserve_feat(c, 0, S.n_corner);
  if (rc) return rc;
  rc = reserve_feat(c, 1, S.n_surf);
  if (rc) return rc;
  // Speculative re-association (one LM iteration per GN iteration, no good-feature selection, one GPU): GN iteration i + 1's
  // matcher needs only the pose it searches at, which is the candidate xc_i whenever iteration i's step is taken.  So it starts
  // as soon as the evaluation at x_i has produced xc_i, next to the evaluation at xc_i that decides the step; the evaluation at
  // x_{i+1} then takes its lists when x_{i+1} == xc_i, or keeps iteration i's lists and fit (SpecState).
  const bool spec = c->fuse_iter && P.max_inner == 1 && P.gf_method == 0 && !c->nccl_comm;
  SpecState *d_spec = nullptr;
  if (spec) {
    MLOAM_CUDA_OK(c, c->knn_spec.reserve(sizeof(SpecState)));
    d_spec = c->knn_spec.as<SpecState>();
  }
  rc = lm_init_state(c, pose_init7, P.max_inner, 0, d_spec);
  if (rc) return rc;
  LMState *st = c->lm_state.as<LMState>();
  const double *d_pose = spec ? d_spec->xc : st->x;  // where the matcher searches
  const double sinfo = map_sqrt_info(P.cov_trace);
  const MatchCfg cfg = match_cfg(c);
  int *h_done = &c->pinned->done;
  const int nc_use = P.point_edge_factor ? S.n_corner : 0, ns_use = P.point_plane_factor ? S.n_surf : 0;
  FeatSet sets[2] = {
      FeatSet{S.corner, c->feat_valid[0].as<unsigned char>(), c->feat_coeff[0].as<float>(), nc_use, 0, S.d_n_corner, S.sinfo_corner},
      FeatSet{S.surf, c->feat_valid[1].as<unsigned char>(), c->feat_coeff[1].as<float>(), ns_use, 1, S.d_n_surf, S.sinfo_surf}};
  // without good-feature selection nothing reads the fit before the solve: its launch folds into the next evaluation at x, which
  // with the speculative schedule is the next GN iteration's
  PendingFit pending;
  const bool defer_fit = c->fuse_iter && P.gf_method == 0;
  first.spec = d_spec, first.fit = &pending;
  // :503-532  match corner then surf at pose_wmap_curr (wo_gf: every feature)
  auto match = [&](int outer) {
    // From the second iteration on the same features meet the same maps at a slightly moved pose: the previous
    // neighbour lists seed the search (exact, see knn.cuh) and unchanged lists keep their line / plane fit.
    const int seeded = (outer > 0 && c->use_seeds) ? 1 : 0;
    MatchJob jobs[2] = {
        MatchJob{MLOAM_MAP_CORNER, 'c', S.corner, nc_use, S.d_n_corner, c->feat_valid[0].as<unsigned char>(),
                 c->feat_coeff[0].as<float>(), nullptr, seeded},
        MatchJob{MLOAM_MAP_SURF, 's', S.surf, ns_use, S.d_n_surf, c->feat_valid[1].as<unsigned char>(),
                 c->feat_coeff[1].as<float>(), nullptr, seeded}};
    return match_pair_device(c, jobs, 2, d_pose, cfg, 0, defer_fit ? &pending : nullptr, spec ? &d_spec->sel : nullptr);
  };
  for (int outer = 0; outer < P.max_outer; outer++) {
    if (!spec || outer == 0) {  // speculative: the previous iteration enqueued this one's matcher
      rc = match(outer);
      if (rc) return rc;
      stamp(c, "match");
    }
    // goodFeatureMatching (:503-532 with FLAGS_gf_method != wo_gf): select gf_ratio of the features per set, on the device;
    // the solve below only sees the selected ones.  Corner first, then surf, as in the reference.
    sets[0].mask = sets[1].mask = nullptr;
    if (P.gf_method != 0) {
      unsigned char *mask[2] = {nullptr, nullptr};
      auto select = [&](int t) {
        if (sets[t].n <= 0) return MLOAM_OK;
        return gf_select_set_device(c, t, sets[t], d_pose, sinfo, P.gf_method, (double)P.gf_ratio,
                                    (unsigned long long)P.gf_seed + 2ull * (unsigned long long)outer + (unsigned long long)t, &mask[t]);
      };
      // the two selections are independent single-CTA chains: corner on the side stream next to surf (also inside a captured graph)
      const bool fork_gf = !c->prof_on && sets[0].n > 0 && sets[1].n > 0;
      rc = on_branch(c, c->br_scan, fork_gf, [&] { return select(0); });
      if (rc == MLOAM_OK) rc = select(1);
      if (rc) return rc;
      if (fork_gf) MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, c->br_scan.join, 0));
      sets[0].mask = mask[0], sets[1].mask = mask[1];
    }
    // :537-582 residual blocks + Evaluate -> J^T J -> evalDegenracy, and iteration 0 of ceres::Solve.  The device
    // only needs the degeneracy decision; scan2map_finish fills in the eigenvalue report of the last iteration.
    if (P.gf_method != 0) stamp(c, "gf");
    const bool speculate = spec && outer + 1 < P.max_outer;  // the last iteration has no next matcher to start early
    // the one LM iteration's second evaluation rides in the same launch, unless it goes next to the speculative matcher
    first.two_pass = c->fuse_iter && P.max_inner == 1 && !speculate;
    first.spec_publish = speculate;
    bool second_done = false;
    rc = linearize_device(c, sets, 2, sinfo, P.huber_a, nullptr, 1, 1, nullptr, first, &second_done);
    if (rc) return rc;
    stamp(c, second_done ? "linearize x2" : "linearize");
    if (speculate) {
      // fork: {matcher of iteration outer + 1 at the published candidate} || {evaluation at the candidate + acceptance}.  The
      // branches share only read-only inputs: the matcher writes the spare half of the lists, the changed and heavy flags; the
      // evaluation writes LMState and the partials.  With stage profiling on they stay serial, like the other forks.
      const bool fork = !c->prof_on;
      rc = on_branch(c, c->br_scan, fork, [&] { return match(outer + 1); });
      if (rc) return rc;
      rc = eval_candidate_device(c, sets, 2, sinfo, P.huber_a, P.eig_thre);
      if (rc) return rc;
      if (fork) MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, c->br_scan.join, 0));
      stamp(c, "match || candidate");
      continue;
    }
    // :586-596 ceres::Solve, at most max_inner LM iterations; the device raises `done`
    for (int it = 0; it < P.max_inner && !second_done; it++) {
      rc = linearize_device(c, sets, 2, sinfo, P.huber_a, nullptr, 2, 2, nullptr, iter);
      if (rc) return rc;
      stamp(c, "linearize (candidate)");
      if (P.max_inner > 1) {
        MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_done, &st->done, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
        if (*h_done) break;
      }
    }
  }
  LMState *hs = &c->pinned->lm;
  int *h_cnt = c->pinned->counts;
  if (want_cov) {  // with_ua: cov_mapping = H^-1 at the returned pose (:600-610), one more tiny launch inside the frame
    rc = pose_cov_device(c);
    if (rc) return rc;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->pinned->pose_cov, c->pose_cov.p, 36 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    stamp(c, "pose covariance");
  }
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hs, st, sizeof(LMState), cudaMemcpyDeviceToHost, c->stream));
  if (S.d_n_surf) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cnt, S.d_n_surf, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  if (S.d_n_corner) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cnt + 1, S.d_n_corner, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  return MLOAM_OK;
}

// ran: the gate passed (scan2map_enqueue's *ran); want_cov as given to scan2map_enqueue
int scan2map_finish(Ctx *c, const ScanRef &S, const double *pose_init7, bool want_cov, int ran, double *pose_out7, mloam_solve_stats_t *stats) {
  if (stats) memset(stats, 0, sizeof(*stats));
  for (int k = 0; k < 7; k++) pose_out7[k] = pose_init7[k];
  memset(c->pose_cov36, 0, sizeof(c->pose_cov36));  // pose_wmap_curr.cov_: zero without with_ua (:621) and for a map-gated frame (:637)
  if (!ran) return MLOAM_OK;
  const LMState *hs = &c->pinned->lm;
  int *h_cnt = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  if (!S.d_n_surf) h_cnt[0] = S.n_surf;
  if (!S.d_n_corner) h_cnt[1] = S.n_corner;
  for (int k = 0; k < 7; k++) pose_out7[k] = hs->x[k];
  if (want_cov && hs->termination != 8 && hs->termination != 9) memcpy(c->pose_cov36, c->pinned->pose_cov, sizeof(c->pose_cov36));
  if (hs->termination == 9) {  // the peer-memory exchange timed out or the ranks lost lock-step: the summed state is not trustworthy
    for (int k = 0; k < 7; k++) pose_out7[k] = pose_init7[k];
    if (stats) stats->ran = 1, stats->termination = 9;
    return fail(c, MLOAM_E_NCCL, "scan2map: peer-memory exchange failed (a rank did not arrive or the ranks lost lock-step); "
                                  "call mloam_comm_p2p_reset on every rank behind a barrier");
  }
  if (hs->termination == 8) {  // k_linearize's grid barrier gave up: a block of the grid never became resident within ~2 s
    for (int k = 0; k < 7; k++) pose_out7[k] = pose_init7[k];
    if (stats) stats->ran = 1, stats->termination = 8;
    return fail(c, MLOAM_E_STATE, "scan2map: the two-evaluation launch timed out at its grid barrier (GPU shared with a kernel that never "
                                   "yields?); set MLOAM_FUSE_ITER=0 to use one launch per evaluation");
  }
  if (c->prof_on) {  // device-side cycle counters of the fused LM tail, reported next to the event-timed stages
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, c->device);
    if (khz > 0) {
      c->prof["lm_tail_reduce"].ms += (double)hs->dbg_cycles[0] / khz, c->prof["lm_tail_reduce"].launches += hs->dbg_cycles[2];
      c->prof["lm_tail_advance"].ms += (double)hs->dbg_cycles[1] / khz, c->prof["lm_tail_advance"].launches += hs->dbg_cycles[2];
    }
  }
  if (stats) {
    stats->ran = 1;
    stats->n_corner = hs->n_valid[0], stats->n_surf = hs->n_valid[1];
    stats->lm_iterations = hs->total_iterations;
    stats->degenerate = hs->is_degenerate;
    stats->termination = hs->termination;
    stats->final_cost = hs->cost;
    memcpy(stats->eig, hs->eig, sizeof(stats->eig));
    memcpy(stats->H, hs->H0, sizeof(stats->H));
    // evalDegenracy's eigenvalues (lidar_mapper_keyframe.cpp:1172-1204): the device decides degeneracy with a
    // Cholesky test of H - thre*I and only runs the eigen-solver when that fails; the report of a healthy Solve is
    // computed here from the same H.
    if (!hs->is_degenerate && !hs->skipped && hs->rows > 0 && c->params.eig_thre > 0.0) eig_report_host(hs->H0, stats->eig);
    stats->n_surf_in = h_cnt[0], stats->n_corner_in = h_cnt[1];
  }
  return MLOAM_OK;
}

int scan2map_run(Ctx *c, const ScanRef &S, const double *pose_init7, bool want_cov, double *pose_out7, mloam_solve_stats_t *stats) {
  int ran = 0;
  int rc = scan2map_enqueue(c, S, pose_init7, want_cov, &ran);
  if (rc) return rc;
  return scan2map_finish(c, S, pose_init7, want_cov, ran, pose_out7, stats);
}

// Device buffers of one frame: feature sets of extractCloud + the down-sampled scans fed to matching.
struct FrameBufs {
  ExtractOut ex;
  float4 *corner_ds, *surf_ds;
  int *n_corner_ds, *n_surf_ds;  // device counts
};
int frame_bufs(Ctx *c, int n, FrameBufs *F, int parity = 0) {
  const size_t N1 = (size_t)n + 16;
  MLOAM_CUDA_OK(c, carve(parity ? c->frame_alt : c->frame_main, [&](Carve &cv) {
    F->ex.sharp = cv.take<float4>(N1), F->ex.less_sharp = cv.take<float4>(N1), F->ex.flat = cv.take<float4>(N1);
    F->ex.less_flat = cv.take<float4>(N1), F->corner_ds = cv.take<float4>(N1), F->surf_ds = cv.take<float4>(N1);
    F->ex.counts = cv.take<int>(16);  // [0..3]
  }));
  F->n_corner_ds = F->ex.counts + 4, F->n_surf_ds = F->ex.counts + 5;
  return MLOAM_OK;
}

// A device sweep + its ScanInfo in one buffer (mloam_frame, the announced next sweep, mloam_extract_features)
struct SweepIn {
  float4 *cloud;
  int *scan_start, *scan_end;
};
int sweep_bufs(Ctx *c, DevBuf &B, int n, int n_scans, SweepIn *S) {
  MLOAM_CUDA_OK(c, carve(B, [&](Carve &cv) {
    S->cloud = cv.take<float4>(n), S->scan_start = cv.take<int>(2 * (size_t)n_scans);
  }));
  S->scan_end = S->scan_start + n_scans;
  return MLOAM_OK;
}

}  // namespace

// Writers of the pinned fields a captured frame graph copies to the device at execution time (PinnedBlock): the enqueue path calls them
// where it stages each field, stage_frame_inputs before every replay.
void mloam::stage_pose(Ctx *c, const double *pose7) { memcpy(c->pinned->pose, pose7, sizeof(c->pinned->pose)); }
void mloam::stage_ext(Ctx *c) { memcpy(c->pinned->ext, c->ext, sizeof(c->pinned->ext)); }
void mloam::stage_rig(Ctx *c) {
  for (int l = 0; l < c->n_lidars; l++) {
    const double *e = c->lidar_ext[l];
    const M33 R = qmat(qnormalized(Q4{e[3], e[4], e[5], e[6]}));  // Pose(q, t): q normalised, T_ = [R | t] (pose.cpp:34-41), cast<float>
    for (int r = 0; r < 3; r++) {
      for (int k = 0; k < 3; k++) c->pinned->rig[l][4 * r + k] = (float)R.m[3 * r + k];
      c->pinned->rig[l][4 * r + 3] = (float)e[r];
    }
  }
}

namespace {

bool rig_merge(const Ctx *c) { return c->n_lidars > 1 || c->lidar_merge; }

void stage_frame_inputs(Ctx *c, const double *pose7) {
  stage_pose(c, pose7);
  if (rig_merge(c)) stage_rig(c);
  else if (c->has_ext) stage_ext(c);
  if (c->with_ua) ua_stage_host(c);
}

// Whether the look-ahead of the previous frame made the features of sw: same caller pointer and sizes; a raw sweep's features are taken by
// a raw frame with the same per-LiDAR counts only, a ring-ordered sweep's by a ring-ordered frame, and a host frame takes a host announcement
bool frame_has_prefetched(const Ctx *c, const Sweep &sw) {
  const Ctx::Features &f = c->prefetched;
  const bool same_kind = sw.raw ? (f.sw.raw && std::memcmp(&f.sw.L, &sw.L, sizeof(RigLayout)) == 0) : !f.sw.raw;
  return f.valid && c->use_lookahead && !c->prof_on && f.sw.key == sw.key && f.sw.n == sw.n && f.sw.n_scans == sw.n_scans && same_kind &&
         (f.sw.host || !sw.host);
}

// extractCloud + (multi-LiDAR merge | base-frame transform) + downsampleCurrentScan of sweep sw on c->stream, into half `parity` of the
// feature double buffer; the corner filter forks onto branch `side`.  A raw sweep goes through the front end (removeNaN + calTimestamp +
// projection, Ctx::front) first, which makes the ring-ordered sweep and its ScanInfo on the device; extraction takes them with the raw
// size n as capacity (no count comes back to the host).
int features_enqueue(Ctx *c, const Sweep &sw, int parity, const Branch &side, ScanRef *S_out) {
  const mloam_params_t &P = c->params;
  const int n = sw.n, n_scans = sw.n_scans;
  FrameBufs F;
  int rc = frame_bufs(c, n, &F, parity);
  if (rc) return rc;
  const float4 *d_cloud = sw.cloud;
  const int *d_scan_start = sw.scan_start, *d_scan_end = sw.scan_end;
  if (sw.raw) {
    const FrontEnd &fe = c->front;
    float4 *proj;
    int *ss, *n_proj;
    MLOAM_CUDA_OK(c, carve(c->front_out, [&](Carve &cv) {
      proj = cv.take<float4>((size_t)n + 1), ss = cv.take<int>(2 * (size_t)n_scans), n_proj = cv.take<int>(4);
    }));
    rc = project_cloud_device(c, d_cloud, sw.L, fe.vertical_scans, fe.horizon_scans, fe.roi_range, &fe, proj, ss, ss + n_scans, n_proj,
                              c->front_work);
    if (rc) return rc;
    stamp(c, "front end");
    d_cloud = proj, d_scan_start = ss, d_scan_end = ss + n_scans;
  }
  rc = extract_device(c, d_cloud, n, d_scan_start, d_scan_end, n_scans, F.ex, nullptr, nullptr);
  if (rc) return rc;
  stamp(c, "extract");
  const int less_cap = n < 120 * n_scans ? n : 120 * n_scans;  // <= 20 less-sharp picks x 6 sectors per ring
  DevCtl *ctl = c->ctl.as<DevCtl>();
  if (rig_merge(c)) {
    // batched sweeps of several LiDARs: features of LiDAR l go to the base frame with its extrinsic, intensity = l
    // (transformCloudFeature, visualization.cpp:40-52), LiDAR after LiDAR as pubPointCloud's `+=` (:93-104)
    if (n_scans % c->n_lidars != 0) return fail(c, MLOAM_E_INVALID, "frame: n_scans must be n_lidars x rings per LiDAR");
    stage_rig(c);
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(ctl->rig, c->pinned->rig, sizeof(float) * 12 * c->n_lidars, cudaMemcpyHostToDevice, c->stream));
    rc = merge_lidars_device(c, F.ex, less_cap, n, c->n_lidars, n_scans / c->n_lidars, &ctl->rig[0][0], ctl->merge_off);
    if (rc) return rc;
  } else if (c->has_ext) {  // features are handed to the mapper in the base frame
    stage_ext(c);
    double *d_ext = ctl->ext;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_ext, c->pinned->ext, 7 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    rc = transform_points_device(c, F.ex.less_sharp, less_cap, F.ex.counts + 1, d_ext);
    if (rc) return rc;
    rc = transform_points_device(c, F.ex.less_flat, n, F.ex.counts + 3, d_ext);
    if (rc) return rc;
  }
  // downsampleCurrentScan, lidar_mapper_keyframe.cpp:356-364 (VoxelGridCovarianceMLOAM<PointI>: xyz mean, last intensity)
  // The two filters are independent chains of small kernels: the corner one runs on a second side stream next to the
  // surf one (own work buffer), also inside a captured graph; with stage profiling on they stay serial.
  const bool fork_voxel = !c->prof_on;
  rc = on_branch(c, side, fork_voxel, [&] {
    return voxel_downsample_device(c, F.ex.less_sharp, less_cap, F.ex.counts + 1, P.corner_leaf, 1, F.corner_ds, F.n_corner_ds, c->voxel_corner);
  });
  if (rc) return rc;
  rc = voxel_downsample_device(c, F.ex.less_flat, n, F.ex.counts + 3, P.surf_leaf, 1, F.surf_ds, F.n_surf_ds, c->voxel_surf);
  if (rc) return rc;
  if (fork_voxel) MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, side.join, 0));
  stamp(c, "voxel (surf; corner on the side stream)");
  ScanRef S{F.surf_ds, n, F.n_surf_ds, F.corner_ds, less_cap, F.n_corner_ds};
  *S_out = S;
  return MLOAM_OK;
}

// mloam_frame copied inputs on a branch's stream outside of any capture, recorded in ev.  Run on that branch (forked), the stream path is
// ordered after them already and a captured graph waits on the record as an external event node; unforked, c->stream waits on it.
int wait_uploads(Ctx *c, cudaEvent_t ev, bool forked) {
  if (!forked) {
    MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, ev, 0));
    return MLOAM_OK;
  }
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  MLOAM_CUDA_OK(c, cudaStreamIsCapturing(c->stream, &cs));
  if (cs == cudaStreamCaptureStatusActive) MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, ev, cudaEventWaitExternal));
  return MLOAM_OK;
}

// The look-ahead state a frame leaves, on the stream path and on a replay alike: the next frame extracts into the other half, and nf
// (valid when this frame ran the look-ahead) describes the announced sweep's features
void frame_advance(Ctx *c, int parity, const Ctx::Features &nf) {
  c->frame_parity = parity ^ 1;
  c->prefetched = nf;
}

// The features of sw — ready from the look-ahead when `have`, else extracted now into half `parity` — the look-ahead of the announced
// sweep, the map builds (rebuild_maps) and the solve on c->stream.  *ran: scan2map_enqueue's.
int frame_enqueue(Ctx *c, const Sweep &sw, bool have, int parity, const float4 *d_surf_map, int n_surf_map, const float4 *d_corner_map,
                  int n_corner_map, int rebuild_maps, const double *pose_init7, ScanRef *S_out, int *ran) {
  // lidar_mapper_keyframe.cpp:433-434 (every frame in the reference).  The two submap builds do not depend on the sweep: they run on a
  // forked side stream, concurrently with extraction + scan down-sampling, and join right before matching (also inside a captured graph).
  // With stage profiling on the branch stays on the main stream so that per-stage event times do not overlap.
  const bool fork_maps = rebuild_maps && !c->prof_on;
  int rc;
  if (rebuild_maps) {
    rc = on_branch(c, c->br_maps, fork_maps, [&] {
      int r = c->maps_pending ? wait_uploads(c, c->ev_maps, fork_maps) : MLOAM_OK;
      if (r == MLOAM_OK) r = map_build_device(c, MLOAM_MAP_SURF, d_surf_map, n_surf_map, pick_cell(c, 0.f));
      if (r == MLOAM_OK) r = map_build_device(c, MLOAM_MAP_CORNER, d_corner_map, n_corner_map, pick_cell(c, 0.f));
      return r;
    });
    if (rc) return rc;
  }
  c->stamp_n = 0;
  stamp(c, "start");
  ScanRef S{};
  if (have) S = c->prefetched.S;
  c->prefetched.valid = false;  // half `parity` is taken or overwritten here
  if (!have) {
    rc = features_enqueue(c, sw, parity, c->br_scan, &S);
    if (rc) return rc;
  }
  // look-ahead: the announced next sweep goes through the same steps on br_ahead into the other half while this frame is matched
  // and solved (it reuses Ctx::extract_work, voxel_corner and voxel_surf of the block above, hence the fork AFTER it)
  Ctx::Features nf{};
  if (c->next.set && c->use_lookahead && !c->prof_on) {
    const Sweep &nx = c->next.sw;
    c->stamp_mute = true;
    rc = on_branch(c, c->br_ahead, true, [&] {
      int r = c->next_pending ? wait_uploads(c, c->ev_next, true) : MLOAM_OK;  // mloam_frame copied the next sweep on br_ahead
      if (r == MLOAM_OK) r = features_enqueue(c, nx, parity ^ 1, c->br_ahead_scan, &nf.S);
      return r;
    });
    c->stamp_mute = false;
    if (rc) return rc;
    nf.valid = true, nf.parity = parity ^ 1, nf.sw = nx;
  }
  stamp(c, have ? "features (prefetched)" : "extract + voxel");
  if (c->with_ua) {  // downsampleCurrentScan's per-point uncertainty + trace gate: on the main stream with the covariances of THIS call
    rc = ua_scan_stage(c, &S);
    if (rc) return rc;
    stamp(c, "uncertainty + gate");
  }
  if (fork_maps) {  // join the map-build branch
    MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, c->br_maps.join, 0));
    stamp(c, "map build join");
  }
  *S_out = S;
  rc = scan2map_enqueue(c, S, pose_init7, c->with_ua != 0, ran);
  if (rc) return rc;
  if (nf.valid) {  // the frame ends when both branches have: the features of the next sweep are complete when this call returns
    MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, c->br_ahead.join, 0));
    stamp(c, "look-ahead join");
  }
  frame_advance(c, parity, nf);
  return MLOAM_OK;
}

// Point the device side of host sweep *sw into B (the points, then room for its ScanInfo) and, with `upload`, copy the sweep there on st.
// The ScanInfo goes through the pinned rows pin: an async copy from pageable memory would block the host behind the sweep's copy.
int sweep_to_device(Ctx *c, DevBuf &B, Sweep *sw, bool upload, int (*pin)[MLOAM_MAX_RINGS], cudaStream_t st) {
  SweepIn D;
  int rc = sweep_bufs(c, B, sw->n, sw->n_scans, &D);
  if (rc) return rc;
  sw->cloud = D.cloud;
  if (!sw->raw) sw->scan_start = D.scan_start, sw->scan_end = D.scan_end;  // a raw sweep has no ScanInfo: the front end makes it
  if (!upload) return MLOAM_OK;
  const int ns = sw->n_scans;
  if (!sw->raw) {
    std::memcpy(pin[0], sw->h_scan_start, sizeof(int) * ns), std::memcpy(pin[1], sw->h_scan_end, sizeof(int) * ns);
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.scan_start, pin[0], sizeof(int) * ns, cudaMemcpyHostToDevice, st));
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.scan_end, pin[1], sizeof(int) * ns, cudaMemcpyHostToDevice, st));
  }
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.cloud, sw->key, sizeof(float4) * (size_t)sw->n, cudaMemcpyHostToDevice, st));
  return MLOAM_OK;
}

// A sweep announced from HOST memory goes up on br_ahead right away (outside of any capture); the look-ahead branch of the frame
// waits on ev_next.  br_ahead's previous work — the look-ahead of the previous frame, which read next_in — was joined by that frame.
int stage_next_sweep(Ctx *c) {
  if (!c->next.set || !c->next.sw.host || !c->use_lookahead || c->prof_on) return MLOAM_OK;
  int rc = sweep_to_device(c, c->next_in, &c->next.sw, true, c->pinned->scan_info_next, c->br_ahead.stream);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaEventRecord(c->ev_next, c->br_ahead.stream));
  c->next_pending = true;
  return MLOAM_OK;
}

unsigned long long fnv1a(unsigned long long h, const void *p, size_t n) {
  const unsigned char *b = static_cast<const unsigned char *>(p);
  for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 1099511628211ull;
  return h;
}

// One frame.  With max_inner == 1 the ~60 launches of a frame form a fixed sequence that depends on the host only
// through the pose guess (staged in pinned memory) — it is captured once per (buffers, sizes, parameters) into a CUDA
// graph and replayed: the first call with a new key runs on the stream (and performs every allocation), the second
// captures + instantiates, later ones replay.  Profiling, multi-GPU (NCCL on the stream) and max_inner > 1 (the host
// polls the LM done flag) use the plain stream path.  have / parity: the look-ahead decision of frame_call, in the key and the
// same on every path.
int frame_run(Ctx *c, const Sweep &sw, bool have, int parity, const float4 *d_surf_map, int n_surf_map, const float4 *d_corner_map,
              int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  ScanRef S{};
  if (c->with_ua && c->nccl_comm)
    return fail(c, MLOAM_E_STATE, "frame: uncertainty-aware frames (mloam_set_uncertainty) are single-GPU only; detach the communicator or set with_ua = 0");
  const bool want_cov = c->with_ua != 0;
  c->last_scan_valid = false;
  const bool can_graph = c->use_graphs && c->params.max_inner == 1 && !c->prof_on && (!c->nccl_comm || c->p2p_on);
  if (can_graph) {
    unsigned long long key = 1469598103934665603ull;
    const void *ptrs[5] = {sw.cloud, sw.scan_start, sw.scan_end, d_surf_map, d_corner_map};
    const int ints[7] = {sw.n, sw.n_scans, n_surf_map, n_corner_map, rebuild_maps, c->has_ext ? 1 : 0, c->maps_pending ? 1 : 0};
    key = fnv1a(key, ptrs, sizeof(ptrs));
    key = fnv1a(key, ints, sizeof(ints));
    if (rebuild_maps && !(c->params.map_cell > 0.f)) {  // the auto cell edges are kernel arguments of the captured build
      const float cells[2] = {c->maps[MLOAM_MAP_SURF].auto_cell_pick(c->pinned, MLOAM_MAP_SURF),
                              c->maps[MLOAM_MAP_CORNER].auto_cell_pick(c->pinned, MLOAM_MAP_CORNER)};
      key = fnv1a(key, cells, sizeof(cells));
    }
    key = fnv1a(key, &c->params, sizeof(c->params));
    key = fnv1a(key, c->ext, sizeof(c->ext));
    key = fnv1a(key, &c->n_lidars, sizeof(c->n_lidars));
    key = fnv1a(key, &c->lidar_merge, sizeof(c->lidar_merge));
    key = fnv1a(key, c->lidar_ext, sizeof(double) * 7 * (size_t)c->n_lidars);
    key = fnv1a(key, &c->stream, sizeof(c->stream));
    key = fnv1a(key, &c->with_ua, sizeof(c->with_ua));  // the covariances and the threshold are staged, not part of the key
    if (sw.raw) {  // raw frame: the per-LiDAR counts and the front-end parameters are kernel arguments of the captured front end
      key = fnv1a(key, &sw.L, sizeof(RigLayout));
      key = fnv1a(key, &c->front, sizeof(c->front));
    }
    if (!rebuild_maps) {
      // the map-size gate (scan2map_enqueue) is decided on the host at capture: with maps built outside the frame (mloam_map_build*,
      // mloam_submap_assemble, mloam_keyframe_submap) a graph captured while it failed must not be replayed once it passes, and back
      const MapStorage &MS = c->maps[MLOAM_MAP_SURF], &MC = c->maps[MLOAM_MAP_CORNER];
      const int gate = (MS.built && MC.built && MS.m > 50 && MC.m > 10) ? 1 : 0;
      key = fnv1a(key, &gate, sizeof(gate));
    }
    {  // look-ahead: which half holds this sweep's features (or that they are extracted now), and the announced next sweep
      const Sweep &nx = c->next.sw;
      const bool ahead = c->next.set && c->use_lookahead;
      const int la[8] = {have ? 1 : 0, parity, ahead ? 1 : 0, ahead ? nx.n : 0, ahead ? nx.n_scans : 0, (ahead && nx.host) ? 1 : 0,
                         (ahead && c->next_pending) ? 1 : 0, c->stamp_on ? 1 : 0};
      const void *lp[5] = {sw.key, ahead ? nx.key : nullptr, ahead ? static_cast<const void *>(nx.cloud) : nullptr,
                           ahead ? static_cast<const void *>(nx.scan_start) : nullptr, ahead ? static_cast<const void *>(nx.scan_end) : nullptr};
      key = fnv1a(key, la, sizeof(la));
      key = fnv1a(key, lp, sizeof(lp));
      if (ahead && nx.raw) key = fnv1a(key, &nx.L, sizeof(RigLayout)), key = fnv1a(key, &c->front, sizeof(c->front));
    }
    Ctx::GraphEntry *e = nullptr;
    for (auto &g : c->graphs)
      if (g.key == key) e = &g;
    if (e && e->exec && e->epoch == alloc_epoch()) {
      stage_frame_inputs(c, pose_init7);  // the captured H2D nodes read them at execution time
      MLOAM_CUDA_OK(c, cudaGraphLaunch(e->exec, c->stream));
      c->launches += e->launches;
      frame_advance(c, parity, e->prefetched_out);
      c->last_scan = e->S, c->last_scan_valid = true;
      return scan2map_finish(c, e->S, pose_init7, want_cov, e->s2m_ran, pose_out7, stats);
    }
    if (e && e->seen >= 1) {  // second sighting: capture
      if (e->exec) cudaGraphExecDestroy(e->exec), e->exec = nullptr;
      const long long l0 = c->launches;
      const unsigned long long ep0 = alloc_epoch();
      cudaGraph_t graph = nullptr;
      const Ctx::Features pf0 = c->prefetched;  // frame_enqueue advances these: put them back when the capture fails
      const int par0 = c->frame_parity;
      int ran = 0;
      MLOAM_CUDA_OK(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
      int rc = frame_enqueue(c, sw, have, parity, d_surf_map, n_surf_map, d_corner_map, n_corner_map, rebuild_maps, pose_init7, &S, &ran);
      cudaError_t ce = cudaStreamEndCapture(c->stream, &graph);
      if (rc == MLOAM_OK && ce == cudaSuccess && graph && ep0 == alloc_epoch() &&
          cudaGraphInstantiate(&e->exec, graph, 0) == cudaSuccess) {
        e->launches = (int)(c->launches - l0), e->epoch = ep0, e->S = S, e->s2m_ran = ran;
        e->prefetched_out = c->prefetched;
        c->launches = l0;
        cudaGraphDestroy(graph);
        MLOAM_CUDA_OK(c, cudaGraphLaunch(e->exec, c->stream));
        c->launches += e->launches;
        c->last_scan = S, c->last_scan_valid = true;
        return scan2map_finish(c, S, pose_init7, want_cov, ran, pose_out7, stats);
      }
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      e->exec = nullptr, e->seen = 0;  // capture failed (e.g. a buffer had to grow, which is illegal while capturing): run this frame on
      c->launches = l0;                // the plain stream path below — it performs the allocation — and capture at a later sighting
      c->graph_capture_failures++;
      c->prefetched = pf0, c->frame_parity = par0;
    } else if (!e) {
      if (c->graphs.size() >= 96) {
        if (c->graphs.front().exec) cudaGraphExecDestroy(c->graphs.front().exec);
        c->graphs.erase(c->graphs.begin());
      }
      Ctx::GraphEntry g;
      g.key = key, g.seen = 1;
      c->graphs.push_back(g);
    }
  }
  int ran = 0;
  int rc = frame_enqueue(c, sw, have, parity, d_surf_map, n_surf_map, d_corner_map, n_corner_map, rebuild_maps, pose_init7, &S, &ran);
  if (rc) return rc;
  c->last_scan = S, c->last_scan_valid = true;
  return scan2map_finish(c, S, pose_init7, want_cov, ran, pose_out7, stats);
}

// A ring-ordered sweep (cloud + ScanInfo, in host or in device memory)
Sweep ring_sweep(const mloam_point_t *cloud, bool host, int n, const int *scan_start, const int *scan_end, int n_scans) {
  Sweep sw;
  sw.key = cloud, sw.host = host, sw.n = n, sw.n_scans = n_scans;
  if (host) sw.h_scan_start = scan_start, sw.h_scan_end = scan_end;
  else sw.cloud = reinterpret_cast<const float4 *>(cloud), sw.scan_start = scan_start, sw.scan_end = scan_end;
  return sw;
}

// The rig's raw sweeps at `raw` (host or device memory; h_counts[l] points of LiDAR l, n_lidars of mloam_set_lidars) after the checks every
// raw entry point makes
int raw_sweep(Ctx *c, const mloam_point_t *raw, bool host, const int *h_counts, Sweep *sw) {
  if (!c->front_set) return fail(c, MLOAM_E_STATE, "frame_raw: call mloam_set_front_end first");
  if (c->nccl_comm) return fail(c, MLOAM_E_STATE, "frame_raw: raw frames are single-GPU only; detach the communicator");
  if (!h_counts) return MLOAM_E_INVALID;
  const FrontEnd &fe = c->front;
  if (c->params.max_ring_points > 0 && c->params.max_ring_points < fe.horizon_scans)
    return fail(c, MLOAM_E_INVALID, "frame_raw: params.max_ring_points is below horizon_scans (a projected ring holds up to horizon_scans points)");
  *sw = Sweep{};
  RigLayout &L = sw->L;
  L.n_lidars = c->n_lidars;
  long long total = 0;
  for (int l = 0; l < c->n_lidars; l++) {
    if (h_counts[l] <= 0)  // the driver node's empty_check (rosNodeRVOxford.cpp:216-220)
      return fail(c, MLOAM_E_INVALID, "frame_raw: every LiDAR of the rig needs a non-empty sweep");
    L.off[l] = (int)total;
    total += h_counts[l];
    if (total > (1 << 30)) return fail(c, MLOAM_E_INVALID, "frame_raw: sweeps too large");
  }
  L.off[c->n_lidars] = (int)total;
  sw->key = raw, sw->host = host, sw->raw = true, sw->n = (int)total, sw->n_scans = c->n_lidars * fe.vertical_scans;
  if (!host) sw->cloud = reinterpret_cast<const float4 *>(raw);
  return MLOAM_OK;
}

// The submaps of a host frame (16 B/point, ~8x the sweep) go up on br_maps so that the copy overlaps extraction and scan down-sampling of
// the sweep; the map-build branch of frame_enqueue is ordered after ev_maps.
int upload_submaps(Ctx *c, const mloam_point_t *h_surf_map, int n_surf_map, const mloam_point_t *h_corner_map, int n_corner_map,
                   const float4 **d_surf_map, const float4 **d_corner_map) {
  DevBuf &ms = c->map_in[0], &mc = c->map_in[1];
  MLOAM_CUDA_OK(c, ms.reserve(sizeof(float4) * (size_t)(n_surf_map + 1)));
  MLOAM_CUDA_OK(c, mc.reserve(sizeof(float4) * (size_t)(n_corner_map + 1)));
  cudaStream_t st = c->br_maps.stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(ms.p, h_surf_map, sizeof(float4) * (size_t)n_surf_map, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(mc.p, h_corner_map, sizeof(float4) * (size_t)n_corner_map, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaEventRecord(c->ev_maps, st));
  c->maps_pending = true;
  *d_surf_map = ms.as<float4>(), *d_corner_map = mc.as<float4>();
  return MLOAM_OK;
}

// What every mloam_frame* entry point does with its sweep sw and submaps (host buffers for a host sweep, device buffers otherwise): the
// sweep — unless the look-ahead made its features —, the announced next sweep and the submaps go up, the frame runs, and the call
// consumes the announcement and the uploads.
int frame_call(Ctx *c, Sweep sw, const mloam_point_t *surf_map, int n_surf_map, const mloam_point_t *corner_map, int n_corner_map,
               int rebuild_maps, const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (sw.host && rebuild_maps && (!surf_map || !corner_map || n_surf_map < 0 || n_corner_map < 0)) return MLOAM_E_INVALID;
  cudaSetDevice(c->device);
  // this sweep's features: extracted while the previous frame was solved (look-ahead), or now into the half after the previous frame's
  const bool have = frame_has_prefetched(c, sw);
  const int parity = have ? c->prefetched.parity : c->frame_parity;
  const float4 *d_sm = sw.host ? nullptr : reinterpret_cast<const float4 *>(surf_map);
  const float4 *d_cm = sw.host ? nullptr : reinterpret_cast<const float4 *>(corner_map);
  int rc = sw.host ? sweep_to_device(c, c->sweep_in, &sw, !have, c->pinned->scan_info, c->stream) : MLOAM_OK;
  if (rc == MLOAM_OK) rc = stage_next_sweep(c);
  if (rc == MLOAM_OK && sw.host && rebuild_maps) rc = upload_submaps(c, surf_map, n_surf_map, corner_map, n_corner_map, &d_sm, &d_cm);
  if (rc == MLOAM_OK) rc = frame_run(c, sw, have, parity, d_sm, n_surf_map, d_cm, n_corner_map, rebuild_maps, pose_init7, pose_out7, stats);
  c->maps_pending = false, c->next_pending = false, c->next.set = false;
  if (rc == MLOAM_OK) memcpy(c->last_pose7, pose_out7, sizeof(c->last_pose7)), c->frame_since_save = true;  // mloam_keyframe_save
  return rc;
}

// What every mloam_frame_set_next* call does after its checks (rc): the previous announcement is withdrawn, and sw — unless the checks
// failed or sw is empty (a withdrawal) — is announced for the next frame
int announce(Ctx *c, const Sweep &sw, int rc) {
  c->next = Ctx::NextSweep{};
  if (rc == MLOAM_OK && sw.key) c->next.set = true, c->next.sw = sw;
  return rc;
}

}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------ scan2map
int mloam_scan2map_device(mloam_ctx_t *h, const mloam_point_t *d_surf_scan, int n_surf, const mloam_point_t *d_corner_scan,
                          int n_corner, const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || n_surf < 0 || n_corner < 0) return MLOAM_E_INVALID;
  cudaSetDevice(h->c.device);
  ScanRef S{reinterpret_cast<const float4 *>(d_surf_scan), n_surf, nullptr, reinterpret_cast<const float4 *>(d_corner_scan), n_corner,
            nullptr};
  return scan2map_run(&h->c, S, pose_init7, false, pose_out7, stats);
}

int mloam_scan2map(mloam_ctx_t *h, const mloam_point_t *h_surf_scan, int n_surf, const mloam_point_t *h_corner_scan, int n_corner,
                   const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || n_surf < 0 || n_corner < 0) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  MLOAM_CUDA_OK(c, c->scan_pts[0].reserve(sizeof(float4) * (size_t)(n_corner + 1)));
  MLOAM_CUDA_OK(c, c->scan_pts[1].reserve(sizeof(float4) * (size_t)(n_surf + 1)));
  if (n_corner > 0)
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->scan_pts[0].p, h_corner_scan, sizeof(float4) * (size_t)n_corner, cudaMemcpyHostToDevice, c->stream));
  if (n_surf > 0)
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->scan_pts[1].p, h_surf_scan, sizeof(float4) * (size_t)n_surf, cudaMemcpyHostToDevice, c->stream));
  ScanRef S{c->scan_pts[1].as<float4>(), n_surf, nullptr, c->scan_pts[0].as<float4>(), n_corner, nullptr};
  return scan2map_run(c, S, pose_init7, false, pose_out7, stats);
}

// scan2MapOptimization with with_ua = true (lidar_mapper_keyframe.cpp:541-545,556-560): every residual is weighted by
// sqrt_info of its scan point's covariance (PointIWithCov::cov_vec, float[6] per point, from mloam_point_uncertainty).
int mloam_scan2map_ua(mloam_ctx_t *h, const mloam_point_t *h_surf_scan, int n_surf, const float *h_surf_cov6,
                      const mloam_point_t *h_corner_scan, int n_corner, const float *h_corner_cov6, const double *pose_init7,
                      double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || n_surf < 0 || n_corner < 0 || (n_surf > 0 && (!h_surf_scan || !h_surf_cov6)) ||
      (n_corner > 0 && (!h_corner_scan || !h_corner_cov6)))
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  cudaStream_t st = c->stream;
  const int ns[2] = {n_corner, n_surf};
  const mloam_point_t *hp[2] = {h_corner_scan, h_surf_scan};
  const float *hc[2] = {h_corner_cov6, h_surf_cov6};
  float *cov[2];
  double *sin[2];
  MLOAM_CUDA_OK(c, carve(c->host_work, [&](Carve &cv) {
    for (int t = 0; t < 2; t++) cov[t] = cv.take<float>(6 * (size_t)(ns[t] + 1)), sin[t] = cv.take<double>((size_t)ns[t] + 1);
  }));
  for (int t = 0; t < 2; t++) {
    MLOAM_CUDA_OK(c, c->scan_pts[t].reserve(sizeof(float4) * (size_t)(ns[t] + 1)));
    if (ns[t] > 0) {
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->scan_pts[t].p, hp[t], sizeof(float4) * (size_t)ns[t], cudaMemcpyHostToDevice, st));
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(cov[t], hc[t], sizeof(float) * 6 * (size_t)ns[t], cudaMemcpyHostToDevice, st));
      int rc = sqrt_info_device(c, cov[t], ns[t], sin[t]);
      if (rc) return rc;
    }
  }
  ScanRef S{c->scan_pts[1].as<float4>(), n_surf, nullptr, c->scan_pts[0].as<float4>(), n_corner, nullptr, sin[1], sin[0]};
  return scan2map_run(c, S, pose_init7, true, pose_out7, stats);  // with_ua: pose_wmap_curr.cov_ = H^-1 at the returned pose (mloam_pose_covariance)
}

// ------------------------------------------------------------------------------------------ extractCloud
int mloam_extract_features(mloam_ctx_t *h, const mloam_point_t *h_cloud, int n, const int *h_scan_start, const int *h_scan_end,
                           int n_scans, mloam_features_t *out) {
  if (!h || !out || n < 0 || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS || (n > 0 && !h_cloud) || !h_scan_start || !h_scan_end)
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  out->n_sharp = out->n_less_sharp = out->n_flat = out->n_less_flat = 0;
  if (n == 0) return MLOAM_OK;
  c->prefetched.valid = false;  // this call reuses half 0 of the frame feature buffers
  c->last_scan_valid = false;
  FrameBufs F;
  int rc = frame_bufs(c, n, &F);
  if (rc) return rc;
  SweepIn D;
  rc = sweep_bufs(c, c->sweep_in, n, n_scans, &D);
  if (rc) return rc;
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.cloud, h_cloud, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.scan_start, h_scan_start, sizeof(int) * n_scans, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.scan_end, h_scan_end, sizeof(int) * n_scans, cudaMemcpyHostToDevice, st));
  rc = extract_device(c, D.cloud, n, D.scan_start, D.scan_end, n_scans, F.ex, nullptr, nullptr);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, F.ex.counts, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc + 4, c->d_extract_status, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  if (hc[4] != 0)
    return fail(c, MLOAM_E_INVALID, "extract: a ring exceeds the on-chip window (12288 points) or ScanInfo is out of range");
  if (hc[0] > out->cap || hc[1] > out->cap || hc[2] > out->cap || hc[3] > out->cap)
    return fail(c, MLOAM_E_INVALID, "extract: output capacity too small");
  out->n_sharp = hc[0], out->n_less_sharp = hc[1], out->n_flat = hc[2], out->n_less_flat = hc[3];
  if (out->corner_points_sharp && hc[0])
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(out->corner_points_sharp, F.ex.sharp, sizeof(float4) * hc[0], cudaMemcpyDeviceToHost, st));
  if (out->corner_points_less_sharp && hc[1])
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(out->corner_points_less_sharp, F.ex.less_sharp, sizeof(float4) * hc[1], cudaMemcpyDeviceToHost, st));
  if (out->surf_points_flat && hc[2])
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(out->surf_points_flat, F.ex.flat, sizeof(float4) * hc[2], cudaMemcpyDeviceToHost, st));
  if (out->surf_points_less_flat && hc[3])
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(out->surf_points_less_flat, F.ex.less_flat, sizeof(float4) * hc[3], cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

int mloam_extract_debug(mloam_ctx_t *h, float *h_curvature, int *h_label, int n) {
  if (!h || n < 0) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  // extract_device's work; curvature and label do not depend on the ring count, and one ring is the smallest extraction of n points
  ExtractWork W;
  Carve cv(c->extract_work.p);
  extract_work_layout(cv, n, 1, &W);
  if (c->extract_work.cap < cv.size) return fail(c, MLOAM_E_STATE, "extract_debug: no extraction of this size has run");
  if (h_curvature) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_curvature, W.curv, sizeof(float) * n, cudaMemcpyDeviceToHost, c->stream));
  if (h_label) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_label, W.label, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ range image
int mloam_project_cloud(mloam_ctx_t *h, const mloam_point_t *h_cloud, int n, int vertical_scans, int horizon_scans, double roi_range,
                        mloam_point_t *h_out, int *n_out, int *h_scan_start, int *h_scan_end) {
  if (!h || n < 0 || !n_out || !h_scan_start || !h_scan_end || (n > 0 && (!h_cloud || !h_out))) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  *n_out = 0;
  if (vertical_scans != 16 && vertical_scans != 32 && vertical_scans != 64)
    return fail(c, MLOAM_E_INVALID, "project_cloud: vertical_scans must be 16, 32 or 64 (ImageSegmenter::setParameter)");
  if (horizon_scans <= 0) return MLOAM_E_INVALID;
  if (n == 0) {  // image_segmenter.hpp:381-387 on an empty cloud
    for (int i = 0; i < vertical_scans; i++) h_scan_start[i] = 5, h_scan_end[i] = -6;
    return MLOAM_OK;
  }
  MLOAM_CUDA_OK(c, c->sweep_in.reserve(sizeof(float4) * (size_t)n));
  float4 *d_out;
  int *d_meta;  // [0] count, [64..] start, [128..] end (PinnedBlock::counts)
  MLOAM_CUDA_OK(c, carve(c->map_in[0], [&](Carve &cv) { d_out = cv.take<float4>(n), d_meta = cv.take<int>(192); }));
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->sweep_in.p, h_cloud, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  RigLayout L{};
  L.n_lidars = 1, L.off[1] = n;
  int rc = project_cloud_device(c, c->sweep_in.as<float4>(), L, vertical_scans, horizon_scans, roi_range, nullptr, d_out, d_meta + 64,
                                d_meta + 128, d_meta, c->front_work);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_meta, sizeof(int) * 192, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  *n_out = hc[0];
  std::memcpy(h_scan_start, hc + 64, sizeof(int) * vertical_scans), std::memcpy(h_scan_end, hc + 128, sizeof(int) * vertical_scans);
  if (hc[0] > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_out, sizeof(float4) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ voxel grid
int mloam_voxel_downsample(mloam_ctx_t *h, const mloam_point_t *h_in, int n, float leaf, int intensity_last, mloam_point_t *h_out,
                           int *n_out) {
  if (!h || n < 0 || !n_out || (n > 0 && (!h_in || !h_out)) || !(leaf > 0.f)) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  *n_out = 0;
  if (n == 0) return MLOAM_OK;
  MLOAM_CUDA_OK(c, c->sweep_in.reserve(sizeof(float4) * (size_t)n));
  float4 *d_out;
  int *d_cnt;
  MLOAM_CUDA_OK(c, carve(c->map_in[0], [&](Carve &cv) { d_out = cv.take<float4>(n), d_cnt = cv.take<int>(16); }));
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->sweep_in.p, h_in, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  int rc = voxel_downsample_device(c, c->sweep_in.as<float4>(), n, nullptr, leaf, intensity_last, d_out, d_cnt, c->voxel_work);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  *n_out = hc[0];
  if (hc[0] > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_out, sizeof(float4) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ frame
int mloam_frame_device(mloam_ctx_t *h, const mloam_point_t *d_cloud, int n, const int *d_scan_start, const int *d_scan_end, int n_scans,
                       const mloam_point_t *d_surf_map, int n_surf_map, const mloam_point_t *d_corner_map, int n_corner_map,
                       int rebuild_maps, const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || n <= 0 || !d_cloud || !d_scan_start || !d_scan_end) return MLOAM_E_INVALID;
  return frame_call(&h->c, ring_sweep(d_cloud, false, n, d_scan_start, d_scan_end, n_scans), d_surf_map, n_surf_map, d_corner_map,
                    n_corner_map, rebuild_maps, pose_init7, pose_out7, stats);
}

// Look-ahead: announce the sweep of the NEXT mloam_frame* call.  While the coming frame is matched and solved, that sweep is extracted
// and down-sampled on a side stream (in the reference the two stages run in different nodes, estimator -> lidar_mapper); the next
// call finds its features ready when it passes the same pointer (and sizes) — otherwise it extracts as usual.  One announcement is
// consumed by one frame; results are identical with or without it.
int mloam_frame_set_next_device(mloam_ctx_t *h, const mloam_point_t *d_cloud, int n, const int *d_scan_start, const int *d_scan_end, int n_scans) {
  if (!h) return MLOAM_E_INVALID;
  if (!d_cloud || n <= 0) return announce(&h->c, Sweep{}, MLOAM_OK);  // withdraw
  const int rc = (!d_scan_start || !d_scan_end || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS) ? MLOAM_E_INVALID : MLOAM_OK;
  return announce(&h->c, ring_sweep(d_cloud, false, n, d_scan_start, d_scan_end, n_scans), rc);
}
int mloam_frame_set_next(mloam_ctx_t *h, const mloam_point_t *h_cloud, int n, const int *h_scan_start, const int *h_scan_end, int n_scans) {
  if (!h) return MLOAM_E_INVALID;
  if (!h_cloud || n <= 0) return announce(&h->c, Sweep{}, MLOAM_OK);  // withdraw
  const int rc = (!h_scan_start || !h_scan_end || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS) ? MLOAM_E_INVALID : MLOAM_OK;
  return announce(&h->c, ring_sweep(h_cloud, true, n, h_scan_start, h_scan_end, n_scans), rc);
}

int mloam_frame(mloam_ctx_t *h, const mloam_point_t *h_cloud, int n, const int *h_scan_start, const int *h_scan_end, int n_scans,
                const mloam_point_t *h_surf_map, int n_surf_map, const mloam_point_t *h_corner_map, int n_corner_map, int rebuild_maps,
                const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || n <= 0 || !h_cloud || !h_scan_start || !h_scan_end || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS)
    return MLOAM_E_INVALID;
  return frame_call(&h->c, ring_sweep(h_cloud, true, n, h_scan_start, h_scan_end, n_scans), h_surf_map, n_surf_map, h_corner_map,
                    n_corner_map, rebuild_maps, pose_init7, pose_out7, stats);
}

// ------------------------------------------------------------------------------------------ raw driver sweeps
// removeNaNFromPointCloud (rosNodeRVKITTI.cpp:154-161, rosNodeRVOxford.cpp:170-177) + FeatureExtract::calTimestamp (feature_extract.cpp:25-114)
int mloam_cal_timestamp(mloam_ctx_t *h, const mloam_point_t *h_cloud, int n, int time_field, float scan_period, mloam_point_t *h_out,
                        int *n_out) {
  if (!h || n < 0 || !n_out || (n > 0 && (!h_cloud || !h_out))) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  *n_out = 0;
  if (n == 0) return MLOAM_OK;
  MLOAM_CUDA_OK(c, c->sweep_in.reserve(sizeof(float4) * (size_t)n));
  float4 *d_out;
  int *d_cnt;
  MLOAM_CUDA_OK(c, carve(c->map_in[0], [&](Carve &cv) { d_out = cv.take<float4>(n), d_cnt = cv.take<int>(16); }));
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->sweep_in.p, h_cloud, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  RigLayout L{};
  L.n_lidars = 1, L.off[1] = n;
  int rc = front_times_device(c, c->sweep_in.as<float4>(), L, time_field ? 1 : 0, scan_period, d_out, d_cnt, c->front_work);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  *n_out = hc[0];
  if (hc[0] > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_out, sizeof(float4) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

int mloam_set_front_end(mloam_ctx_t *h, int vertical_scans, int horizon_scans, double roi_range, float scan_period, int time_field) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (vertical_scans != 16 && vertical_scans != 32 && vertical_scans != 64)
    return fail(c, MLOAM_E_INVALID, "set_front_end: vertical_scans must be 16, 32 or 64 (ImageSegmenter::setParameter)");
  if (horizon_scans <= 0 || !(scan_period > 0.f)) return fail(c, MLOAM_E_INVALID, "set_front_end: horizon_scans and scan_period must be positive");
  if (c->params.max_ring_points > 0 && c->params.max_ring_points < horizon_scans)
    return fail(c, MLOAM_E_INVALID, "set_front_end: params.max_ring_points is below horizon_scans (a projected ring holds up to horizon_scans points)");
  c->front = FrontEnd{vertical_scans, horizon_scans, roi_range, scan_period, time_field ? 1 : 0};
  c->front_set = true;
  c->prefetched.valid = false;  // look-ahead features were made with the previous front end
  return MLOAM_OK;
}

int mloam_front_end(mloam_ctx_t *h, const mloam_point_t *h_raw, const int *h_counts, mloam_point_t *h_out, int *n_out, int *h_scan_start,
                    int *h_scan_end) {
  if (!h || !h_raw || !h_out || !n_out || !h_scan_start || !h_scan_end) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  *n_out = 0;
  Sweep sw;
  int rc = raw_sweep(c, h_raw, true, h_counts, &sw);
  if (rc) return rc;
  cudaSetDevice(c->device);
  const int n = sw.n, n_scans = sw.n_scans;
  c->prefetched.valid = false;  // the front end's output buffer is the frame's
  MLOAM_CUDA_OK(c, c->sweep_in.reserve(sizeof(float4) * (size_t)n));
  float4 *d_out;
  int *d_meta;  // [0] count, then scan starts, scan ends
  MLOAM_CUDA_OK(c, carve(c->front_out, [&](Carve &cv) { d_out = cv.take<float4>((size_t)n + 1), d_meta = cv.take<int>(4 + 2 * (size_t)n_scans); }));
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->sweep_in.p, h_raw, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  const FrontEnd &fe = c->front;
  rc = project_cloud_device(c, c->sweep_in.as<float4>(), sw.L, fe.vertical_scans, fe.horizon_scans, fe.roi_range, &fe, d_out, d_meta + 4,
                            d_meta + 4 + n_scans, d_meta, c->front_work);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_scan_start, d_meta + 4, sizeof(int) * n_scans, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_scan_end, d_meta + 4 + n_scans, sizeof(int) * n_scans, cudaMemcpyDeviceToHost, st));
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_meta, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  *n_out = hc[0];
  if (hc[0] > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_out, sizeof(float4) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

int mloam_frame_raw(mloam_ctx_t *h, const mloam_point_t *h_raw, const int *h_counts, const mloam_point_t *h_surf_map, int n_surf_map,
                    const mloam_point_t *h_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7,
                    mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || !h_raw) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = raw_sweep(&h->c, h_raw, true, h_counts, &sw);
  if (rc) return rc;
  return frame_call(&h->c, sw, h_surf_map, n_surf_map, h_corner_map, n_corner_map, rebuild_maps, pose_init7, pose_out7, stats);
}

int mloam_frame_raw_device(mloam_ctx_t *h, const mloam_point_t *d_raw, const int *h_counts, const mloam_point_t *d_surf_map, int n_surf_map,
                           const mloam_point_t *d_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7,
                           mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || !d_raw) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = raw_sweep(&h->c, d_raw, false, h_counts, &sw);
  if (rc) return rc;
  return frame_call(&h->c, sw, d_surf_map, n_surf_map, d_corner_map, n_corner_map, rebuild_maps, pose_init7, pose_out7, stats);
}

// Look-ahead for raw frames: as mloam_frame_set_next*, picked up by the next mloam_frame_raw* call with the same pointer and counts
int mloam_frame_set_next_raw(mloam_ctx_t *h, const mloam_point_t *h_raw, const int *h_counts) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = h_raw ? raw_sweep(&h->c, h_raw, true, h_counts, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, sw, rc);
}
int mloam_frame_set_next_raw_device(mloam_ctx_t *h, const mloam_point_t *d_raw, const int *h_counts) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = d_raw ? raw_sweep(&h->c, d_raw, false, h_counts, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, sw, rc);
}

int mloam_set_lidars(mloam_ctx_t *h, int n_lidars, const double *ext7) {
  if (!h || n_lidars < 1 || n_lidars > MLOAM_MAX_LIDARS || (n_lidars > 1 && !ext7)) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  c->n_lidars = n_lidars;
  c->prefetched.valid = false;  // look-ahead features were merged with the previous extrinsics
  c->lidar_merge = ext7 != nullptr;  // also for ONE LiDAR with an extrinsic: same float transform + laser id as in a rig
  for (int l = 0; l < n_lidars; l++)
    for (int k = 0; k < 7; k++) c->lidar_ext[l][k] = ext7 ? ext7[7 * l + k] : (k == 6 ? 1.0 : 0.0);
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ uncertainty-aware frames
int mloam_set_uncertainty(mloam_ctx_t *h, int with_ua, const double *ext_cov36, const double *cov_meas9, double trace_threshold) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (with_ua && (!ext_cov36 || !cov_meas9)) return MLOAM_E_INVALID;
  c->with_ua = with_ua ? 1 : 0;
  if (!with_ua) return MLOAM_OK;
  const int n_lasers = (c->n_lidars > 1 || c->lidar_merge) ? c->n_lidars : 1;
  for (int l = 0; l < MLOAM_MAX_LIDARS; l++)
    for (int k = 0; k < 36; k++) c->ua_ext_cov[l][k] = l < n_lasers ? ext_cov36[36 * l + k] : 0.0;
  memcpy(c->ua_cov_meas, cov_meas9, sizeof(c->ua_cov_meas));
  c->ua_trace_threshold = trace_threshold;
  return MLOAM_OK;
}

int mloam_pose_covariance(mloam_ctx_t *h, double *cov36) {
  if (!h || !cov36) return MLOAM_E_INVALID;
  memcpy(cov36, h->c.pose_cov36, sizeof(h->c.pose_cov36));
  return MLOAM_OK;
}

int mloam_frame_scan(mloam_ctx_t *h, mloam_point_t *h_surf, float *h_surf_cov6, int cap_surf, int *n_surf, mloam_point_t *h_corner,
                     float *h_corner_cov6, int cap_corner, int *n_corner) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->last_scan_valid) return fail(c, MLOAM_E_STATE, "frame_scan: no mloam_frame / mloam_frame_device call has run since the last reset");
  cudaSetDevice(c->device);
  const ScanRef &S = c->last_scan;
  cudaStream_t st = c->stream;
  int *hc = c->pinned->counts;
  hc[0] = S.n_surf, hc[1] = S.n_corner;
  if (S.d_n_surf) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, S.d_n_surf, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (S.d_n_corner) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc + 1, S.d_n_corner, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  const int ns = hc[0] < S.n_surf ? hc[0] : S.n_surf, nc = hc[1] < S.n_corner ? hc[1] : S.n_corner;
  if (n_surf) *n_surf = ns;
  if (n_corner) *n_corner = nc;
  if ((h_surf || h_surf_cov6) && ns > cap_surf) return fail(c, MLOAM_E_INVALID, "frame_scan: surf capacity too small");
  if ((h_corner || h_corner_cov6) && nc > cap_corner) return fail(c, MLOAM_E_INVALID, "frame_scan: corner capacity too small");
  const float4 *pts[2] = {S.surf, S.corner};
  const float *cov[2] = {S.cov6_surf, S.cov6_corner};
  mloam_point_t *hp[2] = {h_surf, h_corner};
  float *hcv[2] = {h_surf_cov6, h_corner_cov6};
  const int cnt[2] = {ns, nc};
  for (int t = 0; t < 2; t++) {
    if (cnt[t] <= 0) continue;
    if (hp[t]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hp[t], pts[t], sizeof(float4) * (size_t)cnt[t], cudaMemcpyDeviceToHost, st));
    if (hcv[t]) {
      if (cov[t]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(hcv[t], cov[t], sizeof(float) * 6 * (size_t)cnt[t], cudaMemcpyDeviceToHost, st));
      else memset(hcv[t], 0, sizeof(float) * 6 * (size_t)cnt[t]);  // with_ua = false: PointIWithCov(point, Zero) (:378-386)
    }
  }
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

int mloam_set_extrinsic(mloam_ctx_t *h, const double *ext7) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  c->has_ext = ext7 != nullptr;
  c->prefetched.valid = false;
  for (int k = 0; k < 7; k++) c->ext[k] = ext7 ? ext7[k] : (k == 6 ? 1.0 : 0.0);
  return MLOAM_OK;
}

}  // extern "C"
