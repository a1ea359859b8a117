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
#include "lm.cuh"

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
// captured into a CUDA graph); scan2map_finish() waits and unpacks.  o->ran: the map-size gate passed and the solve is enqueued;
// o->gf_evaluated: gd_float evaluates the full Hessian.  want_cov: also H^-1 at the returned pose (with_ua frame, mloam_scan2map_ua).
int scan2map_enqueue(Ctx *c, const ScanRef &S, const double *pose_init7, bool want_cov, Ctx::FrameOutcome *o) {
  const mloam_params_t &P = c->params;
  o->ran = 0, o->gf_evaluated = false;
  const MapStorage &MS = c->maps[MLOAM_MAP_SURF], &MC = c->maps[MLOAM_MAP_CORNER];
  if (!MS.built || !MC.built) return fail(c, MLOAM_E_STATE, "scan2map: build MLOAM_MAP_SURF and MLOAM_MAP_CORNER first");
  if (!((MS.m > 50) && (MC.m > 10))) return MLOAM_OK;  // lidar_mapper_keyframe.cpp:429 ("Map surf num is not enough")
  o->ran = 1;
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
  // programmatic dependent launch along the chain (launch_chain); the event scopes of stage profiling sit between the kernels, and
  // multi-GPU keeps its NCCL calls and peer-memory flags between ordinary launches
  const bool pdl = c->use_pdl && !c->prof_on && !c->nccl_comm && !c->p2p_on;
  first.pdl = iter.pdl = pdl;
  rc = lm_init_state(c, pose_init7, P.max_inner, 0, d_spec, pdl);
  if (rc) return rc;
  c->lin_trace_n = 0;  // MLOAM_LIN_TRACE: this solve's evaluations at x take the trace slots from 0 on
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
    return match_pair_device(c, jobs, 2, d_pose, cfg, defer_fit ? &pending : nullptr, spec ? &d_spec->sel : nullptr, pdl);
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
      // gd_float: the ratio is read on the device; an evaluation frame's first iteration makes both sets' rows, evaluates the full
      // Hessian over them (which sets that ratio, :456-495) and only then selects
      const double *d_ratio = c->cfg.gf_float_on ? &c->gf_float.as<GfFloatDev>()->st.ratio_cur : nullptr;
      const bool eval = c->cfg.gf_float_on && c->gf_float_eval && outer == 0;
      auto select = [&](int t, int phase) {
        if (sets[t].n <= 0) return MLOAM_OK;
        return gf_select_set_device(c, t, sets[t], d_pose, sinfo, P.gf_method, (double)P.gf_ratio,
                                    (unsigned long long)P.gf_seed + 2ull * (unsigned long long)outer + (unsigned long long)t, &mask[t], d_ratio,
                                    phase);
      };
      if (eval) {
        rc = select(0, 1);
        if (rc == MLOAM_OK) rc = select(1, 1);
        if (rc == MLOAM_OK) rc = gf_full_hessian_device(c, sets);
        if (rc) return rc;
        o->gf_evaluated = true;
      }
      const int phase = eval ? 2 : 3;
      // the two selections are independent single-CTA chains: corner on the side stream next to surf (also inside a captured graph)
      const bool fork_gf = !c->prof_on && sets[0].n > 0 && sets[1].n > 0;
      rc = on_branch(c, c->br_scan, fork_gf, [&] { return select(0, phase); });
      if (rc == MLOAM_OK) rc = select(1, phase);
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
      // fork: {evaluation at the candidate + acceptance} on the side branch || {matcher of iteration outer + 1 at the published
      // candidate} on the main stream, right behind k_linearize, so that the critical path k_linearize -> k_match_knn -> k_linearize
      // is one stream (programmatic edges with pdl).  The branches share only read-only inputs: the matcher writes the spare half of
      // the lists, the changed and heavy flags; the evaluation writes LMState and the partials.  With stage profiling on they stay
      // serial, like the other forks.
      const bool fork = !c->prof_on;
      rc = on_branch(c, c->br_scan, fork, [&] { return eval_candidate_device(c, sets, 2, sinfo, P.huber_a, P.eig_thre, pdl); });
      if (rc) return rc;
      rc = match(outer + 1);
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
    rc = pose_cov_device(c, pdl);
    if (rc) return rc;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->pinned->pose_cov, c->pose_cov.p, 36 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    stamp(c, "pose covariance");
  }
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hs, st, sizeof(LMState), cudaMemcpyDeviceToHost, c->stream));
  if (c->cfg.gf_float_on)  // the report (mloam_gf_float_report) lands with the frame's results
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(&c->pinned->gf_float, &c->gf_float.as<GfFloatDev>()->st, sizeof(GfFloatState), cudaMemcpyDeviceToHost, c->stream));
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
  if (c->cfg.gf_float_on) c->gf_float_host = c->pinned->gf_float;
  if (!S.d_n_surf) h_cnt[0] = S.n_surf;
  if (!S.d_n_corner) h_cnt[1] = S.n_corner;
  for (int k = 0; k < 7; k++) pose_out7[k] = hs->x[k];
  if (want_cov && hs->termination != kTermBarrierTimeout && hs->termination != kTermExchangeFailed) memcpy(c->pose_cov36, c->pinned->pose_cov, sizeof(c->pose_cov36));
  if (hs->termination == kTermExchangeFailed) {  // the peer-memory exchange timed out or the ranks lost lock-step: the summed state is not trustworthy
    for (int k = 0; k < 7; k++) pose_out7[k] = pose_init7[k];
    if (stats) stats->ran = 1, stats->termination = kTermExchangeFailed;
    return fail(c, MLOAM_E_NCCL, "scan2map: peer-memory exchange failed (a rank did not arrive or the ranks lost lock-step); "
                                  "call mloam_comm_p2p_reset on every rank behind a barrier");
  }
  if (hs->termination == kTermBarrierTimeout) {  // k_linearize's grid barrier gave up: a block of the grid never became resident within ~2 s
    for (int k = 0; k < 7; k++) pose_out7[k] = pose_init7[k];
    if (stats) stats->ran = 1, stats->termination = kTermBarrierTimeout;
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

// gd_float: what every solve call does first.  frame_cnt advances before the map gate (lidar_mapper_keyframe.cpp:1059, :429); the 10th,
// 20th, ... call evaluates if it passes the gate (scan2map_enqueue).
int gf_float_begin(Ctx *c) {
  if (!c->cfg.gf_float_on) return MLOAM_OK;
  if (c->params.gf_method != 3) return fail(c, MLOAM_E_STATE, "gd_float is on (mloam_set_gf_float) and params.gf_method is no longer 3");
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "gd_float (mloam_set_gf_float) is single-GPU only; detach the communicator or turn it off");
  c->gf_float_frames++;
  c->gf_float_eval = c->gf_float_frames % 10 == 0;
  c->gf_float_evaluated = false;
  c->gf_float_reported = true;
  return MLOAM_OK;
}

int scan2map_run(Ctx *c, const ScanRef &S, const double *pose_init7, bool want_cov, double *pose_out7, mloam_solve_stats_t *stats) {
  c->reg_valid = false;  // a scan has no sweep: nothing to register
  int rc = gf_float_begin(c);
  if (rc) return rc;
  Ctx::FrameOutcome o;
  rc = scan2map_enqueue(c, S, pose_init7, want_cov, &o);
  c->gf_float_evaluated = o.gf_evaluated;
  if (rc) return rc;
  return scan2map_finish(c, S, pose_init7, want_cov, o.ran, pose_out7, stats);
}

// Device buffers of one frame: feature sets of extractCloud + the down-sampled scans fed to matching.
struct FrameBufs {
  ExtractOut ex;
  float4 *corner_ds, *surf_ds;
  int *n_corner_ds, *n_surf_ds;  // device counts
  float4 *first;                 // the LiDARs' first points (ExtractOut::first) and their flags
  int *first_ok;
  int *off;                      // rig merge: per-LiDAR offsets of the less-sharp and less-flat features (lidar_offsets_device)
  // the registered clouds (reg_scans > 0): the ring-ordered sweep the features were extracted from, and [0] its size on the device (a
  // raw sweep's projection count), [16 ..] its ScanInfo starts
  float4 *reg_sweep = nullptr;
  int *reg_meta = nullptr;
};
// reg_scans: the sweep's ring count when the half also keeps the sweep for the registered clouds; its regions come last, so the other
// regions lie where they lie without them
int frame_bufs(Ctx *c, int n, FrameBufs *F, int parity = 0, int reg_scans = 0) {
  const size_t N1 = (size_t)n + 16;
  MLOAM_CUDA_OK(c, carve(parity ? c->frame_alt : c->frame_main, [&](Carve &cv) {
    F->ex.sharp = cv.take<float4>(N1), F->ex.less_sharp = cv.take<float4>(N1), F->ex.flat = cv.take<float4>(N1);
    F->ex.less_flat = cv.take<float4>(N1), F->corner_ds = cv.take<float4>(N1), F->surf_ds = cv.take<float4>(N1);
    F->ex.counts = cv.take<int>(16);  // [0..3]
    F->first = cv.take<float4>(MLOAM_MAX_LIDARS), F->first_ok = cv.take<int>(MLOAM_MAX_LIDARS);
    F->off = cv.take<int>(2 * (MLOAM_MAX_LIDARS + 1));
    if (reg_scans > 0) F->reg_sweep = cv.take<float4>(N1), F->reg_meta = cv.take<int>(16 + (size_t)reg_scans);
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

void mloam::stage_pose(Ctx *c, const double *pose7) { memcpy(c->pinned->pose, pose7, sizeof(c->pinned->pose)); }

namespace {

// capacity of a frame's less-sharp features: <= 20 picks x 6 sectors per ring
int less_sharp_cap(int n, int n_scans) { return n < 120 * n_scans ? n : 120 * n_scans; }

// The poses the look-ahead branch undistorts the announced sweep with (mloam_frame_set_next_undistort), or nullptr: the branch does not
// run, or it extracts only and the undistortion, merge and scan filters wait for the call that takes the sweep
const UndistPoses *undist_ahead(const Ctx *c) {
  return c->cfg.undist_on && c->next.set && c->next.undist.n > 0 && c->use_lookahead && !c->prof_on ? &c->next.undist : nullptr;
}

// ---- what depends on a sweep's kind: one switch per decision (pcd.cu: pcd_frame_stage, pcd_frame_land, pcd_frame_refusal)
// Whether sweep sw is the announced sweep a: the same kind, caller pointer and sizes, and a host frame takes a host announcement only (a
// device frame may take either).
bool same_sweep(const Sweep &a, const Sweep &sw) {
  if (a.kind != sw.kind || a.key != sw.key || a.n != sw.n || a.n_scans != sw.n_scans || !(a.host || !sw.host)) return false;
  if (std::memcmp(&a.L, &sw.L, sizeof(RigLayout)) != 0) return false;  // a raw-like sweep: the same per-LiDAR counts
  switch (sw.kind) {
    case SweepKind::ring:
    case SweepKind::raw: return true;
    case SweepKind::msg: return std::memcmp(&a.wire, &sw.wire, sizeof(WireMsgs)) == 0;  // the same messages (pointers, shapes) and layouts
    case SweepKind::pcd: return std::memcmp(&a.pcdf, &sw.pcdf, sizeof(PcdFiles)) == 0;  // the same bodies (pointers, sizes, POINTS, tokens)
  }
  return false;
}

// Point the device side of host sweep *sw into B and, with `upload`, copy the sweep there on st.  A ring sweep's ScanInfo goes through
// the pinned rows pin: an async copy from pageable memory would block the host behind the sweep's copy.
int sweep_to_device(Ctx *c, DevBuf &B, Sweep *sw, bool upload, int (*pin)[MLOAM_MAX_RINGS], cudaStream_t st) {
  switch (sw->kind) {
    case SweepKind::ring:
    case SweepKind::raw: {  // the points, then room for the ScanInfo, which a raw sweep has not (the front end makes it)
      SweepIn D;
      int rc = sweep_bufs(c, B, sw->n, sw->n_scans, &D);
      if (rc) return rc;
      sw->cloud = D.cloud;
      const bool ring = sw->kind == SweepKind::ring;
      if (ring) sw->scan_start = D.scan_start, sw->scan_end = D.scan_end;
      if (!upload) return MLOAM_OK;
      const int ns = sw->n_scans;
      if (ring) {
        std::memcpy(pin[0], sw->h_scan_start, sizeof(int) * ns), std::memcpy(pin[1], sw->h_scan_end, sizeof(int) * ns);
        MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.scan_start, pin[0], sizeof(int) * ns, cudaMemcpyHostToDevice, st));
        MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.scan_end, pin[1], sizeof(int) * ns, cudaMemcpyHostToDevice, st));
      }
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(D.cloud, sw->key, sizeof(float4) * (size_t)sw->n, cudaMemcpyHostToDevice, st));
      return MLOAM_OK;
    }
    case SweepKind::msg: return wire_upload(c, B, sw, upload, st);
    case SweepKind::pcd: return pcd_upload(c, B, sw, upload, st);
  }
  return MLOAM_E_INVALID;
}

// The points on the device that extraction reads (a ring sweep) or the front end reads (a raw-like one), on c->stream: the caller's or the
// staged cloud, or the messages unpacked / the PCD bodies decoded into wire_out.  The decode reads the bodies' byte sizes staged for half
// `parity` (pcd_frame_stage).
int sweep_points(Ctx *c, const Sweep &sw, int parity, const float4 **out) {
  switch (sw.kind) {
    case SweepKind::ring:
    case SweepKind::raw: *out = sw.cloud; return MLOAM_OK;
    case SweepKind::msg:
    case SweepKind::pcd: {
      MLOAM_CUDA_OK(c, c->wire_out.reserve(sizeof(float4) * ((size_t)sw.n + 1)));
      float4 *w = c->wire_out.as<float4>();
      *out = w;
      return sw.kind == SweepKind::msg ? wire_unpack_device(c, sw, w) : pcd_decode_half(c, sw, parity, w);
    }
  }
  return MLOAM_E_INVALID;
}

// A sweep's part of the frame graph key (FrameKey)
struct SweepKey {
  const void *ptr[4];  // the sweep on the device (cloud, scan_start, scan_end) and the caller's pointer
  FrontEnd front;      // a raw-like sweep: kernel arguments of the captured front end
  RigLayout L;
  int n, n_scans;
};

// FNV-1a over 8-byte words: the key is built on the frame's host critical path
inline unsigned long long fnv(unsigned long long h, unsigned long long w) { return (h ^ w) * 1099511628211ull; }
unsigned long long fnv_words(unsigned long long h, const void *p, size_t bytes) {
  unsigned long long w;
  for (size_t i = 0; i < bytes; i += 8) memcpy(&w, static_cast<const char *>(p) + i, 8), h = fnv(h, w);
  return h;
}

// Sweep x's part of the frame graph key: *k, and what a message or PCD sweep's capture holds besides, mixed into h before the rest of the
// key — only for such a sweep, so that a context that never takes one keeps the keys it had without them — tagged by kind and by slot
// (next: the announced sweep)
unsigned long long sweep_key(const Sweep &x, const FrontEnd &fe, bool next, SweepKey *k, unsigned long long h) {
  k->ptr[0] = x.cloud, k->ptr[1] = x.scan_start, k->ptr[2] = x.scan_end, k->ptr[3] = x.key;
  k->n = x.n, k->n_scans = x.n_scans;
  if (x.raw_like()) k->front = fe, k->L = x.L;
  switch (x.kind) {
    case SweepKind::ring:
    case SweepKind::raw: return h;
    case SweepKind::msg:  // the messages, layouts and staging are kernel arguments of the captured unpack
      h = fnv(h, next ? 8ull : 4ull);
      h = fnv(h, (unsigned long long)reinterpret_cast<uintptr_t>(x.bytes));
      return fnv_words(h, &x.wire, sizeof(WireMsgs));
    case SweepKind::pcd:
      // the decode's kernel arguments — the staging or the device bodies, POINTS, tokens and token indices — but not the byte sizes, which
      // are staged (pcd_frame_stage), so that files of other sizes replay the same graph.  A host sweep is copied into the staging whatever
      // the caller's buffer: its pointer is no kernel argument (a dataset replay reads every file into a new place).
      if (x.host) k->ptr[3] = nullptr;
      h = fnv(h, next ? 32ull : 16ull);
      h = fnv(h, (unsigned long long)reinterpret_cast<uintptr_t>(x.host ? x.bytes : nullptr));
      for (int l = 0; l < x.L.n_lidars; l++) {
        const mloam_pcd_t &p = x.pcdf.body[l];
        h = fnv(h, (unsigned long long)reinterpret_cast<uintptr_t>(x.host ? nullptr : p.data));
        h = fnv(h, (unsigned long long)(unsigned)p.points << 32 | (unsigned)p.tokens);
        h = fnv(h, (unsigned long long)(unsigned)p.index[0] << 40 ^ (unsigned long long)(unsigned)p.index[1] << 20 ^ (unsigned)p.index[2]);
      }
      return h;
  }
  return h;
}

// One mloam_frame* call as frame_call hands it on.  have: the previous frame's look-ahead made the sweep's features, in half `parity`;
// else they are extracted now into that half.  take_undist: they are complete although the undistortion is on (the look-ahead ran it
// with the poses of mloam_frame_set_next_undistort).  The submaps are on the device.
struct FrameCall {
  Sweep sw;
  bool have;
  int parity;
  const float4 *surf_map, *corner_map;
  int n_surf_map, n_corner_map, rebuild_maps;
  const double *pose_init7;
  bool take_undist;
};

// The pinned inputs of a frame (PinnedBlock), from Ctx::cfg and the pose guess: written once before the frame is enqueued and before
// every replay of its graph, whose captured copies read them at execution time.  The stages only copy them.  The undistortion's poses
// are staged per half: this sweep's into its half, the announced sweep's into the other one when the look-ahead undistorts it.
void stage_frame_inputs(Ctx *c, const FrameCall &fc) {
  const FrameCfg &f = c->cfg;
  stage_pose(c, fc.pose_init7);
  if (f.rig_merge()) {
    for (int l = 0; l < f.n_lidars; l++) pose_mat12(f.lidar_ext[l], c->pinned->rig[l]);
  } else if (f.has_ext) {
    memcpy(c->pinned->ext, f.ext, sizeof(c->pinned->ext));
  }
  if (f.with_ua) ua_stage_host(c);
  if (f.outlier_on) stage_outlier(c);
  if (f.undist_on) stage_undistort(c, fc.parity, undist_ahead(c));
  if (f.gf_float_on) stage_gf_float(c);
  if (!fc.have) pcd_frame_stage(c, fc.sw, fc.parity);  // a sweep the look-ahead made is not read again
  if (c->next.set && c->use_lookahead && !c->prof_on) pcd_frame_stage(c, c->next.sw, fc.parity ^ 1);
}

// Whether the look-ahead of the previous frame made the features of sw.  With the undistortion on they are the extraction only, or
// complete when the look-ahead undistorted with the very bits this call undistorts with (Ctx::undist_pose7, set by frame_call).
bool frame_has_prefetched(const Ctx *c, const Sweep &sw) {
  const Ctx::Features &f = c->prefetched;
  UndistPoses call;
  if (c->cfg.undist_on && f.undist.n > 0) call.n = c->undist_n, std::memcpy(call.pose7, c->undist_pose7, sizeof(double) * 7 * (size_t)call.n);
  const bool undist_ok = !c->cfg.undist_on ? !f.extract_only && f.undist.n == 0 : f.extract_only || (f.undist.n > 0 && f.undist.same_bits(call));
  return f.valid && c->use_lookahead && !c->prof_on && same_sweep(f.sw, sw) && undist_ok && (f.registered || !c->cfg.reg_on);
}

// extractCloud of sweep sw on c->stream into half `parity` of the feature double buffer (*F), with the LiDARs' first points and, for the
// rig merge, each LiDAR's feature offsets — everything that reads Ctx::extract_work.  A raw-like sweep's points (sweep_points) go through
// the front end (removeNaN + calTimestamp + projection, Ctx::front) first, which makes the ring-ordered sweep and its ScanInfo on the
// device; extraction takes them with the raw size n as capacity (no count comes back to the host).
int extract_enqueue(Ctx *c, const Sweep &sw, int parity, FrameBufs *F_out) {
  const int n = sw.n, n_scans = sw.n_scans;
  const FrameCfg &cfg = c->cfg;
  FrameBufs F;
  int rc = frame_bufs(c, n, &F, parity, cfg.reg_on ? n_scans : 0);
  if (rc) return rc;
  const float4 *d_cloud;
  rc = sweep_points(c, sw, parity, &d_cloud);
  if (rc) return rc;
  const int *d_scan_start = sw.scan_start, *d_scan_end = sw.scan_end;
  if (sw.raw_like()) {
    const FrontEnd &fe = cfg.front;
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
    if (cfg.reg_on) MLOAM_CUDA_OK(c, cudaMemcpyAsync(F.reg_meta, n_proj, sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
  }
  if (cfg.reg_on) {  // the registered clouds need the sweep when its frame ends: by then next_in, front_out or the caller's buffer may be reused
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(F.reg_sweep, d_cloud, sizeof(float4) * (size_t)n, cudaMemcpyDeviceToDevice, c->stream));
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(F.reg_meta + 16, d_scan_start, sizeof(int) * (size_t)n_scans, cudaMemcpyDeviceToDevice, c->stream));
  }
  // every frame's extraction records each LiDAR's first point, so that features extracted ahead serve a frame with the outlier cloud on
  const int n_parts = cfg.n_parts();
  if (n_scans % n_parts == 0) F.ex.first = F.first, F.ex.first_ok = F.first_ok, F.ex.first_rings = n_scans / n_parts;  // else the merge
                                                                                                                       // below rejects it
  rc = extract_device(c, d_cloud, n, d_scan_start, d_scan_end, n_scans, F.ex, nullptr, nullptr);
  if (rc) return rc;
  if (cfg.rig_merge()) {  // the merge below may run later (undistortion on): each LiDAR's offsets are kept with the sweep's features
    if (n_scans % n_parts != 0) return fail(c, MLOAM_E_INVALID, "frame: n_scans must be n_lidars x rings per LiDAR");
    rc = lidar_offsets_device(c, n_parts, n_scans / n_parts, F.off);
    if (rc) return rc;
  }
  stamp(c, "extract");
  *F_out = F;
  return MLOAM_OK;
}

// [undistortion] + (multi-LiDAR merge | base-frame transform) + downsampleCurrentScan of the features extract_enqueue left in F (half
// `parity`), on c->stream; the corner filter forks onto branch `side`.
int scan_enqueue(Ctx *c, const Sweep &sw, const FrameBufs &F, int parity, const Branch &side, ScanRef *S_out) {
  const mloam_params_t &P = c->params;
  const FrameCfg &cfg = c->cfg;
  const int n = sw.n, n_scans = sw.n_scans;
  int rc;
  const int less_cap = less_sharp_cap(n, n_scans);
  DevCtl *ctl = c->ctl.as<DevCtl>();
  if (cfg.undist_on) {  // undistortMeasurements (estimator.cpp:376-408): each LiDAR's less-* features in its own frame, before the merge
    rc = undistort_stage(c, parity, F.ex, less_cap, n, cfg.rig_merge() ? F.off : nullptr, cfg.n_parts());
    if (rc) return rc;
    stamp(c, "undistort");
  }
  if (cfg.rig_merge()) {
    // batched sweeps of several LiDARs: features of LiDAR l go to the base frame with its extrinsic, intensity = l
    // (transformCloudFeature, visualization.cpp:40-52), LiDAR after LiDAR as pubPointCloud's `+=` (:93-104)
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(ctl->rig, c->pinned->rig, sizeof(float) * 12 * cfg.n_lidars, cudaMemcpyHostToDevice, c->stream));
    rc = merge_lidars_device(c, F.ex, less_cap, n, cfg.n_lidars, &ctl->rig[0][0], F.off);
    if (rc) return rc;
  } else if (cfg.has_ext) {  // features are handed to the mapper in the base frame
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
  S.first = F.ex.first, S.first_ok = F.ex.first_ok;
  *S_out = S;
  return MLOAM_OK;
}

// The features of sweep sw, all steps: extract_enqueue + scan_enqueue
int features_enqueue(Ctx *c, const Sweep &sw, int parity, const Branch &side, ScanRef *S_out) {
  FrameBufs F;
  int rc = extract_enqueue(c, sw, parity, &F);
  if (rc) return rc;
  return scan_enqueue(c, sw, F, parity, side, S_out);
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

// pubPointCloud of sweep sw, whose features and copy are in half `parity`, on c->stream after the solve: k_registered at pose_wmap_curr,
// LMState::x when the solve ran (ran), else the staged initial pose (the map gate keeps it, lidar_mapper_keyframe.cpp:429, :634-638)
int registered_enqueue(Ctx *c, const Sweep &sw, int parity, int ran, RegOut *out) {
  FrameBufs F;
  int rc = frame_bufs(c, sw.n, &F, parity, sw.n_scans);  // the layout the extraction carved: nothing moves or grows
  if (rc) return rc;
  DevCtl *ctl = c->ctl.as<DevCtl>();
  const double *d_pose;
  if (ran) {
    d_pose = c->lm_state.as<LMState>()->x;
  } else {
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(ctl->pose, c->pinned->pose, 7 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    d_pose = ctl->pose;
  }
  const int less_cap = less_sharp_cap(sw.n, sw.n_scans);
  RegArgs a{};
  a.sweep = F.reg_sweep, a.n_sweep = sw.n, a.d_n_sweep = sw.raw_like() ? F.reg_meta : nullptr, a.scan_start = F.reg_meta + 16;
  a.n_parts = c->cfg.n_parts(), a.rings_per_lidar = sw.n_scans / a.n_parts;
  a.to_base = c->cfg.rig_merge() ? 1 : (c->cfg.has_ext ? 2 : 0), a.rig = &ctl->rig[0][0], a.ext = ctl->ext;  // as scan_enqueue copied them
  a.undist = c->cfg.undist_on ? c->undist.as<UndistStage>() + parity : nullptr;  // undistort_stage's configuration of this sweep's half
  if (c->cfg.outlier_on) a.first = F.first, a.first_ok = F.first_ok, a.outlier = c->outlier.as<OutlierStage>();  // outlier_stage's
  a.less_flat = F.ex.less_flat, a.less_sharp = F.ex.less_sharp, a.cap_flat = sw.n, a.cap_sharp = less_cap;
  a.n_flat = F.ex.counts + 3, a.n_sharp = F.ex.counts + 1, a.pose = d_pose;
  rc = registered_layout(c, sw.n, sw.n, less_cap, out);
  if (rc == MLOAM_OK) rc = registered_stage(c, a, *out);
  if (rc) return rc;
  stamp(c, "registered");
  return MLOAM_OK;
}

// The frame's inputs staged, then on c->stream: the features of the sweep — ready from the look-ahead when f.have, else extracted now
// into half f.parity —, the look-ahead of the announced sweep, the map builds (f.rebuild_maps) and the solve.  Writes nothing of the
// context's frame state: the host-side results go to *o for frame_commit.
int frame_enqueue(Ctx *c, const FrameCall &f, Ctx::FrameOutcome *o) {
  const FrameCfg &cfg = c->cfg;
  const Sweep &sw = f.sw;
  *o = Ctx::FrameOutcome{};
  stage_frame_inputs(c, f);
  // lidar_mapper_keyframe.cpp:433-434 (every frame in the reference).  The two submap builds do not depend on the sweep: they run on a
  // forked side stream, concurrently with extraction + scan down-sampling, and join right before matching (also inside a captured graph).
  // With stage profiling on the branch stays on the main stream so that per-stage event times do not overlap.
  const bool fork_maps = f.rebuild_maps && !c->prof_on;
  int rc;
  if (f.rebuild_maps) {
    rc = on_branch(c, c->br_maps, fork_maps, [&] {
      int r = c->maps_pending ? wait_uploads(c, c->ev_maps, fork_maps) : MLOAM_OK;
      if (r == MLOAM_OK) r = map_build_device(c, MLOAM_MAP_SURF, f.surf_map, f.n_surf_map, pick_cell(c, 0.f));
      if (r == MLOAM_OK) r = map_build_device(c, MLOAM_MAP_CORNER, f.corner_map, f.n_corner_map, pick_cell(c, 0.f));
      return r;
    });
    if (rc) return rc;
  }
  c->stamp_n = 0;
  stamp(c, "start");
  ScanRef &S = o->S;
  const Ctx::Features &pf = c->prefetched;  // the look-ahead's features of this sweep, when f.have
  if (f.have && !pf.extract_only) S = pf.S;
  if (!f.have) {
    rc = features_enqueue(c, sw, f.parity, c->br_scan, &S);
    if (rc) return rc;
  } else if (pf.extract_only) {  // undistortion on: the look-ahead extracted; this sweep's pose is known now
    FrameBufs F;
    rc = frame_bufs(c, sw.n, &F, f.parity, cfg.reg_on ? sw.n_scans : 0);
    F.ex.first = F.first, F.ex.first_ok = F.first_ok;  // recorded by the look-ahead's extraction (extract_enqueue)
    if (rc == MLOAM_OK) rc = scan_enqueue(c, sw, F, f.parity, c->br_scan, &S);
    if (rc) return rc;
  }
  // look-ahead: the announced next sweep goes through the same steps on br_ahead into the other half while this frame is matched
  // and solved (it reuses Ctx::extract_work, voxel_corner and voxel_surf of the block above, hence the fork AFTER it).  With the
  // undistortion on, the branch needs the next sweep's poses: announced with it (mloam_frame_set_next_undistort), it runs every step
  // with them, staged in the other half's UndistStage; else they come with the next call, the branch extracts only (extract_work),
  // and that call runs undistortion, merge and the scan filters on the main stream before it forks its own look-ahead.
  Ctx::Features &nf = o->next;
  if (c->next.set && c->use_lookahead && !c->prof_on) {
    const Sweep &nx = c->next.sw;
    const UndistPoses *nx_undist = undist_ahead(c);
    const bool extract_only = cfg.undist_on && !nx_undist;
    c->stamp_mute = true;
    rc = on_branch(c, c->br_ahead, true, [&] {
      int r = c->next_pending ? wait_uploads(c, c->ev_next, true) : MLOAM_OK;  // mloam_frame copied the next sweep on br_ahead
      if (r == MLOAM_OK && extract_only) {
        FrameBufs F;
        r = extract_enqueue(c, nx, f.parity ^ 1, &F);
      } else if (r == MLOAM_OK) {
        r = features_enqueue(c, nx, f.parity ^ 1, c->br_ahead_scan, &nf.S);
      }
      return r;
    });
    c->stamp_mute = false;
    if (rc) return rc;
    nf.valid = true, nf.parity = f.parity ^ 1, nf.sw = nx, nf.extract_only = extract_only, nf.registered = cfg.reg_on;
    if (nx_undist) nf.undist = *nx_undist;
  }
  stamp(c, f.have ? "features (prefetched)" : "extract + voxel");
  const UaStage *d_ua = nullptr;
  if (cfg.with_ua) {  // downsampleCurrentScan's per-point uncertainty + trace gate: on the main stream with the covariances of THIS call
    rc = ua_scan_stage(c, &S, &d_ua);
    if (rc) return rc;
    stamp(c, "uncertainty + gate");
  }
  if (cfg.outlier_on) {  // the outlier cloud (:366-418): the recorded first points -> base frame -> filter -> the same gate, one launch
    rc = outlier_stage(c, &S, d_ua);
    if (rc) return rc;
    stamp(c, "outlier cloud");
  }
  if (fork_maps) {  // join the map-build branch
    MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, c->br_maps.join, 0));
    stamp(c, "map build join");
  }
  rc = scan2map_enqueue(c, S, f.pose_init7, cfg.with_ua != 0, o);
  if (rc) return rc;
  if (cfg.reg_on) {  // pubPointCloud (:690-714): after the solve, next to the look-ahead's tail
    rc = registered_enqueue(c, sw, f.parity, o->ran, &o->reg);
    if (rc) return rc;
  }
  if (nf.valid) {  // the frame ends when both branches have: the features of the next sweep are complete when this call returns
    MLOAM_CUDA_OK(c, cudaStreamWaitEvent(c->stream, c->br_ahead.join, 0));
    stamp(c, "look-ahead join");
  }
  return pcd_frame_land(c, sw);
}

// A frame's outcome applied to the context, on the stream, capture and replay paths alike
void frame_commit(Ctx *c, int parity, const Ctx::FrameOutcome &o) {
  c->frame_parity = parity ^ 1;
  c->prefetched = o.next;
  // the poses the look-ahead undistorted with are staged, not captured: a replay's are the ones announced for it (same key: announced)
  if (c->prefetched.undist.n > 0) c->prefetched.undist = c->next.undist;
  c->last_scan = o.S, c->last_scan_valid = true;
  c->reg_last = o.reg;
  c->gf_float_evaluated = o.gf_evaluated;
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

// Edges of a captured graph that launch_chain made programmatic (-1: the edges could not be read)
int count_programmatic_edges(cudaGraph_t g) {
  size_t n = 0;
  if (cudaGraphGetEdges_v2(g, nullptr, nullptr, nullptr, &n) != cudaSuccess) return -1;
  std::vector<cudaGraphNode_t> from(n), to(n);
  std::vector<cudaGraphEdgeData> data(n);
  if (n && cudaGraphGetEdges_v2(g, from.data(), to.data(), data.data(), &n) != cudaSuccess) return -1;
  int k = 0;
  for (size_t i = 0; i < n; i++) k += data[i].type == cudaGraphDependencyTypeProgrammatic ? 1 : 0;
  return k;
}

// Everything a frame graph depends on besides its staged inputs (stage_frame_inputs), hashed whole into the graph cache's key.  What a
// frame does not use is zero, so two frames share a key exactly when they enqueue the same graph.
struct FrameKey {
  SweepKey sweep, next;  // the sweep, and the announced one (look-ahead)
  const void *maps[2];   // the submaps of an in-frame rebuild
  cudaStream_t stream;
  mloam_params_t params;
  double ext[7], lidar_ext[MLOAM_MAX_LIDARS][7];  // the rig's first n_lidars
  float cells[2];              // the auto cell edges of an in-frame rebuild: kernel arguments of the captured builds
  // gate: the map-size gate (scan2map_enqueue) is decided on the host at capture: with maps built outside the frame (mloam_map_build*,
  // mloam_submap_assemble, mloam_keyframe_submap) a graph captured while it failed must not be replayed once it passes, and back
  int raw, n_surf_map, n_corner_map, rebuild_maps, maps_pending, gate, has_ext, n_lidars, lidar_merge;
  // the stages' launches and the look-ahead's split with the undistortion on (their staged values are not part of the key)
  int with_ua, outlier_on, undist_on, undist_n, reg_on, gf_float_on, gf_eval;
  // the look-ahead: which half holds this sweep's features (or that they are extracted now), and the announced next sweep
  int have, parity, ahead, next_host, next_pending, stamp_on;
};
static_assert(sizeof(SweepKey) == 4 * sizeof(void *) + sizeof(FrontEnd) + sizeof(RigLayout) + 2 * sizeof(int) &&
                  sizeof(FrameKey) == 2 * sizeof(SweepKey) + 3 * sizeof(void *) + sizeof(mloam_params_t) +
                                          sizeof(double) * 7 * (1 + MLOAM_MAX_LIDARS) + 2 * sizeof(float) + 22 * sizeof(int),
              "hashed whole in 8-byte words: no padding");

unsigned long long frame_key(Ctx *c, const FrameCall &f) {
  const FrameCfg &cfg = c->cfg;
  FrameKey k;
  memset(&k, 0, sizeof(k));
  unsigned long long h = 1469598103934665603ull;
  h = sweep_key(f.sw, cfg.front, false, &k.sweep, h);
  if (c->next.set && c->use_lookahead) {
    const Sweep &nx = c->next.sw;
    h = sweep_key(nx, cfg.front, true, &k.next, h);
    k.ahead = 1, k.next_host = nx.host, k.next_pending = c->next_pending;
  }
  k.maps[0] = f.surf_map, k.maps[1] = f.corner_map, k.stream = c->stream;
  memcpy(&k.params, &c->params, sizeof(k.params));
  memcpy(k.ext, cfg.ext, sizeof(k.ext));
  memcpy(k.lidar_ext, cfg.lidar_ext, sizeof(double) * 7 * (size_t)cfg.n_lidars);
  if (f.rebuild_maps && !(c->params.map_cell > 0.f)) {
    k.cells[0] = c->maps[MLOAM_MAP_SURF].auto_cell_pick(c->pinned, MLOAM_MAP_SURF);
    k.cells[1] = c->maps[MLOAM_MAP_CORNER].auto_cell_pick(c->pinned, MLOAM_MAP_CORNER);
  }
  k.raw = f.sw.raw_like(), k.n_surf_map = f.n_surf_map, k.n_corner_map = f.n_corner_map;
  k.rebuild_maps = f.rebuild_maps, k.maps_pending = c->maps_pending;
  const MapStorage &MS = c->maps[MLOAM_MAP_SURF], &MC = c->maps[MLOAM_MAP_CORNER];
  k.gate = !f.rebuild_maps && MS.built && MC.built && MS.m > 50 && MC.m > 10;
  k.has_ext = cfg.has_ext, k.n_lidars = cfg.n_lidars, k.lidar_merge = cfg.lidar_merge;
  k.with_ua = cfg.with_ua, k.outlier_on = cfg.outlier_on, k.reg_on = cfg.reg_on;
  k.undist_on = cfg.undist_on, k.undist_n = cfg.undist_on ? c->undist_n : 0;
  k.gf_float_on = cfg.gf_float_on, k.gf_eval = cfg.gf_float_on && c->gf_float_eval;  // an evaluation frame's extra launch
  k.have = f.have, k.parity = f.parity, k.stamp_on = c->stamp_on;
  h = fnv_words(h, &k, sizeof(k));
  // the undistortion in the look-ahead branch, and a call that takes a sweep undistorted there (mloam_frame_set_next_undistort): one
  // more word, only when either is on, so that the keys of a context that never announces poses are the ones it had without them
  const unsigned long long w = (undist_ahead(c) ? 1ull : 0ull) | (f.take_undist ? 2ull : 0ull);
  return w ? fnv(h, w) : h;
}

// The single-GPU stages at frame time: their setters refuse a multi-GPU context (multi_gpu), and this refuses a communicator attached
// after them.  raw: the sweep is raw, and the front end is single-GPU too.
int frame_single_gpu(Ctx *c, bool raw) {
  if (!c->nccl_comm) return MLOAM_OK;
  const FrameCfg &f = c->cfg;
  const char *msg =
      raw          ? "frame_raw: raw frames are single-GPU only; detach the communicator"
      : f.with_ua  ? "frame: uncertainty-aware frames (mloam_set_uncertainty) are single-GPU only; detach the communicator or set with_ua = 0"
      : f.outlier_on ? "frame: the outlier cloud (mloam_set_outlier) is single-GPU only; detach the communicator or set it to 0"
      : f.undist_on  ? "frame: the undistortion (mloam_set_distortion) is single-GPU only; detach the communicator or turn it off"
      : f.reg_on     ? "frame: the registered clouds (mloam_set_registered) are single-GPU only; detach the communicator or turn them off"
                     : nullptr;
  return msg ? fail(c, MLOAM_E_STATE, msg) : MLOAM_OK;
}

// One frame.  With max_inner == 1 the ~60 launches of a frame form a fixed sequence that depends on the host only through the staged
// inputs — it is captured once per frame_key into a CUDA graph and replayed: the first call with a new key runs on the stream (and
// performs every allocation), the second captures + instantiates, later ones replay.  Profiling, multi-GPU (NCCL on the stream) and
// max_inner > 1 (the host polls the LM done flag) use the plain stream path.
// A sweep the device refused (pcd_frame_refusal): the call returns its error and commits nothing (the look-ahead's features are dropped;
// the next frame extracts its sweep again)
int frame_refused(Ctx *c, const FrameCall &f, double *pose_out7, mloam_solve_stats_t *stats) {
  const int rc = pcd_frame_refusal(c, f.sw, f.parity);
  if (rc == MLOAM_OK) return rc;
  c->prefetched.valid = false;
  for (int k = 0; k < 7; k++) pose_out7[k] = f.pose_init7[k];
  if (stats) memset(stats, 0, sizeof(*stats));
  return rc;
}

int frame_run(Ctx *c, const FrameCall &f, double *pose_out7, mloam_solve_stats_t *stats) {
  int rc = frame_single_gpu(c, false);
  if (rc) return rc;
  const bool want_cov = c->cfg.with_ua != 0;
  c->last_scan_valid = false;
  c->frame_from_graph = false;
  rc = gf_float_begin(c);
  if (rc) return rc;
  Ctx::FrameOutcome o;
  const bool can_graph = c->use_graphs && c->params.max_inner == 1 && !c->prof_on && (!c->nccl_comm || c->p2p_on);
  if (can_graph) {
    const unsigned long long key = frame_key(c, f);
    Ctx::GraphEntry *e = nullptr;
    for (auto &g : c->graphs)
      if (g.key == key) e = &g;
    if (e && e->seen >= 1 && !(e->exec && e->epoch == alloc_epoch())) {  // second sighting: capture, then replay below
      if (e->exec) cudaGraphExecDestroy(e->exec), e->exec = nullptr;
      const long long l0 = c->launches;
      const unsigned long long ep0 = alloc_epoch();
      cudaGraph_t graph = nullptr;
      MLOAM_CUDA_OK(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
      rc = frame_enqueue(c, f, &o);
      cudaError_t ce = cudaStreamEndCapture(c->stream, &graph);
      const bool ok = rc == MLOAM_OK && ce == cudaSuccess && graph && ep0 == alloc_epoch() &&
                      cudaGraphInstantiate(&e->exec, graph, 0) == cudaSuccess;
      if (ok) e->launches = (int)(c->launches - l0), e->epoch = ep0, e->out = o, c->graph_captures++;
      if (ok) c->graph_pdl_edges = count_programmatic_edges(graph);
      if (graph) cudaGraphDestroy(graph);
      c->launches = l0;
      if (!ok) {
        cudaGetLastError();
        e->exec = nullptr, e->seen = 0;  // capture failed (e.g. a buffer had to grow, which is illegal while capturing): run this frame on
        c->graph_capture_failures++;     // the plain stream path below — it performs the allocation — and capture at a later sighting
      }
    } else if (!e) {
      if (c->graphs.size() >= 96) {
        if (c->graphs.front().exec) cudaGraphExecDestroy(c->graphs.front().exec);
        c->graphs.erase(c->graphs.begin());
      }
      Ctx::GraphEntry g;
      g.key = key, g.seen = 1;
      c->graphs.push_back(g);
    }
    if (e && e->exec && e->epoch == alloc_epoch()) {
      stage_frame_inputs(c, f);  // the captured H2D nodes read them at execution time
      MLOAM_CUDA_OK(c, cudaGraphLaunch(e->exec, c->stream));
      c->frame_from_graph = true;
      c->launches += e->launches;
      rc = frame_refused(c, f, pose_out7, stats);
      if (rc) return rc;
      frame_commit(c, f.parity, e->out);
      return scan2map_finish(c, e->out.S, f.pose_init7, want_cov, e->out.ran, pose_out7, stats);
    }
  }
  rc = frame_enqueue(c, f, &o);
  if (rc) {
    c->prefetched.valid = false;  // half f.parity may be partly overwritten
    return rc;
  }
  rc = frame_refused(c, f, pose_out7, stats);
  if (rc) return rc;
  frame_commit(c, f.parity, o);
  return scan2map_finish(c, o.S, f.pose_init7, want_cov, o.ran, pose_out7, stats);
}

// ---- one constructor per kind, with the checks of every entry point that takes that kind (raw-like: in this order, rig_sweep's last)

// A ring-ordered sweep (cloud + ScanInfo, in host or in device memory)
Sweep ring_sweep(const mloam_point_t *cloud, bool host, int n, const int *scan_start, const int *scan_end, int n_scans) {
  Sweep sw;
  sw.key = cloud, sw.host = host, sw.n = n, sw.n_scans = n_scans;
  if (host) sw.h_scan_start = scan_start, sw.h_scan_end = scan_end;
  else sw.cloud = reinterpret_cast<const float4 *>(cloud), sw.scan_start = scan_start, sw.scan_end = scan_end;
  return sw;
}

// A raw-like sweep of kind `kind` at key (host or device memory) whose LiDAR l has counts[l] points (n_lidars of mloam_set_lidars): the
// checks every raw-like sweep makes last, and its layout
int rig_sweep(Ctx *c, SweepKind kind, const void *key, bool host, const int *counts, Sweep *sw) {
  const FrontEnd &fe = c->cfg.front;
  if (c->params.max_ring_points > 0 && c->params.max_ring_points < fe.horizon_scans)
    return fail(c, MLOAM_E_INVALID, "frame_raw: params.max_ring_points is below horizon_scans (a projected ring holds up to horizon_scans points)");
  *sw = Sweep{};
  RigLayout &L = sw->L;
  L.n_lidars = c->cfg.n_lidars;
  long long total = 0;
  for (int l = 0; l < L.n_lidars; l++) {
    if (counts[l] <= 0)  // the driver node's empty_check (rosNodeRVOxford.cpp:216-220)
      return fail(c, MLOAM_E_INVALID, "frame_raw: every LiDAR of the rig needs a non-empty sweep");
    L.off[l] = (int)total;
    total += counts[l];
    if (total > (1 << 30)) return fail(c, MLOAM_E_INVALID, "frame_raw: sweeps too large");
  }
  L.off[L.n_lidars] = (int)total;
  sw->kind = kind, sw->key = key, sw->host = host, sw->n = (int)total, sw->n_scans = L.n_lidars * fe.vertical_scans;
  return MLOAM_OK;
}

// The rig's raw sweeps at `raw` (host or device memory; h_counts[l] points of LiDAR l)
int raw_sweep(Ctx *c, const mloam_point_t *raw, bool host, const int *h_counts, Sweep *sw) {
  if (!c->cfg.front_set) return fail(c, MLOAM_E_STATE, "frame_raw: call mloam_set_front_end first");
  int rc = frame_single_gpu(c, true);
  if (rc) return rc;
  if (!h_counts) return MLOAM_E_INVALID;
  rc = rig_sweep(c, SweepKind::raw, raw, host, h_counts, sw);
  if (rc == MLOAM_OK && !host) sw->cloud = reinterpret_cast<const float4 *>(raw);
  return rc;
}

// The rig's PointCloud2 messages msgs (data in host or device memory): a raw sweep whose points the unpack launch writes
int msg_sweep(Ctx *c, const mloam_pc2_msg_t *msgs, bool host, Sweep *sw) {
  const FrameCfg &cfg = c->cfg;
  if (!cfg.front_set) return fail(c, MLOAM_E_STATE, "frame_msg: call mloam_set_front_end first");
  if (cfg.n_layouts == 0) return fail(c, MLOAM_E_STATE, "frame_msg: call mloam_set_front_end_layout first");
  if (cfg.n_layouts != cfg.n_lidars)
    return fail(c, MLOAM_E_STATE, "frame_msg: mloam_set_front_end_layout gave another LiDAR count than mloam_set_lidars; give the layouts again");
  int rc = frame_single_gpu(c, true);
  if (rc) return rc;
  if (!msgs) return MLOAM_E_INVALID;
  if (cfg.front.time_field)
    for (int l = 0; l < cfg.n_lidars; l++)
      if (!cfg.layouts[l].datatype[3]) return fail(c, MLOAM_E_INVALID, "frame_msg: time_field 1 needs the timestamp field as lane 3 of every layout");
  int counts[MLOAM_MAX_LIDARS];
  for (int l = 0; l < cfg.n_lidars; l++) {
    const mloam_pc2_msg_t &m = msgs[l];
    const mloam_pc2_layout_t &F = cfg.layouts[l];
    if (!m.data) return fail(c, MLOAM_E_INVALID, "frame_msg: a message without data");
    if (m.width <= 0 || m.height <= 0)  // the driver node's empty_check (rosNodeRVOxford.cpp:216-220)
      return fail(c, MLOAM_E_INVALID, "frame_msg: every LiDAR of the rig needs a non-empty message");
    if ((long long)m.width * m.height > (1 << 30)) return fail(c, MLOAM_E_INVALID, "frame_msg: sweeps too large");
    if (m.row_step < (size_t)m.width * (size_t)F.point_step) return fail(c, MLOAM_E_INVALID, "frame_msg: row_step < width x point_step");
    if (m.row_step > m.size / (size_t)m.height)  // size < height x row_step, without the product's overflow
      return fail(c, MLOAM_E_INVALID, "frame_msg: a message is shorter than height x row_step");
    counts[l] = m.width * m.height;
  }
  rc = rig_sweep(c, SweepKind::msg, msgs[0].data, host, counts, sw);
  if (rc) return rc;
  for (int l = 0; l < cfg.n_lidars; l++) sw->wire.msg[l] = msgs[l], sw->wire.layout[l] = cfg.layouts[l];
  return MLOAM_OK;
}

// The rig's ASCII PCD bodies pcds (data in host or device memory): a raw sweep of POINTS points per LiDAR, which the decode writes
int pcd_sweep(Ctx *c, const mloam_pcd_t *pcds, bool host, Sweep *sw) {
  const FrameCfg &cfg = c->cfg;
  if (!cfg.front_set) return fail(c, MLOAM_E_STATE, "frame_pcd: call mloam_set_front_end first");
  int rc = frame_single_gpu(c, true);
  if (rc) return rc;
  if (!pcds) return MLOAM_E_INVALID;
  if (cfg.front.time_field) return fail(c, MLOAM_E_INVALID, "frame_pcd: a PointXYZ cloud has no timestamp field (time_field 1)");
  rc = pcd_check(c, cfg.n_lidars, pcds);
  if (rc) return rc;
  int counts[MLOAM_MAX_LIDARS];
  for (int l = 0; l < cfg.n_lidars; l++) counts[l] = pcds[l].points;
  rc = rig_sweep(c, SweepKind::pcd, pcds[0].data, host, counts, sw);
  if (rc) return rc;
  for (int l = 0; l < cfg.n_lidars; l++) sw->pcdf.body[l] = pcds[l];
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

// What every mloam_frame* entry point does after its checks and the constructor that made its sweep sw (rc; evaluated with the
// arguments, before sw is read), with sw and the submaps (host buffers for a host sweep, device buffers otherwise): the sweep — unless the look-ahead made its features —, the announced next sweep and the
// submaps go up, the frame runs, and the call consumes the announcement and the uploads.
int frame_call(Ctx *c, int rc, const Sweep &sw, const mloam_point_t *surf_map, int n_surf_map, const mloam_point_t *corner_map,
               int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (rc) return rc;
  c->reg_valid = false;
  if (sw.host && rebuild_maps && (!surf_map || !corner_map || n_surf_map < 0 || n_corner_map < 0)) return MLOAM_E_INVALID;
  // the poses announced with this sweep (mloam_frame_set_next_undistort), consumed by this call whatever it returns
  const Ctx::AnnouncedPoses ann = c->undist_announced;
  c->undist_announced.undist.n = 0;
  if (c->cfg.undist_on) {  // the sweep's pose_undist (mloam_frame_undistort, else the announced one), consumed by this call whatever it returns
    bool set = c->undist_set;
    c->undist_set = false;
    if (!set && ann.undist.n > 0 && same_sweep(ann.sw, sw)) {
      std::memcpy(c->undist_pose7, ann.undist.pose7, sizeof(double) * 7 * (size_t)ann.undist.n);
      c->undist_n = ann.undist.n, set = true;
    }
    if (!set) return fail(c, MLOAM_E_STATE, "frame: the undistortion is on and no pose was given for this sweep (mloam_frame_undistort)");
    if (c->undist_n != c->cfg.n_parts())
      return fail(c, MLOAM_E_INVALID, "frame: mloam_frame_undistort gave a pose count other than the frame's LiDARs (1 without the rig merge)");
  }
  cudaSetDevice(c->device);
  // this sweep's features: extracted while the previous frame was solved (look-ahead), or now into the half after the previous frame's
  FrameCall f{sw, frame_has_prefetched(c, sw), 0, nullptr, nullptr, n_surf_map, n_corner_map, rebuild_maps, pose_init7, false};
  f.parity = f.have ? c->prefetched.parity : c->frame_parity;
  f.take_undist = f.have && c->cfg.undist_on && !c->prefetched.extract_only;
  if (!sw.host) f.surf_map = reinterpret_cast<const float4 *>(surf_map), f.corner_map = reinterpret_cast<const float4 *>(corner_map);
  rc = sw.host ? sweep_to_device(c, c->sweep_in, &f.sw, !f.have, c->pinned->scan_info, c->stream) : MLOAM_OK;
  if (rc == MLOAM_OK) rc = stage_next_sweep(c);
  if (rc == MLOAM_OK && sw.host && rebuild_maps) rc = upload_submaps(c, surf_map, n_surf_map, corner_map, n_corner_map, &f.surf_map, &f.corner_map);
  if (rc == MLOAM_OK) rc = frame_run(c, f, pose_out7, stats);
  if (rc == MLOAM_OK && f.take_undist) c->undist_ahead_taken++;
  if (c->next.set && c->next.undist.n > 0) c->undist_announced = Ctx::AnnouncedPoses{c->next.sw, c->next.undist};
  c->maps_pending = false, c->next_pending = false, c->next.set = false;
  if (rc == MLOAM_OK) memcpy(c->last_pose7, pose_out7, sizeof(c->last_pose7)), c->frame_since_save = true;  // mloam_keyframe_save
  c->reg_valid = rc == MLOAM_OK && c->cfg.reg_on;  // mloam_frame_registered
  return rc;
}

// What every mloam_frame_set_next* call does after its checks and its sweep's constructor (rc): the previous announcement is withdrawn,
// and sw — unless the checks failed or sw is empty (a withdrawal) — is announced for the next frame
int announce(Ctx *c, int rc, const Sweep &sw) {
  c->next = Ctx::NextSweep{};
  if (rc == MLOAM_OK && sw.key) c->next.set = true, c->next.sw = sw, c->next.undist_open = true;
  return rc;
}

// The front end alone (mloam_front_end*) of host sweep sw after the constructor that made it (rc, as frame_call's): its raw points on the device, then the projection
// into front_out and the read-back of the ring-ordered sweep and its ScanInfo
int front_end_call(Ctx *c, int rc, const Sweep &made, mloam_point_t *h_out, int *n_out, int *h_scan_start, int *h_scan_end) {
  *n_out = 0;
  if (rc) return rc;
  Sweep sw = made;  // a message sweep's staging is set below
  cudaSetDevice(c->device);
  const int n = sw.n, n_scans = sw.n_scans;
  cudaStream_t st = c->stream;
  c->prefetched.valid = false;  // the front end's output buffer is the frame's
  const float4 *d_raw = nullptr;
  switch (sw.kind) {
    case SweepKind::ring: return MLOAM_E_INVALID;  // the constructors of the front end make raw-like sweeps only
    case SweepKind::raw:
      MLOAM_CUDA_OK(c, c->sweep_in.reserve(sizeof(float4) * (size_t)n));
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->sweep_in.p, sw.key, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
      d_raw = c->sweep_in.as<float4>();
      break;
    case SweepKind::msg:  // staged in sweep_in and unpacked into wire_out, as in a frame
      rc = sweep_to_device(c, c->sweep_in, &sw, true, nullptr, st);
      if (rc == MLOAM_OK) rc = sweep_points(c, sw, 0, &d_raw);
      break;
    case SweepKind::pcd:  // decoded into wire_out by pcd_decode_device, which waits and refuses a malformed body before the projection
      MLOAM_CUDA_OK(c, c->wire_out.reserve(sizeof(float4) * ((size_t)n + 1)));
      rc = pcd_decode_device(c, sw.L.n_lidars, sw.pcdf.body, true, c->wire_out.as<float4>());
      d_raw = c->wire_out.as<float4>();
      break;
  }
  if (rc) return rc;
  float4 *d_out;
  int *d_meta;  // [0] count, then scan starts, scan ends
  MLOAM_CUDA_OK(c, carve(c->front_out, [&](Carve &cv) { d_out = cv.take<float4>((size_t)n + 1), d_meta = cv.take<int>(4 + 2 * (size_t)n_scans); }));
  const FrontEnd &fe = c->cfg.front;
  rc = project_cloud_device(c, d_raw, sw.L, fe.vertical_scans, fe.horizon_scans, fe.roi_range, &fe, d_out, d_meta + 4, d_meta + 4 + n_scans,
                            d_meta, c->front_work);
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
  return frame_call(&h->c, MLOAM_OK, ring_sweep(d_cloud, false, n, d_scan_start, d_scan_end, n_scans), d_surf_map, n_surf_map,
                    d_corner_map, n_corner_map, rebuild_maps, pose_init7, pose_out7, stats);
}

// Look-ahead: announce the sweep of the NEXT mloam_frame* call.  While the coming frame is matched and solved, that sweep is extracted
// and down-sampled on a side stream (in the reference the two stages run in different nodes, estimator -> lidar_mapper); the next
// call finds its features ready when it passes the same pointer (and sizes) — otherwise it extracts as usual.  One announcement is
// consumed by one frame; results are identical with or without it.
int mloam_frame_set_next_device(mloam_ctx_t *h, const mloam_point_t *d_cloud, int n, const int *d_scan_start, const int *d_scan_end, int n_scans) {
  if (!h) return MLOAM_E_INVALID;
  if (!d_cloud || n <= 0) return announce(&h->c, MLOAM_OK, Sweep{});  // withdraw
  const int rc = (!d_scan_start || !d_scan_end || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS) ? MLOAM_E_INVALID : MLOAM_OK;
  return announce(&h->c, rc, ring_sweep(d_cloud, false, n, d_scan_start, d_scan_end, n_scans));
}
int mloam_frame_set_next(mloam_ctx_t *h, const mloam_point_t *h_cloud, int n, const int *h_scan_start, const int *h_scan_end, int n_scans) {
  if (!h) return MLOAM_E_INVALID;
  if (!h_cloud || n <= 0) return announce(&h->c, MLOAM_OK, Sweep{});  // withdraw
  const int rc = (!h_scan_start || !h_scan_end || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS) ? MLOAM_E_INVALID : MLOAM_OK;
  return announce(&h->c, rc, ring_sweep(h_cloud, true, n, h_scan_start, h_scan_end, n_scans));
}

int mloam_frame(mloam_ctx_t *h, const mloam_point_t *h_cloud, int n, const int *h_scan_start, const int *h_scan_end, int n_scans,
                const mloam_point_t *h_surf_map, int n_surf_map, const mloam_point_t *h_corner_map, int n_corner_map, int rebuild_maps,
                const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || n <= 0 || !h_cloud || !h_scan_start || !h_scan_end || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS)
    return MLOAM_E_INVALID;
  return frame_call(&h->c, MLOAM_OK, ring_sweep(h_cloud, true, n, h_scan_start, h_scan_end, n_scans), h_surf_map, n_surf_map,
                    h_corner_map, n_corner_map, rebuild_maps, pose_init7, pose_out7, stats);
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
  c->cfg.front = FrontEnd{vertical_scans, horizon_scans, roi_range, scan_period, time_field ? 1 : 0};
  c->cfg.front_set = true;
  c->prefetched.valid = false;  // look-ahead features were made with the previous front end
  undist_withdraw(c);
  return MLOAM_OK;
}

int mloam_front_end(mloam_ctx_t *h, const mloam_point_t *h_raw, const int *h_counts, mloam_point_t *h_out, int *n_out, int *h_scan_start,
                    int *h_scan_end) {
  if (!h || !h_out || !n_out || !h_scan_start || !h_scan_end || !h_raw) return MLOAM_E_INVALID;
  Sweep sw;
  return front_end_call(&h->c, raw_sweep(&h->c, h_raw, true, h_counts, &sw), sw, h_out, n_out, h_scan_start, h_scan_end);
}

int mloam_frame_raw(mloam_ctx_t *h, const mloam_point_t *h_raw, const int *h_counts, const mloam_point_t *h_surf_map, int n_surf_map,
                    const mloam_point_t *h_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7,
                    mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || !h_raw) return MLOAM_E_INVALID;
  Sweep sw;
  return frame_call(&h->c, raw_sweep(&h->c, h_raw, true, h_counts, &sw), sw, h_surf_map, n_surf_map, h_corner_map, n_corner_map,
                    rebuild_maps, pose_init7, pose_out7, stats);
}

int mloam_frame_raw_device(mloam_ctx_t *h, const mloam_point_t *d_raw, const int *h_counts, const mloam_point_t *d_surf_map, int n_surf_map,
                           const mloam_point_t *d_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7,
                           mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7 || !d_raw) return MLOAM_E_INVALID;
  Sweep sw;
  return frame_call(&h->c, raw_sweep(&h->c, d_raw, false, h_counts, &sw), sw, d_surf_map, n_surf_map, d_corner_map, n_corner_map,
                    rebuild_maps, pose_init7, pose_out7, stats);
}

// Look-ahead for raw frames: as mloam_frame_set_next*, picked up by the next mloam_frame_raw* call with the same pointer and counts
int mloam_frame_set_next_raw(mloam_ctx_t *h, const mloam_point_t *h_raw, const int *h_counts) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = h_raw ? raw_sweep(&h->c, h_raw, true, h_counts, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, rc, sw);
}
int mloam_frame_set_next_raw_device(mloam_ctx_t *h, const mloam_point_t *d_raw, const int *h_counts) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = d_raw ? raw_sweep(&h->c, d_raw, false, h_counts, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, rc, sw);
}

// ------------------------------------------------------------------------------------------ PointCloud2 messages
int mloam_set_front_end_layout(mloam_ctx_t *h, int n_lidars, const mloam_pc2_layout_t *layouts) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (n_lidars < 1 || n_lidars > MLOAM_MAX_LIDARS || !layouts) return fail(c, MLOAM_E_INVALID, "set_front_end_layout: 1 to 16 layouts");
  for (int l = 0; l < n_lidars; l++) {
    const mloam_pc2_layout_t &F = layouts[l];
    if (F.point_step < 1 || F.point_step > 1024) return fail(c, MLOAM_E_INVALID, "set_front_end_layout: point_step must be 1 .. 1024 bytes");
    for (int k = 0; k < 4; k++) {
      const int dt = F.datatype[k];
      if (k == 3 && dt == 0) continue;  // no lane 3
      if (dt != 7 && dt != 8) return fail(c, MLOAM_E_INVALID, "set_front_end_layout: fields must be FLOAT32 (7) or FLOAT64 (8)");
      if (F.offset[k] < 0 || F.offset[k] > F.point_step - (dt == 8 ? 8 : 4))
        return fail(c, MLOAM_E_INVALID, "set_front_end_layout: a field does not lie inside the point (offset + size > point_step)");
    }
  }
  FrameCfg &f = c->cfg;
  f.n_layouts = n_lidars;
  memset(f.layouts, 0, sizeof(f.layouts));
  memcpy(f.layouts, layouts, sizeof(mloam_pc2_layout_t) * (size_t)n_lidars);
  c->prefetched.valid = false;  // as mloam_set_front_end
  undist_withdraw(c);
  return MLOAM_OK;
}

int mloam_front_end_msg(mloam_ctx_t *h, const mloam_pc2_msg_t *msgs, mloam_point_t *h_out, int *n_out, int *h_scan_start, int *h_scan_end) {
  if (!h || !h_out || !n_out || !h_scan_start || !h_scan_end) return MLOAM_E_INVALID;
  Sweep sw;
  return front_end_call(&h->c, msg_sweep(&h->c, msgs, true, &sw), sw, h_out, n_out, h_scan_start, h_scan_end);
}

// The decode of the rig's ASCII PCD bodies (pcd.cu), then the raw front end, as mloam_front_end_msg
int mloam_front_end_pcd(mloam_ctx_t *h, const mloam_pcd_t *pcds, mloam_point_t *h_out, int *n_out, int *h_scan_start, int *h_scan_end) {
  if (!h || !h_out || !n_out || !h_scan_start || !h_scan_end) return MLOAM_E_INVALID;
  Sweep sw;
  return front_end_call(&h->c, pcd_sweep(&h->c, pcds, true, &sw), sw, h_out, n_out, h_scan_start, h_scan_end);
}

int mloam_frame_msg(mloam_ctx_t *h, const mloam_pc2_msg_t *msgs, const mloam_point_t *h_surf_map, int n_surf_map,
                    const mloam_point_t *h_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7,
                    mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7) return MLOAM_E_INVALID;
  Sweep sw;
  return frame_call(&h->c, msg_sweep(&h->c, msgs, true, &sw), sw, h_surf_map, n_surf_map, h_corner_map, n_corner_map,
                    rebuild_maps, pose_init7, pose_out7, stats);
}

int mloam_frame_msg_device(mloam_ctx_t *h, const mloam_pc2_msg_t *msgs, const mloam_point_t *d_surf_map, int n_surf_map,
                           const mloam_point_t *d_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7,
                           double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7) return MLOAM_E_INVALID;
  Sweep sw;
  return frame_call(&h->c, msg_sweep(&h->c, msgs, false, &sw), sw, d_surf_map, n_surf_map, d_corner_map, n_corner_map,
                    rebuild_maps, pose_init7, pose_out7, stats);
}

// Look-ahead for message frames: as mloam_frame_set_next_raw*, picked up by the next mloam_frame_msg* call with the same messages
int mloam_frame_set_next_msg(mloam_ctx_t *h, const mloam_pc2_msg_t *msgs) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = msgs ? msg_sweep(&h->c, msgs, true, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, rc, sw);
}
int mloam_frame_set_next_msg_device(mloam_ctx_t *h, const mloam_pc2_msg_t *msgs) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = msgs ? msg_sweep(&h->c, msgs, false, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, rc, sw);
}

// PCD frames: as mloam_frame_raw* on the sweep the decode of the rig's bodies gives
int mloam_frame_pcd(mloam_ctx_t *h, const mloam_pcd_t *pcds, const mloam_point_t *h_surf_map, int n_surf_map, const mloam_point_t *h_corner_map,
                    int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7) return MLOAM_E_INVALID;
  Sweep sw;
  return frame_call(&h->c, pcd_sweep(&h->c, pcds, true, &sw), sw, h_surf_map, n_surf_map, h_corner_map, n_corner_map,
                    rebuild_maps, pose_init7, pose_out7, stats);
}

int mloam_frame_pcd_device(mloam_ctx_t *h, const mloam_pcd_t *pcds, const mloam_point_t *d_surf_map, int n_surf_map,
                           const mloam_point_t *d_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7,
                           double *pose_out7, mloam_solve_stats_t *stats) {
  if (!h || !pose_init7 || !pose_out7) return MLOAM_E_INVALID;
  Sweep sw;
  return frame_call(&h->c, pcd_sweep(&h->c, pcds, false, &sw), sw, d_surf_map, n_surf_map, d_corner_map, n_corner_map,
                    rebuild_maps, pose_init7, pose_out7, stats);
}

// Look-ahead for PCD frames: as mloam_frame_set_next_msg*, picked up by the next mloam_frame_pcd* call with the same bodies
int mloam_frame_set_next_pcd(mloam_ctx_t *h, const mloam_pcd_t *pcds) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = pcds ? pcd_sweep(&h->c, pcds, true, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, rc, sw);
}
int mloam_frame_set_next_pcd_device(mloam_ctx_t *h, const mloam_pcd_t *pcds) {
  if (!h) return MLOAM_E_INVALID;
  Sweep sw;
  const int rc = pcds ? pcd_sweep(&h->c, pcds, false, &sw) : MLOAM_OK;  // nullptr: withdraw
  return announce(&h->c, rc, sw);
}

int mloam_set_lidars(mloam_ctx_t *h, int n_lidars, const double *ext7) {
  if (!h || n_lidars < 1 || n_lidars > MLOAM_MAX_LIDARS || (n_lidars > 1 && !ext7)) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  FrameCfg &f = c->cfg;
  f.n_lidars = n_lidars;
  c->prefetched.valid = false;  // look-ahead features were merged with the previous extrinsics
  undist_withdraw(c);           // ... and the announced poses may be of another count
  f.lidar_merge = ext7 != nullptr;  // also for ONE LiDAR with an extrinsic: same float transform + laser id as in a rig
  for (int l = 0; l < n_lidars; l++)
    for (int k = 0; k < 7; k++) f.lidar_ext[l][k] = ext7 ? ext7[7 * l + k] : (k == 6 ? 1.0 : 0.0);
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ uncertainty-aware frames
int mloam_set_uncertainty(mloam_ctx_t *h, int with_ua, const double *ext_cov36, const double *cov_meas9, double trace_threshold) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (with_ua && (!ext_cov36 || !cov_meas9)) return MLOAM_E_INVALID;
  FrameCfg &f = c->cfg;
  f.with_ua = with_ua ? 1 : 0;
  if (!with_ua) return MLOAM_OK;
  const int n_lasers = f.n_parts();
  for (int l = 0; l < MLOAM_MAX_LIDARS; l++)
    for (int k = 0; k < 36; k++) f.ua_ext_cov[l][k] = l < n_lasers ? ext_cov36[36 * l + k] : 0.0;
  memcpy(f.ua_cov_meas, cov_meas9, sizeof(f.ua_cov_meas));
  f.ua_trace_threshold = trace_threshold;
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ outlier cloud (segment_cloud: 0)
int mloam_set_outlier(mloam_ctx_t *h, float map_outlier_res) {
  if (!h || !(map_outlier_res >= 0.f) || map_outlier_res > 3.0e38f) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (multi_gpu(c))
    return fail(c, MLOAM_E_STATE, "set_outlier: the outlier cloud is single-GPU only, like with_ua; detach the communicator");
  c->cfg.outlier_on = map_outlier_res > 0.f;
  c->cfg.outlier_leaf = c->cfg.outlier_on ? map_outlier_res : 0.f;
  return MLOAM_OK;
}

int mloam_frame_outlier(mloam_ctx_t *h, mloam_point_t *h_pts, float *h_cov6, int cap, int *n) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (n) *n = 0;
  if (!c->last_scan_valid) return fail(c, MLOAM_E_STATE, "frame_outlier: no mloam_frame* call has run since the last reset");
  const ScanRef &S = c->last_scan;
  if (!S.d_n_outlier) return fail(c, MLOAM_E_STATE, "frame_outlier: the last frame ran without the outlier cloud (mloam_set_outlier)");
  cudaSetDevice(c->device);
  cudaStream_t st = c->stream;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, S.d_n_outlier, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  const int m = hc[0];
  if (n) *n = m;
  if (!(h_pts || h_cov6) || m == 0) return MLOAM_OK;
  if (m > cap) return fail(c, MLOAM_E_INVALID, "frame_outlier: capacity too small (*n holds the cloud's size)");
  if (h_pts) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_pts, S.outlier, sizeof(float4) * (size_t)m, cudaMemcpyDeviceToHost, st));
  if (h_cov6) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cov6, S.cov6_outlier, sizeof(float) * 6 * (size_t)m, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ gd_float
int mloam_set_gf_float(mloam_ctx_t *h, int on, float map_deg_thre) {
  if (!h || (on && !(map_deg_thre == map_deg_thre))) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!on) {
    c->cfg.gf_float_on = false;
    return MLOAM_OK;
  }
  if (c->params.gf_method != 3) return fail(c, MLOAM_E_STATE, "set_gf_float: gd_float is gd_fix with an adaptive ratio; set params.gf_method = 3 first");
  if (multi_gpu(c))
    return fail(c, MLOAM_E_STATE, "set_gf_float: gd_float is single-GPU only (the 21 sums of sharded features are not exchanged); detach the communicator");
  cudaSetDevice(c->device);
  c->gf_float.in_graphs = false;  // allocated once, so the graphs that hold its address stay valid
  MLOAM_CUDA_OK(c, c->gf_float.reserve(sizeof(GfFloatDev)));
  const double ini = (double)c->params.gf_ratio;
  c->gf_float_host = GfFloatState{ini < 1.0 ? ini : 1.0, 0.0, 0, 0};  // gf_ratio_cur = std::min(1.0, FLAGS_gf_ratio_ini) (:1248)
  c->pinned->gf_float = c->gf_float_host;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(&c->gf_float.as<GfFloatDev>()->st, &c->pinned->gf_float, sizeof(GfFloatState), cudaMemcpyHostToDevice, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  c->cfg.gf_float_on = true, c->cfg.gf_float_thre = map_deg_thre;
  c->gf_float_frames = 0, c->gf_float_eval = c->gf_float_evaluated = c->gf_float_reported = false;
  return MLOAM_OK;
}

int mloam_set_gf_float_threshold(mloam_ctx_t *h, float map_deg_thre) {
  if (!h || !(map_deg_thre == map_deg_thre)) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->cfg.gf_float_on) return fail(c, MLOAM_E_STATE, "set_gf_float_threshold: gd_float is off (mloam_set_gf_float)");
  c->cfg.gf_float_thre = map_deg_thre;
  return MLOAM_OK;
}

int mloam_gf_float_report(mloam_ctx_t *h, double *ratio_cur, double *deg_factor, int *total_feat_num, int *evaluated_last_call, long long *frame_cnt) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->cfg.gf_float_on) return fail(c, MLOAM_E_STATE, "gf_float_report: gd_float is off (mloam_set_gf_float)");
  if (!c->gf_float_reported) return fail(c, MLOAM_E_STATE, "gf_float_report: no solve call has run since gd_float was turned on");
  const GfFloatState &g = c->gf_float_host;
  if (ratio_cur) *ratio_cur = g.ratio_cur;
  if (deg_factor) *deg_factor = g.deg_factor;
  if (total_feat_num) *total_feat_num = g.total_feat_num;
  if (evaluated_last_call) *evaluated_last_call = c->gf_float_evaluated ? 1 : 0;
  if (frame_cnt) *frame_cnt = c->gf_float_frames;
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
  c->cfg.has_ext = ext7 != nullptr;
  c->prefetched.valid = false;
  for (int k = 0; k < 7; k++) c->cfg.ext[k] = ext7 ? ext7[k] : (k == 6 ? 1.0 : 0.0);
  return MLOAM_OK;
}

}  // extern "C"
