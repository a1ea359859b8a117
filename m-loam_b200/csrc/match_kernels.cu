// match_kernels.cu — FeatureExtract::matchCornerFromMap / matchSurfFromMap (feature_extract.hpp:378-643;
// per-point forms :645-883) as two kernels:
//
//   k_match_knn  one WARP per feature: pointAssociateToMap + exact K-nearest search in the dense voxel grid
//                (knn.cuh) + the distance gate sqdist[K-1] < MIN_MATCH_SQ_DIS.  Corner and surf features share one
//                launch; the features that had to search blind in the previous iteration are scheduled first (HeavyQ),
//                so long queries — features in sparse regions — do not form the tail of the launch.  Output: K neighbour positions per feature (20 B).
//   k_match_fit  one THREAD per feature: gathers the K neighbours (5 x 16 B), fits the line (mean + scatter +
//                3x3 eigen) or the plane (5x3 column-pivoted QR), applies the lambda / plane-distance / FOV gates
//                and writes valid + coefficients.  Running the fit one-thread-per-feature instead of redundantly
//                in all 32 lanes of the search warp removes ~1/3 of the matcher's warp instructions and halves its
//                register footprint.  The per-feature routine lives in match_fit.cuh; scan2map without good-feature
//                selection defers it into the first evaluation of the solve (k_linearize), so that a GN iteration is
//                two launches.
#include <climits>
#include <cstdlib>

#include "ctx.h"
#include "fit.cuh"
#include "knn.cuh"
#include "match_fit.cuh"

namespace mloam {

constexpr int MWARPS = 8;  // warps per CTA in k_match_knn

struct KnnSet {
  MapView map;
  const float4 *pts;   // sensor-frame features
  int n;               // count, or launch upper bound when d_n is set
  const int *d_n;      // nullable device-side count
  int *pos;            // out: n * K positions into map.sorted (-1: gate failed); in: the previous result when seeded
  int seeded;          // pos holds this set's result of the previous re-association iteration on the SAME map
  unsigned char *changed;  // out (nullable): 1 when the neighbour list differs from the seed (or there was none)
  float4 *anchor;      // per feature: map-frame position of its last real search + the displacement it tolerates
  int half;            // double-buffered pos / anchor (SpecState): features per half; 0: read and write in place
  const unsigned char *heavy_in;  // nullable: 1 where the previous launch listed the query (HeavyQ) — those go first
  unsigned char *heavy_out;       // this launch's verdict, for the next one
};

// Scheduling of the searches inside a launch.  Queries differ by about 10x in cost (a kept neighbour list is a re-rank,
// a ball search scans a few rows, a blind search grows shells) and a launch is only as fast as its slowest warp, so the
// few features that searched blind in a seeded launch are listed (atomic append — a handful per launch, not one atomic per
// query: tens of thousands of increments of ONE address serialise at the L2) and taken first by the next launch, one per
// warp; everything else is a static stride.  A launch without seeds lists nothing: all its queries search blind, and in
// the next launch they are seeded.  A stride skips the listed queries by a ballot over the list held in the lanes' registers
// (at most 32 entries) or by their heavy_in byte (longer lists).  cnt[3] rotates: a launch reads cnt_in, appends to
// cnt_out and clears cnt_zero for the launch after the next.
// all_searches (MLOAM_KNN_SCHEDULE=0, the earlier schedule): list every ball and blind search, seeded or not.
struct HeavyQ {
  const int *list_in;   // nullable (first iteration): global feature indices (corner set first)
  const int *cnt_in;
  int *list_out;
  int *cnt_out;
  int *cnt_zero;
  int all_searches;
};

// Instances.  The search is a chain of dependent warp-wide operations (prefix loads -> TMA -> REDUX / ballot / shuffle rounds),
// so more resident warps hide more of it, but only without spills (a local-memory round trip inside that chain) and only if one
// k_eval_candidate block (64 threads x 128 registers = 8192) still fits beside the matcher on each SM: the speculative schedule
// runs it next to the matcher, and where it does not fit it lands on the path to the next k_linearize.
//   k_match_knn      the default: at most KNN_LEAN_REGS registers, so three CTAs (3 x 256 x 72 = 55296 of the SM's 65536
//                    registers) sit beside one k_eval_candidate block.  Spill-free with no stack frame: the sets, the schedule's
//                    values and the warp's place in it are read from shared memory where they are used, scan_runs is inlined.
//   k_match_knn_mb2  __launch_bounds__(256, 2), MLOAM_KNN_MB=2: launched with two CTAs per SM, the earlier residency, kept to
//                    compare against;
//                    its STATS = true instance is the one for stage profiling and MLOAM_KNN_TRACE=1, with the per-path counters
//                    (path_stats: the KnnPathStats of ctx.h addressed as 32-bit words; KPS_WORD(field) is a field's word index) and
//                    the per-query trace.
// Both run the same body, so a query does the same operations in the same order in either.  sel_prune: bound-pruned selection
// (scan_runs), 0 under MLOAM_KNN_SCHEDULE=0.
#define KPS_WORD(field) (offsetof(KnnPathStats, field) / sizeof(unsigned))
constexpr int KNN_LEAN_REGS = 72;

// This warp's index in the grid, read afresh from the special registers at every use (volatile: not kept in a register
// across the search).
__device__ __forceinline__ int global_warp() {
  unsigned tid, cta;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(cta));
  return (int)(cta * MWARPS + (tid >> 5));
}

template <int K, bool STATS>
__device__ __forceinline__ void match_knn(const KnnSet &a, const KnnSet &b, const double *__restrict__ pose7, float min_match_sq_dis,
                                          const HeavyQ &hq, const int *__restrict__ d_sel, unsigned *__restrict__ path_stats, unsigned tma_min,
                                          unsigned *__restrict__ trace, int sel_prune) {
  if (!STATS) path_stats = nullptr, trace = nullptr;
  __shared__ KnnSmem ksm[MWARPS];
  const int lane = threadIdx.x & 31;
  KnnSmem &ks = ksm[threadIdx.x >> 5];
  // Prologue: nothing here reads what the kernel before this one on the GN chain (k_linearize) writes.  The maps and the device
  // feature counts were built before the solve; the heavy list and its count were written by the previous matcher, which is two
  // launches back and complete (no kernel of the chain triggers its dependents before its own grid-dependency wait).
  knn_smem_init(ks, lane, tma_min);
  // The two sets live in shared memory: a query reads its set's pointers where it uses them instead of holding them in
  // registers across the search (and a set picked by a runtime index is not copied to local memory).
  __shared__ KnnSet s_set[2];
  __shared__ GridP s_grid[2];
  __shared__ PoseD s_pose;
  if (threadIdx.x == 0) s_set[0] = a, s_set[1] = b, s_grid[0] = load_grid(a.map), s_grid[1] = load_grid(b.map);
  // Schedule: first the listed heavy features of the previous launch (one per warp), then a static stride over the rest.
  // Its CTA-wide values are kept in shared memory too and read where they are used.
  __shared__ int s_na, s_n, s_n_heavy, s_h_in;
  __shared__ int s_listed[32];  // a short heavy list (n_heavy <= 32): the stride skips these
  {
    const int na = a.d_n ? min(a.n, *a.d_n) : a.n;
    const int n = na + (b.d_n ? min(b.n, *b.d_n) : b.n);
    const int n_heavy = hq.list_in ? min(__ldg(hq.cnt_in), n) : 0;
    const int gw = blockIdx.x * MWARPS + (threadIdx.x >> 5);
    if (threadIdx.x == 0) s_na = na, s_n = n, s_n_heavy = n_heavy;
    if (threadIdx.x < 32) s_listed[lane] = n_heavy <= 32 && lane < n_heavy ? __ldg(hq.list_in + lane) : -1;
    if (lane == 0 && gw < n_heavy) ks.first = __ldg(hq.list_in + gw);  // the warp's first listed feature
  }
  // Programmatic dependent launch: the pose searched at (SpecState::xc, published by k_linearize's tail), d_sel (committed there)
  // and the lists, anchors, changed flags and fit inputs k_linearize reads are only touched after the previous kernel completed
  cudaGridDependencySynchronize();
  cudaTriggerProgrammaticLaunchCompletion();
  unsigned long long t_enter = 0ull;
  if (trace) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_enter));
  if (threadIdx.x == 0) s_pose = pose_from_param(pose7), s_h_in = d_sel ? (*d_sel & 1) : 0;  // double-buffered sets: read half s_h_in, write the other
  __syncthreads();
  const int n_warps = gridDim.x * MWARPS;
  if (hq.cnt_zero && global_warp() == 0 && lane == 0) *hq.cnt_zero = 0;
  // The warp's place in the schedule is kept in its shared-memory words too (written by lane 0, read after a __syncwarp):
  // slot < 0 walks the heavy list at slot - INT_MIN, slot >= 0 strides over the features.
  if (lane == 0) ks.slot = global_warp() < s_n_heavy ? INT_MIN + global_warp() : global_warp();
#pragma unroll 1
  for (;; ) {
    __syncwarp();
    int t = ks.slot;
    __syncwarp();  // every lane has read it before lane 0 advances it
    bool from_list = t < 0;
    if (from_list) {
      t -= INT_MIN;
      if (t >= s_n_heavy) t = global_warp(), from_list = false;
    }
    if (!from_list && t >= s_n) break;
    const int na = s_na;
    int i = t;
    if (lane == 0) ks.slot = from_list ? INT_MIN + (t + n_warps) : t + n_warps;
    if (from_list) {
      i = t == global_warp() ? ks.first : __ldg(hq.list_in + t);
    } else if (s_n_heavy > 32) {  // listed ones have been done above
      const unsigned char *hin = s_set[i < na ? 0 : 1].heavy_in;
      if (hin && hin[i < na ? i : i - na]) continue;
    } else if (s_n_heavy > 0 && __any_sync(MLOAM_FULL_MASK, s_listed[lane] == i)) {
      continue;
    }
    const bool in_a = i < na;
    const int j = in_a ? i : i - na;
    const KnnSet &S = s_set[in_a ? 0 : 1];
    const float4 p = __ldg(S.pts + j);
    const long long t_query = (path_stats || trace) ? clock64() : 0ll;
    int path = 3;  // 0 keep (matched), 1 keep (rejected), 2 ball, 3 blind
    const float3 sel = associate(s_pose, p.x, p.y, p.z);  // pointAssociateToMap, utility.h:103-117
    const GridP &g = s_grid[in_a ? 0 : 1];
    Best best;  // selection width K + 1: lane K holds the nearest scanned point outside the K-set (feeds the anchor's slack)
    // read half o_in, write half o_out: every query writes its complete state (list, anchor) to the out half.  The addresses
    // are formed from S where they are used.
    const int o_in = s_h_in ? S.half : 0, o_out = S.half - o_in;
    const int seeded = S.seeded;
    // Temporal coherence between re-association iterations (all three shortcuts are exact, see knn.cuh):
    //   keep    the query moved less than the anchor's slack since its last real search: the K-set cannot have
    //           changed, only its order — recompute the K distances and re-rank (no cell probes, no scan)
    //   ball    otherwise the previous neighbours bound the search ball around the moved query
    //   blind   no previous neighbours (or a ball of more than 32 cells)
    int prev = -1, newpos = -1;
    bool done = false;
    float r2 = 3.0e38f;
    if (seeded) {
      if (lane < K) prev = S.pos[(size_t)(j + o_in) * K + lane];
      const float4 an = S.anchor[j + o_in];
      const float mx = sel.x - an.x, my = sel.y - an.y, mz = sel.z - an.z;
      const float moved = sqrtf(mx * mx + my * my + mz * mz);
      const bool within = an.w > 0.0f && moved + 2e-5f < an.w;
      if (__shfl_sync(MLOAM_FULL_MASK, prev, 0) < 0) {
        // rejected last time with the K-th neighbour at least radius + an.w away from the anchor: still rejected
        if (within) {
          done = true;
          path = 1;
          if (lane == 0 && o_out != o_in) S.anchor[j + o_out] = an;
        }
      } else {
        unsigned long long key = MLOAM_KEY_NONE;
        unsigned d2b = 0u;
        if (lane < K) {
          const float4 v = __ldg(S.map.sorted + prev);
          const float ex = v.x - sel.x, ey = v.y - sel.y, ez = v.z - sel.z;
          d2b = __float_as_uint(ex * ex + ey * ey + ez * ez);  // non-negative floats order like their bit patterns
          key = ((unsigned long long)d2b << 32) | (unsigned)__float_as_int(v.w);
        }
        r2 = __uint_as_float(__reduce_max_sync(MLOAM_FULL_MASK, d2b));
        if (within) {
          int rank = 0;
#pragma unroll
          for (int k = 0; k < K; k++) {
            const unsigned long long other = __shfl_sync(MLOAM_FULL_MASK, key, k);
            if (other < key) rank++;
          }
#pragma unroll
          for (int k = 0; k < K; k++) {
            const int rk = __shfl_sync(MLOAM_FULL_MASK, rank, k), pk = __shfl_sync(MLOAM_FULL_MASK, prev, k);
            if (rk == lane) newpos = pk;
          }
          if (!(r2 < min_match_sq_dis)) {  // :407,571,667,814 — the slack of a match says nothing about a rejection
            newpos = -1;
            if (lane == 0) S.anchor[j + o_out] = make_float4(sel.x, sel.y, sel.z, 0.0f);
          } else if (lane == 0 && o_out != o_in) {
            S.anchor[j + o_out] = an;
          }
          done = true;
          path = 0;
        }
      }
    }
    if (!done) {
      float explored = 0.0f;
      bool found = false;
      if (r2 < min_match_sq_dis)
        found = warp_knn_seeded<K, K + 1>(S.map, g, ks, sel.x, sel.y, sel.z, r2, 0.1f * g.cell,
                                             lane, best, &explored, sel_prune != 0);
      if (!found) {
        KnnDbg dbg = {0, 0, 0, 0, 0, 0};
        const long long t_blind = (path_stats || trace) ? clock64() : 0ll;
        warp_knn<K, true, K + 1>(S.map, g, ks, sel.x, sel.y, sel.z, min_match_sq_dis, lane, best, &explored, 0.05f,
                                 (path_stats || trace) ? &dbg : nullptr, sel_prune != 0);
        if (trace && lane == 0) {
          unsigned *tr = trace + 4 * (size_t)((in_a ? 0 : na) + j);
          tr[1] = (unsigned)dbg.t_ring1, tr[2] = (unsigned)dbg.t_ball, tr[3] = ((unsigned)dbg.ring1_pts << 20) | ((unsigned)(dbg.ball_pts & 0xfff) << 8) | (unsigned)(dbg.ball_steps & 0xff);
        }
        if (path_stats && lane == 0) {
          unsigned long long *q = reinterpret_cast<unsigned long long *>(path_stats + KPS_WORD(blind));
          atomicAdd(q + 0, 0ull), atomicAdd(q + 1, (unsigned long long)dbg.t_ring1);
          atomicAdd(q + 2, (unsigned long long)dbg.t_ball), atomicAdd(q + 3, (unsigned long long)dbg.ring1_pts);
          atomicAdd(q + 4, (unsigned long long)dbg.ball_pts), atomicAdd(q + 5, (unsigned long long)dbg.ball_steps);
          atomicAdd(q + 6, (unsigned long long)dbg.ball_rows), atomicAdd(q + 7, dbg.t_ball ? 1ull : 0ull);
          const long long dt_blind = clock64() - t_blind;
          if (dt_blind > 90000) {  // a record of one very slow blind query (benign race: any of them will do)
            long long *rec = reinterpret_cast<long long *>(path_stats + KPS_WORD(slow_rec));
            rec[0] = dt_blind, rec[1] = 0, rec[2] = dbg.t_ring1, rec[3] = dbg.t_ball, rec[4] = dbg.ring1_pts;
            rec[5] = dbg.ball_pts, rec[6] = dbg.ball_rows, rec[7] = dbg.ball_steps, rec[8] = (in_a ? 0 : 1) * 1000000 + j;
            rec[9] = (long long)(t_blind - t_query);
          }
        }
      }
      path = found ? 2 : 3;
      const unsigned long long kK = best_key(best, K - 1), kK1 = best_key(best, K);
      const bool ok = kK != MLOAM_KEY_NONE && key_d2(kK) < min_match_sq_dis;  // :407,571,667,814
      newpos = (ok && lane < K) ? best.pos : -1;
      // anchor: K-set members are within rK of this position, everything else at least lb away
      float slack = 0.0f;
      if (ok) {
        const float rK = sqrtf(key_d2(kK));
        float lb = explored;
        if (kK1 != MLOAM_KEY_NONE) lb = fminf(lb, sqrtf(key_d2(kK1)));
        slack = 0.5f * (lb - rK) - 2e-5f;
      } else {
        // rejected: the K-th neighbour is at least lbK away; while the query stays within lbK - radius of here the
        // verdict stands
        float lbK = explored;
        if (kK != MLOAM_KEY_NONE) lbK = fminf(lbK, sqrtf(key_d2(kK)));
        slack = lbK - sqrtf(min_match_sq_dis) - 2e-5f;
      }
      if (lane == 0) S.anchor[j + o_out] = make_float4(sel.x, sel.y, sel.z, slack);
    }
    if (lane < K) S.pos[(size_t)(j + o_out) * K + lane] = newpos;
    if (S.changed) {
      const bool diff = __any_sync(MLOAM_FULL_MASK, lane < K && (!seeded || newpos != prev));
      if (lane == 0) S.changed[j] = diff ? 1 : 0;
    }
    if (path_stats && lane == 0) {  // stage profiling: queries and SM cycles per search path, slowest single query
      const unsigned long long dt = (unsigned long long)(clock64() - t_query);
      atomicAdd(path_stats + KPS_WORD(queries) + path, 1u);
      atomicAdd(reinterpret_cast<unsigned long long *>(path_stats + KPS_WORD(cycles)) + path, dt);
      atomicMax(path_stats + KPS_WORD(max_query_cycles), (unsigned)(dt > 0xffffffffull ? 0xffffffffull : dt));
      if (dt > 32768ull) atomicAdd(path_stats + KPS_WORD(over_32k), 1u);
      if (dt > 65536ull) atomicAdd(path_stats + KPS_WORD(over_64k), 1u);
      // slowest query: cycles << 32 | path << 30 | set << 29 | feature index
      atomicMax(reinterpret_cast<unsigned long long *>(path_stats + KPS_WORD(slowest)),
                (dt << 32) | ((unsigned long long)path << 30) | ((unsigned long long)(in_a ? 0 : 1) << 29) | (unsigned)(j & 0x1fffffff));
    }
    if (trace && lane == 0) trace[4 * (size_t)((in_a ? 0 : na) + j)] = (unsigned)(clock64() - t_query) | ((unsigned)path << 30);
    unsigned char *const hout = S.heavy_out;
    if (hout && lane == 0) {
      const bool heavy = hq.all_searches ? path >= 2 : (path == 3 && seeded);
      hout[j] = heavy ? 1 : 0;
      if (heavy && hq.list_out) hq.list_out[atomicAdd(hq.cnt_out, 1)] = in_a ? j : j + s_na;
    }
  }
  if (trace && lane == 0) {  // per-warp timeline after the per-query words: [enter, first query, exit] in ns
    unsigned long long t_exit;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_exit));
    unsigned long long *w = reinterpret_cast<unsigned long long *>(trace + 4 * (size_t)(a.n + b.n + 1)) + 2 * (size_t)(blockIdx.x * MWARPS + (threadIdx.x >> 5));
    w[0] = t_enter, w[1] = t_exit;
  }
}

#define KNN_PARAMS                                                                                                                  \
  KnnSet a, KnnSet b, const double *__restrict__ pose7, float min_match_sq_dis, HeavyQ hq, const int *__restrict__ d_sel,           \
      unsigned *__restrict__ path_stats, unsigned tma_min, unsigned *__restrict__ trace, int sel_prune
template <int K>
__global__ void __maxnreg__(KNN_LEAN_REGS) k_match_knn(KNN_PARAMS) {
  match_knn<K, false>(a, b, pose7, min_match_sq_dis, hq, d_sel, path_stats, tma_min, trace, sel_prune);
}
template <int K, bool STATS>
__global__ void __launch_bounds__(MWARPS * 32, 2) k_match_knn_mb2(KNN_PARAMS) {
  match_knn<K, STATS>(a, b, pose7, min_match_sq_dis, hq, d_sel, path_stats, tma_min, trace, sel_prune);
}
#undef KNN_PARAMS

template <int K>
__global__ void __launch_bounds__(128) k_match_fit(FitSet a, FitSet b, const double *__restrict__ pose7, float min_plane_dis, int check_fov) {
  const int na = a.d_n ? min(a.n, *a.d_n) : a.n;
  const int nb = b.d_n ? min(b.n, *b.d_n) : b.n;
  const PoseD T = pose_from_param(pose7);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < na + nb; i += gridDim.x * blockDim.x) {
    if (i < na) fit_one<K>(a, i, T, min_plane_dis, check_fov);
    else fit_one<K>(b, i - na, T, min_plane_dis, check_fov);
  }
}

// ------------------------------------------------------------------------------------------------ launchers
// Match up to two feature sets (corner against MLOAM_MAP_CORNER-like slot, surf against a surf slot) in one
// kNN launch + one fit launch.  Sets with n == 0 are skipped.
int match_pair_device(Ctx *c, const MatchJob *jobs, int n_jobs, const double *d_pose7, const MatchCfg &cfg, PendingFit *defer, const int *d_sel,
                      bool pdl) {
  if (defer) defer->K = 0;
  if (n_jobs < 1 || n_jobs > 2) {
    c->err = "match: 1 or 2 jobs";
    return MLOAM_E_INVALID;
  }
  if (cfg.n_neigh != 5 && cfg.n_neigh != 10) {
    c->err = "match_from_map: n_neigh must be 5 or 10";
    return MLOAM_E_INVALID;
  }
  const int K = cfg.n_neigh;
  KnnSet ks[2];
  FitSet fs[2];
  int n_upper = 0;
  bool flip = false;
  for (int t = 0; t < 2; t++) {
    KnnSet &k = ks[t];
    FitSet &f = fs[t];
    memset(&k, 0, sizeof(k));
    memset(&f, 0, sizeof(f));
    if (t >= n_jobs || jobs[t].n <= 0) continue;
    const MatchJob &J = jobs[t];
    if (J.slot < 0 || J.slot >= MLOAM_NUM_MAPS || !c->maps[J.slot].built) {
      c->err = "match_from_map: map slot not built";
      return MLOAM_E_STATE;
    }
    if (J.type != 'c' && J.type != 's') {
      c->err = "match_from_map: type must be 'c' or 's'";
      return MLOAM_E_INVALID;
    }
    DevBuf &pb = c->knn_pos[t];
    const int halves = d_sel ? 2 : 1;  // double-buffered (speculative schedule): half 1 follows half 0
    MLOAM_CUDA_OK(c, pb.reserve(sizeof(int) * (size_t)K * (size_t)(J.n + 1) * halves));
    k.map = c->maps[J.slot].view();
    DevBuf &cb = c->knn_changed[t];
    MLOAM_CUDA_OK(c, cb.reserve((size_t)(J.n + 1)));
    k.pts = J.pts, k.n = J.n, k.d_n = J.d_n, k.pos = pb.as<int>();
    DevBuf &ab = c->knn_anchor[t];
    MLOAM_CUDA_OK(c, ab.reserve(sizeof(float4) * (size_t)(J.n + 1) * halves));
    k.seeded = J.seeded, k.changed = cb.as<unsigned char>(), k.anchor = ab.as<float4>();
    k.half = d_sel ? J.n + 1 : 0;
    c->knn_half[t] = k.half, c->knn_k = K, c->knn_map[t] = k.map;
    // search verdicts ("had to search") alternate between two halves from launch to launch: read the previous, write the next
    DevBuf &hb = c->knn_heavy[t];
    const size_t half = ((size_t)J.n + 256) & ~(size_t)255;
    MLOAM_CUDA_OK(c, hb.reserve(2 * half));
    k.heavy_in = J.seeded ? hb.as<unsigned char>() + half * (size_t)c->knn_parity : nullptr;
    k.heavy_out = hb.as<unsigned char>() + half * (size_t)(J.seeded ? (c->knn_parity ^ 1) : c->knn_parity);
    flip = flip || J.seeded;
    f.changed = (J.seeded && !J.nn) ? cb.as<unsigned char>() : nullptr;
    f.sorted = k.map.sorted, f.pts = J.pts, f.n = J.n, f.d_n = J.d_n, f.pos = pb.as<int>(), f.half = k.half;
    f.valid = J.valid, f.coeff = J.coeff, f.nn = J.nn, f.is_plane = J.type == 's' ? 1 : 0;
    n_upper += J.n;
  }
  if (d_sel && (!defer || fs[0].nn || fs[1].nn)) {  // only the deferred fit knows which half is valid
    c->err = "match: double-buffered lists need the deferred fit";
    return MLOAM_E_STATE;
  }
  if (n_upper <= 0) return MLOAM_OK;
  // heavy list of the launch: 2 lists x n_upper ints + 3 rotating counters (zeroed with the buffer; k_lm_init re-zeroes
  // them at the start of every solve, where the rotation restarts)
  HeavyQ hq{nullptr, nullptr, nullptr, nullptr, nullptr, c->knn_all_searches ? 1 : 0};
  {
    DevBuf &hl = c->knn_heavy_list;
    const size_t ints = 2 * ((size_t)n_upper + 64) + 16;
    if (hl.cap < sizeof(int) * ints) {
      MLOAM_CUDA_OK(c, hl.reserve(sizeof(int) * ints));
      MLOAM_CUDA_OK(c, cudaMemsetAsync(hl.p, 0, hl.cap, c->stream));
    }
    int *cnt = hl.as<int>();                 // [0..2] counters
    int *lists = hl.as<int>() + 16;
    const size_t half_l = (size_t)n_upper + 64;
    if (!flip) {                              // a non-seeded launch starts a solve: the rotation restarts with clean counters
      c->knn_rot = 0;
      MLOAM_CUDA_OK(c, cudaMemsetAsync(cnt, 0, 3 * sizeof(int), c->stream));
    }
    const int k = c->knn_rot;
    if (flip) hq.list_in = lists + half_l * (size_t)(k & 1), hq.cnt_in = cnt + k % 3;
    hq.list_out = lists + half_l * (size_t)((k + 1) & 1), hq.cnt_out = cnt + (k + 1) % 3, hq.cnt_zero = cnt + (k + 2) % 3;
    c->knn_rot = k + 1;
  }
  if (flip) c->knn_parity ^= 1;
  cudaStream_t st = c->stream;
  {
    ProfScope ps(c, "match");
    // with stage profiling on: how many queries took the keep (matched / rejected), ball and blind paths
    unsigned *path_stats = (c->prof_on && !getenv("MLOAM_KNN_NO_STATS")) ? reinterpret_cast<unsigned *>(&c->ctl.as<DevCtl>()->knn_stats) : nullptr;
    // one trace slot per launch of a solve: the launch that starts it clears them all, so that no clear sits between the launches of
    // the GN chain
    unsigned *trace = nullptr;
    if (c->knn_trace_on) {
      const size_t slot = 16 * (size_t)(n_upper + 1) + 16 * (size_t)MWARPS * 4 * c->sm_count;
      if (!flip || slot != c->knn_trace_slot) {
        MLOAM_CUDA_OK(c, c->knn_trace.reserve(slot * KNN_TRACE_SLOTS));
        MLOAM_CUDA_OK(c, cudaMemsetAsync(c->knn_trace.p, 0, slot * KNN_TRACE_SLOTS, st));
        c->knn_trace_slot = slot, c->knn_trace_timeline = 16 * (size_t)(n_upper + 1), c->knn_trace_n = 0;
      }
      const int s = c->knn_trace_n < KNN_TRACE_SLOTS ? c->knn_trace_n++ : KNN_TRACE_SLOTS - 1;
      trace = reinterpret_cast<unsigned *>(c->knn_trace.as<unsigned char>() + slot * (size_t)s);
    }
    // the instrumented instance is compiled for two CTAs per SM; the grid never asks for more CTAs than can be resident:
    // warps stride over the features
    const bool stats = path_stats || trace;
    const int mb = stats ? 2 : c->knn_min_blocks;
    int nb = (n_upper + MWARPS - 1) / MWARPS;
    if (nb > mb * c->sm_count) nb = mb * c->sm_count;
    void (*k)(KnnSet, KnnSet, const double *, float, HeavyQ, const int *, unsigned *, unsigned, unsigned *, int);
    if (stats) k = K == 5 ? k_match_knn_mb2<5, true> : k_match_knn_mb2<10, true>;
    else if (mb == 2) k = K == 5 ? k_match_knn_mb2<5, false> : k_match_knn_mb2<10, false>;
    else k = K == 5 ? k_match_knn<5> : k_match_knn<10>;
    MLOAM_CUDA_OK(c, launch_chain(pdl, k, nb, MWARPS * 32, st, ks[0], ks[1], d_pose7, cfg.min_match_sq_dis, hq, d_sel, path_stats,
                                  c->knn_tma_min, trace, c->knn_all_searches ? 0 : 1));
    c->launches++;
  }
  if (defer && !fs[0].nn && !fs[1].nn) {
    defer->set[0] = fs[0], defer->set[1] = fs[1];
    defer->K = K, defer->min_plane_dis = cfg.min_plane_dis, defer->check_fov = cfg.check_fov;
  } else {
    ProfScope ps(c, "fit");
    int nb = (n_upper + 127) / 128;
    if (nb > 4 * c->sm_count) nb = 4 * c->sm_count;
    if (K == 5) k_match_fit<5><<<nb, 128, 0, st>>>(fs[0], fs[1], d_pose7, cfg.min_plane_dis, cfg.check_fov);
    else k_match_fit<10><<<nb, 128, 0, st>>>(fs[0], fs[1], d_pose7, cfg.min_plane_dis, cfg.check_fov);
    c->launches++;
  }
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

int knn_residency(const Ctx *c, int K, int *ctas_per_sm, int *regs) {
  if (K != 5 && K != 10) return MLOAM_E_INVALID;
  const void *k = c->knn_min_blocks == 2 ? (K == 5 ? (const void *)k_match_knn_mb2<5, false> : (const void *)k_match_knn_mb2<10, false>)
                                         : (K == 5 ? (const void *)k_match_knn<5> : (const void *)k_match_knn<10>);
  cudaFuncAttributes fa;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, k, MWARPS * 32, 0) != cudaSuccess || cudaFuncGetAttributes(&fa, k) != cudaSuccess)
    return MLOAM_E_CUDA;
  *regs = fa.numRegs;
  return MLOAM_OK;
}

int match_from_map_device(Ctx *c, int slot, int type, const float4 *d_pts, int n, const int *d_n, const double *d_pose7,
                          const MatchCfg &cfg, unsigned char *d_valid, float *d_coeff, int *d_nn) {
  MatchJob j{slot, type, d_pts, n, d_n, d_valid, d_coeff, d_nn, 0};
  return match_pair_device(c, &j, 1, d_pose7, cfg);
}

}  // namespace mloam
