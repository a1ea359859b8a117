// gf_kernels.cu — good-feature selection (SURVEY.md §8 row a23): ActiveFeatureSelection::goodFeatureMatching,
// estimator/src/lidarMapper/lidar_mapper.h:229-573 (odometry twin: estimator.cpp:1347-1517).
//
// The reference draws candidates at random, matches each lazily against the map, evaluates its 1x6 Jacobian row
// (evaluateFeatJacobianMatching, :130-174) and greedily keeps the one that maximises log det(H + J^T J) — a sequential
// loop with a wall-clock cap.  Matching and the Jacobian depend on the feature and the pose only, so here
//   phase 1 (parallel): every feature is matched (k_match_knn / k_match_fit) and gets its Jacobian row (k_gf_jaco);
//   phase 2 (one CTA):  the selection loop itself runs on the device over those tables (k_gf_select):
//     rnd  one thread, candidate pool as a Fenwick tree (k-th remaining element / erase in O(log n) instead of the
//          reference's vector::erase);
//     gd   stochastic greedy: lane 0 draws the round's candidates (same pool / visited bookkeeping as the reference),
//          the warp evaluates their log-dets in parallel (6x6 Cholesky each) and picks the best;
//     fps  farthest-point sampling: 1024 threads update the min-distance table and arg-max it per pick.
// gd_float (lidar_mapper_keyframe.cpp:456-495): every 10th frame evalFullHessian (lidar_mapper.h:176-227) sums J^T J over every matched
// feature at the pose and with the rows phase 1 already made; k_gf_full_hessian reduces them in the reference's order, takes the
// log-determinant and leaves the ratio of the next ten frames on the device, where k_gf_select reads it.
// The reference's mt19937(random_device) is replaced by an explicit PCG32 seed and its time cap is dropped — see
// oracle/orc_gf.hpp for the restatement the kernels are checked against pick by pick.
#include <cuda_pipeline.h>

#include <vector>

#include "ctx.h"
#include "factors.cuh"
#include "host_util.h"
#include "lm.cuh"

namespace mloam {

constexpr int GF_THREADS = 1024;
constexpr int kGfMaxRandomQueue = 20;  // MAX_RANDOM_QUEUE_TIME, lidar_mapper.h:83
constexpr int kGfSmemInts = 50 * 1024;  // 200 KB of dynamic shared memory for the candidate pool (one CTA per launch)

__global__ void k_gf_jaco(const float4 *__restrict__ pts, const unsigned char *__restrict__ valid, const float *__restrict__ coeff, int n,
                          const int *__restrict__ d_n, int is_plane, const float *__restrict__ cov6, const double *__restrict__ sinfo,
                          double default_sinfo, const double *__restrict__ pose7, double *__restrict__ jaco) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (d_n) n = min(n, *d_n);
  if (i >= n) return;
  double J[6] = {0, 0, 0, 0, 0, 0};
  if (valid[i]) {
    double si = sinfo ? sinfo[i] : default_sinfo;
    if (cov6) {  // extractCov -> trace -> sqrt(1/trace) with the clamp of lidar_map_factor.hpp:34,41
      const double tr = (double)cov6[(size_t)i * 6] + (double)cov6[(size_t)i * 6 + 3] + (double)cov6[(size_t)i * 6 + 5];
      const double s = sqrt(1 / tr);
      si = s >= 3.0 ? 1.0 : s / 3.0;
    }
    const PoseR P = make_poser(pose7);
    const float4 pf = pts[i];
    const D3 p{(double)pf.x, (double)pf.y, (double)pf.z};
    const float *cf = coeff + (size_t)i * 6;
    if (is_plane) plane_factor(P, p, D3{(double)cf[0], (double)cf[1], (double)cf[2]}, (double)cf[3], si, J, true);
    else edge_factor(P, p, D3{(double)cf[0], (double)cf[1], (double)cf[2]}, D3{(double)cf[3], (double)cf[4], (double)cf[5]}, si, J, true);
  }
#pragma unroll
  for (int k = 0; k < 6; k++) jaco[(size_t)i * 6 + k] = J[k];
}

// Odometry-side rows (Estimator::evaluateFeatJacobian, estimator.cpp:1273-1345): surf features carry the pose_i block of
// LidarPureOdomPlaneNormFactor(point, coeffs, 1.0) on (pivot, pose_i, ext); corner features the constant row
// Matrix<double,1,6>::Identity() = [1 0 0 0 0 0] (:1342).
__global__ void k_gf_jaco_odom(const float4 *__restrict__ pts, const unsigned char *__restrict__ valid, const float *__restrict__ coeff, int n,
                               int is_plane, const double *__restrict__ x21 /* pivot | pose_i | ext */, double *__restrict__ jaco) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double J[6] = {0, 0, 0, 0, 0, 0};
  if (valid[i]) {
    if (is_plane) {
      const Chain ch = make_chain(x21, x21 + 7, x21 + 14);
      const float4 pf = pts[i];
      const float *cf = coeff + (size_t)i * 6;
      double Je[6];
      odom_plane_factor(ch, D3{(double)pf.x, (double)pf.y, (double)pf.z}, D3{(double)cf[0], (double)cf[1], (double)cf[2]}, (double)cf[3], 1.0, nullptr, J, Je);
    } else {
      J[0] = 1.0;
    }
  }
#pragma unroll
  for (int k = 0; k < 6; k++) jaco[(size_t)i * 6 + k] = J[k];
}

// ---- PCG32, identical to oracle/orc_gf.hpp
__device__ __forceinline__ unsigned gf_next(unsigned long long &s) {
  const unsigned long long old = s;
  s = old * 6364136223846793005ull + 1442695040888963407ull;
  const unsigned xorshifted = (unsigned)(((old >> 18u) ^ old) >> 27u);
  const unsigned rot = (unsigned)(old >> 59u);
  return (xorshifted >> rot) | (xorshifted << ((32u - rot) & 31u));
}
__device__ __forceinline__ unsigned long long gf_seed(unsigned long long seed) {
  unsigned long long s = seed * 0x9e3779b97f4a7c15ull + 0xda3e39cb94b95bdbull;
  gf_next(s);
  return s;
}
__device__ __forceinline__ int gf_uniform(unsigned long long &s, int lo, int hi) {
  const unsigned long long span = (unsigned long long)(hi - lo) + 1ull;
  return lo + (int)(((unsigned long long)gf_next(s) * span) >> 32);
}

// ---- candidate pool: Fenwick tree over "still in the pool" flags (1-based), all alive initially
__device__ __forceinline__ int fen_find_kth(const int *fen, int n, int top_pow2, int k /* 0-based */) {
  int pos = 0, rem = k + 1;
  for (int step = top_pow2; step > 0; step >>= 1) {
    const int nx = pos + step;
    if (nx <= n && fen[nx] < rem) pos = nx, rem -= fen[nx];
  }
  return pos;  // 0-based physical index of the k-th alive element
}
__device__ __forceinline__ void fen_remove(int *fen, int n, int idx /* 0-based */) {
  for (int i = idx + 1; i <= n; i += i & -i) fen[i] -= 1;
}

__device__ __forceinline__ void gf_add_outer(double *H, const double *j) {
  for (int a = 0; a < 6; a++)
    for (int b = 0; b < 6; b++) H[a * 6 + b] += j[a] * j[b];
}
// common::logDet(A, true): LLT, 2 * sum log(diag)   (math.hpp:172-202); A is overwritten
__device__ __noinline__ double gf_logdet(double *A) {
  if (!chol<6>(A)) return -INFINITY;
  double s = 0.0;
  for (int c = 0; c < 6; c++) s += log(A[c * 6 + c]);
  return 2.0 * s;
}
__device__ double gf_logdet_with(const double *H, const double *j) {  // logDet(H + J^T J, true)
  double A[36];
  for (int a = 0; a < 6; a++)
    for (int b = 0; b < 6; b++) A[a * 6 + b] = H[a * 6 + b] + j[a] * j[b];
  return gf_logdet(A);
}

// ---- evalFullHessian + the gd_float policy.  One CTA.  The reference adds J^T J feature by feature into one mat_H (surf, then corner),
// and the factor feeds a threshold, so the sum keeps that order: thread e < 21 owns element e of the upper triangle and walks the
// rows in index order, one multiply and one add per row like the host loop; the 21 chains are independent, so they run side by side.
// All threads stage the next tile of rows into shared memory (cp.async, double-buffered) while the 21 walk the current one.
// Unmatched features are walked too: k_gf_jaco left them all-zero rows, each product is +0 or -0, and x + (+-0) == x for every partial sum
// that occurs (the diagonal starts at 1e-6 and grows; an off-diagonal starts at +0 and a sum of +0 with +-0 terms stays +0) — the same
// bits as skipping them, without a flag test in the chain.
constexpr int FH_THREADS = 256;
constexpr int FH_TILE = 448;  // rows per tile: 2 x 21 KB of shared memory
struct FhSet {
  const double *jaco;            // n x 6, 16-byte aligned
  const unsigned char *matched;
  int n;
  const int *d_n;                // nullable device-side count
};
__global__ void __launch_bounds__(FH_THREADS) k_gf_full_hessian(FhSet s0, FhSet s1, const double *H_in, const double *__restrict__ cfg,
                                                                GfFloatState *__restrict__ st, double *H_out /* may be H_in */,
                                                                int *__restrict__ feat_io) {
  __shared__ __align__(16) double tile[2][FH_TILE * 6];
  __shared__ double Hs[21], A[36];  // the triangle, then the full matrix the Cholesky overwrites
  __shared__ int s_cnt;
  const int tid = threadIdx.x;
  int ea = 0, eb = 0;  // element tid of the upper triangle, row-major: (0,0) (0,1) ... (0,5) (1,1) ...
  for (int e = 0, a = 0; a < 6; a++)
    for (int b = a; b < 6; b++, e++)
      if (e == tid) ea = a, eb = b;
  double acc = H_in ? H_in[ea * 6 + eb] : (ea == eb ? 1e-6 : 0.0);  // mat_H = I * 1e-6 (:461)
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  int cnt = 0;
  for (int set = 0; set < 2; set++) {
    const FhSet S = set ? s1 : s0;
    const int n = S.d_n ? min(S.n, *S.d_n) : S.n;
    const int tiles = (n + FH_TILE - 1) / FH_TILE;
    auto stage = [&](int k) {  // rows [k * FH_TILE, ...) -> tile[k & 1], 16 B per copy (a row is 3 of them)
      const int rows = min(FH_TILE, n - k * FH_TILE);
      const double *src = S.jaco + (size_t)k * FH_TILE * 6;
      for (int q = tid; q < rows * 3; q += FH_THREADS) __pipeline_memcpy_async(&tile[k & 1][q * 2], src + q * 2, 16);
      __pipeline_commit();
    };
    if (tiles > 0) stage(0);
    for (int k = 0; k < tiles; k++) {
      if (k + 1 < tiles) stage(k + 1);
      __pipeline_wait_prior(k + 1 < tiles ? 1 : 0);
      __syncthreads();
      if (tid < 21) {
        const double *r = tile[k & 1];
        const int rows = min(FH_TILE, n - k * FH_TILE);
        for (int i = 0; i < rows; i++) acc += r[i * 6 + ea] * r[i * 6 + eb];
      }
      __syncthreads();  // tile[k & 1] is staged again two iterations on
    }
    for (int i = tid; i < n; i += FH_THREADS) cnt += S.matched[i] ? 1 : 0;
  }
  if (tid < 21) Hs[tid] = acc;
  if (cnt) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  if (tid == 0) {
    for (int e = 0, a = 0; a < 6; a++)
      for (int b = a; b < 6; b++, e++) A[a * 6 + b] = A[b * 6 + a] = Hs[e];
    if (H_out)
      for (int i = 0; i < 36; i++) H_out[i] = A[i];
    const int total = (feat_io ? *feat_io : 0) + s_cnt;
    if (feat_io) *feat_io = total;
    if (st) {  // :470-492
      const double f = gf_logdet(A);
      st->deg_factor = f, st->total_feat_num = total, st->evaluations += 1;
      st->ratio_cur = f > cfg[0] ? cfg[1] : 0.8;  // <= MAP_DEG_THRE takes 0.8
    }
  }
}

struct GfArgs {
  int method;  // 0 wo_gf, 1 rnd, 2 fps, 3 gd
  double gf_ratio;
  const double *d_ratio;  // nullable: the ratio on the device (gd_float, GfFloatState::ratio_cur), read in place of gf_ratio
  unsigned long long seed;
  int n;
  const int *d_n;  // nullable device-side feature count (n is then the upper bound the buffers are sized for)
  const unsigned char *matched;
  const double *jaco;
  const float4 *pts;
  unsigned char *mask;  // nullable out: mask[i] = 1 for selected features, 0 otherwise (i < n)
  int *fen;      // n + 1
  int *visited;  // n   (gd: round stamp per pool element; fps: visited flag)
  float *dist;   // n   (fps)
  int *sel;      // out, selection order
  int *n_sel;    // out
  double *H;     // out 36
  int smem_ints; // words of dynamic shared memory the launch provides for the pool
};

__global__ void __launch_bounds__(GF_THREADS) k_gf_select(GfArgs a) {
  __shared__ double H[36];
  __shared__ int s_num_sel, s_stop, s_pick;
  __shared__ float red_d[GF_THREADS / 32];
  __shared__ int red_j[GF_THREADS / 32];
  __shared__ int cand[32];
  const int tid = threadIdx.x, lane = tid & 31;
  const int n = a.d_n ? min(a.n, *a.d_n) : a.n;
  // The selection is a chain of dependent pool operations (16-step Fenwick descents, visited marks) issued by ONE thread: in
  // global memory every step is an L2 round trip; the pool lives in shared memory whenever it fits
  // (a.smem_ints words of dynamic shared memory: Fenwick tree first, then the visited marks).
  extern __shared__ int gf_smem[];
  int *const fen = (n + 1 <= a.smem_ints) ? gf_smem : a.fen;
  int *const visited = (2 * n + 1 <= a.smem_ints) ? gf_smem + (n + 1) : a.visited;
  const bool matched_in_smem = 2 * n + 1 + (n + 3) / 4 <= a.smem_ints;
  unsigned char *const matched_s = reinterpret_cast<unsigned char *>(gf_smem + (2 * n + 1));
  if (matched_in_smem)
    for (int i = tid; i < n; i += GF_THREADS) matched_s[i] = a.matched[i];
  const unsigned char *const matched = matched_in_smem ? matched_s : a.matched;
  if (a.mask)
    for (int i = tid; i < n; i += GF_THREADS) a.mask[i] = 0;
  const int num_use = (int)((size_t)((size_t)n * (a.d_ratio ? *a.d_ratio : a.gf_ratio)));  // static_cast<size_t>(num_all_features * gf_ratio), :248
  if (tid < 36) H[tid] = (tid % 7 == 0) ? 1e-6 : 0.0;              // sub_mat_H = I * 1e-6 (:504, :519)
  if (tid == 0) s_num_sel = 0, s_stop = 0, s_pick = -1;
  for (int i = tid; i <= n; i += GF_THREADS) fen[i] = i & -i;    // Fenwick tree of an all-ones array
  for (int i = tid; i < n; i += GF_THREADS) visited[i] = a.method == 2 ? 0 : -1, a.dist[i] = 1e5f;
  __syncthreads();
  int top = 1;
  while (top * 2 <= n) top *= 2;
  unsigned long long rng = gf_seed(a.seed);

  if (a.method == 0) {  // wo_gf (:257-299): every matched feature, in order
    if (tid == 0) {
      int k = 0;
      for (int q = 0; q < n; q++)
        if (matched[q]) gf_add_outer(H, a.jaco + (size_t)q * 6), a.sel[k++] = q;
      s_num_sel = k;
    }
  } else if (a.method == 1) {  // rnd (:300-346)
    if (tid == 0) {
      int k = 0, size = n;
      while (k < num_use && size > 0) {
        const int j = gf_uniform(rng, 0, size - 1);
        const int q = fen_find_kth(fen, n, top, j);
        if (matched[q]) gf_add_outer(H, a.jaco + (size_t)q * 6), a.sel[k++] = q;
        fen_remove(fen, n, q);
        size--;
      }
      s_num_sel = k;
    }
  } else if (a.method == 2) {  // fps (:347-449)
    if (n > 0) {
      int old = 0;
      if (tid == 0) {
        const int k0 = gf_uniform(rng, 0, n - 1);
        visited[k0] = 1;
        if (matched[k0]) a.sel[0] = k0, s_num_sel = 1;  // selected, but never added to sub_mat_H (:375-379)
        s_pick = k0;
      }
      __syncthreads();
      old = s_pick;
      int cnt_visited = 1;
      while (true) {
        if (s_num_sel >= num_use || cnt_visited >= n) break;  // uniform: s_num_sel is only written between barriers
        const float4 po = a.pts[old];
        float best_d = -1.0f;
        int best_j = 0x7fffffff;  // none: no d2 > -1 on this thread
        for (int j = tid; j < n; j += GF_THREADS) {
          if (visited[j]) continue;
          const float4 pn = a.pts[j];
          const float dx = po.x - pn.x, dy = po.y - pn.y, dz = po.z - pn.z;
          const float d = sqrtf(dx * dx + dy * dy + dz * dz);
          const float dj = a.dist[j];
          const float d2 = dj < d ? dj : d;  // std::min(d, dist[j]) (:410): a NaN d stays NaN, so a non-finite point is never the arg-max
          a.dist[j] = d2;
          if (d2 > best_d) best_d = d2, best_j = j;  // ascending j per thread: the first maximum wins, as in the reference
        }
        // arg-max over the block: larger distance, then smaller index
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float od = __shfl_down_sync(MLOAM_FULL_MASK, best_d, o);
          const int oj = __shfl_down_sync(MLOAM_FULL_MASK, best_j, o);
          if (od > best_d || (od == best_d && oj < best_j)) best_d = od, best_j = oj;
        }
        if (lane == 0) red_d[tid >> 5] = best_d, red_j[tid >> 5] = best_j;
        __syncthreads();
        if (tid == 0) {
          float bd = red_d[0];
          int bj = red_j[0];
          for (int w = 1; w < GF_THREADS / 32; w++)
            if (red_d[w] > bd || (red_d[w] == bd && red_j[w] < bj)) bd = red_d[w], bj = red_j[w];
          // no unvisited point with d2 > -1 (all that remain are non-finite): best_j keeps its initial 1 (:402), visited or not
          const int q = bj == 0x7fffffff ? 1 : bj;
          visited[q] = 1;
          if (matched[q]) gf_add_outer(H, a.jaco + (size_t)q * 6), a.sel[s_num_sel] = q, s_num_sel = s_num_sel + 1;
          s_pick = q;
        }
        __syncthreads();
        old = s_pick;
        cnt_visited++;
      }
    }
  } else if (tid < 32) {  // gd_fix / gd_float (:450-556), warp 0
    int size = n, num_sel = 0, num_rnd_que = 0;
    // at least 1: the reference's subset of 0 (num_use > n) pops its first candidate at once (heap.size() >= 0), as a subset of 1 does
    const int size_rnd_subset = num_use > 0 ? max(1, (int)(1.0 * n / num_use)) : 0;
    while (true) {
      if (num_sel >= num_use || size == 0) break;
      int heap_n = 0, best_idx = -1;
      double best_score = 0.0;
      bool round_done = false, give_up = false;
      while (!round_done && !give_up) {
        // lane 0 draws up to 32 matched candidates for this round (or fewer if the round's quota needs fewer)
        int n_cand = 0;
        if (lane == 0) {
          const int want = min(32, size_rnd_subset - heap_n);
          while (n_cand < want) {
            if (size == 0) break;
            num_rnd_que = 0;
            int j = 0, q = -1;
            while (num_rnd_que < kGfMaxRandomQueue) {
              j = gf_uniform(rng, 0, size - 1);
              q = fen_find_kth(fen, n, top, j);
              if (visited[q] < num_sel) {
                visited[q] = num_sel;
                break;
              }
              num_rnd_que++;
            }
            if (num_rnd_que >= kGfMaxRandomQueue) break;
            if (!matched[q]) {  // "not found constraints or outlier constraints" (:518-523): leaves the pool
              fen_remove(fen, n, q);
              size--;
              continue;
            }
            cand[n_cand++] = q;
          }
        }
        n_cand = __shfl_sync(MLOAM_FULL_MASK, n_cand, 0);
        size = __shfl_sync(MLOAM_FULL_MASK, size, 0);
        num_rnd_que = __shfl_sync(MLOAM_FULL_MASK, num_rnd_que, 0);
        __syncwarp();
        // log det(H + J^T J) of the drawn candidates, one per lane; best = larger score, then drawn earlier
        double sc = -INFINITY;
        int order = 0x7fffffff, cidx = -1;
        if (lane < n_cand) {
          cidx = cand[lane];
          // a round of ONE candidate (gf_ratio > 0.5: size_rnd_subset == 1) picks it whatever its score: skip the 6x6 Cholesky
          sc = size_rnd_subset > 1 ? gf_logdet_with(H, a.jaco + (size_t)cidx * 6) : 0.0;
          order = heap_n + lane;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double os = __shfl_down_sync(MLOAM_FULL_MASK, sc, o);
          const int oo = __shfl_down_sync(MLOAM_FULL_MASK, order, o), oi = __shfl_down_sync(MLOAM_FULL_MASK, cidx, o);
          if (oi >= 0 && (cidx < 0 || os > sc || (os == sc && oo < order))) sc = os, order = oo, cidx = oi;
        }
        sc = __shfl_sync(MLOAM_FULL_MASK, sc, 0), cidx = __shfl_sync(MLOAM_FULL_MASK, cidx, 0);
        if (n_cand > 0 && (heap_n == 0 || sc > best_score)) best_score = sc, best_idx = cidx;
        heap_n += n_cand;
        __syncwarp();
        if (heap_n >= size_rnd_subset && heap_n > 0) {  // pop the heap's top: the round's pick
          if (lane < 6) {  // sub_mat_H += J^T J: one row per lane (the same single addition per element as the sequential loop)
            const double *jb = a.jaco + (size_t)best_idx * 6;
            const double ja = jb[lane];
            for (int b = 0; b < 6; b++) H[lane * 6 + b] += ja * jb[b];
          }
          if (lane == 0) {
            fen_remove(fen, n, best_idx);
            a.sel[num_sel] = best_idx;
          }
          size--;
          num_sel++;
          round_done = true;
        } else if (size == 0 || num_rnd_que >= kGfMaxRandomQueue) {
          give_up = true;  // pool exhausted or 20 fruitless draws: the partially filled heap is dropped
        }
        __syncwarp();
      }
      if (num_rnd_que >= kGfMaxRandomQueue) break;
      if (give_up) break;
    }
    if (lane == 0) s_num_sel = num_sel;
  }
  __syncthreads();
  if (tid < 36) a.H[tid] = H[tid];
  if (tid == 0) *a.n_sel = s_num_sel;
  if (a.mask)
    for (int k = tid; k < s_num_sel; k += GF_THREADS) a.mask[a.sel[k]] = 1;
}

// The selection's work for n features in B (Jacobian rows | fen | visited | dist | sel | n_sel | H | mask, then the cov_vec staging of
// the host path when cov != nullptr): *jaco and the work pointers of a are set, a.jaco = *jaco
static int gf_work(Ctx *c, DevBuf &B, int n, GfArgs *a, double **jaco, float **cov) {
  MLOAM_CUDA_OK(c, carve(B, [&](Carve &cv) {
    a->jaco = *jaco = cv.take<double>(6 * (size_t)n), a->fen = cv.take<int>((size_t)n + 1), a->visited = cv.take<int>(n), a->dist = cv.take<float>(n);
    a->sel = cv.take<int>(n), a->n_sel = cv.take<int>(4), a->H = cv.take<double>(36), a->mask = cv.take<unsigned char>((size_t)n + 16);
    if (cov) *cov = cv.take<float>(6 * (size_t)n);
  }));
  return MLOAM_OK;
}

// k_gf_select over the rows of a.jaco (one CTA)
static int gf_select_launch(Ctx *c, GfArgs &a) {
  ProfScope ps(c, "gf_select");
  a.smem_ints = kGfSmemInts;
  if (!c->smem_opt_in_gf) {
    MLOAM_CUDA_OK(c, cudaFuncSetAttribute(k_gf_select, cudaFuncAttributeMaxDynamicSharedMemorySize, kGfSmemInts * (int)sizeof(int)));
    c->smem_opt_in_gf = true;
  }
  k_gf_select<<<1, GF_THREADS, kGfSmemInts * sizeof(int), c->stream>>>(a);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// Device-resident selection of one matched feature set (inside scan2MapOptimization): no host round trip.
int gf_select_set_device(Ctx *c, int t, const FeatSet &fs, const double *d_pose7, double default_sinfo, int method, double gf_ratio,
                         unsigned long long seed, unsigned char **d_mask_out, const double *d_ratio, int phase) {
  const int n = fs.n;
  *d_mask_out = nullptr;
  if (n <= 0) return MLOAM_OK;
  GfArgs a;
  double *d_jaco;
  int rc = gf_work(c, c->gf_work[t], n, &a, &d_jaco, nullptr);
  if (rc) return rc;
  if (phase & 1) {
    k_gf_jaco<<<(n + 127) / 128, 128, 0, c->stream>>>(fs.pts, fs.valid, fs.coeff, n, fs.d_n, fs.is_plane ? 1 : 0, nullptr, fs.sinfo, default_sinfo,
                                                     d_pose7, d_jaco);
    c->launches++;
  }
  if (!(phase & 2)) return MLOAM_OK;
  a.method = method, a.gf_ratio = gf_ratio, a.d_ratio = d_ratio, a.seed = seed, a.n = n, a.d_n = fs.d_n;
  a.matched = fs.valid, a.pts = fs.pts;
  rc = gf_select_launch(c, a);
  if (rc) return rc;
  *d_mask_out = a.mask;
  return MLOAM_OK;
}

static int full_hessian_launch(Ctx *c, const FhSet &s0, const FhSet &s1, const double *d_H_in, const double *d_cfg, GfFloatState *d_st,
                               double *d_H_out, int *d_feat_io) {
  ProfScope ps(c, "gf_full_hessian");
  k_gf_full_hessian<<<1, FH_THREADS, 0, c->stream>>>(s0, s1, d_H_in, d_cfg, d_st, d_H_out, d_feat_io);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

void stage_gf_float(Ctx *c) { c->pinned->gf_float_cfg[0] = (double)c->cfg.gf_float_thre, c->pinned->gf_float_cfg[1] = (double)c->params.gf_ratio; }

int gf_full_hessian_device(Ctx *c, const FeatSet *sets) {
  GfFloatDev *d = c->gf_float.as<GfFloatDev>();
  stage_gf_float(c);
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d->cfg, c->pinned->gf_float_cfg, sizeof(d->cfg), cudaMemcpyHostToDevice, c->stream));
  FhSet fs[2];  // [0] surf (sets[1]), [1] corner (sets[0]): the order of :463-467
  for (int k = 0; k < 2; k++) {
    const FeatSet &S = sets[1 - k];
    GfArgs a;
    double *d_jaco = nullptr;
    if (S.n > 0) {
      const int rc = gf_work(c, c->gf_work[1 - k], S.n, &a, &d_jaco, nullptr);  // where phase 1 left the rows
      if (rc) return rc;
    }
    fs[k] = FhSet{d_jaco, S.valid, S.n > 0 ? S.n : 0, S.d_n};
  }
  return full_hessian_launch(c, fs[0], fs[1], nullptr, d->cfg, &d->st, nullptr, nullptr);
}

}  // namespace mloam

using namespace mloam;

static int good_features_impl(mloam_ctx_t *h, int slot, int type, const mloam_point_t *h_pts, int n, const float *h_cov6, const double *pose7,
                              const double *odom_x21, int method, double gf_ratio, unsigned long long seed, int *h_sel, int *n_sel, double *H36,
                              unsigned char *h_matched, double *h_jaco);

extern "C" int mloam_good_features(mloam_ctx_t *h, int slot, int type, const mloam_point_t *h_pts, int n, const float *h_cov6,
                                   const double *pose7, int method, double gf_ratio, unsigned long long seed, int *h_sel, int *n_sel,
                                   double *H36, unsigned char *h_matched, double *h_jaco) {
  return good_features_impl(h, slot, type, h_pts, n, h_cov6, pose7, nullptr, method, gf_ratio, seed, h_sel, n_sel, H36, h_matched, h_jaco);
}

// Estimator::goodFeatureMatching (estimator.cpp:1347-1517): features of frame i matched at pose_local = pivot^-1 * pose_i * ext
// (n_neigh 5, CHECK_FOV false), rows from evaluateFeatJacobian, every matched feature when gf_ratio == 1.0 (:1380-1414), else the
// stochastic greedy selection.
extern "C" int mloam_good_features_odom(mloam_ctx_t *h, int slot, int type, const mloam_point_t *h_pts, int n, const double *pose_pivot7,
                                        const double *pose_i7, const double *ext7, double gf_ratio, unsigned long long seed, int *h_sel, int *n_sel,
                                        double *H36, unsigned char *h_matched, double *h_jaco) {
  if (!pose_pivot7 || !pose_i7 || !ext7) return MLOAM_E_INVALID;
  double x21[21], local[7];
  for (int k = 0; k < 7; k++) x21[k] = pose_pivot7[k], x21[7 + k] = pose_i7[k], x21[14 + k] = ext7[k];
  {  // Pose(pose_pivot.T_.inverse() * pose_i.T_ * pose_ext.T_) (:1358)
    const PoseD P = pose_from_param(pose_pivot7), I = pose_from_param(pose_i7), E = pose_from_param(ext7);
    const Q4 qpi = qconj(qnormalized(P.q));
    const Q4 q = qnormalized(qmul(qpi, qmul(I.q, E.q)));
    const D3 t = qrot(qpi, (qrot(I.q, E.t) + I.t) - P.t);
    local[0] = t.x, local[1] = t.y, local[2] = t.z, local[3] = q.x, local[4] = q.y, local[5] = q.z, local[6] = q.w;
  }
  return good_features_impl(h, slot, type, h_pts, n, nullptr, local, x21, gf_ratio == 1.0 ? 0 : 3, gf_ratio, seed, h_sel, n_sel, H36, h_matched, h_jaco);
}

// Phase 1 of a host-buffer call: the features go up, are matched against map `slot` at pose7 and get their Jacobian rows (odom_x21: the
// odometry-side rows) in Ctx::host_work, whose regions *a and *d_jaco then name.  fixed5: n_neigh 5 and CHECK_FOV false whatever the
// parameters say (estimator.cpp:1377; lidar_mapper.h:187,193).
static int gf_rows_host(Ctx *c, int slot, int type, const mloam_point_t *h_pts, int n, const float *h_cov6, const double *pose7,
                        const double *odom_x21, bool fixed5, GfArgs *a, double **d_jaco) {
  const int t = type == 's' ? 1 : 0;
  MLOAM_CUDA_OK(c, c->scan_pts[t].reserve(sizeof(float4) * (size_t)n));
  int rc = reserve_feat(c, t, n);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->scan_pts[t].p, h_pts, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  double *d_pose;
  rc = upload_pose(c, pose7, &d_pose);
  if (rc) return rc;
  MatchCfg mcfg = match_cfg(c);
  if (fixed5) mcfg.n_neigh = 5, mcfg.check_fov = 0;
  rc = match_from_map_device(c, slot, type, c->scan_pts[t].as<float4>(), n, nullptr, d_pose, mcfg,
                             c->feat_valid[t].as<unsigned char>(), c->feat_coeff[t].as<float>(), nullptr);
  if (rc) return rc;
  float *d_cov = nullptr;
  rc = gf_work(c, c->host_work, n, a, d_jaco, h_cov6 ? &d_cov : nullptr);
  if (rc) return rc;
  if (h_cov6) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_cov, h_cov6, sizeof(float) * 6 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  if (odom_x21) {
    double *stage = c->pinned->odom_x;
    for (int k = 0; k < 21; k++) stage[k] = odom_x21[k];
    double *d_x21 = c->ctl.as<DevCtl>()->odom_x;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_x21, stage, 21 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    k_gf_jaco_odom<<<(n + 127) / 128, 128, 0, c->stream>>>(c->scan_pts[t].as<float4>(), c->feat_valid[t].as<unsigned char>(), c->feat_coeff[t].as<float>(),
                                                          n, type == 's' ? 1 : 0, d_x21, *d_jaco);
  } else {
    k_gf_jaco<<<(n + 127) / 128, 128, 0, c->stream>>>(c->scan_pts[t].as<float4>(), c->feat_valid[t].as<unsigned char>(), c->feat_coeff[t].as<float>(), n,
                                                     nullptr, type == 's' ? 1 : 0, d_cov, nullptr, map_sqrt_info(c->params.cov_trace), d_pose, *d_jaco);
  }
  c->launches++;
  a->matched = c->feat_valid[t].as<unsigned char>(), a->pts = c->scan_pts[t].as<float4>();
  return MLOAM_OK;
}

static int good_features_impl(mloam_ctx_t *h, int slot, int type, const mloam_point_t *h_pts, int n, const float *h_cov6, const double *pose7,
                              const double *odom_x21, int method, double gf_ratio, unsigned long long seed, int *h_sel, int *n_sel, double *H36,
                              unsigned char *h_matched, double *h_jaco) {
  if (!h || n < 0 || !pose7 || !n_sel || !H36 || method < 0 || method > 3 || !(gf_ratio >= 0.0) || gf_ratio > 1.0 ||
      (n > 0 && (!h_pts || !h_sel)) || (type != 's' && type != 'c'))
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  *n_sel = 0;
  for (int i = 0; i < 36; i++) H36[i] = (i % 7 == 0) ? 1e-6 : 0.0;
  if (n == 0) return MLOAM_OK;
  GfArgs a;
  double *d_jaco;
  int rc = gf_rows_host(c, slot, type, h_pts, n, h_cov6, pose7, odom_x21, odom_x21 != nullptr, &a, &d_jaco);
  if (rc) return rc;
  a.method = method, a.gf_ratio = gf_ratio, a.d_ratio = nullptr, a.seed = seed, a.n = n, a.d_n = nullptr, a.mask = nullptr;
  rc = gf_select_launch(c, a);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(n_sel, a.n_sel, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(H36, a.H, 36 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_sel, a.sel, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  if (h_matched) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_matched, a.matched, (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  if (h_jaco) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_jaco, d_jaco, sizeof(double) * 6 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}

// ActiveFeatureSelection::evalFullHessian (lidar_mapper.h:176-227) for one feature set: H36 and *feat_num accumulate
extern "C" int mloam_full_hessian(mloam_ctx_t *h, int slot, int type, const mloam_point_t *h_pts, int n, const float *h_cov6, const double *pose7,
                                  double *H36, int *feat_num) {
  if (!h || n < 0 || !pose7 || !H36 || !feat_num || (n > 0 && !h_pts) || (type != 's' && type != 'c')) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (n == 0) return MLOAM_OK;
  GfArgs a;
  double *d_jaco;
  int rc = gf_rows_host(c, slot, type, h_pts, n, h_cov6, pose7, nullptr, true, &a, &d_jaco);
  if (rc) return rc;
  // the caller's mat_H and feat_num go to the selection's H and n_sel words, and come back from there
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(a.H, H36, 36 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(a.n_sel, feat_num, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  rc = full_hessian_launch(c, FhSet{d_jaco, a.matched, n, nullptr}, FhSet{nullptr, nullptr, 0, nullptr}, a.H, nullptr, nullptr, a.H, a.n_sel);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(H36, a.H, 36 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(feat_num, a.n_sel, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}
