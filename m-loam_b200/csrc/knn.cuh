// knn.cuh — exact K-nearest-neighbour search over the direct-indexed voxel grid (common.cuh), one WARP per query.
//
// Replaces pcl::KdTreeFLANN::nearestKSearch (feature_extract.hpp:155,293,406,570,666,813).
// Semantics: the K nearest map points in ascending (squared distance, original index) order, where the
// squared distance is FLANN's L2_Simple in float (dx*dx + dy*dy + dz*dz, rounded per operation), limited
// to points with d2 < max_sqdist — which is all the callers look at: every reference caller rejects the
// query unless sqdist[K-1] < MIN_MATCH_SQ_DIS (or sqdist[0] < DISTANCE_SQ_THRESHOLD for K=1).
//
// Search plan per query (all 32 lanes cooperate; the running best list is DISTRIBUTED: lane r holds the r-th best):
//   ring 1  the 3x3x3 cells around the query's cell are 9 ROWS of 3 x-adjacent cells, i.e. 9 contiguous runs of
//           `sorted`: lanes 0..8 read the two prefix entries that delimit their row (computed addresses, no probing),
//           the runs are staged into this warp's shared-memory tile with 1-D TMA bulk copies (cp.async.bulk +
//           mbarrier complete_tx: every run in flight at once, one memory round trip whatever their number), then the
//           tile is read back as conflict-free float4 and reduced with a warp-wide K-selection.
//           Stop if the K-th distance is inside the visited cube — the common case when the cell edge fits the map's
//           point spacing (map_cell = auto picks it from the occupancy statistics of the previous build).
//   ball    otherwise every row (y, z) of cells that reaches into the ball of radius min(radius, K-th so far) is
//           clipped in x to that ball and staged the same way, 32 rows per step; the bound shrinks between steps.
//           The part of a ring-1 row that has been scanned already is cut out.
// Two memory round trips for a typical query (prefix entries -> points), bounded work for every query: nothing in the
// search depends on hash-chain lengths or on how the points are distributed.
//
// Exactness: float distance in FLANN's operation order, ties on the original index, conservative epsilons on every
// pruning bound (cell membership is floorf(p * inv_cell): a point can sit one rounding error outside its cell's box).
#pragma once
#include "common.cuh"

namespace mloam {

#define MLOAM_KEY_NONE 0xffffffffffffffffull

// Running best list of a warp: lane r (r < N) holds the r-th smallest key seen so far, lanes >= N hold NONE.
// key = (float bits of d2) << 32 | original index; pos = position in MapView::sorted.
struct Best {
  unsigned long long key;
  int pos;
};
__device__ __forceinline__ Best best_none() { return Best{MLOAM_KEY_NONE, -1}; }
__device__ __forceinline__ unsigned long long best_key(const Best &b, int r) { return __shfl_sync(MLOAM_FULL_MASK, b.key, r); }
__device__ __forceinline__ float key_d2(unsigned long long k) { return __uint_as_float((unsigned)(k >> 32)); }

// Per-warp staging tile (shared memory): KNN_TILE points per TMA step + the mbarrier the bulk copies complete on.
constexpr int KNN_TILE = 256;
struct __align__(16) KnnSmem {
  float4 pts[KNN_TILE];
  unsigned long long mbar;
  unsigned phase;  // parity of the next wait (kept by lane 0, broadcast)
  int slot, first;  // the caller's (k_match_knn: the warp's place in its schedule, its first listed feature)
};

// Optional per-query instrumentation of the blind search (stage profiling only).
struct KnnDbg {
  long long t_ring1, t_ball;  // SM cycles per phase
  int ring1_pts, ball_pts, ball_rows, ball_steps;
};

// %laneid read where it is used (volatile: not held in a register across a search)
__device__ __forceinline__ unsigned lane_id() {
  unsigned l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
  unsigned hi = (unsigned)(v >> 32);
  unsigned mh = __reduce_min_sync(MLOAM_FULL_MASK, hi);
  unsigned lo = (hi == mh) ? (unsigned)v : 0xffffffffu;
  unsigned ml = __reduce_min_sync(MLOAM_FULL_MASK, lo);
  return ((unsigned long long)mh << 32) | ml;
}

__device__ __forceinline__ int warp_excl_scan(int v, int lane, int *total) {
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(MLOAM_FULL_MASK, inc, o);
    if (lane >= o) inc += t;
  }
  *total = __shfl_sync(MLOAM_FULL_MASK, inc, 31);
  return inc - v;
}

// ------------------------------------------------------------------------------------------- mbarrier / TMA (sm_90a)
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void knn_smem_init(KnnSmem &ks, int lane, unsigned = 0u) {
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&ks.mbar)) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    ks.phase = 0u;
  }
  __syncwarp();
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// Distributed best list in split form: lane r < N holds the r-th smallest (d2 bits, index) + its position.
struct BestS {
  unsigned d, i;
  int p;
};
#define MLOAM_D_NONE 0xffffffffu
__device__ __forceinline__ bool key_less(unsigned da, unsigned ia, unsigned db, unsigned ib) { return da < db || (da == db && ia < ib); }

// Stage the runs (one per lane: `count` points from sorted[start], count 0 = none), KNN_TILE points per step, and merge
// them into the best list: the new list is the N smallest of (current best) U (staged points with d2 <= bound).
// Selection works on the 32-bit distance patterns (non-negative floats order like their bits): one REDUX per extracted
// element, the index only breaks ties (rare, warp-uniform branch).  Once the list is full, a step whose candidates beat
// the N-th at most N times inserts them one by one (ballot + popc gives the slot, one shuffle-up shifts the tail).
// bound: float bits of the caller's squared distance bound, MLOAM_D_NONE for none.  A candidate takes part only if it
// beats min(N-th, bound) — with an empty list too, so the points of a row that lie outside the caller's ball (rows are
// clipped at cell granularity) cost one compare and no selection round.  Entries <= bound are those of the unbounded
// list; the callers only look beyond the bound through min(explored, d) with explored below the bound (warp_knn).
// Inlined: out of line, the call ABI saved the caller's live registers around each of its call sites, which alone kept
// k_match_knn above its 72-register budget (match_kernels.cu).
template <int N>
__device__ __forceinline__ Best scan_runs(const float4 *__restrict__ sorted, KnnSmem *ks, int start, int count, float qx, float qy, float qz,
                                       Best best, int *n_points, unsigned bound) {
  constexpr int U = 2;  // candidates per lane and selection step
  const int lane = threadIdx.x & 31;
  int total;
  const int excl = warp_excl_scan(count, lane, &total);
  if (n_points) *n_points += total;
  unsigned phase = ks->phase;  // same value in every lane (written by lane 0 before a __syncwarp)
  BestS e{best.key == MLOAM_KEY_NONE ? MLOAM_D_NONE : (unsigned)(best.key >> 32), (unsigned)best.key, best.pos};
  for (int base = 0; base < total; base += KNN_TILE) {
    const int chunk = min(KNN_TILE, total - base);
    // ---- stage: this lane's part of [base, base + chunk) as one bulk copy; all copies of the step are in flight together
    {
      const int lo = max(excl, base), hi = min(excl + count, base + chunk);
      if (lane == 0) mbar_expect_tx(&ks->mbar, (unsigned)chunk * 16u);
      __syncwarp();
      if (hi > lo) tma_load_1d(&ks->pts[lo - base], sorted + (start + (lo - excl)), (unsigned)(hi - lo) * 16u, &ks->mbar);
      mbar_wait(&ks->mbar, phase);
      phase ^= 1u;
    }
    // ---- select from the tile, 32 * U candidates per step.  A candidate's position is its flat index in this call's
    // concatenated runs, encoded as -(index) - 2 and converted for the survivors at the end.
#pragma unroll 1
    for (int c0 = 0; c0 < chunk; c0 += 32 * U) {
      unsigned cd[U], ci[U];
      // candidate u's encoded position, formed where it is taken rather than held in registers through the rounds
      auto cp = [&](int u) { return -(base + c0 + u * 32 + lane) - 2; };
#pragma unroll
      for (int u = 0; u < U; u++) {
        const int t = c0 + u * 32 + lane;
        cd[u] = MLOAM_D_NONE, ci[u] = 0xffffffffu;
        if (t < chunk) {
          const float4 v = ks->pts[t];
          const float ex = v.x - qx, ey = v.y - qy, ez = v.z - qz;
          const float d2 = ex * ex + ey * ey + ez * ez;
          cd[u] = __float_as_uint(d2), ci[u] = (unsigned)__float_as_int(v.w);
        }
      }
      // how many candidates beat min(N-th, bound)?  The bound as a key is (bound, 0xffffffff): d2 == bound still enters.
      // The others cannot enter the list; they are dropped here so that the selection rounds end with the admitted ones.
      const unsigned nd = __shfl_sync(MLOAM_FULL_MASK, e.d, N - 1), ni = __shfl_sync(MLOAM_FULL_MASK, e.i, N - 1);
      const bool by_bound = bound < nd;
      const unsigned td = by_bound ? bound : nd, ti = by_bound ? 0xffffffffu : ni;
      unsigned beat[U];
      int n_beat = 0;
#pragma unroll
      for (int u = 0; u < U; u++) {
        const bool in = key_less(cd[u], ci[u], td, ti);
        beat[u] = __ballot_sync(MLOAM_FULL_MASK, in);
        n_beat += __popc(beat[u]);
        if (!in) cd[u] = MLOAM_D_NONE;
      }
      if (n_beat == 0) continue;
      if (nd != MLOAM_D_NONE && n_beat <= N) {
        // ---- insertion: the list is full and few candidates matter
#pragma unroll
        for (int u = 0; u < U; u++) {
          unsigned mk = beat[u];
          while (mk) {
            const int src = __ffs(mk) - 1;
            mk &= mk - 1;
            const unsigned xd = __shfl_sync(MLOAM_FULL_MASK, cd[u], src), xi = __shfl_sync(MLOAM_FULL_MASK, ci[u], src);
            const int xp = -(base + c0 + u * 32 + src) - 2;
            const int slot = __popc(__ballot_sync(MLOAM_FULL_MASK, lane < N && key_less(e.d, e.i, xd, xi)));
            const unsigned ud = __shfl_up_sync(MLOAM_FULL_MASK, e.d, 1), ui = __shfl_up_sync(MLOAM_FULL_MASK, e.i, 1);
            const int up = __shfl_up_sync(MLOAM_FULL_MASK, e.p, 1);
            if (slot < N) {
              if (lane > slot && lane < N) e.d = ud, e.i = ui, e.p = up;
              if (lane == slot) e.d = xd, e.i = xi, e.p = xp;
            }
          }
        }
        continue;
      }
      // ---- selection: N rounds, each extracts the smallest remaining of (old list entry of this lane) U (its candidates)
      BestS o = e, n{MLOAM_D_NONE, 0xffffffffu, -1};
#pragma unroll 1
      for (int r = 0; r < N; r++) {
        unsigned ld = o.d, li = o.i;
        int lp = o.p, which = U;
#pragma unroll
        for (int u = 0; u < U; u++)
          if (key_less(cd[u], ci[u], ld, li)) ld = cd[u], li = ci[u], lp = cp(u), which = u;
        const unsigned md = __reduce_min_sync(MLOAM_FULL_MASK, ld);
        if (md == MLOAM_D_NONE) break;  // fewer than N points so far
        unsigned owners = __ballot_sync(MLOAM_FULL_MASK, ld == md);
        if (owners & (owners - 1)) {  // equal distances: the smaller original index first
          const unsigned mi = __reduce_min_sync(MLOAM_FULL_MASK, ld == md ? li : 0xffffffffu);
          owners = __ballot_sync(MLOAM_FULL_MASK, ld == md && li == mi);
        }
        const int src = __ffs(owners) - 1;
        const unsigned wi = __shfl_sync(MLOAM_FULL_MASK, li, src);
        const int wp = __shfl_sync(MLOAM_FULL_MASK, lp, src);
        if (lane == r) n.d = md, n.i = wi, n.p = wp;
        if (lane == src) {
          if (which == U) o.d = MLOAM_D_NONE;
#pragma unroll
          for (int u = 0; u < U; u++)
            if (which == u) cd[u] = MLOAM_D_NONE;
        }
      }
      e = n;
    }
    __syncwarp();  // every lane has read the tile: the next stage may overwrite it
  }
  if (lane == 0) ks->phase = phase;
  // flat indices -> positions in `sorted`: the owning run is the last lane whose exclusive prefix is <= the index
  {
    const int f = e.p <= -2 ? -(e.p + 2) : 0;
    int j = 0;
#pragma unroll
    for (int step = 16; step > 0; step >>= 1) {
      const int v = __shfl_sync(MLOAM_FULL_MASK, excl, j + step);
      if (v <= f) j += step;
    }
    const int st = __shfl_sync(MLOAM_FULL_MASK, start, j), ex = __shfl_sync(MLOAM_FULL_MASK, excl, j);
    if (e.p <= -2) e.p = st + (f - ex);
  }
  __syncwarp();
  best.key = e.d == MLOAM_D_NONE ? MLOAM_KEY_NONE : (((unsigned long long)e.d << 32) | e.i);
  best.pos = e.d == MLOAM_D_NONE ? -1 : e.p;
  return best;
}

// One row of cells (relative coordinates y, z; x range [xl, xh], all inside the grid): its points are sorted[s .. e).
__device__ __forceinline__ void row_run(const MapView &map, const GridP &g, int y, int z, int xl, int xh, int *start, int *count) {
  const size_t base = ((size_t)z * g.ny + y) * g.nx;
  const unsigned s = __ldg(map.cell_start + base + xl), e = __ldg(map.cell_start + base + xh + 1);
  *start = (int)s, *count = (int)(e - s);
}

__device__ __forceinline__ float knn_eps(const GridP &g, float qx, float qy, float qz) {
  return 1e-6f * (fabsf(qx) + fabsf(qy) + fabsf(qz) + 8.0f * g.cell) + 1e-6f;
}
// squared gap between coordinate q and the slab of cell index c (absolute), deflated by eps
__device__ __forceinline__ float slab_gap(float q, int c_abs, float cell, float eps) {
  const float lo = (float)c_abs * cell;
  return fmaxf(fmaxf(lo - q, q - (lo + cell)) - eps, 0.0f);
}

// Scan every cell that reaches into the ball of squared radius `bound2` around q (rows of cells clipped in x to the
// ball), restricted to the cube of Chebyshev radius clip_r (cells) around the query's cell (cx, cy, cz) when
// clip_r >= 0, and without the cube of radius skip_r that has been scanned already when skip_r >= 0.
// `bound2` shrinks while scanning: lim2 = min(max_sqdist, K-th so far) is what the result needs; prune(lim2) adds the
// caller's padding.  Returns false when the scan needs more than max_slots row slots (nothing scanned); the blind
// search passes an unbounded max_slots, so it always scans.  sel(bound2): the selection bound handed to scan_runs.
template <int K, int N, typename Prune, typename Sel>
__device__ __forceinline__ bool scan_ball(const MapView &map, const GridP &g, KnnSmem &ks, float qx, float qy, float qz, int cx, int cy, int cz,
                                          int clip_r, int skip_r, float &lim2, Prune prune, int max_slots, int lane, Best &out, KnnDbg *dbg,
                                          Sel sel) {
  const float eps = knn_eps(g, qx, qy, qz);
  float bound2 = prune(lim2);
  const float R = sqrtf(bound2) * 1.0002f + eps;
  int ylo = (int)floorf((qy - R) * g.inv_cell) - g.oy, yhi = (int)floorf((qy + R) * g.inv_cell) - g.oy;
  int zlo = (int)floorf((qz - R) * g.inv_cell) - g.oz, zhi = (int)floorf((qz + R) * g.inv_cell) - g.oz;
  int xmin = 0, xmax = g.nx - 1;
  if (clip_r >= 0) {
    ylo = max(ylo, cy - clip_r), yhi = min(yhi, cy + clip_r), zlo = max(zlo, cz - clip_r), zhi = min(zhi, cz + clip_r);
    xmin = max(xmin, cx - clip_r), xmax = min(xmax, cx + clip_r);
  }
  ylo = max(ylo, 0), yhi = min(yhi, g.ny - 1), zlo = max(zlo, 0), zhi = min(zhi, g.nz - 1);
  if (ylo > yhi || zlo > zhi || xmin > xmax) return true;
  // clamped to the grid: wy * wz <= ny * nz <= n_cells (< 2^28), so the row count fits an int whatever the ball's size
  const int wy = yhi - ylo + 1, wz = zhi - zlo + 1;
  const int n_rows = wy * wz;
  // a row through the skipped cube splits into the part left of it and the part right of it: those rows get two slots
  const int sw = 2 * skip_r + 1;
  const int n_slots = skip_r >= 0 ? n_rows + sw * sw : n_rows;
  if (n_slots > max_slots) return false;
#pragma unroll 1
  for (int s0 = 0; s0 < n_slots; s0 += 32) {
    const int s = s0 + lane;
    int start = 0, count = 0;
    if (s < n_slots) {
      int y, z, side = 0;  // side 0: whole row / left part, 1: right part of a row through the skipped cube
      if (s < n_rows) {
        y = ylo + s % wy, z = zlo + s / wy;
      } else {
        const int t = s - n_rows;
        y = cy + t % sw - skip_r, z = cz + t / sw - skip_r, side = 1;
      }
      bool take = y >= ylo && y <= yhi && z >= zlo && z <= zhi;
      const bool in_skip = skip_r >= 0 && abs(y - cy) <= skip_r && abs(z - cz) <= skip_r;
      if (side == 1 && !in_skip) take = false;
      if (take) {
        const float gy = slab_gap(qy, y + g.oy, g.cell, eps), gz = slab_gap(qz, z + g.oz, g.cell, eps);
        const float dyz2 = gy * gy + gz * gz;
        if (dyz2 <= bound2) {
          const float hx = sqrtf(bound2 - dyz2) * 1.0002f + eps;
          int xl = (int)floorf((qx - hx) * g.inv_cell) - g.ox, xh = (int)floorf((qx + hx) * g.inv_cell) - g.ox;
          xl = max(xl, xmin), xh = min(xh, xmax);
          if (in_skip) {
            if (side == 0) xh = min(xh, cx - skip_r - 1);
            else xl = max(xl, cx + skip_r + 1);
          }
          if (xl <= xh) row_run(map, g, y, z, xl, xh, &start, &count);
        }
      }
    }
    if (dbg) dbg->ball_steps++, dbg->ball_rows += __popc(__ballot_sync(MLOAM_FULL_MASK, count > 0));
    if (!__any_sync(MLOAM_FULL_MASK, count > 0)) continue;
    out = scan_runs<N>(map.sorted, &ks, start, count, qx, qy, qz, out, dbg ? &dbg->ball_pts : nullptr, sel(bound2));
    const unsigned long long kk = best_key(out, K - 1);
    if (kk != MLOAM_KEY_NONE) lim2 = fminf(lim2, key_d2(kk)), bound2 = fminf(bound2, prune(lim2));
  }
  return true;
}

// Seeded search (temporal coherence between the re-association iterations of one scan2MapOptimization): the caller
// knows K map points — the previous iteration's neighbours — whose largest squared distance to the moved query is
// r2 < max_sqdist.  Every point of the true K-nearest set then lies in the ball of radius sqrt(r2), so scanning the
// cells that intersect that ball gives the exact result, ties included.  pad > 0 widens the ball so that the (K+1)-th
// distance is seen too.  Returns false (nothing written) when the ball needs more than 32 rows.
// *explored: every map point closer than this has been scanned.
// sel_prune: the selection keeps only points with d2 <= rr * rr rounded up.  The K-set is inside (d2 <= r2); a point left
// out has sqrtf(d2) >= rr > *explored, so min(*explored, d) — all the caller reads beyond the K-th — is unchanged.
template <int K, int N>
__device__ __forceinline__ bool warp_knn_seeded(const MapView &map, const GridP &g, KnnSmem &ks, float qx, float qy, float qz, float r2,
                                                float pad, int lane, Best &out, float *explored, bool sel_prune = false) {
  const float eps = knn_eps(g, qx, qy, qz);
  const float rr = sqrtf(r2) * 1.0002f + eps + pad;
  float lim2 = rr * rr;
  const unsigned sel = sel_prune ? __float_as_uint(__fmul_ru(rr, rr)) : MLOAM_D_NONE;
  Best b = best_none();
  // the ball is fixed (the seed bound): no shrinking, so that the explored radius is known
  if (!scan_ball<K, N>(map, g, ks, qx, qy, qz, 0, 0, 0, -1, -1, lim2, [&](float) { return rr * rr; }, 32, lane, b, nullptr,
                       [&](float) { return sel; }))
    return false;
  out = b;
  *explored = fmaxf(rr - 2.0f * eps, 0.0f);
  return true;
}

// distance from q to the nearest face of the cube of Chebyshev radius r (cells) around the absolute cell (ax, ay, az)
__device__ __forceinline__ float cube_face_gap(const GridP &g, float qx, float qy, float qz, int ax, int ay, int az, int r, float eps) {
  float m = qx - (float)(ax - r) * g.cell;
  m = fminf(m, (float)(ax + r + 1) * g.cell - qx);
  m = fminf(m, qy - (float)(ay - r) * g.cell);
  m = fminf(m, (float)(ay + r + 1) * g.cell - qy);
  m = fminf(m, qz - (float)(az - r) * g.cell);
  m = fminf(m, (float)(az + r + 1) * g.cell - qz);
  return m - eps;
}

// The blind search.  N >= K: selection width; with N = K + 1 the extra slot holds the nearest point outside the
// K-set AMONG THE SCANNED ONES.
// *explored (nullable): every map point closer than this has been scanned into `out`.  Hence min(K-th scanned,
// *explored) bounds the true K-th distance from below, and min((K+1)-th scanned, *explored) the (K+1)-th.  pad > 0
// lets the later phases look that much beyond min(radius, K-th), so that the caller also learns how isolated the K-set
// (or how far from K neighbours a rejected query) is; the result inside the radius is unaffected.
// REJECT_PARTIAL is kept for the callers' sake (every matcher gate only wants full K-sets); the grid search has no
// separate partial path.
// sel_prune: the selection keeps only points inside the current pruning bound (ring 1: prune(max_sqdist); then the
// shrinking bound of the shells).  The bounds never drop below the final prune(lim2), so a point left out has
// sqrtf(d2) >= sqrtf(prune(lim2)) > *explored: the K-set and lim2 are unchanged, and min(*explored, d) of the K-th and
// (K+1)-th entries — all the callers read beyond the bound — is too.
template <int K, bool REJECT_PARTIAL, int N = K>
__device__ __forceinline__ void warp_knn(const MapView &map, const GridP &g, KnnSmem &ks, float qx, float qy, float qz, float max_sqdist,
                                         int lane, Best &out, float *explored = nullptr, float pad = 0.0f, KnnDbg *dbg = nullptr,
                                         bool sel_prune = false) {
  long long t_mark = dbg ? clock64() : 0ll;
  out = best_none();
  if (explored) *explored = 0.0f;
  if (!(fabsf(qx) < 3.0e37f && fabsf(qy) < 3.0e37f && fabsf(qz) < 3.0e37f)) return;  // non-finite query: no neighbours
  const int ax = (int)floorf(qx * g.inv_cell), ay = (int)floorf(qy * g.inv_cell), az = (int)floorf(qz * g.inv_cell);  // absolute cell
  const int cx = ax - g.ox, cy = ay - g.oy, cz = az - g.oz;
  const float eps = knn_eps(g, qx, qy, qz);
  // lim2: min(radius^2, K-th so far) — what the result needs; cells are pruned against prune(lim2), which with pad > 0
  // reaches pad beyond sqrt(lim2).
  const float radius = sqrtf(max_sqdist);
  auto prune = [&](float l2) {
    if (!(pad > 0.0f)) return l2;
    const float r = fminf(sqrtf(l2), radius) + pad;
    return fmaxf(l2, r * r);
  };
  auto sel = [&](float bound2) { return sel_prune ? __float_as_uint(bound2) : MLOAM_D_NONE; };
  // ---- ring 1: 9 rows of (up to) 3 cells
  {
    int start = 0, count = 0;
    if (lane < 9) {
      const int y = cy + (int)(lane_id() % 3u) - 1, z = cz + (int)(lane_id() / 3u) - 1;
      const int xl = max(cx - 1, 0), xh = min(cx + 1, g.nx - 1);
      if (y >= 0 && y < g.ny && z >= 0 && z < g.nz && xl <= xh) row_run(map, g, y, z, xl, xh, &start, &count);
    }
    if (__any_sync(MLOAM_FULL_MASK, count > 0))
      out = scan_runs<N>(map.sorted, &ks, start, count, qx, qy, qz, out, dbg ? &dbg->ring1_pts : nullptr, sel(prune(max_sqdist)));
    if (dbg) {
      const long long t = clock64();
      dbg->t_ring1 = t - t_mark, t_mark = t;
    }
  }
  float lim2 = max_sqdist;
  {
    const unsigned long long kk = best_key(out, K - 1);
    if (kk != MLOAM_KEY_NONE) lim2 = fminf(lim2, key_d2(kk));
  }
  // ---- shells: the cube of Chebyshev radius r around the query's cell is complete after shell r.  Nearest-first
  // matters: the K-th distance found in shell r bounds everything scanned afterwards.  Stop as soon as the covered cube
  // contains the ball the result needs.  (The result itself needs lim2; the pad only steers how much further we look.)
  float covered = cube_face_gap(g, qx, qy, qz, ax, ay, az, 1, eps);
#pragma unroll 1
  for (int r = 2;; r++) {
    if (covered > 0.0f && covered * covered >= lim2) break;
    if (r > 5) {  // many thin shells left (tiny cells): one pass over the rest of the ball
      scan_ball<K, N>(map, g, ks, qx, qy, qz, cx, cy, cz, -1, r - 1, lim2, prune, 1 << 30, lane, out, dbg, sel);
      covered = 3.0e38f;
      break;
    }
    scan_ball<K, N>(map, g, ks, qx, qy, qz, cx, cy, cz, r, r - 1, lim2, prune, 1 << 30, lane, out, dbg, sel);
    covered = cube_face_gap(g, qx, qy, qz, ax, ay, az, r, eps);
  }
  if (dbg) dbg->t_ball = clock64() - t_mark;
  // every point closer than min(covered cube, final pruning bound) has been scanned (bounds never dropped below the final one)
  if (explored) *explored = fmaxf(fminf(covered, sqrtf(prune(lim2)) - eps), 0.0f);
}

}  // namespace mloam
