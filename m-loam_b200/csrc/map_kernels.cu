// map_kernels.cu — GPU map build (direct-indexed voxel grid, common.cuh) and the stand-alone exact kNN (sm_90a).
//
//   map build  : replaces pcl::KdTreeFLANN::setInputCloud (lidar_mapper_keyframe.cpp:433-434): a counting sort of the
//                points by cell over a dense grid — bounding box, per-cell counts (one atomicAdd per point gives its rank
//                inside the cell), exclusive prefix over the cells, scatter.  Every pass streams the points once with
//                coalesced 16-byte loads; grid geometry is decided on the device (no host round trip, graph-capturable).
//   k_knn      : replaces nearestKSearch (feature_extract.hpp:406,570,666,813), see knn.cuh
#include "ctx.h"
#include "knn.cuh"

namespace mloam {

// ------------------------------------------------------------------------------------------- build
constexpr int GB_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_TILE = GB_THREADS * SCAN_ITEMS;  // cells per CTA of the prefix-scan kernels

// order-preserving float <-> int (for atomicMin / atomicMax on coordinates)
__device__ __forceinline__ int f2ord(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }
__device__ __forceinline__ bool finite3(const float4 &p) {
  return fabsf(p.x) < 3.0e37f && fabsf(p.y) < 3.0e37f && fabsf(p.z) < 3.0e37f;  // false for NaN and Inf
}

__global__ void k_grid_reset(GridHdr *h) {
  if (threadIdx.x == 0) {
    for (int k = 0; k < 3; k++) h->bb_min[k] = 0x7fffffff, h->bb_max[k] = (int)0x80000000;
    h->ticket = 0, h->n_sorted = 0, h->n_occupied = 0;
  }
}

// Bounding box of the finite points (pcl::KdTreeFLANN drops non-finite points from the index too).
__global__ void __launch_bounds__(GB_THREADS) k_grid_bbox(const float4 *__restrict__ pts, int m, GridHdr *h) {
  int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {(int)0x80000000, (int)0x80000000, (int)0x80000000};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const float4 p = __ldg(pts + i);
    if (!finite3(p)) continue;
    const int x = f2ord(p.x), y = f2ord(p.y), z = f2ord(p.z);
    lo[0] = min(lo[0], x), lo[1] = min(lo[1], y), lo[2] = min(lo[2], z);
    hi[0] = max(hi[0], x), hi[1] = max(hi[1], y), hi[2] = max(hi[2], z);
  }
  __shared__ int s_lo[3], s_hi[3];
  if (threadIdx.x < 3) s_lo[threadIdx.x] = 0x7fffffff, s_hi[threadIdx.x] = (int)0x80000000;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const int a = __reduce_min_sync(MLOAM_FULL_MASK, lo[k]), b = __reduce_max_sync(MLOAM_FULL_MASK, hi[k]);
    if ((threadIdx.x & 31) == 0) atomicMin(&s_lo[k], a), atomicMax(&s_hi[k], b);
  }
  __syncthreads();
  if (threadIdx.x < 3) atomicMin(&h->bb_min[threadIdx.x], s_lo[threadIdx.x]), atomicMax(&h->bb_max[threadIdx.x], s_hi[threadIdx.x]);
}

// Grid geometry from the bounding box: the requested cell edge doubles until the dense grid fits `cap` cells.
__global__ void k_grid_dims(GridHdr *h, float cell_req, unsigned cap) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float cell = cell_req;
  int level = 0;
  if (h->bb_min[0] > h->bb_max[0]) {  // no finite point
    h->ox = h->oy = h->oz = 0, h->nx = h->ny = h->nz = 1, h->n_cells = 1, h->level = 0, h->cell = cell, h->inv_cell = 1.0f / cell;
    return;
  }
  float lo[3], hi[3];
  for (int k = 0; k < 3; k++) lo[k] = ord2f(h->bb_min[k]), hi[k] = ord2f(h->bb_max[k]);
  for (;; level++, cell *= 2.0f) {
    const float inv = 1.0f / cell;
    long long o[3], n[3];
    bool fits = true;
    for (int k = 0; k < 3; k++) {
      const float a = floorf(lo[k] * inv), b = floorf(hi[k] * inv);
      if (!(fabsf(a) < 1.0e9f && fabsf(b) < 1.0e9f)) fits = false;  // cell index must fit an int
      o[k] = (long long)a, n[k] = (long long)b - (long long)a + 1;
    }
    if (fits && n[0] * n[1] <= (long long)cap && n[0] * n[1] * n[2] <= (long long)cap) {
      h->ox = (int)o[0], h->oy = (int)o[1], h->oz = (int)o[2], h->nx = (int)n[0], h->ny = (int)n[1], h->nz = (int)n[2];
      h->n_cells = (int)(n[0] * n[1] * n[2]), h->level = level, h->cell = cell, h->inv_cell = inv;
      return;
    }
    if (level > 100) {  // cannot happen for finite coordinates; leave a valid one-cell grid
      h->ox = h->oy = h->oz = 0, h->nx = h->ny = h->nz = 1, h->n_cells = 1, h->level = level, h->cell = cell, h->inv_cell = inv;
      return;
    }
  }
}

__global__ void __launch_bounds__(GB_THREADS) k_grid_clear(unsigned *__restrict__ cells, const GridHdr *__restrict__ h) {
  const int n_tot = h->n_cells + 1;
  const int i4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n_tot) return;
  if (i4 + 3 < n_tot) {
    reinterpret_cast<uint4 *>(cells)[i4 >> 2] = make_uint4(0u, 0u, 0u, 0u);
  } else {
    for (int k = i4; k < n_tot; k++) cells[k] = 0u;
  }
}

__device__ __forceinline__ int cell_index(const GridP &g, const float4 &p) {
  const int x = (int)floorf(p.x * g.inv_cell) - g.ox, y = (int)floorf(p.y * g.inv_cell) - g.oy, z = (int)floorf(p.z * g.inv_cell) - g.oz;
  return (z * g.ny + y) * g.nx + x;  // inside the grid by construction (the bounding box covers every finite point)
}

// Pass 1: one atomicAdd per point on its cell's counter; the returned value is the point's rank inside the cell.
// (Only the ORDER of points inside a cell depends on the arrival order; results never do — kNN ties break on the index.)
__global__ void __launch_bounds__(GB_THREADS) k_grid_count(const float4 *__restrict__ pts, int m, MapView mv, unsigned *__restrict__ cells,
                                                          int *__restrict__ rank_of) {
  const GridP g = load_grid(mv);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const float4 p = __ldg(pts + i);
    int rank = -1;
    if (finite3(p)) rank = (int)atomicAdd(cells + cell_index(g, p), 1u);
    rank_of[i] = rank;
  }
}

__device__ __forceinline__ unsigned block_excl_scan_u32(unsigned v, unsigned *total) {
  __shared__ unsigned ws[GB_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned t = __shfl_up_sync(MLOAM_FULL_MASK, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) ws[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    unsigned w = lane < GB_THREADS / 32 ? ws[lane] : 0u;
#pragma unroll
    for (int o = 1; o < GB_THREADS / 32; o <<= 1) {
      const unsigned t = __shfl_up_sync(MLOAM_FULL_MASK, w, o);
      if (lane >= o) w += t;
    }
    if (lane < GB_THREADS / 32) ws[lane] = w;
  }
  __syncthreads();
  const unsigned base = wid > 0 ? ws[wid - 1] : 0u;
  *total = ws[GB_THREADS / 32 - 1];
  __syncthreads();
  return base + inc - v;
}

// Pass 2a: per-tile sums of the cell counts; the CTA that finishes last turns them into exclusive tile offsets.
__global__ void __launch_bounds__(GB_THREADS) k_grid_scan_a(const unsigned *__restrict__ cells, GridHdr *h, unsigned *__restrict__ tile_sums) {
  const int n_tot = h->n_cells + 1;
  const int n_tiles = (n_tot + SCAN_TILE - 1) / SCAN_TILE;
  if ((int)blockIdx.x >= n_tiles) return;
  const int i0 = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  unsigned sum = 0u, occ = 0u;
  if (i0 + SCAN_ITEMS <= n_tot) {
#pragma unroll
    for (int q = 0; q < SCAN_ITEMS / 4; q++) {
      const uint4 v = __ldg(reinterpret_cast<const uint4 *>(cells + i0) + q);
      sum += v.x + v.y + v.z + v.w;
      occ += (v.x != 0u) + (v.y != 0u) + (v.z != 0u) + (v.w != 0u);
    }
  } else {
    for (int k = i0; k < n_tot; k++) sum += cells[k], occ += cells[k] != 0u;
  }
  unsigned total;
  block_excl_scan_u32(sum, &total);
  unsigned occ_total;
  block_excl_scan_u32(occ, &occ_total);
  __shared__ bool is_last;
  if (threadIdx.x == 0) {
    tile_sums[blockIdx.x] = total;
    if (occ_total) atomicAdd(&h->n_occupied, (int)occ_total);
    __threadfence();
    is_last = atomicAdd(&h->ticket, 1) == n_tiles - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  unsigned carry = 0u;
  for (int base = 0; base < n_tiles; base += GB_THREADS) {
    const int t = base + threadIdx.x;
    const unsigned v = t < n_tiles ? __ldcg(tile_sums + t) : 0u;
    unsigned tot;
    const unsigned ex = block_excl_scan_u32(v, &tot);
    if (t < n_tiles) tile_sums[t] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) h->ticket = 0, h->n_sorted = (int)carry;
}

// Pass 2b: exclusive prefix inside each tile + the tile offset, in place: counts become cell_start.
__global__ void __launch_bounds__(GB_THREADS) k_grid_scan_b(unsigned *__restrict__ cells, const GridHdr *__restrict__ h, const unsigned *__restrict__ tile_sums) {
  const int n_tot = h->n_cells + 1;
  const int n_tiles = (n_tot + SCAN_TILE - 1) / SCAN_TILE;
  if ((int)blockIdx.x >= n_tiles) return;
  const int i0 = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  unsigned v[SCAN_ITEMS];
  const bool full = i0 + SCAN_ITEMS <= n_tot;
  if (full) {
#pragma unroll
    for (int q = 0; q < SCAN_ITEMS / 4; q++) {
      const uint4 t = reinterpret_cast<const uint4 *>(cells + i0)[q];
      v[4 * q] = t.x, v[4 * q + 1] = t.y, v[4 * q + 2] = t.z, v[4 * q + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) v[k] = (i0 + k < n_tot) ? cells[i0 + k] : 0u;
  }
  unsigned sum = 0u;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    const unsigned t = v[k];
    v[k] = sum, sum += t;
  }
  unsigned total;
  const unsigned off = block_excl_scan_u32(sum, &total) + tile_sums[blockIdx.x];
  if (full) {
#pragma unroll
    for (int q = 0; q < SCAN_ITEMS / 4; q++)
      reinterpret_cast<uint4 *>(cells + i0)[q] = make_uint4(v[4 * q] + off, v[4 * q + 1] + off, v[4 * q + 2] + off, v[4 * q + 3] + off);
  } else {
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++)
      if (i0 + k < n_tot) cells[i0 + k] = v[k] + off;
  }
}

// Pass 3: scatter.  w of the sorted copy carries the original index.
__global__ void __launch_bounds__(GB_THREADS) k_grid_scatter(const float4 *__restrict__ pts, int m, MapView mv, const int *__restrict__ rank_of,
                                                            float4 *__restrict__ sorted, float4 *__restrict__ orig) {
  const GridP g = load_grid(mv);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    float4 p = __ldg(pts + i);
    if (orig) orig[i] = p;
    const int rank = rank_of[i];
    if (rank < 0) continue;
    const unsigned s = __ldg(mv.cell_start + cell_index(g, p));
    p.w = __int_as_float(i);
    sorted[s + (unsigned)rank] = p;
  }
}

static unsigned grid_capacity(int m) {
  // memory bound of a slot's dense grid (4 B per cell); the device coarsens the cell edge when the bounding box
  // needs more.  Generous on purpose: only the cells of the actual bounding box are ever cleared / scanned.
  unsigned long long want = 16ull * (unsigned long long)(m > 0 ? m : 1);
  if (want < (1ull << 22)) want = 1ull << 22;
  if (want > (1ull << 28)) want = 1ull << 28;
  return (unsigned)want;
}

int map_build_device(Ctx *c, int slot, const float4 *d_pts, int m, float cell) {
  if (slot < 0 || slot >= MLOAM_NUM_MAPS || m < 0) {
    c->err = "map_build: bad slot / size";
    return MLOAM_E_INVALID;
  }
  MapStorage &M = c->maps[slot];
  if (!(cell > 0.f)) cell = M.auto_cell_pick(c->pinned, slot);
  ProfScope ps(c, "map_build");
  const bool keep_orig = slot == MLOAM_MAP_SCAN_CORNER || slot == MLOAM_MAP_SCAN_SURF;
  unsigned cap = grid_capacity(m);
  if (cap < M.capacity) cap = M.capacity;  // never shrink: the buffers are grow-only anyway
  MLOAM_CUDA_OK(c, M.sorted.reserve(sizeof(float4) * (size_t)(m + 1)));
  if (keep_orig) MLOAM_CUDA_OK(c, M.orig.reserve(sizeof(float4) * (size_t)(m + 1)));
  MLOAM_CUDA_OK(c, M.cells.reserve(sizeof(unsigned) * ((size_t)cap + 8)));
  MLOAM_CUDA_OK(c, M.rank_of.reserve(sizeof(int) * (size_t)(m + 1)));
  MLOAM_CUDA_OK(c, M.tile_sums.reserve(sizeof(unsigned) * ((size_t)cap / SCAN_TILE + 8)));
  MLOAM_CUDA_OK(c, M.hdr.reserve(sizeof(GridHdr)));
  M.capacity = cap, M.m = m, M.cell = cell, M.built = true;
  cudaStream_t st = c->stream;
  GridHdr *h = M.hdr.as<GridHdr>();
  const MapView mv = M.view();
  int nb = (m + 4 * GB_THREADS - 1) / (4 * GB_THREADS);  // ~4 points per thread
  if (nb < 1) nb = 1;
  if (nb > 16 * c->sm_count) nb = 16 * c->sm_count;
  k_grid_reset<<<1, 32, 0, st>>>(h);
  if (m > 0) k_grid_bbox<<<nb, GB_THREADS, 0, st>>>(d_pts, m, h);
  k_grid_dims<<<1, 32, 0, st>>>(h, cell, cap);
  const int nb_clear = (int)(((size_t)cap + 1 + 4 * GB_THREADS - 1) / (4 * GB_THREADS));
  k_grid_clear<<<nb_clear, GB_THREADS, 0, st>>>(M.cells.as<unsigned>(), h);
  if (m > 0) k_grid_count<<<nb, GB_THREADS, 0, st>>>(d_pts, m, mv, M.cells.as<unsigned>(), M.rank_of.as<int>());
  const int nb_scan = (int)(((size_t)cap + 1 + SCAN_TILE - 1) / SCAN_TILE);
  k_grid_scan_a<<<nb_scan, GB_THREADS, 0, st>>>(M.cells.as<unsigned>(), h, M.tile_sums.as<unsigned>());
  k_grid_scan_b<<<nb_scan, GB_THREADS, 0, st>>>(M.cells.as<unsigned>(), h, M.tile_sums.as<unsigned>());
  if (m > 0)
    k_grid_scatter<<<nb, GB_THREADS, 0, st>>>(d_pts, m, mv, M.rank_of.as<int>(), M.sorted.as<float4>(), keep_orig ? M.orig.as<float4>() : nullptr);
  c->launches += m > 0 ? 8 : 5;
  // occupancy statistics for the next auto-cell decision of this slot (read lazily by auto_cell_pick; stale is fine)
  if (c->pinned)
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(&c->pinned->map_hdr[slot], h, 48, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------- kNN
constexpr int QWARPS = 8;  // warps (= queries) per block

template <int K>
__global__ void __launch_bounds__(QWARPS * 32)
    k_knn(MapView map, const float4 *__restrict__ q, int nq, const double *__restrict__ pose7, float max_sqdist,
          int *__restrict__ idx, float *__restrict__ sqd, unsigned tma_min) {
  __shared__ KnnSmem ksm[QWARPS];
  const int lane = threadIdx.x & 31;
  KnnSmem &ks = ksm[threadIdx.x >> 5];
  knn_smem_init(ks, lane, tma_min);
  const GridP g = load_grid(map);
  for (int i = blockIdx.x * QWARPS + (threadIdx.x >> 5); i < nq; i += gridDim.x * QWARPS) {
    const float4 p = __ldg(q + i);
    float3 s = make_float3(p.x, p.y, p.z);
    if (pose7) s = associate(pose_from_param(pose7), p.x, p.y, p.z);
    Best best;
    warp_knn<K, false>(map, g, ks, s.x, s.y, s.z, max_sqdist, lane, best);
    if (lane < K) {  // lane r holds the r-th neighbour
      const float d2 = key_d2(best.key);
      const bool ok = best.key != MLOAM_KEY_NONE && d2 < max_sqdist;
      idx[(size_t)i * K + lane] = ok ? (int)(unsigned)(best.key & 0xffffffffu) : -1;
      sqd[(size_t)i * K + lane] = ok ? d2 : INFINITY;
    }
  }
}

int knn_device(Ctx *c, int slot, const float4 *d_q, int nq, const double *d_pose7, int k, float max_sqdist, int *d_idx,
               float *d_sqd) {
  if (slot < 0 || slot >= MLOAM_NUM_MAPS || !c->maps[slot].built) {
    c->err = "knn: map slot not built";
    return MLOAM_E_STATE;
  }
  if (nq <= 0) return MLOAM_OK;
  ProfScope ps(c, "knn");
  MapView mv = c->maps[slot].view();
  int nb = (nq + QWARPS - 1) / QWARPS;
  if (nb > 8 * c->sm_count) nb = 8 * c->sm_count;  // warps stride over the queries
  cudaStream_t st = c->stream;
  switch (k) {
    case 1: k_knn<1><<<nb, QWARPS * 32, 0, st>>>(mv, d_q, nq, d_pose7, max_sqdist, d_idx, d_sqd, c->knn_tma_min); break;
    case 5: k_knn<5><<<nb, QWARPS * 32, 0, st>>>(mv, d_q, nq, d_pose7, max_sqdist, d_idx, d_sqd, c->knn_tma_min); break;
    case 10: k_knn<10><<<nb, QWARPS * 32, 0, st>>>(mv, d_q, nq, d_pose7, max_sqdist, d_idx, d_sqd, c->knn_tma_min); break;
    default: c->err = "knn: k must be 1, 5 or 10"; return MLOAM_E_INVALID;
  }
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

}  // namespace mloam
