// extract_kernels.cu — FeatureExtract::extractCloud (feature_extract.cpp:118-297) and the PCL voxel-grid
// filters on its path (pcl::VoxelGrid<PointI>, feature_extract.cpp:267-270; VoxelGridCovarianceMLOAM<PointI>,
// lidar_mapper_keyframe.cpp:359-364; algorithm mirrored in-tree at voxel_grid_covariance_mloam_impl.hpp:84-250).
//
//   k_curvature      11-tap stencil over the flat ring-major array (:133-142) + consecutive-gap flags (:194-197)
//   k_ring_pick      one CTA per ring: one bitonic sort of (sector, curvature, offset) in shared memory (:160-162),
//                    then the data-dependent sharp / less-sharp / flat picks with +-5 suppression (:165-256)
//   k_ring_voxel     one CTA per ring: label <= 0 compaction (:258-264) + per-ring pcl::VoxelGrid(0.2) (:266-271) with an
//                    in-CTA sort; k_ring_voxel_emit concatenates the rings
//   voxel pipeline   whole-cloud filters: bbox -> voxel index -> stable radix sort (two launches per 8-bit pass) -> run
//                    heads -> ordered centroid sums; clouds of <= 2048 points take the in-CTA path (k_voxel_small)
//
// Float arithmetic follows the reference's evaluation order; integer/index results are exact.
#include "ctx.h"
#include "cal_timestamp.cuh"
#include "project.cuh"
#include "primitives.cuh"

namespace mloam {

// ------------------------------------------------------------------------------------------ primitives
__global__ void k_prim_tile_sums(const int *__restrict__ in, int n, int *__restrict__ tile_sums) {
  const int base = blockIdx.x * PRIM_TILE + threadIdx.x * PRIM_ITEMS;
  int s = 0;
#pragma unroll
  for (int k = 0; k < PRIM_ITEMS; k++)
    if (base + k < n) s += in[base + k];
  int total;
  prim_block_scan(s, &total);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
__global__ void k_prim_scan_tiles(int *tile_sums, int n_tiles, int *total_out) {
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_tiles; base += PRIM_THREADS) {
    const int i = base + threadIdx.x;
    const int v = i < n_tiles ? tile_sums[i] : 0;
    int total;
    const int ex = prim_block_scan(v, &total);
    if (i < n_tiles) tile_sums[i] = carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0 && total_out) *total_out = carry;
}
__global__ void k_prim_scan_apply(const int *__restrict__ in, int n, const int *__restrict__ tile_sums, int *__restrict__ out) {
  const int base = blockIdx.x * PRIM_TILE + threadIdx.x * PRIM_ITEMS;
  int c[PRIM_ITEMS];
  int s = 0;
#pragma unroll
  for (int k = 0; k < PRIM_ITEMS; k++) {
    c[k] = (base + k < n) ? in[base + k] : 0;
    s += c[k];
  }
  int ex = prim_block_scan(s, nullptr) + tile_sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < PRIM_ITEMS; k++) {
    if (base + k < n) out[base + k] = ex;
    ex += c[k];
  }
}

// exclusive scan d_in[0..n) -> d_out (may alias), optional device total.  tmp must hold ceil(n/PRIM_TILE) ints.
void scan_exclusive(Ctx *c, const int *d_in, int *d_out, int n, int *d_tmp, int *d_total) {
  if (n <= 0) {
    if (d_total) cudaMemsetAsync(d_total, 0, sizeof(int), c->stream);
    return;
  }
  const int nt = (n + PRIM_TILE - 1) / PRIM_TILE;
  k_prim_tile_sums<<<nt, PRIM_THREADS, 0, c->stream>>>(d_in, n, d_tmp);
  k_prim_scan_tiles<<<1, PRIM_THREADS, 0, c->stream>>>(d_tmp, nt, d_total);
  k_prim_scan_apply<<<nt, PRIM_THREADS, 0, c->stream>>>(d_in, n, d_tmp, d_out);
  c->launches += 3;
}

// Stable LSD radix sort, 8-bit digits.  Tile layout: warp w of the block owns keys
// [blk*TILE + w*256, +256), visited in 8 rounds of 32 consecutive keys -> input order is preserved per digit.
// hist[b * 256 + d] = keys of block b with digit d.  The block that finishes last turns the table into the exclusive
// prefix the scatter needs (digit-major, block-minor order) — the three scan launches of a pass folded into this one.
// d_n_valid (nullable): device-side key count; blocks beyond it contribute nothing.
__global__ void k_rs_hist(const unsigned long long *__restrict__ keys, int n, const int *__restrict__ d_n_valid, int shift,
                          int *__restrict__ hist, int nblk, unsigned *__restrict__ ticket) {
  __shared__ int h[256];
  __shared__ bool is_last;
  if (d_n_valid) n = min(n, *d_n_valid);
  h[threadIdx.x] = 0;
  __syncthreads();
  const int base = blockIdx.x * PRIM_TILE;
#pragma unroll
  for (int k = 0; k < PRIM_ITEMS; k++) {
    const int i = base + k * PRIM_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&h[(int)((keys[i] >> shift) & 0xffull)], 1);
  }
  __syncthreads();
  hist[blockIdx.x * 256 + threadIdx.x] = h[threadIdx.x];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  int *col = hist + threadIdx.x;  // thread d owns digit d: entries col[b * 256], coalesced across the block
  int sum = 0;
#pragma unroll 8
  for (int b = 0; b < nblk; b++) sum += __ldcg(col + b * 256);
  int run = prim_block_scan(sum, nullptr);
#pragma unroll 8
  for (int b = 0; b < nblk; b++) {
    const int t = __ldcg(col + b * 256);
    col[b * 256] = run;
    run += t;
  }
  if (threadIdx.x == 0) *ticket = 0u;
}
__global__ void k_rs_scatter(const unsigned long long *__restrict__ keys, const unsigned *__restrict__ vals, int n,
                             const int *__restrict__ d_n_valid, int shift, const int *__restrict__ offs, int nblk,
                             unsigned long long *__restrict__ keys_out, unsigned *__restrict__ vals_out) {
  __shared__ int cnt[PRIM_THREADS / 32][256];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (d_n_valid) n = min(n, *d_n_valid);
  if (blockIdx.x * PRIM_TILE >= n) return;
  for (int k = threadIdx.x; k < (PRIM_THREADS / 32) * 256; k += PRIM_THREADS) (&cnt[0][0])[k] = 0;
  __syncthreads();
  const int wbase = blockIdx.x * PRIM_TILE + w * (PRIM_ITEMS * 32);
  unsigned long long kk[PRIM_ITEMS];
  int rank[PRIM_ITEMS];
#pragma unroll
  for (int it = 0; it < PRIM_ITEMS; it++) {
    const int i = wbase + it * 32 + lane;
    const bool ok = i < n;
    kk[it] = ok ? keys[i] : 0ull;
    const int d = (int)((kk[it] >> shift) & 0xffull);
    const unsigned act = __ballot_sync(MLOAM_FULL_MASK, ok);
    rank[it] = 0;
    if (ok) {
      const unsigned peers = __match_any_sync(act, d);
      const int before = __popc(peers & ((1u << lane) - 1u));
      rank[it] = cnt[w][d] + before;
      __syncwarp(act);
      if (before == 0) cnt[w][d] += __popc(peers);
    }
    __syncwarp();
  }
  __syncthreads();
  {  // per digit: exclusive prefix over the block's warps
    const int d = threadIdx.x;
    int run = 0;
#pragma unroll
    for (int ww = 0; ww < PRIM_THREADS / 32; ww++) {
      const int t = cnt[ww][d];
      cnt[ww][d] = run;
      run += t;
    }
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < PRIM_ITEMS; it++) {
    const int i = wbase + it * 32 + lane;
    if (i < n) {
      const int d = (int)((kk[it] >> shift) & 0xffull);
      const int pos = offs[blockIdx.x * 256 + d] + cnt[w][d] + rank[it];
      keys_out[pos] = kk[it];
      vals_out[pos] = vals[i];
    }
  }
}

struct SortBufs {
  unsigned long long *k0, *k1;
  unsigned *v0, *v1;
  int *hist;  // 256 * nblk
  int *tmp;   // scan tiles
  unsigned *ticket;  // zero before the first pass (k_seg_init), self-resetting
};
// Sorts the first min(n, *d_n_valid) entries of (k0,v0) by the low `nbits` of the key; returns which buffer holds the
// result (0 or 1).  Two launches per 8-bit pass.
static int radix_sort(Ctx *c, SortBufs b, int n, const int *d_n_valid, int nbits) {
  if (n <= 0) return 0;
  const int nblk = (n + PRIM_TILE - 1) / PRIM_TILE;
  int cur = 0;
  for (int shift = 0; shift < nbits; shift += 8) {
    unsigned long long *ki = cur ? b.k1 : b.k0, *ko = cur ? b.k0 : b.k1;
    unsigned *vi = cur ? b.v1 : b.v0, *vo = cur ? b.v0 : b.v1;
    k_rs_hist<<<nblk, PRIM_THREADS, 0, c->stream>>>(ki, n, d_n_valid, shift, b.hist, nblk, b.ticket);
    k_rs_scatter<<<nblk, PRIM_THREADS, 0, c->stream>>>(ki, vi, n, d_n_valid, shift, b.hist, nblk, ko, vo);
    c->launches += 2;
    cur ^= 1;
  }
  return cur;
}

// ------------------------------------------------------------------------------------------ voxel grid
__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

struct SegBox {           // per segment
  unsigned mn[3], mx[3];  // ordered-uint encodings of min / max
};

__global__ void k_seg_init(SegBox *box, int n_seg, unsigned *ticket) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *ticket = 0u;
  if (i < n_seg) {
    for (int d = 0; d < 3; d++) box[i].mn[d] = 0xffffffffu, box[i].mx[d] = 0u;
  }
}
// getMinMax3D over finite points (voxel_grid_covariance_mloam_impl.hpp:84-90)
__global__ void k_seg_bbox(const float4 *__restrict__ pts, const int *__restrict__ seg, int n, const int *__restrict__ d_n_valid,
                           SegBox *box) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (d_n_valid) n = min(n, *d_n_valid);
  const bool in = i < n;
  float4 p = in ? pts[i] : make_float4(0, 0, 0, 0);
  const bool ok = in && isfinite(p.x) && isfinite(p.y) && isfinite(p.z);
  const int s = in ? (seg ? seg[i] : 0) : -1;
  const int s0 = __shfl_sync(MLOAM_FULL_MASK, s, 0);
  const bool uniform = __all_sync(MLOAM_FULL_MASK, s == s0 || !in);
  unsigned mn[3] = {ok ? f2ord(p.x) : 0xffffffffu, ok ? f2ord(p.y) : 0xffffffffu, ok ? f2ord(p.z) : 0xffffffffu};
  unsigned mx[3] = {ok ? f2ord(p.x) : 0u, ok ? f2ord(p.y) : 0u, ok ? f2ord(p.z) : 0u};
  if (uniform && s0 >= 0) {
#pragma unroll
    for (int d = 0; d < 3; d++) {
      mn[d] = __reduce_min_sync(MLOAM_FULL_MASK, mn[d]);
      mx[d] = __reduce_max_sync(MLOAM_FULL_MASK, mx[d]);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
      for (int d = 0; d < 3; d++) {
        if (mn[d] != 0xffffffffu) atomicMin(&box[s0].mn[d], mn[d]);
        if (mx[d] != 0u) atomicMax(&box[s0].mx[d], mx[d]);
      }
    }
  } else if (ok) {
#pragma unroll
    for (int d = 0; d < 3; d++) atomicMin(&box[s].mn[d], mn[d]), atomicMax(&box[s].mx[d], mx[d]);
  }
}

// Voxel key per point: (segment << 32) | idx with idx = ijk . (1, div0, div0*div1)   (:206-222).
// A segment whose index space would overflow int32 is passed through unchanged (:92-101): every point gets
// its own key (position inside the segment).  Non-finite points get the all-ones key and are dropped later.
__global__ void k_voxel_keys(const float4 *__restrict__ pts, const int *__restrict__ seg, const int *__restrict__ seg_begin, int n,
                             const int *__restrict__ d_n_valid, float inv, const SegBox *__restrict__ box,
                             unsigned long long *__restrict__ keys, unsigned *__restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  vals[i] = (unsigned)i;
  if (d_n_valid && i >= *d_n_valid) {  // beyond the device-side count: dropped like a non-finite point
    keys[i] = 0xffffffffffffffffull;
    return;
  }
  const float4 p = pts[i];
  const int s = seg ? seg[i] : 0;
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) {
    keys[i] = 0xffffffffffffffffull;
    return;
  }
  const SegBox b = box[s];
  const float mn0 = ord2f(b.mn[0]), mn1 = ord2f(b.mn[1]), mn2 = ord2f(b.mn[2]);
  const float mx0 = ord2f(b.mx[0]), mx1 = ord2f(b.mx[1]), mx2 = ord2f(b.mx[2]);
  const long long dx = (long long)((mx0 - mn0) * inv) + 1, dy = (long long)((mx1 - mn1) * inv) + 1,
                  dz = (long long)((mx2 - mn2) * inv) + 1;
  unsigned idx;
  if (dx * dy * dz > 2147483647ll) {
    idx = (unsigned)(i - (seg_begin ? seg_begin[s] : 0));
  } else {
    const int minb0 = (int)floorf(mn0 * inv), minb1 = (int)floorf(mn1 * inv), minb2 = (int)floorf(mn2 * inv);
    const int maxb0 = (int)floorf(mx0 * inv), maxb1 = (int)floorf(mx1 * inv);
    const int div0 = maxb0 - minb0 + 1, div1 = maxb1 - minb1 + 1;
    const int i0 = (int)(floorf(p.x * inv) - (float)minb0);
    const int i1 = (int)(floorf(p.y * inv) - (float)minb1);
    const int i2 = (int)(floorf(p.z * inv) - (float)minb2);
    idx = (unsigned)(i0 + i1 * div0 + i2 * (div0 * div1));
  }
  keys[i] = ((unsigned long long)(unsigned)s << 32) | idx;
}

__global__ void k_run_heads(const unsigned long long *__restrict__ keys, int n, const int *__restrict__ d_n_valid, int *__restrict__ head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (d_n_valid && i >= *d_n_valid) {  // beyond the device-side count: never sorted, never a run
    head[i] = 0;
    return;
  }
  const unsigned long long k = keys[i];
  head[i] = (k != 0xffffffffffffffffull && (i == 0 || keys[i - 1] != k)) ? 1 : 0;
}

// One thread per run head: accumulate the run in sorted (= input) order in float, divide by the float count
// (Eigen 3.3 `centroid /= float(n)`).  intensity_last: VoxelGridCovarianceMLOAM keeps the last point's intensity
// (voxel_grid_covariance_mloam_impl.hpp:417-428); otherwise pcl::VoxelGrid averages every field.
__global__ void k_centroids(const float4 *__restrict__ pts, const unsigned long long *__restrict__ keys,
                            const unsigned *__restrict__ vals, const int *__restrict__ head, const int *__restrict__ slot, int n,
                            const int *__restrict__ d_n_valid, int intensity_last, float4 *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (d_n_valid) n = min(n, *d_n_valid);
  if (i >= n || !head[i]) return;
  const unsigned long long k = keys[i];
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f, last = 0.f;
  int j = i;
  for (; j < n && keys[j] == k; j++) {
    const float4 p = pts[vals[j]];
    sx = sx + p.x, sy = sy + p.y, sz = sz + p.z, si = si + p.w;
    last = p.w;
  }
  const float cnt = (float)(j - i);
  out[slot[i]] = make_float4(sx / cnt, sy / cnt, sz / cnt, intensity_last ? last : si / cnt);
}

// VoxelGridCovarianceMLOAM<PointIWithCov>: the covariance-weighted merge of a voxel (voxel_grid_covariance_mloam_impl.hpp:293-333),
// one thread per run head, float arithmetic in the reference's order: w = thr - trace (points with |trace| >= thr are skipped),
// mu += w * xyz, intensity of the heaviest point, cov(7) += (w * w) * [cov_vec | cov_trace], then / W and / (W * W);
// the output trace is recomputed from the merged diagonal (:332).
struct CovIO {
  const float *cov6_in;    // n * 6
  const float *trace_in;   // n
  float *cov6_out, *trace_out;
  float trace_threshold;
  const SegBox *box;       // the cloud's bounding box: the int32-overflow case copies the input through (:92-101)
  float inv;
};
__global__ void k_centroids_cov(const float4 *__restrict__ pts, const unsigned long long *__restrict__ keys, const unsigned *__restrict__ vals,
                                const int *__restrict__ head, const int *__restrict__ slot, int n, const int *__restrict__ d_n_valid, CovIO io,
                                float4 *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (d_n_valid) n = min(n, *d_n_valid);
  if (i >= n || !head[i]) return;
  const unsigned long long k = keys[i];
  {
    const SegBox b = io.box[0];
    const float mn0 = ord2f(b.mn[0]), mn1 = ord2f(b.mn[1]), mn2 = ord2f(b.mn[2]);
    const float mx0 = ord2f(b.mx[0]), mx1 = ord2f(b.mx[1]), mx2 = ord2f(b.mx[2]);
    const long long dx = (long long)((mx0 - mn0) * io.inv) + 1, dy = (long long)((mx1 - mn1) * io.inv) + 1, dz = (long long)((mx2 - mn2) * io.inv) + 1;
    if (dx * dy * dz > 2147483647ll) {  // "leaf size is too small": output = input (every point is its own run here)
      const unsigned q = vals[i];
      const int o = slot[i];
      out[o] = pts[q];
#pragma unroll
      for (int a = 0; a < 6; a++) io.cov6_out[(size_t)o * 6 + a] = io.cov6_in[(size_t)q * 6 + a];
      io.trace_out[o] = io.trace_in[q];
      return;
    }
  }
  float mu0 = 0.f, mu1 = 0.f, mu2 = 0.f, ity = 0.f, wt = 0.f, w_max = 0.f;
  float cov[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int j = i; j < n && keys[j] == k; j++) {
    const unsigned q = vals[j];
    const float4 p = pts[q];
    const float *c6 = io.cov6_in + (size_t)q * 6;
    const float tr = c6[0] + c6[3] + c6[5];
    if (fabsf(tr) >= io.trace_threshold) continue;
    const float w = io.trace_threshold - tr;
    mu0 = mu0 + w * p.x, mu1 = mu1 + w * p.y, mu2 = mu2 + w * p.z;
    ity = w > w_max ? p.w : ity;
    w_max = w > w_max ? w : w_max;
    const float ww = w * w;
#pragma unroll
    for (int a = 0; a < 6; a++) cov[a] = cov[a] + ww * c6[a];
    cov[6] = cov[6] + ww * io.trace_in[q];
    wt = wt + w;
  }
  if (wt == 0.f) wt = 1.0f;
  const float w2 = wt * wt;
  const int o = slot[i];
  out[o] = make_float4(mu0 / wt, mu1 / wt, mu2 / wt, ity);
#pragma unroll
  for (int a = 0; a < 6; a++) cov[a] = cov[a] / w2;
#pragma unroll
  for (int a = 0; a < 6; a++) io.cov6_out[(size_t)o * 6 + a] = cov[a];
  io.trace_out[o] = cov[0] + cov[3] + cov[5];
}

// Shared voxel pipeline.  scratch layout is owned by the caller (VoxelWork).
struct VoxelWork {
  SegBox *box;
  unsigned long long *k0, *k1;
  unsigned *v0, *v1;
  int *hist, *tmp, *head, *slot;
  unsigned *ticket;
};
static int voxel_pipeline(Ctx *c, const float4 *d_pts, const int *d_seg, const int *d_seg_begin, int n, const int *d_n_valid,
                          int n_seg, float leaf, int intensity_last, VoxelWork w, float4 *d_out, int *d_n_out, const CovIO *cov = nullptr) {
  cudaStream_t st = c->stream;
  if (n <= 0) {
    cudaMemsetAsync(d_n_out, 0, sizeof(int), st);
    return MLOAM_OK;
  }
  const float inv = 1.0f / leaf;
  const int nb = (n + 255) / 256;
  k_seg_init<<<(n_seg + 127) / 128, 128, 0, st>>>(w.box, n_seg, w.ticket);
  k_seg_bbox<<<nb, 256, 0, st>>>(d_pts, d_seg, n, d_n_valid, w.box);
  k_voxel_keys<<<nb, 256, 0, st>>>(d_pts, d_seg, d_seg_begin, n, d_n_valid, inv, w.box, w.k0, w.v0);
  c->launches += 3;
  int seg_bits = 0;
  while ((1 << seg_bits) < n_seg) seg_bits++;
  SortBufs sb{w.k0, w.k1, w.v0, w.v1, w.hist, w.tmp, w.ticket};
  // all-ones keys (non-finite points) must sort last: include the full 64 bits only when a segment id is present
  const int nbits = n_seg > 1 ? 32 + ((seg_bits + 7) / 8) * 8 : 32;
  const int cur = radix_sort(c, sb, n, d_n_valid, nbits);
  const unsigned long long *ks = cur ? w.k1 : w.k0;
  const unsigned *vs = cur ? w.v1 : w.v0;
  k_run_heads<<<nb, 256, 0, st>>>(ks, n, d_n_valid, w.head);
  c->launches++;
  scan_exclusive(c, w.head, w.slot, n, w.tmp, d_n_out);
  if (cov) {
    CovIO io = *cov;
    io.box = w.box, io.inv = inv;
    k_centroids_cov<<<nb, 256, 0, st>>>(d_pts, ks, vs, w.head, w.slot, n, d_n_valid, io, d_out);
  }
  else k_centroids<<<nb, 256, 0, st>>>(d_pts, ks, vs, w.head, w.slot, n, d_n_valid, intensity_last, d_out);
  c->launches++;
  return MLOAM_OK;
}

static int voxel_work_reserve(Ctx *c, DevBuf &buf, int n, int n_seg, VoxelWork *w) {
  const int nblk = (n + PRIM_TILE - 1) / PRIM_TILE + 1;
  const int n_hist = 256 * nblk;
  const int n_tmp = (std::max(n, n_hist) + PRIM_TILE - 1) / PRIM_TILE + 1;
  const size_t n1 = (size_t)n + 1;
  MLOAM_CUDA_OK(c, carve(buf, [&](Carve &cv) {
    w->box = cv.take<SegBox>(n_seg + 1);
    w->k0 = cv.take<unsigned long long>(n1), w->k1 = cv.take<unsigned long long>(n1);
    w->v0 = cv.take<unsigned>(n1), w->v1 = cv.take<unsigned>(n1);
    w->hist = cv.take<int>(n_hist), w->tmp = cv.take<int>(n_tmp);
    w->head = cv.take<int>(n1), w->slot = cv.take<int>(n1);
    w->ticket = cv.take<unsigned>(4);
  }));
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ range-image projection
// ImageSegmenter::segmentCloud with segment_flag_ == false (image_segmenter.hpp:88-136, 381-389; parameters image_segmenter.cpp:18-63):
// every point gets a (row, column) pixel of the vertical_scans x horizon_scans range image, the first point (input order) of a pixel wins,
// intensity += row, and the output is the rows concatenated, each in input order; ScanInfo = [row begin + 5, row end - 6].
// The float arithmetic follows the reference expression by expression (explicitly rounded operations, fdlibm atanf / atan2f — fd_atan.cuh).
// Batched over a rig (RigLayout): LiDAR l has an image of its own and its rows are rows l * vertical_scans + r of the output.
__device__ __forceinline__ int rig_lidar_of(const RigLayout &L, int i) {
  int l = 0;
  while (l + 1 < L.n_lidars && i >= L.off[l + 1]) l++;
  return l;
}
__global__ void k_project_pixels(const float4 *__restrict__ P, int n, ProjectParam sp, RigLayout L, int *__restrict__ pix,
                                 int *__restrict__ winner) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int row = 0;
  int px = project_pixel(sp, P[i], &row);
  if (px >= 0 && L.n_lidars > 1) px += rig_lidar_of(L, i) * sp.vertical_scans * sp.horizon_scans;
  pix[i] = px;
  if (px >= 0) atomicMin(&winner[px], i);
}
__global__ void k_project_keys(const int *__restrict__ pix, const int *__restrict__ winner, int n, int horizon_scans,
                               unsigned long long none, unsigned long long *__restrict__ keys, unsigned *__restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int px = pix[i];
  keys[i] = (px >= 0 && winner[px] == i) ? (unsigned long long)(px / horizon_scans) : none;  // (lidar, row)
  vals[i] = (unsigned)i;
}
__global__ void k_project_emit(const float4 *__restrict__ P, const unsigned long long *__restrict__ keys, const unsigned *__restrict__ vals,
                               int n, unsigned long long none, int vertical_scans, float4 *__restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned long long k = keys[j];
  if (k >= none) return;
  float4 p = P[vals[j]];
  p.w = __fadd_rn(p.w, (float)(int)(k % (unsigned long long)vertical_scans));
  out[j] = p;
}
// r in 0..n_rows: first sorted position whose (lidar, row) key is >= r
__global__ void k_project_rows(const unsigned long long *__restrict__ keys, int n, int n_rows, int *__restrict__ scan_start,
                               int *__restrict__ scan_end, int *__restrict__ n_out) {
  __shared__ int begin[MLOAM_MAX_RINGS + 1];
  for (int r = threadIdx.x; r <= n_rows; r += blockDim.x) {
    int lo = 0, hi = n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (keys[mid] < (unsigned long long)r) lo = mid + 1;
      else hi = mid;
    }
    begin[r] = lo;
  }
  __syncthreads();
  for (int r = threadIdx.x; r <= n_rows; r += blockDim.x) {
    if (r < n_rows) scan_start[r] = begin[r] + 5, scan_end[r] = begin[r + 1] - 6;
    else *n_out = begin[r];
  }
}

// ------------------------------------------------------------------------------------------ calTimestamp
// FeatureExtract::calTimestamp (feature_extract.cpp:25-114, cal_timestamp.cuh) per LiDAR of a rig after removeNaNFromPointCloud, without a
// compaction: ends[l] / ends[16 + l] = first / last finite point of LiDAR l, ends[32 + l] = its flip index (first point whose first-half
// angle sets half_passed).  The start / end angles of every LiDAR (findStartEndAngle) are computed once per CTA of k_front_flip into shared
// memory, and CTA 0 leaves them in `angles` (start | end) for k_front_times.  The timed cloud keeps the input order; a dropped point
// becomes an all-NaN point, which no pixel takes.
__global__ void k_front_ends(const float4 *__restrict__ P, int n, RigLayout L, int *__restrict__ ends) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !ts_finite(P[i])) return;
  const int l = rig_lidar_of(L, i);
  atomicMin(&ends[l], i);
  atomicMax(&ends[MLOAM_MAX_LIDARS + l], i);
}
__global__ void k_front_flip(const float4 *__restrict__ P, int n, RigLayout L, int *__restrict__ ends, float *__restrict__ angles) {
  __shared__ float ang[2 * MLOAM_MAX_LIDARS];
  const int t = threadIdx.x;
  if (t < L.n_lidars) {
    float start_ori = 0.f, end_ori = 0.f;
    if (ends[MLOAM_MAX_LIDARS + t] >= 0) ts_start_end(P[ends[t]], P[ends[MLOAM_MAX_LIDARS + t]], &start_ori, &end_ori);  // else: no finite point
    ang[t] = start_ori, ang[MLOAM_MAX_LIDARS + t] = end_ori;
    if (blockIdx.x == 0) angles[t] = start_ori, angles[MLOAM_MAX_LIDARS + t] = end_ori;
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + t;
  if (i >= n) return;
  const float4 p = P[i];
  if (!ts_finite(p)) return;
  const int l = rig_lidar_of(L, i);
  bool flips;
  ts_ori_first_half(p, ang[l], &flips);
  if (flips) atomicMin(&ends[2 * MLOAM_MAX_LIDARS + l], i);
}
__global__ void k_front_times(const float4 *__restrict__ P, int n, RigLayout L, int time_field, float scan_period, const int *__restrict__ ends,
                              const float *__restrict__ angles, float4 *__restrict__ out, int *__restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = P[i];
  const bool fin = ts_finite(p);
  if (keep) keep[i] = fin ? 1 : 0;
  if (!fin) {
    const float q = __int_as_float(0x7fc00000);
    out[i] = make_float4(q, q, q, q);
    return;
  }
  float t;
  if (time_field) t = ts_from_stamp(p.w);
  else {
    const int l = rig_lidar_of(L, i);
    t = ts_point_time_at(p, i - L.off[l], angles[l], angles[MLOAM_MAX_LIDARS + l], ends[2 * MLOAM_MAX_LIDARS + l] - L.off[l], 0, scan_period);
  }
  out[i] = make_float4(p.x, p.y, p.z, t);
}

// work of project_cloud_device / front_times_device in `buf` for n points and n_pix pixels
struct ProjectWork {
  SortBufs sb;
  int *pix, *winner, *ends;
  float *angles;
  float4 *timed;
};
static int project_work_reserve(Ctx *c, DevBuf &buf, int n, size_t n_pix, ProjectWork *w) {
  const int nblk = (n + PRIM_TILE - 1) / PRIM_TILE + 1;
  const int n_hist = 256 * nblk;
  const int n_tmp = (std::max(n, n_hist) + PRIM_TILE - 1) / PRIM_TILE + 1;
  const size_t n1 = (size_t)n + 1;
  MLOAM_CUDA_OK(c, carve(buf, [&](Carve &cv) {
    w->sb.k0 = cv.take<unsigned long long>(n1), w->sb.k1 = cv.take<unsigned long long>(n1);
    w->sb.v0 = cv.take<unsigned>(n1), w->sb.v1 = cv.take<unsigned>(n1);
    w->sb.hist = cv.take<int>(n_hist), w->sb.tmp = cv.take<int>(n_tmp), w->sb.ticket = cv.take<unsigned>(4);
    w->pix = cv.take<int>(n1), w->winner = cv.take<int>(n_pix), w->ends = cv.take<int>(3 * MLOAM_MAX_LIDARS);
    w->angles = cv.take<float>(2 * MLOAM_MAX_LIDARS);
    w->timed = cv.take<float4>(n1);
  }));
  return MLOAM_OK;
}

static int front_times(Ctx *c, const float4 *d_in, const RigLayout &L, int time_field, float scan_period, const ProjectWork &w, float4 *d_out,
                       int *d_keep) {
  const int n = L.off[L.n_lidars];
  if (n <= 0) return MLOAM_OK;
  ProfScope ps(c, "front_end");
  cudaStream_t st = c->stream;
  const int nb = (n + 255) / 256;
  if (!time_field) {
    MLOAM_CUDA_OK(c, cudaMemsetAsync(w.ends, 0x7f, sizeof(int) * 3 * MLOAM_MAX_LIDARS, st));
    MLOAM_CUDA_OK(c, cudaMemsetAsync(w.ends + MLOAM_MAX_LIDARS, 0xff, sizeof(int) * MLOAM_MAX_LIDARS, st));
    k_front_ends<<<nb, 256, 0, st>>>(d_in, n, L, w.ends);
    k_front_flip<<<nb, 256, 0, st>>>(d_in, n, L, w.ends, w.angles);
    c->launches += 2;
  }
  k_front_times<<<nb, 256, 0, st>>>(d_in, n, L, time_field, scan_period, w.ends, w.angles, d_out, d_keep);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}
__global__ void k_front_compact(const float4 *__restrict__ timed, const int *__restrict__ keep, const int *__restrict__ slot, int n,
                                float4 *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && keep[i]) out[slot[i]] = timed[i];
}
int front_times_device(Ctx *c, const float4 *d_in, const RigLayout &L, int time_field, float scan_period, float4 *d_out, int *d_n_out,
                       DevBuf &work) {
  const int n = L.off[L.n_lidars];
  ProjectWork w;
  int rc = project_work_reserve(c, work, n, 1, &w);
  if (rc) return rc;
  rc = front_times(c, d_in, L, time_field, scan_period, w, w.timed, w.pix);
  if (rc) return rc;
  int *slot = reinterpret_cast<int *>(w.sb.v0);
  scan_exclusive(c, w.pix, slot, n, w.sb.tmp, d_n_out);
  k_front_compact<<<(n + 255) / 256, 256, 0, c->stream>>>(w.timed, w.pix, slot, n, d_out);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

int project_cloud_device(Ctx *c, const float4 *d_in, const RigLayout &L, int vertical_scans, int horizon_scans, double roi_range,
                         const FrontEnd *fe, float4 *d_out, int *d_scan_start, int *d_scan_end, int *d_n_out, DevBuf &work) {
  const int n = L.off[L.n_lidars];
  if (L.n_lidars < 1 || L.n_lidars > MLOAM_MAX_LIDARS) {
    c->err = "project_cloud: the rig must have 1 to 16 LiDARs";
    return MLOAM_E_INVALID;
  }
  if (n <= 0 || horizon_scans <= 0) {
    c->err = "project_cloud: empty cloud or horizon_scans <= 0";
    return MLOAM_E_INVALID;
  }
  if (vertical_scans != 16 && vertical_scans != 32 && vertical_scans != 64) {
    c->err = "project_cloud: vertical_scans must be 16, 32 or 64 (ImageSegmenter::setParameter)";
    return MLOAM_E_INVALID;
  }
  const ProjectParam sp = project_param(vertical_scans, horizon_scans, roi_range);
  const size_t n_pix = (size_t)L.n_lidars * vertical_scans * horizon_scans;
  ProjectWork w;
  int rc = project_work_reserve(c, work, n, n_pix, &w);
  if (rc) return rc;
  if (fe) {  // removeNaN + calTimestamp of every LiDAR first: the projection reads the timed cloud
    rc = front_times(c, d_in, L, fe->time_field, fe->scan_period, w, w.timed, nullptr);
    if (rc) return rc;
    d_in = w.timed;
  }
  ProfScope ps(c, "project");
  cudaStream_t st = c->stream;
  const int n_rows = L.n_lidars * vertical_scans;
  const int nbits = n_rows < 255 ? 8 : 16;  // (lidar, row) keys; all-ones = no pixel, sorts last
  const unsigned long long none = (1ull << nbits) - 1;
  MLOAM_CUDA_OK(c, cudaMemsetAsync(w.winner, 0x7f, sizeof(int) * n_pix, st));
  MLOAM_CUDA_OK(c, cudaMemsetAsync(w.sb.ticket, 0, 16, st));
  // a frame extracts the projected cloud with the raw size as its capacity: the tail past the projected count is zeros, never stale data
  if (fe) MLOAM_CUDA_OK(c, cudaMemsetAsync(d_out, 0, sizeof(float4) * (size_t)n, st));
  const int nb = (n + 255) / 256;
  k_project_pixels<<<nb, 256, 0, st>>>(d_in, n, sp, L, w.pix, w.winner);
  k_project_keys<<<nb, 256, 0, st>>>(w.pix, w.winner, n, horizon_scans, none, w.sb.k0, w.sb.v0);
  c->launches += 2;
  const int cur = radix_sort(c, w.sb, n, nullptr, nbits);
  const unsigned long long *ks = cur ? w.sb.k1 : w.sb.k0;
  const unsigned *vs = cur ? w.sb.v1 : w.sb.v0;
  k_project_emit<<<nb, 256, 0, st>>>(d_in, ks, vs, n, none, vertical_scans, d_out);
  k_project_rows<<<1, 256, 0, st>>>(ks, n, n_rows, d_scan_start, d_scan_end, d_n_out);
  c->launches += 2;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// in-CTA voxel filter (defined with the per-ring filter below)
constexpr int RV_THREADS = 512;
constexpr int RV_MAX_P2 = 16384;  // >= RING_MAX (defined below)
constexpr int RV_SMALL_MAX = 2048;  // whole-cloud filters up to this size run in one CTA (a bitonic sort of more keys on
                                    // one SM is slower than the multi-CTA radix passes)
__global__ void k_voxel_small(const float4 *__restrict__ P, int n, const int *__restrict__ d_n_valid, float inv, int intensity_last,
                              float4 *__restrict__ out, int *__restrict__ n_out);

int voxel_downsample_device(Ctx *c, const float4 *d_in, int n, const int *d_n_in, float leaf, int intensity_last, float4 *d_out,
                            int *d_n_out, DevBuf &work) {
  if (!(leaf > 0.f) || n < 0) {
    c->err = "voxel_downsample: bad leaf / size";
    return MLOAM_E_INVALID;
  }
  ProfScope ps(c, "voxel");
  if (n > 0 && n <= RV_SMALL_MAX) {
    bool &opt_in = c->smem_opt_in[0];  // function attributes are per device: remembered per context, not per process
    if (!opt_in) {
      MLOAM_CUDA_OK(c, cudaFuncSetAttribute(k_voxel_small, cudaFuncAttributeMaxDynamicSharedMemorySize, RV_MAX_P2 * (int)sizeof(unsigned long long)));
      opt_in = true;
    }
    k_voxel_small<<<1, RV_THREADS, RV_MAX_P2 * sizeof(unsigned long long), c->stream>>>(d_in, n, d_n_in, 1.0f / leaf, intensity_last, d_out, d_n_out);
    c->launches++;
    MLOAM_CUDA_OK(c, cudaGetLastError());
    return MLOAM_OK;
  }
  VoxelWork w;
  int rc = voxel_work_reserve(c, work, n, 1, &w);
  if (rc) return rc;
  rc = voxel_pipeline(c, d_in, nullptr, nullptr, n, d_n_in, 1, leaf, intensity_last, w, d_out, d_n_out);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// VoxelGridCovarianceMLOAM<PointIWithCov>::filter (lidar_mapper_keyframe.cpp:344-347): always the radix pipeline.
int voxel_downsample_cov_device(Ctx *c, const float4 *d_in, const float *d_cov6, const float *d_trace, int n, const int *d_n_in, float leaf,
                                float trace_threshold, float4 *d_out, float *d_cov6_out, float *d_trace_out, int *d_n_out, DevBuf &work) {
  if (!(leaf > 0.f) || n < 0) {
    c->err = "voxel_downsample_cov: bad leaf / size";
    return MLOAM_E_INVALID;
  }
  ProfScope ps(c, "voxel_cov");
  VoxelWork w;
  int rc = voxel_work_reserve(c, work, n, 1, &w);
  if (rc) return rc;
  CovIO io{d_cov6, d_trace, d_cov6_out, d_trace_out, trace_threshold, nullptr, 0.f};
  rc = voxel_pipeline(c, d_in, nullptr, nullptr, n, d_n_in, 1, leaf, 0, w, d_out, d_n_out, &io);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ extractCloud
constexpr int CURV_THREADS = 256;

// :133-142.  Also gap_ok[i] = |p[i+1]-p[i]|^2 <= 0.05 (the suppression test of :194-197 / :205-208, which
// compares a float against the double literal 0.05) and the ring id of every point inside a ring's
// [scan_start, scan_end) window (-1 elsewhere).
__global__ void __launch_bounds__(CURV_THREADS)
    k_curvature(const float4 *__restrict__ P, int n, float *__restrict__ curv, unsigned char *__restrict__ gap_ok,
                int *__restrict__ label) {
  __shared__ float sx[CURV_THREADS + 10], sy[CURV_THREADS + 10], sz[CURV_THREADS + 10];
  const int base = blockIdx.x * CURV_THREADS;
  for (int t = threadIdx.x; t < CURV_THREADS + 10; t += CURV_THREADS) {
    const int g = base + t - 5;
    float4 p = (g >= 0 && g < n) ? P[g] : make_float4(0, 0, 0, 0);
    sx[t] = p.x, sy[t] = p.y, sz[t] = p.z;
  }
  __syncthreads();
  const int i = base + threadIdx.x;
  if (i >= n) return;
  const int t = threadIdx.x + 5;
  float c = 0.f;
  if (i >= 5 && i < n - 5) {
    const float dx = sx[t - 5] + sx[t - 4] + sx[t - 3] + sx[t - 2] + sx[t - 1] - 10 * sx[t] + sx[t + 1] + sx[t + 2] + sx[t + 3] +
                     sx[t + 4] + sx[t + 5];
    const float dy = sy[t - 5] + sy[t - 4] + sy[t - 3] + sy[t - 2] + sy[t - 1] - 10 * sy[t] + sy[t + 1] + sy[t + 2] + sy[t + 3] +
                     sy[t + 4] + sy[t + 5];
    const float dz = sz[t - 5] + sz[t - 4] + sz[t - 3] + sz[t - 2] + sz[t - 1] - 10 * sz[t] + sz[t + 1] + sz[t + 2] + sz[t + 3] +
                     sz[t + 4] + sz[t + 5];
    c = dx * dx + dy * dy + dz * dz;
  }
  curv[i] = c;
  label[i] = 0;
  unsigned char g = 0;
  if (i + 1 < n) {
    const float ex = sx[t + 1] - sx[t], ey = sy[t + 1] - sy[t], ez = sz[t + 1] - sz[t];
    g = ((double)(ex * ex + ey * ey + ez * ez) > 0.05) ? 0 : 1;
  }
  gap_ok[i] = g;
}

constexpr int RING_THREADS = 512;
constexpr int RING_MAX = 12288;      // points per ring handled on chip (sort keys, picked / gap bytes)
constexpr int RING_SORT_MAX = 16384; // power of two >= RING_MAX: capacity of the in-CTA bitonic sort
constexpr int PICK_SHARP = 12, PICK_LESS = 120, PICK_FLAT = 24;  // per ring: 6 sectors x (2, 20, 4)

struct RingStage {  // per ring picks, indices into the cloud
  int n_sharp, n_less, n_flat, pad;
  int sharp[PICK_SHARP];
  int less[PICK_LESS];
  int flat[PICK_FLAT];
};

__global__ void __launch_bounds__(RING_THREADS)
    k_ring_pick(const float *__restrict__ curv, const unsigned char *__restrict__ gap_ok_g, int n, const int *__restrict__ scan_start,
                const int *__restrict__ scan_end, int *__restrict__ label, RingStage *__restrict__ stage, int *__restrict__ status, int smem_keys) {
  extern __shared__ unsigned long long keys[];  // smem_keys (<= RING_SORT_MAX), sized by the launcher from params.max_ring_points
  __shared__ unsigned char picked[RING_MAX + 16];
  __shared__ unsigned char gap[RING_MAX + 16];
  const int ring = blockIdx.x;
  RingStage &S = stage[ring];
  if (threadIdx.x == 0) S.n_sharp = S.n_less = S.n_flat = 0;  // rings that return early emit nothing
  const int s = scan_start[ring], e = scan_end[ring];
  if (e - s < 6) return;  // :155
  // on-chip window [lo, hi) = [s-5, e+5): every index the picks can touch (ind +- 5, ind in [s, e-1])
  const int lo = s - 5, hi = e + 5;
  if (hi - lo > RING_MAX || lo < 0 || hi > n) {
    if (threadIdx.x == 0) atomicExch(status, 1);  // ring too long for the on-chip window / ScanInfo out of range
    return;
  }
  for (int t = threadIdx.x; t < hi - lo; t += RING_THREADS) {
    picked[t] = 0;
    gap[t] = gap_ok_g[lo + t];
  }
  // :160-162 for all six sectors at once: ONE bitonic sort of (sector, curvature, offset in ring).  The sectors tile
  // [s, e-1] in index order, so sector j's sorted run is keys[sp_j - s, ep_j - s]; ties in curvature go by index (the
  // reference's std::sort leaves them unspecified).
  const int len_ring = e - s;  // points s .. e-1; the last sector ends at e-1
  int P2 = 1;
  while (P2 < len_ring) P2 <<= 1;
  if (P2 > smem_keys) {  // ring longer than the launch was sized for (params.max_ring_points)
    if (threadIdx.x == 0) atomicExch(status, 1);
    return;
  }
  for (int t = threadIdx.x; t < P2; t += RING_THREADS) {
    unsigned long long key = 0xffffffffffffffffull;
    if (t < len_ring) {
      int j = 0;
#pragma unroll
      for (int q = 1; q < 6; q++)
        if (s + t >= s + (e - s) * q / 6) j = q;
      key = ((unsigned long long)j << 46) | ((unsigned long long)__float_as_uint(curv[s + t]) << 14) | (unsigned)t;
    }
    keys[t] = key;
  }
  __syncthreads();
  for (int k2 = 2; k2 <= P2; k2 <<= 1) {
    for (int j2 = k2 >> 1; j2 > 0; j2 >>= 1) {
      for (int t = threadIdx.x; t < P2; t += RING_THREADS) {
        const int ixj = t ^ j2;
        if (ixj > t) {
          const unsigned long long a = keys[t], b = keys[ixj];
          const bool up = (t & k2) == 0;
          if ((a > b) == up) keys[t] = b, keys[ixj] = a;
        }
      }
      __syncthreads();
    }
  }
  int n_sharp = 0, n_less = 0, n_flat = 0;  // warp 0 keeps the running pick counts (uniform across its lanes)
  for (int j = 0; j < 6; j++) {
    const int sp = s + (e - s) * j / 6;            // :160
    const int ep = s + (e - s) * (j + 1) / 6 - 1;  // :161
    const int len = ep - sp + 1;
    const unsigned long long *skeys = keys + (sp - s);  // this sector's run, ascending curvature
    if (threadIdx.x < 32) {
      // The picks are inherently sequential (each one suppresses its +-5 neighbours), but finding the NEXT
      // unsuppressed candidate is not: warp 0 inspects 32 sorted candidates per step and ballots for the first
      // one that is still unpicked; lane 0 applies the pick.  Same visiting order as the reference's loops.
      const int lane = threadIdx.x;
      // :165-215 edge points, largest curvature first
      int largest = 0;
      int k = len - 1;
      while (k >= 0) {
        const int idx = k - lane;
        const bool inb = idx >= 0;
        const unsigned long long kk = inb ? skeys[idx] : 0ull;
        const float cv = __uint_as_float((unsigned)(kk >> 14));
        const int ind = s + (int)(unsigned)(kk & 0x3fffull);
        const bool pass = inb && ((double)cv > 0.1);  // sorted: once one fails, everything after it fails
        const unsigned m_fail = __ballot_sync(MLOAM_FULL_MASK, !pass);
        const unsigned before_fail = m_fail ? ((1u << (__ffs(m_fail) - 1)) - 1u) : 0xffffffffu;
        const unsigned m_unp = __ballot_sync(MLOAM_FULL_MASK, pass && picked[ind - lo] == 0) & before_fail;
        if (m_unp == 0) {
          if (m_fail) break;
          k -= 32;
          continue;
        }
        const int sel = __ffs(m_unp) - 1;
        const int pind = __shfl_sync(MLOAM_FULL_MASK, ind, sel);
        largest++;
        if (largest > 20) break;
        if (lane == 0) {
          const int o = pind - lo;
          if (largest <= 2) {
            label[pind] = 2;
            S.sharp[n_sharp] = pind;
            S.less[n_less] = pind;
          } else {
            label[pind] = 1;
            S.less[n_less] = pind;
          }
          picked[o] = 1;
          for (int l = 1; l <= 5; l++) {
            if (!gap[o + l - 1]) break;
            picked[o + l] = 1;
          }
          for (int l = -1; l >= -5; l--) {
            if (!gap[o + l]) break;
            picked[o + l] = 1;
          }
        }
        if (largest <= 2) n_sharp++;
        n_less++;
        __syncwarp();
        k = k - sel - 1;
      }
      // :218-256 flat points, smallest curvature first; the 4th pick breaks before any marking (:227-231)
      int smallest = 0;
      k = 0;
      while (k < len) {
        const int idx = k + lane;
        const bool inb = idx < len;
        const unsigned long long kk = inb ? skeys[idx] : 0ull;
        const float cv = __uint_as_float((unsigned)(kk >> 14));
        const int ind = s + (int)(unsigned)(kk & 0x3fffull);
        const bool pass = inb && ((double)cv < 0.1);
        const unsigned m_fail = __ballot_sync(MLOAM_FULL_MASK, !pass);
        const unsigned before_fail = m_fail ? ((1u << (__ffs(m_fail) - 1)) - 1u) : 0xffffffffu;
        const unsigned m_unp = __ballot_sync(MLOAM_FULL_MASK, pass && picked[ind - lo] == 0) & before_fail;
        if (m_unp == 0) {
          if (m_fail) break;
          k += 32;
          continue;
        }
        const int sel = __ffs(m_unp) - 1;
        const int pind = __shfl_sync(MLOAM_FULL_MASK, ind, sel);
        smallest++;
        if (lane == 0) {
          label[pind] = -1;
          S.flat[n_flat] = pind;
        }
        n_flat++;
        if (smallest >= 4) break;
        if (lane == 0) {
          const int o = pind - lo;
          picked[o] = 1;
          for (int l = 1; l <= 5; l++) {
            if (!gap[o + l - 1]) break;
            picked[o + l] = 1;
          }
          for (int l = -1; l >= -5; l--) {
            if (!gap[o + l]) break;
            picked[o + l] = 1;
          }
        }
        __syncwarp();
        k = k + sel + 1;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) S.n_sharp = n_sharp, S.n_less = n_less, S.n_flat = n_flat;
}

// Emit the staged picks in ring order (the order the reference's push_backs produce).
__global__ void k_emit_picks(const float4 *__restrict__ P, const RingStage *__restrict__ stage, int n_scans, float4 *__restrict__ sharp,
                             float4 *__restrict__ less, float4 *__restrict__ flat, int *__restrict__ counts) {
  // one CTA per ring: offsets = counts of the rings before it (<= 127 small reads), then a parallel gather
  __shared__ int off[3];
  const int r = blockIdx.x;
  if (threadIdx.x < 3) {
    int a = 0;
    for (int q = 0; q < r; q++) a += threadIdx.x == 0 ? stage[q].n_sharp : (threadIdx.x == 1 ? stage[q].n_less : stage[q].n_flat);
    off[threadIdx.x] = a;
    if (r == n_scans - 1)
      counts[threadIdx.x] = a + (threadIdx.x == 0 ? stage[r].n_sharp : (threadIdx.x == 1 ? stage[r].n_less : stage[r].n_flat));
  }
  __syncthreads();
  const RingStage &S = stage[r];
  for (int k = threadIdx.x; k < S.n_sharp; k += blockDim.x) sharp[off[0] + k] = P[S.sharp[k]];
  for (int k = threadIdx.x; k < S.n_less; k += blockDim.x) less[off[1] + k] = P[S.less[k]];
  for (int k = threadIdx.x; k < S.n_flat; k += blockDim.x) flat[off[2] + k] = P[S.flat[k]];
}

// ------------------------------------------------------------------------------------------ per-ring voxel grid
// :258-271 in ONE CTA per ring: gather the ring's less-flat points (label <= 0, ring order), pcl::VoxelGrid(0.2) on
// them — bounding box, voxel index, a bitonic sort of (voxel index << 14 | offset in ring) in shared memory (the
// offset in the low bits makes the order inside a voxel the input order, i.e. what a stable sort gives), run heads,
// ordered float centroid sums — and stage the centroids at the ring's own window of `stage_out`.  Replaces the
// flag / scan / gather kernels and a 5-pass segmented radix sort (about 40 launches) for the per-ring filter.

__device__ __forceinline__ int block_excl_scan_512(int v, int *warp_tot /* smem[17] */, int *total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(MLOAM_FULL_MASK, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  if (w == 0) {
    const int x = lane < RV_THREADS / 32 ? warp_tot[lane] : 0;
    int s = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(MLOAM_FULL_MASK, s, o);
      if (lane >= o) s += t;
    }
    if (lane < RV_THREADS / 32) warp_tot[lane] = s - x;
    if (lane == 31) warp_tot[16] = s;
  }
  __syncthreads();
  const int r = warp_tot[w] + inc - v;
  *total = warp_tot[16];
  __syncthreads();  // warp_tot may be reused right away
  return r;
}

// Voxel-grid filter of the points P[s, s + len) whose label is <= 0 (all of them when label == nullptr), by one CTA of
// RV_THREADS threads; len <= RV_MAX_P2.  Centroids go to out[0..), their number to *out_cnt.
__device__ void voxel_in_cta(const float4 *__restrict__ P, const int *__restrict__ label, int s, int len, float inv, int intensity_last,
                             float4 *__restrict__ out, int *__restrict__ out_cnt) {
  extern __shared__ unsigned long long rv_keys[];  // RV_MAX_P2
  __shared__ int warp_tot[17];
  __shared__ unsigned bb[6];  // ordered-uint min xyz, max xyz
  if (threadIdx.x < 3) bb[threadIdx.x] = 0xffffffffu, bb[3 + threadIdx.x] = 0u;
  __syncthreads();
  // pass 1: bounding box of the finite less-flat points (getMinMax3D) + their number
  int nq = 0;
  {
    unsigned mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u};
    int cnt = 0;
    for (int t = threadIdx.x; t < len; t += RV_THREADS) {
      if (label && label[s + t] > 0) continue;
      cnt++;
      const float4 p = P[s + t];
      if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        mn[0] = min(mn[0], f2ord(p.x)), mn[1] = min(mn[1], f2ord(p.y)), mn[2] = min(mn[2], f2ord(p.z));
        mx[0] = max(mx[0], f2ord(p.x)), mx[1] = max(mx[1], f2ord(p.y)), mx[2] = max(mx[2], f2ord(p.z));
      }
    }
#pragma unroll
    for (int d = 0; d < 3; d++) {
      mn[d] = __reduce_min_sync(MLOAM_FULL_MASK, mn[d]);
      mx[d] = __reduce_max_sync(MLOAM_FULL_MASK, mx[d]);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
      for (int d = 0; d < 3; d++) atomicMin(&bb[d], mn[d]), atomicMax(&bb[3 + d], mx[d]);
    }
    int dummy = block_excl_scan_512(cnt, warp_tot, &nq);
    (void)dummy;
  }
  if (nq == 0) {
    if (threadIdx.x == 0) *out_cnt = 0;
    return;
  }
  const float mn0 = ord2f(bb[0]), mn1 = ord2f(bb[1]), mn2 = ord2f(bb[2]);
  const float mx0 = ord2f(bb[3]), mx1 = ord2f(bb[4]), mx2 = ord2f(bb[5]);
  const long long ddx = (long long)((mx0 - mn0) * inv) + 1, ddy = (long long)((mx1 - mn1) * inv) + 1, ddz = (long long)((mx2 - mn2) * inv) + 1;
  const bool pass_through = ddx * ddy * ddz > 2147483647ll;  // :92-101
  const int minb0 = (int)floorf(mn0 * inv), minb1 = (int)floorf(mn1 * inv), minb2 = (int)floorf(mn2 * inv);
  const int div0 = (int)floorf(mx0 * inv) - minb0 + 1, div1 = (int)floorf(mx1 * inv) - minb1 + 1;
  int P2 = 1;
  while (P2 < nq) P2 <<= 1;
  // pass 2: keys, written densely in ring order (tile by tile so that the compaction keeps that order)
  int carry = 0;
  for (int base = 0; base < len; base += RV_THREADS) {
    const int t = base + threadIdx.x;
    const bool f = t < len && (!label || label[s + t] <= 0);
    int tile_total;
    const int q = carry + block_excl_scan_512(f ? 1 : 0, warp_tot, &tile_total);
    if (f) {
      const float4 p = P[s + t];
      unsigned long long key = 0xffffffffffffffffull;  // non-finite points are dropped
      if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        unsigned idx;
        if (pass_through) {
          idx = (unsigned)q;
        } else {
          const int i0 = (int)(floorf(p.x * inv) - (float)minb0);
          const int i1 = (int)(floorf(p.y * inv) - (float)minb1);
          const int i2 = (int)(floorf(p.z * inv) - (float)minb2);
          idx = (unsigned)(i0 + i1 * div0 + i2 * (div0 * div1));
        }
        key = ((unsigned long long)idx << 14) | (unsigned)t;
      }
      rv_keys[q] = key;
    }
    carry += tile_total;
  }
  for (int t = nq + threadIdx.x; t < P2; t += RV_THREADS) rv_keys[t] = 0xffffffffffffffffull;
  __syncthreads();
  // bitonic sort, ascending
  for (int k2 = 2; k2 <= P2; k2 <<= 1) {
    for (int j2 = k2 >> 1; j2 > 0; j2 >>= 1) {
      for (int t = threadIdx.x; t < P2; t += RV_THREADS) {
        const int ixj = t ^ j2;
        if (ixj > t) {
          const unsigned long long a = rv_keys[t], b = rv_keys[ixj];
          const bool up = (t & k2) == 0;
          if ((a > b) == up) rv_keys[t] = b, rv_keys[ixj] = a;
        }
      }
      __syncthreads();
    }
  }
  // run heads -> output slots -> ordered centroid sums (:239-250 and the centroid loop)
  carry = 0;
  for (int base = 0; base < nq; base += RV_THREADS) {
    const int k = base + threadIdx.x;
    bool head = false;
    unsigned long long key = 0xffffffffffffffffull;
    if (k < nq) {
      key = rv_keys[k];
      head = key != 0xffffffffffffffffull && (k == 0 || (rv_keys[k - 1] >> 14) != (key >> 14));
    }
    int tile_total;
    const int slot = carry + block_excl_scan_512(head ? 1 : 0, warp_tot, &tile_total);
    if (head) {
      float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f, last = 0.f;
      int j = k;
      for (; j < nq && (rv_keys[j] >> 14) == (key >> 14); j++) {
        const float4 p = P[s + (int)(rv_keys[j] & 0x3fffull)];
        sx = sx + p.x, sy = sy + p.y, sz = sz + p.z, si = si + p.w;
        last = p.w;
      }
      const float cnt = (float)(j - k);
      out[slot] = make_float4(sx / cnt, sy / cnt, sz / cnt, intensity_last ? last : si / cnt);
    }
    carry += tile_total;
  }
  if (threadIdx.x == 0) *out_cnt = carry;
}

__global__ void __launch_bounds__(RV_THREADS)
    k_ring_voxel(const float4 *__restrict__ P, const int *__restrict__ label, int n, const int *__restrict__ scan_start,
                 const int *__restrict__ scan_end, float inv, float4 *__restrict__ stage_out, int *__restrict__ ring_cnt, int smem_keys,
                 float4 *__restrict__ first = nullptr, int *__restrict__ first_ok = nullptr, int first_rings = 0) {
  const int ring = blockIdx.x;
  const int s = scan_start[ring], e = scan_end[ring];
  // the first ring of LiDAR l records laser_cloud_out.points[0] of its part (image_segmenter.hpp:390): the part starts at
  // scan_start - 5 of its first ring, and holds sum (end - start + 11) points over its rings (0: empty, no point)
  if (first && threadIdx.x == 0 && ring % first_rings == 0) {
    int cnt = 0;
    for (int r = ring; r < ring + first_rings; r++) cnt += scan_end[r] - scan_start[r] + 11;
    const int at = s - 5, l = ring / first_rings;
    const int ok = (cnt > 0 && at >= 0 && at < n) ? 1 : 0;
    first_ok[l] = ok;
    if (ok) first[l] = P[at];
  }
  const int len = e - s;
  // the rings k_ring_pick processes (:155, the on-chip window check and the sort capacity of this launch)
  if (len < 6 || len + 10 > RING_MAX || s - 5 < 0 || e + 5 > n || len > smem_keys) {
    if (threadIdx.x == 0) ring_cnt[ring] = 0;
    return;
  }
  voxel_in_cta(P, label, s, len, inv, 0, stage_out + s, ring_cnt + ring);
}

// Whole-cloud filter of a SMALL cloud (n <= RV_MAX_P2, e.g. the <= 120 x rings less-sharp corner candidates of a sweep):
// the same in-CTA pipeline, one launch instead of ~28.
__global__ void __launch_bounds__(RV_THREADS)
    k_voxel_small(const float4 *__restrict__ P, int n, const int *__restrict__ d_n_valid, float inv, int intensity_last,
                  float4 *__restrict__ out, int *__restrict__ n_out) {
  if (d_n_valid) n = min(n, *d_n_valid);
  if (n <= 0) {
    if (threadIdx.x == 0) *n_out = 0;
    return;
  }
  voxel_in_cta(P, nullptr, 0, n, inv, intensity_last, out, n_out);
}

// Concatenate the rings' staged centroids in ring order (the order of :271's `+=`).
__global__ void k_ring_voxel_emit(const float4 *__restrict__ stage_out, const int *__restrict__ ring_cnt, const int *__restrict__ scan_start,
                                  int n_scans, float4 *__restrict__ out, int *__restrict__ n_out) {
  __shared__ int off;
  const int r = blockIdx.x;
  if (threadIdx.x == 0) {
    int a = 0;
    for (int q = 0; q < r; q++) a += ring_cnt[q];
    off = a;
    if (r == n_scans - 1) *n_out = a + ring_cnt[r];
  }
  __syncthreads();
  const int cnt = ring_cnt[r], s = scan_start[r];
  for (int k = threadIdx.x; k < cnt; k += blockDim.x) out[off + k] = stage_out[s + k];
}

__global__ void k_transform_points(float4 *pts, int n, const int *__restrict__ d_n, const double *__restrict__ pose7) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (d_n) n = min(n, *d_n);
  if (i >= n) return;
  float4 p = pts[i];
  const float3 q = associate(pose_from_param(pose7), p.x, p.y, p.z);
  pts[i] = make_float4(q.x, q.y, q.z, p.w);
}
int transform_points_device(Ctx *c, float4 *d_pts, int n, const int *d_n, const double *d_pose7) {
  if (n <= 0) return MLOAM_OK;
  k_transform_points<<<(n + 255) / 256, 256, 0, c->stream>>>(d_pts, n, d_n, d_pose7);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// ------------------------------------------------------------------------------------------ multi-LiDAR merge
// One batched extraction over the concatenated sweeps of L LiDARs (rings l * R .. (l + 1) * R - 1 belong to LiDAR l)
// produces the feature clouds in ring order, i.e. LiDAR by LiDAR.  The odometry node hands them to the mapper in the
// base frame, laser id in the intensity (transformCloudFeature, visualization.cpp:40-52; pubPointCloud :93-104):
// pcl::transformPointCloud with the float matrix of Pose(qbl, tbl), then `+=` per LiDAR.
__global__ void k_lidar_offsets(const RingStage *__restrict__ stage, const int *__restrict__ ring_cnt, int rings_per_lidar, int n_lidars,
                                int *__restrict__ off /* [2][n_lidars + 1]: less-sharp, less-flat */) {
  const int l = threadIdx.x;
  if (l > n_lidars) return;
  int a = 0, b = 0;
  for (int q = 0; q < l * rings_per_lidar; q++) a += stage[q].n_less, b += ring_cnt[q];
  off[l] = a, off[n_lidars + 1 + l] = b;
}

__global__ void k_merge_transform(float4 *__restrict__ pts, const int *__restrict__ off, int n_lidars, const float *__restrict__ ext12, int set_id = 1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= off[n_lidars]) return;
  int l = 0;
  while (l + 1 < n_lidars && i >= off[l + 1]) l++;
  const float4 p = pts[i];
  pts[i] = rig_transform(ext12 + 12 * l, p, set_id ? (float)l : p.w);  // p.intensity = n (rig merge) / kept (local map, estimator.cpp:1185-1186)
}

int lidar_offsets_device(Ctx *c, int n_lidars, int rings_per_lidar, int *d_off) {
  if (n_lidars < 1 || n_lidars > MLOAM_MAX_LIDARS || !c->d_ring_stage) {
    c->err = "merge_lidars: 1..16 LiDARs, after an extraction";
    return MLOAM_E_INVALID;
  }
  k_lidar_offsets<<<1, 32, 0, c->stream>>>(static_cast<const RingStage *>(c->d_ring_stage), c->d_ring_cnt, rings_per_lidar, n_lidars, d_off);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

int merge_lidars_device(Ctx *c, ExtractOut out, int n_cap_less, int n_cap_lflat, int n_lidars, const float *d_ext12, const int *d_off) {
  if (n_lidars < 1 || n_lidars > MLOAM_MAX_LIDARS) {
    c->err = "merge_lidars: 1..16 LiDARs";
    return MLOAM_E_INVALID;
  }
  cudaStream_t st = c->stream;
  if (n_cap_less > 0) k_merge_transform<<<(n_cap_less + 255) / 256, 256, 0, st>>>(out.less_sharp, d_off, n_lidars, d_ext12);
  if (n_cap_lflat > 0) k_merge_transform<<<(n_cap_lflat + 255) / 256, 256, 0, st>>>(out.less_flat, d_off + n_lidars + 1, n_lidars, d_ext12);
  c->launches += 2;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// In place: segment l of `pts` (points [off[l], off[l+1])) <- float 3x4 matrix l times the point, intensity kept
// (pcl::transformPointCloud with pose_local_[n][i].T_.cast<float>(), estimator.cpp:1185-1190).
int transform_segments_device(Ctx *c, float4 *d_pts, int n, const int *d_off, int n_seg, const float *d_mat12) {
  if (n <= 0) return MLOAM_OK;
  k_merge_transform<<<(n + 255) / 256, 256, 0, c->stream>>>(d_pts, d_off, n_seg, d_mat12, 0);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

void extract_work_layout(Carve &cv, int n, int n_scans, ExtractWork *W) {
  const size_t N1 = (size_t)n + 16;
  W->curv = cv.take<float>(N1), W->label = cv.take<int>(N1), W->gap = cv.take<unsigned char>(N1);
  W->stage = cv.take<RingStage>(n_scans), W->ring_cnt = cv.take<int>((size_t)n_scans + 2), W->status = cv.take<int>(4);
  W->less_flat = cv.take<float4>(N1);
}

int extract_device(Ctx *c, const float4 *d_cloud, int n, const int *d_scan_start, const int *d_scan_end, int n_scans,
                   ExtractOut out, float *d_curv_or_null, int *d_label_or_null) {
  if (n < 0 || n_scans <= 0 || n_scans > MLOAM_MAX_RINGS || (out.first && (out.first_rings <= 0 || n_scans % out.first_rings != 0 ||
                                                                              n_scans / out.first_rings > MLOAM_MAX_LIDARS))) {
    c->err = "extract: n_scans must be in 1..1024 (rings of all LiDARs of a batched extraction)";
    return MLOAM_E_INVALID;
  }
  // in-CTA sort capacity per ring: params.max_ring_points (0: the on-chip maximum).  A tight bound lets several ring CTAs
  // share an SM (the sort keys are the kernels' shared-memory footprint), which is what a multi-LiDAR batch needs.
  int smem_keys = RING_SORT_MAX;
  if (c->params.max_ring_points > 0) {
    smem_keys = 64;
    while (smem_keys < c->params.max_ring_points && smem_keys < RING_SORT_MAX) smem_keys <<= 1;
  }
  ProfScope ps(c, "extract");
  cudaStream_t st = c->stream;
  ExtractWork W;
  MLOAM_CUDA_OK(c, carve(c->extract_work, [&](Carve &cv) { extract_work_layout(cv, n, n_scans, &W); }));
  float *curv = W.curv;
  int *label = W.label;
  unsigned char *gap = W.gap;
  RingStage *stage = W.stage;
  int *seg_begin = W.ring_cnt;
  int *status = W.status;
  c->d_extract_status = status;
  c->d_ring_stage = stage, c->d_ring_cnt = seg_begin;  // per-ring pick / centroid counts (multi-LiDAR merge)
  float4 *lf = W.less_flat;
  MLOAM_CUDA_OK(c, cudaMemsetAsync(out.counts, 0, 4 * sizeof(int), st));
  MLOAM_CUDA_OK(c, cudaMemsetAsync(status, 0, sizeof(int), st));
  if (n == 0) return MLOAM_OK;
  const int nb = (n + 255) / 256;
  k_curvature<<<(n + CURV_THREADS - 1) / CURV_THREADS, CURV_THREADS, 0, st>>>(d_cloud, n, curv, gap, label);
  bool &pick_opt_in = c->smem_opt_in[1];
  if (!pick_opt_in) {
    MLOAM_CUDA_OK(c, cudaFuncSetAttribute(k_ring_pick, cudaFuncAttributeMaxDynamicSharedMemorySize, RING_SORT_MAX * (int)sizeof(unsigned long long)));
    pick_opt_in = true;
  }
  k_ring_pick<<<n_scans, RING_THREADS, (size_t)smem_keys * sizeof(unsigned long long), st>>>(curv, gap, n, d_scan_start, d_scan_end, label, stage, status, smem_keys);
  k_emit_picks<<<n_scans, 128, 0, st>>>(d_cloud, stage, n_scans, out.sharp, out.less_sharp, out.flat, out.counts);
  // :258-271 less-flat candidates + per-ring pcl::VoxelGrid(0.2): one CTA per ring, then the ring-order concatenation
  bool &smem_opt_in = c->smem_opt_in[2];
  if (!smem_opt_in) {
    MLOAM_CUDA_OK(c, cudaFuncSetAttribute(k_ring_voxel, cudaFuncAttributeMaxDynamicSharedMemorySize, RV_MAX_P2 * (int)sizeof(unsigned long long)));
    smem_opt_in = true;
  }
  k_ring_voxel<<<n_scans, RV_THREADS, (size_t)smem_keys * sizeof(unsigned long long), st>>>(d_cloud, label, n, d_scan_start, d_scan_end, 1.0f / 0.2f,
                                                                                              lf, seg_begin, smem_keys, out.first, out.first_ok,
                                                                                              out.first_rings);
  k_ring_voxel_emit<<<n_scans, 128, 0, st>>>(lf, seg_begin, d_scan_start, n_scans, out.less_flat, out.counts + 3);
  c->launches += 5;
  if (d_curv_or_null) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_curv_or_null, curv, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  if (d_label_or_null) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_label_or_null, label, sizeof(int) * n, cudaMemcpyDeviceToDevice, st));
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

}  // namespace mloam
