// pcd_write.cu — the mapper's clouds, and clouds a caller holds, as the ASCII PCD files pcl::PCDWriter::write gives them (the format:
// include/mloam_b200.h, mloam_cloud_pcd; the characters of one value: csrc/pcd_format.cuh).  Up to 16 files in ONE launch, k_pcd_write:
//
// Each CTA takes a tile of 128 points of one file, in the order of a ticket it draws from a counter (so every tile it waits on is already
// running).  Each thread formats its point's line into a slot of shared memory; a block scan of the line lengths gives the lines' places
// in the tile; a decoupled look-back over the file's earlier tiles gives the tile's place in the file (tile 0 starts after the header,
// which it composes once the file's point count is known, a count that may live on the device).  The lines are compacted in shared
// memory and the tile's bytes stored contiguously.  Tile words carry the call's epoch and tickets count on from the last call, so
// nothing is reset between calls.  The CTA of a file's last tile stores the file's size.
#include <algorithm>
#include <climits>

#include "ctx.h"
#include "host_util.h"
#include "pcd_format.cuh"

namespace mloam {

namespace {

constexpr int PW_THREADS = 128;
constexpr int PW_MAX_FILES = 16;
constexpr int PW_MAX_SEGS = 2 * PW_MAX_FILES;
constexpr int PW_FIELD = pcd::PCD_FMT_MAX + 1;  // a value and its separator
constexpr int PW_LINE = 11 * PW_FIELD;          // the longest line
constexpr int PW_HEADER = 384;                  // the longest header (eleven fields, 10-digit counts) fits
constexpr unsigned PW_AGGREGATE = 1u, PW_INCLUSIVE = 2u;

struct PcdFile {
  unsigned char *out;
  int nf;            // fields per point: 3, 4 or 11
  int seg0, n_segs;  // its segments in PcdWriteBatch::seg, concatenated in order
  int tile0;         // its first tile (files' tiles are consecutive, at least one each)
};

struct PcdWriteBatch {
  PackSeg seg[PW_MAX_SEGS];
  PcdFile file[PW_MAX_FILES];
  int tile_end;                       // tiles of every file
  int n_files;
  unsigned epoch;                     // tags the tile words of this launch (never 0)
  unsigned long long ticket0;         // the counter's value before the launch
  unsigned long long *ticket;
  unsigned long long *tile_word;      // per tile: (epoch << 2 | flag) << 32 | bytes
  int *bytes;                         // out: each file's size
};

__device__ __forceinline__ int seg_count(const PackSeg &g) { return g.d_n ? max(0, min(g.n, *g.d_n)) : g.n; }

__device__ int put_str(char *o, int n, const char *s) {
  while (*s) o[n++] = *s++;
  return n;
}
__device__ int put_int(char *o, int n, int v) {
  char t[10];
  int k = 0;
  do t[k++] = (char)('0' + v % 10), v /= 10;
  while (v);
  while (k) o[n++] = t[--k];
  return n;
}

// generateHeader<PointT> of n points with nf fields into o; returns its length
__device__ int pcd_header(int nf, int n_pts, char *o) {
  const char *const names[11] = {"x", "y", "z", "intensity", "cov_xx", "cov_xy", "cov_xz", "cov_yy", "cov_yz", "cov_zz", "cov_trace"};
  int n = put_str(o, 0, "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS");
  for (int f = 0; f < nf; f++) o[n++] = ' ', n = put_str(o, n, names[f]);
  const char *const rows[3] = {"\nSIZE", "\nTYPE", "\nCOUNT"}, vals[3] = {'4', 'F', '1'};
  for (int r = 0; r < 3; r++) {
    n = put_str(o, n, rows[r]);
    for (int f = 0; f < nf; f++) o[n++] = ' ', o[n++] = vals[r];
  }
  n = put_int(o, put_str(o, n, "\nWIDTH "), n_pts);
  n = put_int(o, put_str(o, n, "\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS "), n_pts);
  return put_str(o, n, "\nDATA ascii\n");
}

__global__ void __launch_bounds__(PW_THREADS) k_pcd_write(const __grid_constant__ PcdWriteBatch B) {
  __shared__ char s_line[PW_THREADS * PW_LINE];  // thread k's line at slot k
  __shared__ char s_out[PW_THREADS * PW_LINE];   // the tile's lines back to back
  __shared__ char s_hdr[PW_HEADER];
  __shared__ int s_warp[PW_THREADS / 32];
  __shared__ int s_tile, s_prefix;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = (int)(atomicAdd(B.ticket, 1ull) - B.ticket0);
  __syncthreads();
  const int t = s_tile;
  int f = 0;
  while (f + 1 < B.n_files && t >= B.file[f + 1].tile0) f++;
  const PcdFile &F = B.file[f];
  const int j = t - F.tile0;
  const bool last = f + 1 < B.n_files ? t + 1 == B.file[f + 1].tile0 : t + 1 == B.tile_end;
  int n_pts = 0;
  for (int s = F.seg0; s < F.seg0 + F.n_segs; s++) n_pts += seg_count(B.seg[s]);

  // this thread's line
  const int i = j * PW_THREADS + tid;
  int len = 0;
  char *line = s_line + tid * PW_LINE;
  if (i < n_pts) {
    int s = F.seg0, k = i;
    for (int m; k >= (m = seg_count(B.seg[s])); s++) k -= m;
    const PackSeg &g = B.seg[s];
    const float4 p = __ldg(g.pts + k);
    uint32_t v[11] = {__float_as_uint(p.x), __float_as_uint(p.y), __float_as_uint(p.z), __float_as_uint(p.w)};
    if (F.nf == 11) {
#pragma unroll
      for (int q = 0; q < 6; q++) v[4 + q] = __float_as_uint(__ldg(g.cov6 + 6 * (size_t)k + q));
      v[10] = __float_as_uint(__ldg(g.trace + k));
    }
    for (int q = 0; q < F.nf; q++) {
      len += pcd::format_float(v[q], line + len);
      line[len++] = q + 1 < F.nf ? ' ' : '\n';
    }
  }

  // block scan of the line lengths
  int incl = len;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int before = 0, agg = 0;
#pragma unroll
  for (int w = 0; w < PW_THREADS / 32; w++) before += w < warp ? s_warp[w] : 0, agg += s_warp[w];
  const int excl = before + incl - len;

  // the tile's place in the file
  if (tid == 0) {
    const unsigned long long tag = (unsigned long long)B.epoch << 2;
    unsigned prefix = 0;
    if (j == 0) {
      prefix = n_pts > 0 ? (unsigned)pcd_header(F.nf, n_pts, s_hdr) : 0u;
    } else {
      atomicExch(B.tile_word + t, ((tag | PW_AGGREGATE) << 32) | (unsigned)agg);
      for (int p = t - 1;;) {
        const unsigned long long w = atomicAdd(B.tile_word + p, 0ull);
        const unsigned long long wt = w >> 32;
        if (wt == (tag | PW_INCLUSIVE)) {
          prefix += (unsigned)w;
          break;
        }
        if (wt == (tag | PW_AGGREGATE)) prefix += (unsigned)w, p--;
      }
    }
    atomicExch(B.tile_word + t, ((tag | PW_INCLUSIVE) << 32) | (prefix + (unsigned)agg));
    s_prefix = (int)prefix;
    if (last) B.bytes[f] = n_pts > 0 ? (int)(prefix + (unsigned)agg) : 0;
  }
  for (int k = 0; k < len; k++) s_out[excl + k] = line[k];
  __syncthreads();
  unsigned char *out = F.out;
  if (j == 0 && n_pts > 0)
    for (int k = tid; k < s_prefix; k += PW_THREADS) out[k] = (unsigned char)s_hdr[k];
  out += s_prefix;
  for (int k = tid; k < agg; k += PW_THREADS) out[k] = (unsigned char)s_out[k];
}

// One file to write: its segments, fields per point and point capacity
struct PcdJob {
  PackSeg seg[2];
  int n_segs = 0, nf = 0;
  long long cap = 0;
};

// The launch for n jobs; sizes and device addresses of the files on return (the stream synchronised)
int pcd_write(Ctx *c, int n, const PcdJob *jobs, size_t *bytes, unsigned char **d_file) {
  PcdWriteBatch B;
  memset(&B, 0, sizeof(B));
  B.n_files = n;
  size_t off[PW_MAX_FILES + 1] = {0};
  int tiles = 0;
  for (int k = 0; k < n; k++) {
    const PcdJob &J = jobs[k];
    const long long bound = PW_HEADER + J.cap * PW_FIELD * J.nf;
    if (bound > INT_MAX) return fail(c, MLOAM_E_INVALID, "pcd: a file could exceed 2^31 - 1 bytes");
    PcdFile &F = B.file[k];
    F.nf = J.nf, F.seg0 = k == 0 ? 0 : B.file[k - 1].seg0 + B.file[k - 1].n_segs, F.n_segs = J.n_segs, F.tile0 = tiles;
    for (int s = 0; s < J.n_segs; s++) B.seg[F.seg0 + s] = J.seg[s];
    tiles += (int)std::max(1ll, (J.cap + PW_THREADS - 1) / PW_THREADS);
    off[k + 1] = off[k] + align256((size_t)bound);
  }
  B.tile_end = tiles;
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, c->pcd_files.reserve(off[n] + 256));
  unsigned char *base = c->pcd_files.as<unsigned char>();
  for (int k = 0; k < n; k++) B.file[k].out = d_file[k] = base + off[k];
  B.bytes = reinterpret_cast<int *>(base + off[n]);
  // the counter and the tile words start zeroed in a new allocation; a zero tag is no call's
  const size_t tile_bytes = sizeof(unsigned long long) * ((size_t)tiles + 1);
  if (tile_bytes > c->pcd_tiles.cap) {
    MLOAM_CUDA_OK(c, c->pcd_tiles.reserve(tile_bytes));
    MLOAM_CUDA_OK(c, cudaMemsetAsync(c->pcd_tiles.p, 0, c->pcd_tiles.cap, st));
    c->pcd_tickets = 0;
  }
  c->pcd_epoch = (c->pcd_epoch + 1) & 0x3fffffffu;
  if (c->pcd_epoch == 0) c->pcd_epoch = 1;
  B.epoch = c->pcd_epoch;
  B.ticket = c->pcd_tiles.as<unsigned long long>();
  B.tile_word = B.ticket + 1;
  B.ticket0 = c->pcd_tickets;
  {
    ProfScope ps(c, "pcd_write");
    k_pcd_write<<<tiles, PW_THREADS, 0, st>>>(B);
    c->launches++;
    MLOAM_CUDA_OK(c, cudaGetLastError());
  }
  c->pcd_tickets += (unsigned long long)tiles;
  int *hb = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hb, B.bytes, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  for (int k = 0; k < n; k++) bytes[k] = (size_t)hb[k];
  return MLOAM_OK;
}

// Copies the files to the caller's host buffers when every one fits (h_data[k] NULL: a size query)
int pcd_copy_out(Ctx *c, int n, unsigned char *const *d_file, const size_t *bytes, void *const *h_data, const size_t *cap_bytes) {
  for (int k = 0; k < n; k++)
    if (h_data[k] && bytes[k] > cap_bytes[k]) return fail(c, MLOAM_E_INVALID, "pcd: a capacity is too small (bytes holds the files' sizes)");
  bool copied = false;
  for (int k = 0; k < n; k++) {
    if (!h_data[k] || bytes[k] == 0) continue;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_data[k], d_file[k], bytes[k], cudaMemcpyDeviceToHost, c->stream));
    copied = true;
  }
  if (copied) MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}

// The checks and the launch of mloam_cloud_pcd*
int cloud_pcd(Ctx *c, int n, const int *sources, size_t *bytes, unsigned char **d_file) {
  if (!sources || !bytes || n < 1 || n > MLOAM_PCD_KEYFRAMES + 1) return fail(c, MLOAM_E_INVALID, "cloud_pcd: 1..7 sources, non-NULL arrays");
  for (int k = 0; k < n; k++) bytes[k] = 0;
  bool seen[MLOAM_PCD_KEYFRAMES + 1] = {false, false, false, false, false, false, false};
  for (int k = 0; k < n; k++) {
    const int s = sources[k];
    if (s < MLOAM_MSG_FULL_RES || s > MLOAM_PCD_KEYFRAMES || seen[s])
      return fail(c, MLOAM_E_INVALID, "cloud_pcd: a source is not one of MLOAM_MSG_* / MLOAM_PCD_KEYFRAMES or is given twice");
    seen[s] = true;
  }
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "cloud_pcd: single-GPU only; detach the communicator");
  for (int k = 0; k < n; k++) {
    if (sources[k] <= MLOAM_MSG_CORNER_LAST && !c->reg_valid)
      return fail(c, MLOAM_E_STATE, "cloud_pcd: the last call was no mloam_frame* call run with the registered clouds on (mloam_set_registered)");
    if (sources[k] > MLOAM_MSG_CORNER_LAST && !c->kf) return fail(c, MLOAM_E_STATE, "cloud_pcd: call mloam_keyframes_init first");
  }
  cudaSetDevice(c->device);
  PcdJob jobs[MLOAM_PCD_KEYFRAMES + 1];
  for (int k = 0; k < n; k++) {
    const int s = sources[k];
    PcdJob &J = jobs[k];
    J.nf = s <= MLOAM_MSG_CORNER_LAST || s == MLOAM_PCD_KEYFRAMES ? 4 : 11;
    if (s <= MLOAM_MSG_CORNER_LAST) {
      const int w = s - MLOAM_MSG_FULL_RES;  // MLOAM_REGISTERED_* of the same order
      J.seg[0] = PackSeg{c->reg_last.cloud[w], nullptr, nullptr, c->reg_last.counts + w, c->reg_last.cap[w], 0}, J.n_segs = 1;
    } else if (s == MLOAM_PCD_KEYFRAMES) {
      std::vector<float4> pos;
      keyframe_positions(c, pos);
      if (!pos.empty()) {
        MLOAM_CUDA_OK(c, c->pcd_src.reserve(sizeof(float4) * pos.size()));
        MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->pcd_src.p, pos.data(), sizeof(float4) * pos.size(), cudaMemcpyHostToDevice, c->stream));
      }
      J.seg[0] = PackSeg{c->pcd_src.as<float4>(), nullptr, nullptr, nullptr, (int)pos.size(), 0}, J.n_segs = 1;
    } else {
      J.n_segs = keyframe_msg_segments(c, s, J.seg);
    }
    for (int g = 0; g < J.n_segs; g++) J.cap += J.seg[g].n;
  }
  return pcd_write(c, n, jobs, bytes, d_file);
}

}  // namespace

}  // namespace mloam

using namespace mloam;

extern "C" {

int mloam_cloud_pcd(mloam_ctx_t *h, int n, const int *sources, void *const *h_data, const size_t *cap_bytes, size_t *bytes) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!h_data || !cap_bytes) return fail(c, MLOAM_E_INVALID, "cloud_pcd: h_data and cap_bytes must not be NULL");
  unsigned char *d_file[PW_MAX_FILES];
  const int rc = cloud_pcd(c, n, sources, bytes, d_file);
  return rc ? rc : pcd_copy_out(c, n, d_file, bytes, h_data, cap_bytes);
}

int mloam_cloud_pcd_device(mloam_ctx_t *h, int n, const int *sources, const void **d_data, size_t *bytes) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!d_data) return fail(c, MLOAM_E_INVALID, "cloud_pcd_device: d_data must not be NULL");
  unsigned char *d_file[PW_MAX_FILES];
  const int rc = cloud_pcd(c, n, sources, bytes, d_file);
  if (rc) return rc;
  for (int k = 0; k < n; k++) d_data[k] = d_file[k];
  return MLOAM_OK;
}

int mloam_pcd_encode(mloam_ctx_t *h, int n, const mloam_pcd_cloud_t *clouds, void *const *h_data, const size_t *cap_bytes, size_t *bytes) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!clouds || !h_data || !cap_bytes || !bytes || n < 1 || n > PW_MAX_FILES)
    return fail(c, MLOAM_E_INVALID, "pcd_encode: 1..16 clouds, non-NULL arrays");
  for (int k = 0; k < n; k++) bytes[k] = 0;
  size_t off[PW_MAX_FILES + 1] = {0};
  for (int k = 0; k < n; k++) {
    const mloam_pcd_cloud_t &q = clouds[k];
    if (q.layout != MLOAM_PCD_XYZ && q.layout != MLOAM_PCD_XYZI && q.layout != MLOAM_PCD_XYZI_COV)
      return fail(c, MLOAM_E_INVALID, "pcd_encode: a layout that is not one of MLOAM_PCD_XYZ / _XYZI / _XYZI_COV");
    if (q.count < 0) return fail(c, MLOAM_E_INVALID, "pcd_encode: a negative count");
    if (q.count > 0 && (!q.pts || (q.layout == MLOAM_PCD_XYZI_COV && (!q.cov6 || !q.trace))))
      return fail(c, MLOAM_E_INVALID, "pcd_encode: a cloud without its points (or cov6 / trace for MLOAM_PCD_XYZI_COV)");
    const size_t m = (size_t)q.count;
    off[k + 1] = off[k] + align256(16 * m) + (q.layout == MLOAM_PCD_XYZI_COV ? align256(24 * m) + align256(4 * m) : 0);
  }
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "pcd_encode: single-GPU only; detach the communicator");
  cudaSetDevice(c->device);
  PcdJob jobs[PW_MAX_FILES];
  for (int k = 0; k < n; k++) {
    const long long bound = PW_HEADER + (long long)clouds[k].count * PW_FIELD * (clouds[k].layout == MLOAM_PCD_XYZI_COV ? 11 : 4);
    if (bound > INT_MAX) return fail(c, MLOAM_E_INVALID, "pcd: a file could exceed 2^31 - 1 bytes");
  }
  MLOAM_CUDA_OK(c, c->pcd_src.reserve(off[n] + 256));
  cudaStream_t st = c->stream;
  for (int k = 0; k < n; k++) {
    const mloam_pcd_cloud_t &q = clouds[k];
    const size_t m = (size_t)q.count;
    unsigned char *p = c->pcd_src.as<unsigned char>() + off[k];
    PcdJob &J = jobs[k];
    J.nf = q.layout == MLOAM_PCD_XYZ ? 3 : q.layout == MLOAM_PCD_XYZI ? 4 : 11, J.cap = q.count, J.n_segs = 1;
    J.seg[0] = PackSeg{reinterpret_cast<const float4 *>(p), nullptr, nullptr, nullptr, q.count, 0};
    if (m == 0) continue;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(p, q.pts, 16 * m, cudaMemcpyHostToDevice, st));
    if (q.layout == MLOAM_PCD_XYZI_COV) {
      unsigned char *pc = p + align256(16 * m), *pt = pc + align256(24 * m);
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(pc, q.cov6, 24 * m, cudaMemcpyHostToDevice, st));
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(pt, q.trace, 4 * m, cudaMemcpyHostToDevice, st));
      J.seg[0].cov6 = reinterpret_cast<const float *>(pc), J.seg[0].trace = reinterpret_cast<const float *>(pt);
    }
  }
  unsigned char *d_file[PW_MAX_FILES];
  const int rc = pcd_write(c, n, jobs, bytes, d_file);
  return rc ? rc : pcd_copy_out(c, n, d_file, bytes, h_data, cap_bytes);
}

}  // extern "C"
