// pcd.cu — the ASCII bodies of the dataset nodes' PCD files -> float4 points (pcl::io::loadPCDFile<pcl::PointXYZ>, rosNodeRVOxford.cpp:
// 355-370, rosNodeRVHercules.cpp:354-368), every file of the rig in two launches.  The rules are host/mloam_io.hpp decodePCDASCII's; a
// token's value is csrc/pcd_ascii.cuh's.
//
// A point is a line that holds a token, and its index is the number of such lines before it, so the decode is a count and a scan:
//  - k_pcd_count: each CTA takes one equal span of one body (pcd_spans spans per body) and counts the lines whose first token starts in
//    it — a byte that is no separator nor '\n' and whose nearest byte before it that is no separator is '\n' or the body's start;
//  - k_pcd_parse: each CTA adds up the counts of the spans before its own, walks its span again in chunks of 16 bytes per thread, numbers
//    the line starts with a block scan and parses every line below POINTS from its start: the x / y / z tokens into float4 (lane 3 = 0),
//    the status word collecting the PCD_E_* bits of a refused body.  The span's last CTA checks the line count against POINTS.
// The bodies' sizes are read on the device (PcdStage), so the launches depend on the point counts and the SM count only.
#include <algorithm>
#include <climits>

#include "ctx.h"
#include "host_util.h"
#include "pcd_ascii.cuh"
#include "primitives.cuh"

namespace mloam {

namespace {

constexpr int PCD_THREADS = PRIM_THREADS;      // prim_block_scan's block
constexpr int PCD_BYTES = 16;                   // bytes per thread and chunk
constexpr int PCD_CHUNK = PCD_THREADS * PCD_BYTES;
constexpr int PCD_MAX_SPANS = 256;

struct PcdRig {
  const unsigned char *data[MLOAM_MAX_LIDARS];  // device bodies; nullptr: the body is at base + PcdStage::off
  const unsigned char *base;                    // the host bodies' staging
  int points[MLOAM_MAX_LIDARS], tokens[MLOAM_MAX_LIDARS], index[MLOAM_MAX_LIDARS][3];
  int out_off[MLOAM_MAX_LIDARS];                // the file's first point in out
  int n_files, spans;                           // spans per body: gridDim.x = n_files x spans
  const PcdStage *stage;
  int *counts;                                  // [n_files][spans] line starts per span
  unsigned *status;
};

__device__ __forceinline__ const unsigned char *pcd_body(const PcdRig &R, int f) { return R.data[f] ? R.data[f] : R.base + R.stage->off[f]; }

// whether the first token of a line starts at byte p of body d.  Only a byte that follows a separator scans back, over that run of
// separators alone: each run is walked once per kernel, so the work stays linear in the body's size.
__device__ __forceinline__ bool pcd_line_start(const unsigned char *d, long long p) {
  const unsigned char ch = __ldg(d + p);
  if (ch == '\n' || pcd::is_sep(ch)) return false;
  long long k = p - 1;
  while (k >= 0 && pcd::is_sep(__ldg(d + k))) k--;
  return k < 0 || __ldg(d + k) == '\n';
}

// the bytes [s0, s1) of span `span` of a body of `size` bytes
__device__ __forceinline__ void pcd_span(long long size, int spans, int span, long long *s0, long long *s1) {
  *s0 = size * span / spans, *s1 = size * (span + 1) / spans;
}

__global__ void __launch_bounds__(PCD_THREADS) k_pcd_count(const __grid_constant__ PcdRig R) {
  const int f = blockIdx.x / R.spans, span = blockIdx.x - f * R.spans;
  const long long size = R.stage->size[f];
  const unsigned char *d = pcd_body(R, f);
  long long s0, s1;
  pcd_span(size, R.spans, span, &s0, &s1);
  int n = 0;
  for (long long c = s0 + (long long)threadIdx.x * PCD_BYTES; c < s1; c += PCD_CHUNK)
    for (int j = 0; j < PCD_BYTES && c + j < s1; j++) n += pcd_line_start(d, c + j) ? 1 : 0;
  int total;
  prim_block_scan(n, &total);
  if (threadIdx.x == 0) R.counts[blockIdx.x] = total;
}

// One line from its first token at p: the x / y / z tokens -> out, or the refusal bits
__device__ unsigned pcd_parse_line(const unsigned char *d, long long size, long long p, int tokens, const int *index, float4 *out) {
  uint32_t v[3] = {0u, 0u, 0u};
  int tok = 0;
  long long k = p;
  unsigned st = 0;
  while (tok < tokens) {
    while (k < size && pcd::is_sep(__ldg(d + k))) k++;
    if (k >= size || __ldg(d + k) == '\n') break;
    const long long a = k;
    while (k < size) {
      const unsigned char ch = __ldg(d + k);
      if (ch == '\n' || pcd::is_sep(ch)) break;
      k++;
    }
    for (int c = 0; c < 3; c++)
      if (index[c] == tok) st |= (unsigned)pcd::parse_float(d + a, k - a, &v[c]) << 1;
    tok++;
  }
  if (tok < tokens) st |= pcd::PCD_E_SHORT_LINE;
  *out = make_float4(__uint_as_float(v[0]), __uint_as_float(v[1]), __uint_as_float(v[2]), 0.f);
  return st;
}

__global__ void __launch_bounds__(PCD_THREADS) k_pcd_parse(const __grid_constant__ PcdRig R, float4 *__restrict__ out) {
  __shared__ int s_base;
  const int f = blockIdx.x / R.spans, span = blockIdx.x - f * R.spans;
  const long long size = R.stage->size[f];
  const unsigned char *d = pcd_body(R, f);
  const int *cnt = R.counts + f * R.spans;
  {  // the line starts of the spans before this one
    int before = 0;
    for (int s = threadIdx.x; s < span; s += PCD_THREADS) before += cnt[s];
    int total;
    prim_block_scan(before, &total);
    if (threadIdx.x == 0) s_base = total;
    __syncthreads();
  }
  int base = s_base;
  const int points = R.points[f], tokens = R.tokens[f];
  const int index[3] = {R.index[f][0], R.index[f][1], R.index[f][2]};
  float4 *o = out + R.out_off[f];
  long long s0, s1;
  pcd_span(size, R.spans, span, &s0, &s1);
  unsigned st = 0;
  for (long long c0 = s0; c0 < s1; c0 += PCD_CHUNK) {  // the same trip count for every thread: the scan below needs the whole block
    const long long c = c0 + (long long)threadIdx.x * PCD_BYTES;
    unsigned mask = 0;
    for (int j = 0; j < PCD_BYTES && c + j < s1; j++) mask |= pcd_line_start(d, c + j) ? 1u << j : 0u;
    int total;
    int i = base + prim_block_scan(__popc(mask), &total);
    for (; mask && i < points; mask &= mask - 1, i++) st |= pcd_parse_line(d, size, c + __ffs(mask) - 1, tokens, index, o + i);
    base += total;
  }
  if (span == R.spans - 1 && threadIdx.x == 0 && base < points) st |= pcd::PCD_E_FEW_LINES;
  if (st) atomicOr(R.status, st);
}

// the spans of a body: as many CTAs as two per SM over the whole decode, at least one per file
int pcd_spans(const Ctx *c, int n) { return std::max(1, std::min(PCD_MAX_SPANS, 2 * c->sm_count / n)); }

// The kernel arguments of n bodies: device bodies at their pointers, host ones at base + PcdStage::off
void pcd_rig(const Ctx *c, int n, const mloam_pcd_t *pcds, bool host, const unsigned char *base, PcdRig *R) {
  memset(R, 0, sizeof(*R));
  R->n_files = n, R->spans = pcd_spans(c, n), R->base = host ? base : nullptr;
  for (int f = 0; f < n; f++) {
    const mloam_pcd_t &p = pcds[f];
    if (!host) R->data[f] = static_cast<const unsigned char *>(p.data);
    R->points[f] = p.points, R->tokens[f] = p.tokens, R->out_off[f] = f ? R->out_off[f - 1] + pcds[f - 1].points : 0;
    for (int k = 0; k < 3; k++) R->index[f][k] = p.index[k];
  }
}

// The PcdStage h_stage (pinned) to the device, the status word cleared, then the two launches on c->stream
int pcd_launch(Ctx *c, PcdRig &R, const PcdStage *h_stage, PcdStage *d_stage, int *d_counts, unsigned *d_status, float4 *out) {
  cudaStream_t st = c->stream;
  R.stage = d_stage, R.counts = d_counts, R.status = d_status;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_stage, h_stage, sizeof(PcdStage), cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemsetAsync(d_status, 0, sizeof(unsigned), st));
  const int grid = R.n_files * R.spans;
  ProfScope ps(c, "pcd_decode");
  k_pcd_count<<<grid, PCD_THREADS, 0, st>>>(R);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  k_pcd_parse<<<grid, PCD_THREADS, 0, st>>>(R, out);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

// the per-half regions of Ctx::pcd_frame: a fixed size, so that it is allocated once
struct PcdHalf {
  PcdStage *stage;
  unsigned *status;
  int *counts;
};
int pcd_frame_bufs(Ctx *c, int half, PcdHalf *H) {
  PcdStage *stage;
  unsigned *status;
  int *counts;
  MLOAM_CUDA_OK(c, carve(c->pcd_frame, [&](Carve &cv) {
    stage = cv.take<PcdStage>(2), status = cv.take<unsigned>(4), counts = cv.take<int>(2 * (size_t)MLOAM_MAX_LIDARS * PCD_MAX_SPANS);
  }));
  H->stage = stage + half, H->status = status + half, H->counts = counts + (size_t)half * MLOAM_MAX_LIDARS * PCD_MAX_SPANS;
  return MLOAM_OK;
}

}  // namespace

int pcd_check(Ctx *c, int n, const mloam_pcd_t *pcds) {
  if (n < 1 || n > MLOAM_MAX_LIDARS || !pcds) return fail(c, MLOAM_E_INVALID, "pcd: 1..MLOAM_MAX_LIDARS files");
  long long total = 0;
  for (int f = 0; f < n; f++) {
    const mloam_pcd_t &p = pcds[f];
    if (!p.data && p.size > 0) return fail(c, MLOAM_E_INVALID, "pcd: a body without data");
    if (p.points < 1) return fail(c, MLOAM_E_INVALID, "pcd: every file needs POINTS >= 1");
    if (p.tokens < 1) return fail(c, MLOAM_E_INVALID, "pcd: tokens per line < 1");
    if (p.size > ((size_t)1 << 40)) return fail(c, MLOAM_E_INVALID, "pcd: a body over 2^40 bytes");
    for (int k = 0; k < 3; k++)
      if (p.index[k] < 0 || p.index[k] >= p.tokens) return fail(c, MLOAM_E_INVALID, "pcd: a token index outside [0, tokens)");
    total += p.points;
    if (total > (1 << 30)) return fail(c, MLOAM_E_INVALID, "pcd: more than 2^30 points");
  }
  return MLOAM_OK;
}

int pcd_refusal(Ctx *c, unsigned s) {
  if (s & pcd::PCD_E_BAD_TOKEN) return fail(c, MLOAM_E_INVALID, "pcd: an x / y / z token outside the grammar (see mloam_pcd_t)");
  if (s & pcd::PCD_E_TOO_LONG) return fail(c, MLOAM_E_INVALID, "pcd: an x / y / z token with more than 19 significant digits");
  if (s & pcd::PCD_E_SHORT_LINE) return fail(c, MLOAM_E_INVALID, "pcd: a line with fewer tokens than the header's");
  if (s & pcd::PCD_E_FEW_LINES) return fail(c, MLOAM_E_INVALID, "pcd: fewer lines than POINTS");
  return MLOAM_OK;
}

// The PcdStage of a PCD sweep: each body's size and, for host bytes, its offset in the device staging (256-byte aligned) — staged per
// frame, never part of a graph key
static void pcd_stage(const Sweep &sw, PcdStage *st) {
  long long off = 0;
  for (int l = 0; l < sw.L.n_lidars; l++) {
    const mloam_pcd_t &p = sw.pcdf.body[l];
    st->size[l] = (long long)p.size, st->off[l] = sw.host ? off : 0;
    off += (long long)((p.size + 255) & ~(size_t)255);
  }
}

int pcd_upload(Ctx *c, DevBuf &B, Sweep *sw, bool upload, cudaStream_t st) {
  PcdStage ps;
  pcd_stage(*sw, &ps);
  const int nl = sw->L.n_lidars;
  const size_t need = (size_t)(ps.off[nl - 1] + ps.size[nl - 1]) + 16;
  if (need > B.cap) MLOAM_CUDA_OK(c, B.reserve(need + need / 2));
  sw->bytes = B.as<unsigned char>();
  for (int l = 0; upload && l < nl; l++)
    if (ps.size[l]) MLOAM_CUDA_OK(c, cudaMemcpyAsync(B.as<unsigned char>() + ps.off[l], sw->pcdf.body[l].data, (size_t)ps.size[l], cudaMemcpyHostToDevice, st));
  return MLOAM_OK;
}

int pcd_decode_half(Ctx *c, const Sweep &sw, int half, float4 *out) {
  PcdHalf H;
  int rc = pcd_frame_bufs(c, half, &H);
  if (rc) return rc;
  PcdRig R;
  pcd_rig(c, sw.L.n_lidars, sw.pcdf.body, sw.host, sw.bytes, &R);
  return pcd_launch(c, R, &c->pinned->pcd_half[half], H.stage, H.counts, H.status, out);
}

void pcd_frame_stage(Ctx *c, const Sweep &sw, int half) {
  if (sw.kind == SweepKind::pcd) pcd_stage(sw, &c->pinned->pcd_half[half]);
}

int pcd_frame_land(Ctx *c, const Sweep &sw) {
  if (sw.kind != SweepKind::pcd) return MLOAM_OK;
  PcdHalf H;
  const int rc = pcd_frame_bufs(c, 0, &H);
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->pinned->pcd_half_status, H.status, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, c->stream));
  return MLOAM_OK;
}

int pcd_frame_refusal(Ctx *c, const Sweep &sw, int half) {
  if (sw.kind != SweepKind::pcd) return MLOAM_OK;
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return pcd_refusal(c, c->pinned->pcd_half_status[half]);
}

int pcd_decode_device(Ctx *c, int n, const mloam_pcd_t *pcds, bool host, float4 *out) {
  int rc = pcd_check(c, n, pcds);
  if (rc) return rc;
  cudaSetDevice(c->device);
  PcdStage &S = c->pinned->pcd;
  long long off = 0;
  for (int f = 0; f < n; f++) {
    S.size[f] = (long long)pcds[f].size, S.off[f] = off;
    if (host) off += (long long)((pcds[f].size + 255) & ~(size_t)255);
  }
  cudaStream_t st = c->stream;
  if (host) {
    MLOAM_CUDA_OK(c, c->pcd_in.reserve((size_t)off + 16));
    for (int f = 0; f < n; f++)
      if (pcds[f].size) MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->pcd_in.as<unsigned char>() + S.off[f], pcds[f].data, pcds[f].size, cudaMemcpyHostToDevice, st));
  }
  PcdRig R;
  pcd_rig(c, n, pcds, host, c->pcd_in.as<unsigned char>(), &R);
  PcdStage *d_stage;
  int *d_counts;
  unsigned *d_status;
  MLOAM_CUDA_OK(c, carve(c->pcd_work, [&](Carve &cv) {
    d_stage = cv.take<PcdStage>(1), d_counts = cv.take<int>((size_t)MLOAM_MAX_LIDARS * PCD_MAX_SPANS), d_status = cv.take<unsigned>(4);
  }));
  rc = pcd_launch(c, R, &S, d_stage, d_counts, d_status, out);
  if (rc) return rc;
  unsigned *hs = &c->pinned->pcd_status;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hs, d_status, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return pcd_refusal(c, *hs);
}

}  // namespace mloam

using namespace mloam;

extern "C" {

int mloam_pcd_decode(mloam_ctx_t *h, int n, const mloam_pcd_t *pcds, mloam_point_t *h_out) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!h_out) return fail(c, MLOAM_E_INVALID, "pcd_decode: h_out must not be NULL");
  long long total = 0;
  for (int f = 0; pcds && f < n && f < MLOAM_MAX_LIDARS; f++) total += std::max(0, pcds[f].points);
  DevBuf &B = c->map_in[0];  // the host entry points' output
  MLOAM_CUDA_OK(c, B.reserve(sizeof(float4) * (size_t)(std::min<long long>(total, 1 << 30) + 1)));
  const int rc = pcd_decode_device(c, n, pcds, true, B.as<float4>());
  if (rc) return rc;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, B.p, sizeof(float4) * (size_t)total, cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}

int mloam_pcd_decode_device(mloam_ctx_t *h, int n, const mloam_pcd_t *pcds, mloam_point_t *d_out) {
  if (!h) return MLOAM_E_INVALID;
  if (!d_out) return fail(&h->c, MLOAM_E_INVALID, "pcd_decode_device: d_out must not be NULL");
  return pcd_decode_device(&h->c, n, pcds, false, reinterpret_cast<float4 *>(d_out));
}

}  // extern "C"
