// wire.cu — the rig's sensor_msgs/PointCloud2 messages -> the float4 raw sweep of the front end (pcl::fromROSMsg in the driver nodes,
// rosNodeRVHercules.cpp:169, rosNodeRVKITTI.cpp:157, rosNodeRVOxford.cpp:173), one launch over every LiDAR of the rig.  The rules are
// host/mloam_io.hpp unpackPointCloud2's: fields at any byte offset, FLOAT32 or FLOAT64 (rounded to float as (float)d), byte-swapped when
// the message's endianness is not the device's, organised clouds row-major with rows row_step bytes apart.  Non-finite points are
// written as they are: the front end's removeNaN drops them.
//
// Memory pattern: a point is point_step bytes (22, 32, 48 in real drivers), so its fields are unaligned in general.  Each warp takes 32
// points of one row — contiguous bytes — and stages them into shared memory with 16-byte loads (byte loads only in the two partial words
// at the ends, so nothing outside the message is read); the fields are then picked from shared memory and the float4s stored coalesced.
//
// The way out (mloam_cloud_msgs*): pcl::toROSMsg of the clouds the mapper publishes (lidar_mapper_keyframe.cpp:690-714, :780-851) into
// the 32-byte PointXYZI or 48-byte PointXYZIWithCov layout, up to six messages in one launch, k_wire_pack.  Point steps are multiples of
// 16 and every message starts 256-byte aligned, so each thread writes its point as 2 or 3 uint4 stores, the warp's stores covering
// contiguous bytes; the float4 points are read coalesced, cov_vec as three float2 per point.
#include <algorithm>
#include <climits>

#include "ctx.h"
#include "host_util.h"

namespace mloam {

namespace {

constexpr int WIRE_MAX_WARPS = 8;
constexpr int WIRE_SMEM = 48 * 1024;  // per CTA, without the opt-in: one warp of 32 x 1024-byte points fits

struct WireRig {
  const unsigned char *data[MLOAM_MAX_LIDARS];  // each LiDAR's bytes on the device
  long long row_step[MLOAM_MAX_LIDARS];
  int width[MLOAM_MAX_LIDARS];
  int task_off[MLOAM_MAX_LIDARS + 1];           // warp tasks (32-point pieces of a row) of the LiDARs before l
  int out_off[MLOAM_MAX_LIDARS];                // the LiDAR's first point in the raw sweep (RigLayout::off)
  mloam_pc2_layout_t layout[MLOAM_MAX_LIDARS];
  int n_lidars;
  int warp_bytes;                               // shared memory per warp: 32 x the rig's largest point_step + 32, a multiple of 16
};

// One field of a point staged in shared memory: 4 or 8 bytes, little-endian unless swap
__device__ __forceinline__ float wire_field(const unsigned char *p, int datatype, bool swap) {
  if (datatype == 8) {
    unsigned long long v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v |= (unsigned long long)p[swap ? 7 - i : i] << (8 * i);
    return __double2float_rn(__longlong_as_double((long long)v));
  }
  unsigned v = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) v |= (unsigned)p[swap ? 3 - i : i] << (8 * i);
  return __uint_as_float(v);
}

__global__ void __launch_bounds__(WIRE_MAX_WARPS * 32) k_wire_unpack(const __grid_constant__ WireRig R, float4 *__restrict__ out) {
  extern __shared__ __align__(16) unsigned char wire_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int task = blockIdx.x * (blockDim.x >> 5) + warp;
  if (task >= R.task_off[R.n_lidars]) return;
  int l = 0;
  while (task >= R.task_off[l + 1]) l++;
  const int w = R.width[l], chunks = (w + 31) >> 5, t = task - R.task_off[l];
  const int row = t / chunks, col0 = (t - row * chunks) << 5;
  const int np = min(32, w - col0);
  const int step = R.layout[l].point_step;
  const unsigned char *src = R.data[l] + (long long)row * R.row_step[l] + (long long)col0 * step;
  const size_t nbytes = (size_t)np * step;
  // the 16-byte words covering [src, src + nbytes); buf[k] holds the byte at a0 + k
  const size_t s = reinterpret_cast<size_t>(src), a0 = s & ~(size_t)15, a1 = (s + nbytes + 15) & ~(size_t)15;
  unsigned char *buf = wire_smem + (size_t)warp * R.warp_bytes;
  for (size_t a = a0 + 16 * (size_t)lane; a < a1; a += 512) {
    uint4 v;
    if (a >= s && a + 16 <= s + nbytes) {
      v = __ldg(reinterpret_cast<const uint4 *>(a));
    } else {  // a partial word at either end: only the message's own bytes
      unsigned char b[16];
#pragma unroll
      for (int k = 0; k < 16; k++) b[k] = (a + k >= s && a + k < s + nbytes) ? *reinterpret_cast<const unsigned char *>(a + k) : 0;
      memcpy(&v, b, 16);
    }
    *reinterpret_cast<uint4 *>(buf + (a - a0)) = v;
  }
  __syncwarp();
  if (lane >= np) return;
  const mloam_pc2_layout_t &F = R.layout[l];
  const unsigned char *p = buf + (s - a0) + (size_t)lane * step;
  const bool swap = F.is_bigendian != 0;  // the device is little-endian
  float4 q;
  q.x = wire_field(p + F.offset[0], F.datatype[0], swap);
  q.y = wire_field(p + F.offset[1], F.datatype[1], swap);
  q.z = wire_field(p + F.offset[2], F.datatype[2], swap);
  q.w = F.datatype[3] ? wire_field(p + F.offset[3], F.datatype[3], swap) : 0.f;
  out[R.out_off[l] + row * w + col0 + lane] = q;
}

// ---- the way out: pcl::toROSMsg of the mapper's published clouds (mloam_cloud_msgs*)
constexpr int PACK_THREADS = 256;
constexpr int PACK_MAX_MSGS = 6;
constexpr int PACK_MAX_SEGS = 2 * PACK_MAX_MSGS;

struct PackBatch {
  PackSeg seg[PACK_MAX_SEGS];               // in message order; a message's segments are consecutive
  unsigned char *out[PACK_MAX_MSGS];        // each message's bytes, 256-byte aligned
  int step[PACK_MAX_MSGS];                  // 32 (PointXYZI) or 48 (PointXYZIWithCov)
  int n_segs, n_msgs;
  int *width;                               // out: the messages' point counts
};

// Grid-stride over the points of every segment.  Every block reads the counts (a registered cloud's lives on the device); block 0
// publishes the widths.  A point is written whole, as 2 or 3 uint4 stores at its 16-byte aligned slot:
//   32 B: x y z 0 | intensity 0 0 0         48 B: x y z 0 | intensity cov_xx cov_xy cov_xz | cov_yy cov_yz cov_zz cov_trace
// Bits are moved, never computed on, so NaN payloads and signed zeros survive.
__global__ void __launch_bounds__(PACK_THREADS) k_wire_pack(const __grid_constant__ PackBatch B) {
  __shared__ int s_start[PACK_MAX_SEGS + 1];  // the segment's first point in the batch
  __shared__ int s_at[PACK_MAX_SEGS];         // ... and in its message
  const int tid = threadIdx.x;
  if (tid == 0) {
    int tot = 0, at = 0;
    for (int s = 0; s < B.n_segs; s++) {
      const PackSeg &g = B.seg[s];
      const int n = g.d_n ? max(0, min(g.n, *g.d_n)) : g.n;
      if (s > 0 && g.cloud != B.seg[s - 1].cloud) at = 0;
      s_start[s] = tot, s_at[s] = at;
      tot += n, at += n;
      if (blockIdx.x == 0 && (s + 1 == B.n_segs || B.seg[s + 1].cloud != g.cloud)) B.width[g.cloud] = at;
    }
    s_start[B.n_segs] = tot;
  }
  __syncthreads();
  const int total = s_start[B.n_segs];
  for (int i = blockIdx.x * PACK_THREADS + tid; i < total; i += gridDim.x * PACK_THREADS) {
    int s = 0;
    while (i >= s_start[s + 1]) s++;
    const PackSeg &g = B.seg[s];
    const int k = i - s_start[s], m = g.cloud;
    const float4 p = __ldg(g.pts + k);
    uint4 *dst = reinterpret_cast<uint4 *>(B.out[m] + (size_t)(s_at[s] + k) * B.step[m]);
    dst[0] = make_uint4(__float_as_uint(p.x), __float_as_uint(p.y), __float_as_uint(p.z), 0u);
    if (B.step[m] == 32) {
      dst[1] = make_uint4(__float_as_uint(p.w), 0u, 0u, 0u);
    } else {
      const float2 *c = reinterpret_cast<const float2 *>(g.cov6 + 6 * (size_t)k);  // 24-byte rows: 8-byte aligned
      const float2 c01 = __ldg(c), c23 = __ldg(c + 1), c45 = __ldg(c + 2);
      dst[1] = make_uint4(__float_as_uint(p.w), __float_as_uint(c01.x), __float_as_uint(c01.y), __float_as_uint(c23.x));
      dst[2] = make_uint4(__float_as_uint(c23.y), __float_as_uint(c45.x), __float_as_uint(c45.y), __float_as_uint(__ldg(g.trace + k)));
    }
  }
}

bool is_registered_msg(int source) { return source <= MLOAM_MSG_CORNER_LAST; }
size_t msg_step(int source) { return is_registered_msg(source) ? 32 : 48; }

// The checks both entry points make, then the launch; widths and device addresses of the n messages on return (the stream synchronised)
int cloud_msgs_pack(Ctx *c, int n, const int *sources, int *width, unsigned char **d_msg) {
  if (!sources || !width || n < 1 || n > PACK_MAX_MSGS) return fail(c, MLOAM_E_INVALID, "cloud_msgs: 1..6 sources, non-NULL arrays");
  for (int k = 0; k < n; k++) width[k] = 0;
  bool seen[PACK_MAX_MSGS] = {false, false, false, false, false, false};
  for (int k = 0; k < n; k++) {
    const int s = sources[k];
    if (s < MLOAM_MSG_FULL_RES || s > MLOAM_MSG_GLOBAL_MAP1 || seen[s])
      return fail(c, MLOAM_E_INVALID, "cloud_msgs: a source is not one of MLOAM_MSG_* or is given twice");
    seen[s] = true;
  }
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "cloud_msgs: single-GPU only; detach the communicator");
  for (int k = 0; k < n; k++) {
    if (is_registered_msg(sources[k]) && !c->reg_valid)
      return fail(c, MLOAM_E_STATE, "cloud_msgs: the last call was no mloam_frame* call run with the registered clouds on (mloam_set_registered)");
    if (!is_registered_msg(sources[k]) && !c->kf) return fail(c, MLOAM_E_STATE, "cloud_msgs: call mloam_keyframes_init first");
  }
  cudaSetDevice(c->device);
  PackBatch B;
  memset(&B, 0, sizeof(B));
  B.n_msgs = n;
  size_t off[PACK_MAX_MSGS + 1] = {0};
  long long bound = 0;
  for (int k = 0; k < n; k++) {
    const int s = sources[k];
    PackSeg *seg = B.seg + B.n_segs;
    int ns = 1;
    if (is_registered_msg(s)) {
      const int w = s - MLOAM_MSG_FULL_RES;  // MLOAM_REGISTERED_* of the same order
      seg[0] = PackSeg{c->reg_last.cloud[w], nullptr, nullptr, c->reg_last.counts + w, c->reg_last.cap[w], 0};
    } else {
      ns = keyframe_msg_segments(c, s, seg);
    }
    B.step[k] = (int)msg_step(s);
    long long cap = 0;
    for (int j = 0; j < ns; j++) seg[j].cloud = k, cap += seg[j].n;
    B.n_segs += ns, bound += cap;
    off[k + 1] = off[k] + align256((size_t)cap * B.step[k]);
  }
  if (bound > INT_MAX) return fail(c, MLOAM_E_INVALID, "cloud_msgs: more than 2^31 points in one call");
  MLOAM_CUDA_OK(c, c->cloud_msgs.reserve(off[n] + 256));
  unsigned char *base = c->cloud_msgs.as<unsigned char>();
  for (int k = 0; k < n; k++) B.out[k] = d_msg[k] = base + off[k];
  B.width = reinterpret_cast<int *>(base + off[n]);
  const long long grid = std::min<long long>(std::max<long long>(1, (bound + PACK_THREADS - 1) / PACK_THREADS), 8ll * c->sm_count);
  {
    ProfScope ps(c, "wire_pack");
    k_wire_pack<<<(unsigned)grid, PACK_THREADS, 0, c->stream>>>(B);
    c->launches++;
    MLOAM_CUDA_OK(c, cudaGetLastError());
  }
  int *hw = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hw, B.width, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  for (int k = 0; k < n; k++) width[k] = hw[k];
  return MLOAM_OK;
}

}  // namespace

// where LiDAR l's bytes lie in a host message sweep's device staging (256-byte aligned), and l = n_lidars: the staging's size
static size_t wire_stage_offset(const WireMsgs &w, int l) {
  size_t off = 0;
  for (int k = 0; k < l; k++) off += ((size_t)w.msg[k].height * w.msg[k].row_step + 255) & ~(size_t)255;
  return off;
}

int wire_upload(Ctx *c, DevBuf &B, Sweep *sw, bool upload, cudaStream_t st) {
  const WireMsgs &w = sw->wire;
  MLOAM_CUDA_OK(c, B.reserve(wire_stage_offset(w, sw->L.n_lidars)));
  sw->bytes = B.as<unsigned char>();
  for (int l = 0; upload && l < sw->L.n_lidars; l++)
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(B.as<unsigned char>() + wire_stage_offset(w, l), w.msg[l].data, (size_t)w.msg[l].height * w.msg[l].row_step,
                                     cudaMemcpyHostToDevice, st));
  return MLOAM_OK;
}

int wire_unpack_device(Ctx *c, const Sweep &sw, float4 *out) {
  WireRig R;
  memset(&R, 0, sizeof(R));
  R.n_lidars = sw.L.n_lidars;
  int max_step = 1;
  for (int l = 0; l < R.n_lidars; l++) {
    const mloam_pc2_msg_t &m = sw.wire.msg[l];
    R.data[l] = sw.host ? sw.bytes + wire_stage_offset(sw.wire, l) : static_cast<const unsigned char *>(m.data);
    R.row_step[l] = (long long)m.row_step, R.width[l] = m.width, R.out_off[l] = sw.L.off[l];
    R.layout[l] = sw.wire.layout[l];
    R.task_off[l + 1] = R.task_off[l] + m.height * ((m.width + 31) / 32);  // <= 2^30 points in all: no overflow
    max_step = max(max_step, R.layout[l].point_step);
  }
  R.warp_bytes = (32 * max_step + 32 + 15) & ~15;
  const int warps = min(WIRE_MAX_WARPS, WIRE_SMEM / R.warp_bytes);
  const int tasks = R.task_off[R.n_lidars];
  ProfScope ps(c, "wire_unpack");
  k_wire_unpack<<<(tasks + warps - 1) / warps, 32 * warps, (size_t)warps * R.warp_bytes, c->stream>>>(R, out);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

}  // namespace mloam

using namespace mloam;

extern "C" {

int mloam_cloud_msgs(mloam_ctx_t *h, int n, const int *sources, void *const *h_data, const size_t *cap_bytes, int *width) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!h_data || !cap_bytes) return fail(c, MLOAM_E_INVALID, "cloud_msgs: h_data and cap_bytes must not be NULL");
  unsigned char *d_msg[PACK_MAX_MSGS];
  const int rc = cloud_msgs_pack(c, n, sources, width, d_msg);
  if (rc) return rc;
  for (int k = 0; k < n; k++)
    if (h_data[k] && (size_t)width[k] * msg_step(sources[k]) > cap_bytes[k])
      return fail(c, MLOAM_E_INVALID, "cloud_msgs: a capacity is too small (width holds the messages' sizes)");
  bool copied = false;
  for (int k = 0; k < n; k++) {
    const size_t bytes = (size_t)width[k] * msg_step(sources[k]);
    if (!h_data[k] || bytes == 0) continue;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_data[k], d_msg[k], bytes, cudaMemcpyDeviceToHost, c->stream));
    copied = true;
  }
  if (copied) MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}

int mloam_cloud_msgs_device(mloam_ctx_t *h, int n, const int *sources, const void **d_data, int *width) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!d_data) return fail(c, MLOAM_E_INVALID, "cloud_msgs_device: d_data must not be NULL");
  unsigned char *d_msg[PACK_MAX_MSGS];
  const int rc = cloud_msgs_pack(c, n, sources, width, d_msg);
  if (rc) return rc;
  for (int k = 0; k < n; k++) d_data[k] = d_msg[k];
  return MLOAM_OK;
}

}  // extern "C"
