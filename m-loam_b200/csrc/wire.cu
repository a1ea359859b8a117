// wire.cu — the rig's sensor_msgs/PointCloud2 messages -> the float4 raw sweep of the front end (pcl::fromROSMsg in the driver nodes,
// rosNodeRVHercules.cpp:169, rosNodeRVKITTI.cpp:157, rosNodeRVOxford.cpp:173), one launch over every LiDAR of the rig.  The rules are
// host/mloam_io.hpp unpackPointCloud2's: fields at any byte offset, FLOAT32 or FLOAT64 (rounded to float as (float)d), byte-swapped when
// the message's endianness is not the device's, organised clouds row-major with rows row_step bytes apart.  Non-finite points are
// written as they are: the front end's removeNaN drops them.
//
// Memory pattern: a point is point_step bytes (22, 32, 48 in real drivers), so its fields are unaligned in general.  Each warp takes 32
// points of one row — contiguous bytes — and stages them into shared memory with 16-byte loads (byte loads only in the two partial words
// at the ends, so nothing outside the message is read); the fields are then picked from shared memory and the float4s stored coalesced.
#include "ctx.h"

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

}  // namespace

size_t wire_stage_offset(const WireMsgs &w, int l) {
  size_t off = 0;
  for (int k = 0; k < l; k++) off += ((size_t)w.msg[k].height * w.msg[k].row_step + 255) & ~(size_t)255;
  return off;
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
