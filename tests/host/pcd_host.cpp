// Host build of csrc/pcd_ascii.cuh and the PCD helpers of m-loam_b200/host/mloam_io.hpp for tests/test_pcd_frames_cpu.py and
// tests/test_pcd_frames.py: the token parser the device runs, libstdc++'s reading of a token as PCL calls it, and the header / body rules.
#include <cstdio>
#include <cstdlib>
#include <locale>
#include <sstream>
#include <string>

#include "../../m-loam_b200/host/mloam_io.hpp"

using namespace mloam::io;

// Tokens: n of them back to back in buf, token k at [off[k], off[k + 1]).  pcd_parse: the device parser, status[k] and bits[k]
extern "C" void pcd_parse(const unsigned char *buf, const long long *off, long long n, int *status, unsigned *bits) {
  for (long long k = 0; k < n; k++) status[k] = pcd::parse_float(buf + off[k], off[k + 1] - off[k], bits + k);
}

// ... and the float PCL's copyStringValue<float> stores: "nan", else istringstream >> f in the classic locale, else (float)atof
extern "C" void pcd_stream(const unsigned char *buf, const long long *off, long long n, unsigned *bits) {
  for (long long k = 0; k < n; k++) {
    const std::string tok(reinterpret_cast<const char *>(buf) + off[k], (size_t)(off[k + 1] - off[k]));
    float v;
    if (tok == "nan") {
      v = std::numeric_limits<float>::quiet_NaN();
    } else {
      std::istringstream is(tok);
      is.imbue(std::locale::classic());
      if (!(is >> v)) v = static_cast<float>(std::atof(tok.c_str()));
    }
    std::memcpy(bits + k, &v, 4);
  }
}

// %.<prec>g of n floats (bits), back to back into buf (cap bytes), token k at [off[k], off[k + 1]); returns the bytes written or -1
extern "C" long long pcd_format(const unsigned *bits, long long n, int prec, char *buf, long long cap, long long *off) {
  long long at = 0;
  for (long long k = 0; k < n; k++) {
    float v;
    std::memcpy(&v, bits + k, 4);
    off[k] = at;
    const int w = std::snprintf(buf + at, (size_t)(cap - at), "%.*g", prec, (double)v);
    if (w < 0 || at + w >= cap) return -1;
    at += w;
  }
  off[n] = at;
  return at;
}

// resolvePCDHeader: 1 and out = {points, body, tokens, ix, iy, iz, binary, point_step, ox, oy, oz}; 0: refused
extern "C" int pcd_header(const uint8_t *bytes, size_t size, long long *out) {
  PCDLayout h;
  if (!resolvePCDHeader(bytes, size, h)) return 0;
  const long long v[11] = {h.points, (long long)h.body, h.tokens, h.index[0], h.index[1], h.index[2], h.binary ? 1 : 0, h.point_step,
                           h.offset[0], h.offset[1], h.offset[2]};
  std::memcpy(out, v, sizeof(v));
  return 1;
}

// pcdBinaryMsg of a binary file: 1 and its layout / message; 0: refused
extern "C" int pcd_binary_msg(const uint8_t *bytes, size_t size, mloam_pc2_layout_t *layout, mloam_pc2_msg_t *msg) {
  PCDLayout h;
  if (!resolvePCDHeader(bytes, size, h)) return 0;
  return pcdBinaryMsg(bytes, size, h, *layout, *msg) ? 1 : 0;
}

// decodePCDASCII: its return value; out holds points float4s
extern "C" int pcd_decode_ascii(const uint8_t *body, size_t size, int points, int tokens, const int *index, float *out) {
  std::vector<mloam_point_t> pts;
  const int rc = decodePCDASCII(body, size, points, tokens, index, pts);
  if (!pts.empty()) std::memcpy(out, pts.data(), sizeof(mloam_point_t) * pts.size());
  return rc;
}

// PCL's own ASCII read of a body, for timing: lines, tokens and copyStringValue<float> of x / y / z, nothing else checked.  Returns the
// points read.
extern "C" int pcd_pcl_read(const uint8_t *body, size_t size, int points, const int *index, float *out) {
  int idx = 0;
  size_t at = 0;
  std::vector<std::string> st;
  while (at < size && idx < points) {
    size_t end = at;
    while (end < size && body[end] != '\n') end++;
    const size_t a = at;
    at = end < size ? end + 1 : end;
    st.clear();
    for (size_t k = a; k < end;) {
      while (k < end && pcd::is_sep(body[k])) k++;
      const size_t t0 = k;
      while (k < end && !pcd::is_sep(body[k])) k++;
      if (k > t0) st.emplace_back(reinterpret_cast<const char *>(body) + t0, k - t0);
    }
    if (st.empty()) continue;
    for (int c = 0; c < 3; c++) {
      const std::string &tok = st[(size_t)index[c]];
      float v;
      if (tok == "nan") {
        v = std::numeric_limits<float>::quiet_NaN();
      } else {
        std::istringstream is(tok);
        is.imbue(std::locale::classic());
        if (!(is >> v)) v = static_cast<float>(std::atof(tok.c_str()));
      }
      out[4 * (size_t)idx + c] = v;
    }
    out[4 * (size_t)idx + 3] = 0.f;
    idx++;
  }
  return idx;
}
