// Host build of csrc/pcd_format.cuh and of host/mloam_io.hpp writePCDASCII for tests/test_pcd_write_cpu.py and tests/test_pcd_write.py:
// the characters the device writes for a float, and PCL's writer restated with iostreams.
#include <cstring>
#include <string>

#include "../../m-loam_b200/csrc/pcd_format.cuh"
#include "../../m-loam_b200/host/mloam_io.hpp"

// pcd::format_float of n floats (bits), back to back into buf (cap bytes), token k at [off[k], off[k + 1]); returns the bytes written or -1
extern "C" long long pcd_format8(const unsigned *bits, long long n, char *buf, long long cap, long long *off) {
  long long at = 0;
  for (long long k = 0; k < n; k++) {
    off[k] = at;
    if (at + pcd::PCD_FMT_MAX > cap) return -1;
    at += pcd::format_float(bits[k], buf + at);
  }
  off[n] = at;
  return at;
}

// writePCDASCII of n points into buf (cap bytes); returns the file's size, or -1 when it does not fit
extern "C" long long pcd_write_ascii(int layout, const mloam_point_t *pts, const float *cov6, const float *trace, long long n, char *buf,
                                     long long cap) {
  const std::string s = mloam::io::writePCDASCII(layout, pts, cov6, trace, (size_t)n);
  if ((long long)s.size() > cap) return -1;
  std::memcpy(buf, s.data(), s.size());
  return (long long)s.size();
}
