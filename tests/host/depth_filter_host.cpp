// Host build of gradslam_b200/csrc/gsx_exp32.cuh (see tests/test_depth_filter_host.py): exp32 of the float32 arguments
// whose bit patterns are [bits_begin, bits_begin + n), into out.
#include "../../gradslam_b200/csrc/gsx_exp32.cuh"

extern "C" void exp32_fill(uint32_t bits_begin, uint32_t n, float *out) {
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t b = bits_begin + i;
    float x;
    memcpy(&x, &b, 4);
    out[i] = gsx::exp32(x);
  }
}

extern "C" int exp32_max_ulps(void) { return gsx::kExp32MaxUlps; }
