// exp32(x): a float32 exponential for the bilateral depth filter's weights exp(-(s + c_r d^2)) (gsx_filter.cu), on
// x in [-17, 0] (the filter skips pairs below -17).  Every step is a separately rounded float32 operation in the order
// written - no FMA (the library builds with -fmad=false, the host test with -ffp-contract=off) and no hardware
// ex2.approx - so numpy float32 states it operation for operation (tests/bilateral_oracle.py exp32) and the filtered
// depth, and everything fused from it, is bit-identical to the CPU oracle:
//     k = rint(x log2e),  r = (x - k ln2_hi) - k ln2_lo  (ln2_hi has 16 significant bits: k ln2_hi and the first
//     subtraction are exact for |k| <= 25),  exp(r) by the degree-7 Taylor polynomial in Horner form
//     (|r| <= 0.35: truncation < 6e-9),  times 2^k built in the exponent field (the result is normal: no underflow).
// exp32(0) = exp32(-0) = 1 exactly; tests/test_depth_filter_host.py checks every float32 in [-17, 0] against the
// oracle bit for bit and against float32(exp(float64 x)) to kExp32MaxUlps.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#ifndef GSX_HD
#ifdef __CUDACC__
#define GSX_HD __host__ __device__
#else
#define GSX_HD
#endif
#endif

namespace gsx {

constexpr int kExp32MaxUlps = 1;        // against float32(exp(float64 x)) on [-17, 0]
constexpr float kExp32Min = -17.0f;     // arguments below are outside the range exp32 is stated for

GSX_HD inline float exp32_scale(int k) {  // 2^k for k in [-126, 127]
  const uint32_t b = (uint32_t)(k + 127) << 23;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f;
  memcpy(&f, &b, 4);
  return f;
#endif
}

GSX_HD inline float exp32(float x) {
  const float kLog2e = 1.44269502f, kLn2Hi = 0.693145751953125f, kLn2Lo = 1.42860677e-06f;
  const float k = rintf(x * kLog2e);
  const float r = (x - k * kLn2Hi) - k * kLn2Lo;
  float p = 1.98412698e-04f;  // 1/7!
  p = p * r + 1.38888889e-03f;  // 1/6!
  p = p * r + 8.33333377e-03f;  // 1/5!
  p = p * r + 4.16666679e-02f;  // 1/4!
  p = p * r + 1.66666672e-01f;  // 1/3!
  p = p * r + 0.5f;
  p = p * r + 1.0f;
  p = p * r + 1.0f;
  return p * exp32_scale((int)k);
}

}  // namespace gsx
