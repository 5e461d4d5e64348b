// Edge-preserving bilateral filter of input depth (KinectFusion, Newcombe et al. 2011; the surfel systems after it
// smooth the depth the same way before they compute vertex and normal maps), with its exact backward.
//
// For a valid centre p (0 < d_p < inf) and the window offsets (du, dv) in the order dv = -r..r outer, du = -r..r inner,
// each in-image valid neighbour q gives, in float32,
//     x = -(float(du^2 + dv^2) c_s + (d_q - d_p)^2 c_r),   skipped if x < -17,   w = exp32(x)
//     num += w d_q,  den += w,      out_p = num / den   (the centre has w = 1, so den >= 1);
// an invalid centre passes through unchanged.  c_s = 1/(2 sigma_s^2), c_r = 1/(2 sigma_r^2) are computed in float64 and
// rounded once.  Skipped pairs and invalid neighbours add w = 0 (num + 0 = num, den + 0 = den), so the sums, and the
// numpy statement in tests/bilateral_oracle.py that vectorises the same loop over pixels, are bit-identical.
//
// Backward (gather, no atomics): for a valid q with W_q = den_q
//     g_in[q] = g_out[q] (1 + 2 c_r sum_{s != q} w_qs (d_s - d_q)(d_s - out_q)) / W_q
//             + sum_{p != q valid, kept} g_out[p] (w_pq / W_p) (1 - 2 c_r (d_q - out_p)(d_q - d_p)),
// where w_pq = w_qp bit for bit (the spatial term and (d_q - d_p)^2 are symmetric); an invalid q has g_in = g_out.
//
// One CTA of 32 x 8 threads owns a 32 x 8 output tile: it stages the tile and its r-pixel halo (out-of-image pixels
// read as 0, i.e. invalid) in shared memory together with the (2r+1)^2 spatial terms, then each thread walks its
// window from shared memory.  The radius is a template parameter so the window loop unrolls to immediate offsets.
// Images go over gridDim.z with a stride, so any number of them fits one launch; image offsets are int64.
#include <math.h>

#include <algorithm>

#include "gsx_common.cuh"
#include "gsx_exp32.cuh"
#include "../../include/gsx.h"

namespace gsx {

constexpr int kBfTileX = 32, kBfTileY = 8, kBfThreads = kBfTileX * kBfTileY, kBfMaxRadius = 7;
constexpr int kBfMaxGridZ = 65535;

__device__ __forceinline__ bool depth_valid(float d) { return d > 0.0f && d < INFINITY; }

// the (2R+1)^2 spatial terms, in window order
template <int R>
__device__ __forceinline__ void bilateral_spatial_terms(float *sp, float c_s, int tid) {
  constexpr int D = 2 * R + 1;
  for (int i = tid; i < D * D; i += kBfThreads) {
    const int dv = i / D - R, du = i % D - R;
    sp[i] = (float)(du * du + dv * dv) * c_s;
  }
}

// the tile of image `src` with its R-pixel halo; 0 outside the image
template <int R>
__device__ __forceinline__ void bilateral_stage(float *dst, const float *__restrict__ src, int H, int W, int tid) {
  constexpr int SW = kBfTileX + 2 * R, SH = kBfTileY + 2 * R;
  const int x0 = (int)blockIdx.x * kBfTileX - R, y0 = (int)blockIdx.y * kBfTileY - R;
  for (int i = tid; i < SH * SW; i += kBfThreads) {
    const int y = y0 + i / SW, x = x0 + i % SW;
    dst[i] = (y >= 0 && y < H && x >= 0 && x < W) ? __ldg(src + (int64_t)y * W + x) : 0.0f;
  }
}

template <int R>
__global__ void __launch_bounds__(kBfThreads) k_depth_bilateral(const float *__restrict__ depth, float *__restrict__ out,
                                                                float *__restrict__ den, int64_t n, int H, int W,
                                                                float c_s, float c_r) {
  constexpr int D = 2 * R + 1, SW = kBfTileX + 2 * R, SH = kBfTileY + 2 * R;
  __shared__ float tile[SH * SW];
  __shared__ float sp[D * D];
  const int tid = threadIdx.y * kBfTileX + threadIdx.x;
  bilateral_spatial_terms<R>(sp, c_s, tid);
  const int w = blockIdx.x * kBfTileX + threadIdx.x, h = blockIdx.y * kBfTileY + threadIdx.y;
  const int64_t P = (int64_t)H * W;
  for (int64_t img = blockIdx.z; img < n; img += gridDim.z) {
    __syncthreads();  // the previous image's window reads are done
    bilateral_stage<R>(tile, depth + img * P, H, W, tid);
    __syncthreads();
    if (h >= H || w >= W) continue;
    const float *c = tile + (threadIdx.y + R) * SW + threadIdx.x + R;
    const float d = c[0];
    float o = d, wsum = 0.0f;
    if (depth_valid(d)) {
      float num = 0.0f, dsum = 0.0f;
#pragma unroll
      for (int dv = -R; dv <= R; ++dv)
#pragma unroll
        for (int du = -R; du <= R; ++du) {
          const float q = c[dv * SW + du];
          const bool ok = depth_valid(q);
          const float dl = q - d;
          const float x = -(sp[(dv + R) * D + du + R] + (dl * dl) * c_r);
          const float wt = (ok && x >= kExp32Min) ? exp32(x) : 0.0f;
          num += wt * (ok ? q : 0.0f);
          dsum += wt;
        }
      o = num / dsum;
      wsum = dsum;
    }
    const int64_t i = img * P + (int64_t)h * W + w;
    out[i] = o;
    if (den) den[i] = wsum;
  }
}

template <int R>
__global__ void __launch_bounds__(kBfThreads) k_depth_bilateral_bwd(const float *__restrict__ depth,
                                                                    const float *__restrict__ out,
                                                                    const float *__restrict__ den,
                                                                    const float *__restrict__ g_out,
                                                                    float *__restrict__ g_depth, int64_t n, int H,
                                                                    int W, float c_s, float c_r) {
  constexpr int D = 2 * R + 1, SW = kBfTileX + 2 * R, SH = kBfTileY + 2 * R;
  __shared__ float t_d[SH * SW], t_o[SH * SW], t_w[SH * SW], t_g[SH * SW];
  __shared__ float sp[D * D];
  const int tid = threadIdx.y * kBfTileX + threadIdx.x;
  bilateral_spatial_terms<R>(sp, c_s, tid);
  const int w = blockIdx.x * kBfTileX + threadIdx.x, h = blockIdx.y * kBfTileY + threadIdx.y;
  const int64_t P = (int64_t)H * W;
  const float two_cr = 2.0f * c_r;
  for (int64_t img = blockIdx.z; img < n; img += gridDim.z) {
    __syncthreads();
    bilateral_stage<R>(t_d, depth + img * P, H, W, tid);
    bilateral_stage<R>(t_o, out + img * P, H, W, tid);
    bilateral_stage<R>(t_w, den + img * P, H, W, tid);
    bilateral_stage<R>(t_g, g_out + img * P, H, W, tid);
    __syncthreads();
    if (h >= H || w >= W) continue;
    const int ci = (threadIdx.y + R) * SW + threadIdx.x + R;
    const float dq = t_d[ci], gq = t_g[ci];
    float g = gq;
    if (depth_valid(dq)) {
      const float oq = t_o[ci];
      float self = 0.0f, cross = 0.0f;
#pragma unroll
      for (int dv = -R; dv <= R; ++dv)
#pragma unroll
        for (int du = -R; du <= R; ++du) {
          if (du == 0 && dv == 0) continue;
          const int si = ci + dv * SW + du;
          const float ds = t_d[si];
          const bool ok = depth_valid(ds);
          const float dl = ds - dq;
          const float x = -(sp[(dv + R) * D + du + R] + (dl * dl) * c_r);
          const bool keep = ok && x >= kExp32Min;
          const float wt = keep ? exp32(x) : 0.0f;
          // q in s's window: s is a valid centre (ok) whose pair with q is kept exactly when q's pair with s is
          const float os = t_o[si];
          self += keep ? wt * (dl * (ds - oq)) : 0.0f;
          cross += keep ? (t_g[si] * (wt / t_w[si])) * (1.0f - two_cr * ((dq - os) * (dq - ds))) : 0.0f;
        }
      g = (gq * (1.0f + two_cr * self)) / t_w[ci] + cross;
    }
    g_depth[img * P + (int64_t)h * W + w] = g;
  }
}

// extents, radius and sigmas -> c_s, c_r (refused before any launch)
static int bilateral_args(const char *fn, int64_t n, int H, int W, int radius, double sigma_space, double sigma_range,
                          float *c_s, float *c_r) {
  GSX_CHECK_ARG(n >= 0 && H >= 1 && W >= 1, "%s: bad extents (n_images %lld, H %d, W %d)", fn, (long long)n, H, W);
  GSX_CHECK_ARG((H + kBfTileY - 1) / kBfTileY <= 65535, "%s: H %d exceeds %d rows", fn, H, 65535 * kBfTileY);
  GSX_CHECK_ARG(radius >= 1 && radius <= kBfMaxRadius, "%s: radius must be in 1..%d, not %d", fn, kBfMaxRadius, radius);
  GSX_CHECK_ARG(isfinite(sigma_space) && sigma_space > 0.0 && isfinite(sigma_range) && sigma_range > 0.0,
                "%s: sigma_space and sigma_range must be finite and > 0 (got %g, %g)", fn, sigma_space, sigma_range);
  *c_s = (float)(1.0 / (2.0 * sigma_space * sigma_space));
  *c_r = (float)(1.0 / (2.0 * sigma_range * sigma_range));
  GSX_CHECK_ARG(isfinite(*c_s) && *c_s > 0.0f && isfinite(*c_r) && *c_r > 0.0f,
                "%s: 1/(2 sigma^2) must be a finite positive float32 (sigma_space %g, sigma_range %g)", fn, sigma_space,
                sigma_range);
  return 0;
}

// do the n-image buffers a and b share a byte?
static bool overlaps(const void *a, const void *b, int64_t bytes) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return a && b && x < y + (uintptr_t)bytes && y < x + (uintptr_t)bytes;
}

static dim3 bilateral_grid(int64_t n, int H, int W) {
  return dim3((unsigned)((W + kBfTileX - 1) / kBfTileX), (unsigned)((H + kBfTileY - 1) / kBfTileY),
              (unsigned)std::min<int64_t>(n, kBfMaxGridZ));
}

}  // namespace gsx

#define GSX_BF_DISPATCH(radius, LAUNCH) \
  switch (radius) {                     \
    case 1: LAUNCH(1); break;           \
    case 2: LAUNCH(2); break;           \
    case 3: LAUNCH(3); break;           \
    case 4: LAUNCH(4); break;           \
    case 5: LAUNCH(5); break;           \
    case 6: LAUNCH(6); break;           \
    default: LAUNCH(7); break;          \
  }

extern "C" int gsx_depth_bilateral(const float *depth, float *out, float *den, int64_t n_images, int H, int W,
                                   int radius, double sigma_space, double sigma_range, void *stream) {
  float c_s, c_r;
  if (int rc = gsx::bilateral_args("gsx_depth_bilateral", n_images, H, W, radius, sigma_space, sigma_range, &c_s, &c_r))
    return rc;
  GSX_CHECK_ARG(depth && out, "gsx_depth_bilateral: null pointer");
  const int64_t bytes = n_images * H * W * (int64_t)sizeof(float);
  GSX_CHECK_ARG(!gsx::overlaps(depth, out, bytes) && !gsx::overlaps(depth, den, bytes) && !gsx::overlaps(out, den, bytes),
                "gsx_depth_bilateral: out and den must not overlap depth or each other (the filter reads neighbours)");
  if (n_images == 0) return 0;
  const dim3 grid = gsx::bilateral_grid(n_images, H, W), block(gsx::kBfTileX, gsx::kBfTileY);
#define GSX_BF_FWD(R) \
  gsx::k_depth_bilateral<R><<<grid, block, 0, (cudaStream_t)stream>>>(depth, out, den, n_images, H, W, c_s, c_r)
  GSX_BF_DISPATCH(radius, GSX_BF_FWD)
#undef GSX_BF_FWD
  GSX_CHECK_LAUNCH("gsx_depth_bilateral");
  return 0;
}

extern "C" int gsx_depth_bilateral_bwd(const float *depth, const float *out, const float *den, const float *g_out,
                                       float *g_depth, int64_t n_images, int H, int W, int radius, double sigma_space,
                                       double sigma_range, void *stream) {
  float c_s, c_r;
  if (int rc = gsx::bilateral_args("gsx_depth_bilateral_bwd", n_images, H, W, radius, sigma_space, sigma_range, &c_s,
                                   &c_r))
    return rc;
  GSX_CHECK_ARG(depth && out && den && g_out && g_depth, "gsx_depth_bilateral_bwd: null pointer");
  const int64_t bytes = n_images * H * W * (int64_t)sizeof(float);
  GSX_CHECK_ARG(!gsx::overlaps(g_depth, depth, bytes) && !gsx::overlaps(g_depth, out, bytes) &&
                    !gsx::overlaps(g_depth, den, bytes) && !gsx::overlaps(g_depth, g_out, bytes),
                "gsx_depth_bilateral_bwd: g_depth must not overlap an input (the backward reads neighbours)");
  if (n_images == 0) return 0;
  const dim3 grid = gsx::bilateral_grid(n_images, H, W), block(gsx::kBfTileX, gsx::kBfTileY);
#define GSX_BF_BWD(R)                                                                                             \
  gsx::k_depth_bilateral_bwd<R><<<grid, block, 0, (cudaStream_t)stream>>>(depth, out, den, g_out, g_depth, n_images, \
                                                                          H, W, c_s, c_r)
  GSX_BF_DISPATCH(radius, GSX_BF_BWD)
#undef GSX_BF_BWD
  GSX_CHECK_LAUNCH("gsx_depth_bilateral_bwd");
  return 0;
}
