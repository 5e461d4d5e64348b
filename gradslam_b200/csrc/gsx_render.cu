// Rendering of a surfel map into per-view images (an extension: the reference has no counterpart).  A map row covers the
// one pixel it projects to, with the projection of the fusion step's association (find_active_map_points,
// gradslam/slam/fusionutils.py:249-274, gsx_common.cuh project()); each pixel keeps the covering row with the smallest
// camera-frame z, ties to the smallest row index.
//   k_render_zbuffer     (R1)  per map row, grid-stride: one 128-bit position load, projection into every view of the
//                              element (cameras staged in shared memory), one 64-bit atomicMin of (bits(z) << 32 | n)
//                              into the pixel's slot of the int64 index image, which the entry point filled with ones.
//   k_render_resolve     (R2)  per pixel: key -> n or -1 in place; depth from the key, gathers of the winning row only for
//                              the outputs requested.
//   k_render_resolve_world (R2w) per pixel of one view per element: key -> n or -1 in place, the winning row's
//                              world-frame point and normal (two 128-bit row loads), zeros where uncovered: the target
//                              images of the projective ICP (gsx_icp.cu, render_icp_targets).
//   k_render_bwd_rows    (R3)  per map row: re-projects the row into every view; where it won the pixel, accumulates the
//                              pixel's upstream gradients in view order (a row wins at most one pixel per view: no atomics).
//   k_render_bwd_pose    (R3)  per pixel tile: d/d(camera-to-world pose) of depth and normals, reduced per tile, then
//                              summed in tile order by k_pose_grad_reduce (gsx_frame.cu).
// Positive floats order like their bit patterns, so the 64-bit key orders like (z, n).
#include "gsx_common.cuh"
#include "../../include/gsx.h"

namespace gsx {

// defined in gsx_frame.cu: partials (img, tile, 12) summed in tile order -> (img, 4, 4), bottom row zero
__global__ void k_pose_grad_reduce(const float *partials, int tiles, float *g_poses, int n_img);

constexpr int kRB = 256;        // threads per CTA of every render kernel
constexpr int kViews = 32;      // cameras staged per CTA (blockIdx.z chunks beyond)
constexpr int kRenderCtasPerSM = 8;
constexpr unsigned long long kEmptyKey = ~0ull;

struct RenderArgs {
  const float *geo;     // (B,cap,8)
  const float *col;     // (B,cap,4) or null
  const int32_t *counts;
  int64_t cap;
  const float *K;
  int64_t K_bstride;
  const float *poses;   // camera-to-world, (B,L,4,4) with element stride pose_bstride
  int64_t pose_bstride;
  int L;
  ImageBounds ib;
  unsigned long long *key;  // (B,L,H,W) the int64 index image
  float *depth, *rgb, *normals, *confidence;  // any may be null
};

// Cameras of views [l0, l0 + nv) of element b (world -> camera and K); the caller synchronises.
__device__ __forceinline__ void load_view_cameras(LiveCamera *s_cam, const float *poses, int64_t pose_bstride,
                                                  const float *K, int64_t K_bstride, int b, int l0, int nv) {
  for (int v = threadIdx.x; v < nv; v += blockDim.x)
    s_cam[v].tinv = rigid_inverse(load_rigid(poses + b * pose_bstride + (int64_t)(l0 + v) * 16));
  for (int i = threadIdx.x; i < nv * 12; i += blockDim.x) s_cam[i / 12].k[i % 12] = __ldg(K + b * K_bstride + i % 12);
}

__global__ void __launch_bounds__(kRB) k_render_zbuffer(RenderArgs a) {
  __shared__ LiveCamera s_cam[kViews];
  const int b = blockIdx.y, l0 = blockIdx.z * kViews;
  const int nv = min(kViews, a.L - l0);
  const int count = a.counts[b];
  if ((int64_t)blockIdx.x * kRB >= count) return;
  load_view_cameras(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b, l0, nv);
  __syncthreads();
  const int64_t P = (int64_t)a.ib.H * a.ib.W;
  const float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
  unsigned long long *key = a.key + ((int64_t)b * a.L + l0) * P;
  const int64_t stride = (int64_t)gridDim.x * kRB;
  for (int64_t n = (int64_t)blockIdx.x * kRB + threadIdx.x; n < count; n += stride) {
    const float4 p = __ldg(reinterpret_cast<const float4 *>(geo + n * kGeoW));
    for (int v = 0; v < nv; ++v) {
      const PixelHit hit = project(s_cam[v], a.ib, p.x, p.y, p.z);
      if (hit.in_frustum) {
        const float z = rigid_apply(s_cam[v].tinv, p.x, p.y, p.z).z;  // project()'s camera-frame z, > 0 here
        atomicMin(key + v * P + hit.h * a.ib.W + hit.w,
                  ((unsigned long long)__float_as_uint(z) << 32) | (unsigned long long)n);
      }
    }
  }
}

__device__ __forceinline__ void st3(float *p, float x, float y, float z) {
  p[0] = x; p[1] = y; p[2] = z;
}

__global__ void __launch_bounds__(kRB) k_render_resolve(RenderArgs a) {
  __shared__ Rigid s_tinv;
  const int img = blockIdx.y;
  const int b = img / a.L, l = img - b * a.L;
  if (a.normals && threadIdx.x == 0) s_tinv = rigid_inverse(load_rigid(a.poses + b * a.pose_bstride + (int64_t)l * 16));
  __syncthreads();
  const int64_t P = (int64_t)a.ib.H * a.ib.W;
  const int64_t pix = (int64_t)blockIdx.x * kRB + threadIdx.x;
  if (pix >= P) return;
  const int64_t i = img * P + pix;
  const unsigned long long k = a.key[i];
  const bool covered = k != kEmptyKey;
  const int64_t n = covered ? (int64_t)(k & 0xffffffffull) : -1;
  reinterpret_cast<int64_t *>(a.key)[i] = n;
  if (a.depth) a.depth[i] = covered ? __uint_as_float((unsigned int)(k >> 32)) : 0.0f;
  const float *row = a.geo + ((int64_t)b * a.cap + (covered ? n : 0)) * kGeoW;
  if (a.normals || a.confidence) {
    float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
    if (covered) {
      if (a.normals) g0 = __ldg(reinterpret_cast<const float4 *>(row));
      g1 = __ldg(reinterpret_cast<const float4 *>(row + 4));
    }
    if (a.normals) {
      const float3 nc = covered ? rotate(s_tinv, g0.w, g1.x, g1.y) : make_float3(0.f, 0.f, 0.f);  // R^T n
      st3(a.normals + i * 3, nc.x, nc.y, nc.z);
    }
    if (a.confidence) a.confidence[i] = g1.z;
  }
  if (a.rgb) {
    float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
    if (covered) c = __ldg(reinterpret_cast<const float4 *>(a.col + ((int64_t)b * a.cap + n) * kColW));
    st3(a.rgb + i * 3, c.x, c.y, c.z);
  }
}

__global__ void __launch_bounds__(kRB) k_render_resolve_world(unsigned long long *key, const float *geo, int64_t cap,
                                                           int64_t P, float *tgt_p, float *tgt_n) {
  const int b = blockIdx.y;
  const int64_t pix = (int64_t)blockIdx.x * kRB + threadIdx.x;
  if (pix >= P) return;
  const int64_t i = b * P + pix;
  const unsigned long long k = key[i];
  const bool covered = k != kEmptyKey;
  const int64_t n = covered ? (int64_t)(k & 0xffffffffull) : -1;
  reinterpret_cast<int64_t *>(key)[i] = n;
  float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
  if (covered) {
    const float *row = geo + ((int64_t)b * cap + n) * kGeoW;
    g0 = __ldg(reinterpret_cast<const float4 *>(row));
    g1 = __ldg(reinterpret_cast<const float4 *>(row + 4));
  }
  st3(tgt_p + i * 3, g0.x, g0.y, g0.z);
  st3(tgt_n + i * 3, g0.w, g1.x, g1.y);
}

// ---- backward -----------------------------------------------------------------------------------------------
struct RenderBwdArgs {
  const float *geo;
  const int32_t *counts;
  int64_t cap;
  const float *K;
  int64_t K_bstride;
  const float *poses;
  int64_t pose_bstride;
  const int64_t *index;  // (B,L,H,W): n or -1
  int L;
  ImageBounds ib;
  const float *g_depth, *g_rgb, *g_normals, *g_confidence;  // any may be null (zero)
  float *d_geo, *d_col;  // (B,cap,8) / (B,cap,4), or null
  float *pose_partials;  // (B*L, tiles, 12), or null
  int tiles;
};

__global__ void __launch_bounds__(kRB) k_render_bwd_rows(RenderBwdArgs a) {
  __shared__ LiveCamera s_cam[kViews];
  const int b = blockIdx.y;
  const int64_t n = (int64_t)blockIdx.x * kRB + threadIdx.x;
  const bool live = n < a.counts[b];
  const int64_t P = (int64_t)a.ib.H * a.ib.W;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
  if (live) p = __ldg(reinterpret_cast<const float4 *>(a.geo + ((int64_t)b * a.cap + n) * kGeoW));
  float dp[3] = {0.f, 0.f, 0.f}, dn[3] = {0.f, 0.f, 0.f}, dc[3] = {0.f, 0.f, 0.f}, dcc = 0.f;
  for (int l0 = 0; l0 < a.L; l0 += kViews) {
    const int nv = min(kViews, a.L - l0);
    __syncthreads();  // the previous chunk's cameras are no longer read
    load_view_cameras(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b, l0, nv);
    __syncthreads();
    if (!live) continue;
    for (int v = 0; v < nv; ++v) {
      const PixelHit hit = project(s_cam[v], a.ib, p.x, p.y, p.z);
      if (!hit.in_frustum) continue;
      const int64_t i = ((int64_t)b * a.L + l0 + v) * P + hit.h * a.ib.W + hit.w;
      if (__ldg(a.index + i) != n) continue;
      const float *r = s_cam[v].tinv.r;  // R^T of the camera-to-world pose
      if (a.g_depth) {  // depth = (R^T (p - t))_z: d/dp = R (0, 0, g)
        const float g = __ldg(a.g_depth + i);
        dp[0] += r[6] * g; dp[1] += r[7] * g; dp[2] += r[8] * g;
      }
      if (a.g_normals) {  // normal = R^T n: d/dn = R g
        const float gx = __ldg(a.g_normals + i * 3), gy = __ldg(a.g_normals + i * 3 + 1),
                    gz = __ldg(a.g_normals + i * 3 + 2);
#pragma unroll
        for (int j = 0; j < 3; ++j) dn[j] += dot3(r[j], r[3 + j], r[6 + j], gx, gy, gz);
      }
      if (a.g_rgb) {
        dc[0] += __ldg(a.g_rgb + i * 3); dc[1] += __ldg(a.g_rgb + i * 3 + 1); dc[2] += __ldg(a.g_rgb + i * 3 + 2);
      }
      if (a.g_confidence) dcc += __ldg(a.g_confidence + i);
    }
  }
  if (n >= a.cap) return;
  const int64_t row = (int64_t)b * a.cap + n;
  if (a.d_geo) {
    float4 *o = reinterpret_cast<float4 *>(a.d_geo + row * kGeoW);
    o[0] = make_float4(dp[0], dp[1], dp[2], dn[0]);
    o[1] = make_float4(dn[1], dn[2], dcc, 0.f);
  }
  if (a.d_col) reinterpret_cast<float4 *>(a.d_col + row * kColW)[0] = make_float4(dc[0], dc[1], dc[2], 0.f);
}

// Per pixel of view (b,l), with q = R^T (p - t) and normal = R^T n of the winning row:
//   dL/dR = (p - t) g_q^T + n g_n^T,  dL/dt = -R g_q,  g_q = (0, 0, g_depth)
// reduced over the tile's pixels (warp shuffles, then the warps in order).
__global__ void __launch_bounds__(kRB) k_render_bwd_pose(RenderBwdArgs a) {
  __shared__ Rigid s_pose;
  __shared__ float s_red[kRB / 32][12];
  const int img = blockIdx.y;
  const int b = img / a.L, l = img - b * a.L;
  if (threadIdx.x == 0) s_pose = load_rigid(a.poses + b * a.pose_bstride + (int64_t)l * 16);
  __syncthreads();
  const int64_t P = (int64_t)a.ib.H * a.ib.W;
  const int64_t pix = (int64_t)blockIdx.x * kRB + threadIdx.x;
  float acc[12];
#pragma unroll
  for (int j = 0; j < 12; ++j) acc[j] = 0.0f;
  const int64_t i = img * P + pix;
  const int64_t n = pix < P ? __ldg(a.index + i) : -1;
  if (n >= 0) {
    const float *row = a.geo + ((int64_t)b * a.cap + n) * kGeoW;
    const float4 g0 = __ldg(reinterpret_cast<const float4 *>(row));
    const float4 g1 = __ldg(reinterpret_cast<const float4 *>(row + 4));
    const float gd = a.g_depth ? __ldg(a.g_depth + i) : 0.0f;
    float gn[3] = {0.f, 0.f, 0.f};
    if (a.g_normals) {
      gn[0] = __ldg(a.g_normals + i * 3); gn[1] = __ldg(a.g_normals + i * 3 + 1); gn[2] = __ldg(a.g_normals + i * 3 + 2);
    }
    const Rigid &T = s_pose;
    const float pt[3] = {g0.x - T.t[0], g0.y - T.t[1], g0.z - T.t[2]};
    const float nw[3] = {g0.w, g1.x, g1.y};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      acc[r * 4 + 0] = nw[r] * gn[0];
      acc[r * 4 + 1] = nw[r] * gn[1];
      acc[r * 4 + 2] = pt[r] * gd + nw[r] * gn[2];
      acc[r * 4 + 3] = -(T.r[r * 3 + 2] * gd);
    }
  }
#pragma unroll
  for (int j = 0; j < 12; ++j) {
    float x = acc[j];
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
    acc[j] = x;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0)
#pragma unroll
    for (int j = 0; j < 12; ++j) s_red[warp][j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 12) {
    float x = 0.0f;
    for (int w = 0; w < kRB / 32; ++w) x += s_red[w][threadIdx.x];
    a.pose_partials[((int64_t)img * a.tiles + blockIdx.x) * 12 + threadIdx.x] = x;
  }
}

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace gsx

using namespace gsx;

// Shared checks of both entry points: sizes, the launch grids' limits and the 32-bit row index of the z-buffer key.
static int check_render_extents(const char *fn, int B, int L, int H, int W, int64_t capacity) {
  GSX_CHECK_ARG(B >= 1 && L >= 1 && H >= 1 && W >= 1, "%s: bad extents B=%d L=%d H=%d W=%d", fn, B, L, H, W);
  GSX_CHECK_ARG((int64_t)L * H * W <= INT32_MAX, "%s: L*H*W = %lld overflows", fn, (long long)L * H * W);
  GSX_CHECK_ARG((int64_t)B * L <= 65535 && B <= 65535, "%s: B*L = %lld views exceed one launch", fn, (long long)B * L);
  GSX_CHECK_ARG(capacity >= 0 && capacity <= INT32_MAX, "%s: bad capacity %lld", fn, (long long)capacity);
  return 0;
}

static inline unsigned pixel_tiles(int H, int W) { return (unsigned)(((int64_t)H * W + kRB - 1) / kRB); }

// Fills the index image with empty keys, then runs R1 over the rows of every element (max_count = host bound on the
// element sizes; no row pass when it is 0).
static void launch_zbuffer(const RenderArgs &a, int B, int64_t max_count, cudaStream_t s) {
  cudaMemsetAsync(a.key, 0xFF, (size_t)B * a.L * a.ib.H * a.ib.W * sizeof(int64_t), s);
  if (max_count > 0) {
    const unsigned chunks = (unsigned)((a.L + kViews - 1) / kViews);
    int64_t bx = (max_count + kRB - 1) / kRB;
    const int64_t cap_blocks = (int64_t)kNumSMs * kRenderCtasPerSM;  // grid-stride beyond
    if (bx * B * chunks > cap_blocks) bx = (cap_blocks + B * chunks - 1) / (B * chunks);
    k_render_zbuffer<<<dim3((unsigned)bx, (unsigned)B, chunks), kRB, 0, s>>>(a);
  }
}

extern "C" int gsx_render_views(const float *map_geometry, const float *map_colors, const int32_t *counts,
                                int64_t capacity, int64_t max_count, const float *intrinsics, int64_t K_bstride,
                                const float *poses, int64_t pose_bstride, int B, int L, int H, int W, int64_t *index,
                                float *depth, float *rgb, float *normals, float *confidence, void *stream) {
  if (check_render_extents("gsx_render_views", B, L, H, W, capacity)) return 1;
  GSX_CHECK_ARG(intrinsics && poses && index, "gsx_render_views: null pointer");
  GSX_CHECK_ARG(max_count >= 0 && max_count <= capacity, "gsx_render_views: max_count %lld outside [0, capacity %lld]",
                (long long)max_count, (long long)capacity);
  if (max_count > 0) GSX_CHECK_ARG(map_geometry && counts, "gsx_render_views: null map pointer");
  if (max_count > 0 && rgb) GSX_CHECK_ARG(map_colors, "gsx_render_views: rgb requested from a map without colours");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors),
                "gsx_render_views: map rows must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  RenderArgs a{map_geometry, map_colors, counts, capacity, intrinsics, K_bstride, poses, pose_bstride, L,
               image_bounds(H, W), reinterpret_cast<unsigned long long *>(index), depth, rgb, normals, confidence};
  launch_zbuffer(a, B, max_count, s);
  k_render_resolve<<<dim3(pixel_tiles(H, W), (unsigned)(B * L)), kRB, 0, s>>>(a);
  GSX_CHECK_LAUNCH("gsx_render_views");
  return 0;
}

namespace gsx {
// Target images of the projective ICP (declared in gsx_icp.cu): one view per element from `poses`, resolved to the
// index image (B, H*W) and the winning rows' world-frame points and normals (B, H*W, 3).  Same checks as
// gsx_render_views; returns non-zero (error set) if they fail.
int render_icp_targets(const float *map_geometry, const int32_t *counts, int64_t capacity, int64_t max_count,
                       const float *intrinsics, int64_t K_bstride, const float *poses, int64_t pose_bstride, int B,
                       int H, int W, int64_t *index, float *tgt_p, float *tgt_n, cudaStream_t s) {
  if (check_render_extents("render_icp_targets", B, 1, H, W, capacity)) return 1;
  GSX_CHECK_ARG(max_count >= 0 && max_count <= capacity, "render_icp_targets: max_count %lld outside [0, capacity %lld]",
                (long long)max_count, (long long)capacity);
  GSX_CHECK_ARG(aligned16(map_geometry), "render_icp_targets: map rows must be 16-byte aligned");
  RenderArgs a{map_geometry, nullptr, counts, capacity, intrinsics, K_bstride, poses, pose_bstride, 1,
               image_bounds(H, W), reinterpret_cast<unsigned long long *>(index), nullptr, nullptr, nullptr, nullptr};
  launch_zbuffer(a, B, max_count, s);
  k_render_resolve_world<<<dim3(pixel_tiles(H, W), (unsigned)B), kRB, 0, s>>>(a.key, map_geometry, capacity,
                                                                             (int64_t)H * W, tgt_p, tgt_n);
  GSX_CHECK_LAUNCH("render_icp_targets");
  return 0;
}
}  // namespace gsx

extern "C" int64_t gsx_render_views_bwd_scratch_bytes(int B, int L, int H, int W) {
  if (B < 1 || L < 1 || H < 1 || W < 1) return -1;
  return (int64_t)B * L * pixel_tiles(H, W) * 12 * 4 + 256;
}

extern "C" int gsx_render_views_bwd(const float *map_geometry, const int32_t *counts, int64_t capacity,
                                    const float *intrinsics, int64_t K_bstride, const float *poses,
                                    int64_t pose_bstride, const int64_t *index, int B, int L, int H, int W,
                                    const float *g_depth, const float *g_rgb, const float *g_normals,
                                    const float *g_confidence, float *d_geometry, float *d_colors, float *d_poses,
                                    void *scratch, int64_t scratch_bytes, void *stream) {
  if (check_render_extents("gsx_render_views_bwd", B, L, H, W, capacity)) return 1;
  GSX_CHECK_ARG(intrinsics && poses && index, "gsx_render_views_bwd: null pointer");
  const bool want_rows = (d_geometry || d_colors) && capacity > 0;
  if (capacity > 0 && (want_rows || d_poses))
    GSX_CHECK_ARG(map_geometry && counts, "gsx_render_views_bwd: null map pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(d_geometry) && aligned16(d_colors),
                "gsx_render_views_bwd: map rows must be 16-byte aligned");
  if (d_poses)
    GSX_CHECK_ARG(scratch && scratch_bytes >= gsx_render_views_bwd_scratch_bytes(B, L, H, W),
                  "gsx_render_views_bwd: scratch too small");
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned tiles = pixel_tiles(H, W);
  RenderBwdArgs a{map_geometry, counts, capacity, intrinsics, K_bstride, poses, pose_bstride, index, L,
                  image_bounds(H, W), g_depth, g_rgb, g_normals, g_confidence, d_geometry, d_colors,
                  (float *)scratch, (int)tiles};
  if (want_rows)
    k_render_bwd_rows<<<dim3((unsigned)((capacity + kRB - 1) / kRB), (unsigned)B), kRB, 0, s>>>(a);
  if (d_poses) {
    k_render_bwd_pose<<<dim3(tiles, (unsigned)(B * L)), kRB, 0, s>>>(a);
    k_pose_grad_reduce<<<B * L, 16, 0, s>>>((const float *)scratch, (int)tiles, d_poses, B * L);
  }
  GSX_CHECK_LAUNCH("gsx_render_views_bwd");
  return 0;
}
