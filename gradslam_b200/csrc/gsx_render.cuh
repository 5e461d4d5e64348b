// Device helpers shared by the renderers (gsx_render.cu: R1 .. R3d, gsx_render_blend.cu: the blended splats): the
// per-CTA view cameras, and the oriented disk of a row in one camera with its ray test.
#pragma once
#include "gsx_common.cuh"

namespace gsx {

constexpr int kRB = 256;    // threads per CTA of every render kernel
constexpr int kViews = 32;  // cameras staged per CTA (blockIdx.z chunks beyond)

// Cameras of views [l0, l0 + nv) of element b (world -> camera and K); the caller synchronises.
__device__ __forceinline__ void load_view_cameras(LiveCamera *s_cam, const float *poses, int64_t pose_bstride,
                                                  const float *K, int64_t K_bstride, int b, int l0, int nv) {
  for (int v = threadIdx.x; v < nv; v += blockDim.x)
    s_cam[v].tinv = rigid_inverse(load_rigid(poses + b * pose_bstride + (int64_t)(l0 + v) * 16));
  for (int i = threadIdx.x; i < nv * 12; i += blockDim.x) s_cam[i / 12].k[i % 12] = __ldg(K + b * K_bstride + i % 12);
}

// A row is a disk when it has a radius and a normal; everything else renders as one pixel.
__device__ __forceinline__ bool is_disk(const float4 &g0, const float4 &g1) {
  return g1.w > 0.0f && (g0.w != 0.0f || g1.x != 0.0f || g1.y != 0.0f);
}

// The disk of a row in one camera: q = T^-1 p, m = R^T n, mq = m.q, rr = r^2, the projected centre (cu, cv) = rint of
// project()'s u, v, and the box of pixels around it (+-M pixels, clipped to the image).
struct Disk {
  float3 q, m;
  float mq, rr;
  int cu, cv;
  int h0, h1, w0, w1;
};
__device__ __forceinline__ Disk make_disk(const LiveCamera &c, const ImageBounds &ib, int M, const float4 &g0,
                                          const float4 &g1) {
  Disk d;
  d.q = rigid_apply(c.tinv, g0.x, g0.y, g0.z);
  d.m = rotate(c.tinv, g0.w, g1.x, g1.y);
  d.mq = dot3(d.m.x, d.m.y, d.m.z, d.q.x, d.q.y, d.q.z);
  d.rr = g1.w * g1.w;
  const float hx = ((c.k[0] * d.q.x + c.k[1] * d.q.y) + c.k[2] * d.q.z) + c.k[3];
  const float hy = ((c.k[4] * d.q.x + c.k[5] * d.q.y) + c.k[6] * d.q.z) + c.k[7];
  const float hz = ((c.k[8] * d.q.x + c.k[9] * d.q.y) + c.k[10] * d.q.z) + c.k[11];
  const float den = (hz != 0.0f) ? hz : 1.0f;
  // clamped first so that the conversion is defined; a centre past the clamp has an empty box either way
  d.cu = (int)rintf(fminf(fmaxf(hx / den, (float)(-M - 2)), (float)(ib.W + M + 1)));
  d.cv = (int)rintf(fminf(fmaxf(hy / den, (float)(-M - 2)), (float)(ib.H + M + 1)));
  d.w0 = max(d.cu - M, 0);
  d.w1 = min(d.cu + M, ib.W - 1);
  d.h0 = max(d.cv - M, 0);
  d.h1 = min(d.cv + M, ib.H - 1);
  if (!(d.q.z > 0.0f)) d.h1 = d.h0 - 1;  // behind the camera: no pixel
  return d;
}

// Pixel (h,w)'s ray d = K^-1 (w, h, 1) against the disk: true, with the plane depth t and m.d, if it meets the disk.
__device__ __forceinline__ bool disk_hit(const Disk &d, const KInv &k, int h, int w, float &t, float &md, float3 &ray) {
  ray = make_float3(k.k00 * (float)w + k.k02, k.k11 * (float)h + k.k12, 1.0f);
  md = dot3(d.m.x, d.m.y, d.m.z, ray.x, ray.y, ray.z);
  if (md == 0.0f) return false;
  t = d.mq / md;
  if (!(t > 0.0f)) return false;
  const float ex = t * ray.x - d.q.x, ey = t * ray.y - d.q.y, ez = t * ray.z - d.q.z;
  return ((ex * ex + ey * ey) + ez * ez) <= d.rr;
}

}  // namespace gsx
