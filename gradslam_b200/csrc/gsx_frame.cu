// K1: depth -> local/global vertex and normal maps.  One thread per pixel; per-image constants (inverse
// intrinsics, pose) are computed once per CTA into shared memory; outputs are staged through shared memory
// so every map is written with coalesced 16-byte stores.
// Reference op chain: gradslam/structures/rgbdimages.py:643-762 (see include/gsx.h).
#include "gsx_common.cuh"
#include "../../include/gsx.h"

namespace gsx {

constexpr int kTile = 256;  // pixels per CTA; 256*3 floats = 3072 B per map tile (16-byte aligned)

struct FrameArgs {
  const float *depth;
  int64_t depth_bstride;
  const float *K;
  int64_t K_bstride;
  const float *poses;  // may be null
  int64_t pose_bstride;
  int B, L, H, W;
  float *out[4];  // vertex, normal, gvertex, gnormal (any may be null)
};

__global__ void __launch_bounds__(kTile) k_backproject_normals(FrameArgs a) {
  __shared__ __align__(16) float stage[4][kTile * 3];
  __shared__ KInv s_k;
  __shared__ Rigid s_pose;
  const int img = blockIdx.y;  // b*L + l
  const int b = img / a.L, l = img - b * a.L;
  const int P = a.H * a.W;
  if (threadIdx.x == 0) s_k = load_kinv(a.K + b * a.K_bstride);
  if (threadIdx.x == 32 && a.poses) s_pose = load_rigid(a.poses + b * a.pose_bstride + (int64_t)l * 16);
  __syncthreads();
  const KInv k = s_k;
  const int tile0 = blockIdx.x * kTile;
  const int pix = tile0 + threadIdx.x;
  const bool want_local = a.out[0] || a.out[1], want_global = a.out[2] || a.out[3];
  if (pix < P) {
    const float *dimg = a.depth + b * a.depth_bstride + (int64_t)l * P;
    const int h = pix / a.W, w = pix - h * a.W;
    const FrameSample f = frame_sample<true>(dimg, k, a.poses ? &s_pose : nullptr, h, w, a.H, a.W);
    const int t3 = threadIdx.x * 3;
    if (want_local) {
      stage[0][t3] = f.v.x; stage[0][t3 + 1] = f.v.y; stage[0][t3 + 2] = f.v.z;
      stage[1][t3] = f.n.x; stage[1][t3 + 1] = f.n.y; stage[1][t3 + 2] = f.n.z;
    }
    if (want_global) {
      stage[2][t3] = f.gv.x; stage[2][t3 + 1] = f.gv.y; stage[2][t3 + 2] = f.gv.z;
      stage[3][t3] = f.gn.x; stage[3][t3 + 1] = f.gn.y; stage[3][t3 + 2] = f.gn.z;
    }
  }
  // make the generic-proxy shared-memory writes visible to the async (bulk-copy) proxy, then sync the CTA
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const int remaining = P - tile0;
  const int nfloat = (remaining < kTile ? remaining : kTile) * 3;
  const int64_t obase = ((int64_t)img * P + tile0) * 3;
  // every image starts 16-byte aligned only if P*3 floats is a multiple of 4
  const bool vec_ok = (nfloat == kTile * 3) && ((obase & 3) == 0);
  if (vec_ok) {
    // full tile: ONE thread hands each 3072-byte map tile to the bulk-copy engine (cp.async.bulk, shared -> global;
    // SASS: UBLKCP), instead of 192 threads issuing 16-byte stores
    if (threadIdx.x == 0) {
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        float *out = a.out[m];
        if (!out) continue;
        const unsigned int src = (unsigned int)__cvta_generic_to_shared(stage[m]);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(out + obase), "r"(src),
                     "n"(kTile * 3 * 4)
                     : "memory");
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // smem must stay intact until it has been read
    }
  } else {
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      float *out = a.out[m];
      if (!out) continue;
      float *dst = out + obase;
      for (int j = threadIdx.x; j < nfloat; j += kTile) dst[j] = stage[m][j];
    }
  }
}

int launch_backproject(const FrameArgs &a, cudaStream_t stream) {
  const int64_t P = (int64_t)a.H * a.W;
  if ((int64_t)a.B * a.L * P == 0) return 0;
  const int64_t bx = (P + kTile - 1) / kTile;
  k_backproject_normals<<<dim3((unsigned)bx, (unsigned)(a.B * a.L)), kTile, 0, stream>>>(a);
  GSX_CHECK_LAUNCH("gsx_backproject_normals_fwd");
  return 0;
}

}  // namespace gsx

extern "C" int gsx_backproject_normals_fwd(const float *depth, int64_t depth_bstride, const float *intrinsics,
                                           int64_t K_bstride, const float *poses, int64_t pose_bstride, int B,
                                           int L, int H, int W, float *vertex, float *normal, float *gvertex,
                                           float *gnormal, void *stream) {
  GSX_CHECK_ARG(depth && intrinsics, "gsx_backproject_normals_fwd: null depth/intrinsics");
  GSX_CHECK_ARG(B >= 0 && L >= 0 && H >= 2 && W >= 2, "gsx_backproject_normals_fwd: need H,W >= 2 (got %d x %d)", H, W);
  GSX_CHECK_ARG((int64_t)B * L <= 65535 && (int64_t)H * W < (1ll << 30), "gsx_backproject_normals_fwd: extents too large");
  float *outs[4] = {vertex, normal, gvertex, gnormal};
  for (float *o : outs)
    GSX_CHECK_ARG(((uintptr_t)o & 15) == 0, "gsx_backproject_normals_fwd: outputs must be 16-byte aligned");
  gsx::FrameArgs a{depth, depth_bstride, intrinsics, K_bstride, poses, pose_bstride, B, L, H, W,
                   {vertex, normal, gvertex, gnormal}};
  return gsx::launch_backproject(a, (cudaStream_t)stream);
}

// =============================================================================================================
// K1 backward: d(loss)/d(depth) and d(loss)/d(pose) from the upstream gradients of the four maps.
// Autograd counterpart of gradslam/structures/rgbdimages.py:643-762 (the reference gets it from PyTorch's tape).
// Gather formulation, no atomics: every pixel q re-evaluates the normal-branch terms of the (at most five)
// pixels whose finite-difference stencil touches q.  Pose gradients are reduced per CTA and summed in tile
// order by a second kernel (deterministic).  The kWantK instantiation also reduces each pixel's K^-1 partials
// (v = ((k00 u + k02) d, (k11 v + k12) d, d) valid) per CTA; a third kernel sums them over the tiles and the L frames of
// each element in a fixed order and maps them to fx, cx, fy, cy.
// =============================================================================================================
namespace gsx {

struct FrameBwdArgs {
  const float *depth;
  int64_t depth_bstride;
  const float *K;
  int64_t K_bstride;
  const float *poses;
  int64_t pose_bstride;
  int B, L, H, W;
  const float *g[4];  // upstream: vertex, normal, gvertex, gnormal (dense (B,L,H,W,3)), any may be null
  float *g_depth;     // (B,L,H,W)
  float *pose_partials;  // (B*L, tiles, 12) or null
  int tiles;
};

__device__ __forceinline__ float3 ld3(const float *p) { return make_float3(__ldg(p), __ldg(p + 1), __ldg(p + 2)); }
__device__ __forceinline__ float3 cross3(const float3 &a, const float3 &b) {
  return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
// R^T g
__device__ __forceinline__ float3 rot_t(const Rigid &r, const float3 &g) {
  return make_float3(r.r[0] * g.x + r.r[3] * g.y + r.r[6] * g.z, r.r[1] * g.x + r.r[4] * g.y + r.r[7] * g.z,
                     r.r[2] * g.x + r.r[5] * g.y + r.r[8] * g.z);
}

// gradient of the loss w.r.t. the two finite differences dh, dv of pixel p (through its normal)
__device__ __forceinline__ void normal_terms(const FrameBwdArgs &a, const float *dimg, const KInv &k, const Rigid *pose,
                                             const float *gn_img, const float *ggn_img, int h, int w, float3 &g_dh,
                                             float3 &g_dv, float3 *n_out) {
  const int W = a.W, H = a.H;
  const int wa = (w < W - 1) ? w : w - 1;
  const int ha = (h < H - 1) ? h : h - 1;
  const float dc = __ldg(dimg + h * W + w);
  const float vf = dc > 0.0f ? 1.0f : 0.0f;
  const float3 a0 = backproject(k, (float)wa, (float)h, __ldg(dimg + h * W + wa));
  const float3 a1 = backproject(k, (float)(wa + 1), (float)h, __ldg(dimg + h * W + wa + 1));
  const float3 b0 = backproject(k, (float)w, (float)ha, __ldg(dimg + ha * W + w));
  const float3 b1 = backproject(k, (float)w, (float)(ha + 1), __ldg(dimg + (ha + 1) * W + w));
  const float3 dh = make_float3(a1.x - a0.x, a1.y - a0.y, a1.z - a0.z);
  const float3 dv = make_float3(b1.x - b0.x, b1.y - b0.y, b1.z - b0.z);
  const float3 c = cross_ref(dh.x, dh.y, dh.z, dv.x, dv.y, dv.z);  // the forward's values (reference rounding)
  const float nrm = norm_ref(c);
  const float den = (nrm == 0.0f) ? 1.0f : nrm;
  const float3 nh = make_float3(c.x / den, c.y / den, c.z / den);
  if (n_out) *n_out = make_float3(nh.x * vf, nh.y * vf, nh.z * vf);
  // upstream gradient w.r.t. the local normal of p
  float3 G = make_float3(0.f, 0.f, 0.f);
  const int64_t o = ((int64_t)h * W + w) * 3;
  if (gn_img) G = ld3(gn_img + o);
  if (ggn_img) {
    float3 t = ld3(ggn_img + o);
    if (pose) t = rot_t(*pose, t);
    G.x += t.x; G.y += t.y; G.z += t.z;
  }
  // n = (c / |c|) * vf  ->  dL/dc = vf * (G - nh (nh.G)) / |c|   (|c| == 0: den is the constant 1)
  float3 gc;
  if (nrm == 0.0f) {
    gc = make_float3(G.x * vf, G.y * vf, G.z * vf);
  } else {
    const float d = nh.x * G.x + nh.y * G.y + nh.z * G.z;
    const float s = vf / den;
    gc = make_float3((G.x - nh.x * d) * s, (G.y - nh.y * d) * s, (G.z - nh.z * d) * s);
  }
  g_dh = cross3(dv, gc);  // c = dh x dv
  g_dv = cross3(gc, dh);
}

// k_partials: (B*L, tiles, 4) per-CTA sums of dL/d(k00, k02, k11, k12), written only by the kWantK instantiation (a
// separate parameter, so that the instantiation without K compiles to the kernel it was before)
template <bool kWantK>
__global__ void __launch_bounds__(kTile) k_backproject_normals_bwd(FrameBwdArgs a, float *k_partials) {
  __shared__ KInv s_k;
  __shared__ Rigid s_pose;
  __shared__ float s_red[kTile / 32][12];
  const int img = blockIdx.y;
  const int b = img / a.L, l = img - b * a.L;
  const int P = a.H * a.W;
  if (threadIdx.x == 0) s_k = load_kinv(a.K + b * a.K_bstride);
  if (threadIdx.x == 32 && a.poses) s_pose = load_rigid(a.poses + b * a.pose_bstride + (int64_t)l * 16);
  __syncthreads();
  const KInv k = s_k;
  const Rigid *pose = a.poses ? &s_pose : nullptr;
  const int pix = blockIdx.x * kTile + threadIdx.x;
  const float *dimg = a.depth + b * a.depth_bstride + (int64_t)l * P;
  const int64_t ibase = (int64_t)img * P * 3;
  const float *gv_img = a.g[0] ? a.g[0] + ibase : nullptr;
  const float *gn_img = a.g[1] ? a.g[1] + ibase : nullptr;
  const float *ggv_img = a.g[2] ? a.g[2] + ibase : nullptr;
  const float *ggn_img = a.g[3] ? a.g[3] + ibase : nullptr;
  float acc[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) acc[i] = 0.0f;
  float kacc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (pix < P) {
    const int h = pix / a.W, w = pix - h * a.W;
    const int W = a.W, H = a.H;
    const float d = __ldg(dimg + pix);
    const float vf = d > 0.0f ? 1.0f : 0.0f;
    const float3 ray = make_float3(k.k00 * (float)w + k.k02, k.k11 * (float)h + k.k12, 1.0f);
    const float3 v = backproject(k, (float)w, (float)h, d);
    // direct vertex gradient
    float3 GV = make_float3(0.f, 0.f, 0.f);
    const int64_t o = (int64_t)pix * 3;
    if (gv_img) GV = ld3(gv_img + o);
    float3 ggv = make_float3(0.f, 0.f, 0.f);
    if (ggv_img) {
      ggv = ld3(ggv_img + o);
      ggv.x *= vf; ggv.y *= vf; ggv.z *= vf;  // gv = (R v + t) * valid
      const float3 t = pose ? rot_t(*pose, ggv) : ggv;
      GV.x += t.x; GV.y += t.y; GV.z += t.z;
    }
    // normal branch: stencil contributions
    const bool any_n = gn_img || ggn_img;
    float3 n_q = make_float3(0.f, 0.f, 0.f);
    if (any_n) {
      float3 gdh, gdv;
      normal_terms(a, dimg, k, pose, gn_img, ggn_img, h, w, gdh, gdv, &n_q);
      const float sh = (w < W - 1) ? -1.0f : 1.0f;  // q is its own a0 (interior) or a1 (last column)
      const float sv = (h < H - 1) ? -1.0f : 1.0f;
      GV.x += sh * gdh.x + sv * gdv.x; GV.y += sh * gdh.y + sv * gdv.y; GV.z += sh * gdh.z + sv * gdv.z;
      if (w >= 1) {  // left neighbour uses q as a1 (for w-1 < W-1, always true here)
        float3 e, f;
        normal_terms(a, dimg, k, pose, gn_img, ggn_img, h, w - 1, e, f, nullptr);
        GV.x += e.x; GV.y += e.y; GV.z += e.z;
      }
      if (w == W - 2) {  // the last column's difference re-uses (W-2, W-1): q is its a0
        float3 e, f;
        normal_terms(a, dimg, k, pose, gn_img, ggn_img, h, W - 1, e, f, nullptr);
        GV.x -= e.x; GV.y -= e.y; GV.z -= e.z;
      }
      if (h >= 1) {
        float3 e, f;
        normal_terms(a, dimg, k, pose, gn_img, ggn_img, h - 1, w, e, f, nullptr);
        GV.x += f.x; GV.y += f.y; GV.z += f.z;
      }
      if (h == H - 2) {
        float3 e, f;
        normal_terms(a, dimg, k, pose, gn_img, ggn_img, H - 1, w, e, f, nullptr);
        GV.x -= f.x; GV.y -= f.y; GV.z -= f.z;
      }
    }
    a.g_depth[(int64_t)img * P + pix] = vf * (ray.x * GV.x + ray.y * GV.y + ray.z * GV.z);
    if constexpr (kWantK) {
      const float dd = vf * d;
      kacc[0] = (dd * (float)w) * GV.x;
      kacc[1] = dd * GV.x;
      kacc[2] = (dd * (float)h) * GV.y;
      kacc[3] = dd * GV.y;
    }
    if (a.pose_partials && pose) {
      // dL/dR = ggv (x) v + ggn (x) n ;  dL/dt = ggv
      float3 ggn = make_float3(0.f, 0.f, 0.f);
      if (ggn_img) ggn = ld3(ggn_img + o);
      const float gg[3] = {ggv.x, ggv.y, ggv.z}, gn3[3] = {ggn.x, ggn.y, ggn.z};
      const float vv[3] = {v.x, v.y, v.z}, nn[3] = {n_q.x, n_q.y, n_q.z};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) acc[i * 4 + j] = gg[i] * vv[j] + gn3[i] * nn[j];
        acc[i * 4 + 3] = gg[i];
      }
    }
  }
  if (a.pose_partials) {
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      float x = acc[i];
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
      acc[i] = x;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0)
#pragma unroll
      for (int i = 0; i < 12; ++i) s_red[warp][i] = acc[i];
    __syncthreads();
    if (threadIdx.x < 12) {
      float x = 0.0f;
      for (int wv = 0; wv < kTile / 32; ++wv) x += s_red[wv][threadIdx.x];
      a.pose_partials[((int64_t)img * a.tiles + blockIdx.x) * 12 + threadIdx.x] = x;
    }
  }
  if constexpr (kWantK) {
    __shared__ float s_kred[kTile / 32][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float x = kacc[i];
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
      kacc[i] = x;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0)
#pragma unroll
      for (int i = 0; i < 4; ++i) s_kred[warp][i] = kacc[i];
    __syncthreads();
    if (threadIdx.x < 4) {
      float x = 0.0f;
      for (int wv = 0; wv < kTile / 32; ++wv) x += s_kred[wv][threadIdx.x];
      k_partials[((int64_t)img * a.tiles + blockIdx.x) * 4 + threadIdx.x] = x;
    }
  }
}

__global__ void k_pose_grad_reduce(const float *partials, int tiles, float *g_poses, int n_img) {
  const int img = blockIdx.x;
  const int i = threadIdx.x;  // 0..15
  if (img >= n_img || i >= 16) return;
  float x = 0.0f;
  if (i < 12)
    for (int t = 0; t < tiles; ++t) x += partials[((int64_t)img * tiles + t) * 12 + i];
  g_poses[(int64_t)img * 16 + i] = x;  // bottom row gets zeros
}

// g_K (B,4,4) of element b from its L frames' per-CTA K^-1 partials, mapped through kinv_chain; every entry load_kinv
// does not read gets 0.  128 threads: warp e sums K^-1 entry e, lane j the tiles j, j+32, ... of frame 0, then of frame
// 1, ..., and the lanes are combined by a fixed butterfly, so the order of every sum is fixed.
__global__ void __launch_bounds__(128) k_intrinsics_grad_reduce(const float *k_partials, int L, int tiles,
                                                                const float *K, int64_t K_bstride, float *g_K) {
  __shared__ float s_g[4];
  const int b = blockIdx.x, lane = threadIdx.x & 31, e = threadIdx.x >> 5;
  float x = 0.0f;
  for (int l = 0; l < L; ++l)
    for (int t = lane; t < tiles; t += 32) x += k_partials[(((int64_t)b * L + l) * tiles + t) * 4 + e];
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
  if (lane == 0) s_g[e] = x;
  __syncthreads();
  if (threadIdx.x < 16) {
    const int i = threadIdx.x;
    const KGrad g = kinv_chain(K + b * K_bstride, KInv{s_g[0], s_g[1], s_g[2], s_g[3]});
    g_K[(int64_t)b * 16 + i] = i == 0 ? g.fx : i == 2 ? g.cx : i == 5 ? g.fy : i == 6 ? g.cy : 0.0f;
  }
}

// scratch of the backward: the pose partials (B*L, tiles, 12), then the K^-1 partials (B*L, tiles, 4)
struct FrameBwdScratch {
  float *pose, *kinv;
  int64_t bytes;
};
inline FrameBwdScratch frame_bwd_scratch(void *base, int B, int L, int64_t tiles) {
  Carver c(base);
  FrameBwdScratch s;
  s.pose = c.take<float>((int64_t)B * L * tiles * 12);
  s.kinv = c.take<float>((int64_t)B * L * tiles * 4);
  s.bytes = c.bytes;
  return s;
}

}  // namespace gsx

extern "C" int64_t gsx_backproject_normals_bwd_scratch_bytes(int B, int L, int H, int W) {
  if (B < 0 || L < 0 || H < 2 || W < 2) return -1;
  const int64_t tiles = ((int64_t)H * W + gsx::kTile - 1) / gsx::kTile;
  return (int64_t)B * L * tiles * 12 * 4 + 256;
}

extern "C" int64_t gsx_backproject_normals_bwd_intrinsics_scratch_bytes(int B, int L, int H, int W) {
  if (B < 0 || L < 0 || H < 2 || W < 2) return -1;
  const int64_t tiles = ((int64_t)H * W + gsx::kTile - 1) / gsx::kTile;
  return gsx::frame_bwd_scratch(nullptr, B, L, tiles).bytes;
}

extern "C" int gsx_backproject_normals_bwd_intrinsics(const float *depth, int64_t depth_bstride,
                                                      const float *intrinsics, int64_t K_bstride, const float *poses,
                                                      int64_t pose_bstride, int B, int L, int H, int W,
                                                      const float *g_vertex, const float *g_normal,
                                                      const float *g_gvertex, const float *g_gnormal, float *g_depth,
                                                      float *g_poses, float *g_intrinsics, void *scratch,
                                                      int64_t scratch_bytes, void *stream) {
  GSX_CHECK_ARG(depth && intrinsics && g_depth, "gsx_backproject_normals_bwd: null pointer");
  GSX_CHECK_ARG(B >= 0 && L >= 0 && H >= 2 && W >= 2, "gsx_backproject_normals_bwd: need H,W >= 2");
  GSX_CHECK_ARG((int64_t)B * L <= 65535, "gsx_backproject_normals_bwd: extents too large");
  if ((int64_t)B * L == 0) return 0;
  const int tiles = (int)(((int64_t)H * W + gsx::kTile - 1) / gsx::kTile);
  const bool want_pose = g_poses && poses, want_k = g_intrinsics != nullptr;
  if (want_k)
    GSX_CHECK_ARG(scratch && scratch_bytes >= gsx_backproject_normals_bwd_intrinsics_scratch_bytes(B, L, H, W),
                  "gsx_backproject_normals_bwd: scratch too small");
  else if (want_pose)
    GSX_CHECK_ARG(scratch && scratch_bytes >= gsx_backproject_normals_bwd_scratch_bytes(B, L, H, W),
                  "gsx_backproject_normals_bwd: scratch too small");
  const gsx::FrameBwdScratch sc = gsx::frame_bwd_scratch(scratch, B, L, tiles);
  gsx::FrameBwdArgs a{depth, depth_bstride, intrinsics, K_bstride, poses, pose_bstride, B, L, H, W,
                      {g_vertex, g_normal, g_gvertex, g_gnormal}, g_depth, want_pose ? sc.pose : nullptr, tiles};
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid((unsigned)tiles, (unsigned)(B * L));
  if (want_k)
    gsx::k_backproject_normals_bwd<true><<<grid, gsx::kTile, 0, s>>>(a, sc.kinv);
  else
    gsx::k_backproject_normals_bwd<false><<<grid, gsx::kTile, 0, s>>>(a, nullptr);
  if (want_pose) gsx::k_pose_grad_reduce<<<B * L, 16, 0, s>>>(sc.pose, tiles, g_poses, B * L);
  if (want_k) gsx::k_intrinsics_grad_reduce<<<B, 128, 0, s>>>(sc.kinv, L, tiles, intrinsics, K_bstride, g_intrinsics);
  GSX_CHECK_LAUNCH("gsx_backproject_normals_bwd");
  return 0;
}

extern "C" int gsx_backproject_normals_bwd(const float *depth, int64_t depth_bstride, const float *intrinsics,
                                           int64_t K_bstride, const float *poses, int64_t pose_bstride, int B,
                                           int L, int H, int W, const float *g_vertex, const float *g_normal,
                                           const float *g_gvertex, const float *g_gnormal, float *g_depth,
                                           float *g_poses, void *scratch, int64_t scratch_bytes, void *stream) {
  return gsx_backproject_normals_bwd_intrinsics(depth, depth_bstride, intrinsics, K_bstride, poses, pose_bstride, B, L,
                                                H, W, g_vertex, g_normal, g_gvertex, g_gnormal, g_depth, g_poses,
                                                nullptr, scratch, scratch_bytes, stream);
}
