// Shared device helpers for libgsx (sm_90a).  Compiled with -fmad=false: every product and sum below
// is rounded separately to fp32, in the association order written, so results are bit-identical to the
// CPU oracle's canonical arithmetic (oracle/gsx_oracle.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>

namespace gsx {

void set_error(const char *fmt, ...);

#define GSX_CHECK_ARG(cond, ...)   \
  do {                             \
    if (!(cond)) {                 \
      gsx::set_error(__VA_ARGS__); \
      return 1;                    \
    }                              \
  } while (0)

#define GSX_CHECK_LAUNCH(name)                                                    \
  do {                                                                            \
    cudaError_t e_ = cudaGetLastError();                                          \
    if (e_ != cudaSuccess) {                                                      \
      gsx::set_error("%s: launch failed: %s", name, cudaGetErrorString(e_));     \
      return 2;                                                                   \
    }                                                                             \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

// floats per packed map row (DESIGN.md section 2): geometry (px,py,pz,nx,ny,nz,ccount,0), colour (r,g,b,0)
constexpr int kGeoW = 8, kColW = 4;

// Scratch and workspace layouts are each written once, as a function that walks a Carver over the allocation:
// take<T>(n) hands out the next 256-byte aligned slot of n T's.  Given the allocation's base the function returns
// pointers; given nullptr the pointers are the slots' byte offsets, and `bytes` is the size the allocation needs.
struct Carver {
  uintptr_t base;
  int64_t bytes = 0;
  explicit Carver(void *p) : base(reinterpret_cast<uintptr_t>(p)) {}
  template <class T>
  T *take(int64_t n) {
    T *p = reinterpret_cast<T *>(base + bytes);
    bytes += (n * (int64_t)sizeof(T) + 255) / 256 * 256;
    return p;
  }
};

struct Rigid {  // row-major rotation + translation of a 4x4 rigid transform
  float r[9];
  float t[3];
};

__device__ __forceinline__ Rigid load_rigid(const float *__restrict__ T) {
  Rigid a;
  a.r[0] = __ldg(T + 0); a.r[1] = __ldg(T + 1); a.r[2] = __ldg(T + 2);  a.t[0] = __ldg(T + 3);
  a.r[3] = __ldg(T + 4); a.r[4] = __ldg(T + 5); a.r[5] = __ldg(T + 6);  a.t[1] = __ldg(T + 7);
  a.r[6] = __ldg(T + 8); a.r[7] = __ldg(T + 9); a.r[8] = __ldg(T + 10); a.t[2] = __ldg(T + 11);
  return a;
}

__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
  return (a0 * b0 + a1 * b1) + a2 * b2;
}

// [R^T, (-R^T) t]   (kornia inverse_transformation as called at gradslam/slam/fusionutils.py:249)
__device__ __forceinline__ Rigid rigid_inverse(const Rigid &a) {
  Rigid o;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) o.r[i * 3 + j] = a.r[j * 3 + i];
    o.t[i] = dot3(-a.r[0 * 3 + i], -a.r[1 * 3 + i], -a.r[2 * 3 + i], a.t[0], a.t[1], a.t[2]);
  }
  return o;
}

__device__ __forceinline__ float3 rigid_apply(const Rigid &a, float x, float y, float z) {
  float3 q;
  q.x = dot3(a.r[0], a.r[1], a.r[2], x, y, z) + a.t[0];
  q.y = dot3(a.r[3], a.r[4], a.r[5], x, y, z) + a.t[1];
  q.z = dot3(a.r[6], a.r[7], a.r[8], x, y, z) + a.t[2];
  return q;
}

__device__ __forceinline__ float3 rotate(const Rigid &a, float x, float y, float z) {
  float3 q;
  q.x = dot3(a.r[0], a.r[1], a.r[2], x, y, z);
  q.y = dot3(a.r[3], a.r[4], a.r[5], x, y, z);
  q.z = dot3(a.r[6], a.r[7], a.r[8], x, y, z);
  return q;
}

// closed-form inverse intrinsics (gradslam/geometry/projutils.py:405-450): eps added to fx, fy.
struct KInv {
  float k00, k02, k11, k12;
};
__device__ __forceinline__ KInv load_kinv(const float *__restrict__ K) {
  const float fx = __ldg(K + 0), fy = __ldg(K + 5), cx = __ldg(K + 2), cy = __ldg(K + 6);
  KInv k;
  k.k00 = 1.0f / (fx + 1e-6f);
  k.k11 = 1.0f / (fy + 1e-6f);
  k.k02 = (-1.0f * cx) / (fx + 1e-6f);
  k.k12 = (-1.0f * cy) / (fy + 1e-6f);
  return k;
}

// local vertex of pixel (u=w, v=h) with depth d, zeroed where d <= 0 (rgbdimages.py:672-679)
__device__ __forceinline__ float3 backproject(const KInv &k, float u, float v, float d) {
  const float vf = d > 0.0f ? 1.0f : 0.0f;
  float3 p;
  p.x = ((k.k00 * u + k.k02) * d) * vf;
  p.y = ((k.k11 * v + k.k12) * d) * vf;
  p.z = d * vf;
  return p;
}

// world-frame vertex of a pixel with depth d and local vertex v: (R v + t) * valid, or v itself when pose == nullptr
// (world frame == camera frame).  K1r's gv, and what the fusion consumers recompute from the depth in the frame record.
__device__ __forceinline__ float3 world_vertex(const Rigid *pose, const float3 &v, float d) {
  if (!pose) return v;
  const float vf = d > 0.0f ? 1.0f : 0.0f;
  float3 g = rigid_apply(*pose, v.x, v.y, v.z);
  g.x *= vf; g.y *= vf; g.z *= vf;
  return g;
}

// The camera a frame was back-projected with (K1r's K^-1 and camera-to-world pose), kept per element in the fusion
// workspace so that K2 and K4 recompute a pixel's vertex from its depth with exactly K1r's operands.
struct FrameCamera {
  Rigid pose;
  KInv k;
  int posed;  // 0: no pose, world frame == camera frame
};
__device__ __forceinline__ float3 frame_local_vertex(const FrameCamera &c, int h, int w, float d) {
  return backproject(c.k, (float)w, (float)h, d);
}
__device__ __forceinline__ float3 frame_world_vertex(const FrameCamera &c, const float3 &v, float d) {
  return world_vertex(c.posed ? &c.pose : nullptr, v, d);
}

// Vertex and normal of pixel (h,w) of depth image `dimg`, in the camera frame and (if pose != nullptr) in the
// world frame: the whole op chain of gradslam/structures/rgbdimages.py:643-762 for one pixel.  Used by K1 (to
// materialise maps) and, on the fly, by the fusion kernels, so both see bit-identical values.
//   v  = K^-1 (w,h,1) d, zeroed where d <= 0            n  = normalize(dh x dv) * valid(centre)
//   dh = forward difference along w (last column re-uses its neighbour's), dv along h likewise
//   gv = (R v + t) * valid                              gn = R n
struct FrameSample {
  float3 v, n, gv, gn;
  float d;
};

// a x b and |c| rounded exactly like the reference's CPU build (torch.cross / Tensor.norm on float32,
// rgbdimages.py:733-734): cross.x = fma(a.y, b.z, -(a.z * b.y)) - first product exact, second rounded - and
// |c| = sqrt(fma(c.z, c.z, fma(c.y, c.y, c.x * c.x))).  Where a valid pixel's right AND lower neighbours are both
// missing, a == b and the contracted cross product is rounding residue rather than 0; normalised, it decides whether
// map points match there, so the kernels and the oracle (oracle/normal_fma.c) reproduce it bit for bit.  The library
// is built with -fmad=false: only these explicit fused operations are fused.
__device__ __forceinline__ float3 cross_ref(float ax, float ay, float az, float bx, float by, float bz) {
  return make_float3(__fmaf_rn(ay, bz, -__fmul_rn(az, by)), __fmaf_rn(az, bx, -__fmul_rn(ax, bz)),
                     __fmaf_rn(ax, by, -__fmul_rn(ay, bx)));
}
__device__ __forceinline__ float norm_ref(const float3 &c) {
  return __fsqrt_rn(__fmaf_rn(c.z, c.z, __fmaf_rn(c.y, c.y, __fmul_rn(c.x, c.x))));
}

// un-normalised local normal dh x dv of pixel (h,w) given its own local vertex v
__device__ __forceinline__ float3 frame_cross(const float *__restrict__ dimg, const KInv &k, int h, int w, int H, int W,
                                              const float3 &v) {
  const int wa = (w < W - 1) ? w : w - 1;
  const int ha = (h < H - 1) ? h : h - 1;
  const float dr = __ldg(dimg + h * W + wa + 1);
  const float db = __ldg(dimg + (ha + 1) * W + w);
  const float3 a1 = backproject(k, (float)(wa + 1), (float)h, dr);
  const float3 b1 = backproject(k, (float)w, (float)(ha + 1), db);
  const float3 a0 = (wa == w) ? v : backproject(k, (float)wa, (float)h, __ldg(dimg + h * W + wa));
  const float3 b0 = (ha == h) ? v : backproject(k, (float)w, (float)ha, __ldg(dimg + ha * W + w));
  const float dhx = a1.x - a0.x, dhy = a1.y - a0.y, dhz = a1.z - a0.z;
  const float dvx = b1.x - b0.x, dvy = b1.y - b0.y, dvz = b1.z - b0.z;
  return cross_ref(dhx, dhy, dhz, dvx, dvy, dvz);
}

// normalize(c) * vf, the zero vector staying zero (rgbdimages.py:731-743)
__device__ __forceinline__ float3 normalize_masked(const float3 &c, float vf) {
  const float nrm = norm_ref(c);
  const float den = (nrm == 0.0f) ? 1.0f : nrm;
  return make_float3((c.x / den) * vf, (c.y / den) * vf, (c.z / den) * vf);
}

// local normal of pixel (h,w) given its own local vertex v and validity vf (1 or 0)
__device__ __forceinline__ float3 frame_normal(const float *__restrict__ dimg, const KInv &k, int h, int w, int H, int W,
                                               const float3 &v, float vf) {
  return normalize_masked(frame_cross(dimg, k, h, w, H, W, v), vf);
}

// The five depth values the sample of pixel (h,w) depends on: centre, the two ends of its horizontal difference
// (w_a, w_a+1) and of its vertical difference (h_a, h_a+1), where w_a = min(w, W-2), h_a = min(h, H-2).  Away from the
// last column / row l and u are the centre itself, so only the centre, its right and its lower neighbour are loaded.
struct DepthStencil {
  float c, l, r, u, d;
};
// the stencil of pixel (h,w) whose own depth c is already loaded
__device__ __forceinline__ DepthStencil load_stencil_around(const float *__restrict__ dimg, float c, int h, int w, int H,
                                                           int W) {
  const int wa = (w < W - 1) ? w : w - 1;
  const int ha = (h < H - 1) ? h : h - 1;
  DepthStencil s;
  s.c = c;
  s.r = __ldg(dimg + h * W + wa + 1);
  s.d = __ldg(dimg + (ha + 1) * W + w);
  s.l = (wa == w) ? s.c : __ldg(dimg + h * W + wa);
  s.u = (ha == h) ? s.c : __ldg(dimg + ha * W + w);
  return s;
}
__device__ __forceinline__ DepthStencil load_stencil(const float *__restrict__ dimg, int h, int w, int H, int W) {
  return load_stencil_around(dimg, __ldg(dimg + h * W + w), h, w, H, W);
}
// frame_sample<true> evaluated from an already loaded stencil (bit-identical arithmetic)
__device__ __forceinline__ FrameSample frame_sample_from(const DepthStencil &t, const KInv &k, const Rigid *pose, int h,
                                                         int w, int H, int W) {
  FrameSample s;
  const int wa = (w < W - 1) ? w : w - 1;
  const int ha = (h < H - 1) ? h : h - 1;
  s.d = t.c;
  const float vf = t.c > 0.0f ? 1.0f : 0.0f;
  s.v = backproject(k, (float)w, (float)h, t.c);
  const float3 a1 = backproject(k, (float)(wa + 1), (float)h, t.r);
  const float3 b1 = backproject(k, (float)w, (float)(ha + 1), t.d);
  const float3 a0 = (wa == w) ? s.v : backproject(k, (float)wa, (float)h, t.l);
  const float3 b0 = (ha == h) ? s.v : backproject(k, (float)w, (float)ha, t.u);
  const float dhx = a1.x - a0.x, dhy = a1.y - a0.y, dhz = a1.z - a0.z;
  const float dvx = b1.x - b0.x, dvy = b1.y - b0.y, dvz = b1.z - b0.z;
  s.n = normalize_masked(cross_ref(dhx, dhy, dhz, dvx, dvy, dvz), vf);
  s.gv = world_vertex(pose, s.v, s.d);
  s.gn = pose ? rotate(*pose, s.n.x, s.n.y, s.n.z) : s.n;
  return s;
}

template <bool kWantNormal>
__device__ __forceinline__ FrameSample frame_sample(const float *__restrict__ dimg, const KInv &k, const Rigid *pose,
                                                    int h, int w, int H, int W) {
  FrameSample s;
  const float dc = __ldg(dimg + h * W + w);
  s.d = dc;
  const float vf = dc > 0.0f ? 1.0f : 0.0f;
  s.v = backproject(k, (float)w, (float)h, dc);
  s.n = kWantNormal ? frame_normal(dimg, k, h, w, H, W, s.v, vf) : make_float3(0.f, 0.f, 0.f);
  s.gv = world_vertex(pose, s.v, dc);
  s.gn = (pose && kWantNormal) ? rotate(*pose, s.n.x, s.n.y, s.n.z) : s.n;
  return s;
}

// High word of the arg-min key of find_best_unique_correspondences (fusionutils.py:491-517): 1/(cc+1e-20), then the
// squared distance d2 >= 0.  Positive floats order like their bit patterns; negatives are flipped so the order stays total.
__device__ __forceinline__ unsigned long long argmin_key_hi(float cc, float d2) {
  const float inv_cc = 1.0f / (cc + 1e-20f);
  unsigned int kb = __float_as_uint(inv_cc);
  kb = (kb & 0x80000000u) ? ~kb : (kb | 0x80000000u);
  const unsigned int rb = __float_as_uint(d2) | 0x80000000u;
  return ((unsigned long long)kb << 32) | rb;
}

// Squared distance between a pixel's frame vertex fv and a map point: the ray distance of the arg-min key and the
// quantity of the distance test.  Negating the difference does not change a square, so map - frame gives the same bits.
__device__ __forceinline__ float ray_d2(const float3 &fv, float x, float y, float z) {
  const float dx = fv.x - x, dy = fv.y - y, dz = fv.z - z;
  return (dx * dx + dy * dy) + dz * dz;
}

// ---- per-pixel arg-min over map rows (find_best_unique_correspondences, fusionutils.py:414-546) ----------------------
// A pixel's 4-byte slot holds n + 1 of the row that currently wins it, 0 for none.  The key of a candidate row n,
// (argmin_key_hi(cc, ray_d2(fv, p)), n), is a fixed function of the row (read-only while the arg-min runs) and of the
// pixel's frame vertex fv, which every candidate of the pixel computes bit for bit; so the slot holds no key, and a
// candidate that finds the slot taken gathers the stored row and recomputes that row's key.
// Claiming is optimistic (most pixels see a single candidate) and returns the slot's previous value; argmin_settle
// finishes the update from it, so that a caller may look at the result of the CAS later.
__device__ __forceinline__ unsigned int argmin_claim(unsigned int *slot, unsigned int n) {
  return atomicCAS(slot, 0u, n + 1u);
}

// geo: the element's geometry rows.  Replaces the stored row while this candidate's key is the smaller one.
__device__ __forceinline__ void argmin_settle(unsigned int *slot, unsigned int n, unsigned long long key_hi,
                                              const float3 &fv, const float *geo, unsigned int old) {
  unsigned int cur = 0u;
  while (old != cur) {  // the last CAS did not take effect: row old - 1 holds the slot
    cur = old;
    const unsigned int m = cur - 1u;
    const float4 p = __ldg(reinterpret_cast<const float4 *>(geo + (int64_t)m * kGeoW));
    const unsigned long long k = argmin_key_hi(__ldg(geo + (int64_t)m * kGeoW + 6), ray_d2(fv, p.x, p.y, p.z));
    if (k < key_hi || (k == key_hi && m <= n)) return;
    old = atomicCAS(slot, cur, n + 1u);
  }
}

// ---- projection of a map point into the live camera (fusionutils.py:249-274) ----------------------------------------
struct ImageBounds {  // frustum limits of an H x W image (kernel argument)
  float u_hi, v_hi;   // float(W - 0.999), float(H - 0.999)
  int H, W;
};
inline ImageBounds image_bounds(int H, int W) { return ImageBounds{(float)(W - 0.999), (float)(H - 0.999), H, W}; }

struct LiveCamera {  // per CTA, in shared memory: world -> camera (T^-1) and the first three rows of the 4x4 K
  Rigid tinv;
  float k[12];
};
// Camera of batch element b.  Called by every thread (thread 0 loads T^-1, threads 32..43 the K entries); the caller
// synchronises.
__device__ __forceinline__ void load_live_camera(LiveCamera &c, const float *poses, int64_t pose_bstride,
                                                 const float *K, int64_t K_bstride, int b) {
  if (threadIdx.x == 0) c.tinv = rigid_inverse(load_rigid(poses + b * pose_bstride));
  if (threadIdx.x >= 32 && threadIdx.x < 44) c.k[threadIdx.x - 32] = __ldg(K + b * K_bstride + (threadIdx.x - 32));
}

struct PixelHit {
  bool in_frustum;
  int h, w;  // pixel under the projection, clamped to the image
  float z;   // camera-frame depth q.z (the free-space test of gsx_prune.cu)
};
// world -> camera (pointclouds.py:526-573), pinhole projection with the 4x4 K on the homogeneous point
// (projutils.py:92-238; z == 0 divides by 1), frustum test, round-half-even like torch.round, then clamp
__device__ __forceinline__ PixelHit project(const LiveCamera &c, const ImageBounds &ib, float x, float y, float z) {
  const float3 q = rigid_apply(c.tinv, x, y, z);
  const float hx = ((c.k[0] * q.x + c.k[1] * q.y) + c.k[2] * q.z) + c.k[3];
  const float hy = ((c.k[4] * q.x + c.k[5] * q.y) + c.k[6] * q.z) + c.k[7];
  const float hz = ((c.k[8] * q.x + c.k[9] * q.y) + c.k[10] * q.z) + c.k[11];
  const float den = (hz != 0.0f) ? hz : 1.0f;
  const float u = hx / den, v = hy / den;
  PixelHit r;
  r.in_frustum = (u > -1e-3f) && (u < ib.u_hi) && (v > -1e-3f) && (v < ib.v_hi) && (q.z > 0.0f);
  r.w = min(max((int)rintf(u), 0), ib.W - 1);
  r.h = min(max((int)rintf(v), 0), ib.H - 1);
  r.z = q.z;
  return r;
}

// ---- stable compaction by single-pass decoupled look-back --------------------------------------------------------
// A scan runs one CTA per tile.  Each tile owns a 64-bit state word  epoch<<34 | flag<<32 | value : flag kTileAggregate
// = `value` counts the tile's own items, kTilePrefix = `value` counts the items of every tile up to and including it.
// A word of another epoch reads as "not yet published": a scan passes a fresh epoch per launch, or zeroes its words
// before each launch and passes epoch 1.  The last tile publishes nothing (no tile waits for it).
constexpr unsigned long long kTileAggregate = 1ull, kTilePrefix = 2ull;

__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u64(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ void publish_tile(unsigned long long *state, int tile, int tiles, unsigned int epoch,
                                             unsigned long long flag, unsigned int value) {
  if (tile + 1 < tiles) st_release_u64(state + tile, ((unsigned long long)epoch << 34) | (flag << 32) | value);
}

// Called by one whole warp once the tile's aggregate `total` is published: returns the tile's exclusive prefix (32
// predecessors per step, back to the nearest one that knows its inclusive prefix); lane 0 then publishes the tile's
// inclusive prefix.
__device__ __forceinline__ unsigned int lookback_warp(unsigned long long *state, int tile, int tiles,
                                                      unsigned int epoch, unsigned int total) {
  const int lane = threadIdx.x & 31;
  unsigned int excl = 0;
  for (int base = tile - 1; base >= 0; base -= 32) {
    const int j = base - lane;
    unsigned long long s = 0ull;
    if (j >= 0) {
      do {
        s = ld_acquire_u64(state + j);
      } while ((unsigned int)(s >> 34) != epoch);
    }
    const bool is_prefix = (j >= 0) && (((s >> 32) & 3ull) == kTilePrefix);
    const unsigned int pm = __ballot_sync(0xffffffffu, is_prefix);
    const int first = pm ? (__ffs(pm) - 1) : 32;  // nearest predecessor that already knows its inclusive prefix
    const unsigned int v = (j >= 0 && lane <= first) ? (unsigned int)s : 0u;
    excl += __reduce_add_sync(0xffffffffu, v);
    if (pm) break;
  }
  if (lane == 0) publish_tile(state, tile, tiles, epoch, kTilePrefix, excl + total);
  return excl;
}

// Dynamic tile id (tiles start in ticket order).  The CTA that draws the last ticket re-arms the counter for the next
// launch (nobody else touches it any more in this one), so the number of tiles may differ from launch to launch.
__device__ __forceinline__ int draw_tile_ticket(unsigned int *ticket, int tiles) {
  const unsigned int t = atomicAdd(ticket, 1u);
  if (t == (unsigned int)tiles - 1u) *ticket = 0u;
  return (int)t;
}

// Stable positions of kPer flags per thread of a kThreads-thread CTA, in row-major order: chunk j, then warp, then lane.
// flag(j) yields this thread's flag j; it is evaluated right before that flag's warp vote, so the work deciding each flag
// is interleaved with the votes.  Every thread calls this: it synchronises the CTA once, and runs at_barrier() right
// after that barrier (CTA-wide work of the caller that needs one).  On return off[j] = the number of set flags before
// this thread's flag j; returns the CTA's total.  s_count is kPer x (kThreads / 32) ints of shared memory.
template <int kThreads, int kPer, class Flag, class AtBarrier>
__device__ __forceinline__ int block_offsets(Flag flag, int (&off)[kPer], int (*s_count)[kThreads / 32],
                                             AtBarrier at_barrier) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    const unsigned int ballot = __ballot_sync(0xffffffffu, flag(j));
    off[j] = __popc(ballot & ((1u << lane) - 1u));
    if (lane == 0) s_count[j][warp] = __popc(ballot);
  }
  __syncthreads();
  at_barrier();
  int total = 0;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    int excl = total;
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) {
      const int c = s_count[j][i];
      if (i < warp) excl += c;
      total += c;
    }
    off[j] += excl;
  }
  return total;
}

}  // namespace gsx
