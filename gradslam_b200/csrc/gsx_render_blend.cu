// Blended disk splats (render_pointclouds(blend_band=eps), an extension: the reference has no counterpart).  A pixel
// shows the normalised, weighted mean of the rows that cover it near the front surface (surface splatting, Zwicker et
// al. 2001), instead of the one row the z-buffer keeps.  Coverage is R1d's (R1's at max_splat_px = 0); the front depth
// z_f and the index image are R1d's, computed by its unchanged launch.  A row n covering pixel p contributes when its
// depth there is t_n(p) <= fp32(z_f(p) + eps), with weight w_n = c_n (1 - s2_n / r_n^2) for a disk (s2 the squared
// in-plane distance disk_hit tests) and c_n otherwise; c_n is the confidence count (slot 6) or 1.
//   k_blend_key       (B1)  per (row, view): the bucket of the row's projected centre on a grid padded by M pixels on
//                           every side (every bucket whose box meets the image), or none; integer counts per bucket.
//   k_scan_*          (B2)  exclusive scan of the bucket counts: tile sums, one CTA over the tile sums, tile rescans.
//   k_blend_place     (B3)  rows into their buckets at the slot the count handed out; k_blend_sort_buckets then sorts
//                           each bucket by row index, so a bucket's order does not depend on the atomics' order.
//   k_blend_resolve   (B4)  per pixel: the buckets of the (2M+1)^2 centres around it in (dy, dx, row) order, the five
//                           sums in registers; no float atomics, so two runs give equal bits.
//   k_blend_bwd_rows  (B5)  per row, the backward: re-enumerates its footprint per view in (view, h, w) order and,
//                           where it contributed, chains dout/dw = (v - out)/W and dout/dv = w/W to its position, normal,
//                           radius, confidence and colour; per view and CTA the pose partials, summed in tile order by
//                           k_pose_grad_reduce.  No atomics.
#include "gsx_render.cuh"
#include "../../include/gsx.h"

namespace gsx {

// defined in gsx_frame.cu: partials (img, tile, 12) summed in tile order -> (img, 4, 4), bottom row zero
__global__ void k_pose_grad_reduce(const float *partials, int tiles, float *g_poses, int n_img);

constexpr int kScanPer = 16;                  // counts per thread of a scan tile
constexpr int kScanTile = kRB * kScanPer;     // counts per scan tile
constexpr int kScanTop = 1024;                // threads of the CTA that scans the tile sums

struct BlendArgs {
  const float *geo, *col;  // (B,cap,8), (B,cap,4) or null
  const int32_t *counts;
  int64_t cap;
  int bound;               // host bound on counts[b]: items are (b, n < bound, l)
  const float *K;
  int64_t K_bstride;
  const float *poses;
  int64_t pose_bstride;
  int L, M;
  ImageBounds ib;
  int BW;                  // bucket grid width W + 2M (height H + 2M)
  int64_t NB;              // buckets per view
  int use_conf;            // weights from slot 6, else 1
  double band;             // eps
};

// The bucket (bh, bw) of a row in one camera, on the grid padded by M: a disk's projected centre when its box meets the
// image, else (one-pixel rows, or M = 0) the pixel project() gives when the row is in the frustum.
__device__ __forceinline__ bool blend_bucket(const LiveCamera &c, const ImageBounds &ib, int M, const float4 &g0,
                                             const float4 &g1, int &bh, int &bw) {
  if (M > 0 && is_disk(g0, g1)) {
    const Disk d = make_disk(c, ib, M, g0, g1);
    bh = d.cv + M;
    bw = d.cu + M;
    return d.h0 <= d.h1 && d.w0 <= d.w1;
  }
  const PixelHit hit = project(c, ib, g0.x, g0.y, g0.z);
  bh = hit.h + M;
  bw = hit.w + M;
  return hit.in_frustum;
}

__global__ void __launch_bounds__(kRB) k_blend_key(BlendArgs a, unsigned int *key, int *rank, int *cnt,
                                                   unsigned int invalid) {
  __shared__ LiveCamera s_cam[kViews];
  const int b = blockIdx.y, l0 = blockIdx.z * kViews;
  const int nv = min(kViews, a.L - l0);
  load_view_cameras(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b, l0, nv);
  __syncthreads();
  const int n = blockIdx.x * kRB + threadIdx.x;
  if (n >= a.bound) return;
  const bool live = n < a.counts[b];
  float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0;
  if (live) {
    g0 = __ldg(reinterpret_cast<const float4 *>(a.geo + ((int64_t)b * a.cap + n) * kGeoW));
    g1 = __ldg(reinterpret_cast<const float4 *>(a.geo + ((int64_t)b * a.cap + n) * kGeoW + 4));
  }
  const int64_t e0 = ((int64_t)b * a.bound + n) * a.L + l0;
  for (int v = 0; v < nv; ++v) {
    int bh, bw;
    unsigned int k = invalid;
    if (live && blend_bucket(s_cam[v], a.ib, a.M, g0, g1, bh, bw)) {
      k = (unsigned int)(((int64_t)b * a.L + l0 + v) * a.NB + (int64_t)bh * a.BW + bw);
      rank[e0 + v] = atomicAdd(cnt + k, 1);
    }
    key[e0 + v] = k;
  }
}

// Exclusive scan of x over a CTA of kThreads threads; *total = the CTA's sum.  s_warp: kThreads / 32 ints.
template <int kThreads>
__device__ __forceinline__ int block_exclusive_scan(int x, int *s_warp, int *total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int pre = 0, tot = 0;
#pragma unroll
  for (int i = 0; i < kThreads / 32; ++i) {
    const int c = s_warp[i];
    if (i < warp) pre += c;
    tot += c;
  }
  __syncthreads();  // s_warp may be reused
  *total = tot;
  return pre + inc - x;
}

__global__ void __launch_bounds__(kRB) k_scan_reduce(const int *cnt, int64_t n, int *tile_sum) {
  __shared__ int s_warp[kRB / 32];
  const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanPer;
  int x = 0;
#pragma unroll
  for (int j = 0; j < kScanPer; ++j)
    if (base + j < n) x += cnt[base + j];
  int total;
  block_exclusive_scan<kRB>(x, s_warp, &total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanTop) k_scan_tiles(int *tile_sum, int tiles) {
  __shared__ int s_warp[kScanTop / 32];
  int carry = 0;
  for (int t0 = 0; t0 < tiles; t0 += kScanTop) {
    const int t = t0 + threadIdx.x;
    const int x = t < tiles ? tile_sum[t] : 0;
    int total;
    const int ex = block_exclusive_scan<kScanTop>(x, s_warp, &total);
    if (t < tiles) tile_sum[t] = carry + ex;
    carry += total;
  }
}

__global__ void __launch_bounds__(kRB) k_scan_apply(int *cnt, int64_t n, const int *tile_prefix) {
  __shared__ int s_warp[kRB / 32];
  const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanPer;
  int v[kScanPer];
  int x = 0;
#pragma unroll
  for (int j = 0; j < kScanPer; ++j) {
    v[j] = base + j < n ? cnt[base + j] : 0;
    x += v[j];
  }
  int total;
  int run = tile_prefix[blockIdx.x] + block_exclusive_scan<kRB>(x, s_warp, &total);
#pragma unroll
  for (int j = 0; j < kScanPer; ++j) {
    if (base + j < n) cnt[base + j] = run;
    run += v[j];
  }
}

__global__ void __launch_bounds__(kRB) k_blend_place(const unsigned int *key, const int *rank, const int *start,
                                                     int64_t items, int bound, int L, unsigned int invalid, int *rows) {
  const int64_t e = (int64_t)blockIdx.x * kRB + threadIdx.x;
  if (e >= items) return;
  const unsigned int k = key[e];
  if (k == invalid) return;
  rows[start[k] + rank[e]] = (int)((e / L) % bound);
}

// Each bucket's rows in ascending order (insertion sort for a few rows, heapsort beyond).
__global__ void __launch_bounds__(kRB) k_blend_sort_buckets(const int *start, int64_t buckets, int *rows) {
  const int64_t k = (int64_t)blockIdx.x * kRB + threadIdx.x;
  if (k >= buckets) return;
  int *r = rows + start[k];
  const int c = start[k + 1] - start[k];
  if (c <= 1) return;
  if (c <= 16) {
    for (int i = 1; i < c; ++i) {
      const int x = r[i];
      int j = i - 1;
      while (j >= 0 && r[j] > x) {
        r[j + 1] = r[j];
        --j;
      }
      r[j + 1] = x;
    }
    return;
  }
  auto sift = [&](int i, int end) {
    const int x = r[i];
    for (int ch = 2 * i + 1; ch < end; ch = 2 * i + 1) {
      if (ch + 1 < end && r[ch + 1] > r[ch]) ++ch;
      if (r[ch] <= x) break;
      r[i] = r[ch];
      i = ch;
    }
    r[i] = x;
  };
  for (int i = c / 2 - 1; i >= 0; --i) sift(i, c);
  for (int end = c - 1; end > 0; --end) {
    const int x = r[0];
    r[0] = r[end];
    r[end] = x;
    sift(0, end);
  }
}

// One contributor of a pixel: depth t, weight w, camera-frame normal m; for a disk also the ray, e = t d - q and s2.
struct Contribution {
  float t, w, s2, md;
  float3 m, q, ray;
  bool disk;
};

// Row (g0, g1) at pixel (h, w), its bucket at offset (dy, dx) from the pixel: false unless it covers the pixel (R1d's
// rule) within the band; z_lim = fp32(z_f + eps).
__device__ __forceinline__ bool contribution(const BlendArgs &a, const LiveCamera &c, const KInv &kinv, const float4 &g0,
                                             const float4 &g1, int h, int w, bool centre, float z_lim,
                                             Contribution &o) {
  const float cc = a.use_conf ? g1.z : 1.0f;
  o.disk = a.M > 0 && is_disk(g0, g1);
  if (o.disk) {
    const Disk d = make_disk(c, a.ib, a.M, g0, g1);
    if (!disk_hit(d, kinv, h, w, o.t, o.md, o.ray)) return false;
    if (!(o.t <= z_lim)) return false;
    const float ex = o.t * o.ray.x - d.q.x, ey = o.t * o.ray.y - d.q.y, ez = o.t * o.ray.z - d.q.z;
    o.s2 = (ex * ex + ey * ey) + ez * ez;
    o.w = cc * (1.0f - o.s2 / d.rr);
    o.m = d.m;
    o.q = d.q;
    return true;
  }
  if (!centre) return false;  // a one-pixel row covers the pixel of its bucket only
  o.q = rigid_apply(c.tinv, g0.x, g0.y, g0.z);
  o.t = o.q.z;
  if (!(o.t <= z_lim)) return false;
  o.w = cc;
  o.s2 = 0.0f;
  o.m = rotate(c.tinv, g0.w, g1.x, g1.y);
  return true;
}

__device__ __forceinline__ float band_limit(float zf, double band) { return __double2float_rn((double)zf + band); }

__global__ void __launch_bounds__(kRB) k_blend_resolve(BlendArgs a, const int64_t *index, const float *zf,
                                                       const int *start, const int *rows, float *weight, float *depth,
                                                       float *rgb, float *normals) {
  __shared__ LiveCamera s_cam;
  __shared__ KInv s_kinv;
  const int img = blockIdx.y;
  const int b = img / a.L, l = img - b * a.L;
  load_view_cameras(&s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b, l, 1);
  if (threadIdx.x == 0) s_kinv = load_kinv(a.K + b * a.K_bstride);
  __syncthreads();
  const int W = a.ib.W;
  const int64_t P = (int64_t)a.ib.H * W;
  const int64_t pix = (int64_t)blockIdx.x * kRB + threadIdx.x;
  if (pix >= P) return;
  const int h = (int)(pix / W), w = (int)(pix - (int64_t)h * W);
  const int64_t i = img * P + pix;
  float sw = 0.f, sd = 0.f, sc[3] = {0.f, 0.f, 0.f}, sn[3] = {0.f, 0.f, 0.f};
  if (__ldg(index + i) >= 0) {
    const float z_lim = band_limit(__ldg(zf + i), a.band);
    const float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
    const int *bucket = start + img * a.NB;
    for (int dy = -a.M; dy <= a.M; ++dy)
      for (int dx = -a.M; dx <= a.M; ++dx) {
        const int64_t k = (int64_t)(h + dy + a.M) * a.BW + (w + dx + a.M);
        const int j1 = __ldg(bucket + k + 1);
        for (int j = __ldg(bucket + k); j < j1; ++j) {
          const int64_t n = __ldg(rows + j);
          const float4 g0 = __ldg(reinterpret_cast<const float4 *>(geo + n * kGeoW));
          const float4 g1 = __ldg(reinterpret_cast<const float4 *>(geo + n * kGeoW + 4));
          Contribution c;
          if (!contribution(a, s_cam, s_kinv, g0, g1, h, w, dy == 0 && dx == 0, z_lim, c)) continue;
          sw += c.w;
          sd += c.w * c.t;
          if (rgb) {
            const float4 col = __ldg(reinterpret_cast<const float4 *>(a.col + ((int64_t)b * a.cap + n) * kColW));
            sc[0] += c.w * col.x; sc[1] += c.w * col.y; sc[2] += c.w * col.z;
          }
          sn[0] += c.w * c.m.x; sn[1] += c.w * c.m.y; sn[2] += c.w * c.m.z;
        }
      }
  }
  const bool any = sw != 0.0f;
  const float den = any ? sw : 1.0f;
  weight[i] = sw;
  depth[i] = any ? sd / den : 0.0f;
  if (rgb)
#pragma unroll
    for (int j = 0; j < 3; ++j) rgb[i * 3 + j] = any ? sc[j] / den : 0.0f;
  if (normals)
#pragma unroll
    for (int j = 0; j < 3; ++j) normals[i * 3 + j] = any ? sn[j] / den : 0.0f;
}

// ---- backward ---------------------------------------------------------------------------------------------------
struct BlendBwdArgs {
  const float *zf, *weight, *depth, *rgb, *normals;      // forward: front depth, W and the outputs
  const float *g_depth, *g_rgb, *g_normals, *g_weight;   // upstream gradients, any may be null (zero)
  float *d_geo, *d_col;                                  // or null
  float *pose_partials;                                  // (B*L, gridDim.x, 12) or null
};

// Per contributing pixel i of a row, with r = w/W and a = dL/dw = sum_k g_k (v_k - out_k)/W + g_weight:
//   value:  dL/dt += g_depth r, dL/dcol = g_rgb r, dL/dm = g_normals r
//   weight: disk w = c (1 - s2/rr): dL/ds2 = -a c/rr, s2 = |e|^2 with e = t d - q, so dL/de = 2 dL/ds2 e,
//           dL/dt += dL/de . d, dL/dq = -dL/de; and t = (m.q)/(m.d): dL/dq += dL/dt m/(m.d),
//           dL/dm += -dL/dt e/(m.d); dL/dc = a (1 - s2/rr), dL/dr = a c 2 s2/(rr r).  One-pixel rows: w = c,
//           t = q.z, dL/dc = a.  Where w = W the row alone makes the pixel: out = v and a = g_weight.
__global__ void __launch_bounds__(kRB) k_blend_bwd_rows(BlendArgs a, BlendBwdArgs g) {
  __shared__ LiveCamera s_cam[kViews];
  __shared__ KInv s_kinv;
  __shared__ float s_red[kRB / 32][12];
  const int b = blockIdx.y;
  const int n = blockIdx.x * kRB + threadIdx.x;
  const bool live = n < a.counts[b];
  const int64_t P = (int64_t)a.ib.H * a.ib.W;
  float4 g0 = make_float4(0.f, 0.f, 0.f, 0.f), g1 = g0, col = g0;
  if (live) {
    g0 = __ldg(reinterpret_cast<const float4 *>(a.geo + ((int64_t)b * a.cap + n) * kGeoW));
    g1 = __ldg(reinterpret_cast<const float4 *>(a.geo + ((int64_t)b * a.cap + n) * kGeoW + 4));
    if (a.col) col = __ldg(reinterpret_cast<const float4 *>(a.col + ((int64_t)b * a.cap + n) * kColW));
  }
  const float cc = a.use_conf ? g1.z : 1.0f;
  if (threadIdx.x == 0) s_kinv = load_kinv(a.K + b * a.K_bstride);
  float dp[3] = {0.f, 0.f, 0.f}, dn[3] = {0.f, 0.f, 0.f}, dcol[3] = {0.f, 0.f, 0.f}, dcc = 0.f, drad = 0.f;
  for (int l0 = 0; l0 < a.L; l0 += kViews) {
    const int nv = min(kViews, a.L - l0);
    __syncthreads();
    load_view_cameras(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b, l0, nv);
    __syncthreads();
    for (int v = 0; v < nv; ++v) {
      float gq[3] = {0.f, 0.f, 0.f}, gm[3] = {0.f, 0.f, 0.f};  // this view's dL/dq, dL/dm (camera frame)
      const int64_t img = (int64_t)b * a.L + l0 + v;
      // one pixel of the footprint
      auto pixel = [&](int h, int w, bool centre) {
        const int64_t i = img * P + (int64_t)h * a.ib.W + w;
        const float Wp = __ldg(g.weight + i);
        if (Wp == 0.0f) return;
        Contribution c;
        if (!contribution(a, s_cam[v], s_kinv, g0, g1, h, w, centre, band_limit(__ldg(g.zf + i), a.band), c)) return;
        const float r = c.w / Wp;
        float acc = 0.f, gt = 0.f;
        if (g.g_depth) {
          const float gd = __ldg(g.g_depth + i);
          acc += gd * (c.t - __ldg(g.depth + i));
          gt = gd * r;
        }
        if (g.g_rgb) {
          const float cv[3] = {col.x, col.y, col.z};
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            const float gc = __ldg(g.g_rgb + i * 3 + j);
            acc += gc * (cv[j] - __ldg(g.rgb + i * 3 + j));
            dcol[j] += gc * r;
          }
        }
        if (g.g_normals) {
          const float mv[3] = {c.m.x, c.m.y, c.m.z};
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            const float gn = __ldg(g.g_normals + i * 3 + j);
            acc += gn * (mv[j] - __ldg(g.normals + i * 3 + j));
            gm[j] += gn * r;
          }
        }
        // a pixel whose whole weight is this row's shows v itself: (v - out) is then rounding only, and W may be tiny
        const float da = (c.w == Wp ? 0.0f : acc / Wp) + (g.g_weight ? __ldg(g.g_weight + i) : 0.0f);
        if (c.disk) {
          const float rr = g1.w * g1.w;
          const float gs2 = -(da * cc) / rr;
          const float e[3] = {c.t * c.ray.x - c.q.x, c.t * c.ray.y - c.q.y, c.t * c.ray.z - c.q.z};
          const float ge[3] = {2.0f * gs2 * e[0], 2.0f * gs2 * e[1], 2.0f * gs2 * e[2]};
          gt += dot3(ge[0], ge[1], ge[2], c.ray.x, c.ray.y, c.ray.z);
          const float s = gt / c.md;
          gq[0] += s * c.m.x - ge[0]; gq[1] += s * c.m.y - ge[1]; gq[2] += s * c.m.z - ge[2];
          gm[0] -= s * e[0]; gm[1] -= s * e[1]; gm[2] -= s * e[2];
          dcc += da * (1.0f - c.s2 / rr);
          drad += (da * cc) * (2.0f * c.s2) / (rr * g1.w);
        } else {
          gq[2] += gt;
          dcc += da;
        }
      };
      if (live) {
        if (a.M > 0 && is_disk(g0, g1)) {
          const Disk d = make_disk(s_cam[v], a.ib, a.M, g0, g1);
          for (int h = d.h0; h <= d.h1; ++h)
            for (int w = d.w0; w <= d.w1; ++w) pixel(h, w, false);
        } else {
          const PixelHit hit = project(s_cam[v], a.ib, g0.x, g0.y, g0.z);
          if (hit.in_frustum) pixel(hit.h, hit.w, true);
        }
      }
      const float *rt = s_cam[v].tinv.r;  // R^T of the camera-to-world pose
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        dp[j] += dot3(rt[j], rt[3 + j], rt[6 + j], gq[0], gq[1], gq[2]);
        dn[j] += dot3(rt[j], rt[3 + j], rt[6 + j], gm[0], gm[1], gm[2]);
      }
      if (g.pose_partials) {
        // dL/dR = (p - c) gq^T + n gm^T, dL/dc = -R gq, with R = rt^T and c = -R t' (t' = T^-1's translation)
        const float *tt = s_cam[v].tinv.t;
        float acc[12];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const float cr = -dot3(rt[r], rt[3 + r], rt[6 + r], tt[0], tt[1], tt[2]);
          const float pt = (r == 0 ? g0.x : r == 1 ? g0.y : g0.z) - cr;
          const float nw = r == 0 ? g0.w : r == 1 ? g1.x : g1.y;
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[r * 4 + c] = pt * gq[c] + nw * gm[c];
          acc[r * 4 + 3] = -dot3(rt[r], rt[3 + r], rt[6 + r], gq[0], gq[1], gq[2]);
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
          g.pose_partials[(img * gridDim.x + blockIdx.x) * 12 + threadIdx.x] = x;
        }
        __syncthreads();
      }
    }
  }
  if (n >= a.bound) return;
  const int64_t row = (int64_t)b * a.cap + n;
  if (g.d_geo) {
    float4 *o = reinterpret_cast<float4 *>(g.d_geo + row * kGeoW);
    o[0] = make_float4(dp[0], dp[1], dp[2], dn[0]);
    o[1] = make_float4(dn[1], dn[2], a.use_conf ? dcc : 0.f, drad);
  }
  if (g.d_col) reinterpret_cast<float4 *>(g.d_col + row * kColW)[0] = make_float4(dcol[0], dcol[1], dcol[2], 0.f);
}

// scratch of the blend forward: bucket starts (B*L*NB + 1), scan tile sums, and per item (b, n < bound, l) its key,
// its slot in the bucket and the bucket-ordered rows
struct BlendScratch {
  int *start, *tile_sum;
  unsigned int *key;
  int *rank, *rows;
  int64_t bytes;
};
inline BlendScratch blend_scratch(void *base, int64_t buckets, int64_t items) {
  Carver c(base);
  BlendScratch r;
  r.start = c.take<int>(buckets + 1);
  r.tile_sum = c.take<int>((buckets + 1 + kScanTile - 1) / kScanTile);
  r.key = c.take<unsigned int>(items);
  r.rank = c.take<int>(items);
  r.rows = c.take<int>(items);
  r.bytes = c.bytes;
  return r;
}

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace gsx

using namespace gsx;

// Buckets per view, (H + 2M)(W + 2M).
static int64_t blend_buckets(int H, int W, int M) { return (int64_t)(H + 2 * M) * (W + 2 * M); }

static int check_blend_extents(const char *fn, int B, int L, int H, int W, int64_t capacity, int64_t max_count,
                               int max_splat_px) {
  GSX_CHECK_ARG(B >= 1 && L >= 1 && H >= 1 && W >= 1, "%s: bad extents B=%d L=%d H=%d W=%d", fn, B, L, H, W);
  GSX_CHECK_ARG(max_splat_px >= 0 && max_splat_px <= GSX_MAX_SPLAT_PX, "%s: max_splat_px %d outside [0, %d]", fn,
                max_splat_px, GSX_MAX_SPLAT_PX);
  GSX_CHECK_ARG((int64_t)L * H * W <= INT32_MAX, "%s: L*H*W = %lld overflows", fn, (long long)L * H * W);
  GSX_CHECK_ARG((int64_t)B * L <= 65535, "%s: B*L = %lld views exceed one launch", fn, (long long)B * L);
  GSX_CHECK_ARG(capacity >= 0 && capacity <= INT32_MAX, "%s: bad capacity %lld", fn, (long long)capacity);
  GSX_CHECK_ARG(max_count >= 0 && max_count <= capacity, "%s: max_count %lld outside [0, capacity %lld]", fn,
                (long long)max_count, (long long)capacity);
  const int64_t buckets = (int64_t)B * L * blend_buckets(H, W, max_splat_px);
  GSX_CHECK_ARG(buckets < INT32_MAX && (int64_t)B * L * max_count < INT32_MAX,
                "%s: %lld buckets / %lld (row, view) pairs exceed 32-bit indexing", fn, (long long)buckets,
                (long long)B * L * max_count);
  return 0;
}

extern "C" int64_t gsx_render_blend_scratch_bytes(int B, int L, int H, int W, int64_t max_count, int max_splat_px) {
  if (B < 1 || L < 1 || H < 1 || W < 1 || max_count < 0 || max_splat_px < 0 || max_splat_px > GSX_MAX_SPLAT_PX)
    return -1;
  return blend_scratch(nullptr, (int64_t)B * L * blend_buckets(H, W, max_splat_px), (int64_t)B * L * max_count).bytes;
}

static BlendArgs blend_args(const float *geo, const float *col, const int32_t *counts, int64_t capacity,
                            int64_t max_count, const float *K, int64_t K_bstride, const float *poses,
                            int64_t pose_bstride, int L, int H, int W, int use_confidence, double band, int M) {
  return BlendArgs{geo, col, counts, capacity, (int)max_count, K, K_bstride, poses, pose_bstride, L, M,
                   image_bounds(H, W), W + 2 * M, blend_buckets(H, W, M), use_confidence ? 1 : 0, band};
}

extern "C" int gsx_render_blend(const float *map_geometry, const float *map_colors, const int32_t *counts,
                                int64_t capacity, int64_t max_count, const float *intrinsics, int64_t K_bstride,
                                const float *poses, int64_t pose_bstride, int B, int L, int H, int W,
                                int use_confidence, double blend_band, int max_splat_px, int64_t *index,
                                float *front_depth, float *weight, float *depth, float *rgb, float *normals,
                                void *scratch, int64_t scratch_bytes, void *stream) {
  if (check_blend_extents("gsx_render_blend", B, L, H, W, capacity, max_count, max_splat_px)) return 1;
  GSX_CHECK_ARG(blend_band >= 0.0, "gsx_render_blend: blend_band %g must be >= 0", blend_band);
  GSX_CHECK_ARG(intrinsics && poses && index && front_depth && weight && depth, "gsx_render_blend: null pointer");
  if (max_count > 0) GSX_CHECK_ARG(map_geometry && counts, "gsx_render_blend: null map pointer");
  if (max_count > 0 && rgb) GSX_CHECK_ARG(map_colors, "gsx_render_blend: rgb requested from a map without colours");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors), "gsx_render_blend: map rows must be 16-byte aligned");
  const int64_t need = gsx_render_blend_scratch_bytes(B, L, H, W, max_count, max_splat_px);
  GSX_CHECK_ARG(scratch && scratch_bytes >= need, "gsx_render_blend: scratch too small (%lld < %lld bytes)",
                (long long)scratch_bytes, (long long)need);
  // R1 / R1d and R2: the index image and the front depth z_f
  if (gsx_render_splats(map_geometry, nullptr, counts, capacity, max_count, intrinsics, K_bstride, poses, pose_bstride,
                        B, L, H, W, index, front_depth, nullptr, nullptr, nullptr, max_splat_px, stream))
    return 1;
  cudaStream_t s = (cudaStream_t)stream;
  const BlendArgs a = blend_args(map_geometry, map_colors, counts, capacity, max_count, intrinsics, K_bstride, poses,
                                 pose_bstride, L, H, W, use_confidence, blend_band, max_splat_px);
  const int64_t buckets = (int64_t)B * L * a.NB, items = (int64_t)B * L * max_count;
  const BlendScratch sc = blend_scratch(scratch, buckets, items);
  if (max_count > 0) {
    const unsigned invalid = (unsigned)buckets;
    cudaMemsetAsync(sc.start, 0, (size_t)(buckets + 1) * sizeof(int), s);
    const dim3 kgrid((unsigned)((max_count + kRB - 1) / kRB), (unsigned)B, (unsigned)((L + kViews - 1) / kViews));
    k_blend_key<<<kgrid, kRB, 0, s>>>(a, sc.key, sc.rank, sc.start, invalid);
    const unsigned tiles = (unsigned)((buckets + 1 + kScanTile - 1) / kScanTile);
    k_scan_reduce<<<tiles, kRB, 0, s>>>(sc.start, buckets + 1, sc.tile_sum);
    k_scan_tiles<<<1, kScanTop, 0, s>>>(sc.tile_sum, (int)tiles);
    k_scan_apply<<<tiles, kRB, 0, s>>>(sc.start, buckets + 1, sc.tile_sum);
    k_blend_place<<<(unsigned)((items + kRB - 1) / kRB), kRB, 0, s>>>(sc.key, sc.rank, sc.start, items,
                                                                      (int)max_count, L, invalid, sc.rows);
    k_blend_sort_buckets<<<(unsigned)((buckets + kRB - 1) / kRB), kRB, 0, s>>>(sc.start, buckets, sc.rows);
  }
  const dim3 pgrid((unsigned)(((int64_t)H * W + kRB - 1) / kRB), (unsigned)(B * L));
  // (no row: every index is -1 and the walk never reads the buckets)
  k_blend_resolve<<<pgrid, kRB, 0, s>>>(a, index, front_depth, sc.start, sc.rows, weight, depth,
                                        map_colors ? rgb : nullptr, normals);
  GSX_CHECK_LAUNCH("gsx_render_blend");
  return 0;
}

extern "C" int64_t gsx_render_blend_bwd_scratch_bytes(int B, int L, int64_t max_count) {
  if (B < 1 || L < 1 || max_count < 0) return -1;
  return (int64_t)B * L * ((max_count + kRB - 1) / kRB) * 12 * (int64_t)sizeof(float) + 256;
}

extern "C" int gsx_render_blend_bwd(const float *map_geometry, const float *map_colors, const int32_t *counts,
                                    int64_t capacity, int64_t max_count, const float *intrinsics, int64_t K_bstride,
                                    const float *poses, int64_t pose_bstride, int B, int L, int H, int W,
                                    int use_confidence, double blend_band, int max_splat_px, const float *front_depth,
                                    const float *weight, const float *depth, const float *rgb, const float *normals,
                                    const float *g_depth, const float *g_rgb, const float *g_normals,
                                    const float *g_weight, float *d_geometry, float *d_colors, float *d_poses,
                                    void *scratch, int64_t scratch_bytes, void *stream) {
  if (check_blend_extents("gsx_render_blend_bwd", B, L, H, W, capacity, max_count, max_splat_px)) return 1;
  GSX_CHECK_ARG(blend_band >= 0.0, "gsx_render_blend_bwd: blend_band %g must be >= 0", blend_band);
  GSX_CHECK_ARG(intrinsics && poses && front_depth && weight, "gsx_render_blend_bwd: null pointer");
  GSX_CHECK_ARG(!g_depth || depth, "gsx_render_blend_bwd: g_depth without the forward's depth");
  GSX_CHECK_ARG(!g_rgb || (rgb && map_colors), "gsx_render_blend_bwd: g_rgb without the forward's rgb and colours");
  GSX_CHECK_ARG(!g_normals || normals, "gsx_render_blend_bwd: g_normals without the forward's normals");
  if (capacity > 0 && (d_geometry || d_colors || d_poses))
    GSX_CHECK_ARG(map_geometry && counts, "gsx_render_blend_bwd: null map pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors) && aligned16(d_geometry) && aligned16(d_colors),
                "gsx_render_blend_bwd: map rows must be 16-byte aligned");
  if (d_poses)
    GSX_CHECK_ARG(scratch && scratch_bytes >= gsx_render_blend_bwd_scratch_bytes(B, L, max_count),
                  "gsx_render_blend_bwd: scratch too small");
  cudaStream_t s = (cudaStream_t)stream;
  if (d_geometry) cudaMemsetAsync(d_geometry, 0, (size_t)B * capacity * kGeoW * sizeof(float), s);
  if (d_colors) cudaMemsetAsync(d_colors, 0, (size_t)B * capacity * kColW * sizeof(float), s);
  const unsigned tiles = (unsigned)((max_count + kRB - 1) / kRB);
  float *partials = d_poses ? reinterpret_cast<float *>(scratch) : nullptr;
  if (tiles > 0 && (d_geometry || d_colors || d_poses)) {
    const BlendArgs a = blend_args(map_geometry, map_colors, counts, capacity, max_count, intrinsics, K_bstride, poses,
                                   pose_bstride, L, H, W, use_confidence, blend_band, max_splat_px);
    const BlendBwdArgs g{front_depth, weight, depth, rgb, normals, g_depth, g_rgb, g_normals, g_weight,
                         d_geometry, d_colors, partials};
    k_blend_bwd_rows<<<dim3(tiles, (unsigned)B), kRB, 0, s>>>(a, g);
  }
  if (d_poses) k_pose_grad_reduce<<<B * L, 16, 0, s>>>(partials, (int)tiles, d_poses, B * L);
  GSX_CHECK_LAUNCH("gsx_render_blend_bwd");
  return 0;
}
