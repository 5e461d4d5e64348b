// Per-surfel embeddings (ConceptFusion-style feature maps) fused beside the colours, for sm_90a.
//   k_embed_merge_append (KE)   after K4 (k_merge_append<kAssoc, kRadii, kEmbRec = true>): for every pixel K4 merged or
//                               appended (assoc != 0), the D channels of its map row.  A merged row n becomes
//                               ((c0 * E[n]) + (alpha * e[pix])) * inv with K4's own c0 and alpha (its record) and
//                               inv = 1 / (c0 + alpha, or 1 where that is 0): the colour merge's expression and operand
//                               order (fusionutils.py:678-699); an appended row is e[pix] (fusionutils.py:702-720).
//                               Rows no pixel touched are not written.  Each merged or appended row belongs to exactly one
//                               pixel, so there are no atomics.  Arithmetic in float32; a half-precision map is read by an
//                               exact upcast and every result is rounded once to the storage type (nearest even).
//   k_embed_bwd_rows / _pixels  the backward (float32 maps): d E_prev and d e, and per merged pixel the quotient rule's
//                               terms of d c0 and d alpha, which K4's backward (k_merge_bwd_pixels<true>) adds to its own.
//   upsampled KE                (k_embed_merge_append<T, V, kUp = true>) the frame's embedding image is coarser than the
//                               depth, (eh, ew) <= (H, W); each pixel samples it bilinearly (F.interpolate, bilinear,
//                               align_corners=False) in registers and merges or appends the unrounded sample.  Its
//                               backward: k_embed_bwd_pixels<true> (d E_prev of merged rows, d c0, d alpha; the sample
//                               recomputed) and k_embed_bwd_gather (d e of each coarse texel, summed over the pixels
//                               whose taps reach it, in a fixed order).  No (B, H, W, D) image exists on either pass.
// Several lanes work on one pixel: C = D / V consecutive threads take V channels each, with 16-byte accesses when the
// channel count and the base pointers allow (V = 16 / sizeof(T)), one channel per thread otherwise.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "gsx_embed.cuh"
#include "../../include/gsx.h"

namespace gsx {

__device__ __forceinline__ float to_f32(float x) { return x; }
__device__ __forceinline__ float to_f32(__half x) { return __half2float(x); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 x) { return __bfloat162float(x); }
template <typename T> __device__ __forceinline__ T from_f32(float x);
template <> __device__ __forceinline__ float from_f32<float>(float x) { return x; }
template <> __device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

// V channels of T as one access: 16 bytes (V = 16 / sizeof(T)) or one element (V = 1)
template <typename T, int V>
struct Chunk {
  T v[V];
};
template <typename T, int V>
__device__ __forceinline__ Chunk<T, V> load_chunk(const T *p) {
  Chunk<T, V> c;
  if constexpr (V * sizeof(T) == 16)
    *reinterpret_cast<uint4 *>(c.v) = *reinterpret_cast<const uint4 *>(p);
  else
    c.v[0] = *p;
  return c;
}
template <typename T, int V>
__device__ __forceinline__ void store_chunk(T *p, const Chunk<T, V> &c) {
  if constexpr (V * sizeof(T) == 16)
    *reinterpret_cast<uint4 *>(p) = *reinterpret_cast<const uint4 *>(c.v);
  else
    *p = c.v[0];
}

// One axis of F.interpolate(mode='bilinear', align_corners=False) from m coarse to n fine samples: fine index i reads
// the coarse taps i0, i1 with weights l0, l1.  Each operation is rounded separately (-fmad=false), as the oracle
// (tests/embedding_upsample_oracle.py) states it.  i0 is non-decreasing in i.
struct Taps {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Taps bilinear_taps(int i, int n, int m) {
  const float scale = (float)m / (float)n;
  float s = scale * ((float)i + 0.5f) - 0.5f;
  if (s < 0.0f) s = 0.0f;
  Taps t;
  t.i0 = (int)s;
  t.i1 = t.i0 + (t.i0 < m - 1 ? 1 : 0);
  t.l1 = s - (float)t.i0;
  t.l0 = 1.0f - t.l1;
  return t;
}

// the bilinear sample f of pixel (v, u) at channels [k0, k0 + V) of a coarse (eh, ew, D) image e, in float32:
// f = ly0 * (lx0 * e[y0,x0] + lx1 * e[y0,x1]) + ly1 * (lx0 * e[y1,x0] + lx1 * e[y1,x1])
template <typename T, int V>
__device__ __forceinline__ void sample_bilinear(const T *e, const Taps &ty, const Taps &tx, int ew, int D, int k0,
                                                float (&f)[V]) {
  const Chunk<T, V> e00 = load_chunk<T, V>(e + ((int64_t)ty.i0 * ew + tx.i0) * D + k0);
  const Chunk<T, V> e01 = load_chunk<T, V>(e + ((int64_t)ty.i0 * ew + tx.i1) * D + k0);
  const Chunk<T, V> e10 = load_chunk<T, V>(e + ((int64_t)ty.i1 * ew + tx.i0) * D + k0);
  const Chunk<T, V> e11 = load_chunk<T, V>(e + ((int64_t)ty.i1 * ew + tx.i1) * D + k0);
#pragma unroll
  for (int k = 0; k < V; ++k)
    f[k] = ty.l0 * (tx.l0 * to_f32(e00.v[k]) + tx.l1 * to_f32(e01.v[k])) +
           ty.l1 * (tx.l0 * to_f32(e10.v[k]) + tx.l1 * to_f32(e11.v[k]));
}

// kUp: the frame is a coarse (eh, ew) image; each thread samples its pixel's four texels (V channels each) and merges
// or appends the sample f, unrounded, by the same rule.  No full-resolution image is formed.
template <typename T, int V, bool kUp = false>
__global__ void __launch_bounds__(256) k_embed_merge_append(EmbedArgs a) {
  const int b = blockIdx.y;
  const int C = a.D / V;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)a.P * C) return;
  const int pix = (int)(i / C), c = (int)(i - (int64_t)pix * C);
  const int32_t as = __ldg(a.assoc + (int64_t)b * a.P + pix);
  if (as == 0) return;
  const int64_t n = (as > 0) ? (int64_t)as - 1 : -(int64_t)as - 1;
  if (n >= a.cap) return;  // (K4 never records a row past capacity: it flags the overflow instead)
  if constexpr (kUp) {
    const int v = pix / a.W, u = pix - v * a.W;
    float f[V];
    sample_bilinear<T, V>(reinterpret_cast<const T *>(a.e) + b * a.e_bstride, bilinear_taps(v, a.H, a.eh),
                          bilinear_taps(u, a.W, a.ew), a.ew, a.D, c * V, f);
    T *dst = reinterpret_cast<T *>(a.E) + ((int64_t)b * a.cap + n) * a.D + c * V;
    if (as < 0) {
      const float2 r = __ldg(a.rec + (int64_t)b * a.P + pix);
      const float c0 = r.x, alpha = r.y;
      const float tot = c0 + alpha;
      const float inv = 1.0f / ((tot == 0.0f) ? 1.0f : tot);
      const Chunk<T, V> m = load_chunk<T, V>(dst);
#pragma unroll
      for (int k = 0; k < V; ++k) f[k] = ((c0 * to_f32(m.v[k])) + (alpha * f[k])) * inv;
    }
    Chunk<T, V> o;
#pragma unroll
    for (int k = 0; k < V; ++k) o.v[k] = from_f32<T>(f[k]);
    store_chunk<T, V>(dst, o);
    return;
  }
  const T *src = reinterpret_cast<const T *>(a.e) + b * a.e_bstride + (int64_t)pix * a.D + c * V;
  T *dst = reinterpret_cast<T *>(a.E) + ((int64_t)b * a.cap + n) * a.D + c * V;
  Chunk<T, V> f = load_chunk<T, V>(src);
  if (as < 0) {
    const float2 r = __ldg(a.rec + (int64_t)b * a.P + pix);
    const float c0 = r.x, alpha = r.y;
    const float tot = c0 + alpha;
    const float inv = 1.0f / ((tot == 0.0f) ? 1.0f : tot);
    const Chunk<T, V> m = load_chunk<T, V>(dst);
#pragma unroll
    for (int k = 0; k < V; ++k) f.v[k] = from_f32<T>(((c0 * to_f32(m.v[k])) + (alpha * to_f32(f.v[k]))) * inv);
  }
  store_chunk<T, V>(dst, f);
}

template <typename T, bool kUp>
static int launch_embed_typed(const EmbedArgs &a, bool vec, cudaStream_t st) {
  constexpr int V = 16 / (int)sizeof(T);
  const int C = vec ? a.D / V : a.D;
  const int64_t blocks = ((int64_t)a.P * C + 255) / 256;
  const dim3 grid((unsigned)blocks, (unsigned)a.B);
  if (vec)
    k_embed_merge_append<T, V, kUp><<<grid, 256, 0, st>>>(a);
  else
    k_embed_merge_append<T, 1, kUp><<<grid, 256, 0, st>>>(a);
  GSX_CHECK_LAUNCH(kUp ? "gsx_embed_merge_append_upsampled" : "gsx_embed_merge_append");
  return 0;
}

template <typename T>
static int launch_embed_typed(const EmbedArgs &a, bool vec, cudaStream_t st) {
  return a.eh > 0 ? launch_embed_typed<T, true>(a, vec, st) : launch_embed_typed<T, false>(a, vec, st);
}

static int elem_bytes(int dtype) { return dtype == 0 ? 4 : 2; }

int launch_embed_merge_append(const EmbedArgs &a, int dtype, cudaStream_t st) {
  if (a.B == 0 || a.P == 0) return 0;
  const int s = elem_bytes(dtype), V = 16 / s;
  const bool vec = a.D % V == 0 && a.e_bstride % V == 0 &&
                   ((reinterpret_cast<uintptr_t>(a.E) | reinterpret_cast<uintptr_t>(a.e)) & 15) == 0;
  if (dtype == 0) return launch_embed_typed<float>(a, vec, st);
  if (dtype == 1) return launch_embed_typed<__half>(a, vec, st);
  return launch_embed_typed<__nv_bfloat16>(a, vec, st);
}

// ---- backward (float32) -------------------------------------------------------------------------------------
//   merged   out = (c0 E + alpha e) inv   =>  d E = g c0 inv,  d e = g alpha inv,
//            d c0 = sum_d g (E inv - num inv^2),  d alpha = sum_d g (e inv - num inv^2)   (num = c0 E + alpha e)
//   appended out = e                      =>  d e = g
//   untouched rows pass g through; rows at or past counts_in (and padding) get 0.
struct EmbedBwdArgs {
  const int32_t *assoc;
  const float2 *rec;
  const int32_t *counts_in;
  const float *E;  // (B, cap_in, D) pre-merge map embeddings
  int64_t cap_in;
  const float *e;  // (B, P, D) frame embeddings
  const float *g;  // (B, cap_out, D) upstream gradient, or null = zero
  int64_t cap_out;
  int B, P, D;
  float *dE, *de, *dc0, *dalpha;
  // upsampled KE only: e and de are coarse (B, eh, ew, D) images sampled at the (H, W) pixels
  int H, W, eh, ew;
};

__global__ void __launch_bounds__(256) k_embed_bwd_rows(EmbedBwdArgs a) {
  const int b = blockIdx.y;
  const int64_t total = a.cap_in * a.D;
  const int cnt = a.counts_in[b];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / a.D;
    const bool live = a.g && n < cnt && n < a.cap_out;
    a.dE[(int64_t)b * total + i] = live ? a.g[((int64_t)b * a.cap_out + n) * a.D + (i - n * a.D)] : 0.0f;
  }
}

// one warp per pixel: lane l takes channels l, l + 32, ... and the weight terms are summed per lane in that order, then
// across the lanes by a fixed butterfly, so the result does not depend on scheduling.
// kUp: the frame is a coarse image; f is re-sampled from its taps and d e is left to k_embed_bwd_gather.
template <bool kUp = false>
__global__ void __launch_bounds__(256) k_embed_bwd_pixels(EmbedBwdArgs a) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (pix >= a.P) return;
  const int64_t pi = (int64_t)b * a.P + pix;
  const int32_t as = a.assoc[pi];
  float *de = kUp ? nullptr : a.de + pi * a.D;
  float dc0 = 0.0f, dal = 0.0f;
  if (as == 0 || !a.g) {
    if constexpr (!kUp)
      for (int d = lane; d < a.D; d += 32) de[d] = 0.0f;
  } else {
    const int64_t n = (as > 0) ? (int64_t)as - 1 : -(int64_t)as - 1;
    const float *g = a.g + ((int64_t)b * a.cap_out + n) * a.D;
    if (as > 0) {
      if constexpr (!kUp)
        for (int d = lane; d < a.D; d += 32) de[d] = g[d];
    } else if constexpr (kUp) {
      const float2 r = a.rec[pi];
      const float c0 = r.x, alpha = r.y;
      const float tot = c0 + alpha;
      const bool degenerate = tot == 0.0f;
      const float inv = 1.0f / (degenerate ? 1.0f : tot);
      const float dinv = degenerate ? 0.0f : -(inv * inv);
      const float *E = a.E + ((int64_t)b * a.cap_in + n) * a.D;
      const float *e = a.e + (int64_t)b * a.eh * a.ew * a.D;
      const int v = pix / a.W, u = pix - v * a.W;
      const Taps ty = bilinear_taps(v, a.H, a.eh), tx = bilinear_taps(u, a.W, a.ew);
      float *dE = a.dE + ((int64_t)b * a.cap_in + n) * a.D;
      for (int d = lane; d < a.D; d += 32) {
        float f[1];
        sample_bilinear<float, 1>(e, ty, tx, a.ew, a.D, d, f);
        const float gd = g[d], m = E[d];
        const float num = c0 * m + alpha * f[0];
        dE[d] = gd * c0 * inv;
        dc0 += gd * (m * inv + num * dinv);
        dal += gd * (f[0] * inv + num * dinv);
      }
    } else {
      const float2 r = a.rec[pi];
      const float c0 = r.x, alpha = r.y;
      const float tot = c0 + alpha;
      const bool degenerate = tot == 0.0f;
      const float inv = 1.0f / (degenerate ? 1.0f : tot);
      const float dinv = degenerate ? 0.0f : -(inv * inv);
      const float *E = a.E + ((int64_t)b * a.cap_in + n) * a.D;
      const float *e = a.e + pi * a.D;
      float *dE = a.dE + ((int64_t)b * a.cap_in + n) * a.D;
      for (int d = lane; d < a.D; d += 32) {
        const float gd = g[d], m = E[d], f = e[d];
        const float num = c0 * m + alpha * f;
        dE[d] = gd * c0 * inv;
        de[d] = gd * alpha * inv;
        dc0 += gd * (m * inv + num * dinv);
        dal += gd * (f * inv + num * dinv);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dc0 += __shfl_xor_sync(0xffffffffu, dc0, o);
    dal += __shfl_xor_sync(0xffffffffu, dal, o);
  }
  if (lane == 0) {
    a.dc0[pi] = dc0;
    a.dalpha[pi] = dal;
  }
}

// the first fine index i in [0, n] whose tap i0 (of bilinear_taps(i, n, m)) is >= t: i0 is non-decreasing in i
__device__ __forceinline__ int first_fine(int t, int n, int m) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (bilinear_taps(mid, n, m).i0 >= t)
      hi = mid;
    else
      lo = mid + 1;
  }
  return lo;
}

// d e of the upsampled KE, (B, eh, ew, D), without atomics: one thread per coarse texel t and V channels.  A pixel's
// taps reach t only if its i0 is t - 1 or t along both axes, a contiguous range of rows and of columns; the thread walks
// it row by row and adds, for every merged or appended pixel p and every tap k of p on t in the order 00, 01, 10, 11,
// w_k(p) * d f(p) with w_00 = ly0 * lx0 and so on and d f = g * alpha * inv (merged) or g (appended).  A fixed order, so
// two runs give the same bits.
template <int V>
__global__ void __launch_bounds__(256) k_embed_bwd_gather(EmbedBwdArgs a) {
  const int b = blockIdx.y;
  const int C = a.D / V;
  const int T = a.eh * a.ew;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)T * C) return;
  const int t = (int)(i / C), c = (int)(i - (int64_t)t * C);
  const int ty = t / a.ew, tx = t - ty * a.ew;
  float acc[V];
#pragma unroll
  for (int k = 0; k < V; ++k) acc[k] = 0.0f;
  if (a.g) {
    const int v0 = first_fine(ty - 1, a.H, a.eh), v1 = first_fine(ty + 1, a.H, a.eh);
    const int u0 = first_fine(tx - 1, a.W, a.ew), u1 = first_fine(tx + 1, a.W, a.ew);
    for (int v = v0; v < v1; ++v) {
      const Taps y = bilinear_taps(v, a.H, a.eh);
      for (int u = u0; u < u1; ++u) {
        const int64_t pi = (int64_t)b * a.P + (int64_t)v * a.W + u;
        const int32_t as = __ldg(a.assoc + pi);
        if (as == 0) continue;
        const int64_t n = (as > 0) ? (int64_t)as - 1 : -(int64_t)as - 1;
        const Chunk<float, V> gc = load_chunk<float, V>(a.g + ((int64_t)b * a.cap_out + n) * a.D + c * V);
        float df[V];
        if (as < 0) {
          const float2 r = __ldg(a.rec + pi);
          const float c0 = r.x, alpha = r.y;
          const float tot = c0 + alpha;
          const float inv = 1.0f / ((tot == 0.0f) ? 1.0f : tot);
#pragma unroll
          for (int k = 0; k < V; ++k) df[k] = gc.v[k] * alpha * inv;
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) df[k] = gc.v[k];
        }
        const Taps x = bilinear_taps(u, a.W, a.ew);
        const float w[4] = {y.l0 * x.l0, y.l0 * x.l1, y.l1 * x.l0, y.l1 * x.l1};
        const bool hit[4] = {y.i0 == ty && x.i0 == tx, y.i0 == ty && x.i1 == tx, y.i1 == ty && x.i0 == tx,
                             y.i1 == ty && x.i1 == tx};
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (hit[q]) {
#pragma unroll
            for (int k = 0; k < V; ++k) acc[k] += w[q] * df[k];
          }
      }
    }
  }
  Chunk<float, V> o;
#pragma unroll
  for (int k = 0; k < V; ++k) o.v[k] = acc[k];
  store_chunk<float, V>(a.de + ((int64_t)b * T + t) * a.D + c * V, o);
}

}  // namespace gsx

using namespace gsx;

static bool aligned_to(const void *p, uintptr_t n) { return (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; }

extern "C" int gsx_embed_merge_append(void *map_embeddings, int64_t capacity, const void *frame_embeddings,
                                      int64_t frame_bstride, const int32_t *assoc, const float *merge_rec, int B, int H,
                                      int W, int D, int dtype, void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2 && D >= 1, "gsx_embed_merge_append: bad extents B=%d H=%d W=%d D=%d", B,
                H, W, D);
  GSX_CHECK_ARG(dtype >= 0 && dtype <= 2, "gsx_embed_merge_append: dtype must be 0 (float32), 1 (float16) or "
                "2 (bfloat16), not %d", dtype);
  GSX_CHECK_ARG(capacity >= 0 && frame_bstride >= (int64_t)H * W * D,
                "gsx_embed_merge_append: bad capacity or frame element stride");
  if (B == 0) return 0;
  GSX_CHECK_ARG(map_embeddings && frame_embeddings && assoc && merge_rec, "gsx_embed_merge_append: null pointer");
  const uintptr_t s = (uintptr_t)elem_bytes(dtype);
  GSX_CHECK_ARG(aligned_to(map_embeddings, s) && aligned_to(frame_embeddings, s) && aligned_to(merge_rec, 8),
                "gsx_embed_merge_append: misaligned embeddings or record");
  const EmbedArgs a{map_embeddings, frame_embeddings, frame_bstride, assoc, reinterpret_cast<const float2 *>(merge_rec),
                    capacity, B, H * W, D};
  return launch_embed_merge_append(a, dtype, (cudaStream_t)stream);
}

extern "C" int gsx_embed_merge_bwd(const int32_t *assoc, const float *merge_rec, const int32_t *counts_in,
                                   const float *map_embeddings, int64_t capacity_in, const float *frame_embeddings,
                                   const float *g_embeddings, int64_t capacity_out, int B, int H, int W, int D,
                                   float *d_map_embeddings, float *d_frame_embeddings, float *d_c0, float *d_alpha,
                                   void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2 && D >= 1, "gsx_embed_merge_bwd: bad extents B=%d H=%d W=%d D=%d", B, H, W,
                D);
  GSX_CHECK_ARG(capacity_in >= 0 && capacity_out >= 0, "gsx_embed_merge_bwd: negative capacity");
  if (B == 0) return 0;
  GSX_CHECK_ARG(assoc && merge_rec && counts_in && frame_embeddings && d_frame_embeddings && d_c0 && d_alpha,
                "gsx_embed_merge_bwd: null pointer");
  GSX_CHECK_ARG(capacity_in == 0 || (map_embeddings && d_map_embeddings), "gsx_embed_merge_bwd: null map pointer");
  GSX_CHECK_ARG(aligned_to(merge_rec, 8), "gsx_embed_merge_bwd: merge_rec must be 8-byte aligned");
  const int P = H * W;
  const EmbedBwdArgs a{assoc, reinterpret_cast<const float2 *>(merge_rec), counts_in, map_embeddings, capacity_in,
                       frame_embeddings, g_embeddings, capacity_out, B, P, D, d_map_embeddings, d_frame_embeddings,
                       d_c0, d_alpha};
  cudaStream_t st = (cudaStream_t)stream;
  if (capacity_in > 0) {
    const int64_t blocks = std::min<int64_t>((capacity_in * D + 255) / 256, 65535);
    k_embed_bwd_rows<<<dim3((unsigned)blocks, (unsigned)B), 256, 0, st>>>(a);
    GSX_CHECK_LAUNCH("gsx_embed_merge_bwd(rows)");
  }
  k_embed_bwd_pixels<false><<<dim3((unsigned)((P + 7) / 8), (unsigned)B), 256, 0, st>>>(a);
  GSX_CHECK_LAUNCH("gsx_embed_merge_bwd(pixels)");
  return 0;
}

extern "C" int gsx_embed_merge_append_upsampled(void *map_embeddings, int64_t capacity, const void *frame_embeddings,
                                                int64_t frame_bstride, const int32_t *assoc, const float *merge_rec,
                                                int B, int H, int W, int eh, int ew, int D, int dtype, void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2 && D >= 1,
                "gsx_embed_merge_append_upsampled: bad extents B=%d H=%d W=%d D=%d", B, H, W, D);
  GSX_CHECK_ARG(eh >= 1 && eh <= H && ew >= 1 && ew <= W,
                "gsx_embed_merge_append_upsampled: the embedding image (%d, %d) must be at most (H, W) = (%d, %d) and "
                "at least (1, 1)", eh, ew, H, W);
  GSX_CHECK_ARG(dtype >= 0 && dtype <= 2, "gsx_embed_merge_append_upsampled: dtype must be 0 (float32), 1 (float16) "
                "or 2 (bfloat16), not %d", dtype);
  GSX_CHECK_ARG(capacity >= 0 && frame_bstride >= (int64_t)eh * ew * D,
                "gsx_embed_merge_append_upsampled: bad capacity or frame element stride");
  if (B == 0) return 0;
  GSX_CHECK_ARG(map_embeddings && frame_embeddings && assoc && merge_rec,
                "gsx_embed_merge_append_upsampled: null pointer");
  const uintptr_t s = (uintptr_t)elem_bytes(dtype);
  GSX_CHECK_ARG(aligned_to(map_embeddings, s) && aligned_to(frame_embeddings, s) && aligned_to(assoc, 4) &&
                aligned_to(merge_rec, 8), "gsx_embed_merge_append_upsampled: misaligned embeddings, assoc or record");
  const EmbedArgs a{map_embeddings, frame_embeddings, frame_bstride, assoc, reinterpret_cast<const float2 *>(merge_rec),
                    capacity, B, H * W, D, H, W, eh, ew};
  return launch_embed_merge_append(a, dtype, (cudaStream_t)stream);
}

extern "C" int gsx_embed_merge_bwd_upsampled(const int32_t *assoc, const float *merge_rec, const int32_t *counts_in,
                                             const float *map_embeddings, int64_t capacity_in,
                                             const float *frame_embeddings, const float *g_embeddings,
                                             int64_t capacity_out, int B, int H, int W, int eh, int ew, int D,
                                             float *d_map_embeddings, float *d_frame_embeddings, float *d_c0,
                                             float *d_alpha, void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2 && D >= 1,
                "gsx_embed_merge_bwd_upsampled: bad extents B=%d H=%d W=%d D=%d", B, H, W, D);
  GSX_CHECK_ARG(eh >= 1 && eh <= H && ew >= 1 && ew <= W,
                "gsx_embed_merge_bwd_upsampled: the embedding image (%d, %d) must be at most (H, W) = (%d, %d) and "
                "at least (1, 1)", eh, ew, H, W);
  GSX_CHECK_ARG(capacity_in >= 0 && capacity_out >= 0, "gsx_embed_merge_bwd_upsampled: negative capacity");
  if (B == 0) return 0;
  GSX_CHECK_ARG(assoc && merge_rec && counts_in && frame_embeddings && d_frame_embeddings && d_c0 && d_alpha,
                "gsx_embed_merge_bwd_upsampled: null pointer");
  GSX_CHECK_ARG(capacity_in == 0 || (map_embeddings && d_map_embeddings),
                "gsx_embed_merge_bwd_upsampled: null map pointer");
  GSX_CHECK_ARG(aligned_to(assoc, 4) && aligned_to(merge_rec, 8) && aligned_to(counts_in, 4) &&
                aligned_to(map_embeddings, 4) && aligned_to(frame_embeddings, 4) && aligned_to(g_embeddings, 4) &&
                aligned_to(d_map_embeddings, 4) && aligned_to(d_frame_embeddings, 4) && aligned_to(d_c0, 4) &&
                aligned_to(d_alpha, 4), "gsx_embed_merge_bwd_upsampled: misaligned embeddings, record or output");
  const int P = H * W;
  const EmbedBwdArgs a{assoc, reinterpret_cast<const float2 *>(merge_rec), counts_in, map_embeddings, capacity_in,
                       frame_embeddings, g_embeddings, capacity_out, B, P, D, d_map_embeddings, d_frame_embeddings,
                       d_c0, d_alpha, H, W, eh, ew};
  cudaStream_t st = (cudaStream_t)stream;
  if (capacity_in > 0) {
    const int64_t blocks = std::min<int64_t>((capacity_in * D + 255) / 256, 65535);
    k_embed_bwd_rows<<<dim3((unsigned)blocks, (unsigned)B), 256, 0, st>>>(a);
    GSX_CHECK_LAUNCH("gsx_embed_merge_bwd_upsampled(rows)");
  }
  k_embed_bwd_pixels<true><<<dim3((unsigned)((P + 7) / 8), (unsigned)B), 256, 0, st>>>(a);
  GSX_CHECK_LAUNCH("gsx_embed_merge_bwd_upsampled(pixels)");
  // 16-byte chunks of the gradient rows and of d e when D and both pointers allow
  const bool vec = D % 4 == 0 && aligned_to(d_frame_embeddings, 16) && (!g_embeddings || aligned_to(g_embeddings, 16));
  const int C = vec ? D / 4 : D;
  const dim3 grid((unsigned)(((int64_t)eh * ew * C + 255) / 256), (unsigned)B);
  if (vec)
    k_embed_bwd_gather<4><<<grid, 256, 0, st>>>(a);
  else
    k_embed_bwd_gather<1><<<grid, 256, 0, st>>>(a);
  GSX_CHECK_LAUNCH("gsx_embed_merge_bwd_upsampled(gather)");
  return 0;
}
