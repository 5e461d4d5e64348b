// Table-returning variants of the data-association steps, kept for API parity with gradslam's module-level
// helpers (find_active_map_points / find_similar_map_points / find_best_unique_correspondences / fuse_with_map,
// gradslam/slam/fusionutils.py:198-722).  They evaluate exactly the same device functions as the fused kernels
// (gsx_fusion.cu) but materialise flags / per-pixel winners so the host can hand out int64 (N,4) tables.
//   k_active_eval        per map slot (b,n): frustum test + pixel                       -> flag, h, w
//   k_similar_eval       per table row: distance + normal test against the frame maps  -> flag
//   k_unique_select      per table row: arg-min per pixel (same key and device functions as K2/K3)
//   k_unique_emit        per pixel: winner present? which n?                            -> flag, n   (and clears)
//   k_records_from_table per table row: store the row as the pixel's winner (input of K4 for fuse_with_map)
//   k_compact            generic stable compaction flag[] -> ascending indices (single-pass decoupled look-back)
#include "gsx_common.cuh"
#include "gsx_fusion_ws.cuh"
#include "gsx_thresholds.h"
#include "../../include/gsx.h"

namespace gsx {

constexpr int kTB = 256;

// ---- generic stable compaction ------------------------------------------------------------------------------
struct CompactArgs {
  const uint8_t *flags;
  int64_t n;
  int64_t *out_idx;
  int64_t *out_count;
  unsigned long long *state;  // (tiles) look-back tile states
  unsigned int *ticket;       // (1)
  int tiles;
  unsigned int epoch;
};

__global__ void __launch_bounds__(kTB) k_compact(CompactArgs a) {
  __shared__ int s_tile, s_excl;
  __shared__ int s_warp[4][kTB / 32];
  if (threadIdx.x == 0) s_tile = draw_tile_ticket(a.ticket, a.tiles);
  __syncthreads();
  const int tile = s_tile;
  int64_t i[4];
  bool f[4];
  int off[4];
  const int total = block_offsets<kTB, 4>(
      [&](int j) {
        i[j] = (int64_t)tile * (kTB * 4) + j * kTB + threadIdx.x;
        f[j] = (i[j] < a.n) && (a.flags[i[j]] != 0);
        return f[j];
      },
      off, s_warp, [] {});
  if (threadIdx.x == 0) publish_tile(a.state, tile, a.tiles, a.epoch, kTileAggregate, (unsigned)total);
  if (threadIdx.x < 32) {
    const unsigned int excl = lookback_warp(a.state, tile, a.tiles, a.epoch, (unsigned)total);
    if (threadIdx.x == 0) s_excl = (int)excl;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (f[j]) a.out_idx[(int64_t)s_excl + off[j]] = i[j];
  if (tile == a.tiles - 1 && threadIdx.x == 0) *a.out_count = (int64_t)s_excl + total;
}

// ---- find_active_map_points ---------------------------------------------------------------------------------
struct ActiveArgs {
  const float *geo;
  const int32_t *counts;
  int64_t cap;
  int64_t width;  // slots per element in the flag arrays (host upper bound of the sizes)
  const float *poses;
  int64_t pose_bstride;
  const float *K;
  int64_t K_bstride;
  ImageBounds ib;
  uint8_t *flags;  // (B, width)
  int32_t *hw;     // (B, width)  h * W + w
};

__global__ void __launch_bounds__(kTB) k_active_eval(ActiveArgs a) {
  __shared__ LiveCamera s_cam;
  const int b = blockIdx.y;
  load_live_camera(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b);
  __syncthreads();
  const int64_t n = (int64_t)blockIdx.x * kTB + threadIdx.x;
  if (n >= a.width) return;
  bool live = n < a.counts[b];
  int pix = 0;
  if (live) {
    const float4 p = __ldg(reinterpret_cast<const float4 *>(a.geo + ((int64_t)b * a.cap + n) * kGeoW));
    const PixelHit hit = project(s_cam, a.ib, p.x, p.y, p.z);
    live = hit.in_frustum;
    pix = hit.h * a.ib.W + hit.w;
  }
  a.flags[(int64_t)b * a.width + n] = live ? 1 : 0;
  a.hw[(int64_t)b * a.width + n] = pix;
}

// ---- rows of an int64 (R,4) table [b, n, h, w] ----------------------------------------------------------------
struct RowArgs {
  const int64_t *table;
  int64_t rows;
  const float *geo;  // (B,cap,8) packed geometry rows
  int64_t cap;
  const float *gv, *gn;  // (B,H,W,3)
  int B, H, W;
  float d2_max, dot_th;  // sqrtf(d2) < dist_th  <=>  d2 <= d2_max (gsx_thresholds.h)
  uint8_t *flags;  // (rows)            k_similar_eval
  unsigned int *win;  // (B,H,W) arg-min slots: k_unique_select / k_records_from_table
};

__device__ __forceinline__ bool row_ok(const RowArgs &a, int64_t b, int64_t n, int64_t h, int64_t w) {
  return b >= 0 && b < a.B && n >= 0 && n < a.cap && h >= 0 && h < a.H && w >= 0 && w < a.W;
}

__global__ void __launch_bounds__(kTB) k_similar_eval(RowArgs a) {
  const int64_t r = (int64_t)blockIdx.x * kTB + threadIdx.x;
  if (r >= a.rows) return;
  const int64_t b = a.table[r * 4], n = a.table[r * 4 + 1], h = a.table[r * 4 + 2], w = a.table[r * 4 + 3];
  bool ok = row_ok(a, b, n, h, w);
  if (ok) {
    const float *p = a.geo + (b * a.cap + n) * kGeoW;
    const float *m = p + 3;
    const float *g = a.gv + ((b * a.H + h) * a.W + w) * 3;
    const float *q = a.gn + ((b * a.H + h) * a.W + w) * 3;
    const float dx = __ldg(g) - __ldg(p), dy = __ldg(g + 1) - __ldg(p + 1), dz = __ldg(g + 2) - __ldg(p + 2);
    const float d2 = (dx * dx + dy * dy) + dz * dz;
    const float dot = (__ldg(q) * __ldg(m) + __ldg(q + 1) * __ldg(m + 1)) + __ldg(q + 2) * __ldg(m + 2);
    ok = (d2 <= a.d2_max) && (dot > a.dot_th);
  }
  a.flags[r] = ok ? 1 : 0;
}

__global__ void __launch_bounds__(kTB) k_unique_select(RowArgs a) {
  const int64_t r = (int64_t)blockIdx.x * kTB + threadIdx.x;
  if (r >= a.rows) return;
  const int64_t b = a.table[r * 4], n = a.table[r * 4 + 1], h = a.table[r * 4 + 2], w = a.table[r * 4 + 3];
  if (!row_ok(a, b, n, h, w)) return;
  const float *geo = a.geo + b * a.cap * kGeoW, *p = geo + n * kGeoW;
  const float *g = a.gv + ((b * a.H + h) * a.W + w) * 3;
  const float3 fv = make_float3(__ldg(g), __ldg(g + 1), __ldg(g + 2));
  const unsigned long long key = argmin_key_hi(__ldg(p + 6), ray_d2(fv, __ldg(p), __ldg(p + 1), __ldg(p + 2)));
  unsigned int *slot = a.win + (b * a.H + h) * a.W + w;
  argmin_settle(slot, (unsigned int)n, key, fv, geo, argmin_claim(slot, (unsigned int)n));
}

__global__ void __launch_bounds__(kTB) k_records_from_table(RowArgs a) {
  const int64_t r = (int64_t)blockIdx.x * kTB + threadIdx.x;
  if (r >= a.rows) return;
  const int64_t b = a.table[r * 4], n = a.table[r * 4 + 1], h = a.table[r * 4 + 2], w = a.table[r * 4 + 3];
  if (!row_ok(a, b, n, h, w)) return;
  a.win[(b * a.H + h) * a.W + w] = (unsigned int)n + 1u;
}

// per pixel: is there a winner?  which map row?
__global__ void __launch_bounds__(kTB) k_unique_emit(const unsigned int *win, int64_t pixels, uint8_t *flags,
                                                     int64_t *n_out) {
  const int64_t i = (int64_t)blockIdx.x * kTB + threadIdx.x;
  if (i >= pixels) return;
  const unsigned int v = win[i];
  flags[i] = v != 0u ? 1 : 0;
  n_out[i] = (int64_t)v - 1;
}

}  // namespace gsx

using namespace gsx;

static inline int64_t tb_blocks(int64_t n) { return (n + kTB - 1) / kTB; }

extern "C" int64_t gsx_compact_scratch_bytes(int64_t n) {
  if (n < 0) return -1;
  const int64_t tiles = (n + kTB * 4 - 1) / (kTB * 4);
  return (tiles + 1) * 8 + 256;
}

extern "C" int gsx_compact_indices(const uint8_t *flags, int64_t n, int64_t *out_idx, int64_t *out_count,
                                   void *scratch, uint32_t epoch, void *stream) {
  GSX_CHECK_ARG(out_count && scratch, "gsx_compact_indices: null pointer");
  GSX_CHECK_ARG(n >= 0 && n < (1ll << 31) * 1024, "gsx_compact_indices: bad n");
  GSX_CHECK_ARG(epoch >= 1 && epoch < (1u << 30), "gsx_compact_indices: epoch out of range");
  cudaStream_t s = (cudaStream_t)stream;
  if (n == 0) {
    cudaMemsetAsync(out_count, 0, 8, s);
    return 0;
  }
  GSX_CHECK_ARG(flags && out_idx, "gsx_compact_indices: null pointer");
  const int tiles = (int)((n + kTB * 4 - 1) / (kTB * 4));
  CompactArgs a{flags, n, out_idx, out_count, (unsigned long long *)((char *)scratch + 256), (unsigned int *)scratch,
                tiles, epoch};
  k_compact<<<tiles, kTB, 0, s>>>(a);
  GSX_CHECK_LAUNCH("gsx_compact_indices");
  return 0;
}

extern "C" int gsx_active_eval(const float *map_geometry, const int32_t *counts, int64_t capacity, int64_t width,
                               const float *poses, int64_t pose_bstride, const float *intrinsics,
                               int64_t K_bstride, int B, int H, int W, uint8_t *flags, int32_t *hw, void *stream) {
  GSX_CHECK_ARG(map_geometry && counts && poses && intrinsics && flags && hw, "gsx_active_eval: null pointer");
  GSX_CHECK_ARG(B >= 1 && H >= 1 && W >= 1 && width >= 0 && width <= capacity, "gsx_active_eval: bad extents");
  GSX_CHECK_ARG((reinterpret_cast<uintptr_t>(map_geometry) & 15) == 0, "gsx_active_eval: geometry rows must be 16-byte aligned");
  if (width == 0) return 0;
  ActiveArgs a{map_geometry, counts, capacity, width, poses, pose_bstride, intrinsics, K_bstride, image_bounds(H, W),
               flags, hw};
  k_active_eval<<<dim3((unsigned)tb_blocks(width), (unsigned)B), kTB, 0, (cudaStream_t)stream>>>(a);
  GSX_CHECK_LAUNCH("gsx_active_eval");
  return 0;
}

extern "C" int gsx_similar_eval(const int64_t *table, int64_t rows, const float *map_geometry, int64_t capacity,
                                const float *gvertex, const float *gnormal, int B, int H, int W, float dist_th,
                                float dot_th, uint8_t *flags, void *stream) {
  if (rows == 0) return 0;
  GSX_CHECK_ARG(table && map_geometry && gvertex && gnormal && flags, "gsx_similar_eval: null pointer");
  RowArgs a{table, rows, map_geometry, capacity, gvertex, gnormal, B, H, W, sqrt_lt_threshold(dist_th), dot_th, flags,
            nullptr};
  k_similar_eval<<<(unsigned)tb_blocks(rows), kTB, 0, (cudaStream_t)stream>>>(a);
  GSX_CHECK_LAUNCH("gsx_similar_eval");
  return 0;
}

// `records`: B*H*W 4-byte arg-min slots (scratch; cleared here)
extern "C" int gsx_unique_select(const int64_t *table, int64_t rows, const float *map_geometry, int64_t capacity,
                                 const float *gvertex, int B, int H, int W, void *records, uint8_t *pixel_flags,
                                 int64_t *pixel_n, void *stream) {
  GSX_CHECK_ARG(records && pixel_flags && pixel_n, "gsx_unique_select: null pointer");
  GSX_CHECK_ARG((reinterpret_cast<uintptr_t>(records) & 3) == 0, "gsx_unique_select: records must be 4-byte aligned");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_unique_select: capacity must fit int32");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t pixels = (int64_t)B * H * W;
  cudaMemsetAsync(records, 0, (size_t)pixels * 4, s);
  if (rows > 0) {
    GSX_CHECK_ARG(table && map_geometry && gvertex, "gsx_unique_select: null pointer");
    RowArgs a{table, rows, map_geometry, capacity, gvertex, nullptr, B, H, W, 0.f, 0.f, nullptr,
              (unsigned int *)records};
    k_unique_select<<<(unsigned)tb_blocks(rows), kTB, 0, s>>>(a);
  }
  k_unique_emit<<<(unsigned)tb_blocks(pixels), kTB, 0, s>>>((const unsigned int *)records, pixels, pixel_flags, pixel_n);
  GSX_CHECK_LAUNCH("gsx_unique_select");
  return 0;
}

// Stores the rows of a unique table as the per-pixel winners of the fusion workspace (after gsx_fusion_frame_records
// re-armed it, before gsx_fusion_merge_append consumes them): fuse_with_map on a caller-supplied table.
extern "C" int gsx_records_from_table(const int64_t *table, int64_t rows, int64_t capacity, int B, int H, int W,
                                      void *workspace, void *stream) {
  if (rows == 0) return 0;
  GSX_CHECK_ARG(table && workspace, "gsx_records_from_table: null pointer");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_records_from_table: capacity must fit int32");
  RowArgs a{table, rows, nullptr, capacity, nullptr, nullptr, B, H, W, 0.f, 0.f, nullptr,
            fusion_workspace(workspace, B, H, W).win};
  k_records_from_table<<<(unsigned)tb_blocks(rows), kTB, 0, (cudaStream_t)stream>>>(a);
  GSX_CHECK_LAUNCH("gsx_records_from_table");
  return 0;
}
