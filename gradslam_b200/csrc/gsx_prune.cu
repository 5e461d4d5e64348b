// Removal of unstable surfels from PointFusion maps for sm_90a (Keller et al. 2013, "Real-time 3D reconstruction in
// dynamic scenes using point-based fusion", section 4.3: a surfel whose confidence is still below c_stable t_max frames
// after it was created is an outlier and is removed).  gradslam has no such step; this is an opt-in extension.
//   k_prune_unstable   (KP)   per batch element, a single-pass stable compaction IN PLACE of the rows [ws, counts[b]):
//                             rows of the window [ws, we) whose confidence is below c_stable are removed, every other
//                             row is kept and moves down; decoupled look-back scan with dynamic tile tickets.
//   k_prune_bwd_rows          one thread per row: the gradient of a kept row comes from its destination row.
// Confidence never decreases (a merge adds alpha > 0), so a row that is stable at any age stays stable: every row is
// tested exactly once, at the step its age reaches t_max.  Rows are appended in step order and the compaction is stable,
// so the rows created at step k are the index range [ring(k-1), ring(k)) of each element, where ring(k) is the row count
// after pruned step k (ring(-1) = 0).  The map keeps ring(k) for the last t_max + 2 steps; the row layout is unchanged.
#include "gsx_common.cuh"
#include "../../include/gsx.h"

namespace gsx {

constexpr int kPB = 256;                 // threads per CTA of the compaction
constexpr int kPRows = 2;                // rows per thread
constexpr int kPTile = kPB * kPRows;     // rows per tile
constexpr int kPruneCtasPerSM = 4;       // resident CTAs per SM (registers, DESIGN.md section 4)
constexpr unsigned int kPruneEpoch = 1u;  // the call zeroes the tile states before the launch

// Scratch of the compaction, per element: tile states of its scan and the dynamic tile ticket.  Sized from the capacity
// (a map that arrives without history has a window as long as the whole map); re-armed by every call, so nothing in it
// survives from one call to the next and a failed call cannot poison a later one.
//   uint64 tile_state[B][T]   look-back state (epoch 1), T = ceil(capacity / kPTile)
//   uint32 ticket[B]          dynamic tile ids
struct PruneScratch {
  unsigned long long *tile_state;
  unsigned int *ticket;
  int64_t tiles;  // T: tile states per element
};

inline PruneScratch prune_scratch(void *base, int B, int64_t capacity, int64_t *bytes = nullptr) {
  Carver c(base);
  PruneScratch s;
  s.tiles = capacity > 0 ? (capacity + kPTile - 1) / kPTile : 1;
  s.tile_state = c.take<unsigned long long>((int64_t)B * s.tiles);
  s.ticket = c.take<unsigned int>(B);
  if (bytes) *bytes = c.bytes;
  return s;
}

struct PruneArgs {
  float *geo, *col;  // (B,cap,8), (B,cap,4) of elements [b0, b0 + nb)
  int32_t *counts;   // (nb,) read and written in place
  int64_t cap;
  int32_t *ring;     // ring(k) of element b at ring[(k mod ring_len) * ring_stride + b]
  int ring_len;
  int64_t ring_stride;
  int step, t_max;
  float c_stable;
  int nb;
  int32_t *keep_map;  // optional (nb,cap): destination row or -1 for every row from the window start on
  PruneScratch sc;    // of elements [b0, b0 + nb)
};

__device__ __forceinline__ int ring_at(const PruneArgs &a, int k, int b) {
  return k < 0 ? 0 : a.ring[(int64_t)(k % a.ring_len) * a.ring_stride + b];
}

// In place is safe under one rule: a tile reads ALL of its rows into registers and issues __threadfence() before it
// publishes its aggregate, and it stores only once it knows its exclusive prefix.  Knowing the prefix means that every
// earlier tile of the element has published, i.e. has read all of its rows.  A row's destination is never above its
// source, and the destinations of tile t end at or before the last row of tile t, so the rows a tile overwrites belong
// to itself (already in registers) or to earlier tiles (already read).  Rows whose destination equals their source are
// not stored, so a window that removes nothing stores nothing.
__global__ void __launch_bounds__(kPB, kPruneCtasPerSM) k_prune_unstable(PruneArgs a) {
  __shared__ int s_tile, s_excl;
  __shared__ int s_warp_sums[kPRows][kPB / 32];
  const int b = blockIdx.x % a.nb;  // batch element varies fastest (as in K4)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // the window: rows created at step s - t_max; before step t_max no row is old enough and nothing is covered
  const int count = a.counts[b];
  const int ws = a.step >= a.t_max ? min(ring_at(a, a.step - a.t_max - 1, b), count) : count;
  const int we = a.step >= a.t_max ? (a.t_max == 0 ? count : min(ring_at(a, a.step - a.t_max, b), count)) : count;
  // tile 0 always exists: the element's last tile records its count and ring entries
  const int ntiles = max(1, (count - ws + kPTile - 1) / kPTile);
  unsigned long long *state = a.sc.tile_state + (int64_t)b * a.sc.tiles;
  float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
  float *col = a.col + (int64_t)b * a.cap * kColW;
  for (;;) {
    // (every thread has read count / ring above, and the previous tile's s_tile, before the next ticket is drawn)
    __syncthreads();
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(a.sc.ticket + b, 1u);
    __syncthreads();
    const int tile = s_tile;
    if (tile >= ntiles) return;
    const int64_t r0 = (int64_t)ws + (int64_t)tile * kPTile;
    float4 g0[kPRows], g1[kPRows], c4[kPRows];
    bool keep[kPRows];
#pragma unroll
    for (int j = 0; j < kPRows; ++j) {
      const int64_t n = r0 + j * kPB + threadIdx.x;
      if (n < count) {
        g0[j] = *reinterpret_cast<const float4 *>(geo + n * kGeoW);
        g1[j] = *reinterpret_cast<const float4 *>(geo + n * kGeoW + 4);
        c4[j] = *reinterpret_cast<const float4 *>(col + n * kColW);
      }
    }
    __threadfence();  // this thread's rows are read before the tile's aggregate is published (see above)
    int off[kPRows];
    const int kept = block_offsets<kPB, kPRows>(
        [&](int j) {
          const int64_t n = r0 + j * kPB + threadIdx.x;
          keep[j] = n < count && !(n < we && g1[j].z < a.c_stable);
          return keep[j];
        },
        off, s_warp_sums, [] {});
    if (threadIdx.x == 0) publish_tile(state, tile, ntiles, kPruneEpoch, kTileAggregate, (unsigned)kept);
    if (warp == 0) {
      const unsigned int excl = lookback_warp(state, tile, ntiles, kPruneEpoch, (unsigned)kept);
      if (lane == 0) s_excl = (int)excl;
    }
    __syncthreads();
    const int64_t base = (int64_t)ws + s_excl;
#pragma unroll
    for (int j = 0; j < kPRows; ++j) {
      const int64_t n = r0 + j * kPB + threadIdx.x;
      if (n >= count) continue;
      const int64_t d = base + off[j];
      if (keep[j] && d != n) {
        *reinterpret_cast<float4 *>(geo + d * kGeoW) = g0[j];
        *reinterpret_cast<float4 *>(geo + d * kGeoW + 4) = g1[j];
        *reinterpret_cast<float4 *>(col + d * kColW) = c4[j];
      }
      if (a.keep_map) a.keep_map[(int64_t)b * a.cap + n] = keep[j] ? (int32_t)d : -1;
    }
    if (tile == ntiles - 1 && threadIdx.x == 0) {
      // new size, ring entries of steps s - t_max .. s - 1 lose the removed rows, ring(s) = new size
      const int total = (int)(base + kept);
      const int removed = count - total;
      a.counts[b] = total;
      for (int k = max(a.step - a.t_max, 0); k < a.step; ++k)
        a.ring[(int64_t)(k % a.ring_len) * a.ring_stride + b] -= removed;
      a.ring[(int64_t)(a.step % a.ring_len) * a.ring_stride + b] = total;
    }
  }
}

int64_t prune_scratch_bytes(int B, int64_t capacity) {
  int64_t bytes;
  prune_scratch(nullptr, B, capacity, &bytes);
  return bytes;
}

// The compaction for the elements [b0, b0 + nb) of a B_total-element map on `st`: all pointers are the full-batch base
// pointers; counts and ring are indexed by element.  Disjoint groups may run concurrently on different streams.
int prune_group(float *geo, float *col, int32_t *counts, int64_t cap, int32_t *ring, int ring_len, int step, int t_max,
                float c_stable, int B_total, int b0, int nb, int32_t *keep_map, void *scratch, cudaStream_t st) {
  if (nb == 0) return 0;
  PruneScratch sc = prune_scratch(scratch, B_total, cap);
  sc.tile_state += (int64_t)b0 * sc.tiles;
  sc.ticket += b0;
  // re-arm this group's tile states and tickets
  if (cudaMemsetAsync(sc.tile_state, 0, (size_t)nb * sc.tiles * sizeof(unsigned long long), st) != cudaSuccess ||
      cudaMemsetAsync(sc.ticket, 0, (size_t)nb * sizeof(unsigned int), st) != cudaSuccess) {
    set_error("gsx_fusion_prune_unstable: re-arming the scratch failed: %s", cudaGetErrorString(cudaGetLastError()));
    return 2;
  }
  PruneArgs a{geo + (int64_t)b0 * cap * kGeoW, col + (int64_t)b0 * cap * kColW, counts + b0, cap, ring + b0, ring_len,
              (int64_t)B_total, step, t_max, c_stable, nb, keep_map ? keep_map + (int64_t)b0 * cap : nullptr, sc};
  // persistent CTAs that draw tiles until the element has none left: the grid does not depend on the (device-side) sizes
  int64_t per_elem = (cap + kPTile - 1) / kPTile;
  const int64_t resident = (int64_t)kNumSMs * kPruneCtasPerSM;
  if (per_elem * nb > resident) per_elem = (resident + nb - 1) / nb;
  if (per_elem < 1) per_elem = 1;
  k_prune_unstable<<<(unsigned)(per_elem * nb), kPB, 0, st>>>(a);
  GSX_CHECK_LAUNCH("gsx_fusion_prune_unstable");
  return 0;
}

// rows before the window carry keep_map[n] = n (the caller's identity fill), removed rows -1, padding rows >= counts_in
// get zero; padding slots (geometry slot 7, colour slot 3) carry zero gradient
__global__ void __launch_bounds__(256) k_prune_bwd_rows(const int32_t *keep_map, const int32_t *counts_in, int64_t cap_in,
                                                       const float *g_geo, const float *g_col, int64_t cap_out,
                                                       float *d_geo, float *d_col) {
  const int b = blockIdx.y;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= cap_in) return;
  const int64_t ri = (int64_t)b * cap_in + n;
  const int32_t k = n < counts_in[b] ? keep_map[ri] : -1;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 g0 = z, g1 = z, gc = z;
  if (k >= 0 && k < cap_out) {
    const int64_t ro = (int64_t)b * cap_out + k;
    if (g_geo) {
      g0 = *reinterpret_cast<const float4 *>(g_geo + ro * kGeoW);
      g1 = *reinterpret_cast<const float4 *>(g_geo + ro * kGeoW + 4);
      g1.w = 0.0f;
    }
    if (g_col) {
      gc = *reinterpret_cast<const float4 *>(g_col + ro * kColW);
      gc.w = 0.0f;
    }
  }
  *reinterpret_cast<float4 *>(d_geo + ri * kGeoW) = g0;
  *reinterpret_cast<float4 *>(d_geo + ri * kGeoW + 4) = g1;
  *reinterpret_cast<float4 *>(d_col + ri * kColW) = gc;
}

}  // namespace gsx

using namespace gsx;

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int64_t gsx_fusion_prune_scratch_bytes(int B, int64_t capacity) {
  if (B < 0 || capacity < 0) return -1;
  return prune_scratch_bytes(B, capacity);
}

extern "C" int gsx_fusion_prune_unstable(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity,
                                         int32_t *ring, int ring_len, int step, int t_max, float c_stable, int B,
                                         int32_t *keep_map, void *scratch, int64_t scratch_bytes, void *stream) {
  GSX_CHECK_ARG(B >= 0 && capacity >= 0, "gsx_fusion_prune_unstable: bad extents B=%d capacity=%lld", B,
                (long long)capacity);
  GSX_CHECK_ARG(t_max >= 0 && ring_len == t_max + 2 && step >= 0,
                "gsx_fusion_prune_unstable: need t_max >= 0, ring_len == t_max + 2, step >= 0 (got %d, %d, %d)", t_max,
                ring_len, step);
  GSX_CHECK_ARG(c_stable >= 0.0f, "gsx_fusion_prune_unstable: c_stable must be >= 0");
  if (B == 0) return 0;
  GSX_CHECK_ARG(map_geometry && map_colors && counts && ring && scratch, "gsx_fusion_prune_unstable: null pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors),
                "gsx_fusion_prune_unstable: map rows must be 16-byte aligned");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_fusion_prune_unstable: capacity must fit int32 (counts are int32)");
  GSX_CHECK_ARG(scratch_bytes >= prune_scratch_bytes(B, capacity),
                "gsx_fusion_prune_unstable: scratch of %lld bytes < gsx_fusion_prune_scratch_bytes = %lld",
                (long long)scratch_bytes, (long long)prune_scratch_bytes(B, capacity));
  return prune_group(map_geometry, map_colors, counts, capacity, ring, ring_len, step, t_max, c_stable, B, 0, B,
                     keep_map, scratch, (cudaStream_t)stream);
}

extern "C" int gsx_fusion_prune_unstable_bwd(const int32_t *keep_map, const int32_t *counts_in, int64_t capacity_in,
                                             const float *g_geometry, const float *g_colors, int64_t capacity_out,
                                             int B, float *d_map_geometry, float *d_map_colors, void *stream) {
  GSX_CHECK_ARG(B >= 0 && capacity_in >= 0 && capacity_out >= 0, "gsx_fusion_prune_unstable_bwd: bad extents");
  if (B == 0 || capacity_in == 0) return 0;
  GSX_CHECK_ARG(keep_map && counts_in && d_map_geometry && d_map_colors, "gsx_fusion_prune_unstable_bwd: null pointer");
  GSX_CHECK_ARG(aligned16(g_geometry) && aligned16(g_colors) && aligned16(d_map_geometry) && aligned16(d_map_colors),
                "gsx_fusion_prune_unstable_bwd: map rows must be 16-byte aligned");
  k_prune_bwd_rows<<<dim3((unsigned)((capacity_in + 255) / 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
      keep_map, counts_in, capacity_in, g_geometry, g_colors, capacity_out, d_map_geometry, d_map_colors);
  GSX_CHECK_LAUNCH("gsx_fusion_prune_unstable_bwd");
  return 0;
}
