// Removal of unstable surfels from PointFusion maps for sm_90a (Keller et al. 2013, "Real-time 3D reconstruction in
// dynamic scenes using point-based fusion", section 4.3: a surfel whose confidence is still below c_stable t_max frames
// after it was created is an outlier and is removed).  gradslam has no such step; this is an opt-in extension.
//   k_prune_unstable   (KP)   per batch element, a single-pass stable compaction IN PLACE of the rows [ws, counts[b]):
//                             rows of the window [ws, we) whose confidence is below c_stable are removed, every other
//                             row is kept and moves down; decoupled look-back scan with dynamic tile tickets.
//   k_prune_bwd_rows          one thread per row: the gradient of a kept row comes from its destination row.
// Free-space violations (the same section's second rule, opt-in beside the first): when a stable surfel is merged with
// new data, every surfel in front of it along that ray is removed.
//   k_free_space_bound (KFb)  one thread per pixel: the camera-frame depth of the row K4 merged the pixel into, if that
//                             row is stable after the merge (-inf otherwise): the pixel's bound.
//   k_free_space_test  (KFt)  grid-stride over the rows like K2: project() into the live camera, a row in front of its
//                             pixel's bound by more than the margin is a violator; one flag bit per row, and the
//                             element's lowest violating row.
//   KP<kFreeSpace>            the compaction starts at min(window start, lowest violator) and also removes the flagged
//                             rows; the ring entries move to the positions of the rows they point at.
// Confidence never decreases (a merge adds alpha > 0), so a row that is stable at any age stays stable: every row is
// tested exactly once, at the step its age reaches t_max.  Rows are appended in step order and the compaction is stable,
// so the rows created at step k are the index range [ring(k-1), ring(k)) of each element, where ring(k) is the row count
// after pruned step k (ring(-1) = 0).  The map keeps ring(k) for the last t_max + 2 steps; the row layout is unchanged.
#include "gsx_common.cuh"
#include "gsx_prune.cuh"
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
  int32_t *keep_map;  // optional (nb,cap): destination row or -1 for every row from the scan start on
  PruneScratch sc;    // of elements [b0, b0 + nb)
  // KP<true> only: KFt's violator bits (nb,words) and lowest violating row (nb), 0xffffffff for none
  const unsigned int *flags;
  int64_t words;
  const unsigned int *lowest;
};

__device__ __forceinline__ int ring_at(const PruneArgs &a, int k, int b) {
  return k < 0 ? 0 : a.ring[(int64_t)(k % a.ring_len) * a.ring_stride + b];
}
__device__ __forceinline__ volatile int32_t &ring_ref(const PruneArgs &a, int k, int b) {
  return reinterpret_cast<volatile int32_t *>(a.ring)[(int64_t)(k % a.ring_len) * a.ring_stride + b];
}

// In place is safe under one rule: a tile reads ALL of its rows into registers and issues __threadfence() before it
// publishes its aggregate, and it stores only once it knows its exclusive prefix.  Knowing the prefix means that every
// earlier tile of the element has published, i.e. has read all of its rows.  A row's destination is never above its
// source, and the destinations of tile t end at or before the last row of tile t, so the rows a tile overwrites belong
// to itself (already in registers) or to earlier tiles (already read).  Rows whose destination equals their source are
// not stored, so a window that removes nothing stores nothing.
//
// kFreeSpace (KP<true>): the scan starts at min(window start, lowest violator) and a row is removed if KFt flagged it OR
// the age rule removes it.  Removals may now lie anywhere, so the ring entries of steps s - t_max .. s - 1 become the
// positions of the rows they point at: new ring(k) = the kept rows below old ring(k).  The tile whose rows contain old
// ring(k) writes it (the last tile: every old ring(k) >= count).  Ring entries are non-decreasing in k, so the entries
// of a tile are a contiguous range of k, found before the tile publishes its aggregate.  Writing in place is then safe:
// a tile writes its entries only once it knows its prefix, i.e. after every earlier tile has found its range; a later
// tile reads entries that an earlier tile may have lowered, but both the old and the new value lie below the later
// tile's first row, so its range does not change.  ring(s - t_max - 1), which gives the window start, is not written.
template <bool kFreeSpace>
__global__ void __launch_bounds__(kPB, kPruneCtasPerSM) k_prune_unstable(PruneArgs a) {
  __shared__ int s_tile, s_excl;
  __shared__ int s_warp_sums[kPRows][kPB / 32];
  __shared__ int s_klo, s_khi;               // KP<true>: the ring entries [s_klo, s_khi) of the tile
  __shared__ int s_pos[kFreeSpace ? kPTile : 1];  // KP<true>: exclusive position of each row among the tile's kept rows
  const int b = blockIdx.x % a.nb;  // batch element varies fastest (as in K4)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // the window: rows created at step s - t_max; before step t_max no row is old enough and nothing is covered
  const int count = a.counts[b];
  const int ws = a.step >= a.t_max ? min(ring_at(a, a.step - a.t_max - 1, b), count) : count;
  const int we = a.step >= a.t_max ? (a.t_max == 0 ? count : min(ring_at(a, a.step - a.t_max, b), count)) : count;
  int start = ws;
  if constexpr (kFreeSpace) start = (int)min((unsigned int)ws, a.lowest[b]);
  // tile 0 always exists: the element's last tile records its count and ring entries
  const int ntiles = max(1, (count - start + kPTile - 1) / kPTile);
  unsigned long long *state = a.sc.tile_state + (int64_t)b * a.sc.tiles;
  float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
  float *col = a.col + (int64_t)b * a.cap * kColW;
  const unsigned int *flags = nullptr;
  if constexpr (kFreeSpace) flags = a.flags + (int64_t)b * a.words;
  for (;;) {
    // (every thread has read count / ring above, and the previous tile's s_tile, before the next ticket is drawn)
    __syncthreads();
    if (threadIdx.x == 0) {
      s_tile = (int)atomicAdd(a.sc.ticket + b, 1u);
      if constexpr (kFreeSpace) s_klo = s_khi = a.step;
    }
    __syncthreads();
    const int tile = s_tile;
    if (tile >= ntiles) return;
    const int64_t r0 = (int64_t)start + (int64_t)tile * kPTile;
    float4 g0[kPRows], g1[kPRows], c4[kPRows];
    bool keep[kPRows];
    unsigned int fw[kPRows];  // KP<true>: the violator word of each row
#pragma unroll
    for (int j = 0; j < kPRows; ++j) {
      const int64_t n = r0 + j * kPB + threadIdx.x;
      if (n < count) {
        g0[j] = *reinterpret_cast<const float4 *>(geo + n * kGeoW);
        g1[j] = *reinterpret_cast<const float4 *>(geo + n * kGeoW + 4);
        c4[j] = *reinterpret_cast<const float4 *>(col + n * kColW);
        if constexpr (kFreeSpace) fw[j] = __ldg(flags + (n >> 5));
      }
    }
    if constexpr (kFreeSpace) {
      // this tile's ring entries: old ring(k) in [r0, r1), the last tile also takes every entry >= count
      const int64_t r1 = tile == ntiles - 1 ? INT64_MAX : r0 + kPTile;
      for (int k = max(a.step - a.t_max, 0) + (int)threadIdx.x; k < a.step; k += kPB) {
        const int old = ring_ref(a, k, b);
        if (old >= r0) atomicMin(&s_klo, k);
        if (old >= r1) atomicMin(&s_khi, k);
      }
    }
    __threadfence();  // this thread's rows are read before the tile's aggregate is published (see above)
    int off[kPRows];
    const int kept = block_offsets<kPB, kPRows>(
        [&](int j) {
          const int64_t n = r0 + j * kPB + threadIdx.x;
          if constexpr (kFreeSpace)
            keep[j] = n < count && !(((fw[j] >> (n & 31)) & 1u) || (n >= ws && n < we && g1[j].z < a.c_stable));
          else
            keep[j] = n < count && !(n < we && g1[j].z < a.c_stable);
          return keep[j];
        },
        off, s_warp_sums, [] {});
    if (threadIdx.x == 0) publish_tile(state, tile, ntiles, kPruneEpoch, kTileAggregate, (unsigned)kept);
    if constexpr (kFreeSpace) {
#pragma unroll
      for (int j = 0; j < kPRows; ++j) s_pos[j * kPB + threadIdx.x] = off[j];
    }
    if (warp == 0) {
      const unsigned int excl = lookback_warp(state, tile, ntiles, kPruneEpoch, (unsigned)kept);
      if (lane == 0) s_excl = (int)excl;
    }
    __syncthreads();
    const int64_t base = (int64_t)start + s_excl;
    if constexpr (kFreeSpace) {
      for (int k = s_klo + (int)threadIdx.x; k < s_khi; k += kPB) {
        volatile int32_t &e = ring_ref(a, k, b);
        const int old = e;
        e = (int32_t)(old >= count ? base + kept : base + s_pos[old - r0]);
      }
    }
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
      a.counts[b] = total;
      if constexpr (!kFreeSpace) {  // (KP<true> moved its ring entries above)
        const int removed = count - total;
        for (int k = max(a.step - a.t_max, 0); k < a.step; ++k)
          a.ring[(int64_t)(k % a.ring_len) * a.ring_stride + b] -= removed;
      }
      a.ring[(int64_t)(a.step % a.ring_len) * a.ring_stride + b] = total;
    }
  }
}

// ---- free-space violations ----------------------------------------------------------------------------------------
constexpr int kFB = 256;               // threads per CTA of KFb and KFt
constexpr int kFreeSpaceCtasPerSM = 8;  // KFt's grid-stride cap, as K2's

// Scratch of the free-space step, per element; re-armed by every call (KFb writes every bound and the lowest violator,
// KFt every flag word below the count), so nothing survives from one call to the next.
//   int32  assoc[B][P]     K4's per-pixel record (the sequence driver's; the step entry point takes the caller's)
//   float  bound[B][P]     KFb's bound image
//   uint32 lowest[B]       lowest violating row, 0xffffffff for none
//   uint32 flags[B][words] one bit per row, words = ceil(capacity / 32)
struct FreeSpaceScratch {
  int32_t *assoc;
  float *bound;
  unsigned int *lowest, *flags;
  int64_t words;
};

inline FreeSpaceScratch free_space_scratch(void *base, int B, int64_t P, int64_t capacity, int64_t *bytes = nullptr) {
  Carver c(base);
  FreeSpaceScratch s;
  s.words = capacity > 0 ? (capacity + 31) / 32 : 1;
  s.assoc = c.take<int32_t>((int64_t)B * P);
  s.bound = c.take<float>((int64_t)B * P);
  s.lowest = c.take<unsigned int>(B);
  s.flags = c.take<unsigned int>((int64_t)B * s.words);
  if (bytes) *bytes = c.bytes;
  return s;
}

int64_t free_space_scratch_bytes(int B, int H, int W, int64_t capacity) {
  int64_t bytes;
  free_space_scratch(nullptr, B, (int64_t)H * W, capacity, &bytes);
  return bytes;
}

struct FreeSpaceArgs {  // of the elements [b0, b0 + nb): every pointer already offset to element b0
  const float *geo;     // (nb,cap,8)
  const int32_t *counts;
  int64_t cap;
  const int32_t *assoc;  // (nb,P)
  const float *poses;
  int64_t pose_bstride;
  const float *K;
  int64_t K_bstride;
  ImageBounds ib;
  float c_stable, margin;
  float *bound;           // (nb,P)
  unsigned int *lowest;   // (nb)
  unsigned int *flags;    // (nb,words)
  int64_t words;
};

// KFb: bound[u] = q.z of the row m that K4 merged pixel u into (assoc = -(m+1)) when m is stable after the merge
// (ccount >= c_stable), with project()'s arithmetic; -inf (no q.z is below it) for every other pixel.
__global__ void __launch_bounds__(kFB) k_free_space_bound(FreeSpaceArgs a) {
  __shared__ LiveCamera s_cam;
  const int b = blockIdx.y;
  load_live_camera(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b);
  __syncthreads();
  const int P = a.ib.H * a.ib.W;
  const int pix = blockIdx.x * kFB + threadIdx.x;
  if (pix == 0) a.lowest[b] = 0xffffffffu;  // (KFt lowers it)
  if (pix >= P) return;
  const int32_t as = __ldg(a.assoc + (int64_t)b * P + pix);
  float bound = __int_as_float(0xff800000);
  if (as < 0) {
    const float *row = a.geo + ((int64_t)b * a.cap + (-(int64_t)as - 1)) * kGeoW;
    const float4 p = __ldg(reinterpret_cast<const float4 *>(row));
    if (__ldg(row + 6) >= a.c_stable) bound = rigid_apply(s_cam.tinv, p.x, p.y, p.z).z;
  }
  a.bound[(int64_t)b * P + pix] = bound;
}

// KFt: row n < counts[b] is a violator iff project() puts it in the frustum at pixel u and q.z < bound[u] - margin
// (the difference rounded to fp32).  Each warp takes 32 consecutive rows (a warp-uniform grid-stride loop over
// 32-aligned chunks), so lane 0 stores the chunk's flag word whole and lowers the element's lowest violator once.
__global__ void __launch_bounds__(kFB, kFreeSpaceCtasPerSM) k_free_space_test(FreeSpaceArgs a) {
  __shared__ LiveCamera s_cam;
  const int b = blockIdx.y;
  const int count = a.counts[b];
  if ((int64_t)blockIdx.x * kFB >= count) return;
  load_live_camera(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
  const float *bound = a.bound + (int64_t)b * a.ib.H * a.ib.W;
  unsigned int *flags = a.flags + (int64_t)b * a.words;
  const int64_t stride = (int64_t)gridDim.x * kFB;
  int64_t n0 = (int64_t)blockIdx.x * kFB + (threadIdx.x & ~31u);
  float4 cur = make_float4(0.f, 0.f, 0.f, 0.f);
  if (n0 + lane < count) cur = __ldg(reinterpret_cast<const float4 *>(geo + (n0 + lane) * kGeoW));
  for (; n0 < count; n0 += stride) {
    const int64_t n = n0 + lane;
    const float4 p = cur;
    if (n + stride < count) cur = __ldg(reinterpret_cast<const float4 *>(geo + (n + stride) * kGeoW));  // next row
    bool viol = false;
    if (n < count) {
      const PixelHit hit = project(s_cam, a.ib, p.x, p.y, p.z);
      if (hit.in_frustum) viol = hit.z < __ldg(bound + hit.h * a.ib.W + hit.w) - a.margin;
    }
    const unsigned int v = __ballot_sync(0xffffffffu, viol);
    if (lane == 0) {
      flags[n0 >> 5] = v;
      if (v) atomicMin(a.lowest + b, (unsigned int)(n0 + __ffs(v) - 1));
    }
  }
}

int64_t prune_scratch_bytes(int B, int64_t capacity) {
  int64_t bytes;
  prune_scratch(nullptr, B, capacity, &bytes);
  return bytes;
}

// The pruned step for the elements [b0, b0 + nb) of a B_total-element map on `st`: all pointers are the full-batch base
// pointers; counts and ring are indexed by element.  Disjoint groups may run concurrently on different streams.  With
// fs, KFb and KFt run first and the compaction is KP<true>; without, KP<false> alone (the age rule).
int prune_group(float *geo, float *col, int32_t *counts, int64_t cap, int32_t *ring, int ring_len, int step, int t_max,
                float c_stable, int B_total, int b0, int nb, int32_t *keep_map, void *scratch, cudaStream_t st,
                const FreeSpaceStep *fs) {
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
              (int64_t)B_total, step, t_max, c_stable, nb, keep_map ? keep_map + (int64_t)b0 * cap : nullptr, sc,
              nullptr, 0, nullptr};
  if (fs) {
    const int64_t P = (int64_t)fs->H * fs->W;
    FreeSpaceScratch fsc = free_space_scratch(fs->scratch, B_total, P, cap);
    FreeSpaceArgs f{a.geo, a.counts, cap, fs->assoc + (int64_t)b0 * P, fs->poses + (int64_t)b0 * fs->pose_bstride,
                    fs->pose_bstride, fs->K + (int64_t)b0 * fs->K_bstride, fs->K_bstride, image_bounds(fs->H, fs->W),
                    c_stable, fs->margin, fsc.bound + (int64_t)b0 * P, fsc.lowest + b0,
                    fsc.flags + (int64_t)b0 * fsc.words, fsc.words};
    k_free_space_bound<<<dim3((unsigned)((P + kFB - 1) / kFB), (unsigned)nb), kFB, 0, st>>>(f);
    GSX_CHECK_LAUNCH("gsx_fusion_prune_free_space(bound)");
    if (fs->max_count > 0) {
      int64_t bx = (fs->max_count + kFB - 1) / kFB;
      const int64_t cap_blocks = (int64_t)kNumSMs * kFreeSpaceCtasPerSM;  // grid-stride beyond this many CTAs
      if (bx * nb > cap_blocks) bx = (cap_blocks + nb - 1) / nb;
      if (bx < 1) bx = 1;
      k_free_space_test<<<dim3((unsigned)bx, (unsigned)nb), kFB, 0, st>>>(f);
      GSX_CHECK_LAUNCH("gsx_fusion_prune_free_space(test)");
    }
    a.flags = f.flags;
    a.words = f.words;
    a.lowest = f.lowest;
  }
  // persistent CTAs that draw tiles until the element has none left: the grid does not depend on the (device-side) sizes
  int64_t per_elem = (cap + kPTile - 1) / kPTile;
  const int64_t resident = (int64_t)kNumSMs * kPruneCtasPerSM;
  if (per_elem * nb > resident) per_elem = (resident + nb - 1) / nb;
  if (per_elem < 1) per_elem = 1;
  if (fs)
    k_prune_unstable<true><<<(unsigned)(per_elem * nb), kPB, 0, st>>>(a);
  else
    k_prune_unstable<false><<<(unsigned)(per_elem * nb), kPB, 0, st>>>(a);
  GSX_CHECK_LAUNCH(fs ? "gsx_fusion_prune_free_space" : "gsx_fusion_prune_unstable");
  return 0;
}

int32_t *free_space_assoc(void *scratch, int B_total, int H, int W, int64_t capacity, int b0) {
  return free_space_scratch(scratch, B_total, (int64_t)H * W, capacity).assoc + (int64_t)b0 * H * W;
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

extern "C" int64_t gsx_fusion_free_space_scratch_bytes(int B, int H, int W, int64_t capacity) {
  if (B < 0 || H < 0 || W < 0 || capacity < 0) return -1;
  return free_space_scratch_bytes(B, H, W, capacity);
}

extern "C" int gsx_fusion_prune_free_space(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity,
                                           int32_t *ring, int ring_len, int step, int t_max, float c_stable, int B,
                                           int32_t *keep_map, void *scratch, int64_t scratch_bytes,
                                           const int32_t *assoc, const float *intrinsics, int64_t K_bstride,
                                           const float *poses, int64_t pose_bstride, int H, int W, float margin,
                                           void *fs_scratch, int64_t fs_scratch_bytes, void *stream) {
  GSX_CHECK_ARG(B >= 0 && capacity >= 0 && H >= 2 && W >= 2,
                "gsx_fusion_prune_free_space: bad extents B=%d capacity=%lld H=%d W=%d", B, (long long)capacity, H, W);
  GSX_CHECK_ARG(t_max >= 0 && ring_len == t_max + 2 && step >= 0,
                "gsx_fusion_prune_free_space: need t_max >= 0, ring_len == t_max + 2, step >= 0 (got %d, %d, %d)", t_max,
                ring_len, step);
  GSX_CHECK_ARG(c_stable >= 0.0f, "gsx_fusion_prune_free_space: c_stable must be >= 0");
  GSX_CHECK_ARG(margin >= 0.0f, "gsx_fusion_prune_free_space: margin must be >= 0 (inf allowed, not NaN)");
  if (B == 0) return 0;
  GSX_CHECK_ARG(map_geometry && map_colors && counts && ring && scratch && assoc && intrinsics && poses && fs_scratch,
                "gsx_fusion_prune_free_space: null pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors) && aligned16(fs_scratch),
                "gsx_fusion_prune_free_space: map rows and scratch must be 16-byte aligned");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_fusion_prune_free_space: capacity must fit int32 (counts are int32)");
  GSX_CHECK_ARG(scratch_bytes >= prune_scratch_bytes(B, capacity),
                "gsx_fusion_prune_free_space: scratch of %lld bytes < gsx_fusion_prune_scratch_bytes = %lld",
                (long long)scratch_bytes, (long long)prune_scratch_bytes(B, capacity));
  GSX_CHECK_ARG(fs_scratch_bytes >= free_space_scratch_bytes(B, H, W, capacity),
                "gsx_fusion_prune_free_space: free-space scratch of %lld bytes < gsx_fusion_free_space_scratch_bytes = "
                "%lld", (long long)fs_scratch_bytes, (long long)free_space_scratch_bytes(B, H, W, capacity));
  const FreeSpaceStep fs{assoc, intrinsics, K_bstride, poses, pose_bstride, H, W, margin, fs_scratch, capacity};
  return prune_group(map_geometry, map_colors, counts, capacity, ring, ring_len, step, t_max, c_stable, B, 0, B,
                     keep_map, scratch, (cudaStream_t)stream, &fs);
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
