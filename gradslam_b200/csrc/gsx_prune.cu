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
// Merging of overlapping surfels (the section's third rule, opt-in; at the merged pixel, at image resolution, not on the
// paper's 4x4-supersampled index map): a pixel the frame merged into a stable row m absorbs its closest candidate n.
//   KFb<true>, KFt<true>      also arm the per-pixel keys, mark the merge targets, and take each candidate's arg-min
//   k_merge_overlapping (KM)  one thread per pixel: m becomes the weighted mean of m and n, n is flagged for KP<true>
//   k_merge_bwd               the quotient rule of each absorption, after k_prune_bwd_rows' gather
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

// What KFb<true> and KFt<true> add for merging (a second kernel argument, so that FreeSpaceArgs and the code of
// KFb<false> / KFt<false> stay as they are): the merge scratch of the elements [b0, b0 + nb), the age window's ring (as
// PruneArgs) and the normal test's threshold.
struct MergeTestArgs {
  unsigned long long *keys;  // (nb,P)
  unsigned int *targets;     // (nb,words)
  const int32_t *ring;
  int ring_len;
  int64_t ring_stride;
  int step, t_max;
  float dot_th;
};

// KFb: bound[u] = q.z of the row m that K4 merged pixel u into (assoc = -(m+1)) when m is stable after the merge
// (ccount >= c_stable), with project()'s arithmetic; -inf (no q.z is below it) for every other pixel.
// KFb<true> also arms the merge: every pixel's key becomes all-ones, and every row some pixel merged into (stable or
// not) gets its target bit (the caller zeroes the bitmap first).
template <bool kMerge>
__global__ void __launch_bounds__(kFB) k_free_space_bound(FreeSpaceArgs a, MergeTestArgs mt) {
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
    if constexpr (kMerge) {
      const unsigned int m = (unsigned int)(-as - 1);
      atomicOr(mt.targets + (int64_t)b * a.words + (m >> 5), 1u << (m & 31));
    }
  }
  a.bound[(int64_t)b * P + pix] = bound;
  if constexpr (kMerge) mt.keys[(int64_t)b * P + pix] = ~0ull;
}

// The merge test of KFt<true> for row n (first half p = (px,py,pz,nx), already loaded) in the frustum at pixel pu,
// whose bound bnd is finite (the pixel has a stable row m) and which is no violator: n is a candidate of m when it is
// not m, not a merge target, not removed by the age rule, both radii are positive, the normals agree and the disks
// overlap; the pixel's key keeps the smallest bits(d2) << 32 | n.  The element's age window [ws, we) is KP's.
__device__ __forceinline__ void merge_candidate(const FreeSpaceArgs &a, const MergeTestArgs &mt, const float *geo,
                                                int b, int64_t n, const float4 &p, int pu, int ws, int we) {
  const int64_t P = (int64_t)a.ib.H * a.ib.W;
  const int64_t m = -(int64_t)__ldg(a.assoc + b * P + pu) - 1;
  if (m == n || ((__ldg(mt.targets + b * a.words + (n >> 5)) >> (n & 31)) & 1u)) return;
  const float4 q1 = __ldg(reinterpret_cast<const float4 *>(geo + n * kGeoW + 4));  // (ny, nz, ccount, radius)
  if ((n >= ws && n < we && q1.z < a.c_stable) || !(q1.w > 0.0f)) return;
  const float4 m0 = __ldg(reinterpret_cast<const float4 *>(geo + m * kGeoW));
  const float4 m1 = __ldg(reinterpret_cast<const float4 *>(geo + m * kGeoW + 4));
  if (!(m1.w > 0.0f)) return;
  const float dot = (m0.w * p.w + m1.x * q1.x) + m1.y * q1.y;
  if (!(dot > mt.dot_th)) return;
  const float dx = p.x - m0.x, dy = p.y - m0.y, dz = p.z - m0.z;
  const float d2 = (dx * dx + dy * dy) + dz * dz;
  const float rr = m1.w + q1.w;
  if (d2 <= rr * rr)
    atomicMin(mt.keys + b * P + pu, ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned long long)n);
}

// KFt: row n < counts[b] is a violator iff project() puts it in the frustum at pixel u and q.z < bound[u] - margin
// (the difference rounded to fp32).  Each warp takes 32 consecutive rows (a warp-uniform grid-stride loop over
// 32-aligned chunks), so lane 0 stores the chunk's flag word whole and lowers the element's lowest violator once.
// KFt<true> also offers every row that is no violator to the stable row of its pixel (merge_candidate).
template <bool kMerge>
__global__ void __launch_bounds__(kFB, kFreeSpaceCtasPerSM) k_free_space_test(FreeSpaceArgs a, MergeTestArgs mt) {
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
  int ws = count, we = count;  // KFt<true>: the age rule's window, as KP computes it
  if constexpr (kMerge) {
    if (mt.step >= mt.t_max) {
      auto ring_at = [&](int k) { return k < 0 ? 0 : mt.ring[(int64_t)(k % mt.ring_len) * mt.ring_stride + b]; };
      ws = min(ring_at(mt.step - mt.t_max - 1), count);
      we = mt.t_max == 0 ? count : min(ring_at(mt.step - mt.t_max), count);
    }
  }
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
      if constexpr (kMerge) {
        if (hit.in_frustum) {
          const int pu = hit.h * a.ib.W + hit.w;
          const float bnd = __ldg(bound + pu);
          viol = hit.z < bnd - a.margin;
          if (!viol && bnd != __int_as_float(0xff800000)) merge_candidate(a, mt, geo, b, n, p, pu, ws, we);
        }
      } else {
        if (hit.in_frustum) viol = hit.z < __ldg(bound + hit.h * a.ib.W + hit.w) - a.margin;
      }
    }
    const unsigned int v = __ballot_sync(0xffffffffu, viol);
    if (lane == 0) {
      flags[n0 >> 5] = v;
      if (v) atomicMin(a.lowest + b, (unsigned int)(n0 + __ffs(v) - 1));
    }
  }
}

// ---- merging of overlapping surfels ---------------------------------------------------------------------------------
// Scratch of the merge, per element; re-armed by every call (the call zeroes the target bits, KFb<true> sets every key).
//   uint64 keys[B][P]        per pixel: the smallest bits(d2) << 32 | n of its candidates, all-ones for none
//   uint32 targets[B][words] one bit per row that some pixel merged into, words = ceil(capacity / 32)
struct MergeScratch {
  unsigned long long *keys;
  unsigned int *targets;
  int64_t words;
};

inline MergeScratch merge_scratch(void *base, int B, int64_t P, int64_t capacity, int64_t *bytes = nullptr) {
  Carver c(base);
  MergeScratch s;
  s.words = capacity > 0 ? (capacity + 31) / 32 : 1;
  s.keys = c.take<unsigned long long>((int64_t)B * P);
  s.targets = c.take<unsigned int>((int64_t)B * s.words);
  if (bytes) *bytes = c.bytes;
  return s;
}

int64_t merge_scratch_bytes(int B, int H, int W, int64_t capacity) {
  int64_t bytes;
  merge_scratch(nullptr, B, (int64_t)H * W, capacity, &bytes);
  return bytes;
}

struct MergeArgs {  // of the elements [b0, b0 + nb): every pointer already offset to element b0
  float *geo, *col;   // (nb,cap,8), (nb,cap,4)
  int64_t cap;
  const int32_t *assoc;                // (nb,P)
  const unsigned long long *keys;      // (nb,P)
  unsigned int *flags, *lowest;        // KFt's violator bits (nb,words) and lowest removed row (nb)
  int64_t words;
  int P;
  int32_t *absorbed;  // optional (nb,cap): absorbed[m] = n for every absorbing row m
};

// KM: one thread per pixel.  A pixel whose key holds a candidate n absorbs it into its stable row m (assoc = -(m+1)),
// unless KFt flagged m: m becomes the confidence-weighted mean of both rows with K4's operand order, and n is flagged
// for KP<true>.  Rows never conflict: n is no merge target, so it absorbs nothing and is read by no other pixel's m
// update; m is a merge target, so it is absorbed nowhere; and each row projects to one pixel.
__global__ void __launch_bounds__(kFB) k_merge_overlapping(MergeArgs a) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * kFB + threadIdx.x;
  if (pix >= a.P) return;
  const unsigned long long key = a.keys[(int64_t)b * a.P + pix];
  if (key == ~0ull) return;
  const int64_t n = (int64_t)(unsigned int)key;
  const int64_t m = -(int64_t)a.assoc[(int64_t)b * a.P + pix] - 1;
  unsigned int *flags = a.flags + (int64_t)b * a.words;
  if ((flags[m >> 5] >> (m & 31)) & 1u) return;  // the free-space rule removes m: no absorber
  float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
  float *col = a.col + (int64_t)b * a.cap * kColW;
  const float4 m0 = *reinterpret_cast<const float4 *>(geo + m * kGeoW);
  const float4 m1 = *reinterpret_cast<const float4 *>(geo + m * kGeoW + 4);
  const float4 mc = *reinterpret_cast<const float4 *>(col + m * kColW);
  const float4 n0 = *reinterpret_cast<const float4 *>(geo + n * kGeoW);
  const float4 n1 = *reinterpret_cast<const float4 *>(geo + n * kGeoW + 4);
  const float4 nc = *reinterpret_cast<const float4 *>(col + n * kColW);
  const float cm = m1.z, cn = n1.z;
  const float tot = cm + cn;
  const float inv = 1.0f / ((tot == 0.0f) ? 1.0f : tot);
  auto mix = [&](float xm, float xn) { return ((cm * xm) + (cn * xn)) * inv; };
  *reinterpret_cast<float4 *>(geo + m * kGeoW) = make_float4(mix(m0.x, n0.x), mix(m0.y, n0.y), mix(m0.z, n0.z),
                                                             mix(m0.w, n0.w));
  *reinterpret_cast<float4 *>(geo + m * kGeoW + 4) = make_float4(mix(m1.x, n1.x), mix(m1.y, n1.y), tot,
                                                                 mix(m1.w, n1.w));
  *reinterpret_cast<float4 *>(col + m * kColW) = make_float4(mix(mc.x, nc.x), mix(mc.y, nc.y), mix(mc.z, nc.z), mc.w);
  atomicOr(flags + (n >> 5), 1u << (n & 31));
  atomicMin(a.lowest + b, (unsigned int)n);
  if (a.absorbed) a.absorbed[(int64_t)b * a.cap + m] = (int32_t)n;
}

int64_t prune_scratch_bytes(int B, int64_t capacity) {
  int64_t bytes;
  prune_scratch(nullptr, B, capacity, &bytes);
  return bytes;
}

// The pruned step for the elements [b0, b0 + nb) of a B_total-element map on `st`: all pointers are the full-batch base
// pointers; counts and ring are indexed by element.  Disjoint groups may run concurrently on different streams.  With
// fs, KFb and KFt run first and the compaction is KP<true>; without, KP<false> alone (the age rule).  With
// fs->merge_scratch, KFb<true> and KFt<true> also find each stable merged pixel's closest overlapping candidate, and KM
// absorbs it before the compaction.
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
    set_error("gsx_fusion_prune: re-arming the scratch failed: %s", cudaGetErrorString(cudaGetLastError()));
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
    const bool merge = fs->merge_scratch != nullptr;
    MergeTestArgs mt{};
    if (merge) {
      MergeScratch ms = merge_scratch(fs->merge_scratch, B_total, P, cap);
      mt = MergeTestArgs{ms.keys + (int64_t)b0 * P, ms.targets + (int64_t)b0 * ms.words, a.ring, ring_len,
                         a.ring_stride, step, t_max, fs->dot_th};
      if (cudaMemsetAsync(mt.targets, 0, (size_t)nb * ms.words * sizeof(unsigned int), st) != cudaSuccess) {
        set_error("gsx_fusion_prune: re-arming the merge scratch failed: %s", cudaGetErrorString(cudaGetLastError()));
        return 2;
      }
    }
    const dim3 pix_grid((unsigned)((P + kFB - 1) / kFB), (unsigned)nb);
    if (merge)
      k_free_space_bound<true><<<pix_grid, kFB, 0, st>>>(f, mt);
    else
      k_free_space_bound<false><<<pix_grid, kFB, 0, st>>>(f, mt);
    GSX_CHECK_LAUNCH("gsx_fusion_prune(free-space bound)");
    if (fs->max_count > 0) {
      int64_t bx = (fs->max_count + kFB - 1) / kFB;
      const int64_t cap_blocks = (int64_t)kNumSMs * kFreeSpaceCtasPerSM;  // grid-stride beyond this many CTAs
      if (bx * nb > cap_blocks) bx = (cap_blocks + nb - 1) / nb;
      if (bx < 1) bx = 1;
      if (merge)
        k_free_space_test<true><<<dim3((unsigned)bx, (unsigned)nb), kFB, 0, st>>>(f, mt);
      else
        k_free_space_test<false><<<dim3((unsigned)bx, (unsigned)nb), kFB, 0, st>>>(f, mt);
      GSX_CHECK_LAUNCH("gsx_fusion_prune(free-space test)");
      if (merge) {
        const MergeArgs mg{a.geo, a.col, cap, f.assoc, mt.keys, f.flags, f.lowest, f.words, (int)P,
                           fs->absorbed ? fs->absorbed + (int64_t)b0 * cap : nullptr};
        k_merge_overlapping<<<pix_grid, kFB, 0, st>>>(mg);
        GSX_CHECK_LAUNCH("gsx_fusion_prune(merge)");
      }
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
  GSX_CHECK_LAUNCH("gsx_fusion_prune");
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

// After k_prune_bwd_rows: one thread per absorbed pair (b, m, n) rewrites the gradients of m and n from the upstream
// gradient G of m's destination row, with the pair's rows as the forward read them (pair_geo / pair_col: m, then n).
// With c = c_m + c_n and every value x = (c_m x_m + c_n x_n) / c: dx/dx_m = c_m / c, dx/dx_n = c_n / c,
// dx/dc_m = (x_m - x_n) c_n / c^2, dx/dc_n = (x_n - x_m) c_m / c^2 (not (x_m - x) / c: confidences are often ~1e-6, and
// the difference against the rounded mean would carry its rounding error times 1 / c), and the ccount adds G_c to
// both.  The radius carries no gradient.
// Pairs are disjoint, so no row is written twice.
__global__ void __launch_bounds__(256) k_merge_bwd(const int32_t *keep_map, const int32_t *counts_in, int64_t cap_in,
                                                   int B, const int32_t *pairs, const float *pair_geo,
                                                   const float *pair_col, int64_t n_pairs, const float *g_geo,
                                                   const float *g_col, int64_t cap_out, float *d_geo, float *d_col) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  const int b = pairs[i * 3];
  if (b < 0 || b >= B) return;
  const int64_t m = pairs[i * 3 + 1], n = pairs[i * 3 + 2];
  if (m < 0 || n < 0 || m >= counts_in[b] || n >= counts_in[b] || m >= cap_in || n >= cap_in) return;
  const int32_t k = keep_map[(int64_t)b * cap_in + m];
  if (k < 0 || k >= cap_out) return;
  const int64_t rm = (int64_t)b * cap_in + m, rn = (int64_t)b * cap_in + n, ro = (int64_t)b * cap_out + k;
  float xm[10], xn[10], g[10];  // px py pz nx ny nz r g b ccount
  const float *gm = pair_geo + i * 2 * kGeoW, *gn = gm + kGeoW;
  const float *cm_ = pair_col + i * 2 * kColW, *cn_ = cm_ + kColW;
#pragma unroll
  for (int j = 0; j < 6; ++j) xm[j] = gm[j], xn[j] = gn[j];
#pragma unroll
  for (int j = 0; j < 3; ++j) xm[6 + j] = cm_[j], xn[6 + j] = cn_[j];
  xm[9] = gm[6], xn[9] = gn[6];
#pragma unroll
  for (int j = 0; j < 10; ++j) g[j] = 0.0f;
  if (g_geo) {
#pragma unroll
    for (int j = 0; j < 6; ++j) g[j] = g_geo[ro * kGeoW + j];
    g[9] = g_geo[ro * kGeoW + 6];
  }
  if (g_col) {
#pragma unroll
    for (int j = 0; j < 3; ++j) g[6 + j] = g_col[ro * kColW + j];
  }
  const float cm = xm[9], cn = xn[9];
  const float tot = cm + cn;
  const float inv = 1.0f / ((tot == 0.0f) ? 1.0f : tot);
  float dm[10], dn[10];
  float dcm = g[9], dcn = g[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    const float d = xm[j] - xn[j];  // x_m - x = (x_m - x_n) c_n / c: no cancellation against the rounded mean
    dm[j] = g[j] * (cm * inv);
    dn[j] = g[j] * (cn * inv);
    dcm += g[j] * ((d * (cn * inv)) * inv);
    dcn -= g[j] * ((d * (cm * inv)) * inv);
  }
  *reinterpret_cast<float4 *>(d_geo + rm * kGeoW) = make_float4(dm[0], dm[1], dm[2], dm[3]);
  *reinterpret_cast<float4 *>(d_geo + rm * kGeoW + 4) = make_float4(dm[4], dm[5], dcm, 0.0f);
  *reinterpret_cast<float4 *>(d_col + rm * kColW) = make_float4(dm[6], dm[7], dm[8], 0.0f);
  *reinterpret_cast<float4 *>(d_geo + rn * kGeoW) = make_float4(dn[0], dn[1], dn[2], dn[3]);
  *reinterpret_cast<float4 *>(d_geo + rn * kGeoW + 4) = make_float4(dn[4], dn[5], dcn, 0.0f);
  *reinterpret_cast<float4 *>(d_col + rn * kColW) = make_float4(dn[6], dn[7], dn[8], 0.0f);
}

}  // namespace gsx

using namespace gsx;

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int64_t gsx_fusion_prune_scratch_bytes(int B, int64_t capacity) {
  if (B < 0 || capacity < 0) return -1;
  return prune_scratch_bytes(B, capacity);
}

extern "C" int64_t gsx_fusion_free_space_scratch_bytes(int B, int H, int W, int64_t capacity) {
  if (B < 0 || H < 0 || W < 0 || capacity < 0) return -1;
  return free_space_scratch_bytes(B, H, W, capacity);
}

extern "C" int64_t gsx_fusion_merge_scratch_bytes(int B, int H, int W, int64_t capacity) {
  if (B < 0 || H < 0 || W < 0 || capacity < 0) return -1;
  return merge_scratch_bytes(B, H, W, capacity);
}

extern "C" int gsx_fusion_prune_merge(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity,
                                      int32_t *ring, int ring_len, int step, int t_max, float c_stable, int B,
                                      int32_t *keep_map, void *scratch, int64_t scratch_bytes, const int32_t *assoc,
                                      const float *intrinsics, int64_t K_bstride, const float *poses,
                                      int64_t pose_bstride, int H, int W, float margin, void *fs_scratch,
                                      int64_t fs_scratch_bytes, float dot_th, void *merge_scratch,
                                      int64_t merge_scratch_bytes_, int32_t *absorbed, void *stream) {
  GSX_CHECK_ARG(B >= 0 && capacity >= 0 && (!assoc || (H >= 2 && W >= 2)),
                "gsx_fusion_prune: bad extents B=%d capacity=%lld H=%d W=%d", B, (long long)capacity, H, W);
  GSX_CHECK_ARG(t_max >= 0 && ring_len == t_max + 2 && step >= 0,
                "gsx_fusion_prune: need t_max >= 0, ring_len == t_max + 2, step >= 0 (got %d, %d, %d)", t_max, ring_len,
                step);
  GSX_CHECK_ARG(c_stable >= 0.0f, "gsx_fusion_prune: c_stable must be >= 0");
  GSX_CHECK_ARG(!assoc || margin >= 0.0f, "gsx_fusion_prune: margin must be >= 0 (inf allowed, not NaN)");
  if (B == 0) return 0;
  GSX_CHECK_ARG(map_geometry && map_colors && counts && ring && scratch, "gsx_fusion_prune: null pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors), "gsx_fusion_prune: map rows must be 16-byte aligned");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_fusion_prune: capacity must fit int32 (counts are int32)");
  GSX_CHECK_ARG(scratch_bytes >= prune_scratch_bytes(B, capacity),
                "gsx_fusion_prune: scratch of %lld bytes < gsx_fusion_prune_scratch_bytes = %lld",
                (long long)scratch_bytes, (long long)prune_scratch_bytes(B, capacity));
  GSX_CHECK_ARG(assoc || !merge_scratch,
                "gsx_fusion_prune_merge: merging needs the free-space inputs (assoc; margin = inf removes no violator)");
  if (!assoc)
    return prune_group(map_geometry, map_colors, counts, capacity, ring, ring_len, step, t_max, c_stable, B, 0, B,
                       keep_map, scratch, (cudaStream_t)stream);
  GSX_CHECK_ARG(intrinsics && poses && fs_scratch, "gsx_fusion_prune: null free-space pointer");
  GSX_CHECK_ARG(aligned16(fs_scratch), "gsx_fusion_prune: the free-space scratch must be 16-byte aligned");
  GSX_CHECK_ARG(fs_scratch_bytes >= free_space_scratch_bytes(B, H, W, capacity),
                "gsx_fusion_prune: free-space scratch of %lld bytes < gsx_fusion_free_space_scratch_bytes = %lld",
                (long long)fs_scratch_bytes, (long long)free_space_scratch_bytes(B, H, W, capacity));
  if (merge_scratch) {
    GSX_CHECK_ARG(!(dot_th != dot_th), "gsx_fusion_prune_merge: dot_th must not be NaN");
    GSX_CHECK_ARG(aligned16(merge_scratch), "gsx_fusion_prune_merge: the merge scratch must be 16-byte aligned");
    GSX_CHECK_ARG(merge_scratch_bytes_ >= merge_scratch_bytes(B, H, W, capacity),
                  "gsx_fusion_prune_merge: merge scratch of %lld bytes < gsx_fusion_merge_scratch_bytes = %lld",
                  (long long)merge_scratch_bytes_, (long long)merge_scratch_bytes(B, H, W, capacity));
  }
  const FreeSpaceStep fs{assoc,    intrinsics, K_bstride,     poses,  pose_bstride, H,
                         W,        margin,     fs_scratch,    capacity, merge_scratch, dot_th,
                         merge_scratch ? absorbed : nullptr};
  return prune_group(map_geometry, map_colors, counts, capacity, ring, ring_len, step, t_max, c_stable, B, 0, B,
                     keep_map, scratch, (cudaStream_t)stream, &fs);
}

extern "C" int gsx_fusion_prune(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity, int32_t *ring,
                                int ring_len, int step, int t_max, float c_stable, int B, int32_t *keep_map,
                                void *scratch, int64_t scratch_bytes, const int32_t *assoc, const float *intrinsics,
                                int64_t K_bstride, const float *poses, int64_t pose_bstride, int H, int W, float margin,
                                void *fs_scratch, int64_t fs_scratch_bytes, void *stream) {
  return gsx_fusion_prune_merge(map_geometry, map_colors, counts, capacity, ring, ring_len, step, t_max, c_stable, B,
                                keep_map, scratch, scratch_bytes, assoc, intrinsics, K_bstride, poses, pose_bstride, H,
                                W, margin, fs_scratch, fs_scratch_bytes, 0.0f, nullptr, 0, nullptr, stream);
}

extern "C" int gsx_fusion_prune_bwd(const int32_t *keep_map, const int32_t *counts_in, int64_t capacity_in,
                                             const float *g_geometry, const float *g_colors, int64_t capacity_out,
                                             int B, float *d_map_geometry, float *d_map_colors, void *stream) {
  GSX_CHECK_ARG(B >= 0 && capacity_in >= 0 && capacity_out >= 0, "gsx_fusion_prune_bwd: bad extents");
  if (B == 0 || capacity_in == 0) return 0;
  GSX_CHECK_ARG(keep_map && counts_in && d_map_geometry && d_map_colors, "gsx_fusion_prune_bwd: null pointer");
  GSX_CHECK_ARG(aligned16(g_geometry) && aligned16(g_colors) && aligned16(d_map_geometry) && aligned16(d_map_colors),
                "gsx_fusion_prune_bwd: map rows must be 16-byte aligned");
  k_prune_bwd_rows<<<dim3((unsigned)((capacity_in + 255) / 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
      keep_map, counts_in, capacity_in, g_geometry, g_colors, capacity_out, d_map_geometry, d_map_colors);
  GSX_CHECK_LAUNCH("gsx_fusion_prune_bwd");
  return 0;
}

extern "C" int gsx_fusion_prune_merge_bwd(const int32_t *keep_map, const int32_t *counts_in, int64_t capacity_in,
                                          const int32_t *pairs, const float *pair_geometry, const float *pair_colors,
                                          int64_t n_pairs, const float *g_geometry, const float *g_colors,
                                          int64_t capacity_out, int B, float *d_map_geometry, float *d_map_colors,
                                          void *stream) {
  GSX_CHECK_ARG(n_pairs >= 0, "gsx_fusion_prune_merge_bwd: bad extents");
  GSX_CHECK_ARG(n_pairs == 0 || (pairs && pair_geometry && pair_colors), "gsx_fusion_prune_merge_bwd: null pointer");
  GSX_CHECK_ARG(n_pairs == 0 || (aligned16(pair_geometry) && aligned16(pair_colors)),
                "gsx_fusion_prune_merge_bwd: pair rows must be 16-byte aligned");
  int rc = gsx_fusion_prune_bwd(keep_map, counts_in, capacity_in, g_geometry, g_colors, capacity_out, B,
                                d_map_geometry, d_map_colors, stream);
  if (rc || B == 0 || capacity_in == 0 || n_pairs == 0) return rc;
  k_merge_bwd<<<(unsigned)((n_pairs + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      keep_map, counts_in, capacity_in, B, pairs, pair_geometry, pair_colors, n_pairs, g_geometry, g_colors,
      capacity_out, d_map_geometry, d_map_colors);
  GSX_CHECK_LAUNCH("gsx_fusion_prune_merge_bwd");
  return 0;
}
