// Fused PointFusion map update for sm_90a.
//   k_frame_records   (K1r)    one thread per live pixel: re-arms the per-frame workspace and writes the element's header
//                              (camera, depth image).  Nothing per pixel is stored from depth: the consumers re-evaluate
//                              the world vertex, world normal (rgbdimages.py:643-762) and confidence weight
//                              (fusionutils.py:16-73) from the pixel's depth stencil, bit for bit.  Caller-supplied maps
//                              (differentiable mode) are packed into per-pixel records instead.
//   k_project_select  (K2+K3)  one thread per map row: project into the live camera, frustum test, gather of the depth
//                              stencil under the projection, distance / normal tests, then each live candidate, with
//                              its key (1/ccount, ray distance, row index), is appended to the bin of the K4 tile that
//                              owns its pixel (a full bin sends it to the pixel's 4-byte arg-min slot instead:
//                              argmin_claim / argmin_settle, gsx_common.cuh).
//   k_merge_append    (K4)     per tile, the arg-min of its binned candidates in shared memory, combined with the slots;
//                              then one thread per pixel: confidence-weighted merge of the selected map row, or stable append of
//                              unmatched valid pixels (single-pass decoupled look-back scan, row-major order per batch
//                              element).  No float atomics anywhere.
// Map rows are sector-packed (DESIGN.md section 2): geometry rows (px,py,pz,nx,ny,nz,ccount,0) of exactly one 32-byte
// sector, colour rows (r,g,b,0) of 16 bytes; every row access is a 128-bit load / store.
// Reference op chains: gradslam/slam/fusionutils.py:198-722 (see include/gsx.h).
#include "gsx_common.cuh"
#include "gsx_exp.cuh"
#include "gsx_fusion_ws.cuh"
#include "gsx_thresholds.h"
#include "../../include/gsx.h"

namespace gsx {

constexpr int kBlock = 256;

// alpha = clamp(exp(-|v|^2 / 2 sigma^2), 1e-7, 1.01) (fusionutils.py:69-72).  The exponential is evaluated in double and
// rounded once: that is the correctly rounded float32 exp (up to 2^-29 odds), so the CUDA path and the CPU oracle agree
// bit for bit and no later threshold / arg-min decision can flip because of a 1-ulp difference in a confidence weight.
__device__ __forceinline__ float confidence_exp(float sq_norm, float two_sigma_sq) {
  const float x = (-sq_norm) / two_sigma_sq;
  if (!(x >= -17.0f)) return 0.0f;  // exp(x) < 4.2e-8: clamps to 1e-7 below (also NaN, like fmaxf(NaN, 1e-7f))
  return exp_f32_via_f64(x);
}
__device__ __forceinline__ float confidence_alpha(float sq_norm, float two_sigma_sq) {
  return fminf(fmaxf(confidence_exp(sq_norm, two_sigma_sq), 1e-7f), 1.01f);
}

// ---- K1r ------------------------------------------------------------------------------------------------
struct FrameRecArgs {
  const float *depth;  // (B,H,W) live depth
  int64_t depth_bstride;
  const float *K;
  int64_t K_bstride;
  const float *poses;  // camera-to-world, or null: world frame == camera frame
  int64_t pose_bstride;
  const float *gv, *gn, *vloc;  // kFromMaps: materialised (B,H,W,3) world vertex / world normal / camera vertex maps
  int B, H, W;
  float two_sigma_sq;
  Workspace ws;
};

constexpr int kRecTW = 32, kRecTH = 8;  // pixel tile of one K1r CTA

// element b's FrameHeader, by one thread of the element's first K1r CTA.  From maps there is no camera; without poses
// world frame == camera frame.  Fields a record kind does not use stay zero.
__device__ __forceinline__ void store_frame_header(const FrameRecArgs &a, int b) {
  FrameHeader hd = {};
  hd.from_maps = a.gv != nullptr;
  if (!hd.from_maps) {
    hd.cam.k = load_kinv(a.K + b * a.K_bstride);
    if (a.poses) hd.cam.pose = load_rigid(a.poses + b * a.pose_bstride);
    hd.cam.posed = a.poses != nullptr;
  }
  hd.two_sigma_sq = a.two_sigma_sq;
  hd.depth = a.depth + b * a.depth_bstride;
  a.ws.hdr[b] = hd;
}

// Pixel (h,w)'s world normal gn and world vertex fv.xyz (and, if kAlpha, its confidence weight fv.w): the values K1
// computes for that pixel, bit for bit.  Packed maps are gathered from nrec / vrec; from depth, the stencil is gathered
// (its centre dc already loaded) and re-evaluated with K1r's camera and the same device functions and operands.
// from_maps is hd.from_maps and pose is hd.cam.posed ? &hd.cam.pose : nullptr, passed separately so that a caller may
// make them compile-time constants.
template <bool kAlpha>
__device__ __forceinline__ void frame_values(const FrameHeader &hd, bool from_maps, const Rigid *pose,
                                             const float4 *nrec, const float4 *vrec, int h, int w, int H, int W, float dc,
                                             float3 &gn, float4 &fv) {
  if (from_maps) {
    const float4 n = __ldg(nrec + h * W + w);
    gn = make_float3(n.x, n.y, n.z);
    fv = __ldg(vrec + h * W + w);
    return;
  }
  const FrameSample f = frame_sample_from(load_stencil_around(hd.depth, dc, h, w, H, W), hd.cam.k, pose, h, w, H, W);
  gn = f.gn;
  // alpha from the LOCAL vertex (fusionutils.py:657, 69-72)
  fv = make_float4(f.gv.x, f.gv.y, f.gv.z,
                   kAlpha ? confidence_alpha((f.v.x * f.v.x + f.v.y * f.v.y) + f.v.z * f.v.z, hd.two_sigma_sq) : 0.0f);
}

// pixel (h,w)'s depth: K1r's copy in nrec for packed maps, else the caller's depth image
__device__ __forceinline__ float frame_depth(const FrameHeader &hd, bool from_maps, const float4 *nrec, int pix) {
  return from_maps ? __ldg(nrec + pix).w : __ldg(hd.depth + pix);
}

// element b's header into shared memory, one word per thread of threads 64..; the caller synchronises
__device__ __forceinline__ void load_frame_header(FrameHeader &s, const FrameHeader *g) {
  constexpr int kWords = (int)(sizeof(FrameHeader) / 4);
  const int i = (int)threadIdx.x - 64;
  if (i >= 0 && i < kWords) reinterpret_cast<int *>(&s)[i] = __ldg(reinterpret_cast<const int *>(g) + i);
}

// From depth, K1r only re-arms the workspace for the frame and writes the header: K2 and K4 evaluate what they need
// from the depth image itself.  From maps it packs them into nrec / vrec.
template <bool kFromMaps>
__global__ void __launch_bounds__(kRecTW *kRecTH) k_frame_records(FrameRecArgs a) {
  const int b = blockIdx.z;
  const int tid = threadIdx.y * kRecTW + threadIdx.x;
  // re-arm the scan state of this element for the frame's K4
  const int lin = (blockIdx.y * gridDim.x + blockIdx.x) * (kRecTW * kRecTH) + tid;
  if (lin < a.ws.tiles) {
    a.ws.tile_state[(int64_t)b * a.ws.tiles + lin] = 0ull;
    a.ws.bin_count[(int64_t)b * a.ws.tiles + lin] = 0u;
  }
  if (lin == 0) {
    a.ws.ticket[b] = 0u;
    store_frame_header(a, b);
  }
  const int w = blockIdx.x * kRecTW + threadIdx.x, h = blockIdx.y * kRecTH + threadIdx.y;
  if (w >= a.W || h >= a.H) return;
  const int P = a.H * a.W;
  const int pix = h * a.W + w;
  const int64_t i = (int64_t)b * P + pix;
  if (kFromMaps) {
    const int64_t o = i * 3;
    const float vx = __ldg(a.vloc + o), vy = __ldg(a.vloc + o + 1), vz = __ldg(a.vloc + o + 2);
    a.ws.nrec[i] = make_float4(__ldg(a.gn + o), __ldg(a.gn + o + 1), __ldg(a.gn + o + 2),
                               __ldg(a.depth + b * a.depth_bstride + pix));
    a.ws.vrec[i] = make_float4(__ldg(a.gv + o), __ldg(a.gv + o + 1), __ldg(a.gv + o + 2),
                               confidence_alpha((vx * vx + vy * vy) + vz * vz, a.two_sigma_sq));
  }
  a.ws.win[i] = 0u;
}

int launch_frame_records(const FrameRecArgs &a, cudaStream_t stream) {
  if (a.B == 0) return 0;
  const dim3 grid((unsigned)((a.W + kRecTW - 1) / kRecTW), (unsigned)((a.H + kRecTH - 1) / kRecTH), (unsigned)a.B);
  const dim3 block(kRecTW, kRecTH);
  if (a.gv)
    k_frame_records<true><<<grid, block, 0, stream>>>(a);
  else
    k_frame_records<false><<<grid, block, 0, stream>>>(a);
  GSX_CHECK_LAUNCH("gsx_fusion_frame_records");
  return 0;
}

// ---- K2 + K3 ------------------------------------------------------------------------------------------
struct ProjectArgs {
  const float *geo;  // (B,cap,8) geometry rows
  const int32_t *counts;
  int64_t cap;
  const float *poses;
  int64_t pose_bstride;
  const float *K;
  int64_t K_bstride;
  int B;
  ImageBounds ib;
  float dot_th;
  float d2_max;  // largest float x with sqrtf(x) < dist_th (-1 if none): sqrtf(d2) < dist_th <=> d2 <= d2_max
  const float4 *nrec, *vrec;
  const FrameHeader *hdr;
  unsigned int *win;
  unsigned long long *stats;
  unsigned int *bin_count;  // (B,T) and (B,T,kBinCap): the candidate bins of K4's tiles
  uint4 *bin;
  int tiles;
  int bin_cap;  // records per bin that K2 fills (<= kBinCap)
};

// 5 CTAs/SM (48 registers, no spill; DESIGN.md section 4)
#ifndef GSX_K2_MINB
#define GSX_K2_MINB 5
#endif

struct MapRow {  // one geometry row
  float4 a, b;   // a = (px,py,pz,nx)  b = (ny,nz,cc,0)
};
__device__ __forceinline__ MapRow load_map_row(const float *geo, int64_t n) {
  MapRow m;
  m.a = __ldg(reinterpret_cast<const float4 *>(geo + n * kGeoW));
  m.b = __ldg(reinterpret_cast<const float4 *>(geo + n * kGeoW + 4));
  return m;
}

// The kernel is bound by (threads in flight) / (length of the dependent memory chain) and by instruction issue, not by
// bytes, so the chain is kept short and the per-row work small:
//   * the map row of the NEXT grid-stride iteration is fetched while the current row is processed (software pipelining);
//   * the tests gather the depth stencil under the projection (centre, right and lower neighbour: the frame's depth
//     image, 1.2 MB per element, stays in L2) and re-evaluate K1's world vertex and world normal from it;
//   * sqrtf(d2) < dist_th is decided as d2 <= d2_max (exact: the correctly rounded square root is monotonic; the
//     threshold is found on the host, gsx_thresholds.h);
//   * a live candidate is not resolved here: it is appended to the bin of the K4 tile that owns its pixel, with one
//     atomicAdd per group of lanes that hit the same tile, and K4 takes the arg-min in shared memory (append_candidate).
// The grid-stride loop of one CTA over element b's rows; the record kind is a template argument so that each of the two
// loops only holds the registers of its own kind.
// Appends candidate row n of pixel pix (key (key_hi, n)) to the bin of the pixel's K4 tile.  The lanes of a warp that
// hit the same tile share one atomicAdd on the tile's count; each lane then stores its 16-byte record.  A lane whose
// slot lies past the bin's capacity resolves its candidate on the pixel's arg-min slot instead, as the table API
// does; the count keeps growing, so K4 knows the tile overflowed.
__device__ __forceinline__ void append_candidate(unsigned int *bin_count, uint4 *bin, int bin_cap, unsigned int *win,
                                                 const float *geo, int pix, unsigned int n,
                                                 unsigned long long key_hi, const float3 &fv) {
  const int t = pix / kTilePix;
  const unsigned int grp = __match_any_sync(__activemask(), t);
  const int lane = (int)(threadIdx.x & 31), leader = __ffs(grp) - 1;
  unsigned int base = 0u;
  if (lane == leader) base = atomicAdd(bin_count + t, (unsigned int)__popc(grp));
  const unsigned int s = __shfl_sync(grp, base, leader) + (unsigned int)__popc(grp & ((1u << lane) - 1u));
  if (s < (unsigned int)bin_cap)
    bin[(int64_t)t * kBinCap + s] =
        make_uint4((unsigned int)key_hi, (unsigned int)(key_hi >> 32), n, (unsigned int)(pix - t * kTilePix));
  else
    argmin_settle(win + pix, n, key_hi, fv, geo, argmin_claim(win + pix, n));
}

template <bool kFromMaps>
__device__ __forceinline__ void select_rows(const ProjectArgs &a, const LiveCamera &s_cam, const FrameHeader &s_hdr,
                                            unsigned int *s_act, int b, int count) {
  const int P = a.ib.H * a.ib.W;
  const float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
  const float4 *nrec = a.nrec + (int64_t)b * P, *vrec = a.vrec + (int64_t)b * P;
  unsigned int *win = a.win + (int64_t)b * P;
  unsigned int *bin_count = a.bin_count + (int64_t)b * a.tiles;
  uint4 *bin = a.bin + (int64_t)b * a.tiles * kBinCap;
  const int64_t stride = (int64_t)gridDim.x * kBlock;
  int64_t n = (int64_t)blockIdx.x * kBlock + threadIdx.x;
  MapRow cur = load_map_row(geo, n < count ? n : 0);
  for (; n < count; n += stride) {
    const MapRow m = cur;
    const int64_t nn = n + stride;
    if (nn < count) cur = load_map_row(geo, nn);  // in flight while this row is processed
    const PixelHit hit = project(s_cam, a.ib, m.a.x, m.a.y, m.a.z);
    if (hit.in_frustum) {
      {  // count the row (bookkeeping): one shared-memory add per converged group of lanes, no register kept for it
        const unsigned int am = __activemask();
        if ((int)(threadIdx.x & 31) == __ffs(am) - 1) atomicAdd(s_act + (threadIdx.x >> 5), (unsigned int)__popc(am));
      }
      const int pix = hit.h * a.ib.W + hit.w;
      float3 gn;
      float4 fv;
      frame_values<false>(s_hdr, kFromMaps, s_hdr.cam.posed ? &s_hdr.cam.pose : nullptr, nrec, vrec, hit.h, hit.w,
                          a.ib.H, a.ib.W, frame_depth(s_hdr, kFromMaps, nrec, pix), gn, fv);
      // are_normals_similar (fusionutils.py:187-195): n_frame . n_map > dot_th
      const float dot = (gn.x * m.a.w + gn.y * m.b.x) + gn.z * m.b.y;
      // are_points_close (fusionutils.py:130): ||frame - map|| < dist_th
      const float3 fv3 = make_float3(fv.x, fv.y, fv.z);
      const float d2 = ray_d2(fv3, m.a.x, m.a.y, m.a.z);
      const bool live = (d2 <= a.d2_max) && (dot > a.dot_th);
      if (live)
        append_candidate(bin_count, bin, a.bin_cap, win, geo, pix, (unsigned int)n, argmin_key_hi(m.b.z, d2), fv3);
    }
  }
}

__global__ void __launch_bounds__(kBlock, GSX_K2_MINB) k_project_select(ProjectArgs a) {
  __shared__ LiveCamera s_cam;
  __shared__ FrameHeader s_hdr;
  __shared__ unsigned int s_act[kBlock / 32];
  const int b = blockIdx.y;
  const int count = a.counts[b];
  if ((int64_t)blockIdx.x * kBlock >= count) return;
  load_live_camera(s_cam, a.poses, a.pose_bstride, a.K, a.K_bstride, b);
  load_frame_header(s_hdr, a.hdr + b);
  if (threadIdx.x < kBlock / 32) s_act[threadIdx.x] = 0u;
  __syncthreads();
  if (s_hdr.from_maps)
    select_rows<true>(a, s_cam, s_hdr, s_act, b, count);
  else
    select_rows<false>(a, s_cam, s_hdr, s_act, b, count);
  // bookkeeping for the roofline's algorithmic-byte count: ONE atomic per CTA (every warp of the grid adding to the same
  // address would serialise thousands of same-address atomics in the L2 when the whole grid works on one map)
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = 0;
#pragma unroll
    for (int i = 0; i < kBlock / 32; ++i) t += s_act[i];
    if (t) atomicAdd(a.stats + 2 * b, (unsigned long long)t);
  }
}

// K2 runs beside the other batch group's K4 (two groups on concurrent streams); a smaller grid most likely leaves SM
// slots to that K4 (not measured on its own).
// H100, bench workload with the binned arg-min: 8 beat 24 by 6.2-6.5 % on the headline, 12 by 1.3-1.5 % and 16 by
// 2.5-3.4 % (DESIGN.md section 4)
#ifndef GSX_K2_CTAS_PER_SM
#define GSX_K2_CTAS_PER_SM 8
#endif

// Test hook (tests/test_gpu_coverage.py): caps K2's total CTA count so that small maps take several grid-stride
// passes.  0 = the shipped cap below.
static int g_k2_grid_cap = 0;

// Test hook (tests/test_gpu_binned_argmin.py): caps the records per candidate bin that K2 fills and K4 reads, so that
// small frames exercise the overflow to the arg-min slots.  Negative = kBinCap.
static int g_bin_cap = -1;
static int bin_capacity() { return g_bin_cap >= 0 && g_bin_cap < kBinCap ? g_bin_cap : kBinCap; }

int launch_project_select(const ProjectArgs &args, int64_t max_count, cudaStream_t stream) {
  if (args.B == 0 || max_count <= 0) return 0;
  ProjectArgs a = args;
  a.bin_cap = bin_capacity();
  int64_t bx = (max_count + kBlock - 1) / kBlock;
  // grid-stride beyond this many CTAs per SM
  const int64_t cap_blocks = g_k2_grid_cap > 0 ? (int64_t)g_k2_grid_cap : (int64_t)kNumSMs * GSX_K2_CTAS_PER_SM;
  if (bx * a.B > cap_blocks) bx = (cap_blocks + a.B - 1) / a.B;
  if (bx < 1) bx = 1;
  k_project_select<<<dim3((unsigned)bx, (unsigned)a.B), kBlock, 0, stream>>>(a);
  GSX_CHECK_LAUNCH("gsx_fusion_project_select");
  return 0;
}

// ---- K4 -------------------------------------------------------------------------------------------------
struct MergeArgs {
  float *geo, *col;  // (B,cap,8), (B,cap,4)
  int with_cc;       // 0: maps without confidence counts (ICPSLAM aggregation): nothing merges, slot 6 stays 0
  const int32_t *counts_in;
  int32_t *counts_out;
  int64_t cap;
  const float *rgb;  // (B,H,W,3) live colours
  int64_t rgb_bstride;
  int B, H, W;
  Workspace ws;
  int32_t *overflow;
  int32_t *assoc;  // optional (B,P): +row+1 appended at `row`, -(row+1) merged into `row`, 0 untouched
  int bin_cap;     // records per candidate bin that K2 filled (set at launch)
};

// K1r zeroes K4's tile states before every frame, so K4's scan always runs in epoch 1
constexpr unsigned int kMergeEpoch = 1u;

#ifndef GSX_K4_MINB
#define GSX_K4_MINB 4
#endif

// Starts moving the sector at p from DRAM into L2 without waiting for it and without a register.  K4 knows the row a
// pixel merges into as soon as its arg-min slot arrives, but gathers the row only after the CTA's scan barrier and the
// vertex re-evaluation: issued here, the DRAM round trip overlaps that work and the gather hits L2.  H100 80GB HBM3,
// 400 W, bench workload: K4 185 -> 178 us per launch, 21.6-21.7 k -> 21.9-22.0 k frames/s (DESIGN.md section 4).
__device__ __forceinline__ void prefetch_l2(const float *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

template <bool kAssoc>
__global__ void __launch_bounds__(kMB, GSX_K4_MINB) k_merge_append(MergeArgs a) {
  __shared__ int s_tile;
  __shared__ int s_warp_sums[kPix][kMB / 32];
  __shared__ int s_matched[kMB / 32];
  __shared__ int s_excl;
  __shared__ __align__(16) float s_rgb[kTilePix * 3];
  __shared__ FrameHeader s_hdr;
  // the tile's arg-min over its binned candidates: per pixel the smallest key_hi, then the smallest n of that key
  __shared__ unsigned long long s_key[kTilePix];
  __shared__ unsigned int s_n[kTilePix];
  // batch element varies fastest in the grid: CTAs resident at the same time belong to different elements, so
  // each element's look-back chain only sees ~1/B of the in-flight tiles
  const int b = blockIdx.x % a.B;
  const int T = a.ws.tiles;
  if (threadIdx.x == 0) s_tile = (int)atomicAdd(a.ws.ticket + b, 1u);  // tiles start in ticket order
  for (int i = threadIdx.x; i < kTilePix; i += kMB) {
    s_key[i] = ~0ull;
    s_n[i] = ~0u;
  }
  load_frame_header(s_hdr, a.ws.hdr + b);
  const int count_in = a.counts_in[b];  // loaded early: its latency hides behind everything below
  __syncthreads();
  const int tile = s_tile;
  const int P = a.H * a.W;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int pix0 = tile * kTilePix;
  const unsigned int *win = a.ws.win + (int64_t)b * P;
  const float4 *nrec = a.ws.nrec + (int64_t)b * P, *vrec = a.ws.vrec + (int64_t)b * P;
  const float *rgb = a.rgb + b * a.rgb_bstride + (int64_t)pix0 * 3;
  const int n_bin = (int)min(a.ws.bin_count[(int64_t)b * T + tile], (unsigned int)a.bin_cap);
  const uint4 *bin = a.ws.bin + ((int64_t)b * T + tile) * kBinCap;

  // live colours of the tile: coalesced 128-bit loads into shared memory (stride-3 reads are conflict free)
  const int tile_px = min(kTilePix, P - pix0);
  if ((reinterpret_cast<uintptr_t>(rgb) & 15) == 0) {
    const int n4 = (tile_px * 3) >> 2;
    for (int i = threadIdx.x; i < n4; i += kMB)
      reinterpret_cast<float4 *>(s_rgb)[i] = __ldg(reinterpret_cast<const float4 *>(rgb) + i);
    for (int i = (n4 << 2) + threadIdx.x; i < tile_px * 3; i += kMB) s_rgb[i] = __ldg(rgb + i);
  } else {
    for (int i = threadIdx.x; i < tile_px * 3; i += kMB) s_rgb[i] = __ldg(rgb + i);
  }

  int pix[kPix];
  unsigned int slot[kPix];  // the matched map row + 1, 0 for none
  float dep[kPix];
  bool matched[kPix], is_new[kPix];
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    pix[j] = pix0 + j * kMB + threadIdx.x;
    slot[j] = 0u;
    dep[j] = 0.0f;
    if (pix[j] < P) {
      slot[j] = win[pix[j]];
      dep[j] = frame_depth(s_hdr, s_hdr.from_maps, nrec, pix[j]);
    }
  }

  // arg-min of the binned candidates, (key_hi, n) lexicographic: the smallest key_hi per pixel, then the smallest n
  // among the records that carry it.  All of a thread's records are loaded at once and kept for the second pass.
  static_assert(kBinCap % kMB == 0, "a bin is read in whole rounds of the CTA");
  constexpr int kRec = kBinCap / kMB;
  uint4 rec[kRec];
#pragma unroll
  for (int k = 0; k < kRec; ++k) {
    const int i = k * kMB + (int)threadIdx.x;
    if (i < n_bin) rec[k] = __ldg(bin + i);
  }
#pragma unroll
  for (int k = 0; k < kRec; ++k)
    if (k * kMB + (int)threadIdx.x < n_bin) atomicMin(s_key + rec[k].w, ((unsigned long long)rec[k].y << 32) | rec[k].x);
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kRec; ++k)
    if (k * kMB + (int)threadIdx.x < n_bin &&
        (((unsigned long long)rec[k].y << 32) | rec[k].x) == s_key[rec[k].w])
      atomicMin(s_n + rec[k].w, rec[k].z);
  __syncthreads();

#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    const int q = j * kMB + (int)threadIdx.x;
    const unsigned int bn = s_n[q];
    if (bn != ~0u) {
      if (slot[j] == 0u) {
        slot[j] = bn + 1u;
      } else {
        // the pixel also has a winner in its arg-min slot (a bin that overflowed, or gsx_records_from_table): that
        // row's key, recomputed from the pixel's frame vertex as argmin_settle does, decides
        const int ph = pix[j] / a.W;
        float3 gn;
        float4 fv;
        frame_values<false>(s_hdr, s_hdr.from_maps, s_hdr.cam.posed ? &s_hdr.cam.pose : nullptr, nrec, vrec, ph,
                            pix[j] - ph * a.W, a.H, a.W, dep[j], gn, fv);
        const unsigned int m = slot[j] - 1u;
        const float4 p = *reinterpret_cast<const float4 *>(a.geo + ((int64_t)b * a.cap + m) * kGeoW);
        const unsigned long long k = argmin_key_hi(a.geo[((int64_t)b * a.cap + m) * kGeoW + 6],
                                                   ray_d2(make_float3(fv.x, fv.y, fv.z), p.x, p.y, p.z));
        if (!(k < s_key[q] || (k == s_key[q] && m < bn))) slot[j] = bn + 1u;
      }
    }
    matched[j] = a.with_cc && slot[j] != 0u;
    if (matched[j]) {  // the matched row's geometry and colour sectors, gathered below
      const int64_t n = (int64_t)slot[j] - 1;
      prefetch_l2(a.geo + ((int64_t)b * a.cap + n) * kGeoW);
      prefetch_l2(a.col + ((int64_t)b * a.cap + n) * kColW);
    }
  }
  int n_matched = 0;
#pragma unroll
  for (int j = 0; j < kPix; ++j) n_matched += matched[j] ? 1 : 0;
  n_matched = __reduce_add_sync(0xffffffffu, n_matched);
  if (lane == 0) s_matched[warp] = n_matched;
  int new_off[kPix];  // position of each new pixel among the tile's new pixels (row-major)
  const int block_total = block_offsets<kMB, kPix>(
      [&](int j) {
        is_new[j] = (pix[j] < P) && (dep[j] > 0.0f) && !matched[j];
        return is_new[j];
      },
      new_off, s_warp_sums,
      [&] {
        if (threadIdx.x == 0) {  // bookkeeping (merged rows of this element): one atomic per CTA
          int t = 0;
#pragma unroll
          for (int i = 0; i < kMB / 32; ++i) t += s_matched[i];
          if (t) atomicAdd(a.ws.stats + 2 * b + 1, (unsigned long long)t);
        }
      });
  unsigned long long *state = a.ws.tile_state + (int64_t)b * T;
  if (threadIdx.x == 0) publish_tile(state, tile, T, kMergeEpoch, kTileAggregate, (unsigned)block_total);

  float *geo = a.geo + (int64_t)b * a.cap * kGeoW;
  float *col = a.col + (int64_t)b * a.cap * kColW;

  // K1's world vertex, confidence weight and world normal of every pixel that is merged or appended (the tile's depth
  // and the row below it are in L1 / L2 by now)
  float4 fv[kPix];
  float3 fn[kPix];
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (matched[j] || is_new[j]) {
      const int ph = pix[j] / a.W;
      frame_values<true>(s_hdr, s_hdr.from_maps, s_hdr.cam.posed ? &s_hdr.cam.pose : nullptr, nrec, vrec, ph, pix[j] - ph * a.W, a.H, a.W, dep[j], fn[j], fv[j]);
    }
  }

  // matched map rows: issue all loads first, then the arithmetic and the stores
  float4 g0[kPix], g1[kPix], c4[kPix];
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (matched[j]) {
      const int64_t n = (int64_t)slot[j] - 1;
      g0[j] = *reinterpret_cast<const float4 *>(geo + n * kGeoW);
      g1[j] = *reinterpret_cast<const float4 *>(geo + n * kGeoW + 4);
      c4[j] = *reinterpret_cast<const float4 *>(col + n * kColW);
    }
  }
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (matched[j]) {
      // confidence-weighted running mean (fusionutils.py:678-699); exactly one pixel owns this map row
      const int64_t n = (int64_t)slot[j] - 1;
      const float alpha = fv[j].w;
      const float c0 = g1[j].z;
      const float tot = c0 + alpha;
      const float inv = 1.0f / ((tot == 0.0f) ? 1.0f : tot);
      const float *fc = s_rgb + (j * kMB + (int)threadIdx.x) * 3;
      float4 o0, o1, oc;
      o0.x = ((c0 * g0[j].x) + (alpha * fv[j].x)) * inv;
      o0.y = ((c0 * g0[j].y) + (alpha * fv[j].y)) * inv;
      o0.z = ((c0 * g0[j].z) + (alpha * fv[j].z)) * inv;
      o0.w = ((c0 * g0[j].w) + (alpha * fn[j].x)) * inv;
      o1.x = ((c0 * g1[j].x) + (alpha * fn[j].y)) * inv;
      o1.y = ((c0 * g1[j].y) + (alpha * fn[j].z)) * inv;
      o1.z = tot;
      o1.w = 0.0f;
      oc.x = ((c0 * c4[j].x) + (alpha * fc[0])) * inv;
      oc.y = ((c0 * c4[j].y) + (alpha * fc[1])) * inv;
      oc.z = ((c0 * c4[j].z) + (alpha * fc[2])) * inv;
      oc.w = 0.0f;
      *reinterpret_cast<float4 *>(geo + n * kGeoW) = o0;
      *reinterpret_cast<float4 *>(geo + n * kGeoW + 4) = o1;
      *reinterpret_cast<float4 *>(col + n * kColW) = oc;
      if (kAssoc) a.assoc[(int64_t)b * P + pix[j]] = -(int32_t)(n + 1);
    }
  }

  // decoupled look-back (warp 0): exclusive prefix of new-point counts over preceding tiles of this element
  if (warp == 0) {
    const unsigned int excl = lookback_warp(state, tile, T, kMergeEpoch, (unsigned)block_total);
    if (lane == 0) s_excl = (int)excl;
  }
  __syncthreads();
  const int64_t base = (int64_t)count_in + s_excl;
#pragma unroll
  for (int j = 0; j < kPix; ++j) {
    if (is_new[j]) {
      // append in row-major pixel order (fusionutils.py:702-720; pointclouds.py:1203-1235)
      const int64_t n = base + new_off[j];
      if (n < a.cap) {
        const float *fc = s_rgb + (j * kMB + (int)threadIdx.x) * 3;
        *reinterpret_cast<float4 *>(geo + n * kGeoW) = make_float4(fv[j].x, fv[j].y, fv[j].z, fn[j].x);
        *reinterpret_cast<float4 *>(geo + n * kGeoW + 4) =
            make_float4(fn[j].y, fn[j].z, a.with_cc ? fv[j].w : 0.0f, 0.0f);
        *reinterpret_cast<float4 *>(col + n * kColW) = make_float4(fc[0], fc[1], fc[2], 0.0f);
        if (kAssoc) a.assoc[(int64_t)b * P + pix[j]] = (int32_t)(n + 1);
      } else {
        *a.overflow = 1;
      }
    }
  }
  if (tile == T - 1 && threadIdx.x == 0) {
    const int64_t total = base + block_total;
    a.counts_out[b] = (int32_t)(total < a.cap ? total : a.cap);
  }
}

int launch_merge_append(const MergeArgs &args, cudaStream_t stream) {
  if (args.B == 0) return 0;
  MergeArgs a = args;
  a.bin_cap = bin_capacity();
  const dim3 grid((unsigned)(a.ws.tiles * a.B));
  if (a.assoc)
    k_merge_append<true><<<grid, kMB, 0, stream>>>(a);  // differentiable forward
  else
    k_merge_append<false><<<grid, kMB, 0, stream>>>(a);
  GSX_CHECK_LAUNCH("gsx_fusion_merge_append");
  return 0;
}

// ---- K4 backward ------------------------------------------------------------------------------------------
// The differentiable forward (k_merge_append<true>) leaves, per pixel, where its sample went: merged into map row n
// (assoc = -(n+1)), appended as row n (assoc = n+1) or dropped (0).  With the pre-merge map and the frame values the
// backward is a pure per-pixel / per-row map - no atomics, no scan:
//   merged   out = (c*m + a*f) * inv,  inv = 1/(c+a)   (fusionutils.py:678-699)
//            d m = g*c*inv      d f = g*a*inv      d c += g*(m*inv - num*inv^2)      d a += g*(f*inv - num*inv^2)
//            cc_out = c + a  =>  d c += g_cc,  d a += g_cc
//   appended out = f, cc_out = a   =>  d f = g,  d a = g_cc
//   alpha    a = clamp(exp(-|v|^2 / 2 sigma^2), 1e-7, 1.01) (fusionutils.py:69-72)  =>  d v = d a * e * (-2 v / 2 sigma^2)
//            inside the clamp range, 0 outside.
// Map tensors and their gradients use the packed row layout (geometry rows of 8 floats, colour rows of 4; the padding
// slots carry zero gradient).
struct MergeBwdArgs {
  const int32_t *assoc;
  const int32_t *counts_in;
  const float *geo, *col;  // pre-merge map (B, cap_in, 8 / 4)
  int with_cc;
  int64_t cap_in;
  const float *g_geo, *g_col;  // upstream gradients (B, cap_out, 8 / 4); null = zero
  int64_t cap_out;
  const float *gv, *gn, *rgb, *vloc;  // frame values (B, P, 3)
  float *d_geo, *d_col;               // (B, cap_in, 8 / 4)
  float *d_gv, *d_gn, *d_rgb, *d_vloc;  // (B, P, 3)
  int B, P;
  float two_sigma_sq;
};

// rows the frame did not touch pass their gradient through; padding rows get zero
__global__ void __launch_bounds__(256) k_merge_bwd_rows(MergeBwdArgs a) {
  const int b = blockIdx.y;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.cap_in) return;
  const bool live = n < a.counts_in[b] && n < a.cap_out;
  const int64_t ri = (int64_t)b * a.cap_in + n, ro = (int64_t)b * a.cap_out + n;
  float4 z = make_float4(0.f, 0.f, 0.f, 0.f), g0 = z, g1 = z, gc = z;
  if (live && a.g_geo) {
    g0 = *reinterpret_cast<const float4 *>(a.g_geo + ro * kGeoW);
    g1 = *reinterpret_cast<const float4 *>(a.g_geo + ro * kGeoW + 4);
    g1.w = 0.0f;
    if (!a.with_cc) g1.z = 0.0f;
  }
  if (live && a.g_col) {
    gc = *reinterpret_cast<const float4 *>(a.g_col + ro * kColW);
    gc.w = 0.0f;
  }
  *reinterpret_cast<float4 *>(a.d_geo + ri * kGeoW) = g0;
  *reinterpret_cast<float4 *>(a.d_geo + ri * kGeoW + 4) = g1;
  *reinterpret_cast<float4 *>(a.d_col + ri * kColW) = gc;
}

__global__ void __launch_bounds__(256) k_merge_bwd_pixels(MergeBwdArgs a) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= a.P) return;
  const int64_t fi = ((int64_t)b * a.P + pix) * 3;
  const int32_t as = a.assoc[(int64_t)b * a.P + pix];
  float dgv[3] = {0.f, 0.f, 0.f}, dgn[3] = {0.f, 0.f, 0.f}, dc[3] = {0.f, 0.f, 0.f}, dv[3] = {0.f, 0.f, 0.f};
  if (as != 0) {
    const int64_t n = (as > 0) ? (int64_t)as - 1 : -(int64_t)as - 1;
    const int64_t ro = (int64_t)b * a.cap_out + n;
    float g[9];
#pragma unroll
    for (int q = 0; q < 6; ++q) g[q] = a.g_geo ? a.g_geo[ro * kGeoW + q] : 0.0f;
#pragma unroll
    for (int q = 0; q < 3; ++q) g[6 + q] = a.g_col ? a.g_col[ro * kColW + q] : 0.0f;
    const float gcc = (a.g_geo && a.with_cc) ? a.g_geo[ro * kGeoW + 6] : 0.0f;
    const float vx = a.vloc[fi], vy = a.vloc[fi + 1], vz = a.vloc[fi + 2];
    const float sq = (vx * vx + vy * vy) + vz * vz;
    const float e = (float)exp((double)((-sq) / a.two_sigma_sq));  // (cold path: library exp)
    float d_alpha = gcc;
    if (as > 0) {
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        dgv[q] = g[q];
        dgn[q] = g[3 + q];
        dc[q] = g[6 + q];
      }
    } else {
      const int64_t ri = (int64_t)b * a.cap_in + n;
      const float alpha = fminf(fmaxf(e, 1e-7f), 1.01f);
      const float c0 = a.geo[ri * kGeoW + 6];
      const float tot = c0 + alpha;
      const bool degenerate = tot == 0.0f;
      const float inv = 1.0f / (degenerate ? 1.0f : tot);
      const float dinv = degenerate ? 0.0f : -(inv * inv);
      float f[9], m[9];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        f[q] = a.gv[fi + q];
        f[3 + q] = a.gn[fi + q];
        f[6 + q] = a.rgb[fi + q];
        m[q] = a.geo[ri * kGeoW + q];
        m[3 + q] = a.geo[ri * kGeoW + 3 + q];
        m[6 + q] = a.col[ri * kColW + q];
      }
      float d_c0 = gcc;
      float dm[9], df[9];
#pragma unroll
      for (int q = 0; q < 9; ++q) {
        const float num = c0 * m[q] + alpha * f[q];
        dm[q] = g[q] * c0 * inv;
        df[q] = g[q] * alpha * inv;
        d_c0 += g[q] * (m[q] * inv + num * dinv);
        d_alpha += g[q] * (f[q] * inv + num * dinv);
      }
#pragma unroll
      for (int q = 0; q < 6; ++q) a.d_geo[ri * kGeoW + q] = dm[q];
      a.d_geo[ri * kGeoW + 6] = d_c0;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        a.d_col[ri * kColW + q] = dm[6 + q];
        dgv[q] = df[q];
        dgn[q] = df[3 + q];
        dc[q] = df[6 + q];
      }
    }
    if (e >= 1e-7f && e <= 1.01f) {
      const float s = d_alpha * e * (-2.0f / a.two_sigma_sq);
      dv[0] = s * vx;
      dv[1] = s * vy;
      dv[2] = s * vz;
    }
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    a.d_gv[fi + q] = dgv[q];
    a.d_gn[fi + q] = dgn[q];
    a.d_rgb[fi + q] = dc[q];
    a.d_vloc[fi + q] = dv[q];
  }
}

// The two halves of one frame for the batch elements [b0, b0 + nb) of a B_total-element problem, on `st`: the frame
// records (K1r), and the map update that consumes them (K2 + K4).  All pointers are the FULL-batch base pointers; batch
// elements are independent, so disjoint groups may run concurrently on different streams, and the records of the next
// frame may be computed (into another workspace) while this frame's update runs (gsx_pointfusion_sequence_gt).
static Workspace group_workspace(void *workspace, int B_total, int b0, int H, int W) {
  const int64_t P = (int64_t)H * W;
  Workspace ws = fusion_workspace(workspace, B_total, H, W);
  ws.nrec += (int64_t)b0 * P;
  ws.vrec += (int64_t)b0 * P;
  ws.hdr += b0;
  ws.win += (int64_t)b0 * P;
  ws.tile_state += (int64_t)b0 * ws.tiles;
  ws.bin_count += (int64_t)b0 * ws.tiles;
  ws.bin += (int64_t)b0 * ws.tiles * kBinCap;
  ws.ticket += b0;
  ws.stats += 2 * b0;
  return ws;
}

int fusion_records_group(const float *poses, int64_t pose_bs, const float *K, int64_t K_bs, const float *depth,
                         int64_t d_bs, int B_total, int b0, int nb, int H, int W, double sigma, void *workspace,
                         cudaStream_t st) {
  FrameRecArgs fa{depth + (int64_t)b0 * d_bs, d_bs, K + (int64_t)b0 * K_bs, K_bs, poses + (int64_t)b0 * pose_bs, pose_bs,
                  nullptr, nullptr, nullptr, nb, H, W, (float)(2.0 * (sigma * sigma)),
                  group_workspace(workspace, B_total, b0, H, W)};
  return launch_frame_records(fa, st);
}

int fusion_update_group(float *geo, float *col, const int32_t *cin, int32_t *cout, int64_t cap, int64_t max_count,
                        const float *poses, int64_t pose_bs, const float *K, int64_t K_bs, const float *rgb,
                        int64_t rgb_bs, int B_total, int b0, int nb, int H, int W, float dist_th, float dot_th,
                        void *workspace, int32_t *overflow, int32_t *assoc, cudaStream_t st) {
  const Workspace ws = group_workspace(workspace, B_total, b0, H, W);
  float *ggeo = geo + (int64_t)b0 * cap * kGeoW, *gcol = col + (int64_t)b0 * cap * kColW;
  if (max_count > 0) {
    ProjectArgs pa{ggeo, cin + b0, cap, poses + (int64_t)b0 * pose_bs, pose_bs, K + (int64_t)b0 * K_bs, K_bs, nb,
                   image_bounds(H, W), dot_th, sqrt_lt_threshold(dist_th), ws.nrec, ws.vrec, ws.hdr, ws.win, ws.stats, ws.bin_count, ws.bin, ws.tiles, 0};
    const int rc = launch_project_select(pa, max_count, st);
    if (rc) return rc;
  }
  // assoc (full-batch base, zeroed by the caller, or null): where each pixel went, for the free-space step
  MergeArgs ma{ggeo, gcol, 1, cin + b0, cout + b0, cap, rgb + (int64_t)b0 * rgb_bs, rgb_bs, nb, H, W, ws, overflow,
               assoc ? assoc + (int64_t)b0 * H * W : nullptr, 0};
  return launch_merge_append(ma, st);
}

int64_t fusion_workspace_bytes(int B, int H, int W) {
  int64_t bytes;
  fusion_workspace(nullptr, B, H, W, &bytes);
  return bytes;
}

}  // namespace gsx

using namespace gsx;

extern "C" int64_t gsx_fusion_workspace_bytes(int B, int H, int W) {
  if (B < 0 || H < 0 || W < 0) return -1;
  return fusion_workspace_bytes(B, H, W);
}

extern "C" int64_t gsx_fusion_workspace_stats_offset(int B, int H, int W) {
  if (B < 0 || H < 0 || W < 0) return -1;
  return (int64_t)reinterpret_cast<uintptr_t>(fusion_workspace(nullptr, B, H, W).stats);
}

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int gsx_fusion_frame_records(const float *depth, int64_t depth_bstride, const float *intrinsics,
                                        int64_t K_bstride, const float *poses, int64_t pose_bstride,
                                        const float *gvertex, const float *gnormal, const float *vertex, int B, int H,
                                        int W, double sigma, void *workspace, void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2, "gsx_fusion_frame_records: bad extents B=%d H=%d W=%d", B, H, W);
  if (B == 0) return 0;
  GSX_CHECK_ARG(depth && workspace, "gsx_fusion_frame_records: null pointer");
  GSX_CHECK_ARG((gvertex && gnormal && vertex) || (!gvertex && !gnormal && !vertex && intrinsics),
                "gsx_fusion_frame_records: pass the three frame maps, or none of them together with the intrinsics");
  GSX_CHECK_ARG(aligned16(workspace), "gsx_fusion_frame_records: the workspace must be 16-byte aligned");
  FrameRecArgs a{depth, depth_bstride, intrinsics, K_bstride, poses, pose_bstride, gvertex, gnormal, vertex, B, H, W,
                 (float)(2.0 * (sigma * sigma)), fusion_workspace(workspace, B, H, W)};
  return launch_frame_records(a, (cudaStream_t)stream);
}

extern "C" int gsx_fusion_project_select(const float *map_geometry, const int32_t *counts, int64_t capacity,
                                         int64_t max_count, const float *poses, int64_t pose_bstride,
                                         const float *intrinsics, int64_t K_bstride, int B, int H, int W,
                                         float dist_th, float dot_th, void *workspace, void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2, "gsx_fusion_project_select: bad extents B=%d H=%d W=%d", B, H, W);
  if (max_count <= 0 || B == 0) return 0;
  GSX_CHECK_ARG(map_geometry && counts, "gsx_fusion_project_select: null map pointer");
  GSX_CHECK_ARG(poses && intrinsics && workspace, "gsx_fusion_project_select: null frame pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(workspace),
                "gsx_fusion_project_select: geometry rows and workspace must be 16-byte aligned");
  GSX_CHECK_ARG(max_count <= capacity, "gsx_fusion_project_select: max_count %lld > capacity %lld",
                (long long)max_count, (long long)capacity);
  const Workspace ws = fusion_workspace(workspace, B, H, W);
  ProjectArgs a{map_geometry, counts, capacity, poses, pose_bstride, intrinsics, K_bstride, B, image_bounds(H, W),
                dot_th, sqrt_lt_threshold(dist_th), ws.nrec, ws.vrec, ws.hdr, ws.win, ws.stats, ws.bin_count, ws.bin, ws.tiles, 0};
  return launch_project_select(a, max_count, (cudaStream_t)stream);
}

extern "C" void gsx_debug_set_k2_grid_cap(int ctas) { g_k2_grid_cap = ctas > 0 ? ctas : 0; }

extern "C" void gsx_debug_set_bin_capacity(int records) { g_bin_cap = records >= 0 ? records : -1; }

extern "C" int gsx_fusion_merge_append(float *map_geometry, float *map_colors, int with_ccounts,
                                       const int32_t *counts_in, int32_t *counts_out, int64_t capacity,
                                       const float *rgb, int64_t rgb_bstride, int B, int H, int W, void *workspace,
                                       int32_t *overflow_flag, int32_t *assoc_out, void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2, "gsx_fusion_merge_append: bad extents B=%d H=%d W=%d", B, H, W);
  if (B == 0) return 0;
  GSX_CHECK_ARG(map_geometry && map_colors && counts_in && counts_out, "gsx_fusion_merge_append: null map pointer");
  GSX_CHECK_ARG(counts_in != counts_out, "gsx_fusion_merge_append: counts_in and counts_out must not alias");
  GSX_CHECK_ARG(rgb && workspace && overflow_flag, "gsx_fusion_merge_append: null frame pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors) && aligned16(workspace),
                "gsx_fusion_merge_append: map rows and workspace must be 16-byte aligned");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_fusion_merge_append: capacity must fit int32 (counts are int32)");
  MergeArgs a{map_geometry, map_colors, with_ccounts ? 1 : 0, counts_in, counts_out, capacity, rgb, rgb_bstride, B, H,
              W, fusion_workspace(workspace, B, H, W), overflow_flag, assoc_out, 0};
  return launch_merge_append(a, (cudaStream_t)stream);
}

extern "C" int gsx_fusion_merge_append_bwd(const int32_t *assoc, const int32_t *counts_in, const float *map_geometry,
                                           const float *map_colors, int with_ccounts, int64_t capacity_in,
                                           const float *g_geometry, const float *g_colors, int64_t capacity_out,
                                           const float *gvertex, const float *gnormal, const float *rgb,
                                           const float *vertex, int B, int H, int W, double sigma,
                                           float *d_map_geometry, float *d_map_colors, float *d_gvertex,
                                           float *d_gnormal, float *d_rgb, float *d_vertex, void *stream) {
  GSX_CHECK_ARG(B >= 0 && H >= 2 && W >= 2, "gsx_fusion_merge_append_bwd: bad extents B=%d H=%d W=%d", B, H, W);
  if (B == 0) return 0;
  GSX_CHECK_ARG(assoc && counts_in && gvertex && gnormal && rgb && vertex, "gsx_fusion_merge_append_bwd: null input");
  GSX_CHECK_ARG(d_gvertex && d_gnormal && d_rgb && d_vertex, "gsx_fusion_merge_append_bwd: null frame gradient");
  GSX_CHECK_ARG(capacity_in == 0 || (map_geometry && map_colors && d_map_geometry && d_map_colors),
                "gsx_fusion_merge_append_bwd: null map pointer");
  GSX_CHECK_ARG(aligned16(map_geometry) && aligned16(map_colors) && aligned16(g_geometry) && aligned16(g_colors) &&
                    aligned16(d_map_geometry) && aligned16(d_map_colors),
                "gsx_fusion_merge_append_bwd: map rows must be 16-byte aligned");
  MergeBwdArgs a{assoc, counts_in, map_geometry, map_colors, with_ccounts ? 1 : 0, capacity_in, g_geometry, g_colors,
                 capacity_out, gvertex, gnormal, rgb, vertex, d_map_geometry, d_map_colors, d_gvertex, d_gnormal, d_rgb,
                 d_vertex, B, H * W, (float)(2.0 * (sigma * sigma))};
  cudaStream_t st = (cudaStream_t)stream;
  if (capacity_in > 0) {
    k_merge_bwd_rows<<<dim3((unsigned)((capacity_in + 255) / 256), (unsigned)B), 256, 0, st>>>(a);
    GSX_CHECK_LAUNCH("gsx_fusion_merge_append_bwd(rows)");
  }
  k_merge_bwd_pixels<<<dim3((unsigned)((a.P + 255) / 256), (unsigned)B), 256, 0, st>>>(a);
  GSX_CHECK_LAUNCH("gsx_fusion_merge_append_bwd(pixels)");
  return 0;
}
