// Workspace of the fused PointFusion map update (gsx_fusion.cu), shared with the table variants (gsx_tables.cu).
#pragma once
#include "gsx_common.cuh"

namespace gsx {

#ifndef GSX_KPIX
#define GSX_KPIX 2
#endif
constexpr int kMB = 256;              // threads per CTA of the merge/append kernel
constexpr int kPix = GSX_KPIX;        // pixels per thread
constexpr int kTilePix = kMB * kPix;  // pixels per merge tile

// Capacity of a tile's candidate bin (records per K4 tile and frame).  On the bench's inputs (make_sequence(8, 32, 480,
// 640, seed=0), counted with the CPU oracle over all 32 frames of elements 0..7) the fullest tile holds 771 live
// candidates, 672 on average in the last frame; 1024 leaves a third in reserve.  Candidates past it fall back to the
// per-pixel arg-min slot, so a fuller tile costs time, not correctness.
#ifndef GSX_BIN_CAP
#define GSX_BIN_CAP 1024
#endif
constexpr int kBinCap = GSX_BIN_CAP;

// How K2 / K4 get a pixel's world vertex, world normal and confidence weight, per batch element (written by K1r).  From
// depth, nothing per pixel is stored: K2 and K4 gather the pixel's depth stencil from the caller's depth image and
// re-evaluate vertex, normal and weight with K1r's camera and device functions, bit for bit.  The 1.2 MB depth image of
// an element stays in L2 where a 4.9 MB record array did not.  Caller-supplied maps (differentiable mode) need not equal
// that re-evaluation, so K1r packs them into nrec / vrec.
struct FrameHeader {
  FrameCamera cam;     // K1r's K^-1 and pose
  float two_sigma_sq;  // of the confidence weight
  int from_maps;       // 1: normal and depth are in nrec, vertex and weight in vrec
  const float *depth;  // the element's (H,W) depth image; it must stay unchanged until the frame's K4 has run
};

//   float4 nrec[B][P]          (gnx,gny,gnz,depth), only for caller-supplied maps               written by K1r
//   float4 vrec[B][P]          (gvx,gvy,gvz,alpha), only for caller-supplied maps               written by K1r
//   FrameHeader hdr[B]         where the depth is, how to re-evaluate vertex / normal / weight  written by K1r
//   uint32 win[B][P]           arg-min slot: n + 1 of the winning row, 0 = none; only K2's      cleared by K1r
//                              bin overflow and gsx_records_from_table write it
//   uint64 tile_state[B][T]    look-back state of K4's scan (epoch 1), T = ceil(P / kTilePix)  cleared by K1r
//   uint32 bin_count[B][T]     candidates K2 appended to the tile's bin (may exceed kBinCap)    cleared by K1r
//   uint4  bin[B][T][kBinCap]  candidates (key_hi lo, key_hi hi, n, pixel offset in the tile)  written by K2
//   uint32 ticket[B]           dynamic tile ids of K4                                           cleared by K1r
//   uint64 stats[B][2]         running totals: {active map rows (in frustum), merged rows}      caller zeroes once
// Nothing in here has to survive from one frame to the next (the stats are bookkeeping only): every frame's K1r
// re-arms what K2 / K4 of that frame consume, so a failed or abandoned call cannot poison a later one.
struct Workspace {
  float4 *nrec, *vrec;
  FrameHeader *hdr;
  unsigned int *win;
  unsigned long long *tile_state;
  unsigned int *bin_count;
  uint4 *bin;
  unsigned int *ticket;
  unsigned long long *stats;
  int tiles;
};

// the workspace at `base` (nullptr: byte offsets); `bytes`, if given, receives its size
inline Workspace fusion_workspace(void *base, int B, int H, int W, int64_t *bytes = nullptr) {
  const int64_t P = (int64_t)H * W;
  Carver c(base);
  Workspace w;
  w.tiles = (int)((P + kTilePix - 1) / kTilePix);
  w.nrec = c.take<float4>(B * P);
  w.vrec = c.take<float4>(B * P);
  w.hdr = c.take<FrameHeader>(B);
  w.win = c.take<unsigned int>(B * P);
  w.tile_state = c.take<unsigned long long>((int64_t)B * w.tiles);
  w.bin_count = c.take<unsigned int>((int64_t)B * w.tiles);
  w.bin = c.take<uint4>((int64_t)B * w.tiles * kBinCap);
  w.ticket = c.take<unsigned int>(B);
  w.stats = c.take<unsigned long long>(2 * (int64_t)B);
  if (bytes) *bytes = c.bytes;
  return w;
}

}  // namespace gsx
