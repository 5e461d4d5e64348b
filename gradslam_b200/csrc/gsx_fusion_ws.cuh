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

// frames whose headers the sequence driver's workspace holds at a time (gsx_fusion.cu: sequence_workspace_bytes)
constexpr int kSeqFrames = 64;

// How K2 / K4 get a pixel's world vertex, world normal and confidence weight, per batch element (written by K1r).
// Nothing per pixel is stored: K2 and K4 gather the pixel's depth stencil from the caller's depth image and re-evaluate
// vertex, normal and weight with K1r's camera and device functions, bit for bit.  The 1.2 MB depth image of an element
// stays in L2 where a 4.9 MB record array did not.
struct FrameHeader {
  FrameCamera cam;     // K1r's K^-1 and pose
  float two_sigma_sq;  // of the confidence weight
  const float *depth;  // the element's (H,W) depth image; it must stay unchanged until the frame's K4 has run
};

//   FrameHeader hdr[B]         where the depth is, how to re-evaluate vertex / normal / weight  written by K1r
//   uint32 win[B][P]           arg-min slot: n + 1 of the winning row, 0 = none; only K2's      zero when K2 starts
//                              bin overflow and gsx_records_from_table write it
//   uint64 tile_state[B][T]    look-back state of K4's scan, T = ceil(P / kTilePix)            epoch from the ticket
//   uint32 bin_count[B][T]     candidates K2 appended to the tile's bin (may exceed kBinCap)    zeroed by K4
//   uint32 ticket[B]           K4's tickets: tile = ticket % T, scan epoch = ticket / T + 1
//   uint32 table[B]            non-zero: gsx_records_from_table filled slots of the element    cleared by K4
//   uint4  bin[B][T][kBinCap]  candidates (key_hi lo, key_hi hi, n, pixel offset in the tile)  written by K2
//   uint64 stats[B][2]         running totals: {active map rows (in frustum), merged rows}      caller zeroes once
// win .. table form the re-arm state, one contiguous byte range (rearm_bytes): all zero is a valid start, and the
// step API's workspace must start so (zero-filled once before first use: no kernel clears the slots per frame).  The
// invariant is kept by the consumer: every slot is zero when a frame's K2 starts.  K4 reads a tile's slots only when
// the tile's bin overflowed or the element's table flag is set, and stores zero to the slots it read; so on a frame
// without overflow no slot is read or written.  K4 zeroes its tile's bin count once it has read it, and the scan's last
// tile clears the table flag.  A frame abandoned before its K4 (K2 or the table fill ran, K4 did not) leaves
// dirty slots: K1r (the per-frame step API) clears the slots of every tile whose bin count exceeds the capacity, and of
// the whole element while its table flag is set, before it re-arms the counts.  The sequence driver runs no K1r: it
// zeroes the re-arm state once per call, so nothing survives from one call to the next.
struct Workspace {
  FrameHeader *hdr;
  unsigned int *win;
  unsigned long long *tile_state;
  unsigned int *bin_count;
  unsigned int *ticket;
  unsigned int *table;
  uint4 *bin;
  unsigned long long *stats;
  int tiles;
};

// the workspace at `base` (nullptr: byte offsets); `bytes`, if given, receives its size; `rearm_bytes`, if given, the
// size of the re-arm state that starts at win
inline Workspace fusion_workspace(void *base, int B, int H, int W, int64_t *bytes = nullptr,
                                  int64_t *rearm_bytes = nullptr) {
  const int64_t P = (int64_t)H * W;
  Carver c(base);
  Workspace w;
  w.tiles = (int)((P + kTilePix - 1) / kTilePix);
  w.hdr = c.take<FrameHeader>(B);
  const int64_t rearm0 = c.bytes;
  w.win = c.take<unsigned int>(B * P);
  w.tile_state = c.take<unsigned long long>((int64_t)B * w.tiles);
  w.bin_count = c.take<unsigned int>((int64_t)B * w.tiles);
  w.ticket = c.take<unsigned int>(B);
  w.table = c.take<unsigned int>(B);
  if (rearm_bytes) *rearm_bytes = c.bytes - rearm0;
  w.bin = c.take<uint4>((int64_t)B * w.tiles * kBinCap);
  w.stats = c.take<unsigned long long>(2 * (int64_t)B);
  if (bytes) *bytes = c.bytes;
  return w;
}

}  // namespace gsx
