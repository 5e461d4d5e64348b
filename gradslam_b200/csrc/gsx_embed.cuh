// The embedding merge KE (gsx_embed.cu), as the sequence driver (gsx_api.cu) launches it.
#pragma once
#include "gsx_common.cuh"

namespace gsx {

struct EmbedArgs {
  void *E;          // (B, cap, D) map embeddings
  const void *e;    // frame embeddings: pixel p of element b starts at b * e_bstride + p * D (elements)
  int64_t e_bstride;
  const int32_t *assoc;  // (B, P): -(n+1) merged into row n, n+1 appended as row n, 0 untouched
  const float2 *rec;     // (B, P): (c0, alpha) of every merged pixel
  int64_t cap;
  int B, P, D;
  // upsampled KE only (eh > 0): the frame is a coarse (eh, ew) image, texel (y, x) of element b at
  // b * e_bstride + (y * ew + x) * D, sampled bilinearly at each pixel of the (H, W) depth; eh = 0: e is at the depth's
  // resolution and these are not read
  int H, W, eh, ew;
};

// KE over the pixels of elements [0, a.B); dtype 0 float32, 1 float16, 2 bfloat16.  a.eh > 0 runs the upsampled KE.
int launch_embed_merge_append(const EmbedArgs &a, int dtype, cudaStream_t st);

}  // namespace gsx
