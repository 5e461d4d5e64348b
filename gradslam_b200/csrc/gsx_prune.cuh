// The pruned step of gsx_prune.cu as the sequence driver (gsx_api.cu) calls it for one batch group.
#pragma once
#include "gsx_common.cuh"

namespace gsx {

// The free-space rule's inputs for one pruned step: the live camera and K4's per-pixel record of that step's merge.
// Pointers are full-batch base pointers; null `fs` = the age rule alone.
struct FreeSpaceStep {
  const int32_t *assoc;  // (B_total, H*W): -(m+1) merged into row m (k_merge_append<true>)
  const float *K;
  int64_t K_bstride;
  const float *poses;  // camera-to-world of the live frame
  int64_t pose_bstride;
  int H, W;
  float margin;
  void *scratch;        // free_space_scratch_bytes(B_total, H, W, cap)
  int64_t max_count;    // host-side upper bound of the counts (KFt's grid)
};

// removal of unstable surfels (and, with fs, of free-space violations) for the elements [b0, b0 + nb)
int prune_group(float *geo, float *col, int32_t *counts, int64_t cap, int32_t *ring, int ring_len, int step, int t_max,
                float c_stable, int B_total, int b0, int nb, int32_t *keep_map, void *scratch, cudaStream_t st,
                const FreeSpaceStep *fs = nullptr);
int64_t prune_scratch_bytes(int B, int64_t capacity);
int64_t free_space_scratch_bytes(int B, int H, int W, int64_t capacity);
// the group's slice of the free-space scratch's assoc image (the sequence driver's K4 writes it)
int32_t *free_space_assoc(void *scratch, int B_total, int H, int W, int64_t capacity, int b0);

}  // namespace gsx
