// libgsx: error reporting, version, and the whole-sequence drivers that chain the kernels without
// returning to Python between frames.
#include <cstdarg>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <algorithm>
#include <mutex>

#include "gsx_common.cuh"
#include "gsx_prune.cuh"
#include "../../include/gsx.h"

namespace gsx {
static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace gsx

extern "C" int gsx_version(void) { return GSX_VERSION; }
extern "C" const char *gsx_last_error(void) { return gsx::g_err; }

namespace gsx {
// gsx_fusion.cu: the two halves of one frame for the batch elements [b0, b0 + nb) of a B_total-element problem
int fusion_records_group(const float *poses, int64_t pose_bs, const float *K, int64_t K_bs, const float *depth,
                         int64_t d_bs, int B_total, int b0, int nb, int H, int W, double sigma, void *workspace,
                         cudaStream_t st);
int fusion_update_group(float *geo, float *col, const int32_t *cin, int32_t *cout, int64_t cap, int64_t max_count,
                        const float *poses, int64_t pose_bs, const float *K, int64_t K_bs, const float *rgb,
                        int64_t rgb_bs, int B_total, int b0, int nb, int H, int W, float dist_th, float dot_th,
                        void *workspace, int32_t *overflow, int32_t *assoc, cudaStream_t st);
int64_t fusion_workspace_bytes(int B, int H, int W);

// Pruning of the sequence driver (Keller et al. 2013): frame s of the call is pruned step s; null = pruning off.
// fs_scratch non-null adds the free-space rule: K4 records where each pixel went (its group's slice of the scratch's
// assoc image, zeroed first) and KFb, KFt and KP<true> run after it.
struct SequencePrune {
  int32_t *ring;  // (t_max + 2, B)
  int t_max;
  float c_stable;
  void *scratch;
  float margin;
  void *fs_scratch;
};

// one group's pruned step s after its K4 (max_count: the host bound of the counts after that K4)
static int sequence_prune_group(const SequencePrune *prune, float *geo, float *col, int32_t *cout, int64_t cap,
                                const float *intrinsics, const float *poses, int64_t pose_bs, int B, int b0, int nb,
                                int s, int H, int W, int64_t max_count, cudaStream_t st) {
  if (!prune->fs_scratch)
    return prune_group(geo, col, cout, cap, prune->ring, prune->t_max + 2, s, prune->t_max, prune->c_stable, B, b0, nb,
                       nullptr, prune->scratch, st);
  const FreeSpaceStep fs{free_space_assoc(prune->fs_scratch, B, H, W, cap, 0), intrinsics, 16, poses, pose_bs, H, W,
                         prune->margin, prune->fs_scratch, max_count};
  return prune_group(geo, col, cout, cap, prune->ring, prune->t_max + 2, s, prune->t_max, prune->c_stable, B, b0, nb,
                     nullptr, prune->scratch, st, &fs);
}

// the group's assoc slice, zeroed for its K4 (null when the free-space rule is off)
static int32_t *sequence_assoc(const SequencePrune *prune, int B, int b0, int nb, int H, int W, int64_t cap,
                               cudaStream_t st) {
  if (!prune || !prune->fs_scratch) return nullptr;
  int32_t *assoc = free_space_assoc(prune->fs_scratch, B, H, W, cap, 0);
  cudaMemsetAsync(assoc + (int64_t)b0 * H * W, 0, (size_t)nb * H * W * sizeof(int32_t), st);
  return assoc;
}

// Batch elements own independent maps, so the sequence driver splits the batch into groups that walk the frame
// sequence on their own streams: the kernels of one group overlap those of another instead of alternating on an otherwise
// idle GPU (none of them saturates a unit on its own: they are bound by memory latency).  Inside a group the frame
// records of frame s+1 (K1r: independent of the map) are computed on a second stream while K2 / K4 of
// frame s (latency-bound) run: the workspace has two halves used alternately, events order
//     K1r(s) -> K2(s), K4(s)      and      K4(s) -> K1r(s+2)  (same half).
constexpr int kMaxGroups = 4, kMaxDevices = 16;
struct GroupStreams {
  bool ready = false;
  cudaStream_t stream[kMaxGroups], rec_stream[kMaxGroups];
  cudaEvent_t fork, join[kMaxGroups], rec_join[kMaxGroups], rec_done[kMaxGroups][2], upd_done[kMaxGroups][2];
};
static GroupStreams g_groups[kMaxDevices];
// The group streams and their fork / join events are shared by every caller on a device: one enqueue (event record ->
// waits -> launches -> join) must not interleave with another thread's, or a group stream could wait on the other
// caller's fork record instead of its own.  Enqueueing is asynchronous, so the lock is held for microseconds.
static std::mutex g_groups_mutex;

static int sequence_groups(int B) {
  int g = 2;
  if (const char *e = getenv("GSX_SEQ_GROUPS")) g = atoi(e);
  if (g > kMaxGroups) g = kMaxGroups;
  if (g > B) g = B;
  return g < 1 ? 1 : g;
}

static GroupStreams *group_streams() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  GroupStreams &gs = g_groups[dev];
  if (!gs.ready) {
    for (int i = 0; i < kMaxGroups; ++i) {
      if (cudaStreamCreateWithFlags(&gs.stream[i], cudaStreamNonBlocking) != cudaSuccess) return nullptr;
      if (cudaStreamCreateWithFlags(&gs.rec_stream[i], cudaStreamNonBlocking) != cudaSuccess) return nullptr;
      if (cudaEventCreateWithFlags(&gs.join[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
      if (cudaEventCreateWithFlags(&gs.rec_join[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
      for (int h = 0; h < 2; ++h) {
        if (cudaEventCreateWithFlags(&gs.rec_done[i][h], cudaEventDisableTiming) != cudaSuccess) return nullptr;
        if (cudaEventCreateWithFlags(&gs.upd_done[i][h], cudaEventDisableTiming) != cudaSuccess) return nullptr;
      }
    }
    if (cudaEventCreateWithFlags(&gs.fork, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    gs.ready = true;
  }
  return &gs;
}
}  // namespace gsx

// Fault injection for the tests of the error path (tests/test_gpu_pointfusion.py): the sequence driver reports a launch
// failure at frame `s` (once), after the earlier frames were enqueued on the group streams.  -1 = off.
static int g_fail_at_frame = -1;
extern "C" void gsx_debug_fail_at_frame(int s) { g_fail_at_frame = s; }

extern "C" int gsx_pointfusion_sequence_groups(int B) { return B <= 0 ? 0 : gsx::sequence_groups(B); }

// The one driver behind gsx_pointfusion_sequence_gt (prune == nullptr) and gsx_pointfusion_sequence_gt_prune.
static int sequence_gt(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity, int64_t max_count0,
                       const float *depth, const float *rgb, const float *intrinsics, const float *poses, int B, int L,
                       int s_begin, int s_end, int H, int W, float dist_th, float dot_th, double sigma, void *workspace,
                       int32_t *overflow_flag, const gsx::SequencePrune *prune, void *stream) {
  GSX_CHECK_ARG(B >= 0 && L >= 0 && H >= 2 && W >= 2, "gsx_pointfusion_sequence_gt: bad extents");
  GSX_CHECK_ARG(0 <= s_begin && s_begin <= s_end && s_end <= L, "gsx_pointfusion_sequence_gt: bad frame range");
  GSX_CHECK_ARG(counts && depth && rgb && intrinsics && poses, "gsx_pointfusion_sequence_gt: null pointer");
  if (B == 0 || s_begin == s_end) return 0;
  GSX_CHECK_ARG(map_geometry && map_colors && workspace && overflow_flag,
                "gsx_pointfusion_sequence_gt: null map / workspace pointer");
  GSX_CHECK_ARG(((reinterpret_cast<uintptr_t>(map_geometry) | reinterpret_cast<uintptr_t>(map_colors) |
                  reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
                "gsx_pointfusion_sequence_gt: map rows and workspace must be 16-byte aligned");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_pointfusion_sequence_gt: capacity must fit int32 (counts are int32)");
  const int64_t P = (int64_t)H * W;
  cudaStream_t user = (cudaStream_t)stream;
  int G = gsx::sequence_groups(B);
  // the group / record streams and their events are shared by every caller on the device: serialise the enqueue
  std::unique_lock<std::mutex> lock(gsx::g_groups_mutex);
  gsx::GroupStreams *gs = gsx::group_streams();
  char *half[2] = {(char *)workspace, (char *)workspace + gsx::fusion_workspace_bytes(B, H, W)};
  int rc = 0;
  if (!gs) {
    // no side streams available: everything in order on the caller's stream
    for (int s = s_begin; s < s_end && rc == 0; ++s) {
      int64_t max_count = max_count0 + (int64_t)(s - s_begin) * P;
      if (max_count > capacity) max_count = capacity;
      rc = gsx::fusion_records_group(poses + (int64_t)s * 16, (int64_t)L * 16, intrinsics, 16, depth + (int64_t)s * P,
                                     (int64_t)L * P, B, 0, B, H, W, sigma, half[0], user);
      if (rc == 0)
        rc = gsx::fusion_update_group(map_geometry, map_colors, counts + (int64_t)(s & 1) * B,
                                      counts + (int64_t)((s + 1) & 1) * B, capacity, max_count, poses + (int64_t)s * 16,
                                      (int64_t)L * 16, intrinsics, 16, rgb + (int64_t)s * P * 3, (int64_t)L * P * 3, B, 0, B,
                                      H, W, dist_th, dot_th, half[0], overflow_flag,
                                      gsx::sequence_assoc(prune, B, 0, B, H, W, capacity, user), user);
      if (rc == 0 && prune)
        rc = gsx::sequence_prune_group(prune, map_geometry, map_colors, counts + (int64_t)((s + 1) & 1) * B, capacity,
                                       intrinsics, poses + (int64_t)s * 16, (int64_t)L * 16, B, 0, B, s, H, W,
                                       std::min(max_count + P, capacity), user);
    }
    return rc;
  }
  cudaEventRecord(gs->fork, user);
  for (int g = 0; g < G; ++g) {
    cudaStreamWaitEvent(gs->stream[g], gs->fork, 0);
    cudaStreamWaitEvent(gs->rec_stream[g], gs->fork, 0);
  }
  for (int s = s_begin; s < s_end && rc == 0; ++s) {
    const int h = s & 1;
    int32_t *cin = counts + (int64_t)(s & 1) * B;
    int32_t *cout = counts + (int64_t)((s + 1) & 1) * B;
    int64_t max_count = max_count0 + (int64_t)(s - s_begin) * P;
    if (max_count > capacity) max_count = capacity;
    for (int g = 0; g < G && rc == 0; ++g) {
      const int b0 = (int)((int64_t)B * g / G), b1 = (int)((int64_t)B * (g + 1) / G);
      if (s == g_fail_at_frame && g == G - 1) {
        g_fail_at_frame = -1;
        gsx::set_error("gsx_pointfusion_sequence_gt: injected failure at frame %d (gsx_debug_fail_at_frame)", s);
        rc = 2;
        break;
      }
      // frame records of frame s into half h, as soon as K4(s-2) has released that half
      if (s >= s_begin + 2) cudaStreamWaitEvent(gs->rec_stream[g], gs->upd_done[g][h], 0);
      rc = gsx::fusion_records_group(poses + (int64_t)s * 16, (int64_t)L * 16, intrinsics, 16, depth + (int64_t)s * P,
                                     (int64_t)L * P, B, b0, b1 - b0, H, W, sigma, half[h], gs->rec_stream[g]);
      if (rc) break;
      cudaEventRecord(gs->rec_done[g][h], gs->rec_stream[g]);
      cudaStreamWaitEvent(gs->stream[g], gs->rec_done[g][h], 0);
      rc = gsx::fusion_update_group(map_geometry, map_colors, cin, cout, capacity, max_count, poses + (int64_t)s * 16,
                                    (int64_t)L * 16, intrinsics, 16, rgb + (int64_t)s * P * 3, (int64_t)L * P * 3, B, b0,
                                    b1 - b0, H, W, dist_th, dot_th, half[h], overflow_flag,
                                    gsx::sequence_assoc(prune, B, b0, b1 - b0, H, W, capacity, gs->stream[g]),
                                    gs->stream[g]);
      if (rc == 0 && prune)
        rc = gsx::sequence_prune_group(prune, map_geometry, map_colors, cout, capacity, intrinsics,
                                       poses + (int64_t)s * 16, (int64_t)L * 16, B, b0, b1 - b0, s, H, W,
                                       std::min(max_count + P, capacity), gs->stream[g]);
      cudaEventRecord(gs->upd_done[g][h], gs->stream[g]);
    }
  }
  // join ALWAYS, also after a failed launch: whatever was already enqueued on the internal streams stays ordered before
  // anything the caller enqueues next on its stream
  for (int g = 0; g < G; ++g) {
    cudaEventRecord(gs->join[g], gs->stream[g]);
    cudaStreamWaitEvent(user, gs->join[g], 0);
    cudaEventRecord(gs->rec_join[g], gs->rec_stream[g]);
    cudaStreamWaitEvent(user, gs->rec_join[g], 0);
  }
  return rc;
}

extern "C" int gsx_pointfusion_sequence_gt(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity,
                                           int64_t max_count0, const float *depth, const float *rgb,
                                           const float *intrinsics, const float *poses, int B, int L, int s_begin,
                                           int s_end, int H, int W, float dist_th, float dot_th, double sigma,
                                           void *workspace, int32_t *overflow_flag, void *stream) {
  return sequence_gt(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb, intrinsics, poses, B, L,
                     s_begin, s_end, H, W, dist_th, dot_th, sigma, workspace, overflow_flag, nullptr, stream);
}

extern "C" int gsx_pointfusion_sequence_gt_prune(float *map_geometry, float *map_colors, int32_t *counts,
                                                 int64_t capacity, int64_t max_count0, const float *depth,
                                                 const float *rgb, const float *intrinsics, const float *poses, int B,
                                                 int L, int s_begin, int s_end, int H, int W, float dist_th,
                                                 float dot_th, double sigma, void *workspace, int32_t *ring, int t_max,
                                                 float c_stable, void *prune_scratch, int64_t prune_scratch_bytes,
                                                 int32_t *overflow_flag, void *stream) {
  GSX_CHECK_ARG(t_max >= 0 && c_stable >= 0.0f, "gsx_pointfusion_sequence_gt_prune: need t_max >= 0, c_stable >= 0");
  if (B > 0 && s_begin < s_end) {
    GSX_CHECK_ARG(ring && prune_scratch, "gsx_pointfusion_sequence_gt_prune: null ring / scratch pointer");
    GSX_CHECK_ARG(prune_scratch_bytes >= gsx::prune_scratch_bytes(B, capacity),
                  "gsx_pointfusion_sequence_gt_prune: prune scratch of %lld bytes < gsx_fusion_prune_scratch_bytes",
                  (long long)prune_scratch_bytes);
  }
  const gsx::SequencePrune prune{ring, t_max, c_stable, prune_scratch, 0.0f, nullptr};
  return sequence_gt(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb, intrinsics, poses, B, L,
                     s_begin, s_end, H, W, dist_th, dot_th, sigma, workspace, overflow_flag, &prune, stream);
}

extern "C" int gsx_pointfusion_sequence_gt_prune_free_space(
    float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity, int64_t max_count0, const float *depth,
    const float *rgb, const float *intrinsics, const float *poses, int B, int L, int s_begin, int s_end, int H, int W,
    float dist_th, float dot_th, double sigma, void *workspace, int32_t *ring, int t_max, float c_stable,
    void *prune_scratch, int64_t prune_scratch_bytes, float margin, void *fs_scratch, int64_t fs_scratch_bytes,
    int32_t *overflow_flag, void *stream) {
  GSX_CHECK_ARG(t_max >= 0 && c_stable >= 0.0f && margin >= 0.0f,
                "gsx_pointfusion_sequence_gt_prune_free_space: need t_max >= 0, c_stable >= 0, margin >= 0");
  if (B > 0 && s_begin < s_end) {
    GSX_CHECK_ARG(ring && prune_scratch && fs_scratch,
                  "gsx_pointfusion_sequence_gt_prune_free_space: null ring / scratch pointer");
    GSX_CHECK_ARG((reinterpret_cast<uintptr_t>(fs_scratch) & 15) == 0,
                  "gsx_pointfusion_sequence_gt_prune_free_space: the free-space scratch must be 16-byte aligned");
    GSX_CHECK_ARG(prune_scratch_bytes >= gsx::prune_scratch_bytes(B, capacity),
                  "gsx_pointfusion_sequence_gt_prune_free_space: prune scratch of %lld bytes < "
                  "gsx_fusion_prune_scratch_bytes", (long long)prune_scratch_bytes);
    GSX_CHECK_ARG(H >= 0 && W >= 0 && capacity >= 0 &&
                      fs_scratch_bytes >= gsx::free_space_scratch_bytes(B, H, W, capacity),
                  "gsx_pointfusion_sequence_gt_prune_free_space: free-space scratch of %lld bytes < "
                  "gsx_fusion_free_space_scratch_bytes", (long long)fs_scratch_bytes);
  }
  const gsx::SequencePrune prune{ring, t_max, c_stable, prune_scratch, margin, fs_scratch};
  return sequence_gt(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb, intrinsics, poses, B, L,
                     s_begin, s_end, H, W, dist_th, dot_th, sigma, workspace, overflow_flag, &prune, stream);
}

extern "C" int64_t gsx_pointfusion_sequence_workspace_bytes(int B, int H, int W) {
  if (B < 0 || H < 0 || W < 0) return -1;
  return 2 * gsx::fusion_workspace_bytes(B, H, W);
}
