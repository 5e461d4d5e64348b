// libgsx: error reporting, version, and the whole-sequence drivers that chain the kernels without
// returning to Python between frames.
#include <cstdarg>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <algorithm>
#include <mutex>

#include "gsx_common.cuh"
#include "gsx_embed.cuh"
#include "gsx_fusion_ws.cuh"
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
// gsx_fusion.cu: the sequence workspace, its per-call re-arm, the frame headers of frames [s, s + F) and the map update
// of frame s (K2 + K4) for the batch elements [b0, b0 + nb) of a B_total-element problem
int64_t sequence_workspace_bytes(int B, int H, int W);
int sequence_rearm(void *workspace, int B, int H, int W, cudaStream_t st);
int sequence_headers_group(const float *poses, const float *K, const float *depth, int L, int s, int F, int B_total,
                           int b0, int nb, int H, int W, double sigma, void *workspace, cudaStream_t st);
int fusion_update_group(float *geo, float *col, const int32_t *cin, int32_t *cout, int64_t cap, int64_t max_count,
                        const float *poses, int64_t pose_bs, const float *K, int64_t K_bs, const float *rgb,
                        int64_t rgb_bs, int B_total, int b0, int nb, int s, int H, int W, float dist_th, float dot_th,
                        void *workspace, int32_t *overflow, int32_t *assoc, float2 *rec, bool radii,
                        cudaStream_t st);

// Embeddings of the sequence driver: map rows E (B, cap, D), frames e (B, L, H, W, D) dense, both of `dtype` (0 float32,
// 1 float16, 2 bfloat16); assoc int32 and rec float2, each (B, H, W): K4's record of every frame, read by KE.
// upsampled: the frames are coarse (B, L, eh, ew, D) images, dense, that the upsampled KE samples at the (H, W) pixels.
struct SequenceEmbed {
  void *E;
  const void *e;
  int D, dtype;
  int32_t *assoc;
  float2 *rec;
  bool upsampled;
  int H, W, eh, ew;
};

// the group's K4 record zeroed, K4 done by the caller, then KE of frame s for elements [b0, b0 + nb)
static int32_t *sequence_embed_assoc(const SequenceEmbed *emb, int b0, int nb, int64_t P, cudaStream_t st) {
  if (!emb) return nullptr;
  cudaMemsetAsync(emb->assoc + (int64_t)b0 * P, 0, (size_t)nb * P * sizeof(int32_t), st);
  return emb->assoc;
}
static int sequence_embed_group(const SequenceEmbed *emb, int64_t cap, int L, int s, int b0, int nb, int64_t P,
                                cudaStream_t st) {
  const int64_t es = emb->dtype == 0 ? 4 : 2;
  const int64_t EP = emb->upsampled ? (int64_t)emb->eh * emb->ew : P;  // embedding texels per frame
  EmbedArgs a{(char *)emb->E + (int64_t)b0 * cap * emb->D * es,
              (const char *)emb->e + ((int64_t)b0 * L + s) * EP * emb->D * es, (int64_t)L * EP * emb->D,
              emb->assoc + (int64_t)b0 * P, emb->rec + (int64_t)b0 * P, cap, nb, (int)P, emb->D};
  if (emb->upsampled) {
    a.H = emb->H;
    a.W = emb->W;
    a.eh = emb->eh;
    a.ew = emb->ew;
  }
  return launch_embed_merge_append(a, emb->dtype, st);
}

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
  void *merge_scratch;  // null: no merging of overlapping surfels
  float dot_th;
};

// one group's pruned step s after its K4 (max_count: the host bound of the counts after that K4)
static int sequence_prune_group(const SequencePrune *prune, float *geo, float *col, int32_t *cout, int64_t cap,
                                const float *intrinsics, const float *poses, int64_t pose_bs, int B, int b0, int nb,
                                int s, int H, int W, int64_t max_count, cudaStream_t st) {
  if (!prune->fs_scratch)
    return prune_group(geo, col, cout, cap, prune->ring, prune->t_max + 2, s, prune->t_max, prune->c_stable, B, b0, nb,
                       nullptr, prune->scratch, st);
  const FreeSpaceStep fs{free_space_assoc(prune->fs_scratch, B, H, W, cap, 0), intrinsics, 16, poses, pose_bs, H, W,
                         prune->margin, prune->fs_scratch, max_count, prune->merge_scratch, prune->dot_th, nullptr};
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
// idle GPU (none of them saturates a unit on its own: they are bound by memory latency).  Per frame a group runs K2 and
// K4 only: the frame headers are written kSeqFrames frames at a time, and K4 re-arms what the next frame consumes.
constexpr int kMaxGroups = 4, kMaxDevices = 16;
struct GroupStreams {
  bool ready = false;
  cudaStream_t stream[kMaxGroups];
  cudaEvent_t fork, join[kMaxGroups];
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
      if (cudaEventCreateWithFlags(&gs.join[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
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

static int sequence_driver(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity,
                           int64_t max_count0, const float *depth, const float *rgb, const float *intrinsics,
                           const float *poses, int B, int L, int s_begin, int s_end, int H, int W, float dist_th,
                           float dot_th, double sigma, void *workspace, int32_t *ring, int t_max, float c_stable,
                           void *prune_scratch, int64_t prune_scratch_bytes, float margin, void *fs_scratch,
                           int64_t fs_scratch_bytes, int32_t *overflow_flag, int surfel_radii, void *merge_scratch,
                           int64_t merge_scratch_bytes, const gsx::SequenceEmbed *emb, void *stream) {
  GSX_CHECK_ARG(B >= 0 && L >= 0 && H >= 2 && W >= 2, "gsx_pointfusion_sequence_gt: bad extents");
  GSX_CHECK_ARG(surfel_radii == 0 || surfel_radii == 1,
                "gsx_pointfusion_sequence_gt: surfel_radii must be 0 or 1, not %d", surfel_radii);
  const bool radii = surfel_radii != 0;
  GSX_CHECK_ARG(0 <= s_begin && s_begin <= s_end && s_end <= L, "gsx_pointfusion_sequence_gt: bad frame range");
  GSX_CHECK_ARG(counts && depth && rgb && intrinsics && poses, "gsx_pointfusion_sequence_gt: null pointer");
  GSX_CHECK_ARG(!ring || (t_max >= 0 && c_stable >= 0.0f && (!fs_scratch || margin >= 0.0f)),
                "gsx_pointfusion_sequence_gt: need t_max >= 0, c_stable >= 0, margin >= 0");
  if (B == 0 || s_begin == s_end) return 0;
  GSX_CHECK_ARG(map_geometry && map_colors && workspace && overflow_flag,
                "gsx_pointfusion_sequence_gt: null map / workspace pointer");
  GSX_CHECK_ARG(((reinterpret_cast<uintptr_t>(map_geometry) | reinterpret_cast<uintptr_t>(map_colors) |
                  reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
                "gsx_pointfusion_sequence_gt: map rows and workspace must be 16-byte aligned");
  GSX_CHECK_ARG(capacity <= 0x7fffffffll, "gsx_pointfusion_sequence_gt: capacity must fit int32 (counts are int32)");
  if (ring) {
    GSX_CHECK_ARG(prune_scratch, "gsx_pointfusion_sequence_gt: null prune scratch pointer");
    GSX_CHECK_ARG(prune_scratch_bytes >= gsx::prune_scratch_bytes(B, capacity),
                  "gsx_pointfusion_sequence_gt: prune scratch of %lld bytes < gsx_fusion_prune_scratch_bytes",
                  (long long)prune_scratch_bytes);
    GSX_CHECK_ARG(!fs_scratch || (reinterpret_cast<uintptr_t>(fs_scratch) & 15) == 0,
                  "gsx_pointfusion_sequence_gt: the free-space scratch must be 16-byte aligned");
    GSX_CHECK_ARG(!fs_scratch || (capacity >= 0 &&
                                  fs_scratch_bytes >= gsx::free_space_scratch_bytes(B, H, W, capacity)),
                  "gsx_pointfusion_sequence_gt: free-space scratch of %lld bytes < "
                  "gsx_fusion_free_space_scratch_bytes", (long long)fs_scratch_bytes);
    GSX_CHECK_ARG(!merge_scratch || fs_scratch,
                  "gsx_pointfusion_sequence_gt_merge: merging needs the free-space scratch (margin = inf removes no "
                  "violator)");
    GSX_CHECK_ARG(!merge_scratch || (reinterpret_cast<uintptr_t>(merge_scratch) & 15) == 0,
                  "gsx_pointfusion_sequence_gt_merge: the merge scratch must be 16-byte aligned");
    GSX_CHECK_ARG(!merge_scratch || merge_scratch_bytes >= gsx::merge_scratch_bytes(B, H, W, capacity),
                  "gsx_pointfusion_sequence_gt_merge: merge scratch of %lld bytes < gsx_fusion_merge_scratch_bytes",
                  (long long)merge_scratch_bytes);
  }
  const gsx::SequencePrune prune_args{ring, t_max, c_stable, prune_scratch, margin, fs_scratch, merge_scratch, dot_th};
  const gsx::SequencePrune *prune = ring ? &prune_args : nullptr;
  const int64_t P = (int64_t)H * W;
  // K4's scan epoch is ticket / tiles + 1 and must fit the 30 bits of a look-back state word
  const int64_t tiles = (P + gsx::kTilePix - 1) / gsx::kTilePix;
  GSX_CHECK_ARG((int64_t)(s_end - s_begin) * tiles < (1ll << 30),
                "gsx_pointfusion_sequence_gt: %d frames of %lld K4 tiles in one call; split the call",
                s_end - s_begin, (long long)tiles);
  cudaStream_t user = (cudaStream_t)stream;
  int G = gsx::sequence_groups(B);
  // the group streams and their events are shared by every caller on the device: serialise the enqueue
  std::unique_lock<std::mutex> lock(gsx::g_groups_mutex);
  gsx::GroupStreams *gs = gsx::group_streams();
  // slots, bin counts, scan states, tickets and table flags: zero once per call, so that nothing a failed or abandoned
  // call left behind reaches this one
  int rc = gsx::sequence_rearm(workspace, B, H, W, user);
  if (rc) return rc;
  // frames [s, s + F) of a header block: from s to the end of its kSeqFrames-aligned block or of the call
  auto header_frames = [&](int s) {
    return (s == s_begin || s % gsx::kSeqFrames == 0) ? std::min(gsx::kSeqFrames - s % gsx::kSeqFrames, s_end - s) : 0;
  };
  if (!gs) {
    // no side streams available: everything in order on the caller's stream
    for (int s = s_begin; s < s_end && rc == 0; ++s) {
      int64_t max_count = max_count0 + (int64_t)(s - s_begin) * P;
      if (max_count > capacity) max_count = capacity;
      if (const int F = header_frames(s))
        rc = gsx::sequence_headers_group(poses, intrinsics, depth, L, s, F, B, 0, B, H, W, sigma, workspace, user);
      if (rc == 0)
        rc = gsx::fusion_update_group(map_geometry, map_colors, counts + (int64_t)(s & 1) * B,
                                      counts + (int64_t)((s + 1) & 1) * B, capacity, max_count, poses + (int64_t)s * 16,
                                      (int64_t)L * 16, intrinsics, 16, rgb + (int64_t)s * P * 3, (int64_t)L * P * 3, B, 0, B,
                                      s, H, W, dist_th, dot_th, workspace, overflow_flag,
                                      emb ? gsx::sequence_embed_assoc(emb, 0, B, P, user)
                                          : gsx::sequence_assoc(prune, B, 0, B, H, W, capacity, user),
                                      emb ? emb->rec : nullptr, radii, user);
      if (rc == 0 && emb) rc = gsx::sequence_embed_group(emb, capacity, L, s, 0, B, P, user);
      if (rc == 0 && prune)
        rc = gsx::sequence_prune_group(prune, map_geometry, map_colors, counts + (int64_t)((s + 1) & 1) * B, capacity,
                                       intrinsics, poses + (int64_t)s * 16, (int64_t)L * 16, B, 0, B, s, H, W,
                                       std::min(max_count + P, capacity), user);
    }
    return rc;
  }
  cudaEventRecord(gs->fork, user);
  for (int g = 0; g < G; ++g) cudaStreamWaitEvent(gs->stream[g], gs->fork, 0);
  for (int s = s_begin; s < s_end && rc == 0; ++s) {
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
      // the group's headers of the next block, after its K4 of the frames that read the block's slots before
      if (const int F = header_frames(s))
        rc = gsx::sequence_headers_group(poses, intrinsics, depth, L, s, F, B, b0, b1 - b0, H, W, sigma, workspace,
                                         gs->stream[g]);
      if (rc) break;
      rc = gsx::fusion_update_group(map_geometry, map_colors, cin, cout, capacity, max_count, poses + (int64_t)s * 16,
                                    (int64_t)L * 16, intrinsics, 16, rgb + (int64_t)s * P * 3, (int64_t)L * P * 3, B, b0,
                                    b1 - b0, s, H, W, dist_th, dot_th, workspace, overflow_flag,
                                    emb ? gsx::sequence_embed_assoc(emb, b0, b1 - b0, P, gs->stream[g])
                                        : gsx::sequence_assoc(prune, B, b0, b1 - b0, H, W, capacity, gs->stream[g]),
                                    emb ? emb->rec : nullptr, radii, gs->stream[g]);
      if (rc == 0 && emb) rc = gsx::sequence_embed_group(emb, capacity, L, s, b0, b1 - b0, P, gs->stream[g]);
      if (rc == 0 && prune)
        rc = gsx::sequence_prune_group(prune, map_geometry, map_colors, cout, capacity, intrinsics,
                                       poses + (int64_t)s * 16, (int64_t)L * 16, B, b0, b1 - b0, s, H, W,
                                       std::min(max_count + P, capacity), gs->stream[g]);
    }
  }
  // join ALWAYS, also after a failed launch: whatever was already enqueued on the internal streams stays ordered before
  // anything the caller enqueues next on its stream
  for (int g = 0; g < G; ++g) {
    cudaEventRecord(gs->join[g], gs->stream[g]);
    cudaStreamWaitEvent(user, gs->join[g], 0);
  }
  return rc;
}

extern "C" int gsx_pointfusion_sequence_gt_merge(float *map_geometry, float *map_colors, int32_t *counts,
                                                 int64_t capacity, int64_t max_count0, const float *depth,
                                                 const float *rgb, const float *intrinsics, const float *poses, int B,
                                                 int L, int s_begin, int s_end, int H, int W, float dist_th,
                                                 float dot_th, double sigma, void *workspace, int32_t *ring, int t_max,
                                                 float c_stable, void *prune_scratch, int64_t prune_scratch_bytes,
                                                 float margin, void *fs_scratch, int64_t fs_scratch_bytes,
                                                 int32_t *overflow_flag, int surfel_radii, void *merge_scratch,
                                                 int64_t merge_scratch_bytes, void *stream) {
  return sequence_driver(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb, intrinsics, poses, B, L,
                         s_begin, s_end, H, W, dist_th, dot_th, sigma, workspace, ring, t_max, c_stable, prune_scratch,
                         prune_scratch_bytes, margin, fs_scratch, fs_scratch_bytes, overflow_flag, surfel_radii,
                         merge_scratch, merge_scratch_bytes, nullptr, stream);
}

extern "C" int gsx_pointfusion_sequence_gt_emb(float *map_geometry, float *map_colors, int32_t *counts,
                                               int64_t capacity, int64_t max_count0, const float *depth,
                                               const float *rgb, const float *intrinsics, const float *poses, int B,
                                               int L, int s_begin, int s_end, int H, int W, float dist_th,
                                               float dot_th, double sigma, void *workspace, int32_t *overflow_flag,
                                               int surfel_radii, void *map_embeddings,
                                               const void *frame_embeddings, int D, int dtype, int32_t *assoc,
                                               float *merge_rec, void *stream) {
  GSX_CHECK_ARG(D >= 1 && dtype >= 0 && dtype <= 2,
                "gsx_pointfusion_sequence_gt_emb: need D >= 1 and dtype 0 (float32), 1 (float16) or 2 (bfloat16)");
  GSX_CHECK_ARG(B == 0 || s_begin == s_end || (map_embeddings && frame_embeddings && assoc && merge_rec),
                "gsx_pointfusion_sequence_gt_emb: null embedding pointer");
  GSX_CHECK_ARG(((reinterpret_cast<uintptr_t>(map_embeddings) | reinterpret_cast<uintptr_t>(frame_embeddings)) &
                 (dtype == 0 ? 3 : 1)) == 0 && (reinterpret_cast<uintptr_t>(merge_rec) & 7) == 0,
                "gsx_pointfusion_sequence_gt_emb: misaligned embeddings or record");
  const gsx::SequenceEmbed emb{map_embeddings, frame_embeddings, D, dtype, assoc,
                               reinterpret_cast<float2 *>(merge_rec)};
  return sequence_driver(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb, intrinsics, poses, B, L,
                         s_begin, s_end, H, W, dist_th, dot_th, sigma, workspace, nullptr, 0, 0.0f, nullptr, 0, 0.0f,
                         nullptr, 0, overflow_flag, surfel_radii, nullptr, 0, &emb, stream);
}

extern "C" int gsx_pointfusion_sequence_gt_emb_upsampled(float *map_geometry, float *map_colors, int32_t *counts,
                                                         int64_t capacity, int64_t max_count0, const float *depth,
                                                         const float *rgb, const float *intrinsics, const float *poses,
                                                         int B, int L, int s_begin, int s_end, int H, int W,
                                                         float dist_th, float dot_th, double sigma, void *workspace,
                                                         int32_t *overflow_flag, int surfel_radii,
                                                         void *map_embeddings, const void *frame_embeddings, int eh,
                                                         int ew, int D, int dtype, int32_t *assoc, float *merge_rec,
                                                         void *stream) {
  GSX_CHECK_ARG(D >= 1 && dtype >= 0 && dtype <= 2, "gsx_pointfusion_sequence_gt_emb_upsampled: need D >= 1 and "
                "dtype 0 (float32), 1 (float16) or 2 (bfloat16)");
  GSX_CHECK_ARG(eh >= 1 && eh <= H && ew >= 1 && ew <= W,
                "gsx_pointfusion_sequence_gt_emb_upsampled: the embedding image (%d, %d) must be at most (H, W) = "
                "(%d, %d) and at least (1, 1)", eh, ew, H, W);
  GSX_CHECK_ARG(B == 0 || s_begin == s_end || (map_embeddings && frame_embeddings && assoc && merge_rec),
                "gsx_pointfusion_sequence_gt_emb_upsampled: null embedding pointer");
  GSX_CHECK_ARG(((reinterpret_cast<uintptr_t>(map_embeddings) | reinterpret_cast<uintptr_t>(frame_embeddings)) &
                 (dtype == 0 ? 3 : 1)) == 0 && (reinterpret_cast<uintptr_t>(merge_rec) & 7) == 0 &&
                (reinterpret_cast<uintptr_t>(assoc) & 3) == 0,
                "gsx_pointfusion_sequence_gt_emb_upsampled: misaligned embeddings, assoc or record");
  const gsx::SequenceEmbed emb{map_embeddings, frame_embeddings, D, dtype, assoc,
                               reinterpret_cast<float2 *>(merge_rec), true, H, W, eh, ew};
  return sequence_driver(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb, intrinsics, poses, B, L,
                         s_begin, s_end, H, W, dist_th, dot_th, sigma, workspace, nullptr, 0, 0.0f, nullptr, 0, 0.0f,
                         nullptr, 0, overflow_flag, surfel_radii, nullptr, 0, &emb, stream);
}

extern "C" int gsx_pointfusion_sequence_gt_radii(float *map_geometry, float *map_colors, int32_t *counts,
                                                 int64_t capacity, int64_t max_count0, const float *depth,
                                                 const float *rgb, const float *intrinsics, const float *poses, int B,
                                                 int L, int s_begin, int s_end, int H, int W, float dist_th,
                                                 float dot_th, double sigma, void *workspace, int32_t *ring, int t_max,
                                                 float c_stable, void *prune_scratch, int64_t prune_scratch_bytes,
                                                 float margin, void *fs_scratch, int64_t fs_scratch_bytes,
                                                 int32_t *overflow_flag, int surfel_radii, void *stream) {
  return gsx_pointfusion_sequence_gt_merge(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb,
                                           intrinsics, poses, B, L, s_begin, s_end, H, W, dist_th, dot_th, sigma,
                                           workspace, ring, t_max, c_stable, prune_scratch, prune_scratch_bytes, margin,
                                           fs_scratch, fs_scratch_bytes, overflow_flag, surfel_radii, nullptr, 0,
                                           stream);
}

extern "C" int gsx_pointfusion_sequence_gt(float *map_geometry, float *map_colors, int32_t *counts, int64_t capacity,
                                           int64_t max_count0, const float *depth, const float *rgb,
                                           const float *intrinsics, const float *poses, int B, int L, int s_begin,
                                           int s_end, int H, int W, float dist_th, float dot_th, double sigma,
                                           void *workspace, int32_t *ring, int t_max, float c_stable,
                                           void *prune_scratch, int64_t prune_scratch_bytes, float margin,
                                           void *fs_scratch, int64_t fs_scratch_bytes, int32_t *overflow_flag,
                                           void *stream) {
  return gsx_pointfusion_sequence_gt_radii(map_geometry, map_colors, counts, capacity, max_count0, depth, rgb,
                                           intrinsics, poses, B, L, s_begin, s_end, H, W, dist_th, dot_th, sigma,
                                           workspace, ring, t_max, c_stable, prune_scratch, prune_scratch_bytes, margin,
                                           fs_scratch, fs_scratch_bytes, overflow_flag, 0, stream);
}

extern "C" int64_t gsx_pointfusion_sequence_workspace_bytes(int B, int H, int W) {
  if (B < 0 || H < 0 || W < 0) return -1;
  return gsx::sequence_workspace_bytes(B, H, W);
}
