"""Per-kernel timing of the PointFusion(odom='gt') sequence, used by bench.py for the roofline line.

Runs exactly the launches of gsx_pointfusion_sequence_gt (K2/K3 -> K4 per frame, same arguments, on a workspace
re-armed once before frame 0 and kept armed by K4 from frame to frame), but from Python with a CUDA event between
launches, and reads the device-side counters after each frame so the
algorithmic byte count of every launch comes from the run itself (SURVEY.md §8d).  The step's algorithmic bytes are
SURVEY's fusion-step formula  16*P + 12*M + 16*A + 12*U + 40*U + 40*New;  they are attributed to the kernels as

    K2  project+select                           12*M + 16*A        (map positions; normal+ccount of active)
    K4  merge+append                             16*P + 52*U + 40*New  (depth and rgb; read colour 12 + write 40 per
                                                                        merged point; write 40 per new point)

K2 and K4 read the depth image: every pixel's depth once in K4, the depth stencils under the projections in K2 (an
intermediate re-read, not algorithmic traffic).
"""
import torch

from . import _C
from .slam.fusionutils import _Workspace
from .structures.pointclouds import Pointclouds


def profile_pointfusion_gt(depth, rgb, K, poses, dist_th, dot_th, sigma):
    """depth (B,L,H,W,1), rgb (B,L,H,W,3), K (B,1,4,4), poses (B,L,4,4): dense CUDA tensors.
    Returns dict kernel -> list of (milliseconds, algorithmic_bytes) per launch, plus per-frame counters."""
    dev = depth.device
    B, L, H, W, _ = depth.shape
    P = H * W
    lib = _C.lib()
    pc = Pointclouds(device=dev)
    pc._allocate(B, L * P, 1, zero=False)
    ws = _Workspace.get(dev, B, H, W)
    off = lib.gsx_fusion_workspace_stats_offset(B, H, W)
    stats = ws.buf[off: off + B * 16].view(torch.int64).view(B, 2)
    stream = _C.stream_ptr(dev)
    out = {"K2_project_select": [], "K4_merge_append": []}
    frames = []
    prev_stats = stats.sum(0).tolist()
    prev_counts = [0] * B
    for s in range(L):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        cin = pc._counts_dev[s & 1]
        cout = pc._counts_dev[(s + 1) & 1]
        # the frame's headers (the driver writes them for a block of frames at once); re-arm once, before frame 0
        _C.check(lib.gsx_fusion_sequence_frame(
            depth.data_ptr() + 4 * s * P, L * P, _C.ptr(K), 16, poses.data_ptr() + 64 * s, L * 16, B, H, W,
            float(sigma), 1 if s == 0 else 0, _C.ptr(ws.buf), stream), "frame headers")
        ev[0].record()
        _C.check(lib.gsx_fusion_project_select(
            _C.ptr(pc._geo), _C.ptr(cin), pc.capacity, min(s * P, pc.capacity), poses.data_ptr() + 64 * s, L * 16,
            _C.ptr(K), 16, B, H, W, float(dist_th), float(dot_th), _C.ptr(ws.buf), stream), "K2")
        ev[1].record()
        _C.check(lib.gsx_fusion_merge_append(
            _C.ptr(pc._geo), _C.ptr(pc._col), 1, _C.ptr(cin), _C.ptr(cout), pc.capacity, rgb.data_ptr() + 12 * s * P,
            L * P * 3, B, H, W, _C.ptr(ws.buf), _C.ptr(pc._overflow_flag()), None, stream), "K4")
        ev[2].record()
        torch.cuda.synchronize(dev)
        counts = cout.tolist()
        cur_stats = stats.sum(0).tolist()
        M = sum(prev_counts)
        New = sum(counts) - M
        A = cur_stats[0] - prev_stats[0]
        U = cur_stats[1] - prev_stats[1]
        if s > 0:
            out["K2_project_select"].append((ev[0].elapsed_time(ev[1]), 12 * M + 16 * A))
        out["K4_merge_append"].append((ev[1].elapsed_time(ev[2]), 16 * B * P + 52 * U + 40 * New))
        frames.append({"frame": s, "map_points": M, "active": A, "merged": U, "new": New})
        prev_counts, prev_stats = counts, cur_stats
    return out, frames
