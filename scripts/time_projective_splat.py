"""What splatted ICP targets (ICPSLAM / PointFusion(target_splat_px=M), gsx_icp_localize_projective) cost and
gain, at 640x480, B=8, gradICP with 20 iterations at dsratio 4, on the bench's inputs (make_sequence(8, 32, 480, 640,
seed=0)), with M = 0 (one pixel per surfel), 1 and 3:

  1. the fused localisation of frame 31 against the radii map of frames 0..30, per call: CUDA events over 5 calls, the
     configurations alternated within each repetition, the median over repetitions;
  2. per-kernel times per launch (R1 / R1d, R2w / R2w<true>, K5p) from a separate torch.profiler run;
  3. the fraction of source points associated at the first iteration (source at the previous pose) and after the last
     (source at the returned pose), M = 0 vs 3;
  4. the tracking error of PointFusion(odom='gradicp', association='projective', surfel_radii=True) over make_sequence
     and make_dynamic_sequence (a box in frames [8, 24)), B=8, L=32: final and maximum translational (m) and rotational
     (degrees) error against the ground-truth poses (the worst element), M = 0 vs 3, dist_thresh None and 0.01.

Prints the GPU's name, power limit and maximum SM clock first."""
import math
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gradslam_b200 as gs
from gradslam_b200.odometry.icputils import (downsample_rgbdimages, localize_projective, project_associate,
                                             projective_targets)
from gradslam_b200.synthetic import make_dynamic_sequence, make_sequence

B, L, H, W, ITERS, DS, REPS = 8, 32, 480, 640, 20, 4, 7
SPLATS = (0, 1, 3)
KERNELS = ("k_render_zbuffer", "k_render_splat", "k_render_resolve_world<false>", "k_render_resolve_world<true>",
           "k_icp_proj_linearize")


def main():
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", torch.cuda.get_device_name(dev), "|", q.stdout.strip().splitlines()[0] if q.stdout else "n/a")
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    frames = gs.RGBDImages(rgb.to(dev), depth.to(dev), K.to(dev), poses.to(dev))
    pc, _ = gs.PointFusion(odom="gt", surfel_radii=True, device=dev)(frames[:, : L - 1])
    print("map: %s rows per element" % pc.num_points_per_pointcloud.tolist())
    odom = gs.PointFusion(odom="gradicp", association="projective", numiters=ITERS, dsratio=DS, device=dev).odomprov
    live, prev = frames[:, L - 1], frames[:, L - 2]
    live.poses = prev.poses
    localize = lambda M: localize_projective(pc, live, prev, DS, odom, M)

    # 1. time per fused localisation
    times = {M: [] for M in SPLATS}
    for M in SPLATS:
        localize(M)
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(REPS):
        for M in SPLATS:
            e0.record()
            for _ in range(5):
                localize(M)
            e1.record()
            torch.cuda.synchronize(dev)
            times[M].append(e0.elapsed_time(e1) / 5)
    print("\n1. fused localisation of one step (B=%d, %dx%d, gradICP %d iterations, ds %d)" % (B, W, H, ITERS, DS))
    for M in SPLATS:
        print("  M=%d  %.3f ms/step  (min/max %.3f/%.3f over %d repetitions)" % (
            M, statistics.median(times[M]), min(times[M]), max(times[M]), REPS))

    # 2. per-kernel times
    from torch.profiler import ProfilerActivity, profile

    print("\n2. per-kernel us per launch (torch.profiler, 5 calls per M)")
    for M in (0, 3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                localize(M)
            torch.cuda.synchronize(dev)
        for ev in prof.key_averages():
            name = ev.key.replace("void ", "").replace("gsx::", "").replace("(", " (")
            short = name.split(" (")[0].replace("<(bool)0>", "<false>").replace("<(bool)1>", "<true>")
            if any(short.startswith(k) for k in KERNELS):
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                print("  M=%d  %-34s %9.1f us x %d" % (M, short, t / max(ev.count, 1), ev.count))

    # 3. associated fraction at the first iteration and after the last
    print("\n3. source points associated (all elements), first iteration / after the last")
    Kd = K[:, 0].to(dev).contiguous()
    for M in (0, 3):
        idx, tgt_p, _ = projective_targets(pc, Kd, prev.poses[:, 0], H, W, M)
        out = localize(M)
        fr = []
        for pose in (prev.poses, out):
            f = gs.RGBDImages(live.rgb_image, live.depth_image, live.intrinsics, pose)
            src = downsample_rgbdimages(f, DS)
            counts = src._counts_dev[src._cur]
            _, j = project_associate(src.points_padded, counts, tgt_p, idx, prev.poses[:, 0], Kd, H, W,
                                     odom.dist_thresh)
            fr.append(float((j >= 0).sum()) / float(counts.sum()))
        print("  M=%d  %.4f / %.4f   (pixels covered %.4f)" % (M, fr[0], fr[1], float((idx >= 0).float().mean())))

    # 4. tracking error
    print("\n4. PointFusion(gradicp, projective, surfel_radii) tracking error over L=%d, B=%d" % (L, B))
    print("  %-9s %4s %6s %12s %12s %12s %12s" % ("sequence", "M", "dth", "final t (m)", "max t (m)", "final R (deg)",
                                                  "max R (deg)"))
    for name, seq in (("static", make_sequence(B, L, H, W, seed=0)),
                      ("dynamic", make_dynamic_sequence(B, L, H, W, 8, 24, seed=0))):
        r, d, k, p = seq
        fr = gs.RGBDImages(r.to(dev), d.to(dev), k.to(dev), p.to(dev))
        for dth in (None, 0.01):
            for M in (0, 3):
                slam = gs.PointFusion(odom="gradicp", association="projective", surfel_radii=True, target_splat_px=M,
                                      dist_thresh=dth, numiters=ITERS, dsratio=DS, device=dev)
                _, rec = slam(fr)
                rec = rec.cpu().double()
                gt = p.double()
                et = (rec[..., :3, 3] - gt[..., :3, 3]).norm(dim=-1)  # (B, L)
                rel = gt[..., :3, :3].transpose(-1, -2) @ rec[..., :3, :3]
                cos = ((rel.diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2).clamp(-1, 1)
                er = torch.rad2deg(torch.acos(cos))
                print("  %-9s %4d %6s %12.4f %12.4f %12.3f %12.3f" % (name, M, dth, et[:, -1].max(), et.max(),
                                                                     er[:, -1].max(), er.max()))


if __name__ == "__main__":
    main()
