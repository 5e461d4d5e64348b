"""Times PointFusion with ICP / gradICP odometry under the two associations, 'nn' (exact 1-NN, the default) and
'projective' (the map rendered from the previous pose), at 640x480, B=8, L=8, 20 iterations, dsratio 4 (and 1 for the
projective association), on the corner-facing scene of bench.py's ICP leg (yaw0=0.6).

Whole-sequence calls and the localisation of the last frame alone are timed with CUDA events over warmed-up calls, the
configurations alternated within each repetition; the median over repetitions is printed.  Per-kernel times come from a
separate torch.profiler run of the localisation calls.  Prints the GPU's name and power limit first."""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gradslam_b200 as gs
from gradslam_b200.odometry.icputils import localize_against_map, localize_projective
from gradslam_b200.synthetic import make_sequence

B, L, H, W, ITERS, REPS = 8, 8, 480, 640, 20, 7
CONFIGS = [(odom, assoc, ds) for odom in ("gradicp", "icp") for assoc, ds in (("nn", 4), ("projective", 4),
                                                                               ("projective", 1))]


def main():
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", torch.cuda.get_device_name(dev), "|", q.stdout.strip().splitlines()[0] if q.stdout else "n/a")
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=100, yaw0=0.6)
    frames = gs.RGBDImages(rgb.to(dev), depth.to(dev), K.to(dev), poses.to(dev))
    pc_map, _ = gs.PointFusion(odom="gt", device=dev)(frames[:, : L - 1])
    slams = {c: gs.PointFusion(odom=c[0], association=c[1], dsratio=c[2], numiters=ITERS, device=dev) for c in CONFIGS}

    def localize(c):
        live, prev = frames[:, L - 1], frames[:, L - 2]
        live.poses = prev.poses
        fn = localize_projective if c[1] == "projective" else localize_against_map
        return fn(pc_map, live, prev, c[2], slams[c].odomprov)

    seq, loc, err = {c: [] for c in CONFIGS}, {c: [] for c in CONFIGS}, {}
    for c in CONFIGS:  # warm-up of every shape
        slams[c](frames)
        localize(c)
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(REPS):
        for c in CONFIGS:
            e0.record()
            _, rec = slams[c](frames)
            e1.record()
            torch.cuda.synchronize(dev)
            seq[c].append(e0.elapsed_time(e1))
            err[c] = float((rec.cpu() - poses).abs().max())
            e0.record()
            for _ in range(5):
                localize(c)
            e1.record()
            torch.cuda.synchronize(dev)
            loc[c].append(e0.elapsed_time(e1) / 5)
    print("%-9s %-11s %3s %12s %10s %14s %12s" % ("odom", "association", "ds", "ms/sequence", "frames/s",
                                                   "ms/localise", "max|p-gt|"))
    for c in CONFIGS:
        ms = statistics.median(seq[c])
        print("%-9s %-11s %3d %12.2f %10.0f %14.3f %12.2e   (sequence min/max %.2f/%.2f ms)" % (
            c[0], c[1], c[2], ms, B * L / ms * 1e3, statistics.median(loc[c]), err[c], min(seq[c]), max(seq[c])))

    from torch.profiler import ProfilerActivity, profile

    for c in CONFIGS:
        if c[0] != "gradicp":
            continue
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                localize(c)
            torch.cuda.synchronize(dev)
        print("\nper-kernel, localisation of one step, %s association=%s ds=%d (5 calls):" % c)
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12))


if __name__ == "__main__":
    main()
