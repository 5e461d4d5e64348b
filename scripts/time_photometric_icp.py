"""What the photometric term (ICPSLAM / PointFusion(photometric_weight=w), gsx_icp_localize_projective) costs and
gains, at 640x480, B=8, gradICP with 20 iterations at dsratio 4, M = 0 (one pixel per surfel) and 3 (disk splats):

  1. the fused localisation of frame 31 against the radii map of frames 0..30 of the bench's inputs
     (make_sequence(8, 32, 480, 640, seed=0)), w = 0 vs w = 0.1, per call: CUDA events over 5 calls, the four
     configurations alternated within each repetition, the median over repetitions;
  2. per-kernel times per launch (k_icp_gather_src, k_icp_model_intensity, k_icp_proj_linearize) from a separate
     torch.profiler run;
  3. the tracking error of PointFusion(odom='gradicp', association='projective', surfel_radii=True) over
     make_textured_sequence(8, 32, 480, 640, seed=0) with yaw0 = 0 (far wall only) and 0.6 (corner), w = 0 vs 0.1:
     final and maximum translational (m) and rotational (degrees) error against the ground-truth poses (worst element).

Prints the GPU's name, power limit and maximum SM clock first."""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gradslam_b200 as gs
from gradslam_b200.odometry.icputils import localize_projective
from gradslam_b200.synthetic import make_sequence, make_textured_sequence

B, L, H, W, ITERS, DS, REPS = 8, 32, 480, 640, 20, 4, 7
WEIGHT = 0.1
CONFIGS = [(M, w) for M in (0, 3) for w in (0.0, WEIGHT)]
KERNELS = ("k_icp_gather_src", "k_icp_model_intensity", "k_icp_proj_linearize")


def main():
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", torch.cuda.get_device_name(dev), "|", q.stdout.strip().splitlines()[0] if q.stdout else "n/a")
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    frames = gs.RGBDImages(rgb.to(dev), depth.to(dev), K.to(dev), poses.to(dev))
    pc, _ = gs.PointFusion(odom="gt", surfel_radii=True, device=dev)(frames[:, : L - 1])
    odom = gs.PointFusion(odom="gradicp", association="projective", numiters=ITERS, dsratio=DS, device=dev).odomprov
    live, prev = frames[:, L - 1], frames[:, L - 2]
    live.poses = prev.poses
    localize = lambda M, w: localize_projective(pc, live, prev, DS, odom, M, w)

    # 1. time per fused localisation
    times = {c: [] for c in CONFIGS}
    for c in CONFIGS:
        localize(*c)
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(REPS):
        for c in CONFIGS:
            e0.record()
            for _ in range(5):
                localize(*c)
            e1.record()
            torch.cuda.synchronize(dev)
            times[c].append(e0.elapsed_time(e1) / 5)
    print("\n1. fused localisation of one step (B=%d, %dx%d, gradICP %d iterations, ds %d)" % (B, W, H, ITERS, DS))
    for c in CONFIGS:
        print("  M=%d w=%-4g %.3f ms/step  (min/max %.3f/%.3f over %d repetitions)" % (
            c[0], c[1], statistics.median(times[c]), min(times[c]), max(times[c]), REPS))

    # 2. per-kernel times
    from torch.profiler import ProfilerActivity, profile

    print("\n2. per-kernel us per launch (torch.profiler, 5 calls per configuration)")
    for c in CONFIGS:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                localize(*c)
            torch.cuda.synchronize(dev)
        for ev in prof.key_averages():
            name = ev.key.replace("void ", "").replace("gsx::", "").replace("(", " (")
            short = name.split(" (")[0].replace("<(bool)0>", "<false>").replace("<(bool)1>", "<true>")
            if any(short.startswith(k) for k in KERNELS):
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                print("  M=%d w=%-4g %-30s %9.2f us x %d" % (c[0], c[1], short, t / max(ev.count, 1), ev.count))

    # 3. tracking error
    print("\n3. PointFusion(gradicp, projective, surfel_radii) on make_textured_sequence, L=%d, B=%d" % (L, B))
    print("  %-5s %3s %5s %12s %12s %12s %12s" % ("yaw0", "M", "w", "final t (m)", "max t (m)", "final R (deg)",
                                                 "max R (deg)"))
    for yaw0 in (0.0, 0.6):
        r, d, k, p = make_textured_sequence(B, L, H, W, seed=0, yaw0=yaw0)
        fr = gs.RGBDImages(r.to(dev), d.to(dev), k.to(dev), p.to(dev))
        for M in (0, 3):
            for w in (0.0, WEIGHT):
                slam = gs.PointFusion(odom="gradicp", association="projective", surfel_radii=True, target_splat_px=M,
                                      photometric_weight=w, numiters=ITERS, dsratio=DS, device=dev)
                _, rec = slam(fr)
                rec, gt = rec.cpu().double(), p.double()
                et = (rec[..., :3, 3] - gt[..., :3, 3]).norm(dim=-1)
                rel = gt[..., :3, :3].transpose(-1, -2) @ rec[..., :3, :3]
                er = torch.rad2deg(torch.acos(((rel.diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2).clamp(-1, 1)))
                print("  %-5g %3d %5g %12.4f %12.4f %12.3f %12.3f" % (yaw0, M, w, et[:, -1].max(), et.max(),
                                                                    er[:, -1].max(), er.max()), flush=True)


if __name__ == "__main__":
    main()
