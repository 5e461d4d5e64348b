"""What the Huber weights (ICPSLAM / PointFusion(huber_delta=, photometric_huber_delta=), finite scales of the ICP
entry points) cost, at 640x480, B=8, gradICP with 20 iterations at dsratio 4, on the bench's inputs
(make_sequence(8, 32, 480, 640, seed=0)): the localisation of frame 31 against the map of frames 0..30.

  1. the fused step per call, with the scales unset and set, the two alternated within each repetition (CUDA events
     over 5 calls, the median over repetitions):
       1-NN association (gsx_icp_localize at delta = +inf vs 0.02 m);
       projective association at M = 0 and M = 3, w = 0 and w = 0.1 (gsx_icp_localize_projective at +inf vs
       delta = 0.02 m and, with w, delta_p = 0.05);
  2. config 3 (ICPSLAM(odom='gradicp', numiters=10) at B=8, two frames, the depth requiring grad): forward and backward
     of the taped run with and without delta.

Prints the GPU's name, power limit and maximum SM clock first."""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gradslam_b200 as gs
from gradslam_b200.synthetic import make_sequence

B, L, H, W, ITERS, DS, REPS = 8, 32, 480, 640, 20, 4, 7
DELTA, DELTA_P, WEIGHT = 0.02, 0.05, 0.1


def _time(fns, reps, calls):
    """{name: fn} -> {name: median ms per call}, the functions alternated within each repetition."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            e0.record()
            for _ in range(calls):
                f()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / calls)
    return {k: (statistics.median(v), min(v), max(v)) for k, v in times.items()}


def main():
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", torch.cuda.get_device_name(dev), "|", q.stdout.strip().splitlines()[0] if q.stdout else "n/a")
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    frames = gs.RGBDImages(rgb.to(dev), depth.to(dev), K.to(dev), poses.to(dev))
    live, prev = frames[:, L - 1], frames[:, L - 2]

    print("\n1. fused localisation of one step (B=%d, %dx%d, gradICP %d iterations, ds %d), ms per step" % (
        B, W, H, ITERS, DS))
    pc_nn, _ = gs.PointFusion(odom="gt", device=dev)(frames[:, : L - 1])
    pc_pr, _ = gs.PointFusion(odom="gt", surfel_radii=True, device=dev)(frames[:, : L - 1])
    configs = [("nn", pc_nn, {})] + [("projective M=%d w=%g" % (M, w), pc_pr,
                                      dict(association="projective", target_splat_px=M, photometric_weight=w))
                                     for M in (0, 3) for w in (0.0, WEIGHT)]
    for name, pc, kw in configs:
        fns = {}
        for robust in (False, True):
            extra = {}
            if robust:
                extra = dict(huber_delta=DELTA)
                if kw.get("photometric_weight"):
                    extra["photometric_huber_delta"] = DELTA_P
            slam = gs.PointFusion(odom="gradicp", numiters=ITERS, dsratio=DS, surfel_radii=pc is pc_pr, device=dev,
                                  **kw, **extra)
            fns[robust] = lambda slam=slam, pc=pc: slam._localize(pc, live, prev)
        t = _time(fns, REPS, 5)
        print("  %-24s unset %.3f  set %.3f  (+%.1f %%)   min/max unset %.3f/%.3f set %.3f/%.3f" % (
            name, t[False][0], t[True][0], 100 * (t[True][0] / t[False][0] - 1), t[False][1], t[False][2], t[True][1],
            t[True][2]), flush=True)

    print("\n2. config 3 (ICPSLAM(odom='gradicp', numiters=10), make_sequence(8, 2, 480, 640, seed=0, yaw0=0.6), the "
          "depth requiring grad): ms per forward + backward")
    r2, d2, k2, p2 = make_sequence(B, 2, H, W, seed=0, yaw0=0.6)
    d2 = d2.to(dev).requires_grad_(True)
    fr2 = gs.RGBDImages(r2.to(dev), d2, k2.to(dev), p2.to(dev))
    fns = {}
    for robust in (False, True):
        slam = gs.ICPSLAM(odom="gradicp", numiters=10, device=dev, **(dict(huber_delta=DELTA) if robust else {}))

        def step(slam=slam):
            _, rec = slam(fr2)
            rec.sum().backward()
        fns[robust] = step
    t = _time(fns, 5, 2)
    print("  unset %.3f  set %.3f  (+%.1f %%)" % (t[False][0], t[True][0], 100 * (t[True][0] / t[False][0] - 1)))


if __name__ == "__main__":
    main()
