"""What d/dK costs in the benchmark's config 3: ICPSLAM(odom='gradicp', numiters=10, dsratio=4) at 640x480, B=8, L=2,
inputs resident, loss = poses.sum(), depth and poses requiring grad, with and without K.requires_grad.

  1. forward and backward per call (CUDA events), the two settings alternated within each repetition, the median over
     repetitions;
  2. per launch of the K1 backward kernels (k_backproject_normals_bwd<false>/<true>, k_intrinsics_grad_reduce) from a
     separate torch.profiler run;
  3. whether the poses, d/d depth and d/d poses are bit for bit the same in two runs of one setting, and in the two
     settings.

Prints the GPU's name, power limit and maximum SM clock first."""
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gradslam_b200 as gs
from gradslam_b200.synthetic import make_sequence

B, L, H, W, ITERS, DS, REPS, CALLS = 8, 2, 480, 640, 10, 4, 7, 3
KERNELS = ("k_backproject_normals_bwd", "k_intrinsics_grad_reduce", "k_pose_grad_reduce")


def main():
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("GPU:", torch.cuda.get_device_name(dev), "|", q.stdout.strip().splitlines()[0] if q.stdout else "n/a")
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0, yaw0=0.6)
    rgb, depth, K, poses = rgb.to(dev), depth.to(dev), K.to(dev), poses.to(dev)
    slam = gs.ICPSLAM(odom="gradicp", numiters=ITERS, dsratio=DS, device=dev)

    def step(k_grad):
        d, p, k = depth.clone().requires_grad_(True), poses.clone().requires_grad_(True), K.clone().requires_grad_(k_grad)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        _, rec = slam(gs.RGBDImages(rgb, d, k, p))
        ev[1].record()
        rec.sum().backward()
        ev[2].record()
        torch.cuda.synchronize(dev)
        return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), (rec.detach(), d.grad, p.grad, k.grad)

    for k_grad in (False, True):
        step(k_grad)
        step(k_grad)
    times = {k: ([], []) for k in (False, True)}
    for _ in range(REPS):
        for k_grad in (False, True):
            f = b = 0.0
            for _ in range(CALLS):
                fm, bm, _ = step(k_grad)
                f, b = f + fm / CALLS, b + bm / CALLS
            times[k_grad][0].append(f)
            times[k_grad][1].append(b)
    print("\n1. config 3 (ICPSLAM gradicp %d iterations, ds %d, %dx%d, B=%d, L=%d), ms per call, median of %d "
          "repetitions of %d calls" % (ITERS, DS, W, H, B, L, REPS, CALLS))
    for k_grad in (False, True):
        f, b = times[k_grad]
        print("  K.requires_grad=%-5s forward %.3f (min/max %.3f/%.3f)  backward %.3f (min/max %.3f/%.3f)" % (
            k_grad, statistics.median(f), min(f), max(f), statistics.median(b), min(b), max(b)))

    from torch.profiler import ProfilerActivity, profile

    print("\n2. K1 backward kernels, us per launch (torch.profiler, 3 calls per setting)")
    for k_grad in (False, True):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                step(k_grad)
        for ev in prof.key_averages():
            name = ev.key.replace("void ", "").replace("gsx::", "")
            short = name.split("(")[0].replace("<(bool)0>", "<false>").replace("<(bool)1>", "<true>")
            if any(short.startswith(k) for k in KERNELS):
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                print("  K.requires_grad=%-5s %-36s %9.2f us x %d" % (k_grad, short, t / max(ev.count, 1), ev.count))

    runs = [step(False)[2], step(False)[2], step(True)[2]]
    print("\n3. bit for bit (poses, d/d depth, d/d poses): two runs without K.requires_grad %s; without vs with %s" % (
        [torch.equal(x, y) for x, y in zip(runs[0][:3], runs[1][:3])],
        [torch.equal(x, y) for x, y in zip(runs[0][:3], runs[2][:3])]))
    g_K = runs[2][3][0, 0]
    print("   d/dK of element 0 (fx, cx, fy, cy):", [float(g_K[i, j]) for i, j in ((0, 0), (0, 2), (1, 1), (1, 2))])


if __name__ == "__main__":
    main()
