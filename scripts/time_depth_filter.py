"""Timing of the bilateral depth filter (gsx_depth_bilateral / gsx_depth_bilateral_bwd) and of its cost inside the
whole-sequence PointFusion(odom='gt') call at the benchmark shape.

  python scripts/time_depth_filter.py [--batch 8] [--seqlen 32] [--reps 20] [--json OUT]

Prints, with the card's name and power limit read in the same run:
  * forward and backward microseconds per 640 x 480 frame at radius 2, 3, 4 and 6 (CUDA events over a B x L stack);
  * PointFusion(odom='gt') on device-resident frames with and without depth_filter, alternated, median ms per call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gradslam_b200 as gs  # noqa: E402
from gradslam_b200.synthetic import add_depth_noise, make_sequence  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def events_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seqlen", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_depth_filter.py needs a GPU")
    dev = torch.device("cuda:0")
    B, L, H, W = args.batch, args.seqlen, 480, 640
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0, yaw0=0.6)
    noisy = add_depth_noise(depth, seed=0)
    res = {"card": card(), "shape": [B, L, H, W], "kernel_us_per_frame": {}, "pointfusion_ms": {}}
    print("card:", res["card"])
    d = noisy.to(dev)
    g = torch.randn(d.shape, device=dev)
    for r in (2, 3, 4, 6):
        f = gs.BilateralFilter(r, 1.5 * r / 2, 0.05)
        out, den = torch.empty_like(d), torch.empty_like(d)
        gd = torch.empty_like(d)
        fwd = lambda: gs._C.launch("gsx_depth_bilateral", d, out, den, B * L, H, W, r, f.sigma_space,  # noqa: E731
                                   f.sigma_range)
        bwd = lambda: gs._C.launch("gsx_depth_bilateral_bwd", d, out, den, g, gd, B * L, H, W, r,  # noqa: E731
                                   f.sigma_space, f.sigma_range)
        t_f = events_ms(fwd, args.reps) * 1e3 / (B * L)
        t_b = events_ms(bwd, args.reps) * 1e3 / (B * L)
        res["kernel_us_per_frame"][r] = {"forward": round(t_f, 2), "backward": round(t_b, 2)}
        print("radius %d: forward %.2f us/frame, backward %.2f us/frame" % (r, t_f, t_b))
    frames = gs.RGBDImages(rgb.to(dev), noisy.to(dev), K.to(dev), poses.to(dev))
    runs = {"no filter": gs.PointFusion(odom="gt", device=dev),
            "filter r=3": gs.PointFusion(odom="gt", device=dev, depth_filter=gs.BilateralFilter(3, 2.0, 0.05))}
    times = {k: [] for k in runs}
    for _ in range(2):  # warm-up
        for slam in runs.values():
            slam(frames)
    torch.cuda.synchronize()
    for _ in range(5):  # alternated
        for k, slam in runs.items():
            times[k].append(events_ms(lambda: slam(frames), 1))
    for k, ts in times.items():
        res["pointfusion_ms"][k] = round(statistics.median(ts), 2)
        print("PointFusion(odom='gt') %s: median %.2f ms per call (%.1f us per frame), runs %s" % (
            k, statistics.median(ts), statistics.median(ts) * 1e3 / L, [round(t, 2) for t in ts]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
