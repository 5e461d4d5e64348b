"""Cost of surfel radii (PointFusion surfel_radii=True) on the fusion step.

Workload: the bench's configuration, PointFusion(odom='gt'), 640x480, B=8, L=32 (make_sequence, seed 0).  Reports:
  * frames/s of the whole-sequence call with radii off and on, alternated within one run (host clock around a device
    synchronise, median of --reps after a warm-up round), and whether slots 0-6 and the colours of the two maps agree;
  * in a separate run of the same call under torch.profiler: K4 (k_merge_append) microseconds per launch both ways;
  * the render of the radii map from a pose halfway between fused frames 15 and 16, L = 1 and L = 8 views per element:
    R1 (one pixel per row) against R1d (disks, --splat-px), z-buffer microseconds per call (torch.profiler, mean of
    --reps calls) and the uncovered-pixel fraction of each;
  * the card's name, power limit and max SM clock, read in the same run.
Writes the results as JSON to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gradslam_b200 as gs  # noqa: E402
from gradslam_b200.synthetic import make_sequence  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed_call(slam, frames):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pc, _ = slam(frames)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, pc


def k4_times(frames, radii):
    """One whole-sequence call under torch.profiler: K4 microseconds per launch (the driver launches it from libgsx)."""
    from torch.profiler import ProfilerActivity, profile

    slam = gs.PointFusion(odom="gt", device="cuda", surfel_radii=radii)
    slam(frames)  # warm-up outside the trace
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        slam(frames)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for short, name in (("K2", "k_project_select"), ("K4", "k_merge_append")):
            if name in e.key:
                out[short] = dict(us_per_launch=e.device_time_total / max(e.count, 1), launches=e.count, kernel=e.key)
    return out


def render_times(pc, K, poses, H, W, M, reps):
    """z-buffer kernel microseconds per call (mean of reps, torch.profiler) and uncovered fraction of one render."""
    from torch.profiler import ProfilerActivity, profile

    out = {}
    for name, m in (("R1_point", 0), ("R1d_disk", M)):
        idx = gs.render_pointclouds(pc, K, poses, H, W, max_splat_px=m).index  # warm-up, and the coverage
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                gs.render_pointclouds(pc, K, poses, H, W, max_splat_px=m)
            torch.cuda.synchronize()
        us = [e.device_time_total / max(e.count, 1) for e in prof.key_averages()
              if "k_render_zbuffer" in e.key or "k_render_splat" in e.key]
        out[name] = dict(zbuffer_us=us[0] if us else None, uncovered=float((idx < 0).float().mean()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--L", type=int, default=32)
    ap.add_argument("--H", type=int, default=480)
    ap.add_argument("--W", type=int, default=640)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--splat-px", type=int, default=3)
    ap.add_argument("--out", default="time_radii.json", help="where the JSON result goes")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_radii.py measures on the GPU"
    res = {"card": card(), "B": a.B, "L": a.L, "H": a.H, "W": a.W}
    print(res["card"], flush=True)
    rgb, depth, K, poses = make_sequence(a.B, a.L, a.H, a.W, seed=0)
    frames = gs.RGBDImages(rgb.cuda(), depth.cuda(), K.cuda(), poses.cuda())
    del rgb, depth
    times = {False: [], True: []}
    maps = {}
    with torch.no_grad():
        for rep in range(a.reps + 1):  # rep 0 warms up both settings
            for radii in (False, True):
                t, pc = timed_call(gs.PointFusion(odom="gt", device="cuda", surfel_radii=radii), frames)
                if rep:
                    times[radii].append(t)
                if rep == a.reps:
                    maps[radii] = pc
                del pc
        off, on = maps[False], maps[True]
        counts = off._host_counts()
        same = counts == on._host_counts() and all(
            torch.equal(off._geo[b, :n, :7], on._geo[b, :n, :7]) and torch.equal(off._col[b, :n], on._col[b, :n])
            for b, n in enumerate(counts))
    for radii in (False, True):
        tm = sorted(times[radii])[len(times[radii]) // 2]
        res["radii_on" if radii else "radii_off"] = dict(fps_call=a.B * a.L / tm, s_call=tm, s_call_spread=times[radii],
                                                        kernels=k4_times(frames, radii))
    # renders of the radii map (one L = 32 call): cameras halfway between fused frames 15 and 16 (L = 1), and 8 such
    # cameras between frames 15 .. 23 (L = 8)
    with torch.no_grad():
        P = frames.poses
        mid = P[:, 15:23].clone()
        mid[..., :3, 3] = 0.5 * (P[:, 15:23, :3, 3] + P[:, 16:24, :3, 3])
        for L in (1, 8):
            res["render_L%d" % L] = render_times(on, frames.intrinsics, mid[:, :L].contiguous(), a.H, a.W, a.splat_px,
                                                 a.reps)
    del off, on
    res["slots_0_6_and_colours_equal"] = bool(same)
    res["rows"] = sum(counts)
    print(json.dumps(res, indent=1), flush=True)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
