"""Cost and effect of removing free-space violations (PointFusion free_space_margin) beside the unstable-surfel rule.

Workload: PointFusion(odom='gt'), 640x480, B=8, L = 32 and 64, on the bench's static scene (make_sequence) and on the
dynamic scene (make_dynamic_sequence: the same room with a box in frames [L/4, L/2)).  Alternated within one run: both
rules off, the age rule alone, and the age rule with the free-space rule at two margins.  Reports, per scene, L and
setting:
  * frames/s of the whole call (host clock around a device synchronise, median of --reps after a warm-up round);
  * final rows per element, rows removed against both rules off, and rows removed by the free-space rule (the age rule
    alone minus the combined rule);
  * in a separate run of the step API under torch.profiler: KFb, KFt and KP microseconds per launch;
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
from gradslam_b200.synthetic import make_dynamic_sequence, make_sequence  # noqa: E402


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


def kernel_times(frames, kw, L):
    """Step API (one fuse_and_prune per frame) under torch.profiler: microseconds per launch of each kernel."""
    from torch.profiler import ProfilerActivity, profile

    slam = gs.PointFusion(odom="gt", device="cuda", **kw)
    pc = gs.Pointclouds(device="cuda")
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(L):
            pc, _ = slam.step(pc, frames[:, s], None, inplace=True)
        torch.cuda.synchronize()
    names = {"KFb": "k_free_space_bound", "KFt": "k_free_space_test", "KP": "k_prune_unstable",
             "K2": "k_project_select", "K4": "k_merge_append"}
    out = {}
    for e in prof.key_averages():
        for short, name in names.items():
            if name in e.key:
                out[short] = dict(us_per_launch=e.device_time_total / max(e.count, 1), launches=e.count)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--L", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--H", type=int, default=480)
    ap.add_argument("--W", type=int, default=640)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--margins", type=float, nargs="+", default=[0.05, 0.2])
    ap.add_argument("--t-max", type=int, default=4)
    ap.add_argument("--quantile", type=float, default=0.25, help="c_stable: this quantile of the unpruned map's confidences")
    ap.add_argument("--out", default="time_free_space.json", help="where the JSON result goes")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_free_space.py measures on the GPU"
    res = {"card": card(), "B": a.B, "H": a.H, "W": a.W, "t_max": a.t_max, "runs": {}}
    print(res["card"], flush=True)
    for scene in ("static", "dynamic"):
        for L in a.L:
            if scene == "static":
                rgb, depth, K, poses = make_sequence(a.B, L, a.H, a.W, seed=0)
            else:
                rgb, depth, K, poses = make_dynamic_sequence(a.B, L, a.H, a.W, L // 4, L // 2, seed=0)
            frames = gs.RGBDImages(rgb.cuda(), depth.cuda(), K.cuda(), poses.cuda())
            del rgb, depth
            with torch.no_grad():
                full, _ = gs.PointFusion(odom="gt", device="cuda")(frames)
                cc = torch.cat(full.features_list)[:, 0].double().cpu()
                c = float(torch.quantile(cc, a.quantile, interpolation="lower"))
                del full, cc
                age = dict(stable_confidence=c, max_unstable_age=a.t_max)
                settings = {"off": {}, "age": age}
                settings.update({"age+free_space(%g)" % m: dict(age, free_space_margin=m) for m in a.margins})
                times = {n: [] for n in settings}
                rows = {}
                for rep in range(a.reps + 1):  # rep 0 warms up every shape
                    for n, kw in settings.items():
                        t, pc = timed_call(gs.PointFusion(odom="gt", device="cuda", **kw), frames)
                        rows[n] = [int(x) for x in pc.num_points_per_pointcloud.tolist()]
                        del pc
                        torch.cuda.empty_cache()
                        if rep:
                            times[n].append(t)
                out = {"c_stable": c, "settings": {}}
                for n in settings:
                    tm = sorted(times[n])[len(times[n]) // 2]
                    out["settings"][n] = dict(fps_call=a.B * L / tm, s_call=tm, s_call_spread=times[n],
                                              rows_per_element=rows[n], removed_vs_off=sum(rows["off"]) - sum(rows[n]))
                    if n.startswith("age+"):
                        out["settings"][n]["removed_by_free_space"] = sum(rows["age"]) - sum(rows[n])
                        out["settings"][n]["removed_by_free_space_fraction"] = 1 - sum(rows[n]) / sum(rows["age"])
                for n, kw in settings.items():
                    if n != "off":
                        out["settings"][n]["kernels_step_api"] = kernel_times(frames, kw, L)
            res["runs"]["%s_L%d" % (scene, L)] = out
            print(json.dumps({"%s_L%d" % (scene, L): out}, indent=1), flush=True)
            del frames
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
