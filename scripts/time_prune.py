"""Cost and effect of removing unstable surfels (PointFusion stable_confidence / max_unstable_age) on long sequences.

Workload: PointFusion(odom='gt'), 640x480, B=8, L frames, on the bench's scene and on the corner-facing scene (yaw0=0.6).
Pruning off and a few (c_stable, t_max) settings are alternated within one run.  Reports, per scene and setting:
  * frames/s of the whole call and of its last 16 frames (t(L) - t(L-16), both whole-sequence calls, host clock around a
    device synchronise, median of --reps);
  * final rows per element and the fraction removed against pruning off;
  * in a separate instrumented run of the step API: K2 and prune kernel times per launch (torch.profiler), and the
    prune's bytes moved, 48 x rows moved + 32 x rows tested, over its time;
  * the confidence quantiles of the unpruned L=32 map, from which c_stable is chosen;
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
from gradslam_b200.slam import fusionutils as fu  # noqa: E402
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


def instrumented(frames, c, t_max, L):
    """Step API with host reads around each prune: rows tested / moved per launch, and kernel times by torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    slam = gs.PointFusion(odom="gt", device="cuda")
    pc = gs.Pointclouds(device="cuda")
    tested = moved = 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(L):
            pc, _ = slam.step(pc, frames[:, s], None, inplace=True)  # fusion only (slam has pruning off)
            h = pc._prune
            step = 0 if h is None else h.step
            counts = pc._counts_dev[pc._cur].tolist()
            if step >= t_max:
                ring = None if h is None else h.ring.cpu()
                at = lambda k, b: 0 if (k < 0 or ring is None) else int(ring[k % (t_max + 2), b])
                cc = pc._geo[..., 6]
                for b, n in enumerate(counts):
                    ws = min(at(step - t_max - 1, b), n)
                    we = n if t_max == 0 else min(at(step - t_max, b), n)
                    rem = (cc[b, ws:we] < c).nonzero()
                    tested += we - ws
                    if rem.numel():
                        first = ws + int(rem[0])
                        moved += (n - first) - rem.numel()
            fu.prune_unstable(pc, c, t_max)
        torch.cuda.synchronize()
    k = {}
    for e in prof.key_averages():
        for name in ("k_project_select", "k_prune_unstable"):
            if name in e.key:
                k[name] = dict(us_per_launch=e.device_time_total / max(e.count, 1), launches=e.count,
                               us_total=e.device_time_total)
    if "k_prune_unstable" in k:
        k["k_prune_unstable"]["rows_tested"] = tested
        k["k_prune_unstable"]["rows_moved"] = moved
        k["k_prune_unstable"]["GB_per_s"] = (48 * moved + 32 * tested) / (k["k_prune_unstable"]["us_total"] * 1e3)
    return k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=8)
    ap.add_argument("--L", type=int, default=64)
    ap.add_argument("--H", type=int, default=480)
    ap.add_argument("--W", type=int, default=640)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="time_prune.json", help="where the JSON result goes")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_prune.py measures on the GPU"
    res = {"card": card(), "B": a.B, "L": a.L, "H": a.H, "W": a.W, "scenes": {}}
    print(res["card"], flush=True)
    for scene, yaw0 in (("bench", 0.0), ("corner", 0.6)):
        rgb, depth, K, poses = make_sequence(a.B, a.L, a.H, a.W, seed=0, yaw0=yaw0)
        frames = gs.RGBDImages(rgb.cuda(), depth.cuda(), K.cuda(), poses.cuda())
        del rgb, depth
        with torch.no_grad():
            m32, _ = gs.PointFusion(odom="gt", device="cuda")(frames[:, :32])
            cc = torch.cat(m32.features_list)[:, 0].double()
            qs = [0.1, 0.25, 0.5, 0.75, 0.9]
            quant = dict(zip(map(str, qs), torch.quantile(cc.cpu(), torch.tensor(qs, dtype=torch.float64)).tolist()))
            del m32
            settings = [None, (quant["0.25"], 4), (quant["0.5"], 4), (quant["0.5"], 16)]
            names = ["off"] + ["c=%.3g,t=%d" % s for s in settings[1:]]
            times = {n: {"L": [], "L-16": []} for n in names}
            rows = {}
            for rep in range(a.reps + 1):  # rep 0 warms up every shape
                for n, st in zip(names, settings):
                    kw = {} if st is None else dict(stable_confidence=st[0], max_unstable_age=st[1])
                    slam = gs.PointFusion(odom="gt", device="cuda", **kw)
                    t_full, pc = timed_call(slam, frames)
                    rows[n] = pc.num_points_per_pointcloud.tolist()
                    del pc
                    t_head, pc = timed_call(slam, frames[:, :a.L - 16])
                    del pc
                    torch.cuda.empty_cache()
                    if rep:
                        times[n]["L"].append(t_full)
                        times[n]["L-16"].append(t_head)
            out = {"confidence_quantiles_L32": quant, "settings": {}}
            for n in names:
                tl = sorted(times[n]["L"])[len(times[n]["L"]) // 2]
                th = sorted(times[n]["L-16"])[len(times[n]["L-16"]) // 2]
                out["settings"][n] = dict(
                    fps_call=a.B * a.L / tl, fps_last16=a.B * 16 / (tl - th), s_call=tl, s_call_spread=times[n]["L"],
                    rows_per_element=rows[n], removed_fraction=1 - sum(rows[n]) / sum(rows["off"]))
            for n, st in zip(names[1:], settings[1:]):
                out["settings"][n]["kernels_step_api"] = instrumented(frames, st[0], st[1], a.L)
            res["scenes"][scene] = out
            print(json.dumps({scene: out}, indent=1), flush=True)
        del frames
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
