"""Cost of blended splats (render_pointclouds(blend_band=...)) against the z-buffer disk render (R1d) alone.

Workload: a PointFusion(odom='gt', surfel_radii=True) map fused from make_sequence (B = 8, 640x480, --frames frames,
seed 0), rendered from the fused poses of the last L frames (L = 1 and L = 8 per element) at max_splat_px
M = 1 and 4.  For each (L, M): milliseconds per call (CUDA events around --reps calls after a warm-up call) of the
forward, and of forward + backward of a loss on depth, normals, rgb and confidence with gradients to the map rows and
poses, for R1d alone and for the blend (--band metres).  Prints the card's name, power limit and max SM clock, read
in the same run, and with --out also writes everything as JSON there."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gradslam_b200 as gs  # noqa: E402
from gradslam_b200.synthetic import make_sequence  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--band", type=float, default=0.02)
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_render_blend: no CUDA device")
    print(card(), flush=True)
    B, H, W = 8, 480, 640
    rgb, depth, K, poses = make_sequence(B, args.frames, H, W, seed=0)
    frames = gs.RGBDImages(rgb.cuda(), depth.cuda(), K.cuda(), poses.cuda())
    pc = gs.PointFusion(odom="gt", device="cuda", surfel_radii=True)(frames)[0]
    Kd = K.cuda()
    rows = {"card": card(), "map_rows": pc._host_counts(), "results": []}
    geo0, col0 = pc._geo.detach().clone(), pc._col.detach().clone()
    for L in (1, 8):
        P = poses[:, -L:].contiguous().cuda()
        for M in (1, 4):
            for band in (None, args.band):
                def fwd():
                    with torch.no_grad():
                        gs.render_pointclouds(pc, Kd, P, H, W, max_splat_px=M, blend_band=band)

                def fwd_bwd():
                    pc._geo, pc._col = geo0.clone().requires_grad_(True), col0.clone().requires_grad_(True)
                    Pg = P.clone().requires_grad_(True)
                    out = gs.render_pointclouds(pc, Kd, Pg, H, W, max_splat_px=M, blend_band=band)
                    (out.depth.sum() + out.normals.sum() + out.rgb.sum() + out.confidence.sum()).backward()

                r = dict(L=L, M=M, band=band, fwd_ms=timed(fwd, args.reps), fwd_bwd_ms=timed(fwd_bwd, args.reps))
                pc._geo, pc._col = geo0, col0
                print(json.dumps(r), flush=True)
                rows["results"].append(r)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
