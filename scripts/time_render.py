#!/usr/bin/env python
"""Times render_pointclouds (R1 z-buffer, R2 resolve, R3 backward) on the benchmark's map: B = 8 sequences of 32 frames,
640x480, seed 0, fused with PointFusion(odom='gt') (~1.1 M rows per element), rendered from all 32 poses and from one.

Reports CUDA-event times per call, per-kernel times from a separate torch.profiler run, the algorithmic bytes of the run
(12 B per map row for the positions; per covered pixel 28 B of row gathers - 16 B of geometry, 12 B of colour - and 40 B
of image writes - index 8, depth 4, rgb 12, normals 12, confidence 4) and, as context, the same render written in ATen
(project_map + scatter_reduce 'amin' + gathers) on the same GPU.  Prints one JSON object (also written to --out if
given)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import gsx_oracle as oracle  # noqa: E402
import gradslam_b200 as gs  # noqa: E402
from gradslam_b200.synthetic import make_sequence  # noqa: E402

KERNELS = {"R1": "k_render_zbuffer", "R2": "k_render_resolve", "R3 rows": "k_render_bwd_rows",
           "R3 pose": "k_render_bwd_pose", "R3 pose reduce": "k_pose_grad_reduce"}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name still identifies the card
        q = "unavailable (%s)" % e
    return {"name": name, "power_limit, max_sm_clock": q}


def event_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_ms(fn, iters):
    """Mean device time per call of each render kernel (torch.profiler, its own run)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for short, name in KERNELS.items():
            if name in ev.key:
                total = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                out[short] = out.get(short, 0.0) + total / 1e3 / iters
    return out


def aten_render(pts, counts, col, K, poses, H, W):
    """The same render in ATen: per view project_map, the frustum test, an int64 key per row, scatter_reduce 'amin'
    per pixel, then gathers of depth and colour."""
    B, N = pts.shape[:2]
    L = poses.shape[1]
    dev = pts.device
    live = torch.arange(N, device=dev).view(1, N) < counts.view(B, 1)
    nn = torch.arange(N, device=dev).view(1, N).expand(B, N)
    bb = torch.arange(B, device=dev).view(B, 1).expand(B, N)
    big = torch.iinfo(torch.int64).max
    index = torch.full((B, L, H * W), big, dtype=torch.int64, device=dev)
    depth = torch.zeros((B, L, H * W), device=dev)
    rgb = torch.zeros((B, L, H * W, 3), device=dev)
    for l in range(L):
        u, v, z = oracle.project_map(pts, poses[:, l], K)
        ok = (u > -1e-3) & (u < W - 0.999) & (v > -1e-3) & (v < H - 0.999) & (z > 0) & live
        w = u.round().long().clamp(0, W - 1)
        h = v.round().long().clamp(0, H - 1)
        key = (z.contiguous().view(torch.int32).to(torch.int64) << 32) | nn
        slot = (bb * L + l) * (H * W) + h * W + w
        index.view(-1).scatter_reduce_(0, slot[ok], key[ok], reduce="amin")
    covered = index != big
    n = torch.where(covered, index & 0xFFFFFFFF, torch.zeros_like(index))
    depth = torch.where(covered, (index >> 32).to(torch.int32).view(torch.float32), depth)
    rgb = torch.where(covered.unsqueeze(-1), torch.gather(col, 1, n.view(B, -1, 1).expand(B, L * H * W, 3)).view(
        B, L, H * W, 3), rgb)
    return torch.where(covered, n, torch.full_like(n, -1)), depth, rgb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_render.py needs a GPU"
    dev = torch.device("cuda:0")
    B, L, H, W = 8, 32, 480, 640
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    K, poses = K.to(dev), poses.to(dev)
    with torch.no_grad():
        pc, _ = gs.PointFusion(odom="gt", device=dev)(gs.RGBDImages(rgb.to(dev), depth.to(dev), K, poses))
    counts = pc.num_points_per_pointcloud
    M = int(counts.sum())
    res = {"card": card(), "map_rows_per_element": counts.tolist(), "image": "%dx%d" % (W, H), "B": B, "cases": {}}
    for Lv, views in ((32, poses), (1, poses[:, -1:].contiguous())):
        call = lambda: gs.render_pointclouds(pc, K, views, H, W)
        with torch.no_grad():
            for _ in range(args.warmup):
                out = call()
            torch.cuda.synchronize()
            fwd_ms = event_ms(call, args.iters)
            fwd_k = kernel_ms(call, args.iters)
            covered = int((out.index >= 0).sum())
        pv = views.clone().requires_grad_(True)
        pcg = pc.clone()
        pcg._geo = pcg._geo.detach().requires_grad_(True)  # gradients w.r.t. the map rows, too

        def fwd_bwd():
            o = gs.render_pointclouds(pcg, K, pv, H, W)
            (o.depth.sum() + o.rgb.sum() + o.normals.sum() + o.confidence.sum()).backward()

        for _ in range(args.warmup):
            fwd_bwd()
        torch.cuda.synchronize()
        fb_ms = event_ms(fwd_bwd, args.iters)
        bwd_k = kernel_ms(fwd_bwd, args.iters)
        pts, col = pc.points_padded.contiguous(), pc.colors_padded.contiguous()
        aten = lambda: aten_render(pts, counts, col, K[:, 0], views, H, W)
        with torch.no_grad():
            a_idx, a_depth, _ = aten()
            same = bool(torch.equal(a_idx.view(B, Lv, H, W), out.index))
            torch.cuda.synchronize()
            aten_ms = event_ms(aten, max(2, args.iters // 4))
        alg_bytes = 12 * M + covered * (28 + 40)
        r1r2 = fwd_k.get("R1", 0.0) + fwd_k.get("R2", 0.0)
        res["cases"]["L=%d" % Lv] = {
            "forward_ms_per_call": fwd_ms, "forward_kernels_ms": fwd_k,
            "forward_plus_backward_ms_per_call": fb_ms, "backward_kernels_ms": {k: v for k, v in bwd_k.items()
                                                                                 if k.startswith("R3")},
            "covered_pixels": covered, "algorithmic_bytes": alg_bytes,
            "R1+R2_GB_per_s": alg_bytes / (r1r2 * 1e-3) / 1e9 if r1r2 > 0 else None,
            "aten_forward_ms_per_call": aten_ms, "aten_index_equal": same}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
