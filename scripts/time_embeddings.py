"""Time that per-surfel embeddings add to PointFusion: the whole-sequence call (odom='gt') per frame, one differentiable
step (forward + backward; skipped, and reported null, where the map's embeddings do not fit four times), and KE's (gsx_embed_merge_append) achieved bandwidth from its algorithmic bytes:
  merged pixels 3 D s (map row read, frame read, store), appended pixels 2 D s, plus the 4-byte assoc of every pixel and
  the 8-byte (c0, alpha) record of every merged pixel.
Each configuration runs with and without embeddings, alternated, on make_sequence frames; L is the longest sequence
(<= 32) whose frames and map fit in half the free device memory, and is printed.  Prints one JSON line per configuration.
Usage: python scripts/time_embeddings.py [--reps 3] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import gradslam_b200 as gs  # noqa: E402
from gradslam_b200.slam import fusionutils as fu  # noqa: E402
from gradslam_b200.synthetic import make_sequence  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def _sync_time(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def _max_L(B, H, W, D, s):
    free, _ = torch.cuda.mem_get_info()
    per_frame = B * H * W * (16 + D * s) + B * H * W * (48 + D * s)  # the frames and L*H*W map rows
    return max(2, min(32, int(0.5 * free // per_frame)))


def run(B, H, W, D, dtype, reps):
    dev = torch.device("cuda:0")
    s = torch.tensor([], dtype=dtype).element_size()
    L = _max_L(B, H, W, D, s)
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    rgb, depth, K, poses = rgb.to(dev), depth.to(dev), K.to(dev), poses.to(dev)
    e = torch.rand((B, L, H, W, D), device=dev).to(dtype)
    plain = gs.RGBDImages(rgb, depth, K, poses)
    emb = gs.RGBDImages(rgb, depth, K, poses, embeddings=e)
    slam = gs.PointFusion(odom="gt", device=dev)
    for f in (plain, emb):
        slam(f)
    t = {"plain": [], "emb": []}
    for _ in range(reps):  # alternated
        for key, f in (("plain", plain), ("emb", emb)):
            t[key].append(_sync_time(lambda: slam(f), 1))
    seq_plain, seq_emb = min(t["plain"]), min(t["emb"])
    # the step-API measurements below use the first Lm frames only: free the rest
    Lm = min(L, 4)
    rgb, depth, poses, e = (x[:, :Lm].clone() for x in (rgb, depth, poses, e))
    del plain, emb, slam
    torch.cuda.empty_cache()
    emb = gs.RGBDImages(rgb, depth, K, poses, embeddings=e)

    # KE alone on the last frame's record of a step-API update (re-merging into the same rows; timing only)
    pc = gs.Pointclouds(device=dev)
    for i in range(Lm - 1):
        pc = fu.update_map_fusion(pc, emb[:, i], 0.05, 0.94, 0.6, inplace=True)
    ws = fu._Workspace.get(dev, B, H, W)
    assoc, rec = ws.assoc, ws.rec
    merged, appended = int((assoc < 0).sum()), int((assoc > 0).sum())
    store = pc._emb.clone()
    ef = e[:, Lm - 2:Lm - 1]
    ef_base, e_bs = fu._embedding_frame(ef, dev)
    code = gs.structures.pointclouds.EMBED_DTYPES[dtype]

    def ke():
        gs._C.launch("gsx_embed_merge_append", store, pc.capacity, ef_base, e_bs, assoc, rec, B, H, W, D, code)

    ke()
    ke_ms = _sync_time(ke, 50)
    del store
    nbytes = B * H * W * 4 + merged * (8 + 3 * D * s) + appended * 2 * D * s

    # one differentiable step (float32 only): forward + backward with and without embeddings
    diff = None
    # the out-of-place step holds the map's embeddings about four times over (input, output, their gradients)
    fits = 4 * B * (pc.capacity + H * W) * D * 4 < torch.cuda.mem_get_info()[0]
    if dtype == torch.float32 and fits:
        base = pc.clone()
        base._emb = None
        res = {}
        for key in ("plain", "emb"):
            def step():
                m = base.clone() if key == "plain" else pc.clone()
                d = depth[:, Lm - 1:Lm].clone().requires_grad_(True)
                kw = {} if key == "plain" else {"embeddings": e[:, Lm - 1:Lm].clone().requires_grad_(True)}
                f = gs.RGBDImages(rgb[:, Lm - 1:Lm], d, K, poses[:, Lm - 1:Lm], **kw)
                out = fu.update_map_fusion(m, f, 0.05, 0.94, 0.6)
                loss = out.points_padded.sum() + (0 if key == "plain" else out.embeddings_padded.sum())
                loss.backward()
            step()
            res[key] = _sync_time(step, 5)
        diff = res
    return {"B": B, "H": H, "W": W, "D": D, "dtype": str(dtype).replace("torch.", ""), "L": L,
            "seq_ms_per_frame_plain": seq_plain / L, "seq_ms_per_frame_emb": seq_emb / L,
            "seq_ms_per_frame_added": (seq_emb - seq_plain) / L,
            "ke_us": ke_ms * 1e3, "ke_bytes": nbytes, "ke_TBps": nbytes / (ke_ms * 1e-3) / 1e12,
            "ke_share_of_3.35TBps": nbytes / (ke_ms * 1e-3) / HBM_BYTES_PER_S, "merged": merged, "appended": appended,
            "diff_step_ms_plain": None if diff is None else diff["plain"],
            "diff_step_ms_emb": None if diff is None else diff["emb"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_embeddings.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    rows = []
    for B in (1, 8):
        for H, W in ((240, 320), (480, 640)):
            for D in (16, 64, 512):
                for dtype in (torch.float32, torch.float16):
                    r = run(B, H, W, D, dtype, args.reps)
                    rows.append(r)
                    print(json.dumps(r), flush=True)
                    torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_embeddings.json"), "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
