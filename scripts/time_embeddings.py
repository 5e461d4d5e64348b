"""Time that per-surfel embeddings add to PointFusion: the whole-sequence call (odom='gt') per frame, one differentiable
step (forward + backward; skipped, and reported null, where the map's embeddings do not fit four times), and KE's (gsx_embed_merge_append) achieved bandwidth from its algorithmic bytes:
  merged pixels 3 D s (map row read, frame read, store), appended pixels 2 D s, plus the 4-byte assoc of every pixel and
  the 8-byte (c0, alpha) record of every merged pixel.
--strides: embedding images of (H / stride, W / stride) texels, fused with upsample_embeddings=True by the upsampled KE
(gsx_embed_merge_append_upsampled); stride 1 is the full-resolution path.  The upsampled KE's bytes count the coarse
image once instead of the frame reads (merged 8 + 2 D s, appended D s, plus eh ew D s per element).
Each configuration runs with and without embeddings, alternated, on make_sequence frames; L is the longest sequence
(<= 32) whose frames fit in half the free device memory, and is printed.  The embedding run passes `out=` maps sized
from the counts of the run without embeddings.  --pinned keeps the frames in pinned host memory (the call uploads them
chunk by chunk).  Prints one JSON line per configuration.
Usage: python scripts/time_embeddings.py [--reps 3] [--out DIR] [--B 1 8] [--hw 480x640] [--D 64 512]
       [--dtypes float32 float16] [--strides 1 8 16] [--pinned]"""
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


def _max_L(B, H, W, eh, ew, D, s):
    free, _ = torch.cuda.mem_get_info()
    # the frames (depth, rgb, embeddings), L*H*W geometry rows of the run without embeddings, and an embedding store of
    # at most L*H*W/2 rows (the maps of make_sequence keep fewer than half the pixels)
    per_frame = B * H * W * 16 + B * eh * ew * D * s + B * H * W * 48 + B * H * W * D * s // 2
    return max(2, min(32, int(0.5 * free // per_frame)))


def _out_maps(B, cap, D, dtype, dev):
    out = gs.Pointclouds(device=dev)
    out._allocate(B, cap, 1)
    out._alloc_embeddings(D, dtype)
    return out


def _rand(shape, dtype, scalar, **kw):
    """uniform [0, 1) embeddings; scalar: based one element past a 16-byte boundary, so KE takes one channel per
    thread (V = 1) instead of 16-byte chunks"""
    n = 1
    for v in shape:
        n *= v
    buf = torch.empty(n + (1 if scalar else 0), dtype=dtype, **kw)
    e = (buf[1:] if scalar else buf).view(shape)
    for b in range(shape[0]):  # (one element at a time: the float32 temporary stays small)
        e[b].copy_(torch.rand(shape[1:], **{k: v for k, v in kw.items() if k == "device"}))
    return e


def run(B, H, W, D, dtype, reps, stride=1, pinned=False, scalar=False):
    dev = torch.device("cuda:0")
    s = torch.tensor([], dtype=dtype).element_size()
    up = stride > 1
    eh, ew = H // stride, W // stride
    L = _max_L(B, H, W, eh, ew, D, s)
    rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
    if pinned:
        rgb, depth, K, poses = rgb.pin_memory(), depth.pin_memory(), K.pin_memory(), poses.pin_memory()
        e = _rand((B, L, eh, ew, D), dtype, scalar, pin_memory=True)
    else:
        rgb, depth, K, poses = rgb.to(dev), depth.to(dev), K.to(dev), poses.to(dev)
        e = _rand((B, L, eh, ew, D), dtype, scalar, device=dev)
    plain = gs.RGBDImages(rgb, depth, K, poses)
    emb = gs.RGBDImages(rgb, depth, K, poses, embeddings=e, upsample_embeddings=up)
    slam = gs.PointFusion(odom="gt", device=dev)
    pc, _ = slam(plain)
    cap = max(pc._host_counts())  # the rows an embedding store needs (INTEGRATION.md section 19, "Memory")
    del pc
    torch.cuda.empty_cache()
    slam(emb, out=_out_maps(B, cap, D, dtype, dev))
    t = {"plain": [], "emb": []}
    for _ in range(reps):  # alternated
        for key, f in (("plain", plain), ("emb", emb)):
            out = None if key == "plain" else _out_maps(B, cap, D, dtype, dev)
            t[key].append(_sync_time(lambda: slam(f, out=out), 1))
            del out
    seq_plain, seq_emb = min(t["plain"]), min(t["emb"])
    # the step-API measurements below use the first Lm frames only, on the device: free the rest
    Lm = min(L, 4)
    rgb, depth, poses = (x[:, :Lm].to(dev) for x in (rgb, depth, poses))
    e_lm = _rand((B, Lm, eh, ew, D), dtype, scalar, device=dev)
    e_lm.copy_(e[:, :Lm])
    e = e_lm
    K = K.to(dev)
    del plain, emb, slam
    torch.cuda.empty_cache()
    emb = gs.RGBDImages(rgb, depth, K, poses, embeddings=e, upsample_embeddings=up)

    # KE alone on the last frame's record of a step-API update (re-merging into the same rows; timing only)
    pc = gs.Pointclouds(device=dev)
    for i in range(Lm - 1):
        pc = fu.update_map_fusion(pc, emb[:, i], 0.05, 0.94, 0.6, inplace=True)
    ws = fu._Workspace.get(dev, B, H, W)
    assoc, rec = ws.assoc, ws.rec
    merged, appended = int((assoc < 0).sum()), int((assoc > 0).sum())
    store = pc._emb  # (re-merged in place: the values do not matter for timing, and a copy may not fit)
    ef = e[:, Lm - 2:Lm - 1]
    ef_base, e_bs = fu._embedding_frame(ef, dev)
    code = gs.structures.pointclouds.EMBED_DTYPES[dtype]

    def ke():
        if up:
            gs._C.launch("gsx_embed_merge_append_upsampled", store, pc.capacity, ef_base, e_bs, assoc, rec, B, H, W,
                         eh, ew, D, code)
        else:
            gs._C.launch("gsx_embed_merge_append", store, pc.capacity, ef_base, e_bs, assoc, rec, B, H, W, D, code)

    ke()
    ke_ms = _sync_time(ke, 50)
    if up:
        nbytes = B * H * W * 4 + merged * (8 + 2 * D * s) + appended * D * s + B * eh * ew * D * s
    else:
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
                kw = {} if key == "plain" else {"embeddings": e[:, Lm - 1:Lm].clone().requires_grad_(True),
                                                "upsample_embeddings": up}
                f = gs.RGBDImages(rgb[:, Lm - 1:Lm], d, K, poses[:, Lm - 1:Lm], **kw)
                out = fu.update_map_fusion(m, f, 0.05, 0.94, 0.6)
                loss = out.points_padded.sum() + (0 if key == "plain" else out.embeddings_padded.sum())
                loss.backward()
            step()
            res[key] = _sync_time(step, 5)
        diff = res
    return {"B": B, "H": H, "W": W, "D": D, "dtype": str(dtype).replace("torch.", ""), "stride": stride, "scalar": scalar,
            "eh": eh, "ew": ew, "pinned": pinned, "L": L, "out_capacity": cap,
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
    ap.add_argument("--B", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--hw", nargs="+", default=["240x320", "480x640"], help="HxW of the depth")
    ap.add_argument("--D", type=int, nargs="+", default=[16, 64, 512])
    ap.add_argument("--dtypes", nargs="+", default=["float32", "float16"])
    ap.add_argument("--strides", type=int, nargs="+", default=[1], help="embedding image stride; 1: full resolution")
    ap.add_argument("--pinned", action="store_true", help="frames in pinned host memory")
    ap.add_argument("--scalar", action="store_true", help="misalign the embeddings: KE's one-channel-per-thread path")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_embeddings.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    rows = []
    for B in args.B:
        for H, W in (tuple(int(v) for v in hw.split("x")) for hw in args.hw):
            for D in args.D:
                for dtype in (getattr(torch, d) for d in args.dtypes):
                    for stride in args.strides:
                        r = run(B, H, W, D, dtype, args.reps, stride, args.pinned, args.scalar)
                        rows.append(r)
                        print(json.dumps(r), flush=True)
                        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_embeddings.json"), "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
