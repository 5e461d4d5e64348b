"""Times K1 (depth -> 4 maps) and its backward on B x L frames (default 8 x 8 at 640x480)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gradslam_b200 as gs
from gradslam_b200.structures.rgbdimages import backproject
from gradslam_b200.synthetic import make_sequence

B, L, H, W = 8, 8, 480, 640
dev = torch.device("cuda:0")
rgb, depth, K, poses = make_sequence(B, L, H, W, seed=0)
depth, K, poses = depth.to(dev), K.to(dev), poses.to(dev)
for want, label, bpp in (((True, True, True, True), "all four maps", 52), ((False, False, True, True), "global maps only", 28)):
    for _ in range(3):
        backproject(depth, K, poses, want)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        backproject(depth, K, poses, want)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    nbytes = B * L * H * W * bpp
    print("K1 %-18s %.1f us for %d frames (%.1f us per 8-frame batch), %.0f GB/s algorithmic (%.1f%% of 3350)" % (
        label, ms * 1e3, B * L, ms * 1e3 / L, nbytes / ms / 1e6, 100 * nbytes / ms / 1e6 / 3350.0))
d = depth.clone().requires_grad_(True)
for _ in range(2):  # warm-up (lazy kernel loading, autograd engine start-up)
    o = backproject(d, K, poses, (True, True, True, True))
    torch.autograd.backward(o, [torch.ones_like(x) for x in o])
outs = backproject(d, K, poses, (True, True, True, True))
g = [torch.randn_like(o) for o in outs]
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
torch.autograd.backward(outs, g)
e1.record()
torch.cuda.synchronize()
print("K1 backward (4 upstream grads -> depth grad): %.1f us for %d frames" % (e0.elapsed_time(e1) * 1e3, B * L))
