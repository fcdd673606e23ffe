"""GPU diagnostic: how accurate is the tensor-core fp32 accumulation behind the fp32-accurate mode?  One conv through the same
six-plane bf16 split the detector uses (yolo.cu / pool.cu split_planes_kernel), built here in torch, against fp64 and fp32
CPU convs of the same fp32 operands.  Prints the signed mean (bias = truncating accumulation) and the rms of the relative
error.  usage: diag_tc_accum.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
import torch.nn.functional as F
from clearcam_b200 import ops


def split3(x):
    hi = x.to(torch.bfloat16)
    r1 = x - hi.float()
    mid = r1.to(torch.bfloat16)
    lo = (r1 - mid.float()).to(torch.bfloat16)
    return hi, mid, lo


def run(N, H, W, Cin, Cout, k, positive):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(N, H, W, Cin, generator=g)
    if positive:
        x = x.abs()                                   # post-SiLU-like activations: sums do not cancel, bias shows
    w = torch.randn(Cout, k, k, Cin, generator=g) * (1.0 / (k * k * Cin) ** 0.5)
    if positive:
        w = w.abs()
    xh, xm, xl = split3(x)
    wh, wm, wl = split3(w)
    xa = torch.cat([xl, xm, xh, xm, xh, xh], dim=-1).contiguous().cuda()             # [lo|mid|hi|mid|hi|hi]
    wa = torch.cat([wh, wm, wl, wh, wm, wh], dim=-1).contiguous().cuda()             # [hi|mid|lo|hi|mid|hi]
    out = torch.empty(N, H, W, Cout, dtype=torch.float32, device="cuda")
    bias = torch.zeros(Cout, device="cuda")
    ops.conv2d(xa, 0, 6 * Cin, wa, bias, k, 1, out, 0, Cout, act=0, impl=1)
    torch.cuda.synchronize()
    got = out.cpu().double()
    xn, wn = x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2)
    ref64 = F.conv2d(xn.double(), wn.double(), padding=k // 2).permute(0, 2, 3, 1)
    ref32 = F.conv2d(xn, wn, padding=k // 2).permute(0, 2, 3, 1).double()
    scale = ref64.abs().mean()
    for tag, t in (("wgmma six-plane  ", got), ("torch fp32 CPU   ", ref32)):
        e = (t - ref64) / scale
        print(f"  {tag}: signed mean {e.mean():+.3e}  rms {e.pow(2).mean().sqrt():.3e}  max {e.abs().max():.3e}")


if __name__ == "__main__":
    for positive in (False, True):
        for (Cin, k) in ((64, 1), (128, 3), (256, 3)):
            print(f"Cin={Cin} k={k} K={Cin * k * k} operands {'positive' if positive else 'signed'}:")
            run(2, 24, 24, Cin, 64, k, positive)
