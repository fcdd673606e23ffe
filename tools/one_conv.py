"""Run single conv shapes through cc_conv (for ncu / timing). usage: one_conv.py [iters]"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from clearcam_b200 import ops
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 3
shapes = [  # N,H,W,Cin,Cout,k,s
    (32, 160, 160, 128, 128, 1, 1),
    (32, 40, 40, 256, 256, 3, 1),
    (32, 160, 160, 64, 64, 3, 1),
    (32, 80, 80, 256, 320, 3, 1),
    (32, 80, 80, 128, 128, 3, 1),
    (32, 160, 160, 256, 256, 1, 1),
    (32, 160, 160, 32, 32, 3, 1),
    (32, 40, 40, 256, 256, 1, 1),
    (32, 40, 40, 128, 128, 3, 1),
    (32, 80, 80, 512, 512, 1, 1),
    (32, 20, 20, 256, 256, 1, 1),
    (32, 320, 320, 64, 128, 3, 2),      # 11: model.1
    (32, 160, 160, 256, 256, 1, 1),     # 12 (= 5): model.2.cv4
    (32, 160, 160, 128, 128, 1, 1),     # 13 (= 0): model.2.cv1
]
sel = [int(a) for a in sys.argv[2:]] or range(len(shapes))
for si in sel:
    N, H, W, Cin, Cout, k, s = shapes[si]
    N = int(os.environ.get("ONE_CONV_N", N))
    x = torch.randn(N, H, W, Cin, device="cuda").to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin, device="cuda") * 0.05).to(torch.bfloat16)
    b = torch.randn(Cout, device="cuda")
    o = torch.empty(N, H // s, W // s, Cout, device="cuda", dtype=torch.bfloat16)
    for _ in range(2):
        ops.conv2d(x, 0, Cin, w, b, k, s, o, 0, Cout, act=1, impl=1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.conv2d(x, 0, Cin, w, b, k, s, o, 0, Cout, act=1, impl=1)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * N * (H // s) * (W // s) * Cout * Cin * k * k
    by = (x.numel() + o.numel()) * 2
    print(f"{shapes[si]}: {ms:.4f} ms  {fl/ms/1e9:.1f} TFLOP/s  {by/ms/1e6:.0f} GB/s")
