"""In-situ timeline of one YOLOv9 forward (cc_yolo_trace: globaltimer stamps written by the conv kernels themselves, no
events between launches, PDL overlap as in production). usage: trace_step.py [size] [B] [res]
Columns: t_in = first CTA entered, t_dep = grid dependency released (previous kernel's memory visible), t_out = last CTA
exited; work = t_out - t_dep; gap = t_dep - previous conv's t_out (launch boundary + any non-conv kernels in between)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from oracle import yolov9 as o
from clearcam_b200.detection.yolov9 import YOLOv9
size = sys.argv[1] if len(sys.argv) > 1 else "c"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 32
res = int(sys.argv[3]) if len(sys.argv) > 3 else 640
fr = o.synthetic_frames(4, res, res, seed=0)
P = o.synthetic_weights(size, seed=0, calib=fr[:2].flip(-1).permute(0, 3, 1, 2).float() / 255)
m = YOLOv9(size, res, weights=P)
frames = fr[torch.arange(B) % 4].cuda()
for _ in range(3):
    m.detect_batch(frames)
torch.cuda.synchronize()
best = None
for _ in range(5):
    tr = m.trace(frames)
    span = max(r["t_out"] for r in tr)
    if best is None or span < best[0]:
        best = (span, tr)
span, tr = best
print(f"span first conv entry -> last conv exit: {span/1e6:.3f} ms (B={B})")
print(f"{'#':>3} {'kind':12s} {'name':34s} {'t_in_us':>9s} {'t_dep_us':>9s} {'t_out_us':>9s} {'work_us':>8s} {'gap_us':>7s} {'ideal_us':>8s} | CTA 0, us after t_dep: operands landed, MMAs issued, first acc done, epilogue done, exit) | first staging pass, SM cycles after 'staging free': (unused)")
prev_out = 0
tw = tg = 0.0
nonconv = []
for i, r in enumerate(tr):
    if r["kind"] != "conv_gemm":
        nonconv.append(r["name"])
        print(f"{i:3d} {r['kind']:12s} {r['name']:34s}")
        continue
    work = (r["t_out"] - r["t_dep"]) / 1e3
    gap = (r["t_dep"] - prev_out) / 1e3
    tw += work
    tg += gap
    c0 = " ".join(f"{(v - r['t_dep'])/1e3:6.2f}" if v else "     -" for v in r["cta0"])     # CTA 0 stamps relative to t_dep
    print(f"{i:3d} {r['kind']:12s} {r['name']:34s} {r['t_in']/1e3:9.2f} {r['t_dep']/1e3:9.2f} {r['t_out']/1e3:9.2f} {work:8.2f} {gap:7.2f} {r['flops']/1443e6:8.2f} | {c0} | {r['pass_cycles']}")
    prev_out = r["t_out"]
print(f"sum of conv work {tw/1e3:.3f} ms, sum of gaps (boundaries + non-conv kernels) {tg/1e3:.3f} ms")
