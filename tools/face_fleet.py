"""AdaFace IR-50 face embeddings on the GPU: correctness first, then device time per call and faces/s.

    python tools/face_fleet.py [--iters 20] [--out results.json]

1. Checks `embed_faces` against the fp32 CPU oracle on synthetic weights and faces (the bar: twice the bf16 mirror's own
   deviation); stops if it fails.
2. For B = 1, 8, 64 and 256: device ms per batched call (CUDA events over --iters calls after warm-up), faces/s and the
   in-situ TFLOP/s from the network's algorithmic FLOPs (computed below from the shapes: 2 x MACs of conv0, the 48 3x3
   convs, the three 1x1 shortcuts and the linear).
3. The reference's call pattern (one face per call, clearcam.py:1234, 675) against one batched call over the same 64 faces,
   alternated over 3 runs.
The card's name and power limit are read in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from clearcam_b200.models import adaface as ca  # noqa: E402
from clearcam_b200.models.objects import ObjectFinder  # noqa: E402
from oracle import adaface as oa  # noqa: E402


def face_flops() -> float:
    """Algorithmic FLOPs of one 112x112 face (2 per multiply-add)."""
    macs = 112 * 112 * 64 * 3 * 9                                     # conv0
    side = 112
    for cin, d, s in ca.SIZES:
        macs += side * side * d * cin * 9                             # conv_layer0 (stride 1)
        side //= s
        macs += side * side * d * d * 9                               # conv_layer1 (stride s)
        if cin != d:
            macs += side * side * d * cin                             # 1x1 shortcut
    macs += 7 * 7 * 512 * 512                                         # linear
    return 2.0 * macs


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card()}
    P = oa.synthetic_weights(seed=5)
    finder = ObjectFinder()
    finder.init_face(weights=P)

    # 1. correctness
    faces = oa.synthetic_faces(8, seed=21)
    got = finder.embed_faces(faces).cpu()
    with torch.no_grad():
        fp32 = oa.forward(P, faces)
        mirror = oa.forward_folded(ca.fold_state_dict(P), faces, bf16=True)
    dev, bar = (got - fp32).abs().max().item(), (mirror - fp32).abs().max().item()
    cos = (got * fp32).sum(-1).min().item()
    res["check"] = {"max_dev_vs_fp32": dev, "mirror_max_dev_vs_fp32": bar, "min_cos": cos}
    print(f"card: {res['card']}")
    print(f"check: max |GPU - fp32 oracle| = {dev:.3e}, bf16 mirror {bar:.3e}, min cosine {cos:.6f}")
    if not dev <= 2 * bar:
        sys.exit("GPU embeddings deviate from the oracle beyond the bar")

    # 2. batched calls
    fl = face_flops()
    res["gflop_per_face"] = fl / 1e9
    res["batched"] = []
    for B in (1, 8, 64, 256):
        x = oa.synthetic_faces(B, seed=B).cuda()
        for _ in range(3):
            finder.embed_faces(x)
        torch.cuda.synchronize()
        ms = timed(lambda: finder.embed_faces(x), args.iters)
        row = {"B": B, "ms_per_call": ms, "faces_per_s": B / ms * 1e3, "tflops": fl * B / ms / 1e9}
        res["batched"].append(row)
        print(f"B={B:4d}: {ms:8.3f} ms/call  {row['faces_per_s']:9.1f} faces/s  {row['tflops']:6.1f} TFLOP/s")

    # 3. the reference's one-face-per-call loop against one batched call, alternated
    B = 64
    x = oa.synthetic_faces(B, seed=64).cuda()
    singles = [x[i:i + 1] for i in range(B)]
    res["loop_vs_batch"] = []
    for run in range(3):
        loop = timed(lambda: [finder.embed_faces(f) for f in singles], max(1, args.iters // 4))
        batch = timed(lambda: finder.embed_faces(x), args.iters)
        res["loop_vs_batch"].append({"run": run, "loop_ms": loop, "batch_ms": batch, "speedup": loop / batch})
        print(f"run {run}: {B} single calls {loop:8.3f} ms, one call of {B} {batch:8.3f} ms: {loop / batch:5.2f}x")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
