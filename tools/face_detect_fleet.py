"""BlazeFace face detection on the GPU: device time per batched call against a per-image loop of the same calls.

    python tools/face_detect_fleet.py [--iters 20] [--out results.json]

For B = 1, 8, 64 and 256 images of 640x640 (the size img_to_face hands the detector), on the reference's weights
(tests/golden/blazeface_ref.npz): device ms of one `BlazeFace.forward` over the B images, and of B single-image calls
(CUDA events over --iters repetitions after warm-up), with images/s.  Before timing, the batched rows are checked equal to
the single calls.  The card's name, power limit and clocks are read in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from clearcam_b200.models.blazeface import BlazeFace  # noqa: E402


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    with np.load(os.path.join(ROOT, "tests", "golden", "blazeface_ref.npz")) as z:
        det = BlazeFace({k: z[k] for k in z.files if k != "firing"})
    g = np.random.default_rng(0)
    ims = [torch.from_numpy(g.integers(0, 256, (640, 640, 3), dtype=np.uint8)).cuda() for _ in range(256)]
    det.forward(ims)                                    # the workspace for the largest batch, allocated once
    batched = det.forward(ims[:8])
    for i in range(8):
        single = det.forward(ims[i:i + 1])
        assert all(torch.equal(s[0], b[i]) for s, b in zip(single, batched)), "batched rows differ from single calls"
    print("card:", card())
    res = {"card": card(), "rows": []}
    for B in (1, 8, 64, 256):
        t_batch = timed(lambda: det.forward(ims[:B]), args.iters)
        t_loop = timed(lambda: [det.forward(ims[i:i + 1]) for i in range(B)], max(1, args.iters // max(1, B // 8)))
        row = {"B": B, "batched_ms": t_batch, "loop_ms": t_loop, "batched_img_s": B / t_batch * 1e3, "loop_img_s": B / t_loop * 1e3}
        res["rows"].append(row)
        print(f"B={B:4d}  batched {t_batch:8.3f} ms ({row['batched_img_s']:8.0f} img/s)   per-image loop {t_loop:8.3f} ms "
              f"({row['loop_img_s']:8.0f} img/s)   x{t_loop / t_batch:.1f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
