"""Per-kernel device time of cc_jpeg_decode on one large file without restart markers, for several library builds
alternated in fresh processes (the DC pass walks such a file's single restart interval).

    python tools/jpeg_dc_ab.py [--reps 3] [--calls 30] -- base "CC_LIB=/path/to/other/libclearcam_b200.so" ...

Variants as in tools/ab.py ("base" = the in-tree build).  Files: seeded synthetic 1080p and 2160p frames (gradients and
noise), q85 4:2:0, no restart interval.  Each process checks its pixels against cv2.imdecode, then times `calls` decodes
under torch.profiler and prints the mean device time of every kernel per call.  Prints the card's name and power limit."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(calls):
    sys.path.insert(0, ROOT)
    import cv2
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from clearcam_b200 import ops
    out = {}
    for H, W in ((1080, 1920), (2160, 3840)):
        rng = np.random.default_rng(H)
        yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
        img = np.clip(np.stack([(xx * (0.9 + 0.3 * c) + yy * (0.6 + 0.2 * c) + 60 * c) % 256 for c in range(3)], -1)
                      + rng.normal(0, 6, (H, W, 3)), 0, 255).astype(np.uint8)
        f = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                       cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])[1].tobytes()
        b = ops.JpegBatch([f])
        o, st = b.decode()
        torch.cuda.synchronize()
        assert int(st[0]) == 0 and np.array_equal(o[0].cpu().numpy(), cv2.imdecode(np.frombuffer(f, np.uint8), 1))
        for _ in range(5):
            b.decode(o)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                b.decode(o)
            torch.cuda.synchronize()
        k = {}
        for e in prof.events():
            if e.device_type.name == "CUDA" and "jdec_" in e.name:
                name = e.name.split("jdec_")[1].split("(")[0].split("ENS")[0]
                k[name] = k.get(name, 0.0) + e.device_time_total / calls
        out[f"{H}p"] = {n: round(v, 1) for n, v in sorted(k.items())} | {"total_us": round(sum(k.values()), 1)}
    print(json.dumps(out))


def main():
    argv = sys.argv[1:]
    if argv and argv[0] == "--child":
        return child(int(argv[1]))
    if "--" not in argv:
        sys.exit(__doc__)
    opts, variants = argv[:argv.index("--")], argv[argv.index("--") + 1:]
    reps = int(opts[opts.index("--reps") + 1]) if "--reps" in opts else 3
    calls = opts[opts.index("--calls") + 1] if "--calls" in opts else "30"
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    for r in range(reps):
        for v in variants:
            env = dict(os.environ)
            if v != "base":
                env.update(kv.split("=", 1) for kv in v.split())
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", calls], env=env, capture_output=True, text=True)
            print(json.dumps({"rep": r, "variant": v, **(json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0
                                                           else {"failed": p.stderr[-2000:]})}), flush=True)


if __name__ == "__main__":
    main()
