"""What reading cameras as yuv420p instead of bgr24 buys on the detector path (YOLOv9-c, res 640, 1080p frames).

    python tools/yuv_ingest.py [--batches 8 32] [--steps 200] [--reps 3] [--out FILE]

Prints the card's name and power limit, then for each batch size B:
  * frames/s from pinned host memory through `YOLOv9.detect_pipelined` (H2D copies overlap the compute), bgr24 against
    yuv420p, alternated `reps` times with `steps` batches per run;
  * the letterbox op's device time per format, from `YOLOv9.profile` (median of 5), which for yuv420p includes the
    conversion to BGR;
  * the H2D bytes per frame, computed from the shapes;
  * a check that both formats give identical detections on the timed inputs (the bgr24 batches are the oracle's
    conversion of the yuv420p ones, oracle/yuv.py, so the detector's input is the same picture).
It also times single-core cv2.cvtColor(COLOR_YUV2BGR_I420) on a 1080p frame: a proxy, not a measurement, of the host
conversion ffmpeg does for `-pix_fmt bgr24` and no longer does for yuv420p.  One JSON line at the end.
Weights are synthetic (oracle.yolov9.synthetic_weights): the speed of the kernels does not depend on their values."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H, W, RES = 1080, 1920, 640


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:                 # the numbers below still carry the device name from torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({ex!r})", "max_sm_clock": "unknown"}


def frames(n, seed):
    """n distinct 1080p frames: yuv420p [n,1620,1920] and their BGR [n,1080,1920,3] = the oracle's conversion."""
    import cv2
    from oracle import yolov9 as o
    from oracle.yuv import i420_to_bgr
    bgr0 = o.synthetic_frames(n, H, W, seed=seed).numpy()
    yuv = np.stack([cv2.cvtColor(np.ascontiguousarray(f), cv2.COLOR_BGR2YUV_I420) for f in bgr0])
    return torch.from_numpy(yuv), torch.from_numpy(i420_to_bgr(yuv))


def run(model, batches, steps, pix_fmt):
    """frames/s of `steps` batches through detect_pipelined; returns (fps, results of the first len(batches) steps)."""
    seq = (batches[i % len(batches)] for i in range(steps))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first = []
    for i, r in enumerate(model.detect_pipelined(seq, pix_fmt=pix_fmt)):
        if i < len(batches):
            first.append(r.clone())
    dt = time.perf_counter() - t0                  # every result has been synchronised on before it was yielded
    return steps * batches[0].shape[0] / dt, first


def cv2_proxy(n=200):
    import cv2
    cv2.setNumThreads(1)
    yuv = np.random.default_rng(0).integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)
    out = np.empty((H, W, 3), np.uint8)
    for _ in range(10):
        cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_I420, dst=out)
    t0 = time.perf_counter()
    for _ in range(n):
        cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_I420, dst=out)
    return (time.perf_counter() - t0) / n * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    from oracle import yolov9 as o
    from clearcam_b200.detection.yolov9 import YOLOv9
    info = card()
    print("card:", info, flush=True)
    fr = o.synthetic_frames(2, 320, 320, seed=9)
    x = torch.stack([o.preprocess(f, 320) for f in fr]).flip(-1).permute(0, 3, 1, 2).float() / 255
    model = YOLOv9("c", RES, weights=o.synthetic_weights("c", seed=9, calib=x))
    result = {"metric": "yuv420p_vs_bgr24_ingest", "card": info, "model": "yolov9-c", "res": RES, "frame": [H, W],
              "steps": a.steps, "reps": a.reps,
              "h2d_bytes_per_frame": {"bgr24": H * W * 3, "yuv420p": H * W * 3 // 2},
              "cv2_yuv2bgr_1thread_ms_per_frame": round(cv2_proxy(), 3), "by_batch": {}}
    print("cv2 single-core I420->BGR per 1080p frame (ms):", result["cv2_yuv2bgr_1thread_ms_per_frame"], flush=True)
    for B in a.batches:
        yuv, bgr = frames(2 * B, seed=B)
        host = {"yuv420p": [yuv[:B].pin_memory(), yuv[B:].pin_memory()],
                "bgr24": [bgr[:B].pin_memory(), bgr[B:].pin_memory()]}
        fps = {"bgr24": [], "yuv420p": []}
        first = {}
        for fmt in fps:                                   # warm-up: plans, graph capture, pinned result buffers
            run(model, host[fmt], 8, fmt)
        for _ in range(a.reps):
            for fmt in ("bgr24", "yuv420p"):
                f, first[fmt] = run(model, host[fmt], a.steps, fmt)
                fps[fmt].append(round(f, 1))
        same = all(torch.equal(p, q) for p, q in zip(first["bgr24"], first["yuv420p"]))
        lb = {}
        for fmt in ("bgr24", "yuv420p"):
            dev = host[fmt][0].cuda()
            ts = []
            for _ in range(5):
                ops = model.profile(dev, pix_fmt=fmt)
                ts.append(sum(op["ms"] for op in ops if op["kind"] == "letterbox"))
            lb[fmt] = round(statistics.median(ts), 4)
        n_det = int(sum(int((r[..., 4] > 0).sum()) for r in first["yuv420p"]))
        row = {"fps": fps, "fps_median": {k: statistics.median(v) for k, v in fps.items()},
               "letterbox_ms": lb, "detections_identical": same, "detections_checked": n_det}
        result["by_batch"][str(B)] = row
        print(f"B={B}:", json.dumps(row), flush=True)
        del host, yuv, bgr
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not all(r["detections_identical"] for r in result["by_batch"].values()):
        sys.exit("bgr24 and yuv420p detections differ")


if __name__ == "__main__":
    main()
