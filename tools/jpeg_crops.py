"""What encoding object thumbnails on the GPU costs, next to cv2 on one host core.

    python tools/jpeg_crops.py [--calls 50] [--reps 3] [--out FILE]

Prints the card's name and power limit, then for two workloads, alternated `reps` times:
  * crops: K = 64 crops of 150-600 px sides from 8 1080p BGR frames at quality 95 (the object thumbnails of
    `save_object`); also from the same frames as yuv420p;
  * frames: the 8 whole 1080p frames at quality 85;
the device time of one cc_jpeg_encode_crops call (CUDA events around `calls` back-to-back calls, buffers allocated once),
the wall time of `ObjectFinder.encode_crops` (launch, lengths back, used bytes back, split into `bytes`), the device time
per kernel from one torch.profiler pass (which stage dominates), the bytes that cross PCIe against the raw crops, and
single-thread cv2.imencode of the same crops on this host.  Every GPU file is checked against cv2's bytes first.
Content: smooth gradients with Gaussian noise (sigma 6), seeded.  One JSON line at the end."""
import argparse
import ctypes
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

H, W, NF = 1080, 1920, 8


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({ex!r})", "max_sm_clock": "unknown"}


def frames(seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    out = []
    for i in range(NF):
        base = np.stack([(xx * (0.1 + 0.05 * c) + yy * (0.07 * (c + 1)) + 40 * i) % 256 for c in range(3)], -1)
        out.append(np.clip(base + rng.normal(0, 6, (H, W, 3)), 0, 255).astype(np.uint8))
    return np.stack(out)


def crop_rects(k=64, seed=1):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(k):
        w, h = (int(v) for v in rng.integers(150, 601, 2))
        x, y = int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1))
        out.append((int(rng.integers(0, NF)), x, y, x + w, y + h))
    return np.array(out, np.int32)


class Call:
    """One cc_jpeg_encode_crops call with its buffers allocated up front."""

    def __init__(self, dev, rects, q, src_fmt):
        from clearcam_b200 import ops
        from clearcam_b200._lib import lib, ptr
        self.lib, n = lib(), dev.shape[0]
        self.rects = np.ascontiguousarray(rects, np.int32)
        bounds = np.array([ops.jpeg_bound(r[3] - r[1], r[4] - r[2]) for r in self.rects], np.int64)
        self.offsets = np.ascontiguousarray(np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.int64))
        need = ctypes.c_size_t(0)
        self.args = (ptr(dev), n, H, W, src_fmt, self.rects.ctypes.data, len(self.rects), q)
        assert self.lib.cc_jpeg_encode_crops(*self.args, None, 0, None, None, None, 0, ctypes.byref(need), None) == 0
        self.out = torch.empty(int(bounds.sum()), dtype=torch.uint8, device="cuda")
        self.lengths = torch.empty(len(self.rects), dtype=torch.int64, device="cuda")
        self.ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
        self.need = need.value
        self.ptr = ptr

    def __call__(self):
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = self.lib.cc_jpeg_encode_crops(*self.args, self.ptr(self.out), self.out.numel(), self.offsets.ctypes.data,
                                           self.ptr(self.lengths), self.ptr(self.ws), self.need, None, s)
        assert rc == 0, self.lib.cc_last_error()


def device_ms(call, n):
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_breakdown(call, n=10):
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "jpeg_" in ev.key:
            name = ev.key.split("jpeg_")[1].split("_kernel")[0]
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out[name] = out.get(name, 0.0) + t / 1e3 / n
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def cv2_ms(fr, rects, q):
    import cv2
    cv2.setNumThreads(1)
    crops = [np.ascontiguousarray(fr[f, y1:y2, x1:x2]) for f, x1, y1, x2, y2 in rects]
    for c in crops[:4]:
        cv2.imencode(".jpg", c, [cv2.IMWRITE_JPEG_QUALITY, q])
    t0 = time.perf_counter()
    for c in crops:
        cv2.imencode(".jpg", c, [cv2.IMWRITE_JPEG_QUALITY, q])
    return (time.perf_counter() - t0) * 1e3, [cv2.imencode(".jpg", c, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes() for c in crops]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    import cv2
    from clearcam_b200.models.objects import ObjectFinder
    info = card()
    print("card:", info, flush=True)
    fr = frames()
    yuv = np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420) for f in fr])
    conv = np.stack([cv2.cvtColor(y, cv2.COLOR_YUV2BGR_I420) for y in yuv])
    dev, dev_y = torch.from_numpy(fr).cuda(), torch.from_numpy(yuv).cuda()
    rects = crop_rects()
    full = np.array([(i, 0, 0, W, H) for i in range(NF)], np.int32)
    work = {"crops_q95_bgr24": (dev, rects, 95, 1, "bgr24", fr), "crops_q95_yuv420p": (dev_y, rects, 95, 2, "yuv420p", conv),
            "frames_q85_bgr24": (dev, full, 85, 1, "bgr24", fr)}
    finder = ObjectFinder()
    result = {"metric": "jpeg_encode_crops", "card": info, "frames": [NF, H, W], "calls": a.calls, "reps": a.reps, "by_workload": {}}
    rows = {}
    for name, (d, r, q, fmt, pix, host) in work.items():
        ref_ms, ref = cv2_ms(host, r, q)
        got = finder.encode_crops(d, r, quality=q, pix_fmt=pix)
        assert got == ref, f"{name}: GPU bytes differ from cv2"
        raw = int(sum((x2 - x1) * (y2 - y1) * 3 for _, x1, y1, x2, y2 in r))
        rows[name] = {"K": len(r), "quality": q, "identical_to_cv2": True, "device_ms": [], "encode_crops_wall_ms": [],
                      "cv2_imencode_1thread_ms": round(ref_ms, 2), "pcie_bytes": int(sum(len(b) for b in got)), "raw_crop_bytes": raw,
                      "call": Call(d, r, q, fmt)}
    for _ in range(a.reps):                                  # alternate the workloads
        for name, (d, r, q, fmt, pix, _) in work.items():
            row = rows[name]
            row["device_ms"].append(round(device_ms(row["call"], a.calls), 4))
            finder.encode_crops(d, r, quality=q, pix_fmt=pix)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(10):
                finder.encode_crops(d, r, quality=q, pix_fmt=pix)
            row["encode_crops_wall_ms"].append(round((time.perf_counter() - t0) * 100, 3))
    for name, row in rows.items():
        row["kernels_ms"] = kernel_breakdown(row.pop("call"))
        row["device_ms_median"] = statistics.median(row["device_ms"])
        row["encode_crops_wall_ms_median"] = statistics.median(row["encode_crops_wall_ms"])
        result["by_workload"][name] = row
        print(f"{name}:", json.dumps(row), flush=True)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
