"""What decoding JPEG files on the GPU costs, next to cv2.imdecode on one host core.

    python tools/jpeg_decode.py [--calls 50] [--reps 3] [--out FILE]

Prints the card's name and power limit, then for three workloads, alternated `reps` times:
  * thumbs: 64 object thumbnails (150-600 px sides, quality 95) made by the project's encoder from seeded synthetic 1080p
    frames, decoded by cc_jpeg_decode (the stored thumbnails `clip_latest_img` / search-by-image read back);
  * frame: one 1080p file at quality 85 (an uploaded image);
  * chain: the same 64 crops through cc_jpeg_crops_decoded (crop -> the pixels of its JPEG file, no entropy coding);
the device time of one call (CUDA events around `calls` back-to-back calls, buffers allocated once), the wall time of the
Python entry point (ops.jpeg_decode: parse, pinned copy, launch, sync; ops.jpeg_crops_decoded), the device time per kernel
from one torch.profiler pass, and single-thread cv2.imdecode of the same files on this host.  Every GPU image is checked
against cv2 first.  One JSON line at the end."""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.jpeg_crops import H, W, NF, card, crop_rects, frames, device_ms  # noqa: E402


class Decode:
    """One cc_jpeg_decode call with its buffers allocated up front."""

    def __init__(self, files):
        from clearcam_b200 import ops
        from clearcam_b200._lib import lib, ptr
        self.b = ops.JpegBatch(files)
        self.out, self.st = self.b.decode()
        self.lib, self.ptr = lib(), ptr
        need = ctypes.c_size_t(0)
        d, h, t = self.b._ptrs()
        assert self.lib.cc_jpeg_decode(d, h, t, self.b.K, None, 0, 0, None, None, None, 0, ctypes.byref(need), None) == 0
        self.ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
        self.need = need.value

    def __call__(self):
        d, h, t = self.b._ptrs()
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = self.lib.cc_jpeg_decode(d, h, t, self.b.K, self.ptr(self.out), self.out.shape[1], self.out.shape[2], self.ptr(self.st),
                                     None, self.ptr(self.ws), self.need, None, s)
        assert rc == 0, self.lib.cc_last_error()


class Chain:
    """One cc_jpeg_crops_decoded call with its buffers allocated up front."""

    def __init__(self, dev, rects, q):
        from clearcam_b200 import ops
        from clearcam_b200._lib import lib, ptr
        self.lib, self.ptr = lib(), ptr
        self.rects = np.ascontiguousarray(rects, np.int32)
        self.out, self.st = ops.jpeg_crops_decoded(dev, self.rects, q, 1)
        self.args = (ptr(dev), dev.shape[0], H, W, 1, self.rects.ctypes.data, len(self.rects), q)
        need = ctypes.c_size_t(0)
        assert self.lib.cc_jpeg_crops_decoded(*self.args, None, 0, 0, None, None, 0, ctypes.byref(need), None) == 0
        self.ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
        self.need = need.value

    def __call__(self):
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = self.lib.cc_jpeg_crops_decoded(*self.args, self.ptr(self.out), self.out.shape[1], self.out.shape[2], self.ptr(self.st),
                                            self.ptr(self.ws), self.need, None, s)
        assert rc == 0, self.lib.cc_last_error()


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
        key = ev.key
        name = key.split("jdec_")[1].split("_kernel")[0] if "jdec_" in key else \
            "encoder_transform" if "jpeg_transform" in key else "memset" if "emset" in key else None
        if name:
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out[name] = out.get(name, 0.0) + t / 1e3 / n
    tot = sum(out.values()) or 1.0
    return {k: {"ms": round(v, 4), "share": round(v / tot, 3)} for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def cv2_ms(files):
    import cv2
    cv2.setNumThreads(1)
    for f in files[:4]:
        cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)
    t0 = time.perf_counter()
    for f in files:
        cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    import cv2
    from clearcam_b200 import ops
    info = card()
    print("card:", info, flush=True)
    fr = frames()
    dev = torch.from_numpy(fr).cuda()
    rects = crop_rects()
    thumbs = ops.jpeg_encode_crops(dev, rects, 95, 1)
    frame = cv2.imencode(".jpg", fr[0], [cv2.IMWRITE_JPEG_QUALITY, 85])[1].tobytes()
    dec = lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)   # noqa: E731
    work = {"thumbs_64_q95": thumbs, "frame_1080p_q85": [frame]}
    result = {"metric": "jpeg_decode", "card": info, "calls": a.calls, "reps": a.reps, "by_workload": {}}
    rows = {}
    for name, files in work.items():
        out, sizes, st = ops.jpeg_decode(files)
        o, st = out.cpu().numpy(), st.cpu().numpy()
        assert (st == 0).all(), f"{name}: status {st}"
        for k, f in enumerate(files):
            w, h = sizes[k]
            assert np.array_equal(o[k, :h, :w], dec(f)), f"{name}: image {k} differs from cv2"
        rows[name] = {"K": len(files), "bytes": int(sum(len(f) for f in files)), "identical_to_cv2": True, "device_ms": [],
                      "wall_ms": [], "cv2_imdecode_1thread_ms": [], "call": Decode(files), "files": files}
    pix, st = ops.jpeg_crops_decoded(dev, rects, 95, 1)
    assert (st.cpu().numpy() == 0).all()
    pix = pix.cpu().numpy()
    for k, (f, x1, y1, x2, y2) in enumerate(rects):
        assert np.array_equal(pix[k, :y2 - y1, :x2 - x1], dec(thumbs[k])), f"chain: crop {k} differs from cv2"
    rows["chain_64_crops_q95"] = {"K": len(rects), "identical_to_cv2": True, "device_ms": [], "wall_ms": [],
                                  "cv2_imdecode_1thread_ms": [], "call": Chain(dev, rects, 95), "files": thumbs}
    for _ in range(a.reps):                                  # alternate the workloads
        for name, row in rows.items():
            row["device_ms"].append(round(device_ms(row["call"], a.calls), 4))
            fn = (lambda: ops.jpeg_crops_decoded(dev, rects, 95, 1)) if name.startswith("chain") else \
                (lambda files=row["files"]: ops.jpeg_decode(files)[2].cpu())
            fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
            row["wall_ms"].append(round((time.perf_counter() - t0) * 100, 3))
            row["cv2_imdecode_1thread_ms"].append(round(cv2_ms(row["files"]), 3))
    for name, row in rows.items():
        row["kernels"] = kernel_breakdown(row.pop("call"))
        row.pop("files")
        for key in ("device_ms", "wall_ms", "cv2_imdecode_1thread_ms"):
            row[key + "_median"] = statistics.median(row[key])
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
