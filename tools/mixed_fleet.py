"""What merging cameras of different resolutions and pixel formats into one detector call buys (YOLOv9-c, res 640).

    python tools/mixed_fleet.py [--steps 200] [--reps 3] [--fleets a b c] [--out FILE]

Prints the card's name and power limit, then for each fleet:
  (a) 8 cameras each of 720p, 1080p, 1440p and 2160p, bgr24 (all letterbox to 384 x 640);
  (b) 5 resolutions (720p, 900p, 1080p, 1440p, 2160p) x 3 cameras, every other camera yuv420p;
  (c) 32 x 1080p bgr24: the control, whose call sequence does not change;
it measures two ways of running a step, alternated `reps` times with `steps` steps per run:
  * grouped: one detect_batch per source shape and format (each padded to its batch bucket), the only way before frame
    tables existed;
  * merged: CameraBatch's grouping with frame tables (one detect_frames per net shape, padded with None rows; a group of
    one source shape still calls detect_batch).
Both ways are timed on device-resident frames (frames/s and device time per step from CUDA events around the detector
calls) and through CameraBatch.step from pinned host frames (frames/s; uploads, detector, result reads and trackers,
synchronised every step).  Before any timing, every camera's rows from the two ways are compared: bit for bit, or at
the >= 0.9 match bar where a camera ran in batches of different sizes.  Last, the letterbox op alone for 32 1080p frames:
the plan's op from YOLOv9.profile (the uniform path, median of 5), and one launch of cc_letterbox (uniform) against
cc_letterbox_frames (table-driven) timed with CUDA events (median of 50).  One JSON line at the end.
Weights are synthetic (oracle.yolov9.synthetic_weights): the speed of the kernels does not depend on their values."""
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

RES = 640
FLEETS = {
    "a": [((h, w), "bgr24") for h, w in ((720, 1280), (1080, 1920), (1440, 2560), (2160, 3840)) for _ in range(8)],
    "b": [((h, w), "yuv420p" if (3 * k + i) % 2 else "bgr24")
          for k, (h, w) in enumerate(((720, 1280), (900, 1600), (1080, 1920), (1440, 2560), (2160, 3840))) for i in range(3)],
    "c": [((1080, 1920), "bgr24")] * 32,
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:                 # the numbers below still carry the device name from torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({ex!r})", "max_sm_clock": "unknown"}


_CONTENT = {}


def frame(shape, fmt, k):
    """Camera k's frame: one of two seeded pictures per resolution, rolled by k so that cameras differ."""
    from oracle import yolov9 as o
    H, W = shape
    key = (H, W, k % 2)
    if key not in _CONTENT:
        _CONTENT[key] = o.synthetic_frames(1, H, W, seed=H + k % 2)[0]
    bgr = torch.roll(_CONTENT[key], 16 * k, dims=1)
    if fmt == "bgr24":
        return bgr
    return torch.cat([bgr[..., 1].reshape(-1), bgr[::2, ::2, 0].reshape(-1), bgr[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)


class Grouped:
    """The model without frame tables: CameraBatch then makes one detect_batch per source shape and format."""
    def __init__(self, m):
        self.m = m

    def detect_batch(self, *a, **kw):
        return self.m.detect_batch(*a, **kw)


def match(ref, got):
    A, Bq = ref[ref[:, 4] > 0], got[got[:, 4] > 0]
    if len(A) == 0:
        return 1.0
    if len(Bq) == 0:
        return 0.0
    d = (A[:, None, :4] - Bq[None, :, :4]).abs().max(-1)[0] + (A[:, None, 5] != Bq[None, :, 5]) * 1e6
    return float(((d < 3.0) & ((A[:, None, 4] - Bq[None, :, 4]).abs() < 0.05)).any(1).float().mean())


def device_step_fn(model, cams, dev, merged):
    """A closure running one step on device-resident frames the way `merged` says; returns {camera: rows} (device)."""
    from clearcam_b200.cameras import CameraBatch
    cb = CameraBatch(model if merged else Grouped(model))
    groups = CameraBatch.group_by_shape({n: dev[n] for n in cams}, {n: f for n, (_, f) in cams.items()})
    plan = []
    for net, keys in cb.merge_groups(groups):
        names = [n for k in keys for n in groups[k]]
        b = cb.bucket(len(names))
        if len(keys) == 1:
            batch = torch.zeros((b,) + tuple(dev[names[0]].shape), dtype=torch.uint8, device="cuda")
            for i, n in enumerate(names):
                batch[i].copy_(dev[n])
            plan.append(("batch", names, batch, keys[0][3]))
        else:
            fr = [dev[n] for n in names] + [None] * (b - len(names))
            fm = [cams[n][1] for n in names] + ["bgr24"] * (b - len(names))
            plan.append(("frames", names, fr, fm))

    def step():
        res = {}
        for kind, names, a, f in plan:
            out = model.detect_batch(a, pix_fmt=f) if kind == "batch" else model.detect_frames(a, pix_fmts=f)
            res.update({n: out[i] for i, n in enumerate(names)})
        return res
    return step, [p[0] + ":" + str(len(p[2])) for p in plan]


def time_device(step, steps, n_frames):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return {"fps": round(steps * n_frames / wall, 1), "device_ms_per_step": round(e0.elapsed_time(e1) / steps, 4)}


def time_camera_batch(model, host, steps, merged):
    from clearcam_b200.cameras import CameraBatch
    cb = CameraBatch(model if merged else Grouped(model))
    for n, (_, fmt) in host["cams"].items():
        cb.add_camera(n, pix_fmt=fmt)
    frames = host["frames"]
    for _ in range(3):
        cb.step(frames)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        cb.step(frames)                       # synchronises on its result reads every step
    return round(steps * len(frames) / (time.perf_counter() - t0), 1)


def letterbox_times(model, reps=50):
    from clearcam_b200._lib import check, lib, ptr, stream_ptr
    from clearcam_b200.detection.yolov9 import frame_table
    out = {}
    for fmt in ("bgr24", "yuv420p"):
        frames = [frame((1080, 1920), fmt, k).cuda() for k in range(32)]
        batch = torch.stack(frames)
        prof = [sum(op["ms"] for op in model.profile(batch, pix_fmt=fmt) if op["kind"] == "letterbox") for _ in range(5)]
        code = 0 if fmt == "bgr24" else 2
        dst = torch.empty(32, 384, 640, 3, dtype=torch.uint8, device="cuda")
        table, _ = frame_table(frames, fmt, RES)
        oh, ow = ctypes.c_int(), ctypes.c_int()
        calls = {
            "uniform": lambda: check(lib().cc_letterbox(ptr(batch), code, 32, 1080, 1920, RES, ptr(dst), ctypes.byref(oh),
                                                        ctypes.byref(ow), stream_ptr()), "cc_letterbox"),
            "table": lambda: check(lib().cc_letterbox_frames(ctypes.cast(table, ctypes.c_void_p), 32, RES, ptr(dst),
                                                             ctypes.byref(oh), ctypes.byref(ow), stream_ptr()), "cc_letterbox_frames"),
        }
        ts = {k: [] for k in calls}
        for _ in range(reps):
            for k, fn in calls.items():           # alternated
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                ts[k].append(e0.elapsed_time(e1))
        out[fmt] = {"plan_op_ms": round(statistics.median(prof), 4),
                    **{f"{k}_launch_ms": round(statistics.median(v), 4) for k, v in ts.items()}}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fleets", nargs="+", default=["a", "b", "c"])
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
    result = {"metric": "mixed_fleet", "card": info, "model": "yolov9-c", "res": RES, "steps": a.steps, "reps": a.reps,
              "fleets": {}}
    ok = True
    for name in a.fleets:
        cams = {f"cam{k:02d}": c for k, c in enumerate(FLEETS[name])}
        hostf = {n: frame(s, f, k) for k, (n, (s, f)) in enumerate(cams.items())}
        dev = {n: t.cuda() for n, t in hostf.items()}
        steps = {}
        calls = {}
        for way in ("grouped", "merged"):
            steps[way], calls[way] = device_step_fn(model, cams, dev, way == "merged")
        # agreement before any timing
        rows = {way: {n: r.cpu() for n, r in steps[way]().items()} for way in steps}
        exact = sum(torch.equal(rows["grouped"][n], rows["merged"][n]) for n in cams)
        worst = min(1.0 if torch.equal(rows["grouped"][n], rows["merged"][n]) else match(rows["grouped"][n], rows["merged"][n])
                    for n in cams)
        n_det = int(sum(int((r[:, 4] > 0).sum()) for r in rows["merged"].values()))
        agree = worst >= 0.9
        ok &= agree
        row = {"cameras": len(cams), "calls": calls, "rows_bitwise_equal": f"{exact}/{len(cams)}", "worst_match": round(worst, 3),
               "detections_checked": n_det}
        print(f"fleet {name}:", json.dumps(row), flush=True)
        if not agree:
            result["fleets"][name] = row
            continue
        for way in steps:                                  # warm-up: plans and graph capture
            time_device(steps[way], 5, len(cams))
        dev_t = {w: [] for w in steps}
        for _ in range(a.reps):
            for way in steps:
                dev_t[way].append(time_device(steps[way], a.steps, len(cams)))
        host = {"cams": cams, "frames": {n: t.pin_memory() for n, t in hostf.items()}}
        cb_t = {w: [] for w in steps}
        for _ in range(a.reps):
            for way in steps:
                cb_t[way].append(time_camera_batch(model, host, a.steps, way == "merged"))
        row.update({"device": dev_t, "camera_batch_fps": cb_t,
                    "device_fps_median": {w: statistics.median(r["fps"] for r in v) for w, v in dev_t.items()},
                    "device_ms_median": {w: statistics.median(r["device_ms_per_step"] for r in v) for w, v in dev_t.items()},
                    "camera_batch_fps_median": {w: statistics.median(v) for w, v in cb_t.items()}})
        result["fleets"][name] = row
        print(f"fleet {name}:", json.dumps(row), flush=True)
        del host, dev, hostf
    result["letterbox_32x1080p"] = letterbox_times(model)
    print("letterbox:", json.dumps(result["letterbox_32x1080p"]), flush=True)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not ok:
        sys.exit("merged and grouped detections disagree")


if __name__ == "__main__":
    main()
