"""Device tracker (one CTA per camera, csrc/ocsort_gpu.cu) against the host tracker (update_many, csrc/ocsort.cu) on B
cameras that replay the golden sequences with per-camera frame offsets.

For each B: outputs are checked equal frame by frame over the warm-up frames (the timed frames are not compared), then
  - device: CUDA events around each cc_ocsort_gpu_update launch after warm-up (the kernel alone; rows stay on the device);
  - host:   wall time of update_many on the same rows (its worker-thread count is printed).
Both trackers are stepped through the same frames, so they carry the same track counts.

Then CameraBatch.step from pinned host frames (YOLOv9-c at res 640, synthetic weights) on the mixed fleets (a) and (c) of
tools/mixed_fleet.py and the c4 shape of bench.py (8 x 1080p), with the device trackers (what CameraBatch does when the
detector's rows are on the GPU) against `HostTracked`, a CameraBatch that hands its rows to the host trackers.  Targets and
preds of every camera are checked equal over the first steps; the two are then alternated in --reps runs of --steps.

    python tools/track_fleet.py [--cams 8 32 128] [--frames 300] [--warmup 30] [--fleets a c c4] [--steps 200] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from clearcam_b200._lib import CC_MAX_FRAMES, cc_track_job, check, lib   # noqa: E402
from clearcam_b200.ocsort_tracker import ocsort                          # noqa: E402


def sequences(F):
    g = os.path.join(ROOT, "tests", "golden")
    seqs = [np.load(os.path.join(g, "ocsort_mot16.npz"))["frames"], np.load(os.path.join(g, "ocsort_street.npz"))["frames"]]
    s = np.load(os.path.join(g, "ocsort_synth.npz"))
    seqs += [s[f"{k}_frames"] for k in "abc"]
    return [q for q in seqs if len(q) >= F]


def run(B, F, warmup):
    seqs = sequences(F + warmup)
    frames = np.stack([seqs[b % len(seqs)][(37 * b) % (len(seqs[b % len(seqs)]) - F - warmup + 1):][:F + warmup]
                       for b in range(B)], 1)                                     # [F, B, 300, 6]
    dev_rows = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    host = [ocsort.OCSort(max_age=100) for _ in range(B)]
    dev = ocsort.DeviceTrackers(slots=B, capacity=512)          # no growth inside the timed frames
    for b in range(B):
        dev.add(b, max_age=100)
    # equality over the warm-up frames, before any timing
    for f in range(warmup):
        got = dev.update([(b, dev_rows[f, b], 0.5) for b in range(B)])
        exp = ocsort.update_many(host, frames[f], 0.5)
        for b in range(B):
            a = np.array([[*t.tlwh, t.score, t.class_id, t.track_id, t.tracklet_len, t.speed] for t in got[b]]).reshape(-1, 9)
            e = np.array([[*t.tlwh, t.score, t.class_id, t.track_id, t.tracklet_len, t.speed] for t in exp[b]]).reshape(-1, 9)
            assert np.array_equal(a, e), f"B={B} camera {b} frame {f}: device and host trackers differ"
    # device: events around each launch
    out = torch.empty((min(B, CC_MAX_FRAMES), 1024, 9), dtype=torch.float64, device="cuda")
    cs = torch.empty((2, min(B, CC_MAX_FRAMES)), dtype=torch.int32, device="cuda")
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(F)]
    st = ctypes_stream()
    dev_ms = []
    for f in range(warmup, warmup + F):
        tables = []
        for c0 in range(0, B, CC_MAX_FRAMES):
            n = min(CC_MAX_FRAMES, B - c0)
            tables.append(((cc_track_job * n)(*[cc_track_job(dev_rows[f, b].data_ptr(), 300, dev._slot[b], 0.5, 0)
                                               for b in range(c0, c0 + n)]), n))
        e0, e1 = ev[f - warmup]
        e0.record()
        for t, n in tables:
            check(lib().cc_ocsort_gpu_update(dev._h, t, n, out.data_ptr(), 1024, cs[0].data_ptr(), cs[1].data_ptr(), st), "update")
        e1.record()
    torch.cuda.synchronize()
    dev_ms = [a.elapsed_time(b) for a, b in ev]
    status = cs[1].cpu().numpy()
    assert (status == 0).all(), f"device tracker status {status}"   # no slot needed room in the timed frames
    # host: update_many on the same frames
    host_ms = []
    for f in range(warmup, warmup + F):
        t0 = time.perf_counter()
        ocsort.update_many(host, frames[f], 0.5)
        host_ms.append((time.perf_counter() - t0) * 1e3)
    tracks = sum(len(h) for h in host) / B
    nthr = max(1, min(B // 4, os.cpu_count() or 1, 16))
    return {"cameras": B, "frames": F, "live_tracks_per_camera": round(tracks, 1),
            "device_ms_per_step": {"median": float(np.median(dev_ms)), "p90": float(np.percentile(dev_ms, 90))},
            "host_ms_per_step": {"median": float(np.median(host_ms)), "p90": float(np.percentile(host_ms, 90)), "threads": nthr}}


def _rows9(tracks):
    return np.array([[*t.tlwh, t.score, t.class_id, t.track_id, t.tracklet_len, t.speed] for t in tracks], np.float64).reshape(-1, 9)


def camera_batch(fleets, steps, reps):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from mixed_fleet import FLEETS, RES, frame
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9

    class HostTracked(CameraBatch):
        """CameraBatch with the detector's rows handed to the host trackers (update_many), as for host rows."""
        def _launch(self, frames):
            return [(names, rows, None) for names, rows, _ in super()._launch(frames)]

    fr = o.synthetic_frames(2, 320, 320, seed=9)
    x = torch.stack([o.preprocess(f, 320) for f in fr]).flip(-1).permute(0, 3, 1, 2).float() / 255
    model = YOLOv9("c", RES, weights=o.synthetic_weights("c", seed=9, calib=x))
    fl = dict(FLEETS, c4=[((1080, 1920), "bgr24")] * 8)
    for name in fleets:
        cams = {f"cam{k:02d}": c for k, c in enumerate(fl[name])}
        frames = {n: frame(s, f, k).pin_memory() for k, (n, (s, f)) in enumerate(cams.items())}
        ways = {"device": CameraBatch(model, max_age=100), "host": HostTracked(model, max_age=100)}
        for cb in ways.values():
            for n, (_, fmt) in cams.items():
                cb.add_camera(n, pix_fmt=fmt)
        for t in range(10):                                     # equality first (also the warm-up)
            got = {w: cb.step(frames) for w, cb in ways.items()}
            for n in cams:
                d, h = got["device"][n], got["host"][n]
                assert np.array_equal(d.rows, h.rows), f"fleet {name} step {t} camera {n}: rows"
                assert np.array_equal(_rows9(d.targets), _rows9(h.targets)), f"fleet {name} step {t} camera {n}: targets"
                assert np.array_equal(d.preds, h.preds), f"fleet {name} step {t} camera {n}: preds"
        fps = {w: [] for w in ways}
        for _ in range(reps):
            for w, cb in ways.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(steps):
                    cb.step(frames)                             # synchronises on its result reads every step
                fps[w].append(round(steps * len(cams) / (time.perf_counter() - t0), 1))
        print(json.dumps({"fleet": name, "cameras": len(cams), "steps": steps, "camera_batch_frames_per_s": fps}), flush=True)


def ctypes_stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, nargs="+", default=[8, 32, 128])
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--fleets", nargs="*", default=["a", "c", "c4"])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "cpus": os.cpu_count()}))
    for B in a.cams:
        print(json.dumps(run(B, a.frames, a.warmup)), flush=True)
    camera_batch(a.fleets, a.steps, a.reps)


if __name__ == "__main__":
    main()
