"""Object events on the device (csrc/events_gpu.cu, right after the tracker launch) against the host loop INTEGRATION.md
used to prescribe (`CameraBatch.step`, then `ObjectEvents` over each camera's STrack list), on B cameras that replay the
golden sequences with per-camera frame offsets, each with its own zone.

For each B: outputs are checked equal frame by frame over the warm-up frames, then
  - device: CUDA events around each cc_ocsort_gpu_events launch (the kernel alone), queued after the tracker launch;
  - host:   wall time of building the STrack lists from the tracker's rows and running ObjectEvents.update per camera.

Then CameraBatch.step_events from pinned host frames (YOLOv9-c at res 640, synthetic weights) on the fleets of
tools/track_fleet.py, against `step` followed by the host loop.  Every camera's preds, flags and saves are checked equal
over the first steps; the two are then alternated in --reps runs of --steps.

    python tools/event_fleet.py [--cams 8 32 128] [--frames 300] [--warmup 30] [--fleets a c c4] [--steps 200] [--reps 3]"""
import argparse
import ctypes
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from clearcam_b200._lib import CC_MAX_FRAMES, cc_track_job, check, lib   # noqa: E402
from clearcam_b200.events import ObjectEvents                            # noqa: E402
from clearcam_b200.ocsort_tracker import ocsort                          # noqa: E402
from track_fleet import sequences                                        # noqa: E402

W, H = 1920, 1080


def zone(b):
    g = np.random.default_rng(b)
    n = int(g.integers(4, 9))
    a = np.sort(g.uniform(0, 2 * np.pi, n))
    r = g.uniform(0.2, 0.6, n)
    return np.stack([0.5 + r * np.cos(a), 0.5 + r * np.sin(a)], 1).tolist()


def host_loop(evs, rows, counts, now):
    """What INTEGRATION.md's loop costs per step: STrack lists from the rows, then ObjectEvents per camera."""
    return [evs[b].update(ocsort._tracks(rows[b], int(counts[b])), W, H, now) for b in range(len(evs))]


def run(B, F, warmup):
    seqs = sequences(F + warmup)
    frames = np.stack([seqs[b % len(seqs)][(37 * b) % (len(seqs[b % len(seqs)]) - F - warmup + 1):][:F + warmup]
                       for b in range(B)], 1)                                     # [F, B, 300, 6]
    dev_rows = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    dev = ocsort.DeviceTrackers(slots=B, capacity=512, event_capacity=512)       # no growth inside the timed frames
    evs = []
    for b in range(B):
        dev.add(b, max_age=100)
        dev.events(b, zone(b), bool(b % 2), bool(b % 3 == 0))
        evs.append(ObjectEvents(zone(b), bool(b % 2), bool(b % 3 == 0)))
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n = min(B, CC_MAX_FRAMES)
    out = torch.empty((n, 1024, 9), dtype=torch.float64, device="cuda")
    cs = torch.empty((2, n), dtype=torch.int32, device="cuda")
    preds = torch.empty((n, 1024, 7), dtype=torch.float64, device="cuda")
    flags = torch.empty((n, 1024), dtype=torch.uint8, device="cuda")
    saves = torch.empty((n, 1024, 6), dtype=torch.int64, device="cuda")
    ecs = torch.empty((3, n), dtype=torch.int32, device="cuda")
    ev_ms, host_ms = [], []
    for f in range(F + warmup):
        now = 1.7e9 + 0.1 * f
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        got, host_rows = [], []
        for c0 in range(0, B, CC_MAX_FRAMES):
            k = min(CC_MAX_FRAMES, B - c0)
            t = (cc_track_job * k)(*[cc_track_job(dev_rows[f, b].data_ptr(), 300, dev._slot[b], 0.5, 0) for b in range(c0, c0 + k)])
            check(lib().cc_ocsort_gpu_update(dev._h, t, k, out.data_ptr(), 1024, cs[0].data_ptr(), cs[1].data_ptr(), st), "update")
            wh = np.array([(W, H)] * k, np.int32).reshape(-1)
            nw = np.full(k, now)
            e0.record()
            check(lib().cc_ocsort_gpu_events(dev._h, t, k, wh.ctypes.data, nw.ctypes.data, out.data_ptr(), 1024, cs[0].data_ptr(),
                                             cs[1].data_ptr(), preds.data_ptr(), flags.data_ptr(), saves.data_ptr(), 1024,
                                             ecs[0].data_ptr(), ecs[2].data_ptr(), st), "events")
            e1.record()
            torch.cuda.synchronize()
            if f >= warmup:
                ms = e0.elapsed_time(e1)
                if c0 == 0:
                    ev_ms.append(ms)
                else:
                    ev_ms[-1] += ms                             # every launch of the step
            c = ecs.cpu().numpy()
            assert (c[2, :k] == 0).all() and (cs[1, :k].cpu().numpy() == 0).all(), "a camera needed room in the run"
            host_rows.append((out[:k].cpu().numpy(), cs[0, :k].cpu().numpy()))
            if f < warmup:
                got += [(preds[b, :c[0, b]].cpu().numpy(), flags[b, :c[0, b]].cpu().numpy(), saves[b, :c[1, b]].cpu().numpy())
                        for b in range(k)]
        rows = np.concatenate([r for r, _ in host_rows])
        counts = np.concatenate([c for _, c in host_rows])
        t0 = time.perf_counter()
        exp = host_loop(evs, rows, counts, now)
        if f >= warmup:
            host_ms.append((time.perf_counter() - t0) * 1e3)
        else:
            for b in range(B):
                for a, e in zip(got[b], exp[b]):
                    assert np.array_equal(a, e), f"B={B} camera {b} frame {f}: device and host events differ"
    return {"cameras": B, "frames": F, "targets_per_camera": round(float(counts.mean()), 1),
            "device_events_ms_per_step": {"median": float(np.median(ev_ms)), "p90": float(np.percentile(ev_ms, 90))},
            "host_loop_ms_per_step": {"median": float(np.median(host_ms)), "p90": float(np.percentile(host_ms, 90))}}


def camera_batch(fleets, steps, reps):
    from mixed_fleet import FLEETS, RES, frame
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9

    fr = o.synthetic_frames(2, 320, 320, seed=9)
    x = torch.stack([o.preprocess(f, 320) for f in fr]).flip(-1).permute(0, 3, 1, 2).float() / 255
    model = YOLOv9("c", RES, weights=o.synthetic_weights("c", seed=9, calib=x))
    fl = dict(FLEETS, c4=[((1080, 1920), "bgr24")] * 8)
    for name in fleets:
        cams = {f"cam{k:02d}": c for k, c in enumerate(fl[name])}
        frames = {n: frame(s, f, k).pin_memory() for k, (n, (s, f)) in enumerate(cams.items())}
        dev, base = CameraBatch(model, max_age=100), CameraBatch(model, max_age=100)
        evs = {}
        for k, (n, ((h, w), fmt)) in enumerate(cams.items()):
            for cb in (dev, base):
                cb.add_camera(n, pix_fmt=fmt)
            dev.set_zone(n, zone(k), bool(k % 2), bool(k % 3 == 0))
            evs[n] = (ObjectEvents(zone(k), bool(k % 2), bool(k % 3 == 0)), w, h)
        clock = [1.7e9]

        def host_way():
            clock[0] += 0.1
            res = base.step(frames)
            return {n: evs[n][0].update(r.targets, evs[n][1], evs[n][2], clock[0]) for n, r in res.items()}

        def device_way():
            return dev.step_events(frames, now=clock[0])
        for t in range(10):                                     # equality first (also the warm-up)
            h = host_way()
            d = device_way()
            for n in cams:
                for a, e in zip((d[n].preds, d[n].flags, d[n].saves), h[n]):
                    assert np.array_equal(a, e), f"fleet {name} step {t} camera {n}: events differ"
        fps = {"step_events": [], "step+host_loop": []}
        for _ in range(reps):
            for w, fn in (("step_events", device_way), ("step+host_loop", host_way)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(steps):
                    fn()
                fps[w].append(round(steps * len(cams) / (time.perf_counter() - t0), 1))
        print(json.dumps({"fleet": name, "cameras": len(cams), "steps": steps, "frames_per_s": fps}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, nargs="*", default=[8, 32, 128])
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
