"""Recorded videos: `CameraBatch.step_video` (one detector pass over a run of T frames, then one launch per stage) against
`step_alerts` once per frame, YOLOv9-c at res 640 with synthetic weights, frames from pinned memory.

Scenarios: one 1080p bgr24 video; 4 videos of mixed resolution and format; one 1080p video next to 8 live 720p cameras
(each live camera delivers one frame per run: in the per-frame mode it steps with the run's first frame, in the video mode
it is a one-frame run of the same step_video call, so both modes do the same work).  Each scenario first checks every
output equal on the same frames (rows, preds, flags, saves, fired ids), then alternates the two modes in --reps timed
windows per T.  A window is the same max(--T) frames of each video for every T (max(--T) / T runs), and every camera's
tracker, events and alert counts start afresh at its start, so both modes and every T see the same tracker load.
It also times, with CUDA events, the three run launches (tracker, events, alerts) of one camera over T frames against T
single-frame chains on the same detector rows.  Prints one JSON line per measurement, with the card and its power limit.

    python tools/video_fleet.py [--T 8 32 128] [--reps 3]"""
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

from clearcam_b200.alerts import Alert                     # noqa: E402
from clearcam_b200.cameras import CameraBatch              # noqa: E402
from clearcam_b200.detection.yolov9 import YOLOv9          # noqa: E402
from clearcam_b200.ocsort_tracker import ocsort            # noqa: E402
from oracle import yolov9 as o                             # noqa: E402

T0 = 1.7e9
SCENARIOS = {
    "1x1080p": {"v0": ((1080, 1920), "bgr24")},
    "4 mixed": {"v0": ((1080, 1920), "bgr24"), "v1": ((720, 1280), "yuv420p"), "v2": ((1440, 2560), "bgr24"),
                "v3": ((1080, 1920), "yuv420p")},
    "1080p+8 live": dict({"v0": ((1080, 1920), "bgr24")}, **{f"live{i}": ((720, 1280), "bgr24") for i in range(8)}),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def frames_for(shape, fmt, n, seed):
    (H, W) = shape
    base = o.synthetic_frames(1, H, W, seed=seed)[0]
    out = []
    for t in range(n):
        f = base.roll(shifts=(5 * t, 8 * t), dims=(0, 1))
        if fmt == "yuv420p":
            f = torch.cat([f[..., 1].reshape(-1), f[::2, ::2, 0].reshape(-1), f[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)
        out.append(f)
    return torch.stack(out).pin_memory()


def batch(model, cams):
    cb = CameraBatch(model)
    for n, (_, fmt) in cams.items():
        cb.add_camera(n, thresh=0.05, pix_fmt=fmt)
        cb.set_zone(n, [[0.1, 0.1], [0.8, 0.1], [0.9, 0.9], [0.2, 0.8]], False, True)
        cb.set_alerts(n, {"default": Alert.make(max=1, classes=[0, 1, 2, 3, 5, 7]), "any": Alert.make(max=3, window=30, zone=False)})
    return cb


def video_step(cb, data, cams, f0, T, t0=T0):
    fr = {n: (data[n][f0:f0 + T] if n.startswith("v") else data[n][f0 // T % len(data[n])][None]) for n in cams}
    clocks = {n: [t0 + 0.1 * (f0 + f) for f in range(len(fr[n]))] for n in cams}
    return cb.step_video(fr, clocks)


def frame_steps(cb, data, cams, f0, T, t0=T0):
    out = {n: [] for n in cams}
    for f in range(T):
        fr = {n: data[n][f0 + f] for n in cams if n.startswith("v")}
        if f == 0:
            fr.update({n: data[n][f0 // T % len(data[n])] for n in cams if not n.startswith("v")})
        for n, r in cb.step_alerts(fr, now=t0 + 0.1 * (f0 + f)).items():
            out[n].append(r)
    return out


def same(a, b):
    for n in a:
        assert len(a[n]) == len(b[n]), n
        for x, y in zip(a[n], b[n]):
            for u, v in zip(x[:4], y[:4]):
                np.testing.assert_array_equal(u, v)
            assert x.fired == y.fired


def launch_times(model, data, T, reps):
    """Device time of tracker + events + alerts for one camera over T frames: 3 run launches against T single chains."""
    rows = model.detect_batch(data["v0"][:T].cuda())
    ms = {}
    for mode in ("runs", "single"):
        trk = ocsort.DeviceTrackers(slots=4, capacity=1024, event_capacity=1024)     # no growth inside the timed window
        trk.add("v0", max_age=100)
        trk.events("v0", None)
        trk.alerts("v0", [Alert.make(max=1), Alert.make(max=3, window=30, zone=False)])
        times = []
        for r in range(reps + 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev = [(1920, 1080, T0 + 0.1 * (r * T + f)) for f in range(T)]
            loc = [(36000.0, 2)] * T
            a.record()
            if mode == "runs":
                j = trk.launch_runs([("v0", rows, 0.05)], [ev], [loc])
            else:
                js = [trk.launch([("v0", rows[f], 0.05)], events=[ev[f]], alerts=[loc[f]]) for f in range(T)]
            b.record()
            torch.cuda.synchronize()
            trk.finish_runs(j) if mode == "runs" else trk.finish_alerts(js[-1])    # single launches share one buffer set
            if r:
                times.append(a.elapsed_time(b))
        ms[mode] = float(np.median(times))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, nargs="+", default=[8, 32, 128])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    gpu = card()
    xc = o.synthetic_frames(2, 384, 640, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    model = YOLOv9("c", 640, weights=o.synthetic_weights("c", seed=5, calib=xc))
    Tmax = max(a.T)
    need = Tmax
    for name, cams in SCENARIOS.items():
        data = {n: frames_for(shape, fmt, need if n.startswith("v") else 4, seed=i) for i, (n, (shape, fmt)) in enumerate(cams.items())}
        for T in a.T:
            vb, fb = batch(model, cams), batch(model, cams)
            same(video_step(vb, data, cams, 0, T), frame_steps(fb, data, cams, 0, T))      # warm-up and the equality check
            res = {"video": [], "per_frame": []}
            for rep in range(a.reps):
                t0 = T0 + 1000.0 * (rep + 1)                  # later clocks for every window: last_det stays in the past
                for mode, fn, cb in (("video", video_step, vb), ("per_frame", frame_steps, fb)):
                    for n in cams:
                        cb.reset_tracker(n)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    for f0 in range(0, Tmax, T):
                        fn(cb, data, cams, f0, T, t0)
                    torch.cuda.synchronize()
                    res[mode].append(time.perf_counter() - t)
            nvid = sum(1 for n in cams if n.startswith("v"))
            fps = {m: nvid * Tmax / float(np.median(v)) for m, v in res.items()}
            print(json.dumps({"scenario": name, "T": T, "video_frames_per_s": round(fps["video"], 1),
                              "per_frame_frames_per_s": round(fps["per_frame"], 1), "speedup": round(fps["video"] / fps["per_frame"], 2),
                              "gpu": gpu}), flush=True)
    data = {"v0": frames_for((1080, 1920), "bgr24", Tmax, seed=0)}
    for T in a.T:
        ms = launch_times(model, data, T, 5)
        print(json.dumps({"launches": "tracker+events+alerts, 1 camera", "T": T, "run_ms": round(ms["runs"], 3),
                          "single_chains_ms": round(ms["single"], 3), "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
