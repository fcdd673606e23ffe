"""Alerts on the device (csrc/alerts_gpu.cu) against the per-alert host loop INTEGRATION.md used to prescribe, at B cameras
with 3 alerts each: init_cam's default alert, a zone alert and a description alert.

Launch mode (per B, cameras replaying the golden sequences with per-camera frame offsets).  Two device handles step the
same rows: one runs the tracker and events, the other the tracker, events and alerts; CUDA events around each launch give
the alerts' share as the difference of the two.  DeviceTrackers.describe runs on each frame's saved objects, whose
embeddings are drawn near the description half of the time so that hits occur.  Fired alerts, hits, similarity matrices
and object counters are checked equal to CameraAlerts (frozen clock) at every frame.  The host loop is timed on its own
state: per preds row and alert, get_counts and add with a clock reading each, then the firing loop and the description
loop with time.localtime() per is_active, as the reference reads them.

End-to-end mode (per B, YOLOv9-c at res 640 with synthetic weights and a synthetic ViT-B/32 finder, 720p bgr24 frames in
pinned memory).  `step_alerts` + `save_objects` + `describe_saves` against `step_events` + `save_objects` + the host loop,
alternated in --reps runs of --steps after --check steps whose fired alerts and hits are checked equal.

    python tools/alert_fleet.py [--cams 8 32 128] [--frames 200] [--warmup 20] [--steps 30] [--reps 2] [--check 14]"""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from clearcam_b200.alerts import WARMUP, Alert, CameraAlerts, local_time   # noqa: E402
from clearcam_b200.ocsort_tracker import ocsort                              # noqa: E402
from track_fleet import sequences                                            # noqa: E402

W, H, D = 1920, 1080, 512
ZONE = [[0.1, 0.1], [0.8, 0.1], [0.9, 0.9], [0.2, 0.8]]


def alerts():
    return [Alert.make(max=1, classes=[0, 1, 2, 3, 5, 7]), Alert.make(max=3, window=30, zone=True),
            Alert.make(desc="a person at the door", threshold=0.3, zone=False)]


def host_loop(al, preds, flags, embs):
    """The loop INTEGRATION.md prescribed before step_alerts, on alerts.py's counters: a clock reading per get_counts,
    add and is_active, as the reference takes them (its answers follow the wall clock, so it runs on its own state)."""
    def max_reached(a, c):
        c.prune(time.time())
        return bool(a.max) and any(len(q) >= a.max for q in c.q.values())
    for row, f in zip(preds, flags):
        cls = int(row[5])
        if f & 1:
            al.counter[cls] += 1
        for a, c in zip(al.alerts, al.counts):
            if not max_reached(a, c) and ((f & 1 and not a.zone) or (f & 2 and a.zone)):
                c.add(cls, time.time())
    if al.warm > WARMUP:
        for i, (a, c) in enumerate(zip(al.alerts, al.counts)):
            if a.desc is not None:
                continue
            if not a.is_active(al.alerts_on, local_time(time.time())):
                c.q = {}
                continue
            if max_reached(a, c) and time.time() - al.last_det[i] >= a.span:
                al.last_det[i] = time.time()
    else:
        al.warm += 1
    for e in embs:
        for i, a in enumerate(al.alerts):
            if time.time() - al.last_det[i] < 60 or not a.is_active(al.alerts_on, local_time(time.time())) or a.desc is None:
                continue
            if float(al.desc_emb[i] @ e) > a.threshold:
                al.last_det[i] = time.time()
                break


def saved_embeddings(g, desc, n):
    """n object embeddings, half of them near the description (row 2 of desc), unit length."""
    e = g.normal(0, 1, (n, D)).astype(np.float32)
    near = g.random(n) < 0.5
    e[near] += 12.0 * desc[2]
    return (e / np.linalg.norm(e, axis=1, keepdims=True)).astype(np.float32)


def launch_mode(B, F, warmup):
    seqs = sequences(F + warmup)
    frames = np.stack([seqs[b % len(seqs)][(37 * b) % (len(seqs[b % len(seqs)]) - F - warmup + 1):][:F + warmup]
                       for b in range(B)], 1)                                     # [F, B, 300, 6]
    dev_rows = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    g = np.random.default_rng(B)
    desc = g.normal(0, 1, (3, D)).astype(np.float32)
    desc /= np.linalg.norm(desc, axis=1, keepdims=True)
    ev_only = ocsort.DeviceTrackers(slots=B, capacity=512, event_capacity=512)
    dev = ocsort.DeviceTrackers(slots=B, capacity=512, event_capacity=512)
    check, ref = [], []
    for b in range(B):
        for d in (ev_only, dev):
            d.add(b, max_age=100)
            d.events(b, ZONE, False, True)
        dev.alerts(b, alerts(), desc)
        check.append(CameraAlerts(alerts(), desc))
        ref.append(CameraAlerts(alerts(), desc))
    t_ev, t_al, t_ds, t_host = [], [], [], []
    fired = hits = 0
    for f in range(F + warmup):
        now, local = 1.76e9 + 0.1 * f, (36000 + f // 10, 2)
        jobs = [(b, dev_rows[f, b], 0.5) for b in range(B)]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        pe = ev_only.launch(jobs, events=[(W, H, now)] * B)
        ev[1].record()
        pa = dev.launch(jobs, events=[(W, H, now)] * B, alerts=[local] * B)
        ev[2].record()
        torch.cuda.synchronize()
        ev_only.finish_events(pe)
        res = dev.finish_alerts(pa)
        n_saves = [len(r[2]) for r in res]
        emb_h = saved_embeddings(g, desc, sum(n_saves))
        emb = torch.from_numpy(emb_h).cuda()
        t0 = time.perf_counter()
        ds = dev.describe([(b, n_saves[b]) for b in range(B)], emb, [now] * B, [local] * B) if sum(n_saves) else None
        t1 = time.perf_counter()
        k = 0
        h0 = time.perf_counter()
        for b in range(B):
            host_loop(ref[b], res[b][0], res[b][1], emb_h[k:k + n_saves[b]])
            k += n_saves[b]
        h1 = time.perf_counter()
        k = 0
        for b in range(B):
            e = emb_h[k:k + n_saves[b]]
            k += n_saves[b]
            assert res[b][3].tolist() == check[b].step(res[b][0], res[b][1], now, local), (B, f, b)
            want = check[b].describe(e, now, local)
            if ds is not None:
                hit, sim = ds[b]
                assert np.array_equal(sim, check[b].similarity(e), equal_nan=True), (B, f, b)   # NaN: no description
                assert [(s, int(a), float(sim[s, a])) for s, a in enumerate(hit) if a >= 0] == want, (B, f, b)
            fired += len(res[b][3])
            hits += len(want)
        if f >= warmup:
            t_ev.append(ev[0].elapsed_time(ev[1]))
            t_al.append(ev[1].elapsed_time(ev[2]))
            t_ds.append((t1 - t0) * 1e3)
            t_host.append((h1 - h0) * 1e3)
    for b in range(B):
        assert (dev.counts(b) == check[b].counter).all()
    pct = lambda v: [round(float(np.median(v)), 4), round(float(np.percentile(v, 90)), 4)]   # noqa: E731
    return {"mode": "launch", "cams": B, "frames": F, "fired": fired, "hits": hits,
            "track_events_ms": pct(t_ev), "track_events_alerts_ms": pct(t_al),
            "alerts_share_ms_median": round(float(np.median(t_al) - np.median(t_ev)), 4),
            "describe_ms": pct(t_ds), "host_loop_ms": pct(t_host)}


def end_to_end(B, steps, reps, n_check):
    from mixed_fleet import frame
    from oracle import clip as oc
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    fr = o.synthetic_frames(2, 320, 320, seed=9)
    x = torch.stack([o.preprocess(f, 320) for f in fr]).flip(-1).permute(0, 3, 1, 2).float() / 255
    model = YOLOv9("c", 640, weights=o.synthetic_weights("c", seed=9, calib=x))
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    cams = [f"cam{k:03d}" for k in range(B)]
    frames = {n: frame((720, 1280), "bgr24", k).pin_memory() for k, n in enumerate(cams)}
    dev, base = CameraBatch(model, max_age=100), CameraBatch(model, max_age=100)
    al = dict(zip(("default", "zone", "desc"), alerts()))
    al["desc"] = al["desc"]._replace(threshold=-1.0)        # every saved object is a candidate: the loop does its work
    for n in cams:
        for cb in (dev, base):
            cb.add_camera(n)
            cb.set_alerts(n, al, of)
            cb.set_zone(n, ZONE, False, True)
    ref = {n: CameraAlerts(list(al.values()), base.cams[n].alerts.desc_emb) for n in cams}
    check = {n: CameraAlerts(list(al.values()), base.cams[n].alerts.desc_emb) for n in cams}
    clock = {"dev": 1.7e9, "host": 1.7e9}              # each way's own clock, advanced alike: both save and embed alike

    def device_way():
        clock["dev"] += 1.5
        now, local = clock["dev"], local_time(clock["dev"])
        res = dev.step_alerts(frames, now=now, local=local)
        return res, dev.describe_saves(dev.save_objects(res, of), now=now, local=local), now, local

    def host_way():
        clock["host"] += 1.5
        res = base.step_events(frames, now=clock["host"])
        saved = base.save_objects(res, of)
        for n, r in res.items():
            e = saved[n][2]
            host_loop(ref[n], r.preds, r.flags, [] if e is None else e.tensor.cpu().numpy())
        return res, saved
    for t in range(n_check):                                  # equality first (also the warm-up)
        res, hits, now, local = device_way()
        hres, saved = host_way()
        for n in cams:
            assert np.array_equal(res[n].preds, hres[n].preds) and np.array_equal(res[n].flags, hres[n].flags)
            ids = list(al)
            assert res[n].fired == [ids[i] for i in check[n].step(hres[n].preds, hres[n].flags, now, local)], (B, t, n)
            e = saved[n][2]
            want = [] if e is None else [(s, ids[a], v) for s, a, v in check[n].describe(e.tensor.cpu().numpy(), now, local)]
            assert hits[n] == want, (B, t, n)
    fps = {"step_alerts+describe_saves": [], "step_events+host_loop": []}
    for _ in range(reps):
        for w, fn in (("step_alerts+describe_saves", device_way), ("step_events+host_loop", host_way)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                fn()
            fps[w].append(round(steps * B / (time.perf_counter() - t0), 1))
    return {"mode": "end_to_end", "cams": B, "steps": steps, "frames_per_s": fps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, nargs="+", default=[8, 32, 128])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--check", type=int, default=14)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"card": card}))
    for B in a.cams:
        print(json.dumps(launch_mode(B, a.frames, a.warmup)), flush=True)
    for B in a.cams:
        print(json.dumps(end_to_end(B, a.steps, a.reps, a.check)), flush=True)


if __name__ == "__main__":
    main()
