"""Alerts on the GPU (csrc/alerts_gpu.cu) behind the device tracker and events: fired alerts, description hits and the
object counter equal to the reference's answers in tests/golden/alerts_ref.npz and to the host form (CameraAlerts) on
the same steps; 128 cameras in one launch with skips, resets, remove / re-add and new settings mid-sequence;
non_zone_alert changed in place; argument errors."""
import ctypes
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from clearcam_b200._lib import CCError, cc_alert, cc_track_job, lib
from clearcam_b200.alerts import Alert, CameraAlerts
from clearcam_b200.ocsort_tracker import ocsort

GOLDEN = Path(__file__).parent / "golden" / "alerts_ref.npz"


def _alert(a):
    return Alert.make(classes=a.get("classes"), max=a.get("max"), window=a.get("window"), sched=a.get("sched"),
                      is_on=a.get("is_on", True), is_notif=a.get("is_notif", True), zone=a.get("zone", True), desc=a.get("desc"),
                      threshold=a.get("threshold", 0.28), last_det=a.get("last_det", 0.0))

pytestmark = pytest.mark.gpu


def _sequences():
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from oracle.make_golden_events import sequences
    return sequences()


def test_device_alerts_equal_the_reference_and_the_host_form():
    g = np.load(GOLDEN)
    cfgs = json.loads(str(g["configs"]))
    seqs = _sequences()
    for k, cfg in enumerate(cfgs):
        p = f"c{k}_"
        frames, thr, kw = seqs[cfg["seq"]]
        settings = [dict(a) for a in cfg["alerts"]]
        al = [_alert(a) for a in settings]
        desc = g[p + "desc"].astype(np.float32) / 1024
        trk = ocsort.DeviceTrackers(slots=4)
        trk.add("c", **kw)
        trk.events("c", cfg["zone"], outside=cfg["outside"], non_zone_alert=any(not a.zone for a in al))
        trk.alerts("c", al, desc)
        host = CameraAlerts(al, desc)
        toggles = {}
        for t in cfg["toggles"]:
            toggles.setdefault(t[0], []).append(t[1:])
        times, tod, wday, ran = g[p + "times"], g[p + "tod"], g[p + "wday"], g[p + "ran"]
        n_saves, emb = g[p + "n_saves"], torch.from_numpy(g[p + "emb"].astype(np.float32) / 1024).cuda()
        exact = bool(ran.all())                 # gated steps skip the tracker: compare with the fixture only without them
        fired, hits, e0 = [], [], 0
        gen = torch.Generator(device="cuda").manual_seed(100 + k)
        for i in range(len(times)):
            for t in toggles.get(i, []):
                if t[0] == "alerts_on":
                    trk.set_alerts_on("c", bool(t[1]))
                    host.alerts_on = bool(t[1])
                else:
                    settings[t[1]]["is_on"] = bool(t[2])
                    new = [_alert(a) for a in settings]
                    new[t[1]] = new[t[1]]._replace(last_det=float(t[3]))
                    keep = [j if j != t[1] else -1 for j in range(len(new))]
                    trk.alerts("c", new, desc, keep)
                    host.replace(new, desc, keep)
            now, local = float(times[i]), (int(tod[i]), int(wday[i]))
            m = int(n_saves[i])
            if not ran[i]:
                e0 += m
                continue
            rows = torch.from_numpy(np.ascontiguousarray(frames[cfg["f0"] + i])).cuda()
            jobs = trk.launch([("c", rows, thr)], events=[(cfg["W"], cfg["H"], now)], alerts=[local])
            torch.cuda.synchronize()
            [(preds, flags, saves, f)] = trk.finish_alerts(jobs)
            want = host.step(preds, flags, now, local)
            assert f.tolist() == want, (k, i)
            fired += [(i, j) for j in f.tolist()]
            if exact:
                assert len(saves) == m, (k, i)
            if len(saves):
                e = emb[e0:e0 + len(saves)].contiguous() if exact else torch.randn(len(saves), emb.shape[1], device="cuda", generator=gen) / 8
                [(hit, sim)] = trk.describe([("c", len(saves))], e, [now], [local])
                want = host.describe(e.cpu().numpy(), now, local)
                got = [(s, int(a), float(sim[s, a])) for s, a in enumerate(hit) if a >= 0]
                assert got == want, (k, i)
                np.testing.assert_array_equal(sim, host.similarity(e.cpu().numpy()))
                hits += [(i, s, a) for s, a, _ in got]
            e0 += m
        np.testing.assert_array_equal(trk.counts("c"), host.counter)
        if exact:
            np.testing.assert_array_equal(np.array(fired, np.int32).reshape(-1, 2), g[p + "fired"], err_msg=f"configuration {k}")
            np.testing.assert_array_equal(np.array(hits, np.int32).reshape(-1, 3), g[p + "hits"], err_msg=f"configuration {k}")
            np.testing.assert_array_equal(trk.counts("c"), g[p + "counts"])


def _scene(rng, t, n):
    rows = np.zeros((n, 6), np.float32)
    for i in range(n):
        x, y = 30 + 70 * i + 6 * t + rng.normal(0, 1), 20 + 25 * i + 3 * t + rng.normal(0, 1)
        rows[i] = [x, y, x + 110, y + 160, 0.9 - 0.02 * i, [0, 2, 5, 7][i % 4]]
    return rows


def test_128_cameras_one_launch_with_skips_resets_and_new_settings():
    rng = np.random.default_rng(5)
    trk = ocsort.DeviceTrackers(slots=256)
    cams = [f"cam{i}" for i in range(128)]
    host = {}

    def settings(i):
        return [Alert.make(max=1, classes=[0, 1, 2, 3, 5, 7]), Alert.make(max=1 + i % 3, window=2 + i % 5, zone=False),
                Alert.make(max=2, window=1.5, classes=[0, 2], sched=[[0, 40 + i]] + [True] * 7)]

    def add(c, i):
        trk.add(c, max_age=30)
        trk.events(c, [[0.0, 0.0], [0.6, 0.0], [0.6, 1.0], [0.0, 1.0]] if i % 2 else None, non_zone_alert=True)
        trk.alerts(c, settings(i))
        host[c] = CameraAlerts(settings(i))

    for i, c in enumerate(cams):
        add(c, i)
    fired = 0
    for t in range(50):
        now, local = 5000.0 + 0.5 * t, (t, 3)
        if t == 20:
            trk.reset("cam3")
            host["cam3"].reset()
            trk.remove("cam4")
            add("cam4", 4)
            new = settings(5)
            new[1] = new[1]._replace(window=9.0)
            trk.alerts("cam5", new, keep=[0, -1, 2])
            host["cam5"].replace(new, keep=[0, -1, 2])
        step = [c for i, c in enumerate(cams) if (t + i) % 7 != 0]              # every camera skips some steps
        rows = {c: torch.from_numpy(_scene(rng, t, 3 + cams.index(c) % 6)).cuda() for c in step}
        jobs = trk.launch([(c, rows[c], 0.5) for c in step], events=[(960, 540, now)] * len(step), alerts=[local] * len(step))
        torch.cuda.synchronize()
        for c, (p, f, s, fi) in zip(step, trk.finish_alerts(jobs)):
            assert fi.tolist() == host[c].step(p, f, now, local), (t, c)
            fired += len(fi)
    assert fired > 0
    for c in cams:
        np.testing.assert_array_equal(trk.counts(c), host[c].counter)
    trk.reset_counts("cam0")
    assert trk.counts("cam0").sum() == 0


def test_events_rerun_carries_the_alerts_and_non_zone_alert_in_place():
    trk = ocsort.DeviceTrackers(slots=4, capacity=2, event_capacity=1)      # room for too few: trackers and events grow
    trk.add("c", max_age=30)
    zone = [[0.0, 0.0], [0.3, 0.0], [0.3, 1.0], [0.0, 1.0]]
    trk.events("c", zone, non_zone_alert=False)
    al = [Alert.make(max=1, window=1, zone=False), Alert.make(max=2, window=3)]
    trk.alerts("c", al)
    host = CameraAlerts(al)
    from clearcam_b200.events import ObjectEvents
    ev = ObjectEvents(zone, False, False)
    solo = ocsort.OCSort(max_age=30)
    rng = np.random.default_rng(2)
    fired = 0
    for t in range(30):
        now, local = 100.0 + 0.5 * t, (0, 0)
        if t == 15:                                    # a non-zone alert appears: the event state must not restart
            trk.set_non_zone_alert("c", True)
            ev.non_zone_alert = True
        r = _scene(rng, t, 6)
        jobs = trk.launch([("c", torch.from_numpy(r).cuda(), 0.5)], events=[(960, 540, now)], alerts=[local])
        torch.cuda.synchronize()
        [(p, f, s, fi)] = trk.finish_alerts(jobs)
        hp, hf, hs = ev.update(solo.update(r, 0.5), 960, 540, now)
        np.testing.assert_array_equal(p, hp)
        np.testing.assert_array_equal(f, hf)
        assert fi.tolist() == host.step(hp, hf, now, local)
        fired += len(fi)
    assert fired > 0


def test_argument_errors():
    trk = ocsort.DeviceTrackers(slots=2)
    trk.add("c")
    trk.events("c")
    with pytest.raises(KeyError):
        trk.counts("c")                                               # no alerts yet
    rows = torch.zeros((0, 6), device="cuda")
    with pytest.raises(KeyError):
        trk.launch([("c", rows, 0.5)], events=[(640, 360, 1.0)], alerts=[(0, 0)])
    with pytest.raises(ValueError):
        trk.launch([("c", rows, 0.5)], alerts=[(0, 0)])               # alerts need the events
    with pytest.raises(ValueError):
        trk.alerts("c", [Alert.make(max=1)] * 65)
    with pytest.raises(ValueError):
        trk.alerts("c", [Alert.make(desc="x")])                       # no embeddings
    trk.alerts("c", [Alert.make(max=1)])
    with pytest.raises(CCError):
        trk.alerts("c", [Alert.make(max=2)], keep=[0])                # kept alert of another shape
    with pytest.raises(ValueError):
        trk.launch([("c", rows, 0.5)], events=[(640, 360, 1.0)], alerts=[(0, 9)])     # weekday out of range
    with pytest.raises(ValueError):
        trk.launch([("c", rows, 0.5)], events=[(640, 360, 1.0)], alerts=[(float("nan"), 0)])
    with pytest.raises(CCError):
        trk.describe([("c", 1)], torch.zeros((1, 8), device="cuda"), [float("inf")], [(0, 0)])
    with pytest.raises(ValueError):
        trk.describe([("c", 2)], torch.zeros((1, 8), device="cuda"), [0.0], [(0, 0)])
    L = lib()
    a = (cc_alert * 1)()
    a[0].window, a[0].max = 1.0, 2000
    assert L.cc_ocsort_gpu_alerts_configure(trk._h, trk._slot["c"], a, 1, None, 0, None, None) != 0
    assert b"max 2000" in L.cc_last_error()
    a[0].max, a[0].window = 1, 0.0
    assert L.cc_ocsort_gpu_alerts_configure(trk._h, trk._slot["c"], a, 1, None, 0, None, None) != 0
    a[0].window, a[0].classes[2] = 1.0, 1 << 20
    assert L.cc_ocsort_gpu_alerts_configure(trk._h, trk._slot["c"], a, 1, None, 0, None, None) != 0
    table = (cc_track_job * 2)(cc_track_job(None, 0, trk._slot["c"], 0.5, 0), cc_track_job(None, 0, trk._slot["c"], 0.5, 0))
    d = ctypes.c_void_p(1)
    t = (ctypes.c_double * 4)(0.0, 0.0, 0.0, 0.0)
    assert L.cc_ocsort_gpu_alerts(trk._h, table, 2, t, t, d, d, 8, d, d, d, d, None) != 0
    assert b"appears twice" in L.cc_last_error()
    assert L.cc_ocsort_gpu_alerts(trk._h, table, 0, t, t, d, d, 8, d, d, d, d, None) != 0
    assert L.cc_ocsort_gpu_alerts(None, table, 1, t, t, None, d, 8, d, d, d, d, None) != 0


def test_describe_many_cameras_in_chunks_equals_the_host_form():
    """DeviceTrackers.describe over 130 cameras (two launches, per-camera row offsets, cameras without rows) against
    CameraAlerts.describe with the same settings."""
    rng = np.random.default_rng(11)
    D, B = 96, 130
    trk = ocsort.DeviceTrackers(slots=B)
    host, jobs, embs, hits = {}, [], [], 0
    for b in range(B):
        desc = rng.normal(0, 1, (3, D)).astype(np.float32)
        al = [Alert.make(desc="a", threshold=float(rng.uniform(-0.1, 0.1)), last_det=-100.0 * (b % 2)),
              Alert.make(max=1), Alert.make(desc="b", threshold=0.05, zone=False)]
        trk.add(b)
        trk.alerts(b, al, desc)
        host[b] = CameraAlerts(al, desc)
        n = int(rng.integers(0, 5)) if b % 9 else 0
        base = desc[rng.integers(0, 3, n) // 2 * 2]
        embs.append(((base * rng.uniform(0, 0.2, (n, 1)) + rng.normal(0, 1, (n, D))) / np.sqrt(D)).astype(np.float32))
        jobs.append((b, n))
    emb = torch.from_numpy(np.concatenate(embs)).cuda()
    now = [30.0 + b for b in range(B)]
    local = [(100, b % 7) for b in range(B)]
    res = trk.describe(jobs, emb, now, local)
    for b, (hit, sim) in enumerate(res):
        np.testing.assert_array_equal(sim, host[b].similarity(embs[b]))
        want = host[b].describe(embs[b], now[b], local[b])
        assert [(s, int(a), float(sim[s, a])) for s, a in enumerate(hit) if a >= 0] == want, b
        hits += len(want)
    assert hits > 10


def _finder():
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    return of


def test_camera_batch_step_alerts_mailboxes_save_objects_describe_saves_mixed_fleet():
    """A mixed-resolution, mixed-format fleet through mailboxes: step_alerts_mailboxes + save_objects + describe_saves on
    the device equal the host form over the same steps — fired alert ids, description hits with their similarities and
    the object counters — with device alerts configured lazily from settings made before the first step (a last_det, a
    camera switched off), a set_alerts mid-sequence that keeps unchanged alerts and encodes a new description, and
    alerts_on toggled."""
    import io
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.ingest import FrameMailbox
    fleet = {"b180": ((180, 320), "bgr24"), "y180": ((180, 320), "yuv420p"), "b360": ((360, 640), "bgr24"),
             "y360": ((360, 640), "yuv420p"), "b720": ((720, 1280), "bgr24"), "y720": ((720, 1280), "yuv420p")}
    xc = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    m = YOLOv9("c", 320, weights=o.synthetic_weights("c", seed=5, calib=xc))
    cb = CameraBatch(m, max_age=100)
    boxes = {n: FrameMailbox(H, W, pix_fmt=fmt) for n, ((H, W), fmt) in fleet.items()}
    of = _finder()
    T0 = 1.7e9

    def settings(i):
        return {"default": Alert.make(max=1, classes=[0, 1, 2, 3, 5, 7]),
                "any": Alert.make(max=1 + i % 2, window=40, zone=False, last_det=T0 + 5.0 if i == 2 else 0.0),
                "person": Alert.make(desc="a person", threshold=-1.0, last_det=T0 - 30.0 if i == 1 else 0.0),
                "car": Alert.make(desc="a red car", threshold=0.0, zone=False)}
    host, ids = {}, {}

    def host_alerts(n, al, keep=None):
        desc = None                                         # the text embeddings set_alerts encoded
        if any(a.desc is not None for a in al.values()):
            D = len(next(cb._desc[a.desc] for a in al.values() if a.desc is not None))
            desc = np.stack([cb._desc[a.desc] if a.desc is not None else np.zeros(D, np.float32) for a in al.values()])
        if n not in host:
            host[n] = CameraAlerts(list(al.values()), desc)
        else:
            host[n].replace(list(al.values()), desc, keep)
        ids[n] = list(al)

    for i, (n, ((H, W), fmt)) in enumerate(fleet.items()):
        cb.add_camera(n, thresh=0.05, pix_fmt=fmt)
        cb.set_alerts(n, settings(i), of)
        host_alerts(n, settings(i))
    cb.set_alerts_on("y360", False)
    host["y360"].alerts_on = False
    fired = hits = 0
    hit_cams = set()
    for t in range(16):
        now, local = T0 + 25.0 * t, (36000 + 25 * t, 1)
        if t == 8:                                          # new settings: "any" changes, a new description appears
            new = dict(settings(4), any=settings(4)["any"]._replace(window=3.0), bike=Alert.make(desc="a bike", threshold=-1.0))
            old = dict(zip(ids["b720"], host["b720"].alerts))
            keep = [ids["b720"].index(k) if k in old and old[k].settings() == a.settings() else -1 for k, a in new.items()]
            cb.set_alerts("b720", new, of)
            host_alerts("b720", new, keep)
            cb.set_alerts_on("y360", True)
            host["y360"].alerts_on = True
        for i, n in enumerate(boxes):
            (H, W), fmt = fleet[n]
            f = o.synthetic_frames(1, H, W, seed=40 + i)[0].roll(shifts=(3 * t, 5 * t), dims=(0, 1))
            if fmt == "yuv420p":
                f = torch.cat([f[..., 1].reshape(-1), f[::2, ::2, 0].reshape(-1), f[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)
            assert boxes[n].fill(io.BytesIO(f.numpy().tobytes()))
        res = cb.step_alerts_mailboxes(boxes, now=now, local=local)
        assert set(res) == set(fleet)
        for n, r in res.items():
            want = [ids[n][j] for j in host[n].step(r.preds, r.flags, now, local)]
            assert r.fired == want, (t, n)
            fired += len(want)
        saved = cb.save_objects(res, of)
        got = cb.describe_saves(saved, now=now, local=local)
        for n, (saves, files, emb) in saved.items():
            e = None if emb is None else emb.tensor.cpu().numpy()
            want = [] if e is None else [(s, ids[n][a], v) for s, a, v in host[n].describe(e, now, local)]
            assert got[n] == want, (t, n)
            hits += len(want)
            if want:
                hit_cams.add(n)
    for n in fleet:
        np.testing.assert_array_equal(cb.object_counts(n), host[n].counter)
    assert hits > 0 and len(hit_cams) >= 2, (hits, hit_cams)
    assert cb._dev_trk is not None and all(cb._dev_trk.has_alerts(n) for n in fleet)   # the device path ran
    print("fired", fired, "hits", hits, "cameras with hits", sorted(hit_cams))
