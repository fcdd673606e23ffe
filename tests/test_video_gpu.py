"""Runs of consecutive frames on the GPU (DeviceTrackers.launch_runs / finish_runs, csrc/*_gpu.cu run kernels) and
CameraBatch.step_video: one launch per stage over T frames equals T single-frame launches and the host objects, frame by
frame; several cameras of different T in one launch; growth in the middle of a run; a failing frame stops its camera only;
description alerts across the frames of a run; the end-to-end video path against step_alerts; argument errors."""
import ctypes
import io
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from clearcam_b200._lib import CC_MAX_FRAMES, CC_TRACK_OVERFLOW, CCError, cc_track_run, lib
from clearcam_b200.alerts import Alert, CameraAlerts
from clearcam_b200.events import ObjectEvents
from clearcam_b200.ocsort_tracker import ocsort

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
GOLDEN = Path(__file__).parent / "golden" / "alerts_ref.npz"


def _alert(a):
    return Alert.make(classes=a.get("classes"), max=a.get("max"), window=a.get("window"), sched=a.get("sched"),
                      is_on=a.get("is_on", True), is_notif=a.get("is_notif", True), zone=a.get("zone", True), desc=a.get("desc"),
                      threshold=a.get("threshold", 0.28), last_det=a.get("last_det", 0.0))


def _sequences():
    sys.path.insert(0, str(ROOT))
    from oracle.make_golden_events import sequences
    return sequences()


def _eq(a, b, msg):
    assert len(a) == len(b), msg
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            np.testing.assert_array_equal(u, v, err_msg=str(msg))


def _setup(trk, cam, kw, zone, outside, al, desc=None):
    trk.add(cam, **kw)
    trk.events(cam, zone, outside=outside, non_zone_alert=any(not a.zone for a in al))
    trk.alerts(cam, al, desc)


def _singles(trk, cam, frames, thr, wh, times, local):
    out = []
    for i, r in enumerate(frames):
        j = trk.launch([(cam, torch.from_numpy(np.ascontiguousarray(r)).cuda(), thr)], events=[wh + (times[i],)], alerts=[local[i]])
        torch.cuda.synchronize()
        out += trk.finish_alerts(j)
    return out


def _runs(trk, cam, frames, thr, wh, times, local, T):
    out = []
    for f0 in range(0, len(frames), T):
        r = torch.from_numpy(np.ascontiguousarray(np.stack(frames[f0:f0 + T]))).cuda()
        n = r.shape[0]
        j = trk.launch_runs([(cam, r, thr)], [[wh + (t,) for t in times[f0:f0 + n]]], [local[f0:f0 + n]])
        torch.cuda.synchronize()
        [got] = trk.finish_runs(j)
        assert len(got) == n
        out += got
    return out


def test_runs_equal_single_steps_and_host_objects_on_the_golden_sequences():
    """Every alerts fixture configuration (zones, schedules, description alerts) on its tracker sequence: runs of T frames
    for T in {1, 2, 7, 32, 128} give, at every frame, what single-frame launches and the host objects give."""
    g = np.load(GOLDEN)
    cfgs = json.loads(str(g["configs"]))
    seqs = _sequences()
    for k, cfg in enumerate(cfgs):
        p = f"c{k}_"
        frames, thr, kw = seqs[cfg["seq"]]
        frames = [np.asarray(f, np.float32) for f in frames[cfg["f0"]:]]
        al = [_alert(dict(a)) for a in cfg["alerts"]]
        desc = g[p + "desc"].astype(np.float32) / 1024
        times = [float(t) for t in g[p + "times"]][:len(frames)]
        local = [(int(a), int(b)) for a, b in zip(g[p + "tod"], g[p + "wday"])][:len(frames)]
        frames = frames[:len(times)]
        wh = (cfg["W"], cfg["H"])
        trk = ocsort.DeviceTrackers(slots=8)
        _setup(trk, "s", kw, cfg["zone"], cfg["outside"], al, desc)
        want = _singles(trk, "s", frames, thr, wh, times, local)
        solo, ev, host = ocsort.OCSort(**kw), ObjectEvents(cfg["zone"], cfg["outside"], any(not a.zone for a in al)), CameraAlerts(al, desc)
        for i, r in enumerate(frames):
            hp, hf, hs = ev.update(solo.update(r, thr), *wh, times[i])
            fired = host.step(hp, hf, times[i], local[i])
            _eq([want[i]], [(hp, hf, hs, np.array(fired, np.int32))], (k, "host", i))
        for T in (1, 2, 7, 32, 128):
            c = f"r{T}"
            _setup(trk, c, kw, cfg["zone"], cfg["outside"], al, desc)
            _eq(_runs(trk, c, frames, thr, wh, times, local, T), want, (k, T))
            np.testing.assert_array_equal(trk.counts(c), trk.counts("s"))
            assert trk.num_tracks(c) == trk.num_tracks("s")


def _scene(rng, t, n, drift=6):
    rows = np.zeros((n, 6), np.float32)
    for i in range(n):
        if rng.random() < 0.15:
            continue                                           # a missed detection now and then
        x, y = 30 + 70 * i + drift * t + rng.normal(0, 1.5), 20 + 25 * i + 3 * t + rng.normal(0, 1.5)
        rows[i] = [x, y, x + 110 + rng.normal(0, 2), y + 160, 0.9 - 0.02 * i, [0, 2, 5, 7][i % 4]]
    return rows


def _zone(rng, n):
    a = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = rng.uniform(0.2, 0.5, n)
    return np.stack([0.5 + r * np.cos(a), 0.5 + r * np.sin(a)], 1).tolist()


def test_random_scenes_many_cameras_different_lengths_growth_and_continuation():
    """12 cameras, zones of 3..256 vertices, 3 alerts each, capacities of 1 (tracker and events grow in the middle of runs):
    one launch per stage over runs of different lengths, then single steps, then runs again, equal at every frame to
    single-frame launches on a second handle; a camera left out keeps its state."""
    rng = np.random.default_rng(7)
    cams = [f"c{i}" for i in range(12)]
    run_trk = ocsort.DeviceTrackers(slots=16, capacity=1, event_capacity=1)
    one_trk = ocsort.DeviceTrackers(slots=16)
    for i, c in enumerate(cams):
        zone = _zone(rng, [3, 17, 256][i % 3]) if i % 4 else None
        al = [Alert.make(max=1, classes=[0, 2]), Alert.make(max=2, window=3, zone=False),
              Alert.make(max=1 + i % 2, window=1.5, classes=[5, 7], sched=[[0, 50000]] + [True] * 7)]
        for trk in (run_trk, one_trk):
            _setup(trk, c, dict(max_age=10 + i), zone, bool(i % 3 == 1), al)
    scenes = {c: [_scene(rng, t, 4 + i % 7, drift=4 + i % 5) for t in range(160)] for i, c in enumerate(cams)}
    pos = {c: 0 for c in cams}
    lengths = [[1, 2, 7, 32, 128, 5], [3], [128], [9, 9, 9]]
    for phase in range(4):
        jobs, evs, als = [], [], []
        for i, c in enumerate(cams):
            if phase == 1:
                continue
            if (phase + i) % 5 == 0:
                continue                                       # left out of this launch
            T = lengths[phase][i % len(lengths[phase])]
            T = min(T, 160 - pos[c])
            if T < 1:
                continue
            f0 = pos[c]
            jobs.append((c, torch.from_numpy(np.stack(scenes[c][f0:f0 + T])).cuda(), 0.5))
            evs.append([(960, 540, 100.0 + 0.4 * f) for f in range(f0, f0 + T)])
            als.append([(36000.0 + f, 2) for f in range(f0, f0 + T)])
        if phase == 1:                                         # single-frame launches on the run handle too
            for f in range(2):
                for trk in (run_trk,):
                    j = trk.launch([(c, torch.from_numpy(scenes[c][pos[c]]).cuda(), 0.5) for c in cams],
                                   events=[(960, 540, 100.0 + 0.4 * pos[c]) for c in cams], alerts=[(36000.0 + pos[c], 2) for c in cams])
                    torch.cuda.synchronize()
                    got = trk.finish_alerts(j)
                j = one_trk.launch([(c, torch.from_numpy(scenes[c][pos[c]]).cuda(), 0.5) for c in cams],
                                   events=[(960, 540, 100.0 + 0.4 * pos[c]) for c in cams], alerts=[(36000.0 + pos[c], 2) for c in cams])
                torch.cuda.synchronize()
                _eq(got, one_trk.finish_alerts(j), ("singles", f))
                for c in cams:
                    pos[c] += 1
            continue
        r = run_trk.launch_runs(jobs, evs, als)
        torch.cuda.synchronize()
        got = run_trk.finish_runs(r)
        for (c, rows, _), per, ev, a in zip(jobs, got, evs, als):
            assert len(per) == rows.shape[0]
            want = []
            for f in range(rows.shape[0]):
                j = one_trk.launch([(c, rows[f].contiguous(), 0.5)], events=[ev[f]], alerts=[a[f]])
                torch.cuda.synchronize()
                want += one_trk.finish_alerts(j)
            _eq(per, want, (phase, c))
            pos[c] += rows.shape[0]
    for c in cams:
        np.testing.assert_array_equal(run_trk.counts(c), one_trk.counts(c))
        assert run_trk.num_tracks(c) == one_trk.num_tracks(c)
    assert run_trk._cap["c0"] > 1 and run_trk._ecap["c0"] > 1          # both grew


def test_a_failing_frame_stops_its_camera_only():
    """A bad class id at frame 5 of camera "bad": frames 0..4 are returned, its tracker is as frame 4 left it, the other
    cameras complete their runs; one CCError names the camera and the frame."""
    rng = np.random.default_rng(3)
    trk = ocsort.DeviceTrackers(slots=4)
    ref = ocsort.DeviceTrackers(slots=4)
    for t in (trk, ref):
        for c in ("bad", "ok"):
            _setup(t, c, dict(max_age=30), None, False, [Alert.make(max=1)])
    sc = {c: [_scene(rng, t, 5) for t in range(12)] for c in ("bad", "ok")}
    sc["bad"][5][0, 5] = 3.5
    sc["bad"][5][0, 4] = 0.9
    jobs = [(c, torch.from_numpy(np.stack(sc[c])).cuda(), 0.5) for c in ("bad", "ok")]
    ev = [[(960, 540, 10.0 + f) for f in range(12)]] * 2
    al = [[(0.0, 0)] * 12] * 2
    r = trk.launch_runs(jobs, ev, al)
    torch.cuda.synchronize()
    with pytest.raises(CCError, match="'bad' frame 5: a detection's class id") as e:
        trk.finish_runs(r)
    res = e.value.results
    assert len(res[0]) == 5 and len(res[1]) == 12
    want = _runs(ref, "bad", sc["bad"][:5], 0.5, (960, 540), [10.0 + f for f in range(5)], [(0.0, 0)] * 5, 5)
    _eq(res[0], want, "bad")
    assert trk.num_tracks("bad") == ref.num_tracks("bad")


def test_overflow_and_argument_errors_of_the_c_abi():
    """cc_ocsort_gpu_update_runs: an output capacity too small for frame 3's targets stops the run there with OVERFLOW
    (done 3); bad arguments fail before the launch; the events, alerts and describe run calls check theirs."""
    trk = ocsort.DeviceTrackers(slots=4)
    _setup(trk, "a", dict(max_age=30, min_hits=0), None, False, [Alert.make(max=1)])
    rng = np.random.default_rng(1)
    T, n = 6, 8
    rows = torch.from_numpy(np.stack([_scene(rng, t, n) for t in range(T)])).cuda()
    rows[3, :, 4] = 0.95                                      # every row of frame 3 above the threshold
    dev = dict(device="cuda")
    out = torch.zeros((1, T, 4, 9), dtype=torch.float64, **dev)
    cnt, live = torch.zeros((1, T), dtype=torch.int32, **dev), torch.zeros((1, T), dtype=torch.int32, **dev)
    ids = torch.zeros((1, T, 64), dtype=torch.int32, **dev)
    ds = torch.zeros(2, dtype=torch.int32, **dev)
    h, st = trk._h, trk._stream()
    slot = trk._slot["a"]

    def call(runs, B=1, fm=T, cap=4, id_cap=64, o=out):
        return lib().cc_ocsort_gpu_update_runs(h, runs, B, fm, o.data_ptr() if o is not None else None, cap, cnt.data_ptr(), ids.data_ptr(),
                                              id_cap, live.data_ptr(), ds[0:1].data_ptr(), ds[1:2].data_ptr(), st)
    ok = (cc_track_run * 1)(cc_track_run(rows.data_ptr(), n, T, slot, 0.5))
    # the first frames fill up to 4 targets at most only when fewer rows pass; use min_hits 0 so every match is output
    assert call(ok) == 0
    torch.cuda.synchronize()
    d, s = ds.tolist()
    assert s == CC_TRACK_OVERFLOW and d <= 3 and int(cnt[0, d]) > 4
    bad = [(cc_track_run * 1)(cc_track_run(rows.data_ptr(), n, 0, slot, 0.5)),           # no frames
           (cc_track_run * 1)(cc_track_run(rows.data_ptr(), n, T + 1, slot, 0.5)),       # more than frames_max
           (cc_track_run * 1)(cc_track_run(None, n, T, slot, 0.5)),                      # NULL rows
           (cc_track_run * 1)(cc_track_run(rows.data_ptr(), 2000, T, slot, 0.5)),        # too many rows
           (cc_track_run * 1)(cc_track_run(rows.data_ptr(), n, T, 3, 0.5)),              # unconfigured slot
           (cc_track_run * 2)(cc_track_run(rows.data_ptr(), n, T, slot, 0.5), cc_track_run(rows.data_ptr(), n, T, slot, 0.5))]
    for i, r in enumerate(bad):
        assert call(r, B=len(r)) != 0, i
    assert call(ok, fm=CC_MAX_FRAMES + 1) != 0
    assert call(ok, id_cap=trk._cap["a"] - 1) != 0
    assert call(ok, o=None) != 0
    # events / alerts / describe runs: a clock that is not finite, a frame size of 0, a weekday of 7, a repeated slot
    wh = np.array([960, 540] * T, np.int32)
    now = np.arange(T, dtype=np.float64)
    preds = torch.zeros((1, T, 4, 7), dtype=torch.float64, **dev)
    flags = torch.zeros((1, T, 4), dtype=torch.uint8, **dev)
    saves = torch.zeros((1, T, 4, 6), dtype=torch.int64, **dev)
    ec = torch.zeros((2, 1, T), dtype=torch.int32, **dev)
    eds = torch.zeros(2, dtype=torch.int32, **dev)

    def ev(runs, wh=wh, now=now, B=1):
        return lib().cc_ocsort_gpu_events_runs(h, runs, B, T, wh.ctypes.data, now.ctypes.data, out.data_ptr(), 4, cnt.data_ptr(),
                                              ids.data_ptr(), 64, live.data_ptr(), ds[0:1].data_ptr(), preds.data_ptr(), flags.data_ptr(),
                                              saves.data_ptr(), 4, ec.data_ptr(), eds[0:1].data_ptr(), eds[1:2].data_ptr(), st)
    assert ev(ok) == 0
    nan = now.copy()
    nan[2] = np.nan
    assert ev(ok, now=nan) != 0
    w0 = wh.copy()
    w0[4] = 0
    assert ev(ok, wh=w0) != 0
    assert ev(bad[-1], B=2) != 0
    loc = np.zeros(2 * T)
    fired = torch.zeros((1, T, 64), dtype=torch.int32, **dev)
    nf = torch.zeros((1, T), dtype=torch.int32, **dev)

    def alr(runs, loc=loc, now=now, B=1):
        return lib().cc_ocsort_gpu_alerts_runs(h, runs, B, T, now.ctypes.data, loc.ctypes.data, preds.data_ptr(), flags.data_ptr(), 4,
                                              ec.data_ptr(), eds[0:1].data_ptr(), fired.data_ptr(), nf.data_ptr(), ds[0:1].data_ptr(),
                                              ds[1:2].data_ptr(), st)
    assert alr(ok) == 0
    l7 = loc.copy()
    l7[3] = 7
    assert alr(ok, loc=l7) != 0
    assert alr(ok, now=nan) != 0
    assert alr(bad[-1], B=2) != 0
    torch.cuda.synchronize()
    emb = torch.zeros((2, 8), **dev)
    hit, sim = torch.zeros(2, dtype=torch.int32, **dev), torch.zeros((2, 64), **dev)
    slots, frames, rws = np.array([slot], np.int32), np.array([2], np.int32), np.array([1, 1], np.int32)
    tt, ll = np.array([0.0, 1.0]), np.zeros(4)

    def ds_(frames=frames, tt=tt):
        return lib().cc_ocsort_gpu_describe_runs(h, slots.ctypes.data, frames.ctypes.data, 1, rws.ctypes.data, tt.ctypes.data, ll.ctypes.data,
                                                emb.data_ptr(), 8, hit.data_ptr(), sim.data_ptr(), st)
    assert ds_() == 0
    assert ds_(frames=np.array([0], np.int32)) != 0
    assert ds_(tt=np.array([0.0, np.inf])) != 0
    torch.cuda.synchronize()


def test_description_alerts_across_the_frames_of_a_run():
    """Hits in consecutive frames: describe_runs applies the 60 s cooldown and last_det frame by frame, exactly as
    per-frame describe calls at each frame's clock."""
    rng = np.random.default_rng(11)
    D = 16
    desc = rng.normal(size=(3, D)).astype(np.float32)
    al = [Alert.make(desc="a", threshold=-0.5), Alert.make(max=1), Alert.make(desc="b", threshold=0.0, sched=[[0, 40000]] + [True] * 7)]
    a = ocsort.DeviceTrackers(slots=4)
    b = ocsort.DeviceTrackers(slots=4)
    for t in (a, b):
        t.add("c")
        t.alerts("c", al, desc)
    T = 40
    rows = [int(r) for r in rng.integers(0, 4, T)]
    clocks = [1000.0 + 7.0 * f for f in range(T)]
    local = [(39000.0 + 30 * f, 2) for f in range(T)]
    emb = torch.from_numpy(rng.normal(size=(sum(rows), D)).astype(np.float32)).cuda()
    [(hit, sim)] = a.describe_runs([("c", rows)], emb, [clocks], [local])
    r0, hits = 0, 0
    for f in range(T):
        if rows[f]:
            [(h1, s1)] = b.describe([("c", rows[f])], emb[r0:r0 + rows[f]].contiguous(), [clocks[f]], [local[f]])
            np.testing.assert_array_equal(hit[r0:r0 + rows[f]], h1)
            np.testing.assert_array_equal(sim[r0:r0 + rows[f]], s1)
            hits += int((h1 >= 0).sum())
        r0 += rows[f]
    assert hits >= 2


def _finder():
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    return of


def _yuv(f):
    H, W = f.shape[:2]
    return torch.cat([f[..., 1].reshape(-1), f[::2, ::2, 0].reshape(-1), f[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)


def test_video_reader_step_video_save_objects_describe_saves_equal_step_alerts():
    """VideoReader -> step_video -> save_objects -> describe_saves for a bgr24 video next to a mixed fleet (a yuv420p video
    of another resolution, a second bgr24 video of the first one's shape): the detector rows equal detect_batch /
    detect_frames of the same frames, and every frame's preds, flags, saves, fired ids, thumbnail files, embeddings and
    description hits equal what step_alerts + save_objects + describe_saves give frame by frame on a second CameraBatch."""
    sys.path.insert(0, str(ROOT))
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.ingest import VideoReader
    xc = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    m = YOLOv9("c", 320, weights=o.synthetic_weights("c", seed=5, calib=xc))
    of = _finder()
    vids = {"v360": ((360, 640), "bgr24"), "y720": ((720, 1280), "yuv420p"), "w360": ((360, 640), "bgr24")}
    N = 13
    data = {}
    for i, (n, ((H, W), fmt)) in enumerate(vids.items()):
        base = o.synthetic_frames(1, H, W, seed=60 + i)[0]
        fr = [base.roll(shifts=(4 * t, 6 * t), dims=(0, 1)) for t in range(N)]
        data[n] = b"".join((_yuv(f) if fmt == "yuv420p" else f).numpy().tobytes() for f in fr)
    T0 = 1.7e9
    al = {"default": Alert.make(max=1, classes=[0, 1, 2, 3, 5, 7]), "any": Alert.make(max=2, window=3, zone=False),
          "thing": Alert.make(desc="a thing", threshold=-1.0)}
    video, single = CameraBatch(m), CameraBatch(m)
    for cb in (video, single):
        for n, ((H, W), fmt) in vids.items():
            cb.add_camera(n, thresh=0.05, pix_fmt=fmt)
            cb.set_zone(n, [[0.0, 0.0], [0.7, 0.0], [0.7, 1.0], [0.0, 1.0]], False, True)
            cb.set_alerts(n, al, of)
    readers = {n: VideoReader(io.BytesIO(data[n]), H, W, fmt, run=4, every=2) for n, ((H, W), fmt) in vids.items()}
    seen = hits = saves = 0
    while True:
        got = {n: next(r, None) for n, r in readers.items()}
        got = {n: g for n, g in got.items() if g is not None}
        if not got:
            break
        clocks = {n: [T0 + 1.5 * pos for pos in p] for n, (_, p) in got.items()}     # 3 s between kept frames: saves
        res = video.step_video({n: f for n, (f, _) in got.items()}, clocks)
        saved = video.save_objects(res, of)
        desc = video.describe_saves(saved, now=clocks)
        for n, (frames, pos) in got.items():
            ws, wf, we, wh = [], [], [], []
            for f in range(len(frames)):
                one = single.step_alerts({n: frames[f]}, now=clocks[n][f])[n]
                r = res[n][f]
                np.testing.assert_array_equal(r.rows, one.rows)
                for u, v in zip(r[1:4], one[1:4]):
                    np.testing.assert_array_equal(u, v)
                assert r.fired == one.fired
                sv = single.save_objects({n: one}, of)
                ws.append(np.asarray(sv[n][0]).reshape(-1, 6))
                wf += sv[n][1]
                if sv[n][2] is not None:
                    we.append(sv[n][2].tensor.cpu())
                wh += [(s + sum(len(x) for x in ws[:-1]), a, v) for s, a, v in single.describe_saves(sv, now=clocks[n][f])[n]]
            s7, files, emb = saved[n]
            np.testing.assert_array_equal(s7[:, 1:], np.concatenate(ws))
            assert files == wf
            if we:
                assert torch.equal(emb.tensor.cpu(), torch.cat(we))
            assert desc[n] == wh, n
            saves += len(files)
            hits += len(wh)
        seen += 4
    assert saves > 0 and hits > 0
    for n in vids:
        np.testing.assert_array_equal(video.object_counts(n), single.object_counts(n))
    assert video._dev_trk is not None and all(video._dev_trk.has_alerts(n) for n in vids)


def _bad_box_scene(kind, F=24, k=9):
    """Frames of 4 objects; at frame k (and k+1 for "huge") rows that make the tracker output a target box the events
    reject: a NaN coordinate on a row that joins an existing track's greedy assignment, or a box beyond 2**60."""
    rng = np.random.default_rng(5)
    frames = [_scene(rng, t, 4) for t in range(F)]
    for f in range(F):
        frames[f][:, 4] = 0.9
    if kind == "nan":
        a = frames[k][1].copy()
        two = a.copy()
        two[:4] += 3.0                                         # a second row on the same track: the greedy assignment
        nan = a.copy()
        nan[2] = np.nan
        frames[k] = np.concatenate([nan[None], frames[k], two[None]]).astype(np.float32)
    else:
        for f in (k, k + 1):
            huge = np.array([[900.0, 600.0, 1e20, 700.0, 0.95, 2.0]], np.float32)
            frames[f] = np.concatenate([frames[f], huge]).astype(np.float32)
    n = max(len(r) for r in frames)
    return [np.concatenate([r, np.zeros((n - len(r), 6), np.float32)]) for r in frames]


@pytest.mark.parametrize("kind", ["nan", "huge"])
def test_a_rejected_box_stops_the_run_where_a_single_step_stops(kind):
    """A target box the events reject at frame e: the run returns frames before e, raises for e, and its tracker has
    applied exactly frame e, so a run resumed at e + 1 equals single-frame launches that went on after the same error.
    A NaN coordinate in a detection row: runs equal single-frame launches frame by frame."""
    frames = _bad_box_scene(kind)
    al = [Alert.make(max=1), Alert.make(max=2, window=3, zone=False)]
    kw = dict(max_age=30, min_hits=1)
    one, run = ocsort.DeviceTrackers(slots=4), ocsort.DeviceTrackers(slots=4)
    for t in (one, run):
        _setup(t, "c", kw, None, False, al)
    ev = [(960, 540, 50.0 + 0.5 * f) for f in range(len(frames))]
    loc = [(36000.0, 3)] * len(frames)
    want, errors = [], []
    for f, r in enumerate(frames):
        j = one.launch([("c", torch.from_numpy(r).cuda(), 0.5)], events=[ev[f]], alerts=[loc[f]])
        torch.cuda.synchronize()
        try:
            want += one.finish_alerts(j)
        except CCError as e:
            assert "not finite" in str(e)
            want.append(None)
            errors.append(f)
    # a box beyond 2**60 reaches the events as a confirmed target; a NaN detection row is gated out by the tracker's IoU
    # tests in this scene (it starts a track that is never confirmed), so there both paths must simply agree
    assert errors or kind == "nan", "the scene must make the events reject a box"
    pos, got = 0, []
    while pos < len(frames):
        r = torch.from_numpy(np.stack(frames[pos:])).cuda()
        j = run.launch_runs([("c", r, 0.5)], [ev[pos:]], [loc[pos:]])
        torch.cuda.synchronize()
        try:
            [per] = run.finish_runs(j)
            got += per
            pos = len(frames)
        except CCError as e:
            e_frame = pos + len(e.results[0])
            assert f"frame {e_frame}: a target's box is not finite" in str(e)
            got += e.results[0] + [None]
            pos = e_frame + 1
    assert [i for i, g in enumerate(got) if g is None] == errors
    _eq([g for g in got if g is not None], [w for w in want if w is not None], kind)
    np.testing.assert_array_equal(run.counts("c"), one.counts("c"))
    assert run.num_tracks("c") == one.num_tracks("c")


@pytest.mark.parametrize("i", range(18))
def test_tracker_runs_equal_single_steps_on_the_pinned_sequences(i):
    """The 18 pinned tracker sequences (mot16, synth a/b/c, street a/b, random scenes; varied min_hits, delta_t, inertia,
    use_byte) through tracker-only runs of 1, 7 and 128 frames: every frame's targets equal DeviceTrackers.update's."""
    sys.path.insert(0, str(ROOT / "oracle"))
    sys.path.insert(0, str(Path(__file__).parent))
    from test_ocsort_gpu import SEQS, _as_rows
    name, frames, thr, kw, _ = SEQS[i]
    frames = np.ascontiguousarray(np.asarray(frames, np.float32)[:256])
    one = ocsort.DeviceTrackers(slots=8)
    one.add("s", **kw)
    d = torch.from_numpy(frames).cuda()
    want = [_as_rows(one.update([("s", d[f], thr)])[0]) for f in range(len(frames))]
    for T in (1, 7, 128):
        trk = ocsort.DeviceTrackers(slots=4, capacity=2)
        trk.add("r", **kw)
        got = []
        for f0 in range(0, len(frames), T):
            j = trk.launch_runs([("r", d[f0:f0 + T].contiguous(), thr)])
            torch.cuda.synchronize()
            got += trk.finish_runs(j)[0]
        assert len(got) == len(want)
        for f, (g, w) in enumerate(zip(got, want)):
            np.testing.assert_array_equal(_as_rows(g), w, err_msg=f"{name} T={T} frame {f}")
        assert trk.num_tracks("r") == one.num_tracks("s")
