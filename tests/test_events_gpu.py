"""Object events on the GPU (csrc/events_gpu.cu through `DeviceTrackers.launch(..., events=)` / `finish_events`, and
`CameraBatch.step_events`) array-equal to the reference fixture (tests/golden/events_ref.npz) and to the host form
`ObjectEvents` on the host tracker's targets: golden and random sequences with seeded zones, 128 cameras in one launch,
track ids far beyond the event storage, growth, a tracker that needs room, a non-finite box, sentinels and every
argument error."""
import ctypes
import io
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from clearcam_b200._lib import cc_track_job, check, lib
from clearcam_b200.events import ObjectEvents
from clearcam_b200.ocsort_tracker import ocsort

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden"
sys.path.insert(0, str(Path(__file__).parent.parent / "oracle"))


def _fixture():
    g = np.load(GOLD / "events_ref.npz")
    return {k: g[k] for k in g.files}, json.loads(str(g["configs"]))


FIX, CFGS = _fixture()


def _sequence(name):
    from make_golden_events import sequences
    if name == "edge":
        return FIX["edge_frames"], 0.5, dict(max_age=30)
    return sequences()[name]


def _eq(got, exp, msg):
    for a, b, what in zip(got, exp, ("preds", "flags", "saves")):
        np.testing.assert_array_equal(a, b, err_msg=f"{msg}: {what}")
        assert a.dtype == b.dtype, f"{msg}: {what} dtype"


def _replay(frames, thr, kw, ev_args, W, H, times, f0=0, f1=None, capacity=64, event_capacity=64, expect=None):
    """Device tracker + events against host OCSort + ObjectEvents on one camera; frames before f0 are tracked only."""
    f1 = len(frames) if f1 is None else f1
    dev = ocsort.DeviceTrackers(slots=4, capacity=capacity, event_capacity=event_capacity)
    dev.add("c", **kw)
    dev.events("c", *ev_args)
    host, ev = ocsort.OCSort(**kw), ObjectEvents(*ev_args)
    rows = torch.from_numpy(np.ascontiguousarray(frames[:f1])).cuda()
    n_out = 0
    for f in range(f1):
        tg = host.update(frames[f], thr)
        if f < f0:
            dev.update([("c", rows[f], thr)])
            continue
        now = float(times[f - f0])
        L = dev.launch([("c", rows[f], thr)], events=[(W, H, now)])
        torch.cuda.current_stream().synchronize()
        [got] = dev.finish_events(L)
        exp = ev.update(tg, W, H, now)
        _eq(got, exp, f"frame {f}")
        if expect is not None:
            _eq(got, expect[f - f0], f"frame {f} against the reference")
        n_out += len(got[0]) + len(got[2])
    return dev, n_out


def _expected(k, frames, thr, kw):
    from make_golden_events import expected, tracker_rows
    exp, times = expected(FIX, CFGS, k, tracker_rows(frames[:CFGS[k]["f1"]], thr, kw))
    return [e[:3] for e in exp], times


@pytest.mark.parametrize("k", range(len(CFGS)))
def test_golden_configuration(k):
    c = CFGS[k]
    frames, thr, kw = _sequence(c["seq"])
    exp, times = _expected(k, frames, thr, kw)
    _replay(frames, thr, kw, (c["zone"], c["outside"], c["non_zone_alert"], c["classes"]), c["W"], c["H"], times,
            c["f0"], c["f1"], expect=exp)


def _random_zone(g, n):
    a = np.sort(g.uniform(0, 2 * np.pi, n))
    r = g.uniform(0.05, 0.6, n)
    z = np.stack([0.5 + r * np.cos(a), 0.5 + r * np.sin(a)], 1)
    if g.random() < 0.3:
        g.shuffle(z)                                     # self-intersecting
    return z.tolist()


def _random_cases():
    from make_golden_ocsort import RANDOM_SEEDS, random_scene_args
    out = []
    for seed in RANDOM_SEEDS:
        kw, thr, frames = random_scene_args(seed)
        g = np.random.default_rng(seed)
        n = 256 if seed == RANDOM_SEEDS[0] else int(g.integers(3, 40))
        out.append((f"random_{seed}", np.asarray(frames, np.float32), thr, kw, _random_zone(g, n), bool(g.integers(0, 2)),
                    bool(g.integers(0, 2)), None if g.random() < 0.5 else [0, 1, 2, 3]))
    for sc in "abc":
        frames, thr, kw = _sequence(f"synth_{sc}")
        g = np.random.default_rng(ord(sc))
        out.append((f"synth_{sc}", frames, thr, kw, _random_zone(g, 12), sc == "b", sc != "a", None))
    return out


RANDOM = _random_cases()


@pytest.mark.parametrize("case", RANDOM, ids=[c[0] for c in RANDOM])
def test_random_sequence_and_zone(case):
    name, frames, thr, kw, zone, outside, nza, classes = case
    times = 1.7e9 + np.arange(len(frames)) * 0.35
    _, n = _replay(frames, thr, kw, (zone, outside, nza, classes), 1280, 720, times)
    assert n > 0


def test_track_ids_far_beyond_the_event_capacity():
    """The street scene reaches ids above 280 while the event storage, starting with room for 64 entries, never holds
    more than the live tracks (at most 114 here): entries of dead tracks are dropped."""
    frames, thr, kw = _sequence("street")
    times = 1.7e9 + np.arange(1500) * 0.1
    dev, _ = _replay(frames, thr, kw, (None, False, False, None), 960, 540, times, event_capacity=64)
    assert dev._ecap["c"] <= 128 and frames is not None


def test_growth_from_a_tiny_capacity_equals_never_growing():
    frames, thr, kw = _sequence("street")
    times = 1.7e9 + np.arange(300) * 0.1
    z = [[0.1, 0.1], [0.9, 0.2], [0.8, 0.9], [0.1, 0.8]]
    small, _ = _replay(frames, thr, kw, (z, False, True, None), 960, 540, times, f1=300, capacity=8, event_capacity=1)
    big, _ = _replay(frames, thr, kw, (z, False, True, None), 960, 540, times, f1=300, capacity=4096, event_capacity=4096)
    assert small._ecap["c"] > 1 and small._cap["c"] > 8       # both the tracker and the events grew, results equal


def _camera_case(b):
    name, frames, thr, kw, zone, outside, nza, classes = RANDOM[b % len(RANDOM)]
    g = np.random.default_rng(1000 + b)
    W, H = [(1280, 720), (1920, 1080), (640, 360)][b % 3]
    zone = None if b % 5 == 0 else _random_zone(g, int(g.integers(3, 20)))
    fps = [10.0, 30.0, 2.0][b % 3]
    return frames, thr, kw, (zone, bool(b % 2), bool(b % 3 == 1), None if b % 4 else [0, 1, 2]), W, H, 1.7e9 + b + np.arange(100) / fps


def test_128_cameras_in_one_launch():
    B, F = 128, 90
    dev = ocsort.DeviceTrackers(slots=256, capacity=16, event_capacity=4)
    cams = [_camera_case(b) for b in range(B)]
    host, evs = {}, {}
    for b, (frames, thr, kw, ea, W, H, times) in enumerate(cams):
        dev.add(b, **kw)
        dev.events(b, *ea)
        host[b], evs[b] = ocsort.OCSort(**kw), ObjectEvents(*ea)
    rows = [torch.from_numpy(np.ascontiguousarray(c[0][:F])).cuda() for c in cams]
    n_out = 0
    for f in range(F):
        if f == 30:
            dev.reset(5)
            host[5], evs[5] = ocsort.OCSort(**cams[5][2]), ObjectEvents(*cams[5][3])
        if f == 40:
            dev.remove(9)
            del host[9], evs[9]
        if f == 50:
            dev.add(9, **cams[9][2])
            dev.events(9, *cams[9][3])
            host[9], evs[9] = ocsort.OCSort(**cams[9][2]), ObjectEvents(*cams[9][3])
        jobs, ev = [], []
        for b, (frames, thr, kw, ea, W, H, times) in enumerate(cams):
            if b not in host or (b % 7 == 3 and f % 4 == 1):
                continue
            jobs.append((b, rows[b][f], thr))
            ev.append((W, H, times[f]))
        L = dev.launch(jobs, events=ev)
        torch.cuda.current_stream().synchronize()
        got = dev.finish_events(L)
        for (b, _, thr), (W, H, now), g in zip(jobs, ev, got):
            exp = evs[b].update(host[b].update(cams[b][0][f], thr), W, H, now)
            _eq(g, exp, f"camera {b} frame {f}")
            n_out += len(g[0]) + len(g[2])
    assert n_out > 0


# ------------------------------------------------------------------------------------------------ raw C-ABI
def _raw(dev, cams, rows, thr, wh, now, doctor=None, cap=1024):
    """Tracker then events through the C-ABI with sentinel-filled outputs -> host arrays."""
    B = len(cams)
    table = (cc_track_job * B)(*[cc_track_job(r.data_ptr(), r.shape[0], dev._slot[c], thr, 0) for c, r in zip(cams, rows)])
    out = torch.full((B, cap, 9), -7.0, dtype=torch.float64, device="cuda")
    cs = torch.full((2, B), -9, dtype=torch.int32, device="cuda")
    check(lib().cc_ocsort_gpu_update(dev._h, table, B, out.data_ptr(), cap, cs[0].data_ptr(), cs[1].data_ptr(), None), "update")
    if doctor is not None:
        doctor(out)
    preds = torch.full((B, cap, 7), -5.0, dtype=torch.float64, device="cuda")
    flags = torch.full((B, cap), 0xAB, dtype=torch.uint8, device="cuda")
    saves = torch.full((B, cap, 6), -3, dtype=torch.int64, device="cuda")
    ecs = torch.full((2, B), -9, dtype=torch.int32, device="cuda")
    est = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    w = np.array(wh, np.int32).reshape(-1)
    t = np.array(now, np.float64)
    check(lib().cc_ocsort_gpu_events(dev._h, table, B, w.ctypes.data, t.ctypes.data, out.data_ptr(), cap, cs[0].data_ptr(),
                                     cs[1].data_ptr(), preds.data_ptr(), flags.data_ptr(), saves.data_ptr(), cap, ecs.data_ptr(),
                                     est.data_ptr(), None), "events")
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (out, cs, preds, flags, saves, ecs, est)]


def test_non_finite_box_and_sentinels():
    """A doctored NaN box fails its own camera only (state unchanged: its next frames still equal the host), nothing is
    written past any camera's rows, and the others' events are intact."""
    frames, thr, kw = _sequence("synth_a")
    cams = ["a", "b", "c"]
    dev = ocsort.DeviceTrackers(slots=4)
    host, evs = {}, {}
    for c in cams:
        dev.add(c, **kw)
        dev.events(c, [[0.1, 0.1], [0.9, 0.1], [0.9, 0.9], [0.1, 0.9]], c == "b", True, None)
        host[c], evs[c] = ocsort.OCSort(**kw), ObjectEvents([[0.1, 0.1], [0.9, 0.1], [0.9, 0.9], [0.1, 0.9]], c == "b", True)
    rows = torch.from_numpy(frames).cuda()
    wh, n_rows = [(1280, 720)] * 3, 0
    for f in range(60):
        now = [1.7e9 + 0.5 * f] * 3

        def doctor(out):
            out[1, 0, 2] = float("nan")
        bad = f == 40
        out, cs, preds, flags, saves, ecs, est = _raw(dev, cams, [rows[f]] * 3, thr, wh, now, doctor if bad else None)
        for b, c in enumerate(cams):
            tg = host[c].update(frames[f], thr)
            if bad and b == 1:
                assert est[b] == 2 and ecs[0, b] == 0 and ecs[1, b] == 0              # CC_EVENT_BAD_BOX
                assert (preds[b] == -5.0).all() and (flags[b] == 0xAB).all() and (saves[b] == -3).all()
                continue
            p, fl, s = evs[c].update(tg, 1280, 720, now[b])
            assert est[b] == 0
            n, m = ecs[0, b], ecs[1, b]
            np.testing.assert_array_equal(preds[b, :n], p)
            np.testing.assert_array_equal(flags[b, :n], fl)
            np.testing.assert_array_equal(saves[b, :m], s)
            assert (preds[b, n:] == -5.0).all() and (flags[b, n:] == 0xAB).all() and (saves[b, m:] == -3).all()
            n_rows += n + m
    assert n_rows > 0


def test_tracker_not_ok_is_not_run():
    frames, thr, kw = _sequence("synth_a")
    dev = ocsort.DeviceTrackers(slots=4, capacity=1)
    dev.add("a", **kw)
    dev.events("a")
    rows = torch.from_numpy(frames).cuda()
    out, cs, preds, flags, saves, ecs, est = _raw(dev, ["a"], [rows[0]], thr, [(640, 480)], [0.0])
    assert cs[1, 0] == 1 and est[0] == 3                                  # tracker NEEDS_ROOM -> events NOT_RUN


def test_argument_errors():
    L = lib()
    dev = ocsort.DeviceTrackers(slots=4)
    dev.add("t", max_age=30)
    h, slot = dev._h, dev._slot["t"]
    free = next(s for s in range(4) if s != slot)
    z = np.array([[0.1, 0.1], [0.9, 0.1], [0.5, 0.9]], np.float64)
    cfg = L.cc_ocsort_gpu_events_configure
    assert cfg(h, free, z.ctypes.data, 3, 0, 0, None, 16, None) != 0 and b"not configured" in L.cc_last_error()
    assert cfg(h, 9, z.ctypes.data, 3, 0, 0, None, 16, None) != 0 and b"slot 9" in L.cc_last_error()
    big = np.zeros((257, 2))
    assert cfg(h, slot, big.ctypes.data, 257, 0, 0, None, 16, None) != 0 and b"257 zone vertices" in L.cc_last_error()
    nan = np.array([[0, 0], [np.inf, 1], [1, 1]], np.float64)
    assert cfg(h, slot, nan.ctypes.data, 3, 0, 0, None, 16, None) != 0 and b"not finite" in L.cc_last_error()
    assert cfg(h, slot, None, 3, 0, 0, None, 16, None) != 0 and b"NULL zone" in L.cc_last_error()
    assert cfg(h, slot, z.ctypes.data, 3, 0, 0, None, 0, None) != 0 and b"capacity 0" in L.cc_last_error()
    assert L.cc_ocsort_gpu_events_grow(h, slot, 64, None) != 0 and b"not configured for events" in L.cc_last_error()
    ok = np.full((256, 2), 0.5)
    assert cfg(h, slot, ok.ctypes.data, 256, 0, 0, None, 16, None) == 0                  # the vertex limit itself is fine
    J = cc_track_job
    p = ctypes.c_void_p(16)
    wh = (ctypes.c_int * 4)(640, 480, 640, 480)
    now = (ctypes.c_double * 2)(0.0, 0.0)
    evt = L.cc_ocsort_gpu_events

    def call(jobs=None, B=1, wh=wh, now=now, cap=8, **nul):
        jobs = jobs if jobs is not None else (J * 1)(J(None, 0, slot, 0.5, 0))
        a = dict(h=h, out=p, cnt=p, st=p, preds=p, flags=p, saves=p, counts=p, status=p)
        a.update(nul)
        return evt(a["h"], jobs, B, wh, now, a["out"], 8, a["cnt"], a["st"], a["preds"], a["flags"], a["saves"], cap, a["counts"],
                   a["status"], None)
    assert call((J * 1)(J(None, 0, free, 0.5, 0))) != 0 and b"not configured" in L.cc_last_error()
    assert call((J * 2)(J(None, 0, slot, 0.5, 0), J(None, 0, slot, 0.5, 0)), B=2) != 0 and b"twice" in L.cc_last_error()
    assert call(B=0) != 0 and b"B 0" in L.cc_last_error()
    assert call(B=129) != 0 and b"B 129" in L.cc_last_error()
    assert call(cap=4) != 0 and b"output capacity" in L.cc_last_error()
    assert call(wh=(ctypes.c_int * 2)(0, 480)) != 0 and b"frame 0 x 480" in L.cc_last_error()
    assert call(now=(ctypes.c_double * 1)(float("nan"))) != 0 and b"clock" in L.cc_last_error()
    for k in ("h", "out", "cnt", "st", "preds", "flags", "saves", "counts", "status"):
        assert call(**{k: None}) != 0 and b"NULL" in L.cc_last_error()
    with pytest.raises(KeyError):
        dev.launch([("t", torch.zeros((0, 6), device="cuda"), 0.5)], events=[(640, 480, 0.0)])   # no events() for t
    with pytest.raises(TypeError):
        dev.events("t", z.tolist(), outside=None)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ CameraBatch
FLEET = {"b180": ((180, 320), "bgr24"), "y180": ((180, 320), "yuv420p"), "b360": ((360, 640), "bgr24"),
         "y360": ((360, 640), "yuv420p"), "b720": ((720, 1280), "bgr24"), "y720": ((720, 1280), "yuv420p")}
ZONES = {"b180": None, "y180": ([[0.0, 0.0], [1.0, 0.0], [1.0, 0.6], [0.0, 0.6]], False, False),
         "b360": ([[0.2, 0.2], [0.8, 0.1], [0.7, 0.9]], True, True), "y360": ([[0.1, 0.1], [0.9, 0.9], [0.9, 0.1], [0.1, 0.9]], False, True),
         "b720": ([[0.0, 0.5], [1.0, 0.5], [1.0, 1.0], [0.0, 1.0]], True, False), "y720": None}


def test_camera_batch_step_events_mailboxes_mixed_fleet():
    """step_events_mailboxes over three resolutions in bgr24 and yuv420p (one merged detector call), 20 steps: each
    camera's preds, flags and saves equal a solo host tracker plus ObjectEvents on the same rows with the picture's W x H;
    frames move every step so targets gain speed; one reset and one remove / re-add."""
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.ingest import FrameMailbox
    x = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    m = YOLOv9("t", 320, weights=o.synthetic_weights("t", seed=5, calib=x))
    cb = CameraBatch(m, max_age=100)
    boxes = {n: FrameMailbox(H, W, pix_fmt=fmt) for n, ((H, W), fmt) in FLEET.items()}
    solo, evs = {}, {}

    def fresh(n):
        solo[n] = ocsort.OCSort(max_age=100)
        evs[n] = ObjectEvents(*(ZONES[n] or (None, False, False)))
    for n in FLEET:
        fresh(n)
    n_rows = 0
    for t in range(20):
        if t == 6:
            cb.reset_tracker("b360")
            fresh("b360")
        if t == 8:
            cb.remove_camera("y720")
            del boxes["y720"], solo["y720"]
        if t == 11:
            boxes["y720"] = FrameMailbox(720, 1280, pix_fmt="yuv420p")
            fresh("y720")
        for i, n in enumerate(boxes):
            (H, W), fmt = FLEET[n]
            f = o.synthetic_frames(1, H, W, seed=40 + i)[0].roll(shifts=(3 * t, 5 * t), dims=(0, 1))
            if fmt == "yuv420p":
                f = torch.cat([f[..., 1].reshape(-1), f[::2, ::2, 0].reshape(-1), f[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)
            assert boxes[n].fill(io.BytesIO(f.numpy().tobytes()))
        if t == 0:
            for n in FLEET:
                cb.add_camera(n, pix_fmt=FLEET[n][1])
                if ZONES[n]:
                    cb.set_zone(n, *ZONES[n])
        if t == 11 and ZONES["y720"]:
            cb.set_zone("y720", *ZONES["y720"])
        now = 1.7e9 + 0.6 * t
        res = cb.step_events_mailboxes(boxes, now=now)
        assert set(res) == set(boxes) and cb._dev_trk is not None
        for n, r in res.items():
            (H, W), _ = FLEET[n]
            exp = evs[n].update(solo[n].update(r.rows, 0.5), W, H, now)
            _eq((r.preds, r.flags, r.saves), exp, f"step {t} camera {n}")
            n_rows += len(r.preds) + len(r.saves)
    assert n_rows > 0
