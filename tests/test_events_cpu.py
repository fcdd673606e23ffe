"""Object events (clearcam_b200/events.py `ObjectEvents`) against the reference's own run_inference / save_object /
point_not_in_polygon, run on the host tracker's rows (tests/golden/events_ref.npz, oracle/make_golden_events.py); plus
plausible bugs that the fixture must catch, the C-ABI's argument errors and `CameraBatch.step_events` on host rows."""
import ctypes
import json
import sys
from functools import lru_cache
from pathlib import Path

import numpy as np
import pytest

from clearcam_b200 import events as ev_mod
from clearcam_b200.events import ObjectEvents
from clearcam_b200.ocsort_tracker.STrack import STrack

GOLD = Path(__file__).parent / "golden"
sys.path.insert(0, str(Path(__file__).parent.parent / "oracle"))


@lru_cache(None)
def fixture():
    g = np.load(GOLD / "events_ref.npz")
    return {k: g[k] for k in g.files}, json.loads(str(g["configs"]))


@lru_cache(None)
def tracker_rows(seq):
    from make_golden_events import sequences, tracker_rows as rows
    frames, thr, kw = sequences()[seq] if seq != "edge" else (fixture()[0]["edge_frames"], 0.5, dict(max_age=30))
    return tuple(rows(frames, thr, kw))


def targets(rows):
    return [STrack(tlwh=r[:4], score=r[4], class_id=r[5], track_id=r[6], age=r[7], speed=r[8]) for r in rows]


def make_events(cfg):
    return ObjectEvents(cfg["zone"], cfg["outside"], cfg["non_zone_alert"], cfg["classes"])


@lru_cache(None)
def expected(k):
    """Config k's per-frame (preds, flags, saves, alert adds [(zone, class)]) and its clock."""
    from make_golden_events import expected as decode
    g, cfgs = fixture()
    return decode(g, cfgs, k, tracker_rows(cfgs[k]["seq"]))


def alert_adds(preds, flags, non_zone_alert):
    """The alert add() calls of clearcam.py:619-620 from the flags, in the reference's order (zone alert first)."""
    out = []
    for r, f in zip(preds, flags):
        out.append((1, int(r[5]))) if f & 2 else None
        if non_zone_alert and f & 1:
            out.append((0, int(r[5])))
    return out


def replay(k, make=make_events, pre=None, post=None):
    """ObjectEvents over config k -> [(preds, flags, saves)] per frame."""
    g, cfgs = fixture()
    cfg = cfgs[k]
    rows = tracker_rows(cfg["seq"])
    ev = make(cfg)
    times = expected(k)[1]
    res = []
    for i, f in enumerate(range(cfg["f0"], cfg["f1"])):
        assert len(rows[f]) == cfg["n_targets"][i]
        tg = targets(rows[f])
        if pre is not None:
            tg = pre(tg)
        res.append(ev.update(tg, cfg["W"], cfg["H"], float(times[i])))
        if post is not None:
            post(ev, tg)
    return res


def differs(k, **kw):
    exp = expected(k)
    for (p, f, s), (ep, ef, es, _) in zip(replay(k, **kw), exp[0]):
        if not (np.array_equal(p, ep) and np.array_equal(f, ef) and np.array_equal(s, es)):
            return True
    return False


N_CFG = len(fixture()[1])


def test_fixture_covers_the_branches():
    g, cfgs = fixture()
    zones = [c["zone"] for c in cfgs if c["zone"] is not None]
    assert any(c["zone"] is None for c in cfgs) and min(map(len, zones)) == 3 and max(map(len, zones)) == 64
    assert {c["outside"] for c in cfgs} == {True, False} and {c["non_zone_alert"] for c in cfgs} == {True, False}
    assert {c["classes"] is None for c in cfgs} == {True, False} and len({(c["W"], c["H"]) for c in cfgs}) >= 2
    assert {c["clock"] for c in cfgs} == {"10fps", "30fps", "gaps"}
    assert sum(len(g[f"c{k}_rejects"]) for k in range(N_CFG)) > 0
    flags = np.concatenate([g[f"c{k}_flags"] for k in range(N_CFG)])
    assert set(np.unique(flags).tolist()) == {0, 1, 2, 3}


@pytest.mark.parametrize("k", range(N_CFG))
def test_object_events_equal_the_reference(k):
    cfg = fixture()[1][k]
    for i, ((p, f, s), (ep, ef, es, adds)) in enumerate(zip(replay(k), expected(k)[0])):
        np.testing.assert_array_equal(p, ep, err_msg=f"config {k} frame {i}: preds")
        assert p.dtype == np.float64 and p.shape[1] == 7
        np.testing.assert_array_equal(f, ef, err_msg=f"config {k} frame {i}: flags")
        np.testing.assert_array_equal(s, es, err_msg=f"config {k} frame {i}: saves")
        assert alert_adds(p, f, cfg["non_zone_alert"]) == adds, f"config {k} frame {i}: alert adds"


# ------------------------------------------------------------------------------------------------ the fixture bites
def _poly_variant(which):
    """point_not_in_polygon with one `<=` turned into `<`."""
    def f(coords, poly):
        n = len(poly)
        for x, y in coords:
            inside = False
            p1x, p1y = poly[0]
            for i in range(1, n + 1):
                p2x, p2y = poly[i % n]
                if y > min(p1y, p2y):
                    if (y < max(p1y, p2y)) if which == "y" else (y <= max(p1y, p2y)):
                        if (x < max(p1x, p2x)) if which == "xmax" else (x <= max(p1x, p2x)):
                            xi = (y - p1y) * (p2x - p1x) / (p2y - p1y) + p1x if p1y != p2y else p1x
                            if p1x == p2x or ((x < xi) if which == "xi" else (x <= xi)):
                                inside = not inside
                p1x, p1y = p2x, p2y
            if inside:
                return False
        return True
    return f


def _any(**kw):
    return any(differs(k, **kw) for k in range(N_CFG))


@pytest.mark.parametrize("which", ["y", "xmax", "xi"])
def test_strict_polygon_comparisons_are_caught(monkeypatch, which):
    monkeypatch.setattr(ev_mod, "point_not_in_polygon", _poly_variant(which))
    assert _any()


def test_truncating_division_is_caught(monkeypatch):
    def rect(b, W, H, min_side=100):
        x1, y1, x2, y2 = (int(v) for v in b)
        cx, cy = int((x1 + x2) / 2), int((y1 + y2) / 2)
        hw, hh = int((x2 - x1) / 2) * 2, int((y2 - y1) / 2) * 2
        nx1, nx2, ny1, ny2 = max(0, min(cx - hw, W)), max(0, min(cx + hw, W)), max(0, min(cy - hh, H)), max(0, min(cy + hh, H))
        return None if (ny2 - ny1) < min_side or (nx2 - nx1) < min_side else (nx1, ny1, nx2, ny2)
    monkeypatch.setattr(ev_mod.ObjectFinder, "crop_rect", staticmethod(rect))
    assert _any()


def test_occurrence_cap_21_is_caught(monkeypatch):
    monkeypatch.setattr(ev_mod, "OCC_CAP", 21)
    assert _any()


def test_saves_after_the_speed_gate_are_caught():
    assert _any(pre=lambda tg: [t for t in tg if t.speed >= ev_mod.MIN_SPEED])


def test_pruning_by_absence_is_caught():
    def prune(ev, tg):
        ids = {t.track_id for t in tg}
        ev.occ = {k: v for k, v in ev.occ.items() if k in ids}
        ev.seen = {k for k in ev.seen if k in ids}
        ev.seen_zone = {k for k in ev.seen_zone if k in ids}
    assert _any(post=prune)


# ------------------------------------------------------------------------------------------------ edge cases
def test_empty_result_and_argument_checks():
    ev = ObjectEvents()
    p, f, s = ev.update([], 640, 480, 0.0)
    assert p.shape == (0, 7) and p.dtype == np.float64 and f.shape == (0,) and f.dtype == np.uint8 and s.shape == (0, 6)
    with pytest.raises(TypeError):
        ObjectEvents([[0, 0], [1, 0], [0, 1]], outside=None)
    with pytest.raises(ValueError):
        ObjectEvents([[0, 0], [1, np.nan], [0, 1]])
    with pytest.raises(ValueError):
        ObjectEvents(np.zeros((257, 2)))
    t = STrack(tlwh=[np.inf, 1, 2, 3], score=0.9, class_id=0, track_id=1, age=3, speed=5)
    with pytest.raises(ValueError, match="not finite"):
        ev.update([t], 640, 480, 0.0)
    t0 = STrack(tlwh=[np.nan, 1, 2, 3], score=0.9, class_id=0, track_id=1, age=0, speed=5)   # tracklet_len 0: never read
    assert ev.update([t0], 640, 480, 0.0)[0].shape == (0, 7)


# ------------------------------------------------------------------------------------------------ C-ABI argument errors
def test_c_abi_rejects_a_null_handle_before_anything():
    """Without a device no handle can be made; what can be checked here is that each entry point refuses a NULL handle
    with a message and no launch.  tests/test_events_gpu.py checks every other argument error on a real handle."""
    from clearcam_b200._lib import lib
    L = lib()
    z = np.array([[0.1, 0.1], [0.9, 0.1], [0.5, 0.9]], np.float64)
    assert L.cc_ocsort_gpu_events_configure(None, 0, z.ctypes.data, 3, 0, 0, None, 16, None) != 0
    assert b"cc_ocsort_gpu_events_configure: bad handle" in L.cc_last_error()
    assert L.cc_ocsort_gpu_events_grow(None, 0, 64, None) != 0
    assert b"cc_ocsort_gpu_events_grow: bad handle" in L.cc_last_error()
    p = ctypes.c_void_p(16)
    assert L.cc_ocsort_gpu_events(None, p, 1, p, p, p, 8, p, p, p, p, p, 8, p, p, None) != 0
    assert b"cc_ocsort_gpu_events: NULL argument" in L.cc_last_error()


# ------------------------------------------------------------------------------------------------ CameraBatch, host rows
class _HostModel:
    """A stand-in detector with host rows: a few boxes that move with the frame's first pixel."""
    def detect_batch(self, frames):
        out = np.zeros((frames.shape[0], 300, 6), np.float32)
        for b in range(frames.shape[0]):
            s = float(frames[b, 0, 0, 0])
            for i in range(5):
                x, y = 20 + 90 * i + 7 * s, 15 + 40 * i + 3 * s
                out[b, i] = [x, y, x + 120 + 10 * i, y + 150, 0.9 - 0.05 * i, i % 3]
        import torch
        return torch.from_numpy(out)


def test_camera_batch_step_events_host_rows_equal_object_events():
    import torch
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.ocsort_tracker import ocsort
    cb = CameraBatch(_HostModel(), max_age=100)
    cams = {"a": ((360, 640), None, False, False), "b": ((480, 640), [[0.1, 0.1], [0.7, 0.1], [0.7, 0.9], [0.1, 0.9]], True, True),
            "c": ((360, 640), [[0.0, 0.0], [0.5, 0.0], [0.5, 1.0]], False, False)}
    solo, evs = {}, {}
    for n, (shape, zone, outside, nza) in cams.items():
        cb.add_camera(n, classes=[0, 1] if n == "c" else None)
        cb.set_zone(n, zone, outside=outside, non_zone_alert=nza)
        solo[n] = ocsort.OCSort(max_age=100)
        evs[n] = ObjectEvents(zone, outside, nza, [0, 1] if n == "c" else None)
    seen = 0
    for t in range(40):
        frames = {n: np.full(shape + (3,), t % 30, np.uint8) for n, (shape, *_ ) in cams.items()}
        res = cb.step_events(frames, now=1000.0 + 0.4 * t)
        for n, r in res.items():
            tg = solo[n].update(r.rows, 0.5)
            p, f, s = evs[n].update(tg, cams[n][0][1], cams[n][0][0], 1000.0 + 0.4 * t)
            np.testing.assert_array_equal(r.preds, p, err_msg=f"step {t} camera {n}")
            np.testing.assert_array_equal(r.flags, f)
            np.testing.assert_array_equal(r.saves, s)
            seen += len(p) + len(s)
    assert seen > 0
