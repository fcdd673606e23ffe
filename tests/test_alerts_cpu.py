"""The host form of the alerts (clearcam_b200/alerts.py) against the reference's answers in tests/golden/alerts_ref.npz
(oracle/make_golden_alerts.py): adds, fired alerts, description hits and the object counter at every step of every
configuration; the similarity's fixed order; bugs that the fixture must catch; settings and argument errors; and
CameraBatch.step_alerts / describe_saves on host rows."""
import inspect
import json
import types
from pathlib import Path

import numpy as np
import pytest

from clearcam_b200 import alerts as alerts_mod
from clearcam_b200.alerts import Alert, CameraAlerts, active, similarity

GOLDEN = Path(__file__).parent / "golden" / "alerts_ref.npz"


def _fixture():
    g = np.load(GOLDEN)
    return g, json.loads(str(g["configs"]))


def _alert(a, mod=alerts_mod):
    return mod.Alert.make(classes=a.get("classes"), max=a.get("max"), window=a.get("window"), sched=a.get("sched"),
                      is_on=a.get("is_on", True), is_notif=a.get("is_notif", True), zone=a.get("zone", True), desc=a.get("desc"),
                      threshold=a.get("threshold", 0.28), last_det=a.get("last_det", 0.0))


def replay(g, cfg, k, mod=alerts_mod):
    """Configuration k through mod.CameraAlerts -> (adds, fired, hits, counts) in the fixture's layout."""
    p = f"c{k}_"
    settings = [dict(a) for a in cfg["alerts"]]
    desc = g[p + "desc"].astype(np.float32) / 1024
    al = mod.CameraAlerts([_alert(a, mod) for a in settings], desc)
    al.adds = []
    toggles = {}
    for t in cfg["toggles"]:
        toggles.setdefault(t[0], []).append(t[1:])
    adds, fired, hits = [], [], []
    r0, e0 = 0, 0
    times, tod, wday, ran, n_rows = g[p + "times"], g[p + "tod"], g[p + "wday"], g[p + "ran"], g[p + "n_rows"]
    cls, flags, n_saves, emb = g[p + "cls"], g[p + "flags"], g[p + "n_saves"], g[p + "emb"].astype(np.float32) / 1024
    for i in range(len(times)):
        for t in toggles.get(i, []):
            if t[0] == "alerts_on":
                al.alerts_on = bool(t[1])
            else:                                     # alert t[1] replaced by one with is_on t[2] at last_det t[3]
                settings[t[1]]["is_on"] = bool(t[2])
                new = [_alert(a, mod) for a in settings]
                new[t[1]] = new[t[1]]._replace(last_det=float(t[3]))
                al.replace(new, desc, [j if j != t[1] else -1 for j in range(len(new))])
        n = int(n_rows[i]) if ran[i] else 0
        preds = np.zeros((n, 7))
        preds[:, 5] = cls[r0:r0 + n]
        del al.adds[:]
        f = al.step(preds, flags[r0:r0 + n], float(times[i]), (int(tod[i]), int(wday[i])))
        r0 += n
        adds += [(i, a, c) for a, c in al.adds]
        fired += [(i, j) for j in f]
        m = int(n_saves[i])
        hits += [(i, s, a) for s, a, _ in al.describe(emb[e0:e0 + m], float(times[i]), (int(tod[i]), int(wday[i])))]
        e0 += m
    assert r0 == len(cls) and e0 == len(emb)
    return (np.array(adds, np.int32).reshape(-1, 3), np.array(fired, np.int32).reshape(-1, 2), np.array(hits, np.int32).reshape(-1, 3),
            al.counter)


def test_host_form_equals_the_reference_at_every_step():
    g, cfgs = _fixture()
    total = np.zeros(4, int)
    for k, cfg in enumerate(cfgs):
        adds, fired, hits, counts = replay(g, cfg, k)
        np.testing.assert_array_equal(adds, g[f"c{k}_adds"], err_msg=f"configuration {k}: adds")
        np.testing.assert_array_equal(fired, g[f"c{k}_fired"], err_msg=f"configuration {k}: fired")
        np.testing.assert_array_equal(hits, g[f"c{k}_hits"], err_msg=f"configuration {k}: description hits")
        np.testing.assert_array_equal(counts, g[f"c{k}_counts"], err_msg=f"configuration {k}: object counter")
        total += [len(adds), len(fired), len(hits), (~g[f"c{k}_ran"]).sum()]
    assert (total > 0).all(), total                  # adds, firings, description hits and gated steps all occur


MUTANTS = {
    "window prune >= for >": ("now - q[0] > w", "now - q[0] >= w"),
    "no break after a description hit": ("hits.append((s, i, float(sims[s, i])))\n                    break",
                                         "hits.append((s, i, float(sims[s, i])))"),
    "inactive alerts keep counting": ("c.q = {}", "pass"),
    "last_det not set on firing": ("self.last_det[i] = now\n                    fired.append(i)", "fired.append(i)"),
    "warm-up off by one": ("if self.warm > WARMUP:", "if self.warm >= WARMUP:"),
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_plausible_bugs_change_an_answer(name):
    old, new = MUTANTS[name]
    src = inspect.getsource(alerts_mod)
    assert old in src
    mod = types.ModuleType("alerts_mutant")
    exec(compile(src.replace(old, new), "alerts_mutant", "exec"), mod.__dict__)
    g, cfgs = _fixture()
    for k, cfg in enumerate(cfgs):
        cfg = json.loads(json.dumps(cfg))
        adds, fired, hits, counts = replay(g, cfg, k, mod)
        if not (np.array_equal(adds, g[f"c{k}_adds"]) and np.array_equal(fired, g[f"c{k}_fired"])
                and np.array_equal(hits, g[f"c{k}_hits"])):
            return
    pytest.fail(f"the fixture does not catch: {name}")


def _lane_order(q, e):
    lanes = [0.0] * 32
    for k in range(len(e)):
        lanes[k % 32] += float(q[k]) * float(e[k])
    for o in (16, 8, 4, 2, 1):
        lanes = [lanes[l] + lanes[l ^ o] for l in range(32)]
    return np.float32(lanes[0])


@pytest.mark.parametrize("D", [512, 768, 45])
def test_similarity_is_the_stated_order(D):
    rng = np.random.default_rng(D)
    q = rng.normal(0, 1, (3, D)).astype(np.float32)
    e = rng.normal(0, 1, (5, D)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    e /= np.linalg.norm(e, axis=1, keepdims=True)
    s = similarity(q, e)
    assert s.dtype == np.float32 and s.shape == (5, 3)
    for n in range(5):
        for a in range(3):
            assert s[n, a].tobytes() == _lane_order(q[a], e[n]).tobytes()
    # unit vectors: float32 BLAS agrees within one ulp of float32 at the scale of the products' sum (|sim| <= 1)
    blas = e @ q.T
    assert (np.abs(s.astype(np.float64) - blas) <= np.spacing(np.float32(1))).all()
    exact = e.astype(np.float64) @ q.T.astype(np.float64)
    assert (np.abs(s - exact) <= np.spacing(np.abs(s)) / 2 + 1e-15).all()     # and rounds the fp64 sum


def test_alert_from_counter_and_activity():
    rc = types.SimpleNamespace(classes={0, 2, "7"}, max=3, window=None, sched=[[100, 200]] + [True] * 5 + [False],
                               is_on=True, is_notif=False, zone=False, desc=None, threshold=0.3, last_det=5.0)
    a = Alert.from_counter(rc)
    assert a.classes == frozenset({0, 2}) and a.max == 3 and a.span == 1.0 and not a.zone
    assert a.sched == ((100.0, 200.0), (True, True, True, True, True, False, False))
    assert a.is_active(True, (150, 0)) and a.is_active(True, (100, 0)) and not a.is_active(True, (99, 0))
    assert not a.is_active(True, (200, 0)) and not a.is_active(True, (150, 5)) and not a.is_active(True, (150, 6))
    assert not a.is_active(False, (150, 0))
    del rc.is_on                                      # is_active: getattr(self, "is_on", False)
    assert not Alert.from_counter(rc).is_on
    b = Alert.make(window=0, is_notif=True, sched=[])
    assert b.span == 60.0 and b.sched is None and b.is_active(True, (0, 6))
    al = [a, b, Alert.make(is_on=False)]
    for local in [(150, 0), (99, 0), (150, 6)]:
        assert active(al, local).tolist() == [x.is_active(True, local) for x in al]
    assert not active(al, (150, 0), alerts_on=False).any()


def test_argument_errors():
    with pytest.raises(ValueError):
        Alert.make(max=1025)
    with pytest.raises(ValueError):
        Alert.make(max=-1)
    with pytest.raises(ValueError):
        Alert.make(window=-3)
    with pytest.raises(ValueError):
        Alert.make(threshold=float("nan"))
    with pytest.raises(ValueError):
        Alert.make(sched=[[0, float("inf")], True])
    with pytest.raises(ValueError):
        CameraAlerts([Alert.make(max=1)] * 65)
    with pytest.raises(ValueError):
        CameraAlerts([Alert.make(desc="x")])                         # no embeddings
    with pytest.raises(TypeError):
        CameraAlerts([{"max": 1}])
    al = CameraAlerts([Alert.make(max=1)])
    with pytest.raises(ValueError):
        al.replace([Alert.make(max=2)], keep=[0])                     # settings differ
    with pytest.raises(ValueError):
        al.replace([Alert.make(max=1)], keep=[3])
    with pytest.raises(ValueError):
        similarity(np.zeros((2, 4), np.float32), np.zeros((1, 5), np.float32))


def test_replace_keeps_unchanged_alerts():
    a, b = Alert.make(max=2, zone=False, window=100), Alert.make(max=2, zone=False, window=50)
    al = CameraAlerts([a, b])
    preds = np.zeros((1, 7))
    for t in range(12):
        al.step(preds, np.array([1], np.uint8), 1000.0 + t, (0, 0))
    assert [sum(len(q) for q in c.q.values()) for c in al.counts] == [2, 2]
    al.replace([b._replace(window=60.0), a], keep=[-1, 0])
    assert [sum(len(q) for q in c.q.values()) for c in al.counts] == [0, 2]
    assert al.last_det[1] > 0 and al.last_det[0] == 0.0


# ------------------------------------------------------------------------------------------------ CameraBatch, host rows
class _HostModel:
    """A stand-in detector with host rows: boxes that move with the frame's first pixel, new ones every few frames."""
    def detect_batch(self, frames):
        out = np.zeros((frames.shape[0], 300, 6), np.float32)
        for b in range(frames.shape[0]):
            s = float(frames[b, 0, 0, 0])
            for i in range(5):
                x, y = 20 + 90 * i + 9 * s, 15 + 40 * i + 4 * s
                out[b, i] = [x, y, x + 120 + 10 * i, y + 150, 0.9 - 0.05 * i, i % 3]
        import torch
        return torch.from_numpy(out)


class _Finder:
    def __init__(self):
        self.calls = []

    def encode_text_batch(self, texts):
        self.calls.append(list(texts))
        return np.stack([np.random.default_rng(len(t)).normal(0, 1, 16).astype(np.float32) for t in texts])


def test_camera_batch_step_alerts_host_rows():
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.events import ObjectEvents
    from clearcam_b200.ocsort_tracker import ocsort
    cb = CameraBatch(_HostModel(), max_age=100)
    finder = _Finder()
    settings = {"a": {"d": Alert.make(max=1, classes=[0, 1, 2, 3, 5, 7]), "z": Alert.make(max=2, window=3, zone=False),
                      "t": Alert.make(desc="a person", threshold=-10.0)},
                "b": {"d": Alert.make(max=3, window=2, is_notif=False), "t2": Alert.make(desc="a car", threshold=0.1, zone=False)}}
    solo, evs, host = {}, {}, {}
    for n in settings:
        cb.add_camera(n)
        cb.set_alerts(n, settings[n], finder)
        solo[n] = ocsort.OCSort(max_age=100)
        nza = any(not a.zone for a in settings[n].values())
        evs[n] = ObjectEvents(None, False, nza)
        desc = np.stack([_Finder().encode_text_batch([a.desc])[0] if a.desc else np.zeros(16, np.float32) for a in settings[n].values()])
        host[n] = CameraAlerts(list(settings[n].values()), desc)
    assert finder.calls == [["a person"], ["a car"]]                  # each new description once
    assert cb.cams["a"].zone[2] and cb.cams["b"].zone[2]
    assert cb.alerting(local=(0, 0)) == ["a", "b"]
    fired_any = 0
    for t in range(60):
        now, local = 1000.0 + 0.7 * t, (3600 + t, 2)
        frames = {n: np.full((360, 640, 3), t % 25, np.uint8) for n in settings}
        res = cb.step_alerts(frames, now=now, local=local)
        for n, r in res.items():
            tg = solo[n].update(r.rows, 0.5)
            p, f, s = evs[n].update(tg, 640, 360, now)
            np.testing.assert_array_equal(r.preds, p)
            np.testing.assert_array_equal(r.flags, f)
            ids = list(settings[n])
            assert r.fired == [ids[i] for i in host[n].step(p, f, now, local)], (t, n)
            fired_any += len(r.fired)
            emb = np.random.default_rng(t).normal(0, 1, (len(s), 16)).astype(np.float32)
            got = cb.describe_saves({n: (s, [], emb)}, now=now, local=local)[n]
            want = [(si, ids[a], v) for si, a, v in host[n].describe(emb, now, local)]
            assert got == want
    assert fired_any > 0
    np.testing.assert_array_equal(cb.object_counts("a"), host["a"].counter)
    assert cb.object_counts("a").sum() > 0
    cb.reset_object_counts("a")
    assert cb.object_counts("a").sum() == 0
    cb.set_alerts_on("b", False)
    assert cb.alerting(local=(0, 0)) == ["a"]
    # unchanged alerts keep their state, a changed one starts afresh; no new description is encoded
    before = [sum(len(q) for q in c.q.values()) for c in cb.cams["a"].alerts.counts]
    changed = dict(settings["a"], z=settings["a"]["z"]._replace(window=4.0))
    cb.set_alerts("a", changed, finder)
    after = [sum(len(q) for q in c.q.values()) for c in cb.cams["a"].alerts.counts]
    assert after[0] == before[0] and after[1] == 0 and len(finder.calls) == 2
    with pytest.raises(ValueError):
        cb.set_alerts("a", {"q": Alert.make(desc="a new text")})     # needs a finder
