"""Golden vectors for the alerts: the adds of `run_inference` (clearcam.py:612-620), the object counter, the firing loop
of `process_frame` (:465-499), its gate (:447) and warm-up, and the description alerts of `clip_latest_img` (:1289-1307).

TEST INFRASTRUCTURE, not product code.  `clearcam.py` needs tinygrad, so it is not imported: the source of
`RollingClassCounter`, `VideoCapture.run_inference`, `VideoCapture.save_object`, `VideoCapture.process_frame`,
`clip_latest_img` and `point_not_in_polygon` is taken from /root/reference/clearcam.py with `ast` (only possible in the
build container) and executed in a namespace of stubs:

  time.time() / localtime()   a frozen clock and local time per step (the reference reads them many times)
  self.tracker[cam].update    the repository's host OCSort on the step's detector rows, stepped only when run_inference
                              runs (the gate skips it, as in the reference)
  cv2, draw_predictions, write_png, send_notif, export_and_upload, threading, database, pickle, open
                              record nothing or return what the code needs; the 5-second live and counter checks never
                              come due
  alerts_on[cam]              set per step from the configuration's toggles
  jit_infer / run_encode_text seeded embeddings: int8 values / 1024, so every product and sum is exact
  sched                       a list whose missing weekday entries read as False: a missing entry counts as inactive (the
                              reference raises IndexError there; alerts.py documents the choice)

Per configuration the file stores the step clock and local time, which steps ran the detector, each ran step's preds
classes and flags, the adds, the fired alerts, the description hits, the object counter at the end, and the embeddings.

    python oracle/make_golden_alerts.py      -> tests/golden/alerts_ref.npz
"""
import ast
import json
from collections import defaultdict, deque
import sys
import types
from pathlib import Path, PurePosixPath

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from oracle.make_golden_events import OUT, REF, T0, clock, sequences   # noqa: E402

D = 64                                         # embedding width of the fixture's descriptions and objects (the kernels take any)


def reference_code():
    tree = ast.parse((REF / "clearcam.py").read_text())
    body = []
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in ("point_not_in_polygon", "clip_latest_img"):
            body.append(node)
        if isinstance(node, ast.ClassDef) and node.name == "RollingClassCounter":
            body.append(node)
        if isinstance(node, ast.ClassDef) and node.name == "VideoCapture":
            body += [f for f in node.body if isinstance(f, ast.FunctionDef) and f.name in ("run_inference", "save_object", "process_frame")]
    assert len(body) == 6, len(body)
    return compile(ast.Module(body=body, type_ignores=[]), str(REF / "clearcam.py"), "exec")


class _Path(str):
    def __truediv__(self, o):
        return _Path(f"{self}/{o}")

    def mkdir(self, **kw):
        pass

    def exists(self):
        return False


class Sched(list):
    """A reference `sched` whose missing weekday entries read as False."""

    def __getitem__(self, i):
        return super().__getitem__(i) if i < len(self) else False


def local_of(now, tod0, wday0):
    secs = tod0 + np.floor(now - T0).astype(np.int64)
    return (secs % 86400).astype(np.int32), ((wday0 + secs // 86400) % 7).astype(np.int32)


def emb_int8(g, base=None, mix=0.0):
    v = g.normal(0, 40, D)
    if base is not None:
        v = (1 - mix) * v + mix * base
    return np.clip(np.round(v), -127, 127).astype(np.int8)


class _Thread:
    def __init__(self, *a, **k):
        pass

    def start(self):
        pass


class _File:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def run_config(code, seq, cfg, k):
    frames, thr, kw = seq
    from clearcam_b200.ocsort_tracker import ocsort
    trk = ocsort.OCSort(**kw)
    n = cfg["f1"] - cfg["f0"]
    times = clock(cfg["clock"], n)
    tods, wdays = local_of(times, cfg["tod0"], cfg["wday0"])
    state = {"now": 0.0, "lt": None}
    ns = {"np": np, "defaultdict": defaultdict, "deque": deque, "model": None, "yolo_jit_cache": None, "jit_cache": None, "classes": None,
          "time": types.SimpleNamespace(time=lambda: state["now"], localtime=lambda *a: state["lt"], sleep=lambda s: None),
          "cv2": types.SimpleNamespace(imwrite=lambda *a, **kw: True, CAP_PROP_POS_FRAMES=1, IMWRITE_JPEG_QUALITY=1),
          "datetime": types.SimpleNamespace(now=lambda: types.SimpleNamespace(strftime=lambda fmt: "2026-01-01")),
          "BASE_DIR": _Path("base"), "object_queue": [], "Tensor": None, "print": lambda *a, **kw: None,
          "draw_predictions": lambda *a: np.zeros((1, 1, 3), np.uint8), "write_png": lambda *a: None, "color_dict": {},
          "send_notif": lambda *a, **kw: None, "export_and_upload": lambda *a, **kw: None, "event_img_info": lambda s: {"ts": 0},
          "threading": types.SimpleNamespace(Thread=_Thread), "pickle": types.SimpleNamespace(dump=lambda *a: None, load=None),
          "open": lambda *a, **kw: _File(), "os": types.SimpleNamespace(path=types.SimpleNamespace(exists=lambda p: False)),
          "alerts_on": {}}
    exec(code, ns)
    RC = ns["RollingClassCounter"]
    cam = "cam"
    g = np.random.default_rng(1000 + k)
    desc_q = {}
    for a in cfg["alerts"]:
        if a.get("desc") is not None and a["desc"] not in desc_q:
            desc_q[a["desc"]] = emb_int8(g)

    def make(i, a, last_det):
        rc = RC(window_seconds=a.get("window"), max=a.get("max"), classes=None if a.get("classes") is None else set(a["classes"]),
                sched=None if a.get("sched") is None else Sched(a["sched"]), cam_name=cam, desc=a.get("desc"),
                threshold=a.get("threshold", 0.28))
        rc.is_on, rc.is_notif, rc.zone, rc.last_det = a.get("is_on", True), a.get("is_notif", True), a.get("zone", True), last_det
        return rc

    alerts = {str(i): make(i, a, a.get("last_det", 0.0)) for i, a in enumerate(cfg["alerts"])}
    adds_now = []

    def wrap(i, rc):
        orig = rc.add

        def add(c):
            orig(c)
            if (rc.classes is None or c in rc.classes) and rc.max and rc.desc is None:     # the alerts that keep counts
                adds_now.append((i, int(c)))
        rc.add = add
        return rc

    for i, (key, rc) in enumerate(alerts.items()):
        wrap(i, rc)
    current = {"frame": None, "emb": None}
    saves_now = []
    self = types.SimpleNamespace()
    self.vod, self.frame_num, self.last_frame_num = {cam: False}, {cam: 0}, {cam: -1}
    self.raw_frame = {cam: np.zeros((1, 1, 3), np.uint8)}
    self.tracker = {cam: types.SimpleNamespace(update=lambda preds, thresh: trk.update(current["frame"], thr))}
    self.settings = {cam: None if cfg["zone"] is None else {"coords": cfg["zone"], "outside": cfg["outside"], "threshold": thr}}
    self.alert_counters = {cam: alerts}
    self.counter = {cam: RC(cam_name=cam, window_seconds=float("inf"))}
    self.object_set, self.object_set_zone, self.pred_occs = {cam: set()}, {cam: set()}, {cam: {}}
    self.last_frames, self.last_preds, self.count = {cam: []}, {cam: []}, {cam: 0}
    self.cap, self.src_fps, self.start_time = {cam: None}, {cam: 30}, {cam: 0.0}
    self.last_det, self.last_preview_time, self.filename = {cam: -1}, {cam: 0.0}, {cam: None}
    self.last_live_check, self.last_counter_update = {cam: float("inf")}, {cam: float("inf")}
    self.live_link = {}

    class _Prev(dict):
        def __getitem__(self, key):
            return state["now"] - 1.0
    self.prev_time = _Prev()

    def _open_ffmpeg(name):
        raise AssertionError("process_frame raised")
    self._open_ffmpeg = _open_ffmpeg
    from clearcam_b200.models.objects import ObjectFinder

    def save_object(p, ts=0, cam_name=None):          # only the crops save_object writes reach clip_latest_img
        t = p.tlwh
        if ObjectFinder.crop_rect((t[0], t[1], t[0] + t[2], t[1] + t[3]), cfg["W"], cfg["H"]) is not None:
            saves_now.append(int(p.track_id))
    self.save_object = save_object
    self.run_inference = lambda frame, cam_name: ns["run_inference"](self, frame, cam_name)
    db = types.SimpleNamespace(run_get=lambda table, name: alerts, run_put=lambda *a, **kw: None)
    ns["database"] = db
    ns["global_settings"] = types.SimpleNamespace(userID="user", use_qwen=False, use_clip=True, key=None)
    W, H = cfg["W"], cfg["H"]
    frame_obj = types.SimpleNamespace(shape=(H, W, 3), numpy=lambda: np.zeros((1, 1, 3), np.uint8))
    frame_obj.unsqueeze = lambda d: frame_obj
    ns["Tensor"] = lambda f: frame_obj
    ns["jit_infer"] = lambda fn, x, cache: types.SimpleNamespace(numpy=lambda: current["emb"])
    ns["run_encode_text"] = lambda clip, text: (desc_q[text].astype(np.float32) / 1024)[None]
    ns["object_finder"] = types.SimpleNamespace(preprocess=lambda img: img, model=types.SimpleNamespace(precompute_embedding=None))
    toggles = {}
    for t in cfg.get("toggles", []):
        toggles.setdefault(t[0], []).append(t[1:])
    out = {"ran": [], "n_rows": [], "cls": [], "flags": [], "adds": [], "fired": [], "hits": [], "n_saves": [], "emb": []}
    desc_keys = [a.get("desc") for a in cfg["alerts"]]
    ns["alerts_on"][cam] = True
    for i, f in enumerate(range(cfg["f0"], cfg["f1"])):
        now = float(times[i])
        state["now"] = now
        state["lt"] = types.SimpleNamespace(tm_hour=int(tods[i]) // 3600, tm_min=int(tods[i]) % 3600 // 60, tm_sec=int(tods[i]) % 60,
                                            tm_wday=int(wdays[i]))
        for t in toggles.get(i, []):
            if t[0] == "alerts_on":
                ns["alerts_on"][cam] = bool(t[1])
            else:                                          # ("is_on", alert, value, last_det): the alert is replaced
                j, v, ld = t[1], t[2], t[3]
                cfg["alerts"][j]["is_on"] = bool(v)
                key = str(j)
                alerts[key] = wrap(j, make(j, cfg["alerts"][j], ld))
        current["frame"] = frames[f]
        self.frame_num[cam] = i
        self.last_frame_num[cam] = i - 1
        del adds_now[:], saves_now[:]
        before = {key: rc.last_det for key, rc in alerts.items()}
        self.last_preds[cam] = None
        seen0, zone0 = set(self.object_set[cam]), set(self.object_set_zone[cam])
        ns["process_frame"](self, cam)
        ran = self.last_frame_num[cam] == i
        preds = np.asarray(self.last_preds[cam], np.float64).reshape(-1, 7) if ran else np.zeros((0, 7))
        out["ran"].append(ran)
        out["flags"] += [int(int(r[6]) in self.object_set[cam] - seen0) | int(int(r[6]) in self.object_set_zone[cam] - zone0) << 1
                         for r in preds]
        out["n_rows"].append(len(preds))
        out["cls"] += [int(r[5]) for r in preds]
        out["adds"] += [(i, a, c) for a, c in adds_now]
        fired = [j for j, (key, rc) in enumerate(alerts.items()) if rc.last_det != before[key]]
        out["fired"] += [(i, j) for j in fired]
        # the saves of this step, each embedded and matched in queue order
        out["n_saves"].append(len(saves_now))
        for s_idx in range(len(saves_now)):
            descs = [d for d in desc_keys if d is not None]
            base = desc_q[descs[g.integers(len(descs))]] if descs and g.random() < 0.5 else None
            q = emb_int8(g, base, float(g.uniform(0.3, 0.9)))
            out["emb"].append(q)
            current["emb"] = (q.astype(np.float32) / 1024)[None]
            before = {key: rc.last_det for key, rc in alerts.items()}
            ns["object_queue"][:] = [PurePosixPath(f"base/cameras/{cam}/objects/2026-01-01/{s_idx}_{saves_now[s_idx]}.jpg")]
            ns["clip_latest_img"](np.zeros((1, 1, 3), np.uint8))
            hit = [j for j, (key, rc) in enumerate(alerts.items()) if rc.last_det != before[key]]
            assert len(hit) <= 1
            out["hits"] += [(i, s_idx, j) for j in hit]
    counts = np.zeros(80, np.int64)
    for c, q in self.counter[cam].data.items():
        counts[int(c)] = len(q)
    return {"times": times, "tod": tods, "wday": wdays, "ran": np.array(out["ran"], bool),
            "n_rows": np.array(out["n_rows"], np.int32), "cls": np.array(out["cls"], np.uint8), "flags": np.array(out["flags"], np.uint8),
            "adds": np.array(out["adds"], np.int32).reshape(-1, 3), "fired": np.array(out["fired"], np.int32).reshape(-1, 2),
            "hits": np.array(out["hits"], np.int32).reshape(-1, 3), "n_saves": np.array(out["n_saves"], np.int32),
            "emb": np.array(out["emb"], np.int8).reshape(-1, D), "counts": counts,
            "desc": np.stack([desc_q[d] if d is not None else np.zeros(D, np.int8) for d in desc_keys])}


WEEK = [[0, 86400]] * 7                       # the UI's default: no entry for Sunday


def configs():
    default = dict(window=None, max=1, classes=[0, 1, 2, 3, 5, 7])                        # init_cam's alert
    cfgs = []

    def add(seq, f0, f1, W, H, zone, alerts, outside=False, clk="10fps", tod0=8 * 3600, wday0=0, toggles=()):
        cfgs.append(dict(seq=seq, f0=f0, f1=f1, W=W, H=H, zone=zone, outside=outside, clock=clk, tod0=tod0, wday0=wday0,
                         alerts=alerts, toggles=list(toggles)))

    hexagon = [[0.1, 0.1], [0.9, 0.15], [0.95, 0.5], [0.8, 0.9], [0.2, 0.8], [0.05, 0.5]]
    lshape = [[0.0, 0.25], [0.5, 0.25], [0.5, 0.5], [0.75, 0.5], [0.75, 1.0], [0.0, 1.0]]
    add("street", 0, 600, 960, 540, None,
        [dict(default), dict(max=3, window=5, classes=[0, 2], zone=False), dict(desc="a person", threshold=0.02, max=1)])
    add("street", 0, 900, 960, 540, hexagon,
        [dict(default), dict(max=3, window=30, zone=True), dict(max=1, zone=False, is_notif=False),
         dict(max=2, window=4, classes=[0], sched=[[8 * 3600 + 20, 8 * 3600 + 50]] + [True] * 7),
         dict(desc="a car", threshold=0.01), dict(desc="a person", threshold=-0.005, zone=False)], clk="gaps",
        toggles=[(300, "is_on", 1, False, 0.0), (420, "is_on", 1, True, T0 + 10.0), (500, "alerts_on", False), (560, "alerts_on", True)])
    add("street", 300, 900, 960, 540, lshape,
        [dict(max=1, window=2, classes=None, zone=False, sched=[[86400 - 40, 86400]] + WEEK[1:]),
         dict(max=3, window=60, classes=[0, 2], sched=[[0, 25]] + WEEK[1:]), dict(desc="a dog", threshold=0.015, sched=WEEK)],
        outside=True, clk="10fps", tod0=86400 - 30, wday0=5)
    add("synth_a", 0, 240, 1280, 720, [[0.2, 0.1], [0.9, 0.5], [0.3, 0.95]],
        [dict(max=1, classes=[1, 3, 5], zone=False), dict(max=3, classes=[1, 3, 5], window=1, is_notif=False),
         dict(desc="a red car", threshold=0.0, zone=False), dict(max=0, zone=False)], clk="30fps")
    add("synth_b", 0, 240, 1280, 720, lshape, [dict(default), dict(max=1, zone=False, window=3)], outside=True, clk="gaps",
        toggles=[(5, "alerts_on", False), (30, "alerts_on", True)])
    add("synth_c", 0, 240, 1920, 1080, None, [dict(max=3, window=10, zone=False), dict(desc="a truck", threshold=0.02)],
        clk="10fps", tod0=3600, wday0=6)
    return cfgs


def main():
    code = reference_code()
    seqs = sequences()
    cfgs = configs()
    out = {}
    for k, cfg in enumerate(cfgs):
        alerts0 = json.loads(json.dumps(cfg["alerts"]))
        r = run_config(code, seqs[cfg["seq"]], cfg, k)
        cfg["alerts"] = alerts0                           # the settings at the start; toggles say what changes
        for name, a in r.items():
            out[f"c{k}_{name}"] = a
        print(k, cfg["seq"], "steps", len(r["ran"]), "ran", int(r["ran"].sum()), "rows", len(r["cls"]), "adds", len(r["adds"]),
              "fired", len(r["fired"]), "saves", len(r["emb"]), "hits", len(r["hits"]), "counted", int(r["counts"].sum()))
    out["configs"] = np.array(json.dumps(cfgs))
    np.savez_compressed(OUT / "alerts_ref.npz", **out)
    print("wrote", OUT / "alerts_ref.npz", (OUT / "alerts_ref.npz").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
