"""Golden vectors for the per-target object events of `run_inference` (clearcam.py:586-621): class filter, the
`pred_occs` clock and `save_object`'s rectangle, the motion gate, the zone test and the new / new-in-zone bookkeeping.

TEST INFRASTRUCTURE, not product code.  `clearcam.py` needs tinygrad, so it is not imported: the source of
`VideoCapture.run_inference`, `VideoCapture.save_object` and `point_not_in_polygon` is taken from
/root/reference/clearcam.py with `ast` (only possible in the build container) and executed in a namespace of stubs:

  time.time()                a frozen clock per frame (the reference reads it several times per target)
  self.tracker[cam].update   replays the host tracker's rows of that frame as STrack-like objects
  self.settings[cam]         None (no zone) or {"coords", "outside", "threshold"}
  self.alert_counters[cam]   a zone alert, plus an alert without a zone when non_zone_alert; get_counts() -> ({}, False),
                             add() is recorded
  self.counter, object_set*  sets and counters that record their adds in order
  cv2.imwrite                records the crop; the frame's pixels hold their own (x, y), so a crop gives its rectangle
  classes                    None or a list of class-id strings, as the reference's global

Nothing of the reference is stored: only arrays of inputs and the answers its code gave.  The tracker rows are the
repository's host tracker (`OCSort`, bit-equal to the device tracker) on the frames already pinned in
tests/golden/ocsort_street.npz (variant a, the product's settings) and ocsort_synth.npz, plus one small scene of this
file's own whose boxes leave the frame to the left and top (negative coordinates: floor division, not truncation).

Each preds row of the reference is one of the frame's targets, in target order, built as
[x1, y1, x2, y2, score, class, track_id] from its tracker row; this is checked bit for bit here.  So the file stores,
per configuration, which targets became preds rows (a bit mask over the frame's targets, `pred_mask`) and the SHA-256 of
the reference's float64 preds bytes (`pred_sha`); `expected` rebuilds the rows from the host tracker and checks that
digest, so the comparison stays exact in float64.  The clock of each configuration is `clock(kind, n)`.

    python oracle/make_golden_events.py      -> tests/golden/events_ref.npz
"""
import ast
import hashlib
import json
import sys
import types
from pathlib import Path

import numpy as np

REF = Path("/root/reference")
ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "tests" / "golden"

T0 = 1.76e9                                   # an epoch-sized clock: differences are taken as the reference takes them


def edge_scene(seed=21, n_frames=150, n_obj=6):
    """Large boxes drifting out of a 640 x 360 frame through its left and top sides, so save rectangles see negative
    corners and odd negative sums."""
    g = np.random.default_rng(seed)
    pos = np.stack([g.uniform(60, 400, n_obj), g.uniform(40, 250, n_obj)], 1)
    vel = np.stack([g.uniform(-5, -2, n_obj), g.uniform(-4, 1, n_obj)], 1)
    size = g.uniform(110, 260, (n_obj, 2))
    frames = np.zeros((n_frames, 16, 6), np.float32)
    for f in range(n_frames):
        pos += vel + g.normal(0, 0.4, vel.shape)
        rows = []
        for i in range(n_obj):
            c, wh = pos[i], size[i] * (1 + g.normal(0, 0.02, 2))
            rows.append([c[0] - wh[0] / 2, c[1] - wh[1] / 2, c[0] + wh[0] / 2, c[1] + wh[1] / 2, g.uniform(0.55, 0.95), i % 3])
        rows.sort(key=lambda r: -r[4])
        frames[f, :len(rows)] = rows
    return frames


def sequences():
    """name -> (frames [F,n,6] float32, det_thresh, OCSort kwargs)."""
    st = np.load(OUT / "ocsort_street.npz")
    a = st["a_args"]
    seqs = {"street": (st["frames"], float(a[0]), dict(max_age=int(a[1]), use_byte=bool(a[2])))}
    sy = np.load(OUT / "ocsort_synth.npz")
    for sc in "abc":
        a = sy[f"{sc}_args"]
        seqs[f"synth_{sc}"] = (sy[f"{sc}_frames"], float(a[0]), dict(max_age=int(a[1]), min_hits=int(a[2]), iou_threshold=float(a[3]),
                                                                    delta_t=int(a[4]), inertia=float(a[5]), use_byte=bool(a[6])))
    seqs["edge"] = (edge_scene(), 0.5, dict(max_age=30))
    return seqs


def tracker_rows(frames, thr, kw):
    """The host tracker's targets per frame: [(n,9) float64] (tlwh, score, class, id, tracklet_len, speed)."""
    sys.path.insert(0, str(ROOT))
    from clearcam_b200.ocsort_tracker import ocsort
    trk = ocsort.OCSort(**kw)
    out = []
    for f in frames:
        tg = trk.update(f, thr)
        out.append(np.array([[*t.tlwh, t.score, t.class_id, t.track_id, t.tracklet_len, t.speed] for t in tg],
                            np.float64).reshape(-1, 9))
    return out


def clock(kind, n):
    f = np.arange(n, dtype=np.float64)
    if kind == "10fps":
        return T0 + f * 0.1
    if kind == "30fps":
        return T0 + f / 30.0
    if kind == "gaps":                                  # 10 frames/s with a 12 s gap every 40 frames
        return T0 + f * 0.1 + 12.0 * (np.arange(n) // 40)
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------------ the reference's code
def reference_functions():
    tree = ast.parse((REF / "clearcam.py").read_text())
    body = []
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == "point_not_in_polygon":
            body.append(node)
        if isinstance(node, ast.ClassDef) and node.name == "VideoCapture":
            body += [f for f in node.body if isinstance(f, ast.FunctionDef) and f.name in ("run_inference", "save_object")]
    assert len(body) == 3
    return compile(ast.Module(body=body, type_ignores=[]), str(REF / "clearcam.py"), "exec")


class _Path(str):
    def __truediv__(self, o):
        return _Path(f"{self}/{o}")

    def mkdir(self, **kw):
        pass


class _Target:
    def __init__(self, r):
        self.tlwh = np.array(r[:4], np.float64)
        self.score, self.class_id, self.track_id, self.tracklet_len, self.speed = r[4], r[5], r[6], r[7], r[8]


class _RecSet(set):
    def __init__(self, log):
        super().__init__()
        self.log = log

    def add(self, v):
        self.log.append(v)
        super().add(v)


class _Alert:
    def __init__(self, zone, log):
        self.zone, self.log = zone, log

    def get_counts(self):
        return {}, False

    def add(self, cls):
        self.log.append((int(self.zone), int(cls)))


def run_config(code, rows, cfg):
    """One camera through the reference's run_inference over frames [f0, f1) of its tracker rows."""
    W, H = cfg["W"], cfg["H"]
    times = clock(cfg["clock"], cfg["f1"] - cfg["f0"])
    state = {"now": 0.0, "writes": []}
    ns = {"np": np, "model": None, "yolo_jit_cache": None,
          "classes": None if cfg["classes"] is None else [str(c) for c in cfg["classes"]],
          "time": types.SimpleNamespace(time=lambda: state["now"]),
          "cv2": types.SimpleNamespace(imwrite=lambda path, crop: state["writes"].append((path, crop)), CAP_PROP_POS_FRAMES=1),
          "datetime": types.SimpleNamespace(now=lambda: types.SimpleNamespace(strftime=lambda fmt: "2026-01-01")),
          "BASE_DIR": _Path("base"), "global_settings": types.SimpleNamespace(use_clip=False, use_face=False),
          "object_queue": [], "Tensor": lambda f: f,
          "jit_infer": lambda model, frame, cache: types.SimpleNamespace(numpy=lambda: None)}
    exec(code, ns)
    cam = "cam"
    adds, oset_log, zset_log, counter_log = [], [], [], []
    current = {"targets": []}
    xy = np.stack(np.meshgrid(np.arange(W, dtype=np.int32), np.arange(H, dtype=np.int32)), -1)    # pixel (y, x) = (x, y)
    self = types.SimpleNamespace()
    self.tracker = {cam: types.SimpleNamespace(update=lambda preds, thresh: current["targets"])}
    self.settings = {cam: None if cfg["zone"] is None else {"coords": cfg["zone"], "outside": cfg["outside"], "threshold": 0.5}}
    alerts = {"zone": _Alert(True, adds)}
    if cfg["non_zone_alert"]:
        alerts["all"] = _Alert(False, adds)
    self.alert_counters = {cam: alerts}
    self.counter = {cam: types.SimpleNamespace(add=lambda c: counter_log.append(c))}
    self.object_set, self.object_set_zone = {cam: _RecSet(oset_log)}, {cam: _RecSet(zset_log)}
    self.pred_occs = {cam: {}}
    self.cap, self.src_fps, self.vod, self.start_time = {cam: None}, {cam: 30}, {cam: False}, {cam: 0.0}
    self.last_frames = {cam: [xy]}
    rejects_now = []

    def save_object(p, ts=0, cam_name=None):
        n = len(state["writes"])
        ns["save_object"](self, p, ts, cam_name=cam_name)
        if len(state["writes"]) == n:
            rejects_now.append(int(p.track_id))
    self.save_object = save_object

    frame = types.SimpleNamespace(shape=(H, W, 3))
    out = {k: [] for k in ("preds", "mask", "flags", "adds", "saves", "save_off", "rejects")}
    out["save_off"].append(0)
    for i, f in enumerate(range(cfg["f0"], cfg["f1"])):
        state["now"], state["writes"] = float(times[i]), []
        del adds[:], oset_log[:], zset_log[:], counter_log[:], rejects_now[:]
        current["targets"] = [_Target(r) for r in rows[f]]
        preds, _ = ns["run_inference"](self, frame, cam)
        preds = np.asarray(preds, np.float64).reshape(-1, 7)
        for r in preds:
            tid = int(r[6])
            out["flags"].append((tid in oset_log) | ((tid in zset_log) << 1))
        assert counter_log == [int(r[5]) for r in preds if int(r[6]) in oset_log]
        # which targets the rows are: one per target at most, in target order, bit-equal to the row built from it
        cand = pred_rows(rows[f])
        ids = [int(r[6]) for r in rows[f]]
        idx = [ids.index(int(r[6])) for r in preds]
        assert idx == sorted(set(idx)) and cand[idx].tobytes() == preds.tobytes()
        mask = np.zeros(len(ids), bool)
        mask[idx] = True
        out["mask"].append(mask)
        out["preds"].append(preds)
        out["adds"] += [(i, z, c) for z, c in adds]
        for path, crop in state["writes"]:
            _, tid, cls = Path(path).stem.rsplit("_", 2)
            out["saves"].append((int(tid), int(cls), int(crop[0, 0, 0]), int(crop[0, 0, 1]), int(crop[-1, -1, 0]) + 1,
                                 int(crop[-1, -1, 1]) + 1))
        out["save_off"].append(out["save_off"][-1] + len(state["writes"]))
        out["rejects"] += [(i, t) for t in rejects_now]
    preds = np.concatenate(out["preds"]).reshape(-1, 7)
    return {"pred_mask": np.packbits(np.concatenate(out["mask"])), "pred_sha": np.array(hashlib.sha256(preds.tobytes()).hexdigest()),
            "flags": np.array(out["flags"], np.uint8), "adds": np.array(out["adds"], np.int32).reshape(-1, 3),
            "saves": np.array(out["saves"], np.int64).reshape(-1, 6), "save_off": np.array(out["save_off"], np.int32),
            "rejects": np.array(out["rejects"], np.int32).reshape(-1, 2)}


def pred_rows(rows):
    """The (n,7) preds row each target (tracker row tlwh, score, class, id, ...) would give (clearcam.py:611)."""
    r = np.asarray(rows, np.float64).reshape(-1, 9)
    return np.stack([r[:, 0], r[:, 1], r[:, 0] + r[:, 2], r[:, 1] + r[:, 3], r[:, 4], r[:, 5], r[:, 6]], 1)


def expected(g, cfgs, k, rows):
    """Configuration k of the fixture `g` (a dict of its arrays) on the host tracker's rows [(n,9)] of its sequence ->
    per frame (preds, flags, saves, alert adds [(zone, class)]) and the clock.  The preds rows are rebuilt from `rows`
    and must hash to the reference's bytes."""
    cfg = cfgs[k]
    f0, f1 = cfg["f0"], cfg["f1"]
    assert [len(rows[f]) for f in range(f0, f1)] == cfg["n_targets"], "the host tracker's rows differ from the fixture's"
    mask = np.unpackbits(g[f"c{k}_pred_mask"], count=sum(cfg["n_targets"])).astype(bool)
    fl, s, so, adds = g[f"c{k}_flags"], g[f"c{k}_saves"], g[f"c{k}_save_off"], g[f"c{k}_adds"]
    out, m0, p0 = [], 0, 0
    for i, f in enumerate(range(f0, f1)):
        m = mask[m0:m0 + len(rows[f])]
        p = pred_rows(rows[f])[m]
        out.append((p, fl[p0:p0 + len(p)], s[so[i]:so[i + 1]], [tuple(int(v) for v in a[1:]) for a in adds[adds[:, 0] == i]]))
        m0 += len(m)
        p0 += len(p)
    assert p0 == len(fl)
    digest = hashlib.sha256(np.concatenate([o[0] for o in out]).reshape(-1, 7).tobytes()).hexdigest()
    assert digest == str(g[f"c{k}_pred_sha"]), f"configuration {k}: rebuilt preds differ from the reference's"
    return out, clock(cfg["clock"], f1 - f0)


# ------------------------------------------------------------------------------------------------ zones
def frac(v, n):
    """A fraction c with c * n == v exactly in float64 (the reference scales coords by the frame size), or None."""
    c = v / n
    for _ in range(8):
        if c * n == v:
            return c
        c = np.nextafter(c, np.inf if c * n < v else -np.inf)
    return None


def star(n, cx, cy, r0, r1, seed):
    g = np.random.default_rng(seed)
    a = np.sort(g.uniform(0, 2 * np.pi, n))
    r = np.where(np.arange(n) % 2 == 0, r0, r1) * g.uniform(0.8, 1.2, n)
    return [[float(cx + r[k] * np.cos(a[k])), float(cy + r[k] * np.sin(a[k]))] for k in range(n)]


def pinned_zones(rows, W, H, f0, f1, thr_speed=2.5):
    """Zones with a box corner of a moving target exactly on a vertical edge, and exactly on a diamond's left vertex (the
    equality branches of point_not_in_polygon): [(zone, frame)]."""
    out = {"edge": None, "vertex": None}
    for f in range(f0, f1):
        for r in rows[f]:
            if r[7] < 1 or r[8] < thr_speed:
                continue
            x2, y1, y2 = r[0] + r[2], r[1], r[1] + r[3]
            if out["edge"] is None:
                cx, ca, cb, cc = frac(x2, W), frac(y1 - 30, H), frac(y2 + 30, H), frac(x2 + 80, W)
                if None not in (cx, ca, cb, cc) and y1 - 30 > 0:
                    out["edge"] = ([[cx, ca], [cc, ca], [cc, cb], [cx, cb]], f)
            elif out["vertex"] is None and f > out["edge"][1] + 5:
                cx, cy = frac(x2, W), frac(y2, H)
                cm, cr, ct, cd, cs = frac(x2 + 60, W), frac(x2 + 120, W), frac(y2 - 60, H), frac(y2 + 60, H), frac(y2 + 10, H)
                if None not in (cx, cy, cm, cr, ct, cd, cs):       # the right vertex lower than the left: no symmetry
                    out["vertex"] = ([[cx, cy], [cm, ct], [cr, cs], [cm, cd]], f)
        if out["vertex"] is not None:
            break
    return out


def configs(rows_of):
    cfgs = []

    def add(seq, f0, f1, W, H, zone, outside=False, nza=False, classes=None, clk="10fps"):
        cfgs.append(dict(seq=seq, f0=f0, f1=f1, W=W, H=H, zone=zone, outside=outside, non_zone_alert=nza, classes=classes, clock=clk))

    hexagon = [[0.1, 0.1], [0.9, 0.15], [0.95, 0.5], [0.8, 0.9], [0.2, 0.8], [0.05, 0.5]]
    bowtie = [[0.1, 0.1], [0.9, 0.9], [0.9, 0.1], [0.1, 0.9]]
    lshape = [[0.0, 0.25], [0.5, 0.25], [0.5, 0.5], [0.75, 0.5], [0.75, 1.0], [0.0, 1.0]]      # horizontal and vertical edges
    add("street", 0, 600, 960, 540, None)
    add("street", 0, 600, 1920, 1080, hexagon, clk="30fps")
    add("street", 300, 900, 960, 540, star(10, 0.5, 0.55, 0.45, 0.2, 1), outside=True, classes=[0, 2], clk="gaps")
    add("street", 600, 1500, 960, 540, bowtie, nza=True)
    add("street", 0, 1500, 960, 540, star(64, 0.5, 0.5, 0.5, 0.3, 2), outside=True, nza=True)
    add("street", 0, 1500, 960, 540, lshape, classes=[0], clk="gaps")
    add("synth_a", 0, 240, 1280, 720, [[0.2, 0.1], [0.9, 0.5], [0.3, 0.95]], classes=[1, 3, 5], clk="30fps")
    add("synth_b", 0, 240, 1280, 720, lshape, outside=True, clk="gaps")
    add("synth_c", 0, 240, 1920, 1080, bowtie, nza=True, clk="10fps")
    add("synth_c", 0, 240, 1280, 720, star(7, 0.5, 0.5, 0.4, 0.15, 3), outside=True, nza=True, clk="30fps")
    add("edge", 0, 150, 640, 360, None, clk="gaps")
    add("edge", 0, 150, 640, 360, [[0.0, 0.0], [0.6, 0.0], [0.6, 0.6], [0.0, 0.6]], clk="10fps")
    for seq, W, H in [("synth_a", 1280, 720), ("synth_b", 1280, 720), ("street", 960, 540)]:
        pz = pinned_zones(rows_of[seq], W, H, 20, 200)
        for kind in ("edge", "vertex"):
            if pz[kind] is not None:
                zone, f = pz[kind]
                add(seq, max(0, f - 40), f + 20, W, H, zone, clk="10fps")
                add(seq, max(0, f - 40), f + 20, W, H, zone, outside=True, nza=True, clk="10fps")
    return cfgs


def main():
    code = reference_functions()
    seqs = sequences()
    rows_of = {name: tracker_rows(*s) for name, s in seqs.items()}
    out = {"edge_frames": seqs["edge"][0]}
    cfgs = configs(rows_of)
    for k, cfg in enumerate(cfgs):
        r = run_config(code, rows_of[cfg["seq"]], cfg)
        cfg["n_targets"] = [int(len(rows_of[cfg["seq"]][f])) for f in range(cfg["f0"], cfg["f1"])]
        for name, a in r.items():
            out[f"c{k}_{name}"] = a
        print(k, cfg["seq"], cfg["f0"], cfg["f1"], "zone", None if cfg["zone"] is None else len(cfg["zone"]), "preds", len(r["flags"]),
              "flags", np.bincount(r["flags"], minlength=4).tolist(), "adds", len(r["adds"]), "saves", len(r["saves"]),
              "rejects", len(r["rejects"]))
    out["configs"] = np.array(json.dumps(cfgs))
    g = {k: v for k, v in out.items()}
    for k in range(len(cfgs)):                                  # the stored form rebuilds the reference's answers
        expected(g, cfgs, k, rows_of[cfgs[k]["seq"]])
    np.savez_compressed(OUT / "events_ref.npz", **out)
    print("wrote", OUT / "events_ref.npz", (OUT / "events_ref.npz").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
