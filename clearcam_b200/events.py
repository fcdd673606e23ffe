"""One camera's object events, as `run_inference` computes them after the tracker (clearcam.py:586-621): the class
filter, `tracklet_len < 1`, the `pred_occs` clock that picks the objects `save_object` writes, the motion gate, the zone
test and the `new` / `new_in_zone` bookkeeping behind the counters and alerts.

    ev = ObjectEvents(zone=settings["coords"], outside=settings["outside"], non_zone_alert=any(not a.zone for a in alerts))
    preds, flags, saves = ev.update(targets, W, H, now)

`preds` is run_inference's return value (k,7) float64 [x1, y1, x2, y2, score, class, track_id], (0,7) when empty.
`flags` (k,) uint8: bit 0 `new` (the id entered object_set: counter.add and the alerts without a zone), bit 1
`new_in_zone` (it entered object_set_zone: the alerts with a zone).  `saves` (m,6) int64 [track_id, class_id, x1, y1,
x2, y2]: the crops save_object writes, in its order; objects whose rectangle is under 100 px still use up their turn.

This is the host path (rows of stand-in models); the GPU runs the same steps in csrc/events_gpu.cu.  Where it has to
choose, it chooses so:
  - one clock reading `now` per camera-step.  The reference reads time.time() several times per target, so the two agree
    whenever its clock does not advance inside the loop;
  - `outside` must be a bool (the reference raises on `True ^ None`);
  - a target that passes the class filter and `tracklet_len` with a box that int() rejects (not finite), or one beyond
    2**60 in magnitude, is an error for the camera (ValueError), not a silent row."""
from typing import Iterable, Optional, Sequence

import numpy as np

from .models.objects import ObjectFinder

MAX_VERTICES = 256          # zone vertices (CC_EVENT_MAX_VERTICES)
OCC_CAP = 20                # pred_occs entries that still count towards the 1 s rule (clearcam.py:592)
MIN_SPEED = 2.5             # clearcam.py:597
BOX_LIMIT = 2.0 ** 60       # save_object's integer steps stay inside int64 on the device


def point_not_in_polygon(coords, poly) -> bool:
    """clearcam.py:647-665: True when no point of `coords` is inside `poly` (ray casting, as written there)."""
    n = len(poly)
    for x, y in coords:
        inside = False
        p1x, p1y = poly[0]
        for i in range(1, n + 1):
            p2x, p2y = poly[i % n]
            if y > min(p1y, p2y):
                if y <= max(p1y, p2y):
                    if x <= max(p1x, p2x):
                        x_intersect = (y - p1y) * (p2x - p1x) / (p2y - p1y) + p1x if p1y != p2y else p1x
                        if p1x == p2x or x <= x_intersect:
                            inside = not inside
            p1x, p1y = p2x, p2y
        if inside:
            return False
    return True


def check_zone(zone) -> Optional[np.ndarray]:
    """zone: None / empty (no zone) or >= 1 (x, y) pairs as fractions of the frame -> float64 (n,2) or None."""
    if zone is None or len(zone) == 0:
        return None
    z = np.array(zone, np.float64)
    if z.ndim != 2 or z.shape[1] != 2 or len(z) > MAX_VERTICES:
        raise ValueError(f"zone must be 1..{MAX_VERTICES} (x, y) pairs, got shape {z.shape}")
    if not np.isfinite(z).all():
        raise ValueError("zone coordinates must be finite")
    return z


class ObjectEvents:
    """One camera's event state (clearcam.py `pred_occs[cam]`, `object_set[cam]`, `object_set_zone[cam]`) and settings."""

    def __init__(self, zone=None, outside: bool = False, non_zone_alert: bool = False, classes: Optional[Iterable[int]] = None):
        """zone: the camera's polygon (settings["coords"], fractions of the frame) or None; outside: settings["outside"];
        non_zone_alert: whether any of the camera's alerts has no zone (clearcam.py:605-609); classes: the class ids the
        product watches (the reference's `classes`, as ints) or None for all."""
        if not isinstance(outside, (bool, np.bool_)) or not isinstance(non_zone_alert, (bool, np.bool_)):
            raise TypeError("outside and non_zone_alert must be bools")
        self.zone = check_zone(zone)
        self.outside, self.non_zone_alert = bool(outside), bool(non_zone_alert)
        self.classes = None if classes is None else {int(c) for c in classes}
        self.occ = {}                # track id -> [number of occurrences, last occurrence time]
        self.seen, self.seen_zone = set(), set()

    def update(self, targets: Sequence, W: int, H: int, now: float):
        """targets: the tracker's output for this frame (STrack-like: tlwh, score, class_id, track_id, tracklet_len,
        speed), W x H the frame's picture size, now the step's clock.  -> (preds, flags, saves) (module doc)."""
        preds, flags, saves = [], [], []
        poly = None if self.zone is None else self.zone * [float(W), float(H)]
        todo = []
        for x in targets:
            if (self.classes is not None and int(x.class_id) not in self.classes) or x.tracklet_len < 1:   # :586, :589
                continue
            t = np.asarray(x.tlwh, np.float64)
            if not (np.isfinite(t).all() and (np.abs(t) < BOX_LIMIT).all() and np.isfinite(t[:2] + t[2:]).all()
                    and (np.abs(t[:2] + t[2:]) < BOX_LIMIT).all()):
                raise ValueError(f"track {x.track_id}: box {t.tolist()} is not finite or beyond 2**60")
            todo.append((x, t))
        for x, t in todo:
            tid = x.track_id
            o = self.occ.get(tid)
            if o is None:                                                                    # :591
                o = self.occ[tid] = [1, now]
            if (o[0] < OCC_CAP and now - o[1] > 1) or now - o[1] > 10:                     # :592-595
                o[0] = min(o[0] + 1, OCC_CAP)
                o[1] = now
                r = ObjectFinder.crop_rect((t[0], t[1], t[0] + t[2], t[1] + t[3]), W, H)
                if r is not None:
                    saves.append((int(tid), int(x.class_id)) + tuple(r))
            if x.speed < MIN_SPEED:                                                          # :597
                continue
            outside = False
            if poly is not None:                                                             # :599-603
                x1, y1, x2, y2 = t[0], t[1], t[0] + t[2], t[1] + t[3]
                outside = point_not_in_polygon([[x1, y1], [x2, y1], [x1, y2], [x2, y2]], poly) ^ self.outside
            if outside and not self.non_zone_alert:                                          # :604-610
                continue
            preds.append([t[0], t[1], t[0] + t[2], t[1] + t[3], x.score, x.class_id, x.track_id])   # :611
            k = int(tid)
            new = k not in self.seen                                                         # :612-618
            new_in_zone = k not in self.seen_zone and not outside
            if new:
                self.seen.add(k)
            if new_in_zone:
                self.seen_zone.add(k)
            flags.append(int(new) | int(new_in_zone) << 1)
        return (np.array(preds, np.float64).reshape(-1, 7), np.array(flags, np.uint8),
                np.array(saves, np.int64).reshape(-1, 6))
