"""One camera's alerts, as the reference decides them (clearcam.py `RollingClassCounter` :47-103, the adds of
`run_inference` :612-620, the firing loop of `process_frame` :465-499 and the description alerts of `clip_latest_img`
:1289-1307).  What an alert then does (the event image, the notification, the upload) stays with the caller.

    al = CameraAlerts([Alert.from_counter(rc) for rc in alert_counters[cam].values()], desc_emb)
    fired = al.step(preds, flags, now, local)      # indices of the alerts that fired, in alert order
    hits = al.describe(embs, now, local)           # [(save index, alert index, similarity)]

`preds` / `flags` are ObjectEvents.update's (clearcam_b200/events.py).  `local` is (seconds of day, weekday with 0 =
Monday), what `time.localtime()` gives; `local_time(now)` makes it from the clock.

This is the host path; the GPU runs the same steps in csrc/alerts_gpu.cu.  Where it has to choose, it chooses so:
  - one clock `now` and one local (seconds of day, weekday) per step (the reference reads time.time() and
    time.localtime() many times);
  - a `sched` without an entry for the weekday counts as inactive that day (the reference raises IndexError inside
    process_frame and restarts ffmpeg; the UI's default seven-entry `sched` has none for Sunday);
  - alerts with `max` 0/None and description alerts keep no counts: they can never fire on counts and nothing reads
    their counts, so this cannot be observed; it bounds the storage to `max` timestamps per (alert, class);
  - the warm-up (`self.count[cam] > 10`) counts the camera's steps since it was added or its tracker reset;
  - a camera left out of a step (the reference's gate of :447, when none of its alerts is active) keeps its counts and
    its warm-up count until its next step.  The reference still runs its firing loop on such a frame: it resets the
    counts of the inactive alerts (all of them) and advances the warm-up.  Stepping the camera with no preds rows
    (`step(empty, empty, now, local)`) does exactly that, which is how the host form replays a gated frame;
  - a description alert whose threshold is None (what /edit_alert stores when the request has none; the reference's
    comparison then raises) never fires;
  - the similarity of a description and an object is the exact fp32 x fp32 products, summed in fp64 in one fixed
    order (`similarity`), rounded to fp32.  The reference's float32 BLAS product can differ by about 1 ulp, so only a
    similarity within about 1e-7 of the threshold can decide differently."""
import math
import time
from collections import deque
from typing import List, NamedTuple, Optional, Sequence

import numpy as np

MAX_ALERTS = 64              # alerts per camera (CC_ALERT_MAX_ALERTS)
MAX_COUNT = 1024             # largest `max` (CC_ALERT_MAX_COUNT)
CLASSES = 80                 # the detector's class ids
WARMUP = 10                  # process_frame fires only once self.count[cam] > 10
DESC_COOLDOWN = 60.0         # clip_latest_img: `time.time() - v.last_det < 60`
DEFAULT_THRESHOLD = 0.28     # RollingClassCounter's default


def local_time(now: float):
    """(seconds of day, weekday with 0 = Monday) of `now` in local time, as is_active reads time.localtime()."""
    t = time.localtime(now)
    return t.tm_hour * 3600 + t.tm_min * 60 + t.tm_sec, t.tm_wday


def _number(v, what):
    if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(float(v)):
        raise ValueError(f"{what} must be a finite number, got {v!r}")
    return float(v)


class Alert(NamedTuple):
    """One alert's settings (RollingClassCounter's fields, :47-64, as /edit_alert sets them, :804-851).

    classes: frozenset of class ids, or None for every class; max: 0 for none; window: seconds, or None for the default
    (60 s when is_notif, else 1 s); sched: None (always) or ((start, end), seven weekday flags, Monday first, a missing
    entry False); desc: the description text of a description alert, or None; threshold: its similarity threshold
    (None: never fires); last_det: the clock of its last firing."""
    classes: Optional[frozenset] = None
    max: int = 0
    window: Optional[float] = None
    sched: Optional[tuple] = None
    is_on: bool = True
    is_notif: bool = True
    zone: bool = True
    desc: Optional[str] = None
    threshold: Optional[float] = DEFAULT_THRESHOLD
    last_det: float = 0.0

    @classmethod
    def make(cls, classes=None, max=None, window=None, sched=None, is_on=True, is_notif=True, zone=True, desc=None,
             threshold=DEFAULT_THRESHOLD, last_det=0.0) -> "Alert":
        """Checked construction from RollingClassCounter-style values (sched as the reference stores it:
        [[start, end], mon, ..., sun])."""
        if classes is not None:
            # add() tests `class_id not in self.classes` with an int class id: members that are not ints never match
            classes = frozenset(int(c) for c in classes if isinstance(c, (int, np.integer)) and not isinstance(c, bool))
        if max is None or max is False:
            max = 0
        if isinstance(max, bool) or not isinstance(max, (int, np.integer)) or not 0 <= max <= MAX_COUNT:
            raise ValueError(f"max must be None or an int in 0..{MAX_COUNT}, got {max!r}")
        if window is not None and window != 0:         # the reference treats a falsy window as unset
            window = _number(window, "window")
            if window <= 0:
                raise ValueError(f"window must be positive, got {window}")
        else:
            window = None
        if sched is not None and len(sched) > 0:
            start, end = (_number(v, "sched[0]") for v in sched[0])
            sched = ((start, end), tuple(bool(sched[d]) if d < len(sched) else False for d in range(1, 8)))
        else:
            sched = None
        if desc is not None and not isinstance(desc, str):
            raise ValueError(f"desc must be a string or None, got {desc!r}")
        if threshold is not None:
            threshold = _number(threshold, "threshold")
        return cls(classes, int(max), window, sched, bool(is_on), bool(is_notif), bool(zone), desc, threshold,
                   _number(last_det, "last_det"))

    @classmethod
    def from_counter(cls, rc) -> "Alert":
        """The settings of a reference RollingClassCounter `rc` (is_on read as is_active reads it)."""
        return cls.make(classes=rc.classes, max=rc.max, window=rc.window, sched=rc.sched, is_on=getattr(rc, "is_on", False),
                        is_notif=rc.is_notif, zone=rc.zone, desc=rc.desc, threshold=rc.threshold, last_det=rc.last_det)

    @property
    def span(self) -> float:
        """The window in seconds (RollingClassCounter: `self.window if self.window else (60 if self.is_notif else 1)`)."""
        return self.window if self.window else (60.0 if self.is_notif else 1.0)

    @property
    def keeps_counts(self) -> bool:
        return self.max > 0 and self.desc is None

    def settings(self) -> "Alert":
        """The alert without its clock: two alerts with equal settings are the same alert to `CameraAlerts.replace`."""
        return self._replace(last_det=0.0)

    def is_active(self, alerts_on: bool, local) -> bool:
        """RollingClassCounter.is_active (:95-103) at local (seconds of day, weekday)."""
        if not alerts_on or not self.is_on:
            return False
        if self.sched is None:
            return True
        tod, wday = local
        if not self.sched[1][wday]:
            return False
        start, end = self.sched[0]
        return tod < end and tod > start - self.span


def active(alerts: Sequence[Alert], local, alerts_on: bool = True) -> np.ndarray:
    """Every alert's is_active at local (seconds of day, weekday) as a bool array (the gate of :447 is its any())."""
    n = len(alerts)
    if not alerts_on or n == 0:
        return np.zeros(n, bool)
    tod, wday = local
    on = np.array([a.is_on for a in alerts], bool)
    has = np.array([a.sched is not None for a in alerts], bool)
    day = np.array([a.sched is not None and a.sched[1][wday] for a in alerts], bool)
    start = np.array([a.sched[0][0] if a.sched else 0.0 for a in alerts], np.float64)
    end = np.array([a.sched[0][1] if a.sched else 0.0 for a in alerts], np.float64)
    span = np.array([a.span for a in alerts], np.float64)
    return on & (~has | (day & (tod < end) & (tod > start - span)))


def similarity(desc_emb, emb) -> np.ndarray:
    """desc_emb [A,D] and emb [N,D] float32 -> [N,A] float32: each dot product as the exact fp32 x fp32 products summed
    in fp64 in one fixed order — lane l of 32 sums elements l, l+32, ... in turn, then an xor butterfly over 16, 8, 4,
    2, 1 — rounded to fp32.  csrc/alerts_gpu.cu sums in the same order, so both give the same bits."""
    q = np.asarray(desc_emb, np.float32).astype(np.float64)
    e = np.asarray(emb, np.float32).astype(np.float64)
    if q.ndim != 2 or e.ndim != 2 or q.shape[1] != e.shape[1]:
        raise ValueError(f"embeddings must be [A,D] and [N,D] with one D, got {q.shape} and {e.shape}")
    p = e[:, None, :] * q[None, :, :]
    acc = np.zeros(p.shape[:2] + (32,), np.float64)
    for k in range(0, p.shape[2], 32):
        seg = p[:, :, k:k + 32]
        acc[:, :, :seg.shape[2]] += seg
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, :, lanes ^ o]
    return acc[:, :, 0].astype(np.float32)


class _Counts:
    """One alert's class deques (RollingClassCounter.data), pruned as add / get_counts prune them."""

    def __init__(self, alert: Alert):
        self.alert, self.q = alert, {}

    def prune(self, now):
        w = self.alert.span
        for q in self.q.values():
            while q and now - q[0] > w:
                q.popleft()

    def max_reached(self, now) -> bool:                   # get_counts()[1]
        self.prune(now)
        return any(len(q) >= self.alert.max for q in self.q.values())

    def add(self, cls, now):
        if self.alert.classes is not None and cls not in self.alert.classes:
            return
        q = self.q.setdefault(cls, deque())
        q.append(now)
        w = self.alert.span
        while q and now - q[0] > w:
            q.popleft()


class CameraAlerts:
    """One camera's alerts and their state, with its object counter (self.counter[cam], a window of inf: the count of new
    ids per class) and its warm-up count."""

    def __init__(self, alerts: Sequence[Alert] = (), desc_emb=None, alerts_on: bool = True):
        self.alerts: List[Alert] = []
        self.counts: List[_Counts] = []
        self.last_det: List[float] = []
        self.desc_emb = None
        self.alerts_on = bool(alerts_on)
        self.counter = np.zeros(CLASSES, np.int64)
        self.warm = 0
        self.adds = None             # a list to record each count added as (alert index, class id)
        self.replace(alerts, desc_emb)

    def replace(self, alerts: Sequence[Alert], desc_emb=None, keep: Optional[Sequence[int]] = None):
        """New settings.  keep[i]: the index of the current alert whose counts and last_det alert i keeps (its settings
        must be equal), or -1: it starts empty with its own last_det.  desc_emb: [len(alerts), D] float32 (rows of
        alerts without a description are not read), or None when no alert has one."""
        alerts = list(alerts)
        if len(alerts) > MAX_ALERTS:
            raise ValueError(f"{len(alerts)} alerts (at most {MAX_ALERTS} per camera)")
        for a in alerts:
            if not isinstance(a, Alert):
                raise TypeError("alerts must be Alert settings (Alert.make / Alert.from_counter)")
        keep = [-1] * len(alerts) if keep is None else [int(k) for k in keep]
        if len(keep) != len(alerts):
            raise ValueError("one keep entry per alert")
        emb = None
        if any(a.desc is not None for a in alerts):
            if desc_emb is None:
                raise ValueError("description alerts need their embeddings")
            emb = np.asarray(desc_emb, np.float32)
            if emb.ndim != 2 or emb.shape[0] != len(alerts) or emb.shape[1] < 1:
                raise ValueError(f"desc_emb must be [{len(alerts)}, D], got {emb.shape}")
        counts, last = [], []
        for a, k in zip(alerts, keep):
            if k >= 0:
                if k >= len(self.alerts) or self.alerts[k].settings() != a.settings():
                    raise ValueError(f"alert to keep {k} does not exist or has other settings")
                c = self.counts[k]
                c.alert = a
                counts.append(c)
                last.append(self.last_det[k])
            else:
                counts.append(_Counts(a))
                last.append(a.last_det)
        self.alerts, self.counts, self.last_det, self.desc_emb = alerts, counts, last, emb

    def reset(self):
        """A restarted camera (init_cam): a fresh object counter and warm-up; the alerts keep their state."""
        self.counter[:] = 0
        self.warm = 0

    def active(self, local) -> np.ndarray:
        return active(self.alerts, local, self.alerts_on)

    def step(self, preds, flags, now: float, local) -> List[int]:
        """The adds of run_inference over this step's preds rows and flags (:612-620), then the firing loop of
        process_frame (:465-499) -> the indices of the alerts that fired, in alert order."""
        now = float(now)
        for row, f in zip(np.asarray(preds, np.float64).reshape(-1, 7), np.asarray(flags, np.uint8)):
            cls = int(row[5])
            if f & 1:
                self.counter[cls] += 1
            for i, (a, c) in enumerate(zip(self.alerts, self.counts)):
                if not a.keeps_counts:
                    continue
                if not c.max_reached(now) and ((f & 1 and not a.zone) or (f & 2 and a.zone)):
                    c.add(cls, now)
                    if self.adds is not None and (a.classes is None or cls in a.classes):
                        self.adds.append((i, cls))
        fired = []
        if self.warm > WARMUP:
            for i, (a, c) in enumerate(zip(self.alerts, self.counts)):
                if a.desc is not None:
                    continue
                if not a.is_active(self.alerts_on, local):
                    c.q = {}
                    continue
                if a.keeps_counts and c.max_reached(now) and now - self.last_det[i] >= a.span:
                    self.last_det[i] = now
                    fired.append(i)
        else:
            self.warm += 1
        return fired

    def similarity(self, emb) -> np.ndarray:
        """[N,A] float32 similarity of N object embeddings with every alert's description (NaN for alerts without one)."""
        emb = np.asarray(emb, np.float32)
        emb = emb.reshape(len(emb), -1) if emb.size else emb.reshape(len(emb), emb.shape[-1] if emb.ndim == 2 else 0)
        out = np.full((len(emb), len(self.alerts)), np.nan, np.float32)
        if self.desc_emb is not None and len(emb):
            d = [i for i, a in enumerate(self.alerts) if a.desc is not None]
            out[:, d] = similarity(self.desc_emb[d], emb)
        return out

    def describe(self, emb, now: float, local):
        """clip_latest_img's description alerts (:1289-1307) on the embeddings of one step's saved objects, in save order
        -> [(save index, alert index, similarity)] of the alerts that fired (at most one per object)."""
        now = float(now)
        sims = self.similarity(emb)
        act = self.active(local)
        hits = []
        for s in range(len(sims)):
            for i, a in enumerate(self.alerts):
                if now - self.last_det[i] < DESC_COOLDOWN or not act[i] or a.desc is None:
                    continue
                if a.threshold is not None and float(sims[s, i]) > a.threshold:
                    self.last_det[i] = now
                    hits.append((s, i, float(sims[s, i])))
                    break
        return hits
