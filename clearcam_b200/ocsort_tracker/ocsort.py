"""`OCSort` with the reference's constructor and `update` contract (ocsort_tracker/ocsort.py:163-177), running in the
C++ tracker of libclearcam_b200 (csrc/ocsort.cu) instead of per-frame numpy.

    tracker = ocsort.OCSort(max_age=100)                 # clearcam.py:239
    online_targets = tracker.update(preds, thresh)       # clearcam.py:585, preds = the detector's (300,6) array

`update_many` steps the trackers of several cameras on one batched detector result in a single library call;
`DeviceTrackers` does the same on the GPU for rows that stay on the device, and can run each camera's object events
(clearcam_b200/events.py, csrc/events_gpu.cu) right after its tracker, and its alerts (clearcam_b200/alerts.py,
csrc/alerts_gpu.cu) right after those."""
import ctypes
from typing import List, Optional, Sequence

import numpy as np

from .._lib import (CC_ALERT_DESC, CC_ALERT_MAX_ALERTS, CC_ALERT_OK, CC_ALERT_ON, CC_ALERT_SCHED, CC_ALERT_ZONE, CC_EVENT_BAD_BOX,
                    CC_EVENT_BAD_ORDER, CC_EVENT_NEEDS_ROOM, CC_EVENT_OK, CC_TRACK_BAD_BOX, CC_TRACK_BAD_CLASS, CC_TRACK_NEEDS_ROOM, CC_TRACK_OK,
                    CC_TRACK_OVERFLOW, CCError, cc_alert, cc_track_run, check, lib)
from .STrack import STrack

_CAP = 1024          # rows of the result buffer (the detector emits at most 300 boxes per frame)
_HEAD = 128          # DeviceTrackers: rows per camera copied to the host with every launch; longer results are read after


def _rows(output_results) -> np.ndarray:
    a = output_results.numpy() if hasattr(output_results, "numpy") and not isinstance(output_results, np.ndarray) else output_results
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] < 6:
        raise ValueError("detections must be (n, 6): x1, y1, x2, y2, score, class")
    return a if a.shape[1] == 6 else np.ascontiguousarray(a[:, :6])


def _tracks(buf: np.ndarray, n: int) -> List[STrack]:
    return [STrack(tlwh=r[:4], score=r[4], class_id=r[5], track_id=r[6], age=r[7], speed=r[8]) for r in buf[:n]]


class _Launched(list):
    """The jobs of one DeviceTrackers.launch; `events` holds each job's (W, H, now) when the events ran with them, and
    `alerts` each job's local time (seconds of day, weekday) when the alerts ran after the events."""
    events = None
    alerts = None


def _cc_alert(a) -> cc_alert:
    """alerts.Alert -> the library's cc_alert."""
    words = [0xffffffff, 0xffffffff, 0xffff] if a.classes is None else [0, 0, 0]
    if a.classes is not None:
        for c in a.classes:
            if 0 <= c < 80:
                words[c >> 5] |= 1 << (c & 31)
    flags = ((CC_ALERT_ON if a.is_on else 0) | (CC_ALERT_ZONE if a.zone else 0) | (CC_ALERT_DESC if a.desc is not None else 0)
             | (CC_ALERT_SCHED if a.sched is not None else 0))
    days = 0 if a.sched is None else sum(1 << d for d in range(7) if a.sched[1][d])
    start, end = (0.0, 0.0) if a.sched is None else a.sched[0]
    r = cc_alert()
    r.classes[:] = words
    r.max, r.flags, r.days = a.max, flags, days
    r.window, r.start, r.end = a.span, start, end
    r.threshold = float("inf") if a.threshold is None else a.threshold
    r.last_det = a.last_det
    return r


class _Runs(list):
    """The jobs of one DeviceTrackers.launch_runs: per job its per-frame events and alerts arguments, the frames read so far,
    the errors, and the launch groups whose results are still to be read."""

    def __init__(self, jobs, events, alerts):
        super().__init__(jobs)
        self.events, self.alerts = events, alerts
        self.res = [[] for _ in jobs]
        self.errors = {}
        self.pending = []


class _RunGroup:
    """One launch per stage over up to CC_MAX_FRAMES runs.  items[b] = (job, first frame, carry): carry is None when the
    tracker ran in this group, else (tracker status, capacity it needs) of the tracker launch whose rows the events rerun."""

    def __init__(self, items):
        self.items = items


def _host(t):
    """A pinned host copy of device tensor t, enqueued on the current stream."""
    h = t.new_empty(tuple(t.shape), device="cpu", pin_memory=True)
    h.copy_(t, non_blocking=True)
    return h


class _EventBuffers:
    """Device outputs of one events launch, their first _HEAD rows packed on the device, pinned host copies of those,
    and the tracker outputs (rows [B,_CAP,9], counts [B], statuses [B]) the launch read."""

    def __init__(self, torch, B):
        dev = dict(device="cuda")
        self.preds = torch.empty((B, _CAP, 7), dtype=torch.float64, **dev)
        self.flags = torch.empty((B, _CAP), dtype=torch.uint8, **dev)
        self.saves = torch.empty((B, _CAP, 6), dtype=torch.int64, **dev)
        self.cs = torch.empty((3, B), dtype=torch.int32, **dev)            # preds rows, save rows, status (3 x launch B)
        self.head = (torch.empty((B, _HEAD, 7), dtype=torch.float64, **dev), torch.empty((B, _HEAD), dtype=torch.uint8, **dev),
                     torch.empty((B, _HEAD, 6), dtype=torch.int64, **dev))
        self.host = tuple(torch.empty(tuple(t.shape), dtype=t.dtype, pin_memory=True) for t in self.head)
        self.hcs = torch.empty((3, B), dtype=torch.int32, pin_memory=True)
        self.trk, self.B = None, 0
        self.fired = torch.empty((B, CC_ALERT_MAX_ALERTS), dtype=torch.int32, **dev)   # alerts: fired indices, then
        self.ares = torch.empty((2, B), dtype=torch.int32, **dev)                      # their count and status
        self.hfired = torch.empty((B, CC_ALERT_MAX_ALERTS), dtype=torch.int32, pin_memory=True)
        self.hares = torch.empty((2, B), dtype=torch.int32, pin_memory=True)
        self.alerts = False                                                           # whether the alerts ran


class OCSort:
    def __init__(self, det_thresh=0.25, max_age=30, min_hits=3, iou_threshold=0.3, delta_t=3, asso_func="iou", inertia=0.2,
                 use_byte=False):
        if asso_func != "iou":
            raise ValueError("only the IoU association the reference uses is implemented")    # ocsort.py:175
        self.max_age, self.min_hits, self.iou_threshold, self.delta_t = max_age, min_hits, iou_threshold, delta_t
        self.inertia, self.use_byte = inertia, use_byte
        self.frame_count = 0
        self._h = ctypes.c_void_p()
        check(lib().cc_ocsort_create(int(max_age), int(min_hits), float(iou_threshold), int(delta_t), float(inertia),
                                     int(bool(use_byte)), ctypes.byref(self._h)), "cc_ocsort_create")
        self._out = np.empty((_CAP, 9), np.float64)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().cc_ocsort_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def __len__(self):
        return lib().cc_ocsort_num_tracks(self._h)

    def update(self, output_results, det_thresh=0.25) -> List[STrack]:
        if output_results is None:                          # ocsort.py:185-186
            return np.empty((0, 5))
        a = _rows(output_results)
        n = ctypes.c_int()
        check(lib().cc_ocsort_update(self._h, a.ctypes.data, a.shape[0], float(det_thresh), self._out.ctypes.data, _CAP,
                                     ctypes.byref(n)), "cc_ocsort_update")
        self.frame_count += 1
        return _tracks(self._out, n.value)


def update_many(trackers: Sequence[Optional[OCSort]], results, det_thresh) -> List[List[STrack]]:
    """Step tracker b on results[b] (a (B,n,6) float32 array — one batched detector output) for every b; entries of
    `trackers` may be None (camera without a tracker).  det_thresh: scalar or one value per camera."""
    r = results.numpy() if hasattr(results, "numpy") and not isinstance(results, np.ndarray) else results
    r = np.ascontiguousarray(r, dtype=np.float32)
    B = len(trackers)
    if r.ndim != 3 or r.shape[0] != B or r.shape[2] != 6:
        raise ValueError("results must be (len(trackers), n, 6)")
    thr = np.ascontiguousarray(np.broadcast_to(np.asarray(det_thresh, np.float32), (B,)))
    hs = (ctypes.c_void_p * B)(*[t._h if t is not None else None for t in trackers])
    out = np.empty((B, _CAP, 9), np.float64)
    n = np.zeros(B, np.int32)
    check(lib().cc_ocsort_update_batch(hs, B, r.ctypes.data, r.shape[1], thr.ctypes.data, out.ctypes.data, _CAP, n.ctypes.data),
          "cc_ocsort_update_batch")
    for t in trackers:
        if t is not None:
            t.frame_count += 1
    return [_tracks(out[b], int(n[b])) if trackers[b] is not None else [] for b in range(B)]


class DeviceTrackers:
    """One `OCSort` per camera, all on the GPU (csrc/ocsort_gpu.cu): `update` steps every camera of a list of jobs in one
    launch per CC_MAX_FRAMES cameras, on detector rows that never leave the device, and returns what `update_many` returns
    for the same rows, bit for bit (track ids included).

        trk = DeviceTrackers()
        trk.add("cam0", max_age=100)                         # OCSort.__init__'s arguments
        [targets] = trk.update([("cam0", rows, 0.5)])       # rows: CUDA float32 (n,6), e.g. one row of detect_batch's output

    `launch` / `finish` split `update` around a synchronisation the caller does anyway (CameraBatch.step)."""

    def __init__(self, slots: int = 1024, max_delta_t: int = 8, capacity: int = 64, event_capacity: int = 64):
        import torch
        from .._lib import CC_MAX_FRAMES
        self._torch, self._B = torch, CC_MAX_FRAMES
        self._h = ctypes.c_void_p()
        check(lib().cc_ocsort_gpu_create(int(slots), int(max_delta_t), ctypes.byref(self._h)), "cc_ocsort_gpu_create")
        self._free = list(range(slots - 1, -1, -1))
        self._slot, self._args, self._cap = {}, {}, {}
        self._capacity = int(capacity)
        self._bufs = []                                        # per launch of one update: device and pinned results
        self._ev, self._ecap, self._event_capacity = {}, {}, int(event_capacity)   # events: settings and room per camera
        self._ebufs, self._rbufs = [], []                      # events outputs: per launch, and for reruns after growth
        self._al = set()                                       # cameras with alerts configured
        self._n_alerts = {}                                    # camera -> its number of alerts

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                lib().cc_ocsort_gpu_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def __contains__(self, cam):
        return cam in self._slot

    def _stream(self):
        return ctypes.c_void_p(self._torch.cuda.current_stream().cuda_stream)

    def _configure(self, cam):
        a = self._args[cam]
        check(lib().cc_ocsort_gpu_configure(self._h, self._slot[cam], a["max_age"], a["min_hits"], a["iou_threshold"], a["delta_t"],
                                            a["inertia"], a["use_byte"], self._cap[cam], self._stream()),
              f"cc_ocsort_gpu_configure (camera {cam!r})")

    def add(self, cam, det_thresh=0.25, max_age=30, min_hits=3, iou_threshold=0.3, delta_t=3, asso_func="iou", inertia=0.2,
            use_byte=False):
        """A tracker for camera `cam` with OCSort.__init__'s arguments (an existing one is replaced)."""
        if asso_func != "iou":
            raise ValueError("only the IoU association the reference uses is implemented")
        if cam not in self._slot:
            if not self._free:
                raise ValueError("every tracker slot is in use")
            self._slot[cam] = self._free.pop()
            self._cap[cam] = self._capacity
        self._args[cam] = dict(max_age=int(max_age), min_hits=int(min_hits), iou_threshold=float(iou_threshold),
                               delta_t=int(delta_t), inertia=float(inertia), use_byte=int(bool(use_byte)))
        try:
            self._configure(cam)
        except Exception:
            self._free.append(self._slot.pop(cam))
            del self._args[cam], self._cap[cam]
            raise

    def reset(self, cam):
        """Start camera `cam`'s tracker afresh (as a new OCSort with the same arguments), and its events with it (as
        init_cam makes both fresh)."""
        self._configure(cam)                                   # also clears the slot's event state

    def events(self, cam, zone=None, outside: bool = False, non_zone_alert: bool = False, classes=None):
        """Run camera `cam`'s object events after its tracker, with ObjectEvents' settings; starts its event state afresh.
        Launches that pass `events=` then give `finish_events` results."""
        from ..events import check_zone
        if cam not in self._slot:
            raise KeyError(f"camera {cam!r} has no tracker: add() it first")
        if not isinstance(outside, (bool, np.bool_)) or not isinstance(non_zone_alert, (bool, np.bool_)):
            raise TypeError("outside and non_zone_alert must be bools")
        z = check_zone(zone)
        self._ev[cam] = (np.zeros((0, 2)) if z is None else np.ascontiguousarray(z), bool(outside), bool(non_zone_alert),
                         None if classes is None else sorted({int(c) for c in classes}))
        self._ecap.setdefault(cam, self._event_capacity)
        self._configure_events(cam)

    def has_events(self, cam) -> bool:
        return cam in self._ev

    def _configure_events(self, cam):
        z, outside, nza, classes = self._ev[cam]
        mask = None
        if classes is not None:
            words = [0, 0, 0]
            for c in classes:
                if 0 <= c < 96:
                    words[c >> 5] |= 1 << (c & 31)
            mask = (ctypes.c_uint32 * 3)(*words)
        check(lib().cc_ocsort_gpu_events_configure(self._h, self._slot[cam], z.ctypes.data if len(z) else None, len(z), int(outside),
                                                   int(nza), mask, self._ecap[cam], self._stream()),
              f"cc_ocsort_gpu_events_configure (camera {cam!r})")

    def set_non_zone_alert(self, cam, non_zone_alert: bool):
        """Change camera `cam`'s non_zone_alert (events()) without starting its event state afresh: the reference reads it
        from the alerts at every target (clearcam.py:604-609)."""
        if cam not in self._ev:
            raise KeyError(f"camera {cam!r} has no events: events() it first")
        if not isinstance(non_zone_alert, (bool, np.bool_)):
            raise TypeError("non_zone_alert must be a bool")
        z, outside, _, classes = self._ev[cam]
        self._ev[cam] = (z, outside, bool(non_zone_alert), classes)
        check(lib().cc_ocsort_gpu_events_set_non_zone_alert(self._h, self._slot[cam], int(bool(non_zone_alert)), self._stream()),
              f"cc_ocsort_gpu_events_set_non_zone_alert (camera {cam!r})")

    def alerts(self, cam, alerts, desc_emb=None, keep=None):
        """Run camera `cam`'s alerts (a list of alerts.Alert, in order) after its events.  desc_emb: [len(alerts), D]
        float32 description embeddings (rows of alerts without a description are not read), None when none has one.
        keep[i]: the index of the camera's current alert whose counts and last_det alert i keeps (equal settings), or -1.
        The object counter, the warm-up count and alerts_on stay."""
        from ..alerts import MAX_ALERTS, Alert
        if cam not in self._slot:
            raise KeyError(f"camera {cam!r} has no tracker: add() it first")
        alerts = list(alerts)
        if len(alerts) > MAX_ALERTS or not all(isinstance(a, Alert) for a in alerts):
            raise ValueError(f"alerts must be at most {MAX_ALERTS} alerts.Alert")
        table = (cc_alert * max(1, len(alerts)))(*[_cc_alert(a) for a in alerts])
        emb, dim = None, 0
        if any(a.desc is not None for a in alerts):
            if desc_emb is None:
                raise ValueError("description alerts need their embeddings")
            t = desc_emb.detach().cpu().numpy() if hasattr(desc_emb, "detach") else desc_emb
            emb = np.ascontiguousarray(t, np.float32)
            if emb.ndim != 2 or emb.shape[0] != len(alerts):
                raise ValueError(f"desc_emb must be [{len(alerts)}, D], got {emb.shape}")
            dim = emb.shape[1]
        kp = None if keep is None else np.ascontiguousarray(keep, np.int32)
        if kp is not None and kp.shape != (len(alerts),):
            raise ValueError("one keep entry per alert")
        check(lib().cc_ocsort_gpu_alerts_configure(self._h, self._slot[cam], table, len(alerts), None if emb is None else emb.ctypes.data,
                                                   dim, None if kp is None else kp.ctypes.data, self._stream()),
              f"cc_ocsort_gpu_alerts_configure (camera {cam!r})")
        self._al.add(cam)
        self._n_alerts[cam] = len(alerts)

    def has_alerts(self, cam) -> bool:
        return cam in self._al

    def set_alerts_on(self, cam, on: bool):
        """The reference's alerts_on[cam] (is_active's first test); True after the first alerts()."""
        self._need_alerts(cam)
        check(lib().cc_ocsort_gpu_alerts_set_on(self._h, self._slot[cam], int(bool(on)), self._stream()),
              f"cc_ocsort_gpu_alerts_set_on (camera {cam!r})")

    def counts(self, cam) -> np.ndarray:
        """Camera `cam`'s object counter (self.counter[cam]): int64 [80], new ids per class id.  Waits for the stream."""
        self._need_alerts(cam)
        out = np.zeros(80, np.int64)
        check(lib().cc_ocsort_gpu_alerts_counts(self._h, self._slot[cam], out.ctypes.data, self._stream()),
              f"cc_ocsort_gpu_alerts_counts (camera {cam!r})")
        return out

    def reset_counts(self, cam):
        """Zero camera `cam`'s object counter (/reset_counts, clearcam.py:512-517)."""
        self._need_alerts(cam)
        check(lib().cc_ocsort_gpu_alerts_reset_counts(self._h, self._slot[cam], self._stream()),
              f"cc_ocsort_gpu_alerts_reset_counts (camera {cam!r})")

    def _need_alerts(self, cam):
        if cam not in self._al:
            raise KeyError(f"camera {cam!r} has no alerts: alerts() it first")

    def describe(self, jobs, emb, now, local):
        """clip_latest_img's description alerts on the device.  jobs: [(camera, rows)], the cameras' consecutive rows of
        emb (a CUDA float32 [N,D] tensor, e.g. the embeddings of save_objects), each camera at most once; now and local
        (seconds of day, weekday) per job.  One launch per CC_MAX_FRAMES cameras, one wait -> per job (hits (rows,) int32:
        the index of the alert that fired per row or -1, similarities (rows, alerts) float32, NaN for alerts without a
        description)."""
        torch = self._torch
        if len(jobs) != len(now) or len(jobs) != len(local):
            raise ValueError("one clock and one local time per job")
        if not (isinstance(emb, torch.Tensor) and emb.is_cuda and emb.dtype == torch.float32 and emb.dim() == 2 and emb.is_contiguous()):
            raise ValueError("emb must be a contiguous CUDA float32 [N, D] tensor")
        n = sum(int(r) for _, r in jobs)
        if n != emb.shape[0]:
            raise ValueError(f"the jobs cover {n} rows, emb has {emb.shape[0]}")
        for cam, _ in jobs:
            self._need_alerts(cam)
        hit = torch.empty(max(n, 1), dtype=torch.int32, device="cuda")
        sim = torch.empty((max(n, 1), CC_ALERT_MAX_ALERTS), dtype=torch.float32, device="cuda")
        r0 = 0
        for c0 in range(0, len(jobs), self._B):
            chunk = jobs[c0:c0 + self._B]
            rows = np.array([int(r) for _, r in chunk], np.int32)
            slots = np.array([self._slot[cam] for cam, _ in chunk], np.int32)
            t = np.array([float(x) for x in now[c0:c0 + self._B]], np.float64)
            loc = np.array([(float(a), float(b)) for a, b in local[c0:c0 + self._B]], np.float64).reshape(-1)
            check(lib().cc_ocsort_gpu_describe(self._h, slots.ctypes.data, rows.ctypes.data, len(chunk), t.ctypes.data, loc.ctypes.data,
                                               emb[r0:].data_ptr() if r0 < n else emb.data_ptr(), emb.shape[1], hit[r0:].data_ptr(),
                                               sim[r0:].data_ptr(), self._stream()), "cc_ocsort_gpu_describe")
            r0 += int(rows.sum())
        h, s = hit.cpu().numpy(), sim.cpu().numpy()
        out, r0 = [], 0
        for cam, r in jobs:
            A = self._n_alerts[cam]
            out.append((h[r0:r0 + r].copy(), s[r0:r0 + r, :A].copy()))
            r0 += r
        return out

    def remove(self, cam):
        slot = self._slot.pop(cam, None)
        if slot is None:
            return
        del self._args[cam], self._cap[cam]
        self._ev.pop(cam, None)
        self._al.discard(cam)
        self._n_alerts.pop(cam, None)
        self._ecap.pop(cam, None)
        check(lib().cc_ocsort_gpu_free(self._h, slot, self._stream()), "cc_ocsort_gpu_free")   # frees its events too
        self._free.append(slot)

    def num_tracks(self, cam) -> int:
        n = ctypes.c_int()
        check(lib().cc_ocsort_gpu_num_tracks(self._h, self._slot[cam], ctypes.byref(n), self._stream()), "cc_ocsort_gpu_num_tracks")
        return n.value

    def _buffers(self, i):
        """Buffer set i: device results [B,_CAP,9], counts and statuses, their first _HEAD rows packed on the device, and
        pinned host copies of those (only the head crosses PCIe with every launch)."""
        torch = self._torch
        while len(self._bufs) <= i:
            self._bufs.append((torch.empty((self._B, _CAP, 9), dtype=torch.float64, device="cuda"),
                               torch.empty((2, self._B), dtype=torch.int32, device="cuda"),
                               torch.empty((self._B, _HEAD, 9), dtype=torch.float64, device="cuda"),
                               torch.empty((self._B, _HEAD, 9), dtype=torch.float64, pin_memory=True),
                               torch.empty((2, self._B), dtype=torch.int32, pin_memory=True)))
        return self._bufs[i]

    def _launch(self, jobs, i, events=None, alerts=None):
        """Enqueue one launch for <= CC_MAX_FRAMES jobs into buffer set i and the copy of its results to the host; with
        `events` ((W, H, now) per job), the events launch on its outputs follows, and with `alerts` (local time per job)
        the alerts launch after that."""
        from .._lib import cc_track_job
        table = (cc_track_job * len(jobs))()
        for b, (cam, rows, thr) in enumerate(jobs):
            if cam not in self._slot:
                raise KeyError(f"camera {cam!r} has no tracker: add() it first")
            if rows.dtype != self._torch.float32 or not rows.is_cuda or rows.dim() != 2 or rows.shape[1] != 6 or not rows.is_contiguous():
                raise ValueError(f"camera {cam!r}: rows must be a contiguous CUDA float32 (n, 6) tensor")
            table[b] = cc_track_job(rows.data_ptr() if rows.shape[0] else None, rows.shape[0], self._slot[cam], float(thr), 0)
        out, cs, head, hout, hcs = self._buffers(i)
        B = len(jobs)
        check(lib().cc_ocsort_gpu_update(self._h, table, B, out.data_ptr(), _CAP, cs[0].data_ptr(), cs[1].data_ptr(),
                                         self._stream()), "cc_ocsort_gpu_update")
        head[:B].copy_(out[:B, :_HEAD])
        hcs.copy_(cs, non_blocking=True)
        hout[:B].copy_(head[:B], non_blocking=True)
        if events is not None:
            while len(self._ebufs) <= i:
                self._ebufs.append(_EventBuffers(self._torch, self._B))
            self._launch_events(table, [j[0] for j in jobs], events, (out, cs[0], cs[1]), self._ebufs[i], alerts)

    def _launch_events(self, table, cams, events, trk, eb, alerts=None):
        """Enqueue the events of `cams` (slots in `table`) on tracker outputs `trk` into event buffers `eb`, and with
        `alerts` (local time per camera) the alerts on the events' outputs."""
        for cam in cams:
            if cam not in self._ev:
                raise KeyError(f"camera {cam!r} has no events: events() it first")
            if alerts is not None:
                self._need_alerts(cam)
        B = len(cams)
        wh = np.array([(int(W), int(H)) for W, H, _ in events], np.int32).reshape(-1)
        now = np.array([float(t) for _, _, t in events], np.float64)
        eb.trk, eb.B = trk, B
        cs = eb.cs.view(-1)[:3 * B]                            # [3,B]: preds rows, save rows (d_counts [2,B]), status
        check(lib().cc_ocsort_gpu_events(self._h, table, B, wh.ctypes.data, now.ctypes.data, trk[0].data_ptr(), _CAP, trk[1].data_ptr(),
                                         trk[2].data_ptr(), eb.preds.data_ptr(), eb.flags.data_ptr(), eb.saves.data_ptr(), _CAP,
                                         cs.data_ptr(), cs[2 * B:].data_ptr(), self._stream()), "cc_ocsort_gpu_events")
        for h, d, full in zip(eb.head, eb.host, (eb.preds, eb.flags, eb.saves)):
            h[:B].copy_(full[:B, :_HEAD])
        eb.hcs.view(-1)[:3 * B].copy_(cs, non_blocking=True)
        for h, d in zip(eb.head, eb.host):
            d[:B].copy_(h[:B], non_blocking=True)
        eb.alerts = alerts is not None
        if eb.alerts:
            loc = np.array([(float(t), float(d)) for t, d in alerts], np.float64).reshape(-1)
            ares = eb.ares.view(-1)[:2 * B]
            check(lib().cc_ocsort_gpu_alerts(self._h, table, B, now.ctypes.data, loc.ctypes.data, eb.preds.data_ptr(), eb.flags.data_ptr(),
                                             _CAP, cs.data_ptr(), cs[2 * B:].data_ptr(), eb.fired.data_ptr(), ares.data_ptr(),
                                             self._stream()), "cc_ocsort_gpu_alerts")
            eb.hfired[:B].copy_(eb.fired[:B], non_blocking=True)
            eb.hares.view(-1)[:2 * B].copy_(ares, non_blocking=True)

    def launch(self, jobs, events=None, alerts=None):
        """Enqueue `update(jobs)` without waiting; pass the result to `finish` after the stream is synchronised.
        events: (W, H, now) per job — the frame's picture size and the step's clock — to run each camera's object events
        right after its tracker (`finish_events` then returns them).  alerts: (seconds of day, weekday) per job — the
        step's local time — to run each camera's alerts right after its events (`finish_alerts` then returns them)."""
        jobs = _Launched(jobs)
        if events is not None:
            jobs.events = list(events)
            if len(jobs.events) != len(jobs):
                raise ValueError("one (W, H, now) per job")
        if alerts is not None:
            if events is None:
                raise ValueError("alerts run on the events' outputs: pass events= too")
            jobs.alerts = [(float(t), int(d)) for t, d in alerts]
            if len(jobs.alerts) != len(jobs):
                raise ValueError("one (seconds of day, weekday) per job")
            if not all(np.isfinite(t) and 0 <= d <= 6 for t, d in jobs.alerts):    # checked before the tracker launches
                raise ValueError("local time: a finite time of day and a weekday in 0..6")
            for cam, _, _ in jobs:
                self._need_alerts(cam)
        for i, c0 in enumerate(range(0, len(jobs), self._B)):
            self._launch(jobs[c0:c0 + self._B], i, None if jobs.events is None else jobs.events[c0:c0 + self._B],
                         None if jobs.alerts is None else jobs.alerts[c0:c0 + self._B])
        return jobs

    def finish(self, jobs, targets: bool = True) -> list:
        """The targets of `launch(jobs)` once the stream has been synchronised.  A camera whose tracker lacked room is
        grown and stepped again here (one more launch and wait).  Every other camera's frame is complete before anything
        is raised: if cameras failed (a class id that is not an integer in 0..79: that tracker is unchanged; more than
        _CAP tracks: the frame was applied), one CCError names them all, and its `results` holds every camera's targets,
        None for the failed ones.  targets=False: (number of targets, CC_TRACK_OK) per camera instead, no STrack built."""
        res, _, errors = self._collect(jobs, targets)
        if errors:
            e = CCError("; ".join(errors))
            e.results = res
            raise e
        return res

    def finish_events(self, jobs) -> list:
        """The object events of `launch(jobs, events=...)` once the stream has been synchronised: per camera
        (preds (k,7) float64, flags (k,) uint8, saves (m,6) int64) as ObjectEvents.update returns them.  Trackers or event
        storage that lacked room are grown and run again here.  Failed cameras (the tracker's errors, or a box that is
        not finite: that camera's events are unchanged) are named in one CCError after every other camera has finished,
        whose `results` holds the others' events and None for the failed ones."""
        if getattr(jobs, "events", None) is None:
            raise ValueError("these jobs were launched without events")
        _, res, errors = self._collect(jobs, False)
        res = [None if r is None else r[:3] for r in res]
        if errors:
            e = CCError("; ".join(errors))
            e.results = res
            raise e
        return res

    def finish_alerts(self, jobs) -> list:
        """The events and alerts of `launch(jobs, events=..., alerts=...)` once the stream has been synchronised: per camera
        (preds, flags, saves, fired) with fired the (n,) int32 indices of the alerts that fired, in alert order.  Events
        run again after growth carry their alerts along.  Errors as finish_events."""
        if getattr(jobs, "alerts", None) is None:
            raise ValueError("these jobs were launched without alerts")
        _, res, errors = self._collect(jobs, False)
        if errors:
            e = CCError("; ".join(errors))
            e.results = res
            raise e
        return res

    def _read_events(self, jobs, k, eb, b, evr, grow, errors):
        cam = jobs[k][0]
        hcs = eb.hcs.view(-1)
        n, m, st = (int(hcs[r * eb.B + b]) for r in range(3))
        if st == CC_EVENT_OK:
            if n <= _HEAD and m <= _HEAD:
                p, f, s = (h[b, :c].numpy().copy() for h, c in zip(eb.host, (n, n, m)))
            else:
                p, f, s = eb.preds[b, :n].cpu().numpy(), eb.flags[b, :n].cpu().numpy(), eb.saves[b, :m].cpu().numpy()
            fired = None
            if eb.alerts:
                if int(eb.hares.view(-1)[eb.B + b]) != CC_ALERT_OK:
                    errors.append(f"camera {cam!r}: its alerts did not run")
                    return
                fired = eb.hfired[b, :int(eb.hares.view(-1)[b])].numpy().copy()
            evr[k] = (p, f, s, fired)
        elif st == CC_EVENT_NEEDS_ROOM:
            grow.append((k, eb, b, n))
        elif st == CC_EVENT_BAD_BOX:
            errors.append(f"camera {cam!r}: a target's box is not finite or beyond 2**60 (its events are unchanged)")
        elif st == CC_EVENT_BAD_ORDER:
            errors.append(f"camera {cam!r}: the tracker's ids are out of order (its events are unchanged)")
        # CC_EVENT_NOT_RUN: the tracker failed (reported) or lacked room (stepped again with its events)

    def _collect(self, jobs, targets):
        """Read every result of `launch(jobs)`, growing and rerunning what lacked room -> (targets, events, errors)."""
        from .._lib import cc_track_job
        res, evr, errors = [None] * len(jobs), [None] * len(jobs), []
        ev = getattr(jobs, "events", None)
        al = getattr(jobs, "alerts", None)
        pend = [(k, k // self._B, k % self._B) for k in range(len(jobs))]    # (job, buffer set, row) of tracker launches
        ev_pend = []                                                            # (job, event buffers, row) of event reruns
        while pend or ev_pend:
            grow, ev_grow = [], []
            for k, i, b in pend:
                out, _, _, hout, hcs = self._bufs[i]
                cam, n, st = jobs[k][0], int(hcs[0, b]), int(hcs[1, b])
                if st == CC_TRACK_NEEDS_ROOM:
                    grow.append((k, n))
                    continue
                if st == CC_TRACK_BAD_CLASS:
                    errors.append(f"camera {cam!r}: a detection's class id is not an integer in 0..79 (its tracker is unchanged)")
                elif st == CC_TRACK_OVERFLOW:
                    errors.append(f"camera {cam!r}: {n} tracks do not fit the output capacity {_CAP}")
                elif not targets:
                    res[k] = (n, st)
                elif n <= _HEAD:                               # copies: the buffers are reused by the next launch
                    res[k] = _tracks(hout[b, :n].numpy().copy(), n)
                else:
                    res[k] = _tracks(out[b, :n].cpu().numpy(), n)
                if ev is not None:
                    self._read_events(jobs, k, self._ebufs[i], b, evr, ev_grow, errors)
            for k, eb, b in ev_pend:
                self._read_events(jobs, k, eb, b, evr, ev_grow, errors)
            ev_pend = []
            # events that lacked room: grow, and run them again on the same tracker rows (gathered before any relaunch
            # below reuses the buffers those rows sit in)
            for c0 in range(0, len(ev_grow), self._B):
                chunk = ev_grow[c0:c0 + self._B]
                for k, _, _, need in chunk:
                    cam = jobs[k][0]
                    cap = max(2 * self._ecap[cam], need)
                    check(lib().cc_ocsort_gpu_events_grow(self._h, self._slot[cam], cap, self._stream()),
                          f"cc_ocsort_gpu_events_grow (camera {cam!r})")
                    self._ecap[cam] = cap
                trk = tuple(self._torch.stack([eb.trk[r][b] for _, eb, b, _ in chunk]) for r in range(3))
                j = c0 // self._B
                while len(self._rbufs) <= j:
                    self._rbufs.append(_EventBuffers(self._torch, self._B))
                table = (cc_track_job * len(chunk))(*[cc_track_job(None, 0, self._slot[jobs[k][0]], 0.0, 0) for k, _, _, _ in chunk])
                self._launch_events(table, [jobs[k][0] for k, _, _, _ in chunk], [ev[k] for k, _, _, _ in chunk], trk, self._rbufs[j],
                                    None if al is None else [al[k] for k, _, _, _ in chunk])
                ev_pend += [(k, self._rbufs[j], b) for b, (k, _, _, _) in enumerate(chunk)]
            for k, need in grow:
                cam = jobs[k][0]
                cap = max(2 * self._cap[cam], need)
                check(lib().cc_ocsort_gpu_grow(self._h, self._slot[cam], cap, self._stream()), f"cc_ocsort_gpu_grow (camera {cam!r})")
                self._cap[cam] = cap
            idx = [k for k, _ in grow]
            pend = []
            if idx:
                again = [jobs[k] for k in idx]
                for i, c0 in enumerate(range(0, len(idx), self._B)):
                    self._launch(again[c0:c0 + self._B], i, None if ev is None else [ev[k] for k in idx[c0:c0 + self._B]],
                                 None if al is None else [al[k] for k in idx[c0:c0 + self._B]])
                pend = [(k, p // self._B, p % self._B) for p, k in enumerate(idx)]
            if pend or ev_pend:
                self._torch.cuda.current_stream().synchronize()
        return res, evr, errors

    # -- runs: several consecutive frames of one camera per job (a recorded video), one launch per stage
    def launch_runs(self, jobs, events=None, alerts=None):
        """Enqueue runs without waiting; pass the result to `finish_runs` after the stream is synchronised.  jobs: [(camera,
        rows, det_thresh)] with rows a contiguous CUDA float32 [T,n,6] tensor (T consecutive frames, 1 <= T <= CC_MAX_FRAMES),
        each camera at most once.  events: per job, a list of T (W, H, now), one per frame; alerts: per job, a list of T
        (seconds of day, weekday).  Each camera's frames are applied in order, exactly as T `launch` calls would."""
        from .._lib import CC_MAX_FRAMES
        jobs = [(cam, rows, float(thr)) for cam, rows, thr in jobs]
        if len({cam for cam, _, _ in jobs}) != len(jobs):
            raise ValueError("each camera at most once per launch_runs")
        for cam, rows, _ in jobs:
            if cam not in self._slot:
                raise KeyError(f"camera {cam!r} has no tracker: add() it first")
            if (rows.dtype != self._torch.float32 or not rows.is_cuda or rows.dim() != 3 or rows.shape[2] != 6 or not rows.is_contiguous()
                    or not 1 <= rows.shape[0] <= CC_MAX_FRAMES):
                raise ValueError(f"camera {cam!r}: rows must be a contiguous CUDA float32 (T, n, 6) tensor, 1 <= T <= {CC_MAX_FRAMES}")
        ev = al = None
        if events is not None:
            ev = [[(int(W), int(H), float(t)) for W, H, t in e] for e in events]
            if len(ev) != len(jobs) or any(len(e) != rows.shape[0] for e, (_, rows, _) in zip(ev, jobs)):
                raise ValueError("one (W, H, now) per frame of every job")
            for cam, _, _ in jobs:
                if cam not in self._ev:
                    raise KeyError(f"camera {cam!r} has no events: events() it first")
        if alerts is not None:
            if ev is None:
                raise ValueError("alerts run on the events' outputs: pass events= too")
            al = [[(float(t), int(d)) for t, d in a] for a in alerts]
            if len(al) != len(jobs) or any(len(a) != rows.shape[0] for a, (_, rows, _) in zip(al, jobs)):
                raise ValueError("one (seconds of day, weekday) per frame of every job")
            if not all(np.isfinite(t) and 0 <= d <= 6 for a in al for t, d in a):
                raise ValueError("local time: a finite time of day and a weekday in 0..6")
            for cam, _, _ in jobs:
                self._need_alerts(cam)
        run = _Runs(jobs, ev, al)
        for c0 in range(0, len(jobs), self._B):
            self._launch_runs(run, [(k, 0, None) for k in range(c0, min(len(jobs), c0 + self._B))])
        return run

    def _launch_runs(self, run, items, trk=None):
        """One group: the tracker runs of items (job, first frame) — or, with trk (tracker rows, counts, ids, live, done of
        an earlier launch, gathered per item), only the events — then the events and alerts behind them."""
        torch = self._torch
        g = _RunGroup(items)
        B = len(items)
        frames = [run[k][1].shape[0] - f0 for k, f0, _ in items]
        Tm = max(frames)
        dev = dict(device="cuda")
        table = (cc_track_run * B)()
        for b, (k, f0, _) in enumerate(items):
            cam, rows, thr = run[k]
            r = rows[f0:]
            table[b] = cc_track_run(r.data_ptr() if r.shape[1] else None, r.shape[1], frames[b], self._slot[cam], thr)
        if trk is None:
            cap = max(1, max(run[k][1].shape[1] for k, _, _ in items))       # a frame emits at most one target per row
            id_cap = max(self._cap[run[k][0]] for k, _, _ in items)
            trk = (torch.empty((B, Tm, cap, 9), dtype=torch.float64, **dev), torch.empty((B, Tm), dtype=torch.int32, **dev),
                   torch.empty((B, Tm, id_cap), dtype=torch.int32, **dev), torch.empty((B, Tm), dtype=torch.int32, **dev),
                   torch.empty((2, B), dtype=torch.int32, **dev))
            out, cnt, ids, live, ds = trk
            check(lib().cc_ocsort_gpu_update_runs(self._h, table, B, Tm, out.data_ptr(), cap, cnt.data_ptr(), ids.data_ptr(), id_cap,
                                                  live.data_ptr(), ds[0].data_ptr(), ds[1].data_ptr(), self._stream()),
                  "cc_ocsort_gpu_update_runs")
            g.hcnt, g.hds = _host(cnt), _host(ds)
            if run.events is None:
                g.hout = _host(out)
        else:
            g.avail = trk[4][0].tolist()                                       # tracker frames the gathered rows hold
        g.trk = trk
        out, cnt, ids, live, ds = trk
        if run.events is not None:
            cap = out.shape[2]
            ev = [e for k, f0, _ in items for e in run.events[k][f0:]]
            wh = np.array([(W, H) for W, H, _ in ev], np.int32).reshape(-1)
            now = np.array([t for _, _, t in ev], np.float64)
            preds = torch.empty((B, Tm, cap, 7), dtype=torch.float64, **dev)
            flags = torch.empty((B, Tm, cap), dtype=torch.uint8, **dev)
            saves = torch.empty((B, Tm, cap, 6), dtype=torch.int64, **dev)
            ecnt = torch.empty((2, B, Tm), dtype=torch.int32, **dev)
            eds = torch.empty((2, B), dtype=torch.int32, **dev)
            check(lib().cc_ocsort_gpu_events_runs(self._h, table, B, Tm, wh.ctypes.data, now.ctypes.data, out.data_ptr(), cap, cnt.data_ptr(),
                                                  ids.data_ptr(), ids.shape[2], live.data_ptr(), ds[0].data_ptr(), preds.data_ptr(),
                                                  flags.data_ptr(), saves.data_ptr(), cap, ecnt.data_ptr(), eds[0].data_ptr(),
                                                  eds[1].data_ptr(), self._stream()), "cc_ocsort_gpu_events_runs")
            g.hev = tuple(_host(t) for t in (preds, flags, saves, ecnt, eds))
            if run.alerts is not None:
                loc = np.array([a for k, f0, _ in items for a in run.alerts[k][f0:]], np.float64).reshape(-1)
                fired = torch.empty((B, Tm, CC_ALERT_MAX_ALERTS), dtype=torch.int32, **dev)
                nf = torch.empty((B, Tm), dtype=torch.int32, **dev)
                ads = torch.empty((2, B), dtype=torch.int32, **dev)
                check(lib().cc_ocsort_gpu_alerts_runs(self._h, table, B, Tm, now.ctypes.data, loc.ctypes.data, preds.data_ptr(),
                                                      flags.data_ptr(), cap, ecnt.data_ptr(), eds[0].data_ptr(), fired.data_ptr(),
                                                      nf.data_ptr(), ads[0].data_ptr(), ads[1].data_ptr(), self._stream()),
                      "cc_ocsort_gpu_alerts_runs")
                g.hal = (_host(fired), _host(nf))
        run.pending.append(g)

    def finish_runs(self, run) -> list:
        """The results of `launch_runs(jobs, ...)` once the stream has been synchronised: per camera a list with one entry
        per frame — its targets, or with events (preds, flags, saves) as `finish_events` gives them, or with alerts (preds,
        flags, saves, fired) as `finish_alerts`.  Trackers or event storage that lacked room are grown here and the run goes
        on from the frame that stopped (more launches and waits).  A camera whose frame k failed (as `finish_events`
        describes) keeps frames 0..k-1; after every other camera has finished its run, one CCError names every failed camera
        and frame, and its `results` holds what each camera completed."""
        from .._lib import CC_EVENT_NOT_RUN
        torch = self._torch
        while run.pending:
            torch.cuda.current_stream().synchronize()
            groups, run.pending = run.pending, []
            full, again = [], []                     # (job, first frame): rerun everything / only the events from there
            for g in groups:
                for b, (k, f0, carry) in enumerate(g.items):
                    cam, T = run[k][0], run[k][1].shape[0] - f0
                    if carry is None:
                        td, ts = int(g.hds[0, b]), int(g.hds[1, b])
                        need = int(g.hcnt[b, td]) if td < T else 0
                    else:
                        td, (ts, need) = g.avail[b], carry
                    if run.events is None:
                        for f in range(td):
                            n = int(g.hcnt[b, f])
                            run.res[k].append(_tracks(g.hout[b, f, :n].numpy().copy(), n))
                        stop = td
                    else:
                        p, fl, sv, ecnt, eds = g.hev
                        ed, es = int(eds[0, b]), int(eds[1, b])
                        for f in range(ed):
                            n, m = int(ecnt[0, b, f]), int(ecnt[1, b, f])
                            r = (p[b, f, :n].numpy().copy(), fl[b, f, :n].numpy().copy(), sv[b, f, :m].numpy().copy())
                            if run.alerts is not None:
                                r += (g.hal[0][b, f, :int(g.hal[1][b, f])].numpy().copy(),)
                            run.res[k].append(r)
                        stop = ed
                        if es == CC_EVENT_NEEDS_ROOM:
                            c = max(2 * self._ecap[cam], int(ecnt[0, b, ed]))
                            check(lib().cc_ocsort_gpu_events_grow(self._h, self._slot[cam], c, self._stream()),
                                  f"cc_ocsort_gpu_events_grow (camera {cam!r})")
                            self._ecap[cam] = c
                            again.append((k, f0 + ed, (g, b, ed, td, ts, need)))
                            continue
                        # the tracker run ends right after a frame with such a box (CC_TRACK_BAD_BOX), so here it has applied
                        # exactly frames ..f0 + ed, as after a failing single-frame step
                        if es == CC_EVENT_BAD_BOX:
                            run.errors[k] = (f"camera {cam!r} frame {f0 + ed}: a target's box is not finite or beyond 2**60 (its events "
                                             f"are unchanged; its tracker applied frame {f0 + td - 1} and stopped)")
                            continue
                        if es == CC_EVENT_BAD_ORDER:
                            run.errors[k] = (f"camera {cam!r} frame {f0 + ed}: the tracker's ids are out of order (its events are "
                                             f"unchanged; its tracker applied frame {f0 + td - 1} and stopped)")
                            continue
                        assert es in (CC_EVENT_OK, CC_EVENT_NOT_RUN)
                    if ts == CC_TRACK_BAD_BOX:        # the events of that frame ran and passed: the run goes on
                        full.append((k, f0 + stop, None))
                    elif ts == CC_TRACK_NEEDS_ROOM:
                        c = max(2 * self._cap[cam], need)
                        check(lib().cc_ocsort_gpu_grow(self._h, self._slot[cam], c, self._stream()), f"cc_ocsort_gpu_grow (camera {cam!r})")
                        self._cap[cam] = c
                        full.append((k, f0 + stop, None))
                    elif ts == CC_TRACK_BAD_CLASS:
                        run.errors[k] = f"camera {cam!r} frame {f0 + stop}: a detection's class id is not an integer in 0..79 (its tracker is unchanged)"
                    elif ts == CC_TRACK_OVERFLOW:
                        run.errors[k] = f"camera {cam!r} frame {f0 + stop}: {need} tracks do not fit the output capacity (the frame was applied)"
            # events that lacked room run again on the tracker rows of their frames (gathered before anything reuses them)
            for c0 in range(0, len(again), self._B):
                chunk = again[c0:c0 + self._B]
                Tm = max(run[k][1].shape[0] - f for k, f, _ in chunk)
                cap = max(src[0].trk[0].shape[2] for _, _, src in chunk)
                id_cap = max(src[0].trk[2].shape[2] for _, _, src in chunk)
                B = len(chunk)
                trk = (torch.zeros((B, Tm, cap, 9), dtype=torch.float64, device="cuda"), torch.zeros((B, Tm), dtype=torch.int32, device="cuda"),
                       torch.zeros((B, Tm, id_cap), dtype=torch.int32, device="cuda"), torch.zeros((B, Tm), dtype=torch.int32, device="cuda"))
                for i, (_, _, (g, b, ed, td, _, _)) in enumerate(chunk):
                    out, cnt, ids, live = g.trk[:4]
                    trk[0][i, :td - ed, :out.shape[2]] = out[b, ed:td]
                    trk[1][i, :td - ed] = cnt[b, ed:td]
                    trk[2][i, :td - ed, :ids.shape[2]] = ids[b, ed:td]
                    trk[3][i, :td - ed] = live[b, ed:td]
                done = torch.tensor([[td - ed for _, _, (_, _, ed, td, _, _) in chunk], [0] * B], dtype=torch.int32)
                self._launch_runs(run, [(k, f, (ts, need)) for k, f, (_, _, _, _, ts, need) in chunk], trk + (done.cuda(),))
            for c0 in range(0, len(full), self._B):
                self._launch_runs(run, full[c0:c0 + self._B])
        if run.errors:
            e = CCError("; ".join(run.errors[k] for k in sorted(run.errors)))
            e.results = run.res
            raise e
        return run.res

    def describe_runs(self, jobs, emb, now, local):
        """`describe` for the saves of runs: jobs [(camera, rows per frame)], the rows of each job consecutive in emb (frame
        after frame, job after job); now and local: per job, one clock and one (seconds of day, weekday) per frame.  Each
        camera's frames are matched in order, each at its own clock -> per job (hits, similarities) over all its rows."""
        torch = self._torch
        if len(jobs) != len(now) or len(jobs) != len(local):
            raise ValueError("one list of clocks and one of local times per job")
        if not (isinstance(emb, torch.Tensor) and emb.is_cuda and emb.dtype == torch.float32 and emb.dim() == 2 and emb.is_contiguous()):
            raise ValueError("emb must be a contiguous CUDA float32 [N, D] tensor")
        counts = [[int(r) for r in rows] for _, rows in jobs]
        if any(len(c) != len(t) or len(c) != len(l) for c, t, l in zip(counts, now, local)):
            raise ValueError("one clock and one local time per frame")
        n = sum(sum(c) for c in counts)
        if n != emb.shape[0]:
            raise ValueError(f"the jobs cover {n} rows, emb has {emb.shape[0]}")
        for cam, _ in jobs:
            self._need_alerts(cam)
        hit = torch.empty(max(n, 1), dtype=torch.int32, device="cuda")
        sim = torch.empty((max(n, 1), CC_ALERT_MAX_ALERTS), dtype=torch.float32, device="cuda")
        r0 = 0
        for c0 in range(0, len(jobs), self._B):
            sl = slice(c0, c0 + self._B)
            slots = np.array([self._slot[cam] for cam, _ in jobs[sl]], np.int32)
            frames = np.array([len(c) for c in counts[sl]], np.int32)
            rows = np.array([r for c in counts[sl] for r in c], np.int32)
            t = np.array([float(x) for ts in now[sl] for x in ts], np.float64)
            loc = np.array([(float(a), float(d)) for ls in local[sl] for a, d in ls], np.float64).reshape(-1)
            check(lib().cc_ocsort_gpu_describe_runs(self._h, slots.ctypes.data, frames.ctypes.data, len(slots), rows.ctypes.data,
                                                    t.ctypes.data, loc.ctypes.data, emb[r0:].data_ptr() if r0 < n else emb.data_ptr(),
                                                    emb.shape[1], hit[r0:].data_ptr(), sim[r0:].data_ptr(), self._stream()),
                  "cc_ocsort_gpu_describe_runs")
            r0 += int(rows.sum())
        h, s = hit.cpu().numpy(), sim.cpu().numpy()
        out, r0 = [], 0
        for (cam, _), c in zip(jobs, counts):
            A, r = self._n_alerts[cam], sum(c)
            out.append((h[r0:r0 + r].copy(), s[r0:r0 + r, :A].copy()))
            r0 += r
        return out

    def update(self, jobs) -> List[List[STrack]]:
        """jobs: [(camera, rows, det_thresh)] with rows a CUDA float32 (n,6) tensor; one camera at most once.  Returns each
        camera's targets, as OCSort.update / update_many would."""
        p = self.launch(jobs)
        self._torch.cuda.current_stream().synchronize()
        return self.finish(p)

