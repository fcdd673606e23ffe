"""`OCSort` with the reference's constructor and `update` contract (ocsort_tracker/ocsort.py:163-177), running in the
C++ tracker of libclearcam_b200 (csrc/ocsort.cu) instead of per-frame numpy.

    tracker = ocsort.OCSort(max_age=100)                 # clearcam.py:239
    online_targets = tracker.update(preds, thresh)       # clearcam.py:585, preds = the detector's (300,6) array

`update_many` steps the trackers of several cameras on one batched detector result in a single library call;
`DeviceTrackers` does the same on the GPU for rows that stay on the device, and can run each camera's object events
(clearcam_b200/events.py, csrc/events_gpu.cu) right after its tracker."""
import ctypes
from typing import List, Optional, Sequence

import numpy as np

from .._lib import (CC_EVENT_BAD_BOX, CC_EVENT_BAD_ORDER, CC_EVENT_NEEDS_ROOM, CC_EVENT_OK, CC_TRACK_BAD_CLASS,
                    CC_TRACK_NEEDS_ROOM, CC_TRACK_OVERFLOW, CCError, check, lib)
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
    """The jobs of one DeviceTrackers.launch; `events` holds each job's (W, H, now) when the events ran with them."""
    events = None


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

    def remove(self, cam):
        slot = self._slot.pop(cam, None)
        if slot is None:
            return
        del self._args[cam], self._cap[cam]
        self._ev.pop(cam, None)
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

    def _launch(self, jobs, i, events=None):
        """Enqueue one launch for <= CC_MAX_FRAMES jobs into buffer set i and the copy of its results to the host; with
        `events` ((W, H, now) per job), the events launch on its outputs follows."""
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
            self._launch_events(table, [j[0] for j in jobs], events, (out, cs[0], cs[1]), self._ebufs[i])

    def _launch_events(self, table, cams, events, trk, eb):
        """Enqueue the events of `cams` (slots in `table`) on tracker outputs `trk` into event buffers `eb`."""
        for cam in cams:
            if cam not in self._ev:
                raise KeyError(f"camera {cam!r} has no events: events() it first")
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

    def launch(self, jobs, events=None):
        """Enqueue `update(jobs)` without waiting; pass the result to `finish` after the stream is synchronised.
        events: (W, H, now) per job — the frame's picture size and the step's clock — to run each camera's object events
        right after its tracker (`finish_events` then returns them)."""
        jobs = _Launched(jobs)
        if events is not None:
            jobs.events = list(events)
            if len(jobs.events) != len(jobs):
                raise ValueError("one (W, H, now) per job")
        for i, c0 in enumerate(range(0, len(jobs), self._B)):
            self._launch(jobs[c0:c0 + self._B], i, None if jobs.events is None else jobs.events[c0:c0 + self._B])
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
            evr[k] = (p, f, s)
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
                self._launch_events(table, [jobs[k][0] for k, _, _, _ in chunk], [ev[k] for k, _, _, _ in chunk], trk, self._rbufs[j])
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
                    self._launch(again[c0:c0 + self._B], i, None if ev is None else [ev[k] for k in idx[c0:c0 + self._B]])
                pend = [(k, p // self._B, p % self._B) for p, k in enumerate(idx)]
            if pend or ev_pend:
                self._torch.cuda.current_stream().synchronize()
        return res, evr, errors

    def update(self, jobs) -> List[List[STrack]]:
        """jobs: [(camera, rows, det_thresh)] with rows a CUDA float32 (n,6) tensor; one camera at most once.  Returns each
        camera's targets, as OCSort.update / update_many would."""
        p = self.launch(jobs)
        self._torch.cuda.current_stream().synchronize()
        return self.finish(p)

