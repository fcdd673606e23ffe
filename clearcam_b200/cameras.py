"""All cameras in one detector call (SURVEY.md §8f N1).

The reference walks its cameras round-robin and runs the detector on one frame at a time (`VideoCapture.start`,
clearcam.py:270-271 -> `process_frame` :423-461 -> `run_inference` :580-586: Tensor(frame) -> jit_infer(model) ->
.numpy() -> tracker.update).  On an H100 a single 1080p frame leaves the GPU mostly idle, so `CameraBatch.step` takes the
latest frame of every camera, groups the frames by shape (cameras differ in resolution; the detector's letterbox plan is
per input shape), runs ONE `detect_batch` per group with uploads and result reads queued back to back, waits once, and
then steps every camera's tracker in one library call.  When the detector's rows are on the GPU, the trackers run there
too (`ocsort.DeviceTrackers`): one launch over every group of the step, queued right after the detector calls and
before that single wait, bit for bit what the host trackers give.  Rows on the host (stand-in models) keep the host
trackers.  What `step` returns per camera is what `run_inference` computes up to clearcam.py:589 — the (300,6)
detector rows and the tracker's targets.  `step_events` goes on to :621: each camera's zone, motion gate, object-save
picks and new-object flags (clearcam_b200/events.py), on the GPU right after the trackers (csrc/events_gpu.cu) for
device rows and by `ObjectEvents` for host rows, and returns run_inference's preds.  `step_alerts` goes on to decide the
camera's alerts (clearcam_b200/alerts.py: the adds of :612-620, the object counter and the firing loop of :465-499), on
the GPU right after the events (csrc/alerts_gpu.cu) for device rows and by `CameraAlerts` for host rows, and
`describe_saves` runs the description alerts of clip_latest_img (:1289-1307) on `save_objects`' embeddings; what a fired
alert then does (image, notification, upload) and the saving of the picked crops stay with the caller.

Each camera has a pixel format (clearcam_b200/pixfmt.py): "bgr24" [H,W,3] frames (the default) or "yuv420p" [H*3/2,W]
frames, which the detector converts on the GPU, or "mjpeg": one JPEG file per frame (bytes-like, e.g. a JpegMailbox
view).  Groups are keyed by (H, W, dtype, format).

An MJPEG camera's device frame is always cv2.imdecode of the file received, as bgr24, whichever side decodes it.  Each
step has one decode stage ahead of the detector: every MJPEG frame of the step is gathered, with the Huffman tables its
scan lacks (ingest.default_tables), into one pinned staging buffer and parsed in one call; the sizes place each picture
in the step's shape and net-shape groups like any bgr24 frame; one host-to-device copy and one decode call
(cc_jpeg_decode_frames) write the pixels straight into the buffers the detector reads (a camera's own buffer or a row
of a uniform batch); the step then waits for the statuses.  Frames the parse or the device leaves to the host are
decoded by cv2.imdecode and uploaded into their place; a frame cv2 also rejects is dropped for the step (the camera is
not stepped and gets no result, its batch row is padding, `dropped_frames` counts it).  With host rows (no CUDA) every
MJPEG frame is decoded by cv2.imdecode.

With the detector's frame tables (a model with `net_shape` and `detect_frames`), uint8 groups whose frames letterbox to
the same net input are merged: a fleet of 720p, 1080p, 1440p and 2160p cameras, bgr24 and yuv420p alike, runs as ONE
batch at res 640 (all of them give a 384 x 640 net input).  A merged group copies each frame into its camera's own
device buffer and makes one `detect_frames` call per CC_MAX_FRAMES cameras, padded to the batch bucket with None rows.
A group with a single source shape and format still calls `detect_batch`, as do float32 frames and models without
frame tables."""
import time
from typing import Dict, Hashable, List, NamedTuple, Optional

import numpy as np
import torch

from ._lib import CC_MAX_FRAMES
from .alerts import Alert, CameraAlerts, local_time
from .events import ObjectEvents
from .ocsort_tracker import ocsort
from .pixfmt import BGR24, MJPEG, check_camera_pix_fmt, yuv420p_size
from .utils.helpers import batch_bucket
from .ocsort_tracker.STrack import STrack


class CameraResult(NamedTuple):
    rows: np.ndarray            # (300,6) float32 detector output in this camera's frame coordinates
    targets: List[STrack]       # tracker.update(rows, thresh), unfiltered (clearcam.py:585)
    preds: np.ndarray           # (k,7) x1,y1,x2,y2,score,class,track_id of targets seen for more than one frame


class CameraEvents(NamedTuple):
    rows: np.ndarray            # (300,6) float32 detector output in this camera's frame coordinates
    preds: np.ndarray           # (k,7) float64: run_inference's return value (clearcam.py:611, 622)
    flags: np.ndarray           # (k,) uint8 per preds row: bit 0 new (object_set), bit 1 new in the zone (object_set_zone)
    saves: np.ndarray           # (m,6) int64 track_id, class_id, x1, y1, x2, y2: the crops save_object writes


class CameraAlertResult(NamedTuple):
    rows: np.ndarray            # (300,6) float32 detector output in this camera's frame coordinates
    preds: np.ndarray           # (k,7) float64: run_inference's return value (clearcam.py:611, 622)
    flags: np.ndarray           # (k,) uint8 per preds row: bit 0 new (object_set), bit 1 new in the zone (object_set_zone)
    saves: np.ndarray           # (m,6) int64 track_id, class_id, x1, y1, x2, y2: the crops save_object writes
    fired: list                 # the ids of the alerts that fired this step, in alert order (clearcam.py:485-499)


class _Camera:
    def __init__(self, thresh, classes, max_age, pix_fmt=BGR24):
        self.thresh, self.classes, self.pix_fmt = thresh, classes, pix_fmt
        self.tracker = ocsort.OCSort(max_age=max_age)          # clearcam.py:239
        self.zone = (None, False, False)                       # settings["coords"], settings["outside"], non-zone alert
        self.events = ObjectEvents(classes=classes)            # host rows' events (pred_occs, object_set, object_set_zone)
        self.alerts = CameraAlerts()                           # host rows' alerts and the settings of every alert
        self.alert_ids: list = []                              # the alerts' ids, in order (alert_counters[cam]'s keys)

    def fresh_events(self):
        self.events = ObjectEvents(*self.zone, classes=self.classes)


class CameraBatch:
    def __init__(self, model, max_age: int = 100):
        """model: a clearcam_b200 YOLOv9 (anything with detect_batch(frames[B,H,W,3]) -> (B,300,6); for yuv420p cameras
        also detect_batch(frames[B,H*3/2,W], pix_fmt="yuv420p")).  When it also has net_shape(H, W, pix_fmt=...) and
        detect_frames(frames, pix_fmts=...), uint8 cameras of different shapes and formats share calls (module doc)."""
        self.model, self.max_age = model, max_age
        self.cams: Dict[Hashable, _Camera] = {}
        self._stage: Dict[tuple, tuple] = {}                   # (H,W,dtype,pix_fmt,bucket) -> (device frame batch, pinned rows)
        self._pin = torch.cuda.is_available()
        self._seen: Dict[Hashable, int] = {}                   # last frame_num taken from each camera's mailbox
        self._where: Dict[Hashable, tuple] = {}                # camera -> (device batch, row) of its frame in the last detect()
        self._tables = hasattr(model, "net_shape") and hasattr(model, "detect_frames")
        self._net: Dict[tuple, tuple] = {}                     # (H,W,dtype,pix_fmt) -> (net_h, net_w)
        self._cam_dev: Dict[Hashable, torch.Tensor] = {}       # camera -> its device frame buffer (merged groups)
        self._table_rows: Dict[tuple, torch.Tensor] = {}       # (net_h, net_w, chunk, bucket) -> pinned rows
        self._dev_trk: Optional[ocsort.DeviceTrackers] = None  # device trackers, made on the first step with device rows
        self._desc: Dict[str, np.ndarray] = {}                 # description text -> its CLIP text embedding (D,) float32
        self._jpeg = None                                      # ops.JpegDecoder of the MJPEG cameras, made on first use
        self.dropped_frames: Dict[Hashable, int] = {}          # MJPEG frames neither the GPU nor cv2 could decode, per camera

    # -- camera set (clearcam.py:207-240 init_cam; settings threshold :584, class filter :586)
    def add_camera(self, name, thresh: float = 0.5, classes=None, pix_fmt: str = BGR24):
        """pix_fmt: the format of this camera's frames, "bgr24" [H,W,3], "yuv420p" [H*3/2,W] or "mjpeg" (one JPEG file per
        frame) (clearcam_b200/pixfmt.py)."""
        self.cams[name] = _Camera(thresh or 0.5, None if classes is None else {int(c) for c in classes}, self.max_age,
                                  check_camera_pix_fmt(pix_fmt))

    def remove_camera(self, name):
        self.cams.pop(name, None)
        if self._dev_trk is not None:
            self._dev_trk.remove(name)
        self._where.pop(name, None)
        self._cam_dev.pop(name, None)
        self._drop_run_frames(name, 0)
        self._seen.pop(name, None)             # a re-added camera starts a new mailbox whose frame_num restarts at 0
        self.dropped_frames.pop(name, None)

    def _drop_run_frames(self, name, T):
        """Forget camera `name`'s per-frame device buffers of step_video (keys (name, f)) for frames f >= T."""
        for d in (self._where, self._cam_dev):
            for key in [k for k in d if isinstance(k, tuple) and len(k) == 2 and k[0] == name and k[1] >= T]:
                del d[key]

    def reset_tracker(self, name):
        """A fresh tracker and fresh events for camera `name`, as init_cam makes them."""
        self.cams[name].tracker = ocsort.OCSort(max_age=self.max_age)
        self.cams[name].fresh_events()
        self.cams[name].alerts.reset()                         # init_cam: a fresh object counter and warm-up
        if self._dev_trk is not None and name in self._dev_trk:
            self._dev_trk.reset(name)
        self._seen.pop(name, None)

    def set_zone(self, name, zone=None, outside: bool = False, non_zone_alert: bool = False):
        """Camera `name`'s zone for `step_events`: settings["coords"] (fractions of the frame; None for no zone),
        settings["outside"] and whether any of its alerts has no zone (clearcam.py:599-610).  Its event state (which ids
        were saved, counted and alerted on) starts afresh.  non_zone_alert replaces what `set_alerts` derived, so pass
        the current value (any(not a.zone for a in alerts)) when the camera has alerts."""
        cam = self.cams[name]
        cam.zone = (zone, outside, non_zone_alert)
        cam.fresh_events()                                     # checks the arguments
        if self._dev_trk is not None and name in self._dev_trk:
            self._dev_trk.events(name, zone, outside, non_zone_alert, cam.classes)

    # -- alerts (clearcam.py RollingClassCounter :47-103, alert_counters[cam], alerts_on[cam])
    def set_alerts(self, name, alerts, finder=None):
        """Camera `name`'s alerts: {id: alert} in order (alert_counters[cam]), each an alerts.Alert or a reference
        RollingClassCounter (Alert.from_counter).  Descriptions not seen before are encoded in one
        `encode_text_batch` call of the finder's CLIP model (finder: an ObjectFinder with CLIP initialised).  Alerts whose id and settings are unchanged keep their counts
        and last_det; new or changed ones start empty at their own last_det.  The camera's non_zone_alert (set_zone)
        becomes whether any alert has no zone, without starting its event state afresh (a later `set_zone` sets it
        again from its own argument).  The object counter and the warm-up stay."""
        cam = self.cams[name]
        items = list(alerts.items())
        al = [a if isinstance(a, Alert) else Alert.from_counter(a) for _, a in items]
        ids = [k for k, _ in items]
        new = sorted({a.desc for a in al if a.desc is not None and a.desc not in self._desc})
        if new:
            clip = getattr(finder, "model", finder)           # an ObjectFinder's CLIP model, or a CLIP model itself
            if clip is None:
                raise ValueError("description alerts need a finder with CLIP initialised to encode their text")
            t = clip.encode_text_batch(new)
            t = getattr(t, "tensor", t)
            t = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
            for text, row in zip(new, np.asarray(t, np.float32)):
                self._desc[text] = row
        desc_emb = None
        if any(a.desc is not None for a in al):
            D = len(next(self._desc[a.desc] for a in al if a.desc is not None))
            desc_emb = np.stack([self._desc[a.desc] if a.desc is not None else np.zeros(D, np.float32) for a in al])
        old = {k: i for i, k in enumerate(cam.alert_ids)}
        keep = [old[k] if k in old and cam.alerts.alerts[old[k]].settings() == a.settings() else -1 for k, a in zip(ids, al)]
        cam.alerts.replace(al, desc_emb, keep)
        dev = self._dev_trk is not None and name in self._dev_trk
        if dev and self._dev_trk.has_alerts(name):
            self._dev_trk.alerts(name, al, desc_emb, keep)
        cam.alert_ids = ids
        nza = any(not a.zone for a in al)
        cam.zone = cam.zone[:2] + (nza,)
        cam.events.non_zone_alert = nza
        if dev and self._dev_trk.has_events(name):
            self._dev_trk.set_non_zone_alert(name, nza)

    def set_alerts_on(self, name, on: bool):
        """The reference's alerts_on[cam]: False makes every alert of the camera inactive."""
        cam = self.cams[name]
        cam.alerts.alerts_on = bool(on)
        if self._dev_trk is not None and self._dev_trk.has_alerts(name):
            self._dev_trk.set_alerts_on(name, bool(on))

    def alerting(self, now: Optional[float] = None, local=None) -> List[Hashable]:
        """The cameras process_frame runs the detector for (clearcam.py:447): those with an active alert at local time
        `local` ((seconds of day, weekday); time.localtime(now) when None)."""
        if local is None:
            local = local_time(time.time() if now is None else float(now))
        return [name for name, cam in self.cams.items() if cam.alerts.active(local).any()]

    def object_counts(self, name) -> np.ndarray:
        """Camera `name`'s object counter (self.counter[cam], /get_counts): int64 [80], the new ids per class id."""
        if self._dev_trk is not None and self._dev_trk.has_alerts(name):
            return self._dev_trk.counts(name)
        return self.cams[name].alerts.counter.copy()

    def reset_object_counts(self, name):
        """/reset_counts (clearcam.py:512-517)."""
        self.cams[name].alerts.counter[:] = 0
        if self._dev_trk is not None and self._dev_trk.has_alerts(name):
            self._dev_trk.reset_counts(name)

    def describe_saves(self, saved: Dict[Hashable, tuple], now: Optional[float] = None, local=None) -> Dict[Hashable, list]:
        """clip_latest_img's description alerts (clearcam.py:1289-1307) on what `save_objects` returned, in save order,
        at clock `now` (time.time() when None) and local time `local` (time.localtime(now) when None) ->
        {camera: [(save index, alert id, similarity)]} of the alerts that fired.  Cameras stepped on the GPU are matched in
        one launch per CC_MAX_FRAMES cameras on the device embeddings, the others by CameraAlerts.  A run's saves (from
        `step_video`) are matched frame by frame, each at its own clock: pass now={camera: the run's clocks, one per frame} and
        local=None (time.localtime of each) or {camera: one local time per frame}; with a dict `now`, cameras with a single
        step's saves are matched at time.time()."""
        runs_now, runs_local = now, local
        if isinstance(now, dict):
            now, local = None, None
        now = time.time() if now is None else float(now)
        if local is None:
            local = local_time(now)
        out = {name: [] for name in saved}
        dev, host = [], []
        runs, hruns = [], []
        for name, (saves, _, emb) in saved.items():
            if emb is None or len(saves) == 0 or not self.cams[name].alerts.alerts:
                continue
            t = getattr(emb, "tensor", emb)
            on_dev = isinstance(t, torch.Tensor) and t.is_cuda and self._dev_trk is not None and self._dev_trk.has_alerts(name)
            if np.asarray(saves).shape[1] == 7:                # a run's saves: each frame at its own clock (step_video)
                if not isinstance(runs_now, dict) or name not in runs_now:
                    raise ValueError(f"camera {name!r}: a run's saves need now={{camera: one clock per frame of the run}}")
                clocks = [float(t) for t in runs_now[name]]
                locs = ([local_time(t) for t in clocks] if runs_local is None
                        else [(float(a), int(d)) for a, d in runs_local[name]])
                if len(locs) != len(clocks) or int(np.asarray(saves)[:, 0].max()) >= len(clocks):
                    raise ValueError(f"camera {name!r}: one clock and one local time per frame of the run")
                rows = np.bincount(np.asarray(saves)[:, 0], minlength=len(clocks)).tolist()
                (runs if on_dev else hruns).append((name, t, rows, clocks, locs))
                continue
            (dev if on_dev else host).append((name, t))
        if runs:
            emb = torch.cat([t.float() for _, t, _, _, _ in runs]).contiguous()
            res = self._dev_trk.describe_runs([(name, rows) for name, _, rows, _, _ in runs], emb, [c for _, _, _, c, _ in runs],
                                              [lc for _, _, _, _, lc in runs])
            for (name, _, _, _, _), (hit, sim) in zip(runs, res):
                ids = self.cams[name].alert_ids
                out[name] = [(s, ids[a], float(sim[s, a])) for s, a in enumerate(hit.tolist()) if a >= 0]
        for name, t, rows, clocks, locs in hruns:
            e = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
            ids, r0 = self.cams[name].alert_ids, 0
            for n, c, lc in zip(rows, clocks, locs):
                out[name] += [(r0 + s, ids[a], v) for s, a, v in self.cams[name].alerts.describe(e[r0:r0 + n], c, lc)]
                r0 += n
        if dev:
            emb = torch.cat([t.float() for _, t in dev]).contiguous()
            res = self._dev_trk.describe([(name, t.shape[0]) for name, t in dev], emb, [now] * len(dev), [local] * len(dev))
            for (name, _), (hit, sim) in zip(dev, res):
                ids = self.cams[name].alert_ids
                out[name] = [(s, ids[a], float(sim[s, a])) for s, a in enumerate(hit.tolist()) if a >= 0]
        for name, t in host:
            e = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
            ids = self.cams[name].alert_ids
            out[name] = [(s, ids[a], v) for s, a, v in self.cams[name].alerts.describe(e, now, local)]
        return out

    bucket = staticmethod(batch_bucket)   # group sizes are padded to a small set of batch sizes (bounded plan count)

    # -- one pass over every camera that has a new frame
    @staticmethod
    def group_by_shape(frames: Dict[Hashable, np.ndarray], pix_fmts: Optional[Dict[Hashable, str]] = None
                       ) -> Dict[tuple, List[Hashable]]:
        """{camera: frame} -> {(H, W, dtype, pix_fmt): cameras}; H, W in pixels.  pix_fmts: each camera's format (missing
        cameras are bgr24).  A frame that does not match its camera's format raises ValueError."""
        groups: Dict[tuple, List[Hashable]] = {}
        for name, f in frames.items():
            if f is None:
                continue
            fmt = (pix_fmts or {}).get(name, BGR24)
            if not hasattr(f, "dtype"):
                raise ValueError(f"camera {name!r}: a {fmt} frame must be an array, got {type(f).__name__}")
            dt = {torch.uint8: "|u1", torch.float32: "<f4"}.get(f.dtype) if isinstance(f, torch.Tensor) else \
                (f.dtype.str if f.dtype in (np.uint8, np.float32) else None)
            if fmt == BGR24:
                if f.ndim != 3 or f.shape[2] != 3 or dt is None:
                    raise ValueError(f"camera {name!r}: frame must be HWC BGR uint8 or float32, got {f.dtype} {tuple(f.shape)}")
                H, W = int(f.shape[0]), int(f.shape[1])
            else:
                if f.ndim != 2 or dt != "|u1":
                    raise ValueError(f"camera {name!r}: a yuv420p frame must be uint8 [H*3/2,W], got {f.dtype} {tuple(f.shape)}")
                try:
                    H, W = yuv420p_size(f.shape)
                except ValueError as ex:
                    raise ValueError(f"camera {name!r}: {ex}") from None
            groups.setdefault((H, W, dt, fmt), []).append(name)
        return groups

    def _buffers(self, key, n):
        k = key + (self.bucket(n),)
        if k not in self._stage:
            H, W, dt, fmt = key
            tdt = torch.uint8 if np.dtype(dt) == np.uint8 else torch.float32
            dev = "cuda" if self._pin else "cpu"
            shape = (H, W, 3) if fmt == BGR24 else (H * 3 // 2, W)
            self._stage[k] = (torch.zeros((k[-1],) + shape, dtype=tdt, device=dev),
                              torch.empty((k[-1], 300, 6), dtype=torch.float32, pin_memory=self._pin))
        return self._stage[k]

    def merge_groups(self, groups: Dict[tuple, List[Hashable]]) -> List[tuple]:
        """Shape groups -> [(net shape or None, [shape keys])]: with frame tables, the uint8 groups of one net shape go
        together; float32 groups (and every group without frame tables) stay alone with net shape None."""
        merged: Dict[tuple, tuple] = {}
        for key in groups:
            H, W, dt, fmt = key
            if not self._tables or dt != "|u1":
                merged[("shape",) + key] = (None, [key])
                continue
            if key not in self._net:
                self._net[key] = tuple(self.model.net_shape(H, W, pix_fmt=fmt))
            net = self._net[key]
            merged.setdefault(("net",) + net, (net, []))[1].append(key)
        return list(merged.values())

    def _camera_buffer(self, name, f) -> torch.Tensor:
        buf = self._cam_dev.get(name)
        if buf is None or tuple(buf.shape) != tuple(f.shape):
            buf = self._cam_dev[name] = torch.empty(tuple(f.shape), dtype=torch.uint8, device="cuda" if self._pin else "cpu")
        return buf

    def detect(self, frames: Dict[Hashable, np.ndarray]) -> Dict[Hashable, np.ndarray]:
        """Detector only: {camera: HWC frame} -> {camera: (300,6) rows}.  One batched call per distinct frame shape, or
        with frame tables per distinct net shape (module doc).
        Each frame goes host -> its row of the device batch (or its camera's device buffer) directly (asynchronously when it
        lives in pinned memory, e.g. a FrameMailbox slot): no host-side stacking copy."""
        pending = self._launch(frames)
        if self._pin:
            torch.cuda.current_stream().synchronize()
        return {name: rows[i].numpy().copy() for names, rows, _ in pending for i, name in enumerate(names) if name is not None}

    def _launch(self, frames, fmts=None, run=False) -> list:
        """Queue every detector call of `detect` and the copies of its rows to the host: [(cameras, host rows, detector
        output)], a camera None where its MJPEG frame was dropped.  fmts: each frame's pixel format when the keys of
        `frames` are not camera names (its camera's by default).  run: the frames are a step_video run, in which a frame
        that cannot be decoded raises ValueError."""
        pending = []
        if fmts is None:
            fmts = {name: cam.pix_fmt for name, cam in self.cams.items() if cam.pix_fmt != BGR24}
        frames, fmts, jpeg, staged = self._stage_jpeg(frames, fmts, run)
        groups = self.group_by_shape(frames, fmts)
        calls = []                             # placed first, so that MJPEG frames are decoded before any detector call
        for net, keys in self.merge_groups(groups):
            if len(keys) > 1:
                calls += self._detect_table(net, [(name, key[3]) for key in keys for name in groups[key]], frames, jpeg)
                continue
            key = keys[0]
            names = groups[key]
            dev, rows = self._buffers(key, len(names))
            for i, name in enumerate(names):
                self._where[name] = (dev, i)
                if name in jpeg:
                    jpeg[name] = dev[i]
                    continue
                f = frames[name]
                dev[i].copy_(f if isinstance(f, torch.Tensor) else torch.from_numpy(f), non_blocking=True)

            def call(names=names, dev=dev, rows=rows, fmt=key[3], dropped=()):
                # bgr24 groups call detect_batch exactly as before the format existed (stand-in models need not know it)
                out = self.model.detect_batch(dev) if fmt == BGR24 else self.model.detect_batch(dev, pix_fmt=fmt)
                rows.copy_(out, non_blocking=True)
                return [([None if n in dropped else n for n in names], rows, out)]
            calls.append(call)
        dropped = self._decode_jpeg(jpeg, staged, run) if jpeg else set()
        for c in calls:
            pending += c(dropped=dropped)
        return pending

    def _stage_jpeg(self, frames, fmts, run):
        """The first half of the decode stage (module doc): gather and parse every MJPEG frame -> (frames, formats, {frame
        key: None}, (staged frame keys, their files)): MJPEG frames the GPU decodes become meta [H,W,3] placeholders and
        the others cv2.imdecode's host pictures, all bgr24; frames cv2 rejects are left out (in a run: ValueError, before
        anything is queued on the device)."""
        keys = [k for k, f in frames.items() if f is not None and fmts.get(k) == MJPEG]
        if not keys:
            return frames, fmts, {}, None
        frames, fmts = dict(frames), dict(fmts)
        files = []
        for k in keys:
            f = frames[k]
            if isinstance(f, torch.Tensor):
                ok = f.dtype == torch.uint8 and f.dim() == 1 and not f.is_cuda
            elif isinstance(f, np.ndarray):
                ok = f.dtype == np.uint8 and f.ndim == 1
            else:
                ok = isinstance(f, (bytes, bytearray, memoryview))
            if not ok:
                raise ValueError(f"camera {k!r}: an mjpeg frame is one JPEG file (bytes-like or a 1-D uint8 host array)")
            files.append(f.numpy() if isinstance(f, torch.Tensor) else f)
            fmts[k] = BGR24
        jpeg = {}
        if self._pin:
            from . import ops
            from .ingest import default_tables
            if self._jpeg is None:
                self._jpeg = ops.JpegDecoder()
            ins = [default_tables(f) for f in files]
            sizes, status = self._jpeg.stage(files, [i if i[1] else None for i in ins])
        for i, k in enumerate(keys):
            if self._pin and status[i] == 0:
                frames[k] = torch.empty((int(sizes[i, 1]), int(sizes[i, 0]), 3), dtype=torch.uint8, device="meta")
                jpeg[k] = None
                continue
            img = self._imdecode(files[i])
            if img is None:
                self._drop(k, run)
                del frames[k]
            else:
                frames[k] = img
        return frames, fmts, jpeg, (keys, files)

    @staticmethod
    def _imdecode(f):
        import cv2
        a = f if isinstance(f, np.ndarray) else np.frombuffer(f, np.uint8)
        return cv2.imdecode(a, cv2.IMREAD_COLOR) if len(a) else None

    def _drop(self, key, run):
        name = key[0] if run else key
        if run:
            raise ValueError(f"camera {name!r}: frame {key[1]} of the run is not a JPEG file cv2 can decode")
        self.dropped_frames[name] = self.dropped_frames.get(name, 0) + 1
        self._where.pop(name, None)

    def _decode_jpeg(self, jpeg, staged, run) -> set:
        """The second half of the decode stage: one decode into the placed buffers, the status wait, cv2 for the frames
        the device left -> the frame keys dropped.  In a run, a frame cv2 rejects after the device did raises ValueError
        here: the uploads and the decode are then queued, but no detector, tracker or event state has changed."""
        keys, files = staged
        dests = [jpeg.get(k) for k in keys]
        status = self._jpeg.decode(dests)
        torch.cuda.current_stream().synchronize()
        dropped = set()
        for i, k in enumerate(keys):
            if dests[i] is None or int(status[i]) == 0:
                continue
            img = self._imdecode(files[i])
            if img is None or tuple(img.shape) != tuple(dests[i].shape):
                self._drop(k, run)
                dropped.add(k)
                continue
            dests[i].copy_(torch.from_numpy(img))
        return dropped

    def _detect_table(self, net, cams, frames, jpeg) -> list:
        """Place the frames of one net shape in their cameras' buffers (an MJPEG frame's buffer goes to `jpeg` for the
        decode) -> one call per CC_MAX_FRAMES cameras, each queueing one detect_frames call; cams: [(camera, pix_fmt)]."""
        calls = []
        for c0 in range(0, len(cams), CC_MAX_FRAMES):
            chunk = cams[c0:c0 + CC_MAX_FRAMES]
            devs = []
            for name, _ in chunk:
                f = frames[name]
                buf = self._camera_buffer(name, f)
                if name in jpeg:
                    jpeg[name] = buf
                else:
                    buf.copy_(f if isinstance(f, torch.Tensor) else torch.from_numpy(f), non_blocking=True)
                self._where[name] = (buf.unsqueeze(0), 0)
                devs.append(buf)

            def call(chunk=chunk, devs=devs, c0=c0, dropped=()):
                names = [None if name in dropped else name for name, _ in chunk]
                b = self.bucket(len(chunk))
                out = self.model.detect_frames([d if n is not None else None for d, n in zip(devs, names)] + [None] * (b - len(chunk)),
                                               pix_fmts=[fmt for _, fmt in chunk] + [BGR24] * (b - len(chunk)))
                k = tuple(net) + (c0 // CC_MAX_FRAMES, b)
                if k not in self._table_rows:
                    self._table_rows[k] = torch.empty((b, 300, 6), dtype=torch.float32, pin_memory=self._pin)
                rows = self._table_rows[k]
                rows.copy_(out, non_blocking=True)
                return [(names, rows, out)]
            calls.append(call)
        return calls

    def device_frame(self, name) -> torch.Tensor:
        """The device copy of the frame camera `name` contributed to the last detect()/step(), in the camera's own format
        ([H,W,3] bgr24 or [H*3/2,W] yuv420p; an MJPEG camera's is the bgr24 [H,W,3] picture of its file) — what the object crops for CLIP are cut from
        (ObjectFinder.embed_crops(..., pix_fmt=...)) without a second upload.  Valid until the next step."""
        dev, i = self._where[name]
        return dev[i]

    def save_objects(self, results: Dict[Hashable, CameraEvents], finder, quality: int = 95) -> Dict[Hashable, tuple]:
        """The thumbnails and embeddings of every camera's object saves of the last step in ONE call (`save_object` and
        `clip_latest_img`, clearcam.py:373-399, 272-279, 1278-1287): results is what `step_events` /
        `step_events_mailboxes` returned, or what `step_video` returned (a list per camera); every camera's saves[:, 2:6]
        are cut from its `device_frame` — for a run, from the device copy of the save's own frame — in its own pixel format
        by one `finder.encode_embed_frames` call -> {camera: (saves, files, embeddings)}, files and embedding rows in saves
        order (embeddings None when CLIP is not initialised, or when the camera has no saves).  A run's saves are (m,7):
        the frame index in the run, then the six save columns, frame after frame.  A step without saves makes no library
        call.  Reads the device frames of the last step, so it is valid until the next step."""
        # (camera, frame key, saves): a step's result is one frame; a step_video result (a list) one per frame of the run,
        # whose saves are returned with their frame index in front
        srcs, out = [], {}
        for name, ev in results.items():
            if isinstance(ev, list):
                for f, e in enumerate(ev):
                    if len(e.saves):
                        srcs.append((name, (name, f), e.saves))
                out[name] = (np.concatenate([np.concatenate([np.full((len(e.saves), 1), f, np.int64), np.asarray(e.saves, np.int64)
                                                             .reshape(-1, 6)], 1) for f, e in enumerate(ev)]).reshape(-1, 7), [], None)
            else:
                if len(ev.saves):
                    srcs.append((name, name, ev.saves))
                out[name] = (ev.saves, [], None)
        if not srcs:
            return out
        frames = [self.device_frame(key) for _, key, _ in srcs]
        rects = np.concatenate([np.concatenate([np.full((len(sv), 1), j, np.int64), np.asarray(sv, np.int64)[:, 2:6]], 1)
                                for j, (_, _, sv) in enumerate(srcs)]).astype(np.int32)
        files, emb = finder.encode_embed_frames(frames, [self._device_fmt(name) for name, _, _ in srcs], rects, quality)
        from .detection.yolov9 import DeviceResult
        k, first = 0, {}
        for name, _, sv in srcs:
            first.setdefault(name, k)
            k += len(sv)
        for name, k0 in first.items():
            n = len(out[name][0])
            out[name] = (out[name][0], files[k0:k0 + n], None if emb is None else DeviceResult(emb.tensor[k0:k0 + n]))
        return out

    def step_mailboxes(self, mailboxes: Dict[Hashable, "FrameMailbox"]) -> Dict[Hashable, CameraResult]:
        """`step` on every camera whose mailbox (clearcam_b200.ingest) holds a frame this object has not seen yet —
        the reference's `if frame_num == last_frame_num: return` per camera (clearcam.py:446).  A camera seen here for
        the first time is added with its mailbox's pixel format."""
        frames = self._from_mailboxes(mailboxes)
        return self.step(frames) if frames else {}

    def step_events_mailboxes(self, mailboxes: Dict[Hashable, "FrameMailbox"], now: Optional[float] = None
                              ) -> Dict[Hashable, CameraEvents]:
        """`step_events` on the cameras whose mailboxes hold a new frame (as `step_mailboxes`)."""
        frames = self._from_mailboxes(mailboxes)
        return self.step_events(frames, now) if frames else {}

    def step_alerts_mailboxes(self, mailboxes: Dict[Hashable, "FrameMailbox"], now: Optional[float] = None, local=None
                              ) -> Dict[Hashable, CameraAlertResult]:
        """`step_alerts` on the cameras whose mailboxes hold a new frame (as `step_mailboxes`)."""
        frames = self._from_mailboxes(mailboxes)
        return self.step_alerts(frames, now, local) if frames else {}

    def step_alerts(self, frames: Dict[Hashable, np.ndarray], now: Optional[float] = None, local=None
                    ) -> Dict[Hashable, CameraAlertResult]:
        """`step_events`, then each camera's alerts (clearcam_b200/alerts.py) at clock `now` and local time `local`
        ((seconds of day, weekday with 0 = Monday); time.localtime(now) when None) -> {camera: CameraAlertResult}.
        Device rows run the alerts on the GPU right after the events, before the step's one wait; host rows run
        `CameraAlerts`.  Which cameras to step is the caller's (`alerting`, the gate of clearcam.py:447)."""
        now = time.time() if now is None else float(now)
        return self._step(frames, now, local_time(now) if local is None else (float(local[0]), int(local[1])))

    def _from_mailboxes(self, mailboxes):
        frames = {}
        for name, mb in mailboxes.items():
            got = mb.latest(self._seen.get(name, -1))
            if got is not None:
                if name not in self.cams:
                    self.add_camera(name, pix_fmt=getattr(mb, "pix_fmt", BGR24))
                self._seen[name], frames[name] = got
        return frames

    def step(self, frames: Dict[Hashable, np.ndarray]) -> Dict[Hashable, CameraResult]:
        return self._step(frames, None)

    def step_events(self, frames: Dict[Hashable, np.ndarray], now: Optional[float] = None) -> Dict[Hashable, CameraEvents]:
        """`step`, then each camera's object events (clearcam.py:586-621, clearcam_b200/events.py) at clock `now`
        (time.time() when None; one reading for the whole step) -> {camera: CameraEvents}.  Device rows run the events on
        the GPU right after the trackers, before the step's one wait; host rows run `ObjectEvents`.  A camera's frame
        size is its picture's (a yuv420p frame [H*3/2,W] is W x H)."""
        return self._step(frames, time.time() if now is None else float(now))

    def step_video(self, frames: Dict[Hashable, object], clocks: Dict[Hashable, object], local=None
                   ) -> Dict[Hashable, List[CameraAlertResult]]:
        """`step_alerts` over runs of consecutive frames: frames {camera: [T,H,W,3] bgr24 or [T,H*3/2,W] yuv420p frames of
        one video, in order}, clocks {camera: T clocks}, local None (time.localtime of each clock) or {camera: T (seconds
        of day, weekday)} -> {camera: [CameraAlertResult per frame]}, what T successive `step_alerts` calls with those
        clocks would return.  Every frame of every camera goes through the detector grouping of `step` (one detect_batch
        per shape, or frame tables of at most CC_MAX_FRAMES frames per net shape); device rows then run one launch per stage
        (tracker, events, alerts) for all cameras and one wait, host rows the host objects frame by frame.  A video camera
        is a normal camera: `step` and `step_video` may alternate on it.  An "mjpeg" camera's run is a list of JPEG files;
        a file neither the GPU nor cv2 can decode raises ValueError before any detector call and leaves every camera's
        tracker, events and alerts as they were (when the device found the fault, the decode had already been queued)."""
        flat, runs = {}, {}
        for name, fr in frames.items():
            if name not in self.cams:
                self.add_camera(name)
            T = len(fr)
            if not 1 <= T <= CC_MAX_FRAMES:
                raise ValueError(f"camera {name!r}: {T} frames (1..{CC_MAX_FRAMES} per run)")
            c = [float(t) for t in clocks[name]]
            if len(c) != T or not all(np.isfinite(c)):
                raise ValueError(f"camera {name!r}: one finite clock per frame")
            lc = [local_time(t) for t in c] if local is None else [(float(a), int(d)) for a, d in local[name]]
            if len(lc) != T:
                raise ValueError(f"camera {name!r}: one local time per frame")
            runs[name] = (T, c, lc)
            for f in range(T):
                flat[(name, f)] = fr[f]
        fmts = {(name, f): self.cams[name].pix_fmt for name, (T, _, _) in runs.items() for f in range(T)}
        pending = self._launch(flat, fmts, run=True)
        for name, (T, _, _) in runs.items():
            self._drop_run_frames(name, T)     # buffers of a longer earlier run
        size = {name: self._picture_size(name, frames[name][0], (name, 0)) for name in runs}
        on_device = bool(pending) and all(isinstance(out, torch.Tensor) and out.is_cuda for _, _, out in pending)
        if on_device:
            if self._dev_trk is None:
                self._dev_trk = ocsort.DeviceTrackers()
            for n in runs:
                self._device_camera(n, True, True)
            where = {key: (out, i) for keys, _, out in pending for i, key in enumerate(keys)}
            jobs = [(n, torch.stack([where[(n, f)][0][where[(n, f)][1]] for f in range(T)]), self.cams[n].thresh)
                    for n, (T, _, _) in runs.items()]
            launched = self._dev_trk.launch_runs(jobs, [[size[n] + (t,) for t in c] for n, (_, c, _) in runs.items()],
                                                 [lc for _, _, lc in runs.values()])
        if self._pin:
            torch.cuda.current_stream().synchronize()
        det = {key: rows[i].numpy().copy() for keys, rows, _ in pending for i, key in enumerate(keys) if key is not None}
        res = {}
        if on_device:
            for n, per in zip(runs, self._dev_trk.finish_runs(launched)):
                ids = self.cams[n].alert_ids
                res[n] = [CameraAlertResult(det[(n, f)], p, fl, s, [ids[i] for i in fired.tolist()]) for f, (p, fl, s, fired) in enumerate(per)]
            return res
        for n, (T, c, lc) in runs.items():
            cam, res[n] = self.cams[n], []
            for f in range(T):
                [tg] = ocsort.update_many([cam.tracker], det[(n, f)][None], [cam.thresh])
                ev = cam.events.update(tg, *size[n], c[f])
                fired = cam.alerts.step(ev[0], ev[1], c[f], lc[f])
                res[n].append(CameraAlertResult(det[(n, f)], *ev, [cam.alert_ids[i] for i in fired]))
        return res

    def _device_fmt(self, name):
        fmt = self.cams[name].pix_fmt
        return BGR24 if fmt == MJPEG else fmt

    def _picture_size(self, name, f, key=None):
        if self.cams[name].pix_fmt == MJPEG:
            f = self.device_frame(name if key is None else key)
        if self._device_fmt(name) == BGR24:
            return int(f.shape[1]), int(f.shape[0])
        H, W = yuv420p_size(f.shape)
        return W, H

    def _device_camera(self, n, events: bool, alerts: bool):
        """Camera n's device tracker, and its device events and alerts when the step runs them, made on first use."""
        if n not in self._dev_trk:
            self._dev_trk.add(n, max_age=self.max_age)
        if events and not self._dev_trk.has_events(n):
            self._dev_trk.events(n, *self.cams[n].zone, self.cams[n].classes)
        if alerts and not self._dev_trk.has_alerts(n):
            al = self.cams[n].alerts
            self._dev_trk.alerts(n, [a._replace(last_det=t) for a, t in zip(al.alerts, al.last_det)], al.desc_emb)
            if not al.alerts_on:
                self._dev_trk.set_alerts_on(n, False)

    def _step(self, frames, now, local=None):
        for name in frames:
            if name not in self.cams:
                self.add_camera(name)
        pending = self._launch(frames)
        on_device = bool(pending) and all(isinstance(out, torch.Tensor) and out.is_cuda for _, _, out in pending)
        if on_device:                          # track on the GPU, queued before the one wait below
            if self._dev_trk is None:
                self._dev_trk = ocsort.DeviceTrackers()
            for names, _, _ in pending:
                for n in names:
                    if n is not None:
                        self._device_camera(n, now is not None, local is not None)
            jobs = [(n, out[i], self.cams[n].thresh) for names, _, out in pending for i, n in enumerate(names) if n is not None]
            launched = self._dev_trk.launch(jobs, None if now is None else
                                            [self._picture_size(n, frames[n]) + (now,) for n, _, _ in jobs],
                                            None if local is None else [local] * len(jobs))
        if self._pin:
            torch.cuda.current_stream().synchronize()
        det = {name: rows[i].numpy().copy() for names, rows, _ in pending for i, name in enumerate(names) if name is not None}
        names = list(det)
        if not names:
            return {}
        if on_device:
            if local is not None:
                return {name: CameraAlertResult(det[name], p, f, s, [self.cams[name].alert_ids[i] for i in fired.tolist()])
                        for name, (p, f, s, fired) in zip(names, self._dev_trk.finish_alerts(launched))}
            if now is not None:
                return {name: CameraEvents(det[name], *e) for name, e in zip(names, self._dev_trk.finish_events(launched))}
            targets = self._dev_trk.finish(launched)
        else:
            targets = ocsort.update_many([self.cams[n].tracker for n in names], np.stack([det[n] for n in names]),
                                         [self.cams[n].thresh for n in names])
        res = {}
        for name, tg in zip(names, targets):
            cam = self.cams[name]
            if now is not None:
                ev = cam.events.update(tg, *self._picture_size(name, frames[name]), now)
                if local is not None:
                    fired = cam.alerts.step(ev[0], ev[1], now, local)
                    res[name] = CameraAlertResult(det[name], *ev, [cam.alert_ids[i] for i in fired])
                else:
                    res[name] = CameraEvents(det[name], *ev)
                continue
            if cam.classes is not None:
                tg = [t for t in tg if int(t.class_id) in cam.classes]                       # clearcam.py:586
            keep = [t for t in tg if t.tracklet_len >= 1]                                     # clearcam.py:589
            preds = np.array([[t.tlwh[0], t.tlwh[1], t.tlwh[0] + t.tlwh[2], t.tlwh[1] + t.tlwh[3], t.score, t.class_id, t.track_id]
                              for t in keep], np.float64).reshape(-1, 7)
            res[name] = CameraResult(det[name], tg, preds)
        return res
