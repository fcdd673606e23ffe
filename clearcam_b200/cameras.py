"""All cameras in one detector call (SURVEY.md §8f N1).

The reference walks its cameras round-robin and runs the detector on one frame at a time (`VideoCapture.start`,
clearcam.py:270-271 -> `process_frame` :423-461 -> `run_inference` :580-586: Tensor(frame) -> jit_infer(model) ->
.numpy() -> tracker.update).  On an H100 a single 1080p frame leaves the GPU mostly idle, so `CameraBatch.step` takes the
latest frame of every camera, groups the frames by shape (cameras differ in resolution; the detector's letterbox plan is
per input shape), runs ONE `detect_batch` per group with uploads and result reads queued back to back, waits once, and
then steps every camera's tracker in one library call.  What comes back per camera is what `run_inference` computes up
to clearcam.py:589 — the (300,6) detector rows and the tracker's targets; zones, alerts and clip saving (:590-621) are
the product's control plane and stay with the caller."""
from typing import Dict, Hashable, List, NamedTuple, Optional

import numpy as np
import torch

from .ocsort_tracker import ocsort
from .utils.helpers import batch_bucket
from .ocsort_tracker.STrack import STrack


class CameraResult(NamedTuple):
    rows: np.ndarray            # (300,6) float32 detector output in this camera's frame coordinates
    targets: List[STrack]       # tracker.update(rows, thresh), unfiltered (clearcam.py:585)
    preds: np.ndarray           # (k,7) x1,y1,x2,y2,score,class,track_id of targets seen for more than one frame


class _Camera:
    def __init__(self, thresh, classes, max_age):
        self.thresh, self.classes = thresh, classes
        self.tracker = ocsort.OCSort(max_age=max_age)          # clearcam.py:239


class CameraBatch:
    def __init__(self, model, max_age: int = 100):
        """model: a clearcam_b200 YOLOv9 (anything with detect_batch(frames[B,H,W,3]) -> (B,300,6))."""
        self.model, self.max_age = model, max_age
        self.cams: Dict[Hashable, _Camera] = {}
        self._stage: Dict[tuple, tuple] = {}                   # (H,W,dtype,bucket) -> (device frame batch, pinned rows)
        self._pin = torch.cuda.is_available()
        self._seen: Dict[Hashable, int] = {}                   # last frame_num taken from each camera's mailbox
        self._where: Dict[Hashable, tuple] = {}                # camera -> (device batch, row) of its frame in the last detect()

    # -- camera set (clearcam.py:207-240 init_cam; settings threshold :584, class filter :586)
    def add_camera(self, name, thresh: float = 0.5, classes=None):
        self.cams[name] = _Camera(thresh or 0.5, None if classes is None else {int(c) for c in classes}, self.max_age)

    def remove_camera(self, name):
        self.cams.pop(name, None)
        self._where.pop(name, None)
        self._seen.pop(name, None)             # a re-added camera starts a new mailbox whose frame_num restarts at 0

    def reset_tracker(self, name):
        self.cams[name].tracker = ocsort.OCSort(max_age=self.max_age)
        self._seen.pop(name, None)

    bucket = staticmethod(batch_bucket)   # group sizes are padded to a small set of batch sizes (bounded plan count)

    # -- one pass over every camera that has a new frame
    @staticmethod
    def group_by_shape(frames: Dict[Hashable, np.ndarray]) -> Dict[tuple, List[Hashable]]:
        groups: Dict[tuple, List[Hashable]] = {}
        for name, f in frames.items():
            if f is None:
                continue
            dt = {torch.uint8: "|u1", torch.float32: "<f4"}.get(f.dtype) if isinstance(f, torch.Tensor) else \
                (f.dtype.str if f.dtype in (np.uint8, np.float32) else None)
            if f.ndim != 3 or f.shape[2] != 3 or dt is None:
                raise ValueError(f"camera {name!r}: frame must be HWC BGR uint8 or float32, got {f.dtype} {tuple(f.shape)}")
            groups.setdefault((int(f.shape[0]), int(f.shape[1]), dt), []).append(name)
        return groups

    def _buffers(self, key, n):
        k = key + (self.bucket(n),)
        if k not in self._stage:
            H, W, dt = key
            tdt = torch.uint8 if np.dtype(dt) == np.uint8 else torch.float32
            dev = "cuda" if self._pin else "cpu"
            self._stage[k] = (torch.zeros((k[-1], H, W, 3), dtype=tdt, device=dev),
                              torch.empty((k[-1], 300, 6), dtype=torch.float32, pin_memory=self._pin))
        return self._stage[k]

    def detect(self, frames: Dict[Hashable, np.ndarray]) -> Dict[Hashable, np.ndarray]:
        """Detector only: {camera: HWC frame} -> {camera: (300,6) rows}.  One batched call per distinct frame shape.
        Each frame goes host -> its row of the device batch directly (asynchronously when it lives in pinned memory, e.g. a
        FrameMailbox slot): no host-side stacking copy."""
        pending = []
        for key, names in self.group_by_shape(frames).items():
            dev, rows = self._buffers(key, len(names))
            for i, name in enumerate(names):
                f = frames[name]
                dev[i].copy_(f if isinstance(f, torch.Tensor) else torch.from_numpy(f), non_blocking=True)
                self._where[name] = (dev, i)
            out = self.model.detect_batch(dev)
            rows.copy_(out, non_blocking=True)
            pending.append((names, rows))
        if self._pin:
            torch.cuda.current_stream().synchronize()
        return {name: rows[i].numpy().copy() for names, rows in pending for i, name in enumerate(names)}

    def device_frame(self, name) -> torch.Tensor:
        """The [H,W,3] device copy of the frame camera `name` contributed to the last detect()/step() — what the object
        crops for CLIP are cut from (ObjectFinder.embed_crops) without a second upload.  Valid until the next step."""
        dev, i = self._where[name]
        return dev[i]

    def step_mailboxes(self, mailboxes: Dict[Hashable, "FrameMailbox"]) -> Dict[Hashable, CameraResult]:
        """`step` on every camera whose mailbox (clearcam_b200.ingest) holds a frame this object has not seen yet —
        the reference's `if frame_num == last_frame_num: return` per camera (clearcam.py:446)."""
        frames = {}
        for name, mb in mailboxes.items():
            got = mb.latest(self._seen.get(name, -1))
            if got is not None:
                self._seen[name], frames[name] = got
        return self.step(frames) if frames else {}

    def step(self, frames: Dict[Hashable, np.ndarray]) -> Dict[Hashable, CameraResult]:
        for name in frames:
            if name not in self.cams:
                self.add_camera(name)
        det = self.detect(frames)
        names = list(det)
        if not names:
            return {}
        targets = ocsort.update_many([self.cams[n].tracker for n in names], np.stack([det[n] for n in names]),
                                     [self.cams[n].thresh for n in names])
        res = {}
        for name, tg in zip(names, targets):
            cam = self.cams[name]
            if cam.classes is not None:
                tg = [t for t in tg if int(t.class_id) in cam.classes]                       # clearcam.py:586
            keep = [t for t in tg if t.tracklet_len >= 1]                                     # clearcam.py:589
            preds = np.array([[t.tlwh[0], t.tlwh[1], t.tlwh[0] + t.tlwh[2], t.tlwh[1] + t.tlwh[3], t.score, t.class_id, t.track_id]
                              for t in keep], np.float64).reshape(-1, 7)
            res[name] = CameraResult(det[name], tg, preds)
        return res
