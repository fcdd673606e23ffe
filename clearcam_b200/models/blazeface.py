"""BlazeFace face detection on the H100: the reference's `BlazeFace` (models/blazeface.py:62-232) with the same call form.

    from clearcam_b200.models.blazeface import BlazeFace
    det = BlazeFace(weights)                 # state dict, .safetensors path, or None for the reference's models/blazeface.safetensors
    rows = det(img).numpy()                  # img: HWC uint8 -> (896,17) [ymin, xmin, ymax, xmax, 6 keypoints (x, y), score]
    dets = det.detect(images)                # many images of any sizes -> device [B,896,17], row b = det(images[b])
    first = first_detections(dets)           # device [B,17]: the one row img_to_face reads per image

The network, the decode and the suppression run in fp32 in libclearcam_b200.so (csrc/blazeface.cu); there is no CPU
fallback.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from .._lib import Handle, cc_face_warp, cc_frame, check, create, lib, ptr, stream_ptr
from ..detection.yolov9 import DeviceResult, _as_tensor, load_weights_arg
from ..pixfmt import CC_FRAME_BGR_U8

ANCHORS, COORDS = 896, 16
WEIGHTS_PATH = "models/blazeface.safetensors"          # models/blazeface.py:134, relative to the reference's working directory
FACE = 112
TARGET_LEFT_EYE = np.array([38, 51])
TARGET_RIGHT_EYE = np.array([73, 51])


def _images(images):
    """A uint8 [B,H,W,3] batch or a list of uint8 [h,w,3] images (numpy or torch, host or device) -> device tensors."""
    if isinstance(images, DeviceResult):
        images = images.tensor
    if isinstance(images, (torch.Tensor, np.ndarray)) and images.ndim == 4:
        t = images if isinstance(images, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(images))
        if t.dtype != torch.uint8 or t.shape[3] != 3 or min(t.shape) < 1:
            raise ValueError(f"images must be uint8 [B,h,w,3], got {t.dtype} {tuple(t.shape)}")
        t = t.to("cuda", non_blocking=True).contiguous()           # one copy; the images are views of it
        return list(t.unbind(0))
    out = []
    for i, im in enumerate(images):
        t = im.tensor if isinstance(im, DeviceResult) else im
        if not isinstance(t, torch.Tensor):
            t = torch.from_numpy(np.ascontiguousarray(t))
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError(f"image {i} must be uint8 [h,w,3], got {t.dtype} {tuple(t.shape)}")
        out.append(t.to("cuda", non_blocking=True).contiguous())
    if not out:
        raise ValueError("no images")
    return out


class BlazeFace(Handle):
    """models/blazeface.py:62-232.  `weights`: the reference's state dict (tensors or arrays under its key names, the
    anchors included), a .safetensors path, or None for the reference's relative path models/blazeface.safetensors."""
    _destroy = "cc_blazeface_destroy"

    def __init__(self, weights=None):
        weights = load_weights_arg(weights, WEIGHTS_PATH)
        self._adopt(create("cc_blazeface_create", lambda: weights))
        self._ws = None

    def _workspace(self, B: int) -> None:
        need = ctypes.c_size_t()
        check(lib().cc_blazeface_workspace_bytes(self._h, B, ctypes.byref(need)), "cc_blazeface_workspace_bytes")
        if self._ws is None or self._ws.numel() < need.value:
            torch.cuda.current_stream().synchronize()          # the old workspace may still be read by queued work
            self._ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
            check(lib().cc_blazeface_set_workspace(self._h, ptr(self._ws), self._ws.numel()), "cc_blazeface_set_workspace")

    def forward(self, images):
        """images: uint8 [B,H,W,3] or a list of uint8 [h,w,3] of any sizes -> device (dets [B,896,17], raw boxes [B,896,16],
        raw scores [B,896]) from one batched call; row b of dets is what `self(images[b])` returns."""
        ims = _images(images)
        B = len(ims)
        self._workspace(B)
        table = frame_table(ims)
        boxes = torch.empty(B, ANCHORS, COORDS, device="cuda", dtype=torch.float32)
        scores = torch.empty(B, ANCHORS, device="cuda", dtype=torch.float32)
        dets = torch.empty(B, ANCHORS, COORDS + 1, device="cuda", dtype=torch.float32)
        check(lib().cc_blazeface_forward(self._h, table, B, ptr(boxes), ptr(scores), ptr(dets), stream_ptr()),
              "cc_blazeface_forward")
        return dets, boxes, scores

    def detect(self, images) -> torch.Tensor:
        return self.forward(images)[0]

    def decode(self, boxes, scores, sizes) -> torch.Tensor:
        """The decode, order, suppression and scaling alone on given head outputs: boxes [B,896,16], scores [B,896] (fp32,
        host or device), sizes: B (height, width) of the images they stand for -> device [B,896,17]."""
        b = torch.as_tensor(boxes, dtype=torch.float32).to("cuda").contiguous()
        s = torch.as_tensor(scores, dtype=torch.float32).to("cuda").contiguous()
        B = b.shape[0]
        if b.shape != (B, ANCHORS, COORDS) or s.shape != (B, ANCHORS) or B < 1:
            raise ValueError(f"boxes must be [B,{ANCHORS},{COORDS}] and scores [B,{ANCHORS}], got {tuple(b.shape)}, {tuple(s.shape)}")
        hw = np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(-1, 2))
        if len(hw) != B:
            raise ValueError(f"{len(hw)} sizes for {B} images")
        out = torch.empty(B, ANCHORS, COORDS + 1, device="cuda", dtype=torch.float32)
        check(lib().cc_blazeface_decode(self._h, ptr(b), ptr(s), B, hw.ctypes.data, ptr(out), stream_ptr()), "cc_blazeface_decode")
        return out

    def __call__(self, img) -> DeviceResult:
        """BlazeFace.__call__: one HWC uint8 image -> DeviceResult (896,17)."""
        return DeviceResult(self.detect([_as_tensor(img)])[0])


def frame_table(ims):
    """Device uint8 [h,w,3] images -> a cc_frame table."""
    return (cc_frame * len(ims))(*[cc_frame(t.data_ptr(), CC_FRAME_BGR_U8, t.shape[0], t.shape[1]) for t in ims])


def face_canvas(ims) -> torch.Tensor:
    """The pre-resize of img_to_face (models/objects.py:265-272) for device uint8 [h,w,3] images in one launch ->
    device uint8 [B,640,640,3], each cv2.copyMakeBorder(cv2.resize(img, long side 640), centred zero border) exactly."""
    out = torch.empty(len(ims), 640, 640, 3, dtype=torch.uint8, device="cuda")
    check(lib().cc_face_canvas(frame_table(ims), len(ims), ptr(out), stream_ptr()), "cc_face_canvas")
    return out


def face_geometry(detections: np.ndarray, h: int, w: int):
    """models/objects.py:273-346 as the reference writes it (numpy and cv2 on the host, float32 where its rows are float32):
    the BlazeFace rows of the 640x640 canvas of an h x w image -> (x1_crop, y1_crop, x2_crop, y2_crop, rot_mat, new_w,
    new_h, transform_mat), or None where the reference returns None."""
    import cv2
    scale = 640 / max(h, w)
    delta_w, delta_h = 640 - int(w * scale), 640 - int(h * scale)
    top, left = delta_h // 2, delta_w // 2
    detections = detections[detections[:, 0] != 0]
    if detections.shape[0] == 0:
        return None
    y1, x1, y2, x2 = detections[0][:4]
    left_eye = np.array([detections[0][4], detections[0][5]])
    right_eye = np.array([detections[0][6], detections[0][7]])
    x1 -= left; x2 -= left
    y1 -= top; y2 -= top
    left_eye -= np.array([left, top])
    right_eye -= np.array([left, top])
    x1 /= scale; x2 /= scale
    y1 /= scale; y2 /= scale
    left_eye /= scale
    right_eye /= scale
    if (x2 - x1) < 50:
        return None
    eye_center = (left_eye + right_eye) / 2
    target_eye_distance = np.linalg.norm(TARGET_RIGHT_EYE - TARGET_LEFT_EYE)
    angle_rad = np.arctan2(right_eye[1] - left_eye[1], right_eye[0] - left_eye[0])
    angle = np.degrees(angle_rad)
    face_width = x2 - x1
    face_height = y2 - y1
    crop_size = max(face_width, face_height) * 2.0
    x1_crop = int(eye_center[0] - crop_size / 2)
    y1_crop = int(eye_center[1] - crop_size / 2)
    x2_crop = int(eye_center[0] + crop_size / 2)
    y2_crop = int(eye_center[1] + crop_size / 2)
    x1_crop = max(0, x1_crop)
    y1_crop = max(0, y1_crop)
    x2_crop = min(w, x2_crop)
    y2_crop = min(h, y2_crop)
    if x2_crop <= x1_crop or y2_crop <= y1_crop:
        return None
    crop_h, crop_w = y2_crop - y1_crop, x2_crop - x1_crop
    left_eye_crop = left_eye - np.array([x1_crop, y1_crop])
    right_eye_crop = right_eye - np.array([x1_crop, y1_crop])
    rot_mat = cv2.getRotationMatrix2D((crop_w / 2, crop_h / 2), angle, 1.0)
    cos_a = np.abs(rot_mat[0, 0])
    sin_a = np.abs(rot_mat[0, 1])
    new_w = int(crop_h * sin_a + crop_w * cos_a)
    new_h = int(crop_h * cos_a + crop_w * sin_a)
    rot_mat[0, 2] += (new_w / 2) - crop_w / 2
    rot_mat[1, 2] += (new_h / 2) - crop_h / 2
    left_eye_rot = rot_mat[:, :2] @ left_eye_crop + rot_mat[:, 2]
    right_eye_rot = rot_mat[:, :2] @ right_eye_crop + rot_mat[:, 2]
    rot_eye_distance = np.linalg.norm(right_eye_rot - left_eye_rot)
    final_scale = target_eye_distance / rot_eye_distance
    tx = TARGET_LEFT_EYE[0] - left_eye_rot[0] * final_scale
    ty = TARGET_LEFT_EYE[1] - left_eye_rot[1] * final_scale
    transform_mat = np.array([[final_scale, 0, tx], [0, final_scale, ty]], dtype=np.float32)
    return x1_crop, y1_crop, x2_crop, y2_crop, rot_mat, new_w, new_h, transform_mat


def _warps(jobs):
    """jobs: (image pointer or None, h, w, face_geometry result) per face -> a cc_face_warp table."""
    table = (cc_face_warp * len(jobs))()
    for k, (src, h, w, (x1, y1, x2, y2, rot, nw, nh, tm)) in enumerate(jobs):
        f = table[k]
        f.src, f.h, f.w = src, h, w
        f.x1, f.y1, f.x2, f.y2, f.rot_w, f.rot_h = x1, y1, x2, y2, nw, nh
        f.rot[:] = [float(v) for v in np.asarray(rot, np.float64).ravel()]
        f.transform[:] = [float(v) for v in np.asarray(tm, np.float32).astype(np.float64).ravel()]
    return table


def align_faces(jobs) -> torch.Tensor:
    """jobs: (device uint8 [h,w,3] image, face_geometry result) pairs -> device uint8 [K,112,112,3] in one launch: face k is
    exactly the reference's two cv2.warpAffine calls and RGB2BGR on its image."""
    out = torch.empty(len(jobs), FACE, FACE, 3, dtype=torch.uint8, device="cuda")
    if not jobs:
        return out
    table = _warps([(t.data_ptr(), t.shape[0], t.shape[1], g) for t, g in jobs])
    check(lib().cc_face_align(table, len(jobs), ptr(out), stream_ptr()), "cc_face_align")
    return out


# ---- the same on the images of a padded BGR batch [n,Hmax,Wmax,3] (image k in the h x w corner of its slot), as the device
# JPEG decoders write them: each slot is read as the RGB image cv2.cvtColor(slot, BGR2RGB) that img_to_face receives
def _slots(slots, index):
    assert slots.is_cuda and slots.dtype == torch.uint8 and slots.is_contiguous() and slots.dim() == 4 and slots.shape[3] == 3
    return (ptr(slots), *slots.shape[:3], np.ascontiguousarray(index, np.int32))


def face_canvas_slots(slots, index, sizes, rows=None) -> torch.Tensor:
    """The canvas of image b: the (height, width) = sizes[b] corner of slots[index[b]] -> device uint8 [max(rows, B),640,640,3]
    in one launch; canvas b equals `face_canvas` of the contiguous RGB copy of that image, and rows past B are zero (batch
    padding)."""
    B = len(index)
    out = torch.empty(max(rows or B, B), 640, 640, 3, dtype=torch.uint8, device="cuda")
    out[B:].zero_()
    p, n, H, W, idx = _slots(slots, index)
    hw = np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(-1, 2))
    check(lib().cc_face_canvas_slots(p, n, H, W, idx.ctypes.data, hw.ctypes.data, B, ptr(out), stream_ptr()), "cc_face_canvas_slots")
    return out


def align_faces_slots(slots, jobs) -> torch.Tensor:
    """jobs: (slot, (height, width), face_geometry result) -> device uint8 [K,112,112,3] in one launch: face k equals
    `align_faces` on the contiguous RGB copy of its image."""
    out = torch.empty(len(jobs), FACE, FACE, 3, dtype=torch.uint8, device="cuda")
    if not jobs:
        return out
    p, n, H, W, idx = _slots(slots, [s for s, _, _ in jobs])
    table = _warps([(None, h, w, g) for _, (h, w), g in jobs])
    check(lib().cc_face_align_slots(p, n, H, W, idx.ctypes.data, table, len(jobs), ptr(out), stream_ptr()), "cc_face_align_slots")
    return out


def first_detections(dets) -> torch.Tensor:
    """Device dets [B,896,17] -> device [B,17]: row b is detections[detections[:, 0] != 0][0] of image b (models/objects.py:
    283-284), or zeros where no row is kept; `face_geometry` of that one row is that of all 896."""
    d = dets.contiguous()
    B = d.shape[0]
    out = torch.empty(B, COORDS + 1, device="cuda", dtype=torch.float32)
    if B:
        check(lib().cc_blazeface_first(ptr(d), B, ptr(out), stream_ptr()), "cc_blazeface_first")
    return out
