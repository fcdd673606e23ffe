"""The image arithmetic of the reference's `img_to_face` (models/objects.py:263-354), restated in numpy and held byte for
byte to the installed cv2 (4.13) by tests/test_face_detect_cpu.py:

  * `resize_linear`: cv2.resize(INTER_LINEAR) of uint8 HWC images.  Fixed point: per output column x, fx =
    float((x + 0.5) * (1 / (dw / sw)) - 0.5), sx = floor(fx), clamped at both ends with fx = 0; column weights
    rint((1 - fx) * 2048), rint(fx * 2048); rows the same without the clamp of the weight (the row index is clamped
    instead); out = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2 on the 11-bit column sums.  An exact 2x
    reduction on both axes is cv2's INTER_AREA: (a + b + c + d + 2) >> 2.
  * `warp_affine`: cv2.warpAffine(INTER_LINEAR, BORDER_CONSTANT 0).  M inverted in float64; per pixel
    X = (rint((M1 * y + M2) * 1024) + 16 + rint(M0 * x * 1024)) >> 5 (likewise Y), integer part X >> 5, fraction X & 31;
    weights (32 - f) * (32 - g) * 32 ... summing to 32768; taps outside the source read 0; out = (sum + 16384) >> 15.
  * `geometry`: the reference's own numpy lines from the first surviving detection row to the crop, the rotation and
    the final float32 transform.
"""
from __future__ import annotations

import numpy as np

TARGET_LEFT_EYE = np.array([38, 51])
TARGET_RIGHT_EYE = np.array([73, 51])


def _axis(dst: int, src: int, clamp_weight: bool):
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_weight:
        lo, hi = s < 0, s >= src - 1
        f[lo | hi] = 0
        s[lo] = 0
        s[hi] = src - 1
    w0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    w1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), w0, w1


def resize_linear(img: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """cv2.resize(img, (dw, dh)) (INTER_LINEAR) of a uint8 [h,w,C] image."""
    h, w = img.shape[:2]
    if (dw, dh) == (w, h):
        return img.copy()
    x = img.astype(np.int64)
    if w == 2 * dw and h == 2 * dh:
        return ((x[0::2, 0::2] + x[0::2, 1::2] + x[1::2, 0::2] + x[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    xs, xs1, a0, a1 = _axis(dw, w, True)
    ys, ys1, b0, b1 = _axis(dh, h, False)
    hr = x[:, xs] * a0[None, :, None] + x[:, xs1] * a1[None, :, None]
    out = (((b0[:, None, None] * (hr[ys] >> 4)) >> 16) + ((b1[:, None, None] * (hr[ys1] >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)


def invert_affine(M) -> np.ndarray:
    """cv2.invertAffineTransform as warpAffine does it, in float64: 6 values."""
    m = np.asarray(M, np.float64).ravel().copy()
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    a11, a22 = m[4] * D, m[0] * D
    m[0], m[4] = a11, a22
    m[1] *= -D
    m[3] *= -D
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return m


def warp_affine(img: np.ndarray, M, dsize) -> np.ndarray:
    """cv2.warpAffine(img, M, dsize) (INTER_LINEAR, zero border) of a uint8 [h,w,3] image."""
    W, H = dsize
    m = invert_affine(M)
    h, w = img.shape[:2]
    x, y = np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64)
    X = (np.rint((m[1] * y + m[2]) * 1024).astype(np.int64)[:, None] + 16 + np.rint(m[0] * x * 1024).astype(np.int64)[None]) >> 5
    Y = (np.rint((m[4] * y + m[5]) * 1024).astype(np.int64)[:, None] + 16 + np.rint(m[3] * x * 1024).astype(np.int64)[None]) >> 5
    ix, fx, iy, fy = X >> 5, X & 31, Y >> 5, Y & 31
    src = img.astype(np.int64)

    def tap(yy, xx):
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        return np.where(ok[..., None], src[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)], 0)

    v = (tap(iy, ix) * ((32 - fy) * (32 - fx) * 32)[..., None] + tap(iy, ix + 1) * ((32 - fy) * fx * 32)[..., None]
         + tap(iy + 1, ix) * (fy * (32 - fx) * 32)[..., None] + tap(iy + 1, ix + 1) * (fy * fx * 32)[..., None])
    return np.clip((v + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def rotation_matrix(center, angle, scale) -> np.ndarray:
    """cv2.getRotationMatrix2D."""
    a = np.deg2rad(float(angle))
    alpha, beta = np.cos(a) * scale, np.sin(a) * scale
    cx, cy = center
    return np.array([[alpha, beta, (1 - alpha) * cx - beta * cy], [-beta, alpha, beta * cx + (1 - alpha) * cy]])


def canvas_geometry(h: int, w: int):
    """The pre-resize of img_to_face (:265-272): (new_w, new_h, top, left, scale)."""
    scale = 640 / max(h, w)
    rw, rh = int(w * scale), int(h * scale)
    return rw, rh, (640 - rh) // 2, (640 - rw) // 2, scale


def geometry(detections: np.ndarray, h: int, w: int, rotation=rotation_matrix, rounded_crop: bool = False):
    """models/objects.py:273-346, line for line, from the BlazeFace rows on the 640x640 canvas of an h x w image to
    (x1_crop, y1_crop, x2_crop, y2_crop, rot_mat [2,3] float64, new_w, new_h, transform_mat [2,3] float32), or None.
    rounded_crop=True is the mutation the tests check against (round instead of int)."""
    _, _, top, left, scale = canvas_geometry(h, w)
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
    cut = (lambda v: int(round(float(v)))) if rounded_crop else int
    x1_crop = cut(eye_center[0] - crop_size / 2)
    y1_crop = cut(eye_center[1] - crop_size / 2)
    x2_crop = cut(eye_center[0] + crop_size / 2)
    y2_crop = cut(eye_center[1] + crop_size / 2)
    x1_crop = max(0, x1_crop)
    y1_crop = max(0, y1_crop)
    x2_crop = min(w, x2_crop)
    y2_crop = min(h, y2_crop)
    if x2_crop <= x1_crop or y2_crop <= y1_crop:
        return None
    crop_h, crop_w = y2_crop - y1_crop, x2_crop - x1_crop
    left_eye_crop = left_eye - np.array([x1_crop, y1_crop])
    right_eye_crop = right_eye - np.array([x1_crop, y1_crop])
    rot_mat = rotation((crop_w / 2, crop_h / 2), angle, 1.0)
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


def canvas(orig: np.ndarray) -> np.ndarray:
    """cv2.resize to a long side of 640, then the zero border to 640x640 (:265-272)."""
    h, w = orig.shape[:2]
    rw, rh, top, left, _ = canvas_geometry(h, w)
    out = np.zeros((640, 640, orig.shape[2]), np.uint8)
    out[top:top + rh, left:left + rw] = resize_linear(orig, rw, rh)
    return out


def align(orig: np.ndarray, g, swap: bool = True) -> np.ndarray:
    """The two warps and the channel swap of :325-346 for geometry `g`.  swap=False is the mutation the tests check."""
    x1c, y1c, x2c, y2c, rot_mat, new_w, new_h, transform_mat = g
    rotated = warp_affine(orig[y1c:y2c, x1c:x2c], rot_mat, (new_w, new_h))
    face = warp_affine(rotated, transform_mat, (112, 112))
    return np.ascontiguousarray(face[..., ::-1]) if swap else face


def img_to_face(detect, orig: np.ndarray):
    """ObjectFinder.img_to_face with `detect(canvas) -> (896,17)` standing for `self.blazeface(Tensor(canvas)).numpy()`."""
    g = geometry(np.asarray(detect(canvas(orig)), np.float32), *orig.shape[:2])
    return None if g is None else align(orig, g)
