"""Torch-CPU restatement of the reference's BlazeFace face detector (models/blazeface.py), the specification
csrc/blazeface.cu is tested against.

    P = load_weights("tests/golden/blazeface_ref.npz")        # the reference's own weights and 896 anchors
    r, c = forward(P, normalize(letterboxed_u8))              # [B,896,16] raw boxes, [B,896] raw scores
    dets = call(P, img)                                       # BlazeFace.__call__: (896,17) for one HWC uint8 image

Choices where the reference's arithmetic is tinygrad's and not stated by the model code (the device follows them):
  * divisions (x / 127.5, the IoU, `/= scale`) are true fp32 divisions;
  * the sigmoid is computed in float64 and rounded once to fp32 (the most accurate fp32 sigmoid), so the 0.85 decision
    depends only on the fp32 logit;
  * topk orders scores descending with ties in ascending anchor index (the detector's postprocess does the same).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.yolov9 import resize as tiny_resize

SIDE, ANCHORS = 256, 896
SCORE_CLIP, MIN_SCORE, IOU_THR = 100.0, 0.85, 0.3
X_SCALE = Y_SCALE = W_SCALE = H_SCALE = 256.0

# (in channels, out channels, stride) of backbone_tiny.list.0 .. 30 (models/blazeface.py:98-127)
BLOCKS = [(24, 24, 1)] * 7 + [(24, 24, 2)] + [(24, 24, 1)] * 7 + [(24, 48, 2)] + [(48, 48, 1)] * 7 + [(48, 96, 2)] + \
    [(96, 96, 1)] * 7


def state_dict_keys():
    """The 139 keys of the reference's safetensors file (tinygrad names; a Seq's blocks sit under `.list`)."""
    keys = ["conv_tiny.weight", "conv_tiny.bias"]
    for h in ("classifier_8", "classifier_16", "regressor_8", "regressor_16"):
        keys += [f"{h}_tiny.weight", f"{h}_tiny.bias"]
    keys += ["final.conv0_tiny.weight", "final.conv0_tiny.bias", "final.conv1_tiny.weight", "final.conv1_tiny.bias"]
    for i in range(len(BLOCKS)):
        keys += [f"backbone_tiny.list.{i}.conv{j}_tiny.{p}" for j in (0, 1) for p in ("weight", "bias")]
    return keys + ["anchors"]


def load_weights(src) -> dict:
    """A state dict, a .safetensors file or an .npz (tests/golden/blazeface_ref.npz) -> {key: fp32 CPU tensor}."""
    if isinstance(src, dict):
        d = src
    elif str(src).endswith(".npz"):
        with np.load(src) as z:
            d = {k: z[k] for k in z.files}
    else:
        from safetensors.numpy import load_file
        d = load_file(str(src))
    return {k: torch.as_tensor(np.asarray(d[k], np.float32)) for k in state_dict_keys()}


def normalize(u8: torch.Tensor) -> torch.Tensor:
    """uint8 [B,256,256,C] -> float [B,C,256,256]: x / 127.5 - 1 (models/blazeface.py:167-169)."""
    return u8.permute(0, 3, 1, 2).float() / 127.5 - 1.0


def _block(P, pfx, x, cin, cout, stride, dt):
    w0, b0 = P[f"{pfx}.conv0_tiny.weight"].to(dt), P[f"{pfx}.conv0_tiny.bias"].to(dt)
    w1, b1 = P[f"{pfx}.conv1_tiny.weight"].to(dt), P[f"{pfx}.conv1_tiny.bias"].to(dt)
    if stride == 2:
        h = F.pad(x, (0, 2, 0, 2))
        x = F.max_pool2d(x, 2, 2)
        h = F.conv2d(h, w0, b0, stride=2, groups=cin)
    else:
        h = F.conv2d(x, w0, b0, padding=1, groups=cin)
    if cout > cin:
        x = F.pad(x, (0, 0, 0, 0, 0, cout - cin))
    return torch.relu(x + F.conv2d(h, w1, b1))


def forward(P, x: torch.Tensor, dtype=torch.float32, taps=None):
    """BlazeFace.forward (models/blazeface.py:136-164): x [B,3,256,256] -> (r [B,896,16], c [B,896]).  dtype=float64 gives
    the high-precision reference the device's error bars are measured against.  taps: a list that receives the stem's,
    every block's and the final block's NCHW outputs."""
    dt = dtype
    x = F.pad(x.to(dt), (1, 2, 1, 2))
    b = x.shape[0]
    x = torch.relu(F.conv2d(x, P["conv_tiny.weight"].to(dt), P["conv_tiny.bias"].to(dt), stride=2))
    if taps is not None:
        taps.append(x)
    for i, (cin, cout, s) in enumerate(BLOCKS):
        x = _block(P, f"backbone_tiny.list.{i}", x, cin, cout, s, dt)
        if taps is not None:
            taps.append(x)
    h = F.pad(x, (0, 2, 0, 2))
    h = F.conv2d(h, P["final.conv0_tiny.weight"].to(dt), P["final.conv0_tiny.bias"].to(dt), stride=2, groups=96)
    h = torch.relu(F.conv2d(h, P["final.conv1_tiny.weight"].to(dt), P["final.conv1_tiny.bias"].to(dt)))
    if taps is not None:
        taps.append(h)

    def head(name, t, n):
        y = F.conv2d(t, P[f"{name}_tiny.weight"].to(dt), P[f"{name}_tiny.bias"].to(dt))
        return y.permute(0, 2, 3, 1).reshape(b, -1, n)

    c = torch.cat([head("classifier_8", x, 1), head("classifier_16", h, 1)], 1)
    r = torch.cat([head("regressor_8", x, 16), head("regressor_16", h, 16)], 1)
    return r, c[..., 0]


def sigmoid(x: torch.Tensor) -> torch.Tensor:
    return torch.sigmoid(x.double()).float()


def decode(r: torch.Tensor, c: torch.Tensor, anchors: torch.Tensor) -> torch.Tensor:
    """_tensors_to_detections with _decode_boxes (models/blazeface.py:177-211), per image: (B,896,16), (B,896) ->
    (B,896,17) [ymin, xmin, ymax, xmax, 6 keypoints (x, y), score], rows under the 0.85 score zeroed."""
    ax, ay, aw, ah = anchors[:, 0], anchors[:, 1], anchors[:, 2], anchors[:, 3]
    xc = r[..., 0] / X_SCALE * aw + ax
    yc = r[..., 1] / Y_SCALE * ah + ay
    w = r[..., 2] / W_SCALE * aw
    h = r[..., 3] / H_SCALE * ah
    kp = r[..., 4:].reshape(*r.shape[:-1], 6, 2)
    kx = kp[..., 0] / X_SCALE * aw[:, None] + ax[:, None]
    ky = kp[..., 1] / Y_SCALE * ah[:, None] + ay[:, None]
    boxes = torch.cat([torch.stack([yc - h / 2., xc - w / 2., yc + h / 2., xc + w / 2.], -1),
                       torch.stack([kx, ky], -1).reshape(*r.shape[:-1], 12)], -1)
    scores = sigmoid(c.clamp(-SCORE_CLIP, SCORE_CLIP))
    mask = scores >= MIN_SCORE
    return torch.cat([boxes, scores[..., None]], -1) * mask[..., None]


def iou_matrix(b: torch.Tensor) -> torch.Tensor:
    """compute_iou_matrix (models/blazeface.py:234-247) on (N,4), its operation order; 0/0 gives NaN, which compares false."""
    x1s, y1s, x2s, y2s = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    areas = (x2s - x1s) * (y2s - y1s)
    x1 = torch.maximum(x1s[:, None], x1s[None, :])
    y1 = torch.maximum(y1s[:, None], y1s[None, :])
    x2 = torch.minimum(x2s[:, None], x2s[None, :])
    y2 = torch.minimum(y2s[:, None], y2s[None, :])
    w = torch.clamp(x2 - x1, min=0)
    h = torch.clamp(y2 - y1, min=0)
    inter = w * h
    return inter / (areas[:, None] + areas[None, :] - inter)


def postprocess(d: torch.Tensor, kept_only: bool = False) -> torch.Tensor:
    """BlazeFace.postprocess (models/blazeface.py:213-232) of one image's (896,17): all rows in score order, a row zeroed
    when it is under 0.85 or when ANY earlier row (masked and suppressed ones included) overlaps it at IoU > 0.3.
    kept_only=True is the classic greedy NMS (only kept rows suppress); it exists for the tests' mutation check."""
    order = torch.sort(d[:, 16], descending=True, stable=True)[1]
    d = d[order]
    high = torch.triu(iou_matrix(d[:, :4]), diagonal=1) > IOU_THR
    if kept_only:
        keep = torch.ones(len(d), dtype=torch.bool)
        for j in range(len(d)):
            keep[j] = not bool((high[:j, j] & keep[:j]).any())
    else:
        keep = high.sum(0) == 0
    keep = keep & (d[:, 16] >= MIN_SCORE)
    return d * keep[:, None]


def letterbox(img: torch.Tensor):
    """The resize and pad of BlazeFace.__call__ (models/blazeface.py:155-165): HWC uint8 -> (256x256 uint8, scale, pad_top,
    pad_left).  The resize is utils/helpers.resize (tinygrad's linear interpolate, oracle.yolov9.resize)."""
    h0, w0 = img.shape[:2]
    scale = min(256 / w0, 256 / h0)
    new_w, new_h = int(w0 * scale), int(h0 * scale)
    r = tiny_resize(img, (new_w, new_h))
    top, left = (256 - new_h) // 2, (256 - new_w) // 2
    return F.pad(r, (0, 0, left, 256 - new_w - left, top, 256 - new_h - top)), scale, top, left


def unletterbox(d: torch.Tensor, scale: float, top: int, left: int, pad_keypoints: bool = False) -> torch.Tensor:
    """The tail of BlazeFace.__call__: *256, pads off the box columns only (the keypoints keep them: the reference's
    quirk), then every column, the score included, divided by the fp32 scale.  pad_keypoints=True is the mutation the tests
    check against."""
    d = d * 256
    d[:, [0, 2]] -= top
    d[:, [1, 3]] -= left
    if pad_keypoints:
        d[:, 4:16:2] -= left
        d[:, 5:16:2] -= top
    return d / torch.tensor(scale, dtype=torch.float32)


def call(P, img) -> torch.Tensor:
    """BlazeFace.__call__ for one HWC uint8 image (numpy or torch) -> (896,17) fp32."""
    img = torch.as_tensor(np.asarray(img))
    x, scale, top, left = letterbox(img)
    r, c = forward(P, normalize(x[None]))
    return unletterbox(postprocess(decode(r, c, P["anchors"])[0]), scale, top, left)
