"""AdaFace IR-50 face embeddings on the H100: the reference's `ADAFACE` (models/adaface.py:24-96) with the same call form.

    from clearcam_b200.models.adaface import ADAFACE
    model = ADAFACE(weights=state_dict)                  # the reference's own key names ("body.list.3.res_layer0.weight", ...)
    emb = model(face).numpy()                            # face: (112,112,3) uint8 -> (1,512), as the reference returns
    embs = model.embed(faces)                            # faces: [B,112,112,3] uint8 -> device (B,512)

The weights are folded on the host in float64 (`fold_state_dict`) and the network runs as one plan of wgmma convs in
libclearcam_b200.so (csrc/adaface.cu); there is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, List

import numpy as np
import torch

from .._lib import CCError, check, lib, ptr, stream_ptr
from ..detection.yolov9 import DeviceResult, fetch, safe_load
from ..utils.helpers import batch_bucket

SIDE, DIM = 112, 512
EPS = 1e-5                                 # tinygrad BatchNorm's default (the reference keeps it)
# (in channels, depth, stride) of the 24 BasicBlockIR_tiny blocks: models/adaface.py:61
SIZES = [[64, 64, 2], [64, 64, 1], [64, 64, 1], [64, 128, 2], [128, 128, 1], [128, 128, 1], [128, 128, 1], [128, 256, 2]] + \
    [[256, 256, 1]] * 13 + [[256, 512, 2], [512, 512, 1], [512, 512, 1]]
WEIGHTS_URL = "https://huggingface.co/roryclear/AdaFace/resolve/main/adaface_ir50_ms1mv2.safetensors"   # :76


def _bn_keys(p: str, affine: bool = True) -> List[str]:
    # tinygrad's BatchNorm attributes in definition order: weight, bias (affine only), num_batches_tracked, running stats
    return ([f"{p}.weight", f"{p}.bias"] if affine else []) + [f"{p}.num_batches_tracked", f"{p}.running_mean", f"{p}.running_var"]


def state_dict_keys() -> List[str]:
    """The keys tinygrad's `get_state_dict(ADAFACE())` yields: attributes in assignment order (:64-75, :25-41), a `Seq`'s
    blocks under its attribute `list` (:15), and no entry for the None bias of a bias-free conv or of `bn2` (affine=False)."""
    keys = ["linear.weight", "linear.bias"] + _bn_keys("bn") + _bn_keys("bn2", affine=False) + ["prelu_weight", "conv0.weight"]
    keys += _bn_keys("bn0")
    for i, (cin, depth, _) in enumerate(SIZES):
        p = f"body.list.{i}"
        keys += _bn_keys(f"{p}.res_layer0") + [f"{p}.conv_layer0.weight"] + _bn_keys(f"{p}.res_layer1")
        keys += [f"{p}.prelu_weight", f"{p}.conv_layer1.weight"] + _bn_keys(f"{p}.res_layer2")
        if cin != depth:
            keys += [f"{p}.shortcut_layer0.weight"] + _bn_keys(f"{p}.shortcut_layer1")
    return keys


def _f64(t) -> np.ndarray:
    if isinstance(t, torch.Tensor):
        return t.detach().to("cpu", torch.float64).numpy()
    if hasattr(t, "numpy") and not isinstance(t, np.ndarray):
        t = t.numpy()
    return np.asarray(t, np.float64)


def _bn(sd, p: str, affine: bool = True):
    """BatchNorm in eval form (x - mean) * weight / sqrt(var + eps) + bias as (scale, shift)."""
    inv = 1.0 / np.sqrt(_f64(sd[f"{p}.running_var"]) + EPS)
    scale = _f64(sd[f"{p}.weight"]) * inv if affine else inv
    shift = (_f64(sd[f"{p}.bias"]) if affine else 0.0) - _f64(sd[f"{p}.running_mean"]) * scale
    return scale, shift


def border_bias(w: np.ndarray, shift: np.ndarray) -> np.ndarray:
    """w [O,I,3,3], a per-input-channel shift applied before the zero-padded conv -> [9,O]: for each border class
    3 * (top / interior / bottom) + (left / interior / right) the shift's contribution summed over the taps that read inside
    the map (a tap that reads the padding sees 0, not the shift)."""
    tap = np.einsum("oirs,i->ors", w, shift)
    inside = ([1, 2], [0, 1, 2], [0, 1])          # filter rows (cols) inside the map for the top / interior / bottom class
    return np.stack([tap[:, inside[rc]][:, :, inside[cc]].sum((1, 2)) for rc in range(3) for cc in range(3)])


def fold_state_dict(sd) -> Dict[str, np.ndarray]:
    """The reference's state dict -> the folded float64 network that cc_face_create takes (names in
    include/clearcam_b200.h).  Every BatchNorm folds into its conv / the linear; the input normalisation
    ((x[:,:,::-1] / 255 - 0.5) / 0.5, :81) and each block's res_layer0 are affine maps in front of a zero-padded 3x3 conv, so
    their scale goes into the weights and their shift into a border-class bias table (`border_bias`), exact at every pixel.
    `num_batches_tracked` is ignored.  Conv weights come out as [O][3][3][I] (the stem's I in the uint8 image's channel order),
    1x1 shortcuts as [O][I], and the linear's columns in NHWC order."""
    missing = [k for k in state_dict_keys() if not k.endswith("num_batches_tracked") and k not in sd]
    if missing:
        raise CCError(f"ADAFACE weights: {len(missing)} tensors missing, e.g. {missing[:3]}")
    F = {}
    s0, t0 = _bn(sd, "bn0")
    w = _f64(sd["conv0.weight"])                                        # [64, 3 (x channel = image channel 2 - c), 3, 3]
    F["stem.w"] = (s0[:, None, None, None] * w[:, ::-1] / 127.5).transpose(0, 2, 3, 1)
    F["stem.cls"] = s0[None] * border_bias(w, -np.ones(3)) + t0[None]
    F["stem.slope"] = _f64(sd["prelu_weight"])
    for i, (cin, depth, stride) in enumerate(SIZES):
        p, q = f"body.list.{i}", f"body.{i}"
        a, b = _bn(sd, f"{p}.res_layer0")
        s1, t1 = _bn(sd, f"{p}.res_layer1")
        s2, t2 = _bn(sd, f"{p}.res_layer2")
        w0 = _f64(sd[f"{p}.conv_layer0.weight"])
        F[f"{q}.c0.w"] = (s1[:, None, None, None] * w0 * a[None, :, None, None]).transpose(0, 2, 3, 1)
        F[f"{q}.c0.cls"] = s1[None] * border_bias(w0, b) + t1[None]
        F[f"{q}.c0.slope"] = _f64(sd[f"{p}.prelu_weight"])
        F[f"{q}.c1.w"] = (s2[:, None, None, None] * _f64(sd[f"{p}.conv_layer1.weight"])).transpose(0, 2, 3, 1)
        F[f"{q}.c1.b"] = t2
        if cin != depth:
            ss, ts = _bn(sd, f"{p}.shortcut_layer1")
            F[f"{q}.sc.w"] = ss[:, None] * _f64(sd[f"{p}.shortcut_layer0.weight"])[:, :, 0, 0]
            F[f"{q}.sc.b"] = ts
        elif stride != 1:                                               # MaxPool2d(1, s): a subsample = identity 1x1 conv
            F[f"{q}.sc.w"] = np.eye(depth)
            F[f"{q}.sc.b"] = np.zeros(depth)
    sb, tb = _bn(sd, "bn")
    s2, t2 = _bn(sd, "bn2", affine=False)
    W = _f64(sd["linear.weight"]).reshape(DIM, DIM, 49)                 # [out, c, h*7 + w]: the NCHW flatten of :90
    bias = _f64(sd["linear.bias"]) + np.einsum("ocp,c->o", W, tb)
    F["linear.w"] = (s2[:, None, None] * W * sb[None, :, None]).transpose(0, 2, 1).reshape(DIM, 49 * DIM)
    F["linear.b"] = s2 * bias + t2
    return F


def _face_batch(faces) -> torch.Tensor:
    t = faces.tensor if isinstance(faces, DeviceResult) else faces
    if not isinstance(t, torch.Tensor):
        if hasattr(t, "numpy") and not isinstance(t, np.ndarray):
            t = t.numpy()
        t = torch.from_numpy(np.ascontiguousarray(t))
    if t.dtype != torch.uint8 or t.dim() != 4 or tuple(t.shape[1:]) != (SIDE, SIDE, 3) or t.shape[0] < 1:
        raise ValueError(f"faces must be uint8 [B,{SIDE},{SIDE},3] with B >= 1, got {t.dtype} {tuple(t.shape)}")
    return t.to("cuda", non_blocking=True).contiguous()


class ADAFACE:
    """models/adaface.py:63-96.  `weights`: the reference's state dict (tensors or arrays under its key names), a
    .safetensors path, or None for the reference's file (found through `fetch`)."""

    def __init__(self, weights=None):
        self._h = None
        if weights is None:
            weights = safe_load(fetch(WEIGHTS_URL))
        elif isinstance(weights, (str, os.PathLike)):
            weights = safe_load(weights)
        L = lib()
        if L.cc_device_check() <= 0:
            raise CCError("clearcam_b200 needs an H100 (sm_90) GPU: " + L.cc_last_error().decode())
        items = [(k, np.ascontiguousarray(v, np.float32)) for k, v in fold_state_dict(weights).items()]
        names = (ctypes.c_char_p * len(items))(*[k.encode() for k, _ in items])
        ptrs = (ctypes.c_void_p * len(items))(*[a.ctypes.data for _, a in items])
        nums = (ctypes.c_int64 * len(items))(*[a.size for _, a in items])
        h = ctypes.c_void_p()
        check(L.cc_face_create(len(items), names, ptrs, nums, ctypes.byref(h)), "cc_face_create")
        self._h = h

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                lib().cc_face_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def embed(self, faces) -> torch.Tensor:
        """faces uint8 [B,112,112,3] (host or device, each as the reference's call receives it) -> device (B,512) fp32; row b
        is what `self(faces[b])` returns.  The batch runs padded to batch_bucket(B) so the plans stay few."""
        t = _face_batch(faces)
        B = t.shape[0]
        Bp = batch_bucket(B)
        if Bp > B:
            t = torch.cat([t, torch.zeros(Bp - B, SIDE, SIDE, 3, dtype=torch.uint8, device=t.device)])
        out = torch.empty(Bp, DIM, device="cuda", dtype=torch.float32)
        check(lib().cc_face_embed(self._h, ptr(t), Bp, ptr(out), DIM, stream_ptr()), "cc_face_embed")
        return out[:B]

    def __call__(self, x) -> DeviceResult:
        """ADAFACE.__call__: one HWC uint8 (112,112,3) image -> DeviceResult (1,512)."""
        t = x.tensor if isinstance(x, DeviceResult) else x
        if not isinstance(t, torch.Tensor):
            if hasattr(t, "numpy") and not isinstance(t, np.ndarray):
                t = t.numpy()
            t = torch.from_numpy(np.ascontiguousarray(t))
        if tuple(t.shape) != (SIDE, SIDE, 3):
            raise ValueError(f"ADAFACE takes one ({SIDE},{SIDE},3) image, got {tuple(t.shape)}")
        return DeviceResult(self.embed(t.unsqueeze(0)))

    def layer_output(self, faces, layer: int) -> torch.Tensor:
        """Parity tap (cc_face_layer_output): 0 the stem, 1..24 the output of block layer-1, 25 the linear -> bn2 output before
        the L2 norm, as fp32 NHWC [B,H,W,C] ([B,1,1,512] for 25), from the plan of exactly B faces."""
        t = _face_batch(faces)
        B = t.shape[0]
        C, H, W = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        check(lib().cc_face_layer_output(self._h, ptr(t), B, layer, None, ctypes.byref(C), ctypes.byref(H), ctypes.byref(W), None),
              "cc_face_layer_output")
        out = torch.empty(B, H.value, W.value, C.value, device="cuda", dtype=torch.float32)
        check(lib().cc_face_layer_output(self._h, ptr(t), B, layer, ptr(out), ctypes.byref(C), ctypes.byref(H), ctypes.byref(W),
                                         stream_ptr()), "cc_face_layer_output")
        return out
