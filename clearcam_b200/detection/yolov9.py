"""Drop-in for the reference's `detection/yolov9.py` on H100 (same import names and call signatures).

    from clearcam_b200.detection.yolov9 import YOLOv9
    model = YOLOv9(size="c", res=640, weights=state_dict_or_path)
    preds = model(frame).numpy()          # (300,6) float32 [x1,y1,x2,y2,conf,class]   (clearcam.py:583)

Mirrors: class YOLOv9 (/root/reference/detection/yolov9.py:298-421), postprocess (:439-458), and the names
test/run_mot.py:1-2 imports from the module.  All arithmetic runs in libclearcam_b200.so (hand-written sm_90a
kernels) through ctypes; torch tensors are only device containers.  There is no CPU fallback: without the
library or without an H100 every call raises CCError.

Differences the reference cannot express (additions): `detect_batch(frames[B,H,W,3])`, explicit `weights=`
(the reference downloads from HuggingFace at construction, :372; there is no network here), `pix_fmt="yuv420p"`:
frames as a camera decodes them, uint8 [H*3/2,W] (a batch [B,H*3/2,W]), converted to BGR on the GPU bit-exactly as
cv2.cvtColor(COLOR_YUV2BGR_I420) would (clearcam_b200/pixfmt.py), and `detect_frames([...])`: frames of different
shapes and formats in one batch, as long as they letterbox to the same net input (`net_shape`).
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import padding
from .._lib import CC_MAX_FRAMES, CCError, Handle, _to_host_fp32, check, create, lib, ptr, stream_ptr
from ..pixfmt import BGR24, CC_FRAME_BGR_F32, CC_FRAME_BGR_U8, CC_FRAME_I420_U8, check_pix_fmt, yuv420p_rows, yuv420p_size


# ----------------------------------------------------------------------------------------------- helpers
class DeviceResult:
    """What the reference returns is a tinygrad Tensor; callers only use `.numpy()` (clearcam.py:583)."""

    def __init__(self, t: torch.Tensor):
        self.tensor = t

    def numpy(self) -> np.ndarray:
        return self.tensor.detach().to("cpu", torch.float32).numpy()

    @property
    def shape(self):
        return tuple(self.tensor.shape)

    def __array__(self, dtype=None):
        a = self.numpy()
        return a if dtype is None else a.astype(dtype)


def _as_tensor(v) -> torch.Tensor:
    """numpy / torch / tinygrad-like -> torch tensor, dtype and device unchanged."""
    if isinstance(v, DeviceResult):
        v = v.tensor
    if not isinstance(v, torch.Tensor):
        if hasattr(v, "numpy") and not isinstance(v, np.ndarray):
            v = v.numpy()
        v = torch.from_numpy(np.ascontiguousarray(v))
    return v


def _yuv_geometry(t: torch.Tensor):
    """A yuv420p batch [B,H*3/2,W] uint8 -> (B, H, W); ValueError for anything else."""
    if t.dtype != torch.uint8 or t.dim() != 3:
        raise ValueError(f"yuv420p frames must be uint8 [B,H*3/2,W], got {t.dtype} {tuple(t.shape)}")
    return (int(t.shape[0]),) + yuv420p_size(t.shape)


def _frame_code(t: torch.Tensor, pix_fmt: str) -> int:
    if check_pix_fmt(pix_fmt) == BGR24:
        return CC_FRAME_BGR_F32 if t.dtype == torch.float32 else CC_FRAME_BGR_U8
    return CC_FRAME_I420_U8


def net_shape(H: int, W: int, res: int, pix_fmt: str = BGR24) -> Tuple[int, int]:
    """(net_h, net_w): the detector's input extent for an H x W frame at `res` — the letterboxed extent of
    YOLOv9.preprocess rounded up to a multiple of 32.  Frames with the same net shape can share one `detect_frames`
    batch (720p, 1080p, 1440p and 2160p all give (384, 640) at res 640).  Host only, needs no GPU."""
    if check_pix_fmt(pix_fmt) != BGR24:
        yuv420p_rows(int(H), int(W))                # ValueError for odd sides
    code = CC_FRAME_BGR_U8 if pix_fmt == BGR24 else CC_FRAME_I420_U8
    nh, nw = ctypes.c_int(), ctypes.c_int()
    check(lib().cc_yolo_net_shape(code, int(H), int(W), int(res), ctypes.byref(nh), ctypes.byref(nw)), "cc_yolo_net_shape")
    return nh.value, nw.value


def frame_table(frames, pix_fmts, res: int):
    """Validate a list of device frames for one frame-table call -> (ctypes cc_frame array, (net_h, net_w)).
    frames: uint8 CUDA tensors, [H,W,3] for "bgr24" or [H*3/2,W] for "yuv420p", or None for a padding row; pix_fmts: one
    format for all, or one per frame.  Raises ValueError before any library call that launches work."""
    from ..ops import frame_table as check_frames
    frames = list(frames)
    B = len(frames)
    fmts = [pix_fmts] * B if isinstance(pix_fmts, str) else list(pix_fmts)
    if len(fmts) != B:
        raise ValueError(f"{B} frames but {len(fmts)} pixel formats")
    if not 1 <= B <= CC_MAX_FRAMES:
        raise ValueError(f"a frame table holds 1 to {CC_MAX_FRAMES} frames, got {B}")
    table, sizes = check_frames(frames, fmts, padding=True)
    net = None
    for i, (hw, fmt) in enumerate(zip(sizes, fmts)):
        if hw is None:
            continue
        ns = net_shape(*hw, res, fmt)
        if net is not None and ns != net:
            raise ValueError(f"frame {i} ({hw[0]}x{hw[1]}) has net shape {ns}, an earlier frame {net}: one call takes one net shape")
        net = ns
    if net is None:
        raise ValueError("every frame of the table is a padding row (None)")
    return table, net


def safe_load(path) -> Dict[str, torch.Tensor]:
    """tinygrad.nn.state.safe_load equivalent (detection/yolov9.py:5,372)."""
    from safetensors.torch import load_file
    return load_file(str(path))


def fetch(url: str) -> str:
    """tinygrad.helpers.fetch equivalent: there is no network here, so only a local mirror is honoured:
    $CLEARCAM_B200_WEIGHTS/<basename(url)>."""
    root = os.environ.get("CLEARCAM_B200_WEIGHTS", "")
    cand = os.path.join(root, os.path.basename(url)) if root else ""
    if cand and os.path.exists(cand):
        return cand
    raise CCError(f"cannot fetch {url}: no network; put the file under $CLEARCAM_B200_WEIGHTS or pass weights=")


def load_weights_arg(weights, default: str):
    """A model's `weights` argument -> its state dict: a state dict as it is, a path through safe_load, None the model's
    own file at `default`, a URL (found through `fetch`) or a local path."""
    if weights is None:
        if "://" in default:
            weights = fetch(default)
        elif not os.path.exists(default):
            raise CCError(f"weights not found at {default} (the reference's path); pass weights=")
        else:
            weights = default
    return safe_load(weights) if isinstance(weights, (str, os.PathLike)) else weights


def load_state_dict(model: "YOLOv9", state_dict) -> None:
    """tinygrad.nn.state.load_state_dict equivalent for this model (detection/yolov9.py:373)."""
    model.load_weights(state_dict)


# Importable layer names (test/run_mot.py:1-2 imports them).  The graph itself lives in the C++ plan builder
# (csrc/yolo.cu); these carry the constructor arguments so user code that builds/inspects layer lists still works.
class _Spec:
    def __init__(self, *args, f=-1, **kw):
        self.args, self.kw, self.f = args, kw, f


class Sequential(_Spec):
    def __init__(self, size=0, list=None):
        self.size = size
        self.list = list if list is not None else [None] * size

    def __len__(self): return len(self.list)
    def __setitem__(self, k, v): self.list[k] = v
    def __getitem__(self, k): return self.list[k]


class Conv(_Spec): pass
class ADown(_Spec): pass
class AConv(_Spec): pass
class ELAN1(_Spec): pass
class RepNBottleneck(_Spec): pass
class RepNCSP(_Spec): pass
class RepNCSPELAN4(_Spec): pass
class SP(_Spec): pass
class SPPELAN(_Spec): pass
class Concat(_Spec): pass
class DDetect(_Spec): pass
class CBLinear(_Spec): pass
class CBFuse(_Spec): pass
class DFL(_Spec): pass
class Upsample(_Spec): pass
class Silence(_Spec): pass


def postprocess(output, max_det=300, conf_threshold=0.25, iou_threshold=0.45):
    """detection/yolov9.py:439-458 on device. output: (B,84,A) [xc,yc,w,h,80 probs] -> DeviceResult (B,max_det,6)."""
    t = output.tensor if isinstance(output, DeviceResult) else output
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(np.asarray(t))
    t = t.to("cuda", torch.float32).contiguous()
    B, C, A = t.shape
    pred = torch.empty(B, A, 6, device="cuda", dtype=torch.float32)
    check(lib().cc_detect_pred_from_raw(ptr(t), B, C - 4, A, conf_threshold, ptr(pred), stream_ptr()), "cc_detect_pred_from_raw")
    out = torch.empty(B, max_det, 6, device="cuda", dtype=torch.float32)
    check(lib().cc_detect_postprocess(ptr(pred), B, A, max_det, iou_threshold, 0, 0.0, 0.0, 1.0, 0.0, 0.0, ptr(out),
                                      stream_ptr()), "cc_detect_postprocess")
    return DeviceResult(out)


# ----------------------------------------------------------------------------------------------- model
class YOLOv9(Handle):
    """YOLOv9(size, res) — same constructor/call contract as the reference (detection/yolov9.py:298-388)."""
    _destroy = "cc_yolo_destroy"

    def __init__(self, size: str = "t", res: int = 1280, weights=None, pad: bool = True, precise: bool = False):
        """pad=False keeps a size with odd widths (t) on its literal graph, whose narrow convs then take the generic
        CUDA-core kernel; m only runs padded.
        precise=True: the fp32-accurate mode (CC_YOLO_FP32_ACCURATE) — fp32 activations, every conv as six bf16 plane
        products on the tensor cores with fp32 accumulation, exact SiLU.  The reference is fp32 end to end; this is the
        mode that reproduces its boxes / scores at the north-star tolerance (the default stores activations in bf16)."""
        self.size, self.res, self.pad, self.precise = size, res, pad, bool(precise)
        self.load_weights(load_weights_arg(weights, f"https://huggingface.co/roryclear/yolov9/resolve/main/yolov9-{size}.safetensors"))

    # -- weights
    def load_weights(self, state_dict) -> None:
        # t and m have widths that are not multiples of 16: run their zero-padded equivalents (same function, every conv
        # on the tensor-core kernel) — see detection/padding.py
        lib_size = padding.padded_size(self.size) if self.pad and padding.padded_size(self.size) else self.size

        def tensors():
            sd = {k.replace(".list.", "."): _to_host_fp32(v) for k, v in state_dict.items() if not k.endswith(("anchors", "strides"))}
            return padding.pad_state_dict(self.size, sd) if lib_size != self.size else sd
        self._adopt(create("cc_yolo_create_ex", tensors, lib_size.encode(), 1 if self.precise else 0))

    # -- inference
    @staticmethod
    def _as_device_frames(frames) -> torch.Tensor:
        t = _as_tensor(frames)
        if t.dtype not in (torch.uint8, torch.float32):
            t = t.to(torch.float32)
        return t.to("cuda", non_blocking=True).contiguous()

    def _device_batch(self, frames, pix_fmt: str):
        """-> (device tensor, frame_fmt code, B, Hf, Wf) of a batch in `pix_fmt`, validated before any library call."""
        if check_pix_fmt(pix_fmt) == BGR24:
            t = self._as_device_frames(frames)
            assert t.dim() == 4 and t.shape[-1] == 3, "frames must be [B,H,W,3]"
            B, Hf, Wf, _ = t.shape
        else:
            t = _as_tensor(frames)
            B, Hf, Wf = _yuv_geometry(t)
            t = t.to("cuda", non_blocking=True).contiguous()
        return t, _frame_code(t, pix_fmt), B, Hf, Wf

    def detect_batch(self, frames, raw: bool = False, stream=None, pix_fmt: str = BGR24):
        """frames: [B,H,W,3] BGR uint8|float32 (pix_fmt="bgr24"), or [B,H*3/2,W] uint8 (pix_fmt="yuv420p"; H, W even);
        host or device.  Returns device tensor (B,300,6) in frame pixels (and the (B,84,A) head tap when raw=True)."""
        t, code, B, Hf, Wf = self._device_batch(frames, pix_fmt)
        out = torch.empty(B, 300, 6, device="cuda", dtype=torch.float32)
        rawt = None
        if raw:
            A = self.plan_info(B, Hf, Wf, is_f32=code == CC_FRAME_BGR_F32, pix_fmt=pix_fmt)["anchors"]
            rawt = torch.empty(B, 84, A, device="cuda", dtype=torch.float32)
        check(lib().cc_yolo_forward(self._h, ptr(t), code, B, Hf, Wf, self.res, ptr(out), ptr(rawt), stream_ptr(stream)),
              "cc_yolo_forward")
        return (out, rawt) if raw else out

    def net_shape(self, H: int, W: int, pix_fmt: str = BGR24) -> Tuple[int, int]:
        """(net_h, net_w) of an H x W frame at this model's res: frames with equal net shapes can share a
        `detect_frames` call."""
        return net_shape(H, W, self.res, pix_fmt)

    def detect_frames(self, frames, pix_fmts=BGR24, raw: bool = False, stream=None):
        """Frames of different shapes and formats in one batch.  frames: a list of B <= CC_MAX_FRAMES (128) device uint8
        tensors, [H,W,3] bgr24 or [H*3/2,W] yuv420p as `pix_fmts` says (one format, or one per frame), None for a padding
        row; every frame must have the same `net_shape`.  Returns the device tensor (B,300,6): row b is frame b's
        detections in its own pixels, what `detect_batch` of B frames of its shape and format gives at row b (and the
        (B,84,A) head tap when raw=True).  Shapes and formats are checked before the library is called (ValueError)."""
        table, (nh, nw) = frame_table(frames, pix_fmts, self.res)
        B = len(table)
        out = torch.empty(B, 300, 6, device="cuda", dtype=torch.float32)
        rawt = None
        if raw:
            A = sum((nh // s) * (nw // s) for s in (8, 16, 32))
            rawt = torch.empty(B, 84, A, device="cuda", dtype=torch.float32)
        check(lib().cc_yolo_forward_frames(self._h, ctypes.cast(table, ctypes.c_void_p), B, self.res, ptr(out), ptr(rawt),
                                           stream_ptr(stream)), "cc_yolo_forward_frames")
        return (out, rawt) if raw else out

    def detect_pipelined(self, host_batches, depth: int = 2, pix_fmt: str = BGR24):
        """Throughput API for host-resident frames: iterates over pinned host batches ([B,H,W,3] bgr24 or [B,H*3/2,W]
        yuv420p, as `pix_fmt` says) and yields one
        pinned host result (B,300,6) per batch.  The H2D copy of batch i+1 and the D2H read of result i-1 run on a side
        stream while batch i computes (double-buffered device frames / results), so PCIe time hides behind the kernels."""
        main = torch.cuda.current_stream()
        side = getattr(self, "_side_stream", None)
        if side is None:
            side = self._side_stream = torch.cuda.Stream()
        it = iter(host_batches)
        slots = []          # per in-flight batch: (device frames, device out, host out, ready event, done event)
        pending = []

        def stage(hb):
            if not hb.is_pinned():
                hb = hb.pin_memory()
            with torch.cuda.stream(side):
                dev = hb.to("cuda", non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(side)
            return dev, ev

        nxt = next(it, None)
        staged = stage(nxt) if nxt is not None else None
        while staged is not None:
            dev, ev = staged
            nxt = next(it, None)
            staged = stage(nxt) if nxt is not None else None          # H2D of the next batch overlaps this compute
            main.wait_event(ev)
            out = self.detect_batch(dev, pix_fmt=pix_fmt)
            done = torch.cuda.Event()
            done.record(main)
            dev.record_stream(main)
            with torch.cuda.stream(side):
                side.wait_event(done)
                host_out = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
                host_out.copy_(out, non_blocking=True)
                fin = torch.cuda.Event()
                fin.record(side)
            out.record_stream(side)
            pending.append((host_out, fin))
            while len(pending) > depth:
                h, f = pending.pop(0)
                f.synchronize()
                yield h
        for h, f in pending:
            f.synchronize()
            yield h

    def __call__(self, frame, pix_fmt: str = BGR24):
        """frame: HWC BGR image (uint8 or float32; numpy / torch / anything with .numpy()), or with pix_fmt="yuv420p" a
        uint8 [H*3/2,W] planar frame.  -> (300,6)
        The single-frame call of the reference's camera loop (clearcam.py:580-583).  A host frame is copied into a device
        buffer this object keeps per frame shape and format, and the result is produced in a kept buffer too, so the library
        sees the same pointers call after call and replays its captured CUDA graph of the plan instead of re-launching ~140
        kernels."""
        single_dim = 3 if check_pix_fmt(pix_fmt) == BGR24 else 2
        t = frame
        if isinstance(t, DeviceResult):
            t = t.tensor
        if isinstance(t, torch.Tensor) and t.is_cuda:
            if pix_fmt == BGR24:
                t = self._as_device_frames(t)
            if t.dim() == single_dim:
                t = t.unsqueeze(0)
            return DeviceResult(self.detect_batch(t, pix_fmt=pix_fmt)[0])
        t = _as_tensor(t)
        if pix_fmt == BGR24 and t.dtype not in (torch.uint8, torch.float32):
            t = t.to(torch.float32)
        if t.dim() == single_dim:
            t = t.unsqueeze(0)
        if pix_fmt != BGR24:
            _yuv_geometry(t)
        key = (tuple(t.shape), t.dtype, pix_fmt)
        bufs = getattr(self, "_single", None)
        if bufs is None or bufs[0] != key:
            bufs = self._single = (key, torch.empty(t.shape, dtype=t.dtype, device="cuda"),
                                   torch.empty(t.shape[0], 300, 6, device="cuda", dtype=torch.float32))
        _, dev, out = bufs
        dev.copy_(t, non_blocking=True)
        B, Hf, Wf = _yuv_geometry(dev) if pix_fmt != BGR24 else dev.shape[:3]
        check(lib().cc_yolo_forward(self._h, ptr(dev), _frame_code(dev, pix_fmt), B, Hf, Wf, self.res, ptr(out), None,
                                    stream_ptr()), "cc_yolo_forward")
        return DeviceResult(out[0].clone())

    def plan_info(self, B, Hf, Wf, is_f32=False, pix_fmt: str = BGR24) -> dict:
        """Facts of the plan for B frames of Hf x Wf pixels (is_f32: float32 bgr24 frames)."""
        code = (CC_FRAME_BGR_F32 if is_f32 else CC_FRAME_BGR_U8) if check_pix_fmt(pix_fmt) == BGR24 else CC_FRAME_I420_U8
        i = [ctypes.c_int() for _ in range(4)]
        d = [ctypes.c_double() for _ in range(2)]
        check(lib().cc_yolo_plan_info(self._h, code, B, Hf, Wf, self.res, *[ctypes.byref(x) for x in i],
                                      *[ctypes.byref(x) for x in d]), "cc_yolo_plan_info")
        return {"net_h": i[0].value, "net_w": i[1].value, "anchors": i[2].value, "launches": i[3].value,
                "conv_flops": d[0].value, "act_bytes": d[1].value}

    def profile(self, frames, pix_fmt: str = BGR24):
        """Per-op device times of one forward: list of dicts {kind, name, ms, flops}."""
        t, code, B, Hf, Wf = self._device_batch(frames, pix_fmt)
        out = torch.empty(B, 300, 6, device="cuda", dtype=torch.float32)
        cap = 1024
        ms = (ctypes.c_float * cap)()
        fl = (ctypes.c_double * cap)()
        by = (ctypes.c_double * cap)()
        kinds = (ctypes.c_char_p * cap)()
        names = (ctypes.c_char_p * cap)()
        n = ctypes.c_int()
        check(lib().cc_yolo_profile(self._h, ptr(t), code, B, Hf, Wf, self.res, ptr(out), cap,
                                    ms, fl, by, kinds, names, ctypes.byref(n), stream_ptr()), "cc_yolo_profile")
        return [{"kind": kinds[i].decode(), "name": names[i].decode(), "ms": ms[i], "flops": fl[i], "bytes": by[i]}
                for i in range(n.value)]

    def trace(self, frames):
        """In-situ device timeline of one forward (no events between launches): list of dicts {kind, name, flops,
        t_in, t_dep, t_out, cta0} in ns relative to the first kernel (zeros for the non-GEMM kernels); cta0 = five stamps of
        CTA 0: first operands landed, all MMAs issued, first accumulator complete, last epilogue group done, exit."""
        t = self._as_device_frames(frames)
        B, Hf, Wf, _ = t.shape
        out = torch.empty(B, 300, 6, device="cuda", dtype=torch.float32)
        cap = 1024
        ns = (ctypes.c_ulonglong * (12 * cap))()
        fl = (ctypes.c_double * cap)()
        kinds = (ctypes.c_char_p * cap)()
        names = (ctypes.c_char_p * cap)()
        n = ctypes.c_int()
        check(lib().cc_yolo_trace(self._h, ptr(t), 1 if t.dtype == torch.float32 else 0, B, Hf, Wf, self.res, ptr(out), cap,
                                  ns, kinds, names, fl, ctypes.byref(n), stream_ptr()), "cc_yolo_trace")
        t0 = min(ns[12 * i] for i in range(n.value) if ns[12 * i])
        rel = lambda v: (v - t0) if v else 0
        return [{"kind": kinds[i].decode(), "name": names[i].decode(), "flops": fl[i], "t_in": rel(ns[12 * i]),
                 "t_dep": rel(ns[12 * i + 1]), "t_out": rel(ns[12 * i + 2]),
                 "cta0": [rel(ns[12 * i + j]) for j in range(3, 8)],
                 "pass_cycles": [int(ns[12 * i + j]) - int(ns[12 * i + 8]) for j in range(9, 12)]} for i in range(n.value)]

    def layer_output(self, layer: int, B, Hf, Wf, is_f32=False):
        """Parity tap: output of graph layer `layer` of the last forward with this shape, as fp32 (B,C,H,W), or None."""
        c, hh, ww = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        f = 1 if is_f32 else 0
        check(lib().cc_yolo_layer_output(self._h, f, B, Hf, Wf, self.res, layer, None, ctypes.byref(c), ctypes.byref(hh),
                                         ctypes.byref(ww), None), "cc_yolo_layer_output")
        if c.value == 0:
            return None
        out = torch.empty(B, hh.value, ww.value, c.value, device="cuda", dtype=torch.float32)
        check(lib().cc_yolo_layer_output(self._h, f, B, Hf, Wf, self.res, layer, ptr(out), ctypes.byref(c),
                                         ctypes.byref(hh), ctypes.byref(ww), stream_ptr()), "cc_yolo_layer_output")
        if self.pad and padding.padded_size(self.size):        # padded equivalent: report the model's own channels
            maps = padding.layer_channel_maps(self.size)
            if layer < len(maps):
                idx = torch.from_numpy(maps[layer]).cuda()
                pads = torch.ones(c.value, dtype=torch.bool, device="cuda")
                pads[idx] = False
                if bool(pads.any()) and float(out[..., pads].abs().max()) != 0.0:
                    raise CCError(f"layer {layer}: padding channels are not zero")
                out = out[..., idx]
        return out.permute(0, 3, 1, 2)

    # -- host-side helpers kept for API parity
    def preprocess(self, image, new_shape=None, pix_fmt: str = BGR24):
        """YOLOv9.preprocess (:390-404) on device; returns DeviceResult HWC BGR (same dtype; uint8 for yuv420p frames,
        [H*3/2,W] or [B,H*3/2,W])."""
        if check_pix_fmt(pix_fmt) == BGR24:
            t = self._as_device_frames(image)
            squeeze = t.dim() == 3
            if squeeze:
                t = t.unsqueeze(0)
            B, Hf, Wf, _ = t.shape
        else:
            t = _as_tensor(image)
            squeeze = t.dim() == 2
            if squeeze:
                t = t.unsqueeze(0)
            B, Hf, Wf = _yuv_geometry(t)
            t = t.to("cuda", non_blocking=True).contiguous()
        res = self.res if new_shape is None else int(new_shape)
        oh, ow = ctypes.c_int(), ctypes.c_int()
        code = _frame_code(t, pix_fmt)
        check(lib().cc_letterbox(None, code, B, Hf, Wf, res, None, ctypes.byref(oh), ctypes.byref(ow), None), "cc_letterbox")
        out = torch.empty(B, oh.value, ow.value, 3, device="cuda", dtype=t.dtype)
        check(lib().cc_letterbox(ptr(t), code, B, Hf, Wf, res, ptr(out), ctypes.byref(oh), ctypes.byref(ow), stream_ptr()),
              "cc_letterbox")
        return DeviceResult(out[0] if squeeze else out)
