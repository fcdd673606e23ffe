"""CPU ORACLE (test infrastructure, NOT product code) — torch-CPU fp32 restatement of the reference detector.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
PARITY UNPINNED: the reference runs on tinygrad (pinned git fe39cf1, not in /root/reference, not installable
here) and fetches its weights from HuggingFace, so it cannot be executed in this environment and its tests hold
no detector tensors (SURVEY.md §8c).  Fidelity rests on line-by-line correspondence with

    /root/reference/detection/yolov9.py   (whole file; line numbers cited per function below)
    /root/reference/utils/helpers.py:127-131 (resize)

plus the param/FLOP identities (tests/test_oracle_cpu.py) and the YOLOv9-t real-weight smoke check against the
reference's recorded tracker inputs (tests/golden/, made by oracle/make_golden.py).

Structure is deliberately different from the reference (a flat op-spec interpreter over a {name: tensor}
dict instead of module objects); the arithmetic is the same.  `quant="bf16"` rounds every stored activation
and every weight to bf16 at the points where the CUDA path stores bf16, so the CUDA path can be compared both
with the true fp32 oracle and with its own number format.
"""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F

# channel tables of detection/yolov9.py:461-464 (SIZES); index names follow YOLOv9.__init__ :302
_SIZES = {
    "t": [16, 64, 96, 24, 128, 256, 224, 160, 48, 144, 192, 80, 32, 16, 3, 96, 32, 64, 128, 64, 64, 128],
    "s": [32, 128, 192, 48, 256, 512, 448, 320, 96, 288, 384, 128, 64, 32, 3, 192, 64, 64, 128, 128, 128, 256],
    "m": [32, 240, 360, 90, 480, 960, 840, 600, 184, 544, 720, 240, 128, 60, 1, 360, 120, 64, 128, 240, 240, 480],
    "c": [64, 256, 512, 128, 256, 1024, 1024, 1024, 128, 768, 1024, 256, 128, 64, 1, 256, 128, 128, 256, 128, 512, 512],
    # zero-padded equivalents the CUDA path runs t and m as (clearcam_b200/detection/padding.py): same graph, widths
    # rounded up to multiples of 16; tests/test_oracle_cpu.py proves the weight transform leaves the function unchanged
    "t@16": [16, 64, 96, 32, 128, 256, 224, 160, 48, 144, 192, 96, 32, 16, 3, 96, 32, 64, 128, 64, 64, 128],
    "m@16": [32, 240, 384, 96, 480, 960, 864, 624, 192, 576, 720, 240, 128, 64, 1, 384, 128, 64, 128, 240, 240, 480],
}


# ------------------------------------------------------------------------------------------------ graph spec
def _conv(cin, cout, k, s=1, g=1, act=True):
    return {"op": "conv", "cin": cin, "cout": cout, "k": k, "s": s, "g": g, "act": act}


def _repncsp(a, b, n):
    # detection/yolov9.py:92-105
    return {"op": "repncsp", "a": a, "b": b, "n": n}


def _elan4(a, b, c, n, f=-1):
    # detection/yolov9.py:107-125  RepNCSPELAN4(a, b, c, n)
    return {"op": "elan4", "a": a, "b": b, "c": c, "n": n, "f": f}


def build_spec(size: str) -> List[dict]:
    """Layer list equivalent to YOLOv9.__init__ (detection/yolov9.py:299-371)."""
    L: List[dict] = []
    if size != "e":
        a, b, c, d, e, f, g, h, i, j, k, l, m, n, p, q, r, s, t, u, v, w = _SIZES[size]
        small = size.split("@")[0] in ("t", "s")
        L.append({**_conv(3, a, 3, 2), "f": -1})
        L.append({**_conv(a, a * 2, 3, 2), "f": -1})
        L.append({"op": "elan1", "ch0": a * 2, "ch1": m, "ch2": a, "ch3": b, "f": -1} if small else _elan4(s, 32, t, p))
        L.append({"op": "adown", "ch": 128, "f": -1} if size == "c" else {"op": "aconv", "cin": m, "cout": u, "f": -1})
        L.append(_elan4(b, n, v, p))
        L.append({"op": "adown", "ch": 256, "f": -1} if size == "c" else {"op": "aconv", "cin": b, "cout": q, "f": -1})
        L.append(_elan4(c, d, c, p))
        L.append({"op": "adown", "ch": 256, "f": -1} if size == "c" else {"op": "aconv", "cin": q, "cout": e, "f": -1})
        L.append(_elan4(w, r, w, p))
        L.append({"op": "sppelan", "ch0": w, "ch1": b, "ch2": f, "ch3": w, "f": -1})
        L.append({"op": "upsample", "f": -1})
        L.append({"op": "concat", "f": [-1, 6]})
        L.append(_elan4(g, d, c, p))
        L.append({"op": "upsample", "f": -1})
        L.append({"op": "concat", "f": [-1, 4]})
        L.append(_elan4(h, n, b, p))
        L.append({"op": "adown", "ch": 128, "f": -1} if size == "c" else {"op": "aconv", "cin": v, "cout": i, "f": -1})
        L.append({"op": "concat", "f": [-1, 12]})
        L.append(_elan4(j, d, c, p))
        L.append({"op": "adown", "ch": 256, "f": -1} if size == "c" else {"op": "aconv", "cin": q, "cout": b, "f": -1})
        L.append({"op": "concat", "f": [-1, 9]})
        L.append(_elan4(k, r, w, p))
        L.append({"op": "detect", "chs": [b, c, w], "d": l, "f": [15, 18, 21]})
    else:
        # detection/yolov9.py:328-371 (hard-coded 43-layer graph)
        L.append({"op": "silence", "f": -1})
        L.append({**_conv(3, 64, 3, 2), "f": -1})
        L.append({**_conv(64, 128, 3, 2), "f": -1})
        L.append(_elan4(128, 32, 256, 2))
        L.append({"op": "adown", "ch": 128, "f": -1})
        L.append(_elan4(256, 64, 512, 2))
        L.append({"op": "adown", "ch": 256, "f": -1})
        L.append(_elan4(512, 128, 1024, 2))
        L.append({"op": "adown", "ch": 512, "f": -1})
        L.append(_elan4(1024, 128, 1024, 2))
        L.append({"op": "cblinear", "cin": 64, "c2s": [64], "f": 1})
        L.append({"op": "cblinear", "cin": 256, "c2s": [64, 128], "f": 3})
        L.append({"op": "cblinear", "cin": 512, "c2s": [64, 128, 256], "f": 5})
        L.append({"op": "cblinear", "cin": 1024, "c2s": [64, 128, 256, 512], "f": 7})
        L.append({"op": "cblinear", "cin": 1024, "c2s": [64, 128, 256, 512, 1024], "f": 9})
        L.append({**_conv(3, 64, 3, 2), "f": 0})
        L.append({"op": "cbfuse", "f": [10, 11, 12, 13, 14, -1], "idx": [0, 0, 0, 0, 0]})
        L.append({**_conv(64, 128, 3, 2), "f": -1})
        L.append({"op": "cbfuse", "f": [11, 12, 13, 14, -1], "idx": [1, 1, 1, 1]})
        L.append(_elan4(128, 32, 256, 2))
        L.append({"op": "adown", "ch": 128, "f": -1})
        L.append({"op": "cbfuse", "f": [12, 13, 14, -1], "idx": [2, 2, 2]})
        L.append(_elan4(256, 64, 512, 2))
        L.append({"op": "adown", "ch": 256, "f": -1})
        L.append({"op": "cbfuse", "f": [13, 14, -1], "idx": [3, 3]})
        L.append(_elan4(512, 128, 1024, 2))
        L.append({"op": "adown", "ch": 512, "f": -1})
        L.append({"op": "cbfuse", "f": [14, -1], "idx": [4]})
        L.append(_elan4(1024, 128, 1024, 2))
        L.append({"op": "sppelan", "ch0": 1024, "ch1": 256, "ch2": 1024, "ch3": 512, "f": 28})
        L.append({"op": "upsample", "f": -1})
        L.append({"op": "concat", "f": [-1, 25]})
        L.append(_elan4(1536, 128, 512, 2))
        L.append({"op": "upsample", "f": -1})
        L.append({"op": "concat", "f": [-1, 22]})
        L.append(_elan4(1024, 64, 256, 2))
        L.append({"op": "adown", "ch": 128, "f": -1})
        L.append({"op": "concat", "f": [-1, 32]})
        L.append(_elan4(768, 128, 512, 2))
        L.append({"op": "adown", "ch": 256, "f": -1})
        L.append({"op": "concat", "f": [-1, 29]})
        L.append(_elan4(1024, 256, 512, 2))
        L.append({"op": "detect", "chs": [256, 512, 512], "d": 256, "f": [35, 38, 41]})
    return L


def conv_table(size: str) -> List[tuple]:
    """[(state-dict prefix, cin, cout, k, stride, groups, has_act)] in the reference's definition order.

    Prefixes follow the reference's attribute paths with Sequential.list elided: `model.4.cv2.0.cv1.conv`,
    `model.22.cv2.0.2` (bare nn.Conv2d), `model.22.dfl.conv`."""
    out = []

    def add(prefix, cin, cout, k, s=1, g=1, act=True):
        out.append((prefix + (".conv" if act else ""), cin, cout, k, s, g, act))

    def add_repncsp(pfx, a, b, n):
        add(pfx + ".cv1", a, b, 1)
        add(pfx + ".cv2", a, b, 1)
        add(pfx + ".cv3", a, a, 1)
        for i in range(n):
            add(f"{pfx}.m.{i}.cv1", b, b, 3)
            add(f"{pfx}.m.{i}.cv2", b, b, 3)

    for i, l in enumerate(build_spec(size)):
        pfx = f"model.{i}"
        op = l["op"]
        if op == "conv":
            add(pfx, l["cin"], l["cout"], l["k"], l["s"])
        elif op == "elan1":
            add(pfx + ".cv1", l["ch0"], l["ch1"], 1)
            add(pfx + ".cv2", l["ch2"], l["ch2"], 3)
            add(pfx + ".cv3", l["ch2"], l["ch2"], 3)
            add(pfx + ".cv4", l["ch3"], l["ch1"], 1)
        elif op == "elan4":
            a, b, c, n = l["a"], l["b"], l["c"], l["n"]
            add(pfx + ".cv1", a, b * 4, 1)
            add_repncsp(pfx + ".cv2.0", b * 2, b, n)
            add(pfx + ".cv2.1", b * 2, b * 2, 3)
            add_repncsp(pfx + ".cv3.0", b * 2, b, n)
            add(pfx + ".cv3.1", b * 2, b * 2, 3)
            add(pfx + ".cv4", b * 8, c, 1)
        elif op == "adown":
            add(pfx + ".cv1", l["ch"], l["ch"], 3, 2)
            add(pfx + ".cv2", l["ch"], l["ch"], 1)
        elif op == "aconv":
            add(pfx + ".cv1", l["cin"], l["cout"], 3, 2)
        elif op == "sppelan":
            add(pfx + ".cv1", l["ch0"], l["ch1"], 1)
            add(pfx + ".cv5", l["ch2"], l["ch3"], 1)
        elif op == "cblinear":
            add(pfx + ".conv", l["cin"], sum(l["c2s"]), 1, act=False)
        elif op == "detect":
            d = l["d"]
            for j, ch in enumerate(l["chs"]):
                add(f"{pfx}.cv2.{j}.0", ch, 64, 3)
                add(f"{pfx}.cv2.{j}.1", 64, 64, 3, g=4)
                add(f"{pfx}.cv2.{j}.2", 64, 64, 1, g=4, act=False)
            for j, ch in enumerate(l["chs"]):
                add(f"{pfx}.cv3.{j}.0", ch, d, 3)
                add(f"{pfx}.cv3.{j}.1", d, d, 3)
                add(f"{pfx}.cv3.{j}.2", d, 80, 1, act=False)
    return out


def normalize_keys(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Accept the reference's safetensors naming (attribute paths, possibly with `.list.` segments)."""
    return {k.replace(".list.", "."): v for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------ forward
class _Q:
    """Quantisation policy: identity (fp32 oracle) or bf16 rounding at the CUDA path's storage points."""

    def __init__(self, mode):
        assert mode in (None, "bf16")
        self.mode = mode

    def act(self, t):
        return t if self.mode is None else t.to(torch.bfloat16).to(torch.float32)

    def w(self, t):
        return t if self.mode is None else t.to(torch.bfloat16).to(torch.float32)


def _cv(P, q, name, x, s=1, g=1, act=True, res=None, quant_w=True, store=True):
    """Conv (detection/yolov9.py:33-38): Conv2d(bias, padding=k//2) -> SiLU; bare nn.Conv2d when act=False."""
    w = P[name + ".weight"]
    b = P[name + ".bias"]
    if quant_w:
        w = q.w(w)
    y = F.conv2d(x, w, b, stride=s, padding=w.shape[-1] // 2, groups=g)
    if act:
        y = y * torch.sigmoid(y)
    if res is not None:
        y = res + y
    return q.act(y) if store else y


def _repncsp_fwd(P, q, pfx, x, n):
    # detection/yolov9.py:100-105 ; RepNBottleneck :89  x + cv2(cv1(x))
    x1 = _cv(P, q, pfx + ".cv1.conv", x)
    for i in range(n):
        t = _cv(P, q, f"{pfx}.m.{i}.cv1.conv", x1)
        x1 = _cv(P, q, f"{pfx}.m.{i}.cv2.conv", t, res=x1)
    x3 = _cv(P, q, pfx + ".cv2.conv", x)
    return _cv(P, q, pfx + ".cv3.conv", torch.cat([x1, x3], 1))


def _elan4_fwd(P, q, pfx, x, n):
    # detection/yolov9.py:119-125
    x = _cv(P, q, pfx + ".cv1.conv", x)
    y0, y1 = x.chunk(2, 1)
    y2 = _cv(P, q, pfx + ".cv2.1.conv", _repncsp_fwd(P, q, pfx + ".cv2.0", y1, n))
    y3 = _cv(P, q, pfx + ".cv3.1.conv", _repncsp_fwd(P, q, pfx + ".cv3.0", y2, n))
    return _cv(P, q, pfx + ".cv4.conv", torch.cat([y0, y1, y2, y3], 1))


def _avg2(x):
    # Tensor.avg_pool2d(x, 2, 1, 1, 0, False, True): kernel 2, stride 1, dilation 1, pad 0  (yolov9.py:47,:62)
    return F.avg_pool2d(x, 2, 1, 0)


def make_anchors(hw_list, strides=(8, 16, 32)):
    """detection/yolov9.py:247-261: centres (x+0.5, y+0.5), row-major per level; returns (2,A), (1,A)."""
    pts, st = [], []
    for (h, w), s in zip(hw_list, strides):
        sx = torch.arange(w, dtype=torch.float32) + 0.5
        sy = torch.arange(h, dtype=torch.float32) + 0.5
        gx = sx.reshape(1, -1).repeat(h, 1).reshape(-1)
        gy = sy.reshape(-1, 1).repeat(1, w).reshape(-1)
        pts.append(torch.stack([gx, gy], 0))
        st.append(torch.full((h * w,), float(s)))
    return torch.cat(pts, 1), torch.cat(st).unsqueeze(0)


def _detect_fwd(P, q, pfx, xs, d):
    """DDetect.__call__ (detection/yolov9.py:202-220) + DFL (:279-282) + dist2bbox (:263-271). -> (B,84,A)"""
    outs = []
    for j, x in enumerate(xs):
        b = _cv(P, q, f"{pfx}.cv2.{j}.0.conv", x)
        b = _cv(P, q, f"{pfx}.cv2.{j}.1.conv", b, g=4)
        b = _cv(P, q, f"{pfx}.cv2.{j}.2", b, g=4, act=False, store=False)   # fp32 logits on the CUDA path too
        c = _cv(P, q, f"{pfx}.cv3.{j}.0.conv", x)
        c = _cv(P, q, f"{pfx}.cv3.{j}.1.conv", c)
        c = _cv(P, q, f"{pfx}.cv3.{j}.2", c, act=False, store=False)
        outs.append(torch.cat([b, c], 1))
    B = xs[0].shape[0]
    cat = torch.cat([o.reshape(B, 144, -1) for o in outs], 2)
    box, cls = cat.split((64, 80), 1)
    A = box.shape[-1]
    # DFL: view (B,4,16,A) -> softmax over the 16 bins -> 1x1 conv with weight arange(16) (P[dfl]) = expectation
    dflw = P[f"{pfx}.dfl.conv.weight"].reshape(1, 1, 16, 1)
    dist = (box.reshape(B, 4, 16, A).softmax(2) * dflw).sum(2)             # (B,4,A)
    anchors, strides = make_anchors([o.shape[2:] for o in outs])
    lt, rb = dist.chunk(2, 1)
    x1y1 = anchors.unsqueeze(0) - lt
    x2y2 = anchors.unsqueeze(0) + rb
    cxy = (x1y1 + x2y2) / 2
    wh = x2y2 - x1y1
    dbox = torch.cat([cxy, wh], 1) * strides
    return torch.cat([dbox, torch.sigmoid(cls)], 1)


def forward_raw(size: str, P: Dict[str, torch.Tensor], x: torch.Tensor, quant=None, taps: list | None = None,
                stem_int: bool = True) -> torch.Tensor:
    """x: (B,3,H,W) fp32 RGB in [0,1] -> (B,84,A). Mirrors the routing loop of YOLOv9.__call__ (:380-385)."""
    q = _Q(quant)
    spec = build_spec(size)
    ys: List[object] = []
    cur: object = x
    for i, l in enumerate(spec):
        f = l["f"]
        if f != -1:
            cur = ys[f] if isinstance(f, int) else [cur if j == -1 else ys[j] for j in f]
        pfx = f"model.{i}"
        op = l["op"]
        if op == "conv":
            if l["cin"] == 3 and q.mode == "bf16" and stem_int:
                # uint8 frames on the CUDA path: exact integer pixels x bf16(w/255) on tensor cores
                w = q.w(P[pfx + ".conv.weight"] / 255.0)
                y = F.conv2d(torch.round(cur * 255.0), w, P[pfx + ".conv.bias"], stride=l["s"], padding=1)
                cur = q.act(y * torch.sigmoid(y))
            else:
                # float frames: the 3-channel stems keep fp32 weights (CUDA-core kernel)
                cur = _cv(P, q, pfx + ".conv", cur, s=l["s"], quant_w=(l["cin"] != 3))
        elif op == "elan4":
            cur = _elan4_fwd(P, q, pfx, cur, l["n"])
        elif op == "elan1":
            # detection/yolov9.py:73-80
            y = _cv(P, q, pfx + ".cv1.conv", cur)
            y0, y1 = y.chunk(2, 1)
            y2 = _cv(P, q, pfx + ".cv2.conv", y1)
            y3 = _cv(P, q, pfx + ".cv3.conv", y2)
            cur = _cv(P, q, pfx + ".cv4.conv", torch.cat([y0, y1, y2, y3], 1))
        elif op == "adown":
            # detection/yolov9.py:45-52
            t = q.act(_avg2(cur))
            x1, x2 = t.chunk(2, 1)
            x1 = _cv(P, q, pfx + ".cv1.conv", x1, s=2)
            x2 = F.max_pool2d(x2, 3, 2, 1)
            x2 = _cv(P, q, pfx + ".cv2.conv", x2)
            cur = torch.cat([x1, x2], 1)
        elif op == "aconv":
            # detection/yolov9.py:61-63
            cur = _cv(P, q, pfx + ".cv1.conv", q.act(_avg2(cur)), s=2)
        elif op == "sppelan":
            # detection/yolov9.py:143-149 with SP = max_pool2d(k=5, s=1, p=2) (:132)
            y = [_cv(P, q, pfx + ".cv1.conv", cur)]
            for _ in range(3):
                y.append(F.max_pool2d(y[-1], 5, 1, 2))
            cur = _cv(P, q, pfx + ".cv5.conv", torch.cat(y, 1))
        elif op == "upsample":
            cur = cur.repeat_interleave(2, 2).repeat_interleave(2, 3)      # :292
        elif op == "concat":
            cur = torch.cat([cur[0], cur[1]], 1)                           # :155
        elif op == "silence":
            pass
        elif op == "cblinear":
            y = _cv(P, q, pfx + ".conv", cur, act=False)                   # :228
            cur = tuple(y.split(l["c2s"], 1))
        elif op == "cbfuse":
            # detection/yolov9.py:235-245: nearest-resize the selected chunk of each source to the last input, sum
            tgt = cur[-1].shape[2:]
            acc = None
            for k_, src in enumerate(cur[:-1]):
                u = F.interpolate(src[l["idx"][k_]], size=tuple(tgt), mode="nearest")
                acc = u if acc is None else acc + u
            cur = q.act(acc + cur[-1])
        elif op == "detect":
            cur = _detect_fwd(P, q, pfx, list(cur), l["d"])
        else:
            raise ValueError(op)
        ys.append(cur)
    if taps is not None:
        taps.extend(ys)
    return cur


# ------------------------------------------------------------------------------------------------ pre / post
def _interp_axis_float(img: torch.Tensor, out: int, axis: int) -> torch.Tensor:
    """tinygrad Tensor.interpolate(mode='linear', align_corners=False) on one axis (SURVEY App. A4):
    idx = clip((i+0.5)*in/out - 0.5, 0, in-1); lo=floor, hi=ceil; lo + (hi-lo)*w."""
    n = img.shape[axis]
    if n == out:
        return img
    idx = ((torch.arange(out, dtype=torch.float32) + 0.5) * (n / out) - 0.5).clamp(0, n - 1)
    lo = idx.floor().long()
    hi = idx.ceil().long()
    w = (idx - lo.float())
    shape = [1] * img.dim()
    shape[axis] = out
    a = img.index_select(axis, lo)
    b = img.index_select(axis, hi)
    return a + (b - a) * w.reshape(shape)


def _interp_axis_u8(img: torch.Tensor, out: int, axis: int) -> torch.Tensor:
    """uint8 variant: tinygrad lerp in 7-bit fixed point with int8 wrap-around on the difference (App. A4,
    recalled behaviour, flagged): w_i = int16(w*128+0.5); out = lo + ((int8(hi-lo)*w_i + 64) >> 7)."""
    n = img.shape[axis]
    if n == out:
        return img
    idx = ((torch.arange(out, dtype=torch.float32) + 0.5) * (n / out) - 0.5).clamp(0, n - 1)
    lo = idx.floor().long()
    hi = idx.ceil().long()
    wi = ((idx - lo.float()) * 128 + 0.5).to(torch.int16).to(torch.int32)
    shape = [1] * img.dim()
    shape[axis] = out
    a = img.index_select(axis, lo).to(torch.int32)
    b = img.index_select(axis, hi).to(torch.int32)
    diff = ((b - a + 128) % 256) - 128                                      # int8 wrap
    r = a + ((diff * wi.reshape(shape) + 64) >> 7)
    return (r % 256).to(torch.uint8)


def resize(img: torch.Tensor, new_size) -> torch.Tensor:
    """utils/helpers.py:127-131: HWC -> bilinear to (new_size[1], new_size[0]); last axis (W) first, then H."""
    fn = _interp_axis_u8 if img.dtype == torch.uint8 else _interp_axis_float
    t = fn(img, new_size[0], 1)
    return fn(t, new_size[1], 0)


def letterbox_params(h, w, res, stride=32):
    """detection/yolov9.py:390-403 (auto=True, scaleup=True): returns (new_w, new_h, pad_x, pad_y)."""
    r = min(res / h, res / w)
    new_w, new_h = int(round(w * r)), int(round(h * r))
    dw, dh = (res - new_w) % stride, (res - new_h) % stride
    dw /= 2
    dh /= 2
    return new_w, new_h, int(round(dw - 0.1)), int(round(dh - 0.1))


def preprocess(image: torch.Tensor, res: int) -> torch.Tensor:
    """YOLOv9.preprocess (:390-404): HWC (uint8 or float) -> letterboxed HWC, zero padded, same dtype."""
    h, w = image.shape[:2]
    new_w, new_h, px, py = letterbox_params(h, w, res)
    img = resize(image, (new_w, new_h))
    return F.pad(img, (0, 0, px, px, py, py))


def compute_iou_matrix(boxes):
    """detection/yolov9.py:423-437, same operation order (areas, max/min, clamp, w*h, a_i + a_j - inter)."""
    x1s, y1s, x2s, y2s = boxes[..., 0], boxes[..., 1], boxes[..., 2], boxes[..., 3]
    areas = (x2s - x1s) * (y2s - y1s)
    x1 = torch.maximum(x1s[:, :, None], x1s[:, None, :])
    y1 = torch.maximum(y1s[:, :, None], y1s[:, None, :])
    x2 = torch.minimum(x2s[:, :, None], x2s[:, None, :])
    y2 = torch.minimum(y2s[:, :, None], y2s[:, None, :])
    w = (x2 - x1).clamp(min=0)
    h = (y2 - y1).clamp(min=0)
    inter = w * h
    union = areas[:, :, None] + areas[:, None, :] - inter
    return inter / union


def postprocess(output, max_det=300, conf_threshold=0.25, iou_threshold=0.45):
    """detection/yolov9.py:439-458: one-shot class-aware suppression on the stable top-300. (B,84,A)->(B,300,6)"""
    xc, yc, w, h, cls = output[:, 0], output[:, 1], output[:, 2], output[:, 3], output[:, 4:]
    x1 = xc - w / 2
    y1 = yc - h / 2
    x2 = xc + w / 2
    y2 = yc + h / 2
    probs, class_ids = cls.max(1)               # torch.max returns the first maximal index like argmax
    class_ids = cls.argmax(1)
    probs = torch.where(probs >= conf_threshold, probs, torch.zeros_like(probs))
    return postprocess_boxes(torch.stack([x1, y1, x2, y2, probs, class_ids.float()], 2), max_det, iou_threshold)


def postprocess_boxes(boxes, max_det=300, iou_threshold=0.45):
    """The selection half of postprocess: (B,A,6) [x1,y1,x2,y2,conf (0 below the threshold),class] -> (B,max_det,6)."""
    order = torch.sort(boxes[..., 4], dim=1, descending=True, stable=True)[1][:, :max_det]
    boxes = torch.gather(boxes, 1, order.unsqueeze(-1).expand(-1, -1, 6))
    ious = torch.triu(compute_iou_matrix(boxes[:, :, :4]), diagonal=1)
    cid = boxes[:, :, -1]
    same = cid[:, :, None] == cid[:, None, :]
    high = (ious > iou_threshold) & same
    keep = high.sum(1) == 0
    return boxes * keep.unsqueeze(-1)


def scale_boxes(img1_shape, preds, img0_shape):
    """detection/yolov9.py:406-421: undo letterbox with FLOAT pads, clip to the original frame."""
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    pad_x = (img1_shape[1] - img0_shape[1] * gain) / 2
    pad_y = (img1_shape[0] - img0_shape[0] * gain) / 2
    out = preds.clone()
    b = out[..., :4]
    b[..., [0, 2]] -= pad_x
    b[..., [1, 3]] -= pad_y
    b /= gain
    b[..., [0, 2]] = b[..., [0, 2]].clamp(0, img0_shape[1])
    b[..., [1, 3]] = b[..., [1, 3]].clamp(0, img0_shape[0])
    return out


def detect(size: str, P, frames, res: int, quant=None, bgr_swap=True, stem_int=None) -> torch.Tensor:
    """YOLOv9.__call__ (:375-388) for a batch of same-shape HWC BGR frames (uint8 or float32).

    Returns (B,300,6) [x1,y1,x2,y2,conf,cls] in original-frame pixels (the reference returns image 0 only)."""
    if frames.dim() == 3:
        frames = frames.unsqueeze(0)
    pre = torch.stack([preprocess(f, res) for f in frames])
    x = pre.flip(-1) if bgr_swap else pre
    x = x.permute(0, 3, 1, 2).to(torch.float32) / 255.0
    with torch.no_grad():
        raw = forward_raw(size, P, x, quant=quant, stem_int=(frames.dtype == torch.uint8) if stem_int is None else stem_int)
        preds = postprocess(raw)
    return scale_boxes(pre.shape[1:3], preds, frames.shape[1:3])


# ------------------------------------------------------------------------------------------------ weights
def synthetic_frames(B: int, H: int, W: int, seed: int = 0) -> torch.Tensor:
    """Seeded uint8 BGR frames with structure (gradient + random filled rectangles + mild noise), so features vary
    with position the way a camera image's do (uniform noise averages out to position-independent features)."""
    g = torch.Generator().manual_seed(1000 + seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    frames = []
    for b in range(B):
        ph = torch.rand(3, generator=g)
        img = torch.stack([(yy * (0.5 + ph[0]) + xx * ph[1]) % 1.0, (xx * (0.5 + ph[1]) + 0.3 * yy) % 1.0,
                           (0.5 * yy * xx + ph[2]) % 1.0], -1) * 160 + 40
        for _ in range(24):
            rh = int(torch.randint(max(H // 24, 4), max(H // 3, 8), (1,), generator=g))
            rw = int(torch.randint(max(W // 24, 4), max(W // 3, 8), (1,), generator=g))
            y0 = int(torch.randint(0, max(H - rh, 1), (1,), generator=g))
            x0 = int(torch.randint(0, max(W - rw, 1), (1,), generator=g))
            img[y0:y0 + rh, x0:x0 + rw] = torch.rand(3, generator=g) * 255
        img = img + torch.randn(H, W, 3, generator=g) * 6
        frames.append(img.clamp(0, 255).to(torch.uint8))
    return torch.stack(frames)


def synthetic_weights(size: str, seed: int = 0, calib: torch.Tensor | None = None, anchors_frac=0.04,
                      ) -> Dict[str, torch.Tensor]:
    """Seeded weights with the reference's state-dict names.

    Every conv is normalised per output channel on one calibration image (data-dependent init: weight /= std_c,
    bias = -mean_c/std_c + N(0,0.1)), so all ~60 sequential layers stay numerically relevant and position
    dependent (a plain N(0,2/fan_in) draw collapses to bias-dominated constants).  The class head is shifted so
    about `anchors_frac` of the anchors pass the 0.25 threshold on the calibration image (top-300 selection and
    the class-aware suppression are both exercised).  DFL weight = arange(16) as in the reference checkpoint.
    `calib`: (1,3,H,W) fp32 RGB in [0,1]; default = synthetic_frames(1,320,320,seed) preprocessed."""
    g = torch.Generator().manual_seed(seed)
    P: Dict[str, torch.Tensor] = {}
    table = conv_table(size)
    for name, cin, cout, k, s, grp, act in table:
        fan_in = (cin // grp) * k * k
        P[name + ".weight"] = torch.randn(cout, cin // grp, k, k, generator=g) * (1.0 / fan_in) ** 0.5
        P[name + ".bias"] = torch.zeros(cout)
    det = max(int(n.split(".")[1]) for n, *_ in table)
    P[f"model.{det}.dfl.conv.weight"] = torch.arange(16, dtype=torch.float32).reshape(1, 16, 1, 1)
    if calib is None:
        calib = synthetic_frames(2, 320, 320, seed).flip(-1).permute(0, 3, 1, 2).float() / 255.0
    # z-quantile such that P(any of 80 classes passes) = anchors_frac
    p_pair = 1.0 - (1.0 - anchors_frac) ** (1.0 / 80.0)
    zq = float(torch.distributions.Normal(0.0, 1.0).icdf(torch.tensor(1.0 - p_pair)))
    scaled = set()
    global _cv
    orig_cv = _cv

    def cv_cal(P_, q, name, x_, s=1, g=1, act=True, res=None, quant_w=True, store=True):
        if name not in scaled:
            w = P_[name + ".weight"]
            y = F.conv2d(x_, w, None, stride=s, padding=w.shape[-1] // 2, groups=g)
            is_cls = ".cv3." in name and name.endswith(".2")
            is_dfl = ".cv2." in name and name.endswith(".2")
            shift = torch.randn(w.shape[0], generator=globals()["_gen"]) * 0.1
            if is_cls or is_dfl:
                # heads: centre/scale the logits over the whole map (one scalar pair per head -> still contractive)
                mu, sd = y.mean(), y.std().clamp(min=1e-6)
                gain = 0.35 if is_cls else 1.5
                if is_cls:   # threshold logit(0.25) sits at the z-quantile giving ~anchors_frac passing anchors
                    shift = shift * 2 + (math.log(0.25 / 0.75) - gain * zq)
                P_[name + ".weight"] = w * (gain / sd)
                P_[name + ".bias"] = -mu / sd * gain + shift
            else:
                # body: one scalar per conv so the pre-activation RMS is 1 (keeps relative perturbations O(1) per
                # layer; per-channel whitening would divide by tiny stds and make the net chaotic)
                rms = y.pow(2).mean().sqrt().clamp(min=1e-6)
                P_[name + ".weight"] = w / rms
                P_[name + ".bias"] = shift
            scaled.add(name)
        return orig_cv(P_, q, name, x_, s=s, g=g, act=act, res=res, quant_w=quant_w, store=store)

    globals()["_gen"] = g
    _cv = cv_cal
    try:
        with torch.no_grad():
            forward_raw(size, P, calib)
    finally:
        _cv = orig_cv
        globals().pop("_gen", None)
    return P


def count_params(P) -> int:
    return sum(int(v.numel()) for v in P.values())


def conv_flops(size: str, h: int, w: int) -> float:
    """2*MACs over all convs for one (h,w) input — must reproduce SURVEY.md §6 (c: 102.14 GFLOP at 640^2)."""
    P = {}
    for name, cin, cout, k, s, grp, act in conv_table(size):
        P[name + ".weight"] = torch.empty(cout, cin // grp, k, k, device="meta")
        P[name + ".bias"] = torch.empty(cout, device="meta")
    total = [0.0]
    global _cv
    orig_cv = _cv

    def cv_count(P_, q, name, x_, s=1, g=1, act=True, res=None, quant_w=True, store=True):
        wt = P_[name + ".weight"]
        k = wt.shape[-1]
        ho = (x_.shape[2] + 2 * (k // 2) - k) // s + 1
        wo = (x_.shape[3] + 2 * (k // 2) - k) // s + 1
        total[0] += 2.0 * x_.shape[0] * ho * wo * wt.shape[0] * wt.shape[1] * k * k
        return torch.empty(x_.shape[0], wt.shape[0], ho, wo, device="meta")

    _cv = cv_count
    try:
        det = max(int(n.split(".")[1]) for n, *_ in conv_table(size))
        P[f"model.{det}.dfl.conv.weight"] = torch.empty(1, 16, 1, 1, device="meta")
        try:
            forward_raw(size, P, torch.empty(1, 3, h, w, device="meta"))
        except (RuntimeError, NotImplementedError):
            pass  # the detect tail (anchors on CPU vs meta) is irrelevant for counting convs
    finally:
        _cv = orig_cv
    return total[0]
