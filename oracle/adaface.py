"""CPU oracle of the reference's AdaFace IR-50 face embedder (/root/reference/models/adaface.py), in torch.

* `forward(P, faces)`: fp32 restatement of ADAFACE.__call__ (:79-96) on a batch, one face per reference call.
* `forward_folded(F, faces, bf16=...)`: the folded network that libclearcam_b200 runs (clearcam_b200/models/adaface.py
  `fold_state_dict`), in float64 (the fold check) or as the bf16 mirror that rounds exactly where the GPU path stores bf16.
* `state_dict_keys()`: the reference's key names, walked from a restatement of its attribute tree as tinygrad's
  `get_state_dict` walks it.
* `synthetic_weights(seed)`: seeded weights whose activations stay O(1) through the 24 residual blocks.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as Fn

EPS = 1e-5                                  # tinygrad nn.BatchNorm default
SIZES = [[64, 64, 2], [64, 64, 1], [64, 64, 1], [64, 128, 2], [128, 128, 1], [128, 128, 1], [128, 128, 1], [128, 256, 2]] + \
    [[256, 256, 1]] * 13 + [[256, 512, 2], [512, 512, 1], [512, 512, 1]]   # adaface.py:61


# ---- the attribute tree (adaface.py:12-75) and tinygrad's get_state_dict walk over it
class _T:
    """Stands for a tinygrad Tensor leaf."""


class _BatchNorm:           # tinygrad.nn.BatchNorm(sz, eps, affine, track_running_stats, momentum)
    def __init__(self, affine=True):
        self.eps, self.track_running_stats, self.momentum = EPS, True, 0.1
        self.weight = _T() if affine else None
        self.bias = _T() if affine else None
        self.num_batches_tracked = _T()
        self.running_mean, self.running_var = _T(), _T()


class _Conv2d:              # tinygrad.nn.Conv2d(..., bias=False)
    def __init__(self, bias=False):
        self.kernel_size, self.stride, self.padding = None, None, None
        self.weight = _T()
        self.bias = _T() if bias else None


class _Linear:
    def __init__(self):
        self.weight, self.bias = _T(), _T()


class _MaxPool2d:           # adaface.py:4-10: no tensors
    def __init__(self):
        self.kernel_size, self.stride, self.padding = 1, 1, 0


class _Seq:                 # adaface.py:12-22: the blocks live in the attribute `list`
    def __init__(self, size):
        self.list = [None] * size


class _Block:               # BasicBlockIR_tiny.__init__, adaface.py:25-41
    def __init__(self, cin, depth, stride):
        self.in_channel, self.depth, self.stride = cin, depth, stride
        self.res_layer0 = _BatchNorm()
        self.conv_layer0 = _Conv2d()
        self.res_layer1 = _BatchNorm()
        self.prelu_weight = _T()
        self.conv_layer1 = _Conv2d()
        self.res_layer2 = _BatchNorm()
        if depth == cin:
            self.shortcut_layer = _MaxPool2d()
        else:
            self.shortcut_layer0 = _Conv2d()
            self.shortcut_layer1 = _BatchNorm()


class _AdaFace:             # ADAFACE.__init__, adaface.py:64-75
    def __init__(self):
        self.linear = _Linear()
        self.bn = _BatchNorm()
        self.bn2 = _BatchNorm(affine=False)
        self.prelu_weight = _T()
        self.conv0 = _Conv2d()
        self.bn0 = _BatchNorm()
        self.body = _Seq(24)
        for i in range(24):
            self.body.list[i] = _Block(*SIZES[i])


def _walk(obj, prefix=""):
    """tinygrad.nn.state.get_state_dict: a Tensor is a leaf; lists / tuples enumerate; objects walk their __dict__."""
    if isinstance(obj, _T):
        return [prefix.strip(".")]
    if isinstance(obj, (list, tuple)):
        return [k for i, x in enumerate(obj) for k in _walk(x, f"{prefix}{i}.")]
    if hasattr(obj, "__dict__"):
        return [k for n, v in obj.__dict__.items() for k in _walk(v, f"{prefix}{n}.")]
    return []


def state_dict_keys():
    return _walk(_AdaFace())


# ---- synthetic weights
def synthetic_weights(seed: int = 0):
    """Seeded weights under the reference's names.  He-scaled convs, BN statistics and affines near what a trained IR-50 has
    (gammas ~1, small means, variances ~1), PReLU slopes in [0.05, 0.35] and res_layer2 gammas ~0.15 so that the residual
    stream stays O(1) through the 24 blocks."""
    g = torch.Generator().manual_seed(seed)

    def rn(*s, std=1.0):
        return torch.randn(*s, generator=g) * std

    def ru(lo, hi, *s):
        return lo + (hi - lo) * torch.rand(*s, generator=g)

    P = {}

    def bn(p, n, gamma=(0.8, 1.2), affine=True):
        if affine:
            P[f"{p}.weight"] = ru(*gamma, n)
            P[f"{p}.bias"] = rn(n, std=0.1)
        P[f"{p}.num_batches_tracked"] = torch.zeros(1)
        P[f"{p}.running_mean"] = rn(n, std=0.1)
        P[f"{p}.running_var"] = ru(0.5, 1.5, n)

    def conv(p, o, i, k):
        P[f"{p}.weight"] = rn(o, i, k, k, std=(2.0 / (i * k * k)) ** 0.5)

    P["linear.weight"] = rn(512, 512 * 49, std=(1.0 / (512 * 49)) ** 0.5)
    P["linear.bias"] = rn(512, std=0.05)
    bn("bn", 512)
    bn("bn2", 512, affine=False)
    P["prelu_weight"] = ru(0.05, 0.35, 64)
    conv("conv0", 64, 3, 3)
    bn("bn0", 64)
    for i, (cin, d, _) in enumerate(SIZES):
        p = f"body.list.{i}"
        bn(f"{p}.res_layer0", cin)
        conv(f"{p}.conv_layer0", d, cin, 3)
        bn(f"{p}.res_layer1", d)
        P[f"{p}.prelu_weight"] = ru(0.05, 0.35, d)
        conv(f"{p}.conv_layer1", d, d, 3)
        bn(f"{p}.res_layer2", d, gamma=(0.1, 0.2))
        if cin != d:
            conv(f"{p}.shortcut_layer0", d, cin, 1)
            bn(f"{p}.shortcut_layer1", d)
    return P


def synthetic_faces(B: int, seed: int = 0) -> torch.Tensor:
    """uint8 [B,112,112,3]: smooth random blobs plus noise, full 0..255 range."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(B, 3, 7, 7, generator=g)
    x = Fn.interpolate(low, size=(112, 112), mode="bicubic", align_corners=False) * 255
    x = x + torch.randn(B, 3, 112, 112, generator=g) * 20
    return x.clamp(0, 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


# ---- the reference's forward (adaface.py:45-57, 79-96), fp32
def _bn_eval(x, P, p, affine=True):
    """tinygrad BatchNorm eval: (x - mean) * (weight * rsqrt(var + eps)) + bias."""
    inv = (P[f"{p}.running_var"].to(x.dtype) + EPS).rsqrt()
    w = P[f"{p}.weight"].to(x.dtype) * inv if affine else inv
    y = (x - P[f"{p}.running_mean"].to(x.dtype).view(1, -1, *([1] * (x.dim() - 2)))) * w.view(1, -1, *([1] * (x.dim() - 2)))
    return y + P[f"{p}.bias"].to(x.dtype).view(1, -1, *([1] * (x.dim() - 2))) if affine else y


def _prelu(x, w):
    return torch.where(x > 0, x, w.to(x.dtype).view(1, -1, 1, 1) * x)         # :54, :86


def forward(P, faces: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """faces uint8 [B,112,112,3] -> [B,512]: row b is ADAFACE()(faces[b]) (each face its own call, so its own norm)."""
    x = faces.to(dtype)
    x = ((x.flip(-1) / 255.0) - 0.5) / 0.5                                       # :81
    x = x.permute(0, 3, 1, 2)                                                    # :82
    W = {k: v.to(dtype) for k, v in P.items()}
    x = _prelu(_bn_eval(Fn.conv2d(x, W["conv0.weight"], padding=1), W, "bn0"), W["prelu_weight"])
    for i, (cin, d, s) in enumerate(SIZES):                                      # BasicBlockIR_tiny.__call__, :45-57
        p = f"body.list.{i}"
        sc = x[:, :, ::s, ::s] if cin == d else \
            _bn_eval(Fn.conv2d(x, W[f"{p}.shortcut_layer0.weight"], stride=s), W, f"{p}.shortcut_layer1")
        y = Fn.conv2d(_bn_eval(x, W, f"{p}.res_layer0"), W[f"{p}.conv_layer0.weight"], padding=1)
        y = _prelu(_bn_eval(y, W, f"{p}.res_layer1"), W[f"{p}.prelu_weight"])
        y = _bn_eval(Fn.conv2d(y, W[f"{p}.conv_layer1.weight"], stride=s, padding=1), W, f"{p}.res_layer2")
        x = y + sc
    x = _bn_eval(x, W, "bn").reshape(x.shape[0], -1)                            # :89-90, NCHW flatten
    x = Fn.linear(x, W["linear.weight"], W["linear.bias"])
    x = _bn_eval(x, W, "bn2", affine=False)
    return x / (x * x).sum(-1, keepdim=True).sqrt()                              # :93-95, per face


# ---- the folded network (what csrc/adaface.cu runs)
def class_map(H: int, W: int) -> torch.Tensor:
    """[H,W] border class 3 * (top 0 / interior 1 / bottom 2) + (left 0 / interior 1 / right 2)."""
    r = torch.ones(H, dtype=torch.long)
    c = torch.ones(W, dtype=torch.long)
    r[0], r[-1], c[0], c[-1] = 0, 2, 0, 2
    return 3 * r[:, None] + c[None, :]


def _bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(x.dtype)


def forward_folded(F, faces: torch.Tensor, bf16: bool = False, dtype=torch.float64, taps: bool = False):
    """The folded network on uint8 faces [B,112,112,3] -> [B,512] (and, with taps=True, the list of the stem's and every
    block's NCHW output and the pre-norm linear output, as cc_face_layer_output numbers them).  bf16=True is the GPU path's
    mirror: weights rounded fp32 -> bf16 as cc_face_create does, every stored activation rounded to bf16 (the shortcut
    before conv_layer1 adds it), fp32 arithmetic, the linear's output kept in fp32."""
    if bf16:
        dtype = torch.float32

    def w(name, conv=True):
        t = torch.as_tensor(np.asarray(F[name], np.float32) if bf16 else np.asarray(F[name])).to(dtype)
        if bf16 and conv:
            t = _bf16(t)
        return t

    def st(x):                     # a store of the GPU path
        return _bf16(x) if bf16 else x

    def conv3(x, name, stride=1):  # [O][3][3][I] -> NCHW conv
        return Fn.conv2d(x, w(name).permute(0, 3, 1, 2), stride=stride, padding=1)

    def prelu_cls(y, base):
        cls = w(f"{base}.cls", False)                                            # [9, O]
        y = y + cls[class_map(*y.shape[-2:])].permute(2, 0, 1)[None]
        return torch.where(y > 0, y, w(f"{base}.slope", False).view(1, -1, 1, 1) * y)

    out = []
    x = faces.to(dtype).permute(0, 3, 1, 2)                                      # raw 0..255, image channel order
    x = st(prelu_cls(conv3(x, "stem.w"), "stem"))
    out.append(x)
    for i, (cin, d, s) in enumerate(SIZES):
        q = f"body.{i}"
        t = st(prelu_cls(conv3(x, f"{q}.c0.w"), f"{q}.c0"))
        if f"{q}.sc.w" in F:
            sc = st(Fn.conv2d(x, w(f"{q}.sc.w")[:, :, None, None], stride=s) + w(f"{q}.sc.b", False).view(1, -1, 1, 1))
        else:
            sc = x
        x = st(conv3(t, f"{q}.c1.w", s) + w(f"{q}.c1.b", False).view(1, -1, 1, 1) + sc)
        out.append(x)
    feat = x.permute(0, 2, 3, 1).reshape(x.shape[0], -1) @ w("linear.w").T + w("linear.b", False)
    out.append(feat)
    emb = feat / (feat * feat).sum(-1, keepdim=True).sqrt()
    return (emb, out) if taps else emb
