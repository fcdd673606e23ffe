"""The AdaFace oracle, the host weight fold and the face helpers of ObjectFinder, without a GPU.

* The oracle (oracle/adaface.py `forward`) equals an independent torch.nn build of the same network in eval mode.
* The folded network (clearcam_b200.models.adaface `fold_state_dict`, what cc_face_create runs) evaluated in float64 equals
  the unfolded float64 oracle to ~1e-12, at border pixels too; a naive fold (the interior bias at every pixel) and a
  row-major instead of NCHW linear permutation each fail that check.
* The key names are the reference's (tinygrad get_state_dict over its attribute tree) and round-trip through the fold.
* preprocess_face returns the RGB image of a 112x112 file and raises otherwise.
"""
import cv2
import numpy as np
import pytest
import torch
import torch.nn as nn

from clearcam_b200._lib import CCError
from clearcam_b200.models import adaface as ca
from clearcam_b200.models.objects import ObjectFinder
from oracle import adaface as oa


@pytest.fixture(scope="module")
def weights():
    return oa.synthetic_weights(seed=7)


@pytest.fixture(scope="module")
def faces():
    return oa.synthetic_faces(2, seed=3)


@pytest.fixture(scope="module")
def unfolded(weights, faces):
    with torch.no_grad():
        return oa.forward(weights, faces, dtype=torch.float64)


class _TorchBlock(nn.Module):
    def __init__(self, cin, d, s):
        super().__init__()
        self.cin, self.d, self.s = cin, d, s
        self.bn0, self.c0, self.bn1 = nn.BatchNorm2d(cin, eps=1e-5), nn.Conv2d(cin, d, 3, 1, 1, bias=False), nn.BatchNorm2d(d, eps=1e-5)
        self.act, self.c1, self.bn2 = nn.PReLU(d), nn.Conv2d(d, d, 3, s, 1, bias=False), nn.BatchNorm2d(d, eps=1e-5)
        if cin == d:
            self.sc = nn.MaxPool2d(1, s)
        else:
            self.sc = nn.Sequential(nn.Conv2d(cin, d, 1, s, bias=False), nn.BatchNorm2d(d, eps=1e-5))

    def forward(self, x):
        return self.bn2(self.c1(self.act(self.bn1(self.c0(self.bn0(x)))))) + self.sc(x)


def _torch_net(P):
    """The same network from torch.nn modules, weights copied from the reference's names."""
    stem = nn.Sequential(nn.Conv2d(3, 64, 3, 1, 1, bias=False), nn.BatchNorm2d(64, eps=1e-5), nn.PReLU(64))
    blocks = nn.ModuleList([_TorchBlock(*s) for s in oa.SIZES])
    bn, lin, bn2 = nn.BatchNorm2d(512, eps=1e-5), nn.Linear(512 * 49, 512), nn.BatchNorm1d(512, eps=1e-5, affine=False)

    def set_bn(m, p, affine=True):
        if affine:
            m.weight.data.copy_(P[f"{p}.weight"]); m.bias.data.copy_(P[f"{p}.bias"])
        m.running_mean.copy_(P[f"{p}.running_mean"]); m.running_var.copy_(P[f"{p}.running_var"])

    stem[0].weight.data.copy_(P["conv0.weight"]); set_bn(stem[1], "bn0"); stem[2].weight.data.copy_(P["prelu_weight"])
    for i, b in enumerate(blocks):
        p = f"body.list.{i}"
        set_bn(b.bn0, f"{p}.res_layer0"); b.c0.weight.data.copy_(P[f"{p}.conv_layer0.weight"]); set_bn(b.bn1, f"{p}.res_layer1")
        b.act.weight.data.copy_(P[f"{p}.prelu_weight"]); b.c1.weight.data.copy_(P[f"{p}.conv_layer1.weight"])
        set_bn(b.bn2, f"{p}.res_layer2")
        if b.cin != b.d:
            b.sc[0].weight.data.copy_(P[f"{p}.shortcut_layer0.weight"]); set_bn(b.sc[1], f"{p}.shortcut_layer1")
    set_bn(bn, "bn"); lin.weight.data.copy_(P["linear.weight"]); lin.bias.data.copy_(P["linear.bias"]); set_bn(bn2, "bn2", False)
    mods = nn.ModuleList([stem, blocks, bn, lin, bn2]).double().eval()

    def run(faces):
        x = ((faces.double().flip(-1) / 255.0) - 0.5) / 0.5
        x = stem(x.permute(0, 3, 1, 2))
        for b in blocks:
            x = b(x)
        x = bn2(lin(bn(x).flatten(1)))
        return x / x.norm(dim=-1, keepdim=True)
    return mods, run


def test_oracle_matches_torch_nn(weights, faces, unfolded):
    _, run = _torch_net(weights)
    with torch.no_grad():
        want = run(faces)
        got32 = oa.forward(weights, faces)
    assert (unfolded - want).abs().max() < 1e-12
    assert (got32.double() - want).abs().max() < 1e-5


def test_folded_equals_unfolded_at_every_pixel(weights, faces, unfolded):
    F = ca.fold_state_dict(weights)
    with torch.no_grad():
        emb, taps = oa.forward_folded(F, faces, taps=True)
        # the stem by hand: conv0 -> bn0 -> PReLU on the normalised, channel-flipped input, every pixel including the borders
        x = (((faces.double().flip(-1) / 255.0) - 0.5) / 0.5).permute(0, 3, 1, 2)
        W = {k: v.double() for k, v in weights.items()}
        stem = oa._prelu(oa._bn_eval(torch.nn.functional.conv2d(x, W["conv0.weight"], padding=1), W, "bn0"), W["prelu_weight"])
    assert (taps[0] - stem).abs().max() < 1e-11
    assert (taps[0][..., 0, :] - stem[..., 0, :]).abs().max() < 1e-11 and (taps[0][..., :, -1] - stem[..., :, -1]).abs().max() < 1e-11
    assert (emb - unfolded).abs().max() < 1e-10


def test_naive_fold_and_row_major_linear_fail(weights, faces, unfolded):
    F = ca.fold_state_dict(weights)
    naive = dict(F)
    for k in [k for k in F if k.endswith(".cls")]:
        naive[k] = np.repeat(F[k][4:5], 9, axis=0)               # the interior bias at every pixel
    W = ca._f64(weights["linear.weight"])
    sb, _ = ca._bn(weights, "bn")
    s2, _ = ca._bn(weights, "bn2", affine=False)
    rowmajor = dict(F)
    rowmajor["linear.w"] = s2[:, None] * W * np.repeat(sb, 49)[None]   # folded, but the columns left in NCHW order
    with torch.no_grad():
        e_naive = oa.forward_folded(naive, faces)
        e_row = oa.forward_folded(rowmajor, faces)
    assert (e_naive - unfolded).abs().max() > 1e-4
    assert (e_row - unfolded).abs().max() > 1e-3


def test_key_names_round_trip(weights):
    keys = ca.state_dict_keys()
    assert keys == oa.state_dict_keys()
    assert sorted(weights) == sorted(keys)
    assert "body.list.3.shortcut_layer0.weight" in keys and "body.list.0.shortcut_layer0.weight" not in keys
    assert "bn2.weight" not in keys and "conv0.bias" not in keys
    # num_batches_tracked is ignored; any other missing tensor is named
    lean = {k: v for k, v in weights.items() if not k.endswith("num_batches_tracked")}
    F = ca.fold_state_dict(lean)
    assert set(F) >= {"stem.w", "stem.cls", "stem.slope", "linear.w", "linear.b", "body.0.sc.w", "body.23.c1.b"}
    assert "body.1.sc.w" not in F
    with pytest.raises(CCError, match="res_layer1"):
        ca.fold_state_dict({k: v for k, v in weights.items() if k != "body.list.5.res_layer1.running_var"})


def test_preprocess_face_rgb_and_refusal(tmp_path):
    rng = np.random.default_rng(0)
    bgr = rng.integers(0, 256, (112, 112, 3), dtype=np.uint8)
    ok, png = cv2.imencode(".png", bgr)
    f = ObjectFinder()
    got = f.preprocess_face(png.tobytes())
    assert got.shape == (112, 112, 3) and np.array_equal(got, bgr[:, :, ::-1])
    ok, big = cv2.imencode(".png", rng.integers(0, 256, (160, 120, 3), dtype=np.uint8))
    with pytest.raises(CCError, match="face detection"):
        f.preprocess_face(big.tobytes())
