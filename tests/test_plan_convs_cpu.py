"""The per-op checks of tests/test_plan_convs_gpu.py see the launches they are there to catch (no GPU needed).

Two conv ops on CPU tensors in a small workspace, laid out as a plan lays them out, over a batch of B = 7 images that are
copies of 3 distinct ones: a 3x3 / stride-2 SiLU conv between channel slices of wider buffers with a residual, and an
activation-free 1x1 conv of 3 x 384 x 64 outputs.  Then the face embedder's PReLU conv (a [9][Cout] border-class bias table
and per-channel slopes) and the CLIP patch embedding's form: a GEMM into fp32 tokens 1..L-1 of each image of an L-token
stream (out_ns = L).  Their exact results (the float64 conv rounded to nearest bf16 / fp32) pass every check; each corruption
below is flagged by the check named with it."""
import ctypes
import types

import pytest
import torch
import torch.nn.functional as F

import test_conv_gpu as tc
import test_plan_convs_gpu as tp
from clearcam_b200._lib import CC_CONV_OP_GEMM, CCError, cc_conv_op, cc_slice, check, lib
from oracle.adaface import class_map

B = 7
BF16 = torch.bfloat16


def _layout():
    """(workspace before the ops, conv op, 1x1 op): buffers back to back, the inputs and residual filled."""
    g = torch.Generator().manual_seed(11)
    sizes = {"x": (32, 48, 48), "o": (16, 24, 64), "r": (16, 24, 32), "x2": (16, 24, 64), "o2": (16, 24, 64)}
    off, offs = 0, {}
    for k, (H, W, cs) in sizes.items():
        offs[k] = off
        off += B * H * W * cs * 2
    ws = torch.zeros(off, dtype=torch.uint8)

    def buf(k, co, C):
        H, W, cs = sizes[k]
        return tp.Slice(offs[k], cs, co, C, B, H, W, 0)

    def fill(s):
        v = torch.randn((tp.REPS,) + tuple(tp.sbuf(ws, s).shape[1:]), generator=g)
        tp.sbuf(ws, s).copy_(v[torch.arange(B) % tp.REPS].to(BF16))

    def op(in_, out, res, k, stride, act):
        Cout, Cin = out.C, in_.C
        w = (torch.randn(Cout, k, k, Cin, generator=g) * (k * k * Cin) ** -0.5).to(BF16)
        bias = torch.randn(Cout, generator=g) * 0.5
        return types.SimpleNamespace(kind=CC_CONV_OP_GEMM, name=f"{k}x{k}/s{stride}", in_=in_, out=out, res=res, w=w, bias=bias,
                                     k=k, stride=stride, groups=1, act=act, pre=None, store1=1, slope=None)

    conv = op(buf("x", 16, 32), buf("o", 16, 32), buf("r", 0, 32), 3, 2, 1)
    conv1 = op(buf("x2", 0, 64), buf("o2", 0, 64), None, 1, 1, 0)
    for s in (conv.in_, conv.res, conv1.in_):
        fill(s)
    return ws, conv, conv1


def _ref(ws, op):
    res = None if op.res is None else tp.sview(ws, op.res)
    return tp.ref64(tp.sview(ws, op.in_), op.w, op.bias, op.k, op.stride, 1, op.act, res)


def _exact(snap, op):
    after = snap.clone()
    tp.sview(after, op.out).copy_(_ref(snap, op)[1].float().to(BF16))
    return after


def _check(snap, after, op):
    tp.check_op(op, snap, after, {})


def test_exact_results_pass():
    snap, conv, conv1 = _layout()
    _check(snap, _exact(snap, conv), conv)
    _check(snap, _exact(snap, conv1), conv1)


def _tile(y, img, h0, w0):
    """the 128-pixel tile box of 8 rows x 16 columns at (h0, w0) of image img"""
    return y[img, h0:h0 + 8, w0:w0 + 16]


def _shifted_tap(snap, op, after):
    """image 5 (a copy of image 2): one tile computed with the top-left tap reading one column to the right"""
    x = tp.sview(snap, op.in_)[5:6].double().permute(0, 3, 1, 2)
    wt = torch.zeros_like(op.w, dtype=torch.float64)
    wt[:, 0, 0] = op.w[:, 0, 0].double()
    wt = wt.permute(0, 3, 1, 2)
    delta = F.conv2d(torch.roll(x, -1, 3), wt, None, 2, 1) - F.conv2d(x, wt, None, 2, 1)
    z = _ref(snap, op)[0][5] + delta[0].permute(1, 2, 0)
    y = F.silu(z) + tp.sview(snap, op.res)[5].double()
    assert (_tile(y[None], 0, 0, 0) - _tile(_ref(snap, op)[1], 5, 0, 0)).abs().max() > 1e-2
    _tile(tp.sview(after, op.out), 5, 0, 0).copy_(_tile(y[None], 0, 0, 0).float().to(BF16))


def _no_bias(snap, op, after):
    """images 1 and its copy 4: one tile without the bias (the copies still agree, so only the float64 check can see it)"""
    z = _ref(snap, op)[0] - op.bias.double()
    y = F.silu(z) + tp.sview(snap, op.res).double()
    for img in (1, 4):
        _tile(tp.sview(after, op.out), img, 8, 8).copy_(_tile(y, img, 8, 8).float().to(BF16))


def _past_the_slice(snap, op, after):
    """one channel written past co + C (the next channel of the wider output buffer), at one pixel"""
    o = op.out
    tp.sbuf(after, o)[0, 3, 4, o.co + o.C] = 1.0


def _unwritten(snap, op, after):
    """one output element left as it was before the op: the NaN the test fills outputs with"""
    tp.sview(after, op.out)[6, 15, 23, 31] = float("nan")


def _truncated(snap, op, after):
    """every output of the activation-free 1x1 truncated to bf16 instead of rounded to nearest"""
    tp.sview(after, op.out).copy_(tc.bf16_trunc(_ref(snap, op)[1]).float().to(BF16))


CORRUPTIONS = [pytest.param(_shifted_tap, 0, r"\(b\) image 5 differs from its copy, image 2", id="shifted-tap-image-5"),
               pytest.param(_no_bias, 0, r"\(a\) worst \|err\|/bar", id="tile-without-bias"),
               pytest.param(_past_the_slice, 0, r"\(d\) workspace byte", id="channel-past-the-slice"),
               pytest.param(_truncated, 1, r"\(a\) rounding bias", id="truncated-bf16-store"),
               pytest.param(_unwritten, 0, r"\(c\) output not finite", id="unwritten-element")]


@pytest.mark.parametrize("corrupt,which,flag", CORRUPTIONS)
def test_corruption_is_flagged(corrupt, which, flag):
    snap, conv, conv1 = _layout()
    op = (conv, conv1)[which]
    after = _exact(snap, op)
    _check(snap, after, op)
    corrupt(snap, op, after)
    with pytest.raises(AssertionError, match=flag):
        _check(snap, after, op)


# ------------------------------------------------------------------------------------------------ PReLU and out_ns ops
HP, WP, CP = 12, 20, 32                  # the PReLU conv's map: a 16-channel input, 32 outputs
PN, KP, WT = 9, 64, 32                   # the patch GEMM: 9 patches of 64 values per image into a 32-wide stream of L = 10


def _face_and_patch_layout():
    """(workspace before the ops, PReLU conv op, patch GEMM op)."""
    g = torch.Generator().manual_seed(12)
    L = PN + 1
    sizes = {"x": B * HP * WP * 16 * 2, "o": B * HP * WP * CP * 2, "p": B * PN * KP * 2, "s": B * L * WT * 4}
    off, offs = 0, {}
    for k, n in sizes.items():
        offs[k] = off
        off += n
    ws = torch.zeros(off, dtype=torch.uint8)
    xin = tp.Slice(offs["x"], 16, 0, 16, B, HP, WP, 0)
    v = torch.randn(tp.REPS, HP, WP, 16, generator=g)
    tp.sview(ws, xin).copy_(v[torch.arange(B) % tp.REPS].to(BF16))
    slope = torch.cat([torch.rand(CP - 4, generator=g) * 0.5, torch.tensor([1.5, -0.3, 0.0, 2.0])])
    prelu = types.SimpleNamespace(kind=CC_CONV_OP_GEMM, name="prelu 3x3", in_=xin, out=tp.Slice(offs["o"], CP, 0, CP, B, HP, WP, 0),
                                  res=None, w=(torch.randn(CP, 3, 3, 16, generator=g) / 12).to(BF16),
                                  bias=torch.randn(9, CP, generator=g), slope=slope, k=3, stride=1, groups=1, act=tp.ACT_PRELU,
                                  pre=None, store1=1)
    pin = tp.Slice(offs["p"], KP, 0, KP, B, 1, PN, 0)
    v = torch.randn(tp.REPS, 1, PN, KP, generator=g)
    tp.sview(ws, pin).copy_(v[torch.arange(B) % tp.REPS].to(BF16))
    stream = tp.Slice(offs["s"], WT, 0, WT, B, 1, L, 1)
    tp.sview(ws, stream).copy_(torch.randn(B, 1, L, WT, generator=g))      # what the stream held before (token 0 included)
    patch = types.SimpleNamespace(kind=CC_CONV_OP_GEMM, name="patch_embed", in_=pin,
                                  out=tp.Slice(offs["s"] + WT * 4, WT, 0, WT, B, 1, PN, 1, L), res=None,
                                  w=(torch.randn(WT, 1, 1, KP, generator=g) / 8).to(BF16), bias=None, slope=None, k=1, stride=1,
                                  groups=1, act=0, pre=None, store1=1)
    return ws, prelu, patch


def _ref2(ws, op, cls=None):
    """float64 (z, y) of op on ws; cls: a border-class map to index the PReLU table with instead of the true one"""
    x = tp.sview(ws, op.in_).double().permute(0, 3, 1, 2)
    z = F.conv2d(x, op.w.double().permute(0, 3, 1, 2), None, op.stride, op.k // 2).permute(0, 2, 3, 1)
    if op.act != tp.ACT_PRELU:
        return z, z
    z = z + op.bias.double()[class_map(HP, WP) if cls is None else cls]
    return z, torch.where(z > 0, z, op.slope.double() * z)


def _exact2(snap, op):
    after = snap.clone()
    y = _ref2(snap, op)[1]
    tp.sview(after, op.out).copy_(y.float().to(BF16) if op.act == tp.ACT_PRELU else y.float())
    return after


def test_exact_prelu_and_pitched_results_pass():
    snap, prelu, patch = _face_and_patch_layout()
    _check(snap, _exact2(snap, prelu), prelu)
    _check(snap, _exact2(snap, patch), patch)


def _class_of_neighbour(snap, op, after, imgs=(2, 5)):
    """the top-left tile's left column (left-border pixels) biased with the interior column's class, in an image and its copy"""
    cls = class_map(HP, WP).clone()
    cls[:, 0] += 1
    y = _ref2(snap, op, cls)[1]
    assert (y[:, :8, 0] - _ref2(snap, op)[1][:, :8, 0]).abs().max() > 1e-2
    for img in imgs:
        _tile(tp.sview(after, op.out), img, 0, 0).copy_(_tile(y, img, 0, 0).float().to(BF16))


def _class_of_neighbour_one_image(snap, op, after):
    _class_of_neighbour(snap, op, after, (5,))


def _slope_on_positive_side(snap, op, after):
    """images 1 and its copy 4: the slope applied to z > 0 instead of z <= 0"""
    z = _ref2(snap, op)[0]
    y = torch.where(z > 0, op.slope.double() * z, z)
    for img in (1, 4):
        tp.sview(after, op.out)[img].copy_(y[img].float().to(BF16))


def _one_token_early(snap, op, after):
    """image 4's patches written to tokens 0..L-2 instead of 1..L-1 of its stream"""
    y = _ref2(snap, op)[1]
    tp.sview(after, op.out._replace(off=op.out.off - WT * 4))[4].copy_(y[4].float())


PRELU_PATCH_CORRUPTIONS = [
    pytest.param(_class_of_neighbour, 0, r"\(a\) worst \|err\|/bar", id="neighbour-class-bias-image-and-copy"),
    pytest.param(_class_of_neighbour_one_image, 0, r"\(b\) image 5 differs from its copy, image 2", id="neighbour-class-bias-image-5"),
    pytest.param(_slope_on_positive_side, 0, r"\(a\) worst \|err\|/bar", id="slope-on-positive-side"),
    pytest.param(_one_token_early, 1, r"\(d\) workspace byte", id="patch-image-one-token-early")]


@pytest.mark.parametrize("corrupt,which,flag", PRELU_PATCH_CORRUPTIONS)
def test_prelu_and_pitched_corruption_is_flagged(corrupt, which, flag):
    snap, prelu, patch = _face_and_patch_layout()
    op = (prelu, patch)[which]
    after = _exact2(snap, op)
    _check(snap, after, op)
    corrupt(snap, op, after)
    with pytest.raises(AssertionError, match=flag):
        _check(snap, after, op)


def test_cc_conv_refuses_a_short_image_pitch():
    """out_ns below the output's pixels per image, or on a kernel that does not take it, is refused before any device query"""
    fake = 1 << 20

    def op(kind, out_ns):
        return cc_conv_op(kind=kind, in_=cc_slice(fake, KP, 0, KP, B, 1, PN, 0), out=cc_slice(fake, WT, 0, WT, B, 1, PN, 1),
                          w=fake, k=1, stride=1, groups=1, out_ns=out_ns)

    for kind, out_ns, msg in ((CC_CONV_OP_GEMM, PN - 1, "cc_conv: out_ns=8 pixels per image is less than the output's 1x9"),
                              (CC_CONV_OP_GEMM, -1, "cc_conv: out_ns=-1 pixels per image"),
                              (3, PN + 1, "cc_conv: out_ns=10 needs kind GEMM, got 3")):
        with pytest.raises(CCError, match=msg):
            check(lib().cc_conv(ctypes.byref(op(kind, out_ns)), None), "cc_conv")
