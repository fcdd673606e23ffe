"""The per-op checks of tests/test_plan_convs_gpu.py see the launches they are there to catch (no GPU needed).

Two conv ops on CPU tensors in a small workspace, laid out as a plan lays them out, over a batch of B = 7 images that are
copies of 3 distinct ones: a 3x3 / stride-2 SiLU conv between channel slices of wider buffers with a residual, and an
activation-free 1x1 conv of 3 x 384 x 64 outputs.  Their exact results (the float64 conv rounded to nearest bf16) pass every
check; each corruption below is flagged by the check named with it."""
import types

import pytest
import torch
import torch.nn.functional as F

import test_conv_gpu as tc
import test_plan_convs_gpu as tp
from clearcam_b200._lib import CC_CONV_OP_GEMM

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
                                     k=k, stride=stride, groups=1, act=act, pre=None, store1=1)

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
