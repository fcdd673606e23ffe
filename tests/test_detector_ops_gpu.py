"""The detector's kernels outside the conv GEMM mainloop, called directly through their C-ABI taps and compared element by
element with exact or float64 references:

* the pools, upsample, SPP and CBFuse (pool.cu): bit-exact against torch restatements in the kernels' float order, then the
  storage rounding;
* the fp32-accurate mode's plane split (bit-exact) and finishing pass, and the whole fp32-accurate conv (split, hi x hi
  segment GEMMs, cross-product GEMM, finish) against float64;
* both stems (stem_tc.cu, stem_kernel) and the conv GEMM's half-resolution `pre` addend (the fused Upsample -> Concat ->
  RepNCSPELAN4 first conv) against float64.

Each tolerance-based test prints its worst |err|/bar.  The CPU test `test_bars_see_detector_bugs` shows, on the inputs the
GPU tests use, that the typical bugs of these kernels leave every tolerance-based bar by at least 4x.
"""
import ctypes
import math
import re

import pytest
import torch
import torch.nn.functional as F

from clearcam_b200 import ops
from clearcam_b200._lib import CC_CONV_OP_DIRECT, CC_CONV_OP_GEMM, CC_CONV_OP_NONE, cc_conv_op, cc_slice, lib

SENT = -7.0
F32_BAR = 2.0 ** -18          # fp32 conv GEMM outputs (tests/test_conv_gpu.py): per element, x (sum|x.w| + |bias| + |pre|)
FIN_BAR = 2.0 ** -21          # finish_f32: 8 ulps of |acc + bias| + |res|
PREC_BAR = 1.625 * 2.0 ** -20  # fp32-accurate conv: x (sum|x.w| + |bias| + |res|)
TANH_ERR = 2.0 ** -11         # tanh.approx.f32 absolute error bound; the SiLU h + h tanh(h) then errs by <= 2^-12 |z|
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(_WORST):
        print(f"\nworst |err|/bar, {key}: {_WORST[key]:.3f}")


def _ratio(key, err, bar, what=""):
    r = (err / bar).max().item()
    _WORST[key] = max(_WORST.get(key, 0.0), r)
    print(f"{key} {what}: worst |err|/bar {r:.3f}")
    assert math.isfinite(r) and r <= 1.0, f"{key} {what}: worst |err|/bar {r:.3f}"


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _store(x, dtype):
    """x (fp32) as the kernel stores it."""
    return x.to(dtype).float() if dtype == torch.bfloat16 else x


def _sentinel_buf(N, H, W, cs, dtype):
    return torch.full((N, H, W, cs), SENT, dtype=dtype, device="cuda")


def _assert_outside_untouched(buf, co, C):
    mask = torch.ones(buf.shape[-1], dtype=torch.bool, device=buf.device)
    mask[co:co + C] = False
    assert bool((buf[..., mask] == SENT).all()), "channels outside the output slice were written"


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------ pools (bit-exact)
POOL_MAPS = [(1, 160, 160), (3, 80, 80), (1, 40, 40), (3, 20, 20), (3, 48, 80), (1, 24, 40), (3, 12, 20), (3, 2, 2)]
# (C, in_cs, in_co, out_cs, out_co): a slice inside wider buffers, and a dense map
POOL_SLICES = [(32, 48, 8, 64, 24), (64, 64, 0, 64, 0)]


def _avg2(x):
    """((a + b) + (d + e)) * 0.25 over the (H-1) x (W-1) map, in fp32 in the kernel's order."""
    a, b, d, e = x[:, :-1, :-1], x[:, :-1, 1:], x[:, 1:, :-1], x[:, 1:, 1:]
    return ((a + b) + (d + e)) * 0.25


def ref_pool(op, x, dtype):
    """x: fp32 NHWC holding stored values."""
    if op == "avg2_pad":
        out = torch.zeros_like(x)
        out[:, :-1, :-1] = _avg2(x)
        return _store(out, dtype)
    if op == "avgmax":
        return _nhwc(F.max_pool2d(_nchw(_store(_avg2(x), dtype)), 3, 2, 1))
    if op == "max5":
        return _nhwc(F.max_pool2d(_nchw(x), 5, 1, 2))
    return x.repeat_interleave(2, 1).repeat_interleave(2, 2)


def _run_pool(op, dtype, N, H, W, C, in_cs, in_co, out_cs, out_co, seed):
    x_all = _store(torch.randn(N, H, W, in_cs, generator=_gen(seed)) * 3, dtype)
    xbuf = x_all.to(dtype).cuda()
    Ho, Wo = {"avgmax": (H // 2, W // 2), "upsample2": (2 * H, 2 * W)}.get(op, (H, W))
    obuf = _sentinel_buf(N, Ho, Wo, out_cs, dtype)
    ops.pool(op, xbuf, in_co, C, obuf, out_co)
    torch.cuda.synchronize()
    _assert_outside_untouched(obuf, out_co, C)
    assert torch.equal(xbuf.cpu().float(), x_all), "the input was written"
    return x_all[..., in_co:in_co + C], obuf[..., out_co:out_co + C].float().cpu()


POOL_CASES = [(op, m, s) for op in ("avg2_pad", "avgmax", "max5", "upsample2") for m in POOL_MAPS for s in POOL_SLICES
              if s[0] == 32 or m[1] in (20, 48)]
POOL_CASES += [("max5", (2, 30, 30), POOL_SLICES[0])]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("op,nhw,sl", POOL_CASES, ids=[f"{o}-{m[0]}x{m[1]}x{m[2]}-C{s[0]}co{s[2]}" for o, m, s in POOL_CASES])
def test_pool_bit_exact(op, nhw, sl, dtype):
    """avg2_pad, avgmax, max5 and upsample2 equal their torch restatement bit for bit; the fp32 averages are also within
    one ulp of float64, and avg2_pad's last row and column are zero."""
    N, H, W = nhw
    C, in_cs, in_co, out_cs, out_co = sl
    x, got = _run_pool(op, dtype, N, H, W, C, in_cs, in_co, out_cs, out_co, seed=H * 7 + W + N + C)
    want = ref_pool(op, x, dtype)
    assert got.shape == want.shape
    bad = (got != want).nonzero()
    assert len(bad) == 0, f"{len(bad)} elements differ, first at {bad[0].tolist()}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}"
    if op == "avg2_pad":
        assert bool((got[:, -1] == 0).all()) and bool((got[:, :, -1] == 0).all())
    if dtype == torch.float32 and op in ("avg2_pad", "avgmax"):
        # the three fp32 additions round once each: within one ulp of (|a| + |b| + |d| + |e|) / 4 of float64 (a plain ulp of
        # the result does not bound them where the pairs cancel)
        x64 = x.double()
        avg64 = (x64[:, :-1, :-1] + x64[:, :-1, 1:] + x64[:, 1:, :-1] + x64[:, 1:, 1:]) / 4
        mag = (x64[:, :-1, :-1].abs() + x64[:, :-1, 1:].abs() + x64[:, 1:, :-1].abs() + x64[:, 1:, 1:].abs()) / 4
        assert bool(((_avg2(x).double() - avg64).abs() <= 2.0 ** -23 * mag).all()), "an fp32 average is further from float64"


# (N, H, W, c1, cs, co): H*W = 800 is the largest map spp3 takes
SPP_CASES = [(1, 1, 1, 64, 256, 0), (3, 2, 2, 128, 544, 16), (32, 20, 20, 256, 1024, 0), (2, 20, 20, 512, 2064, 8),
             (4, 12, 20, 64, 288, 32), (1, 20, 40, 128, 512, 0), (2, 40, 20, 512, 2048, 0), (3, 10, 80, 64, 264, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,c1,cs,co", SPP_CASES)
def test_spp3_bit_exact(N, H, W, c1, cs, co):
    """spp3 writes max_pool2d(5, 1, 2) applied once, twice and three times into the three slices after cv1's, leaving cv1's
    slice and every other channel untouched."""
    x = (torch.randn(N, H, W, c1, generator=_gen(N + H + c1)) * 2).to(torch.bfloat16)
    buf = _sentinel_buf(N, H, W, cs, torch.bfloat16)
    buf[..., co:co + c1] = x.cuda()
    ops.spp3(buf, co, c1)
    torch.cuda.synchronize()
    got = buf.cpu()
    assert torch.equal(got[..., co:co + c1], x), "spp3 wrote into cv1's slice"
    _assert_outside_untouched(buf, co, 4 * c1)
    p = x.float()
    for q in range(1, 4):
        p = ref_pool("max5", p, torch.bfloat16)
        assert torch.equal(got[..., co + q * c1:co + (q + 1) * c1].float(), p), f"pool {q} differs"


# ------------------------------------------------------------------------------------------------ CBFuse (bit-exact)
# (dtype, N, H, W, C, ratios of the sources): e's five-source fuse at 80x80 and 48x80 (ratios up to 16), fewer sources, and
# the general (non-power-of-two) path
CBF_CASES = [(torch.bfloat16, 2, 80, 80, 64, [1, 2, 4, 8, 16]), (torch.float32, 2, 80, 80, 64, [1, 2, 4, 8, 16]),
             (torch.bfloat16, 3, 48, 80, 128, [16, 8, 4, 2, 1]), (torch.bfloat16, 1, 40, 40, 256, [1]),
             (torch.float32, 3, 20, 20, 512, [2, 4]), (torch.bfloat16, 2, 48, 48, 64, [3, 1, 2]),
             (torch.float32, 1, 48, 48, 32, [8, 4, 2, 3])]


def _nearest_idx(n_out, n_in):
    return (torch.arange(n_out) * n_in) // n_out


def ref_cbfuse(srcs, last, dtype):
    H, W = last.shape[1:3]
    acc = None
    for s in srcs:
        up = s[:, _nearest_idx(H, s.shape[1])][:, :, _nearest_idx(W, s.shape[2])]
        acc = up if acc is None else acc + up
    return _store(acc + last, dtype)


def cbfuse_inputs(dtype, N, H, W, C, ratios, seed):
    g = _gen(seed)
    srcs = [_store(torch.randn(N, H // r, W // r, C, generator=g), dtype) for r in ratios]
    last = _store(torch.randn(N, H, W, C, generator=g), dtype)
    return srcs, last


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,N,H,W,C,ratios", CBF_CASES,
                         ids=[f"{'f32' if c[0] == torch.float32 else 'bf16'}-{c[1]}x{c[2]}x{c[3]}-C{c[4]}-r{'.'.join(map(str, c[5]))}"
                              for c in CBF_CASES])
def test_cbfuse_bit_exact(dtype, N, H, W, C, ratios):
    """out = sum_i nearest(src_i) + last in source order, every source and the output a slice of a wider buffer."""
    srcs, last = cbfuse_inputs(dtype, N, H, W, C, ratios, seed=H + W + C + len(ratios))
    for s in srcs:       # the integer index restates F.interpolate(nearest) at these ratios
        up = F.interpolate(_nchw(s), size=(H, W), mode="nearest")
        assert torch.equal(_nhwc(up), s[:, _nearest_idx(H, s.shape[1])][:, :, _nearest_idx(W, s.shape[2])])
    bufs = []
    for k, s in enumerate(srcs):
        b = _sentinel_buf(N, s.shape[1], s.shape[2], C + 8 * (k + 1), dtype)
        b[..., 8 * k:8 * k + C] = s.to(dtype).cuda()
        bufs.append((b, 8 * k))
    lb = _sentinel_buf(N, H, W, 2 * C, dtype)
    lb[..., C:] = last.to(dtype).cuda()
    ob = _sentinel_buf(N, H, W, C + 16, dtype)
    ops.cbfuse(bufs, (lb, C), (ob, 16), C)
    torch.cuda.synchronize()
    _assert_outside_untouched(ob, 16, C)
    assert torch.equal(ob[..., 16:].float().cpu(), ref_cbfuse(srcs, last, dtype))


# ------------------------------------------------------------------------------------------------ fp32-accurate pieces
def split3(x):
    """x (fp32) -> bf16 planes hi, mid, lo as the kernels split them."""
    hi = x.to(torch.bfloat16)
    r1 = x - hi.float()
    mid = r1.to(torch.bfloat16)
    lo = (r1 - mid.float()).to(torch.bfloat16)
    return hi, mid, lo


def split_inputs(npix, cs, seed):
    g = _gen(seed)
    e = torch.randint(-100, 101, (npix, cs), generator=g).double()
    x = (torch.rand(npix, cs, generator=g, dtype=torch.float64) + 1) * torch.pow(2.0, e)
    x = torch.where(torch.rand(npix, cs, generator=g) < 0.5, -x, x).float()
    x[: npix // 4] = x[: npix // 4].to(torch.bfloat16).float()        # exact bf16 values: mid = lo = 0
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("cs,co,C", [(40, 4, 28), (64, 0, 64), (36, 12, 4)])
def test_split_planes_bit_exact(cs, co, C):
    """The six planes [lo | mid | hi | mid | hi | hi] equal the torch split bit for bit, and hi + mid + lo == x exactly."""
    x = split_inputs(1000, cs, seed=cs + co)
    got = ops.split_planes(x.cuda(), co, C).cpu()
    torch.cuda.synchronize()
    hi, mid, lo = split3(x[:, co:co + C])
    want = torch.cat([lo, mid, hi, mid, hi, hi], 1)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    assert torch.equal(hi.double() + mid.double() + lo.double(), x[:, co:co + C].double())
    assert bool((mid[: 250] == 0).all()) and bool((lo[: 250] == 0).all())


def silu64(z, tanh_err=0.0):
    h = z / 2
    return h + h * (torch.tanh(h) + tanh_err)


def finish_inputs(npix, C, with_res, seed):
    g = _gen(seed)
    acc = torch.randn(npix, C, generator=g) * 4
    acc[:, :4] = acc[:, :4] * 20          # silu deep into both tails
    bias = torch.randn(C, generator=g)
    res = torch.randn(npix, C + 8, generator=g) if with_res else None
    return acc, bias, res


FIN_CASES = [(act, r) for act in (0, 1) for r in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("act,with_res", FIN_CASES, ids=[f"act{a}-{'res' if r else 'nores'}" for a, r in FIN_CASES])
def test_finish_f32_matches_float64(act, with_res):
    """out = [res +] act(acc + bias) within 8 ulps of |acc + bias| + |res|; the residual is a slice of another buffer."""
    npix, C = 3000, 96
    acc, bias, res = finish_inputs(npix, C, with_res, seed=act + 2 * with_res)
    out = torch.full((npix, C + 12), SENT, device="cuda")
    ops.finish_f32(acc.cuda(), bias.cuda(), act, out, 12, None if res is None else res.cuda(), 8)
    torch.cuda.synchronize()
    assert bool((out[:, :12] == SENT).all())
    got = out[:, 12:].cpu().double()
    z = acc.double() + bias.double()
    want = silu64(z) if act else z
    r = res[:, 8:].double() if with_res else torch.zeros_like(z)
    want = want + r
    _ratio("finish_f32", (got - want).abs(), FIN_BAR * (z.abs() + r.abs()) + 1e-300, f"act {act} res {with_res}")


# the fp32-accurate conv: (N, H, W, Cin, Cout, k, stride, act, residual).  3x3 over 256 and 512 channels runs several hi x hi
# segments; 96 channels split in 16-channel units
PREC_CASES = [(2, 20, 20, 256, 256, 3, 1, 1, True), (1, 20, 20, 512, 512, 3, 1, 1, False), (2, 40, 40, 256, 128, 3, 2, 1, False),
              (3, 24, 40, 128, 64, 1, 1, 1, True), (2, 16, 16, 16, 32, 3, 1, 0, False), (1, 12, 20, 96, 48, 3, 1, 1, True),
              (1, 20, 20, 512, 16, 1, 1, 0, False), (2, 10, 10, 64, 512, 3, 2, 1, True), (1, 20, 20, 1024, 256, 1, 1, 1, False)]
PREC_KINDS = ["gaussian", "coherent"]


def _coherent(shape, g, scale):
    """Positive fp32 values x = hi + mid + lo whose three bf16 planes are all positive and near their largest (mid >= 0.9
    2^-8 hi, lo >= 0.9 2^-17 hi, hi in {1, 1.125}): the hi x hi sums are exact in fp32, while every cross product adds up with
    one sign, so a dropped or misplaced plane product shows at its full size."""
    hi = 1 + torch.randint(0, 2, shape, generator=g).double() / 8
    mid = ((0.9 + 0.09 * torch.rand(shape, generator=g, dtype=torch.float64)) * 2.0 ** -8).float().to(torch.bfloat16).double()
    lo = torch.round((0.9 + 0.09 * torch.rand(shape, generator=g, dtype=torch.float64)) * 2.0 ** -17 / 2.0 ** -23) * 2.0 ** -23
    x = (hi + mid + lo) * scale
    assert torch.equal(x.float().double(), x)
    return x.float()


def prec_inputs(case, kind):
    N, H, W, Cin, Cout, k, s, act, use_res = case
    g = _gen(((N * 101 + H) * 101 + W) * 10007 + Cin * 1009 + Cout * 11 + k * 3 + s + 7919 * PREC_KINDS.index(kind))
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    if kind == "gaussian":
        x = torch.randn(N, H, W, Cin, generator=g)
        w = torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
        res = torch.randn(N, Ho, Wo, Cout, generator=g) if use_res else None
    else:
        x = _coherent((N, H, W, Cin), g, 1.0)
        w = _coherent((Cout, Cin, k, k), g, 2.0 ** -4)
        res = torch.randn(N, Ho, Wo, Cout, generator=g) * 0.01 if use_res else None
    b = torch.randn(Cout, generator=g) * 0.1
    return x, w, b, res


def prec_ref(x, w, b, res, s, act, dev):
    """float64 [res +] act(conv(x, w) + b) and the bar's magnitude sum|x.w| + |b| + |res|."""
    k = w.shape[-1]
    x64, w64, b64 = x.to(dev).double(), w.to(dev).double(), b.to(dev).double()
    z = _nhwc(F.conv2d(_nchw(x64), w64, b64, stride=s, padding=k // 2))
    mag = _nhwc(F.conv2d(_nchw(x64.abs()), w64.abs(), b64.abs(), stride=s, padding=k // 2))
    y = silu64(z) if act else z
    if res is not None:
        y = y + res.to(dev).double()
        mag = mag + res.to(dev).double().abs()
    return z, y, mag


@pytest.mark.gpu
@pytest.mark.parametrize("kind", PREC_KINDS)
@pytest.mark.parametrize("case", PREC_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3]}to{c[4]}-k{c[5]}s{c[6]}-act{c[7]}{'-res' if c[8] else ''}"
                                                  for c in PREC_CASES])
def test_conv_fp32_accurate_matches_float64(case, kind):
    """The whole fp32-accurate conv (plane split, hi x hi segments, cross products, finish) within 1.625 x 2^-20 (sum|x.w| +
    |b| + |res|) of float64; input, residual and output are slices of wider buffers.  The coherent inputs are the hard case:
    the cross-product GEMM's accumulator truncates in one direction over up to 5 x 9 x Cin / 16 steps."""
    N, H, W, Cin, Cout, k, s, act, use_res = case
    x, w, b, res = prec_inputs(case, kind)
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    xbuf = torch.full((N, H, W, Cin + 8), SENT, device="cuda")
    xbuf[..., 4:4 + Cin] = x.cuda()
    obuf = torch.full((N, Ho, Wo, Cout + 12), SENT, device="cuda")
    rbuf = None
    if use_res:
        rbuf = torch.full((N, Ho, Wo, Cout + 4), SENT, device="cuda")
        rbuf[..., 4:] = res.cuda()
    ops.conv2d_fp32_accurate(xbuf, 4, Cin, w, b, s, act, obuf, 12, rbuf, 4)
    torch.cuda.synchronize()
    assert bool((obuf[..., :12] == SENT).all())
    _, y, mag = prec_ref(x, w, b, res, s, act, "cuda")
    got = obuf[..., 12:].double()
    assert bool(torch.isfinite(got).all())
    _ratio("fp32-accurate conv", (got - y).abs(), PREC_BAR * mag, f"{case} {kind}")


# ------------------------------------------------------------------------------------------------ stems
# (impl, B, H, W, Cout, frame dtype, out dtype, out_cs, out_co)
STEM_CASES = [(1, 1, 62, 46, 16, "u8", "bf16", 16, 0), (1, 2, 384, 640, 32, "u8", "bf16", 48, 16),
              (1, 1, 640, 640, 64, "u8", "bf16", 64, 0), (1, 3, 66, 98, 64, "u8", "bf16", 96, 32),
              (1, 2, 384, 640, 16, "u8", "bf16", 32, 8)]
STEM_CASES += [(2, 2, 62, 98, Cout, fd, od, Cout + 8, 8) for Cout, fd, od in
               [(16, "u8", "bf16"), (32, "u8", "f32"), (64, "f32", "bf16"), (64, "f32", "f32"), (16, "f32", "f32")]]
STEM_CASES += [(2, 1, 384, 640, 64, "u8", "f32", 64, 0)]


def stem_inputs(B, H, W, Cout, fdt, seed):
    g = _gen(seed)
    fr = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    if fdt == "f32":
        fr = fr.float() * torch.rand(B, H, W, 3, generator=g)
    w = torch.randn(Cout, 3, 3, 3, generator=g) * 0.3
    b = torch.randn(Cout, generator=g) * 0.1
    return fr, w, b


def stem_ref(fr, w, b, impl, flip=True, shift=0, dev="cpu"):
    """float64 (pre-activation, SiLU, sum|x.w| + |b|) of the stem on the operands it uses: exact integer pixels with
    bf16(w / 255) for stem_tc, fp32(pixel / 255) with fp32 w for stem_kernel.  flip / shift: the bugs the bars must see."""
    x = fr.to(dev)
    if flip:
        x = x.flip(-1)
    if impl == 1:
        x = x.double()
        wk = (w.float() / torch.full_like(w, 255.0)).to(torch.bfloat16).double().to(dev)
    else:
        x = (x.float() / torch.full(x.shape, 255.0, device=dev)).double()
        wk = w.double().to(dev)
    pad = (1 - shift, 1 + shift, 1 - shift, 1 + shift)
    xp, xa = F.pad(_nchw(x), pad), F.pad(_nchw(x.abs()), pad)
    z = _nhwc(F.conv2d(xp, wk, b.double().to(dev), stride=2))
    mag = _nhwc(F.conv2d(xa, wk.abs(), b.double().abs().to(dev), stride=2))
    return z, silu64(z), mag


def stem_bar(z, y, mag, out_f32):
    if out_f32:
        return 2.0 ** -20 * mag
    return 2.0 ** -7 * y.abs() + TANH_ERR * z.abs() + F32_BAR * mag


@pytest.mark.gpu
@pytest.mark.parametrize("impl,B,H,W,Cout,fdt,odt,out_cs,out_co", STEM_CASES)
def test_stem_matches_float64(impl, B, H, W, Cout, fdt, odt, out_cs, out_co):
    """Both stems against float64 on their own packed operands: clipped last tiles (output pixel counts that are not a
    multiple of 128), more tiles than 5 CTAs per SM cover at once, output slices with co != 0."""
    fr, w, b = stem_inputs(B, H, W, Cout, fdt, seed=B + H + W + Cout + impl)
    dt = torch.float32 if odt == "f32" else torch.bfloat16
    obuf = _sentinel_buf(B, H // 2, W // 2, out_cs, dt)
    ops.stem(fr.cuda(), w, b, obuf, out_co, impl)
    torch.cuda.synchronize()
    _assert_outside_untouched(obuf, out_co, Cout)
    z, y, mag = stem_ref(fr, w, b, impl, dev="cuda")
    got = obuf[..., out_co:out_co + Cout].double()
    name = "stem_tc" if impl == 1 else f"stem_kernel {fdt}->{odt}"
    _ratio(name, (got - y).abs(), stem_bar(z, y, mag, odt == "f32"), f"{B}x{H}x{W} Cout {Cout}")


# ------------------------------------------------------------------------------------------------ conv GEMM + pre addend
# the fused first convs of c (layers 12, 15) and e (32, 35) at 640x640 and 384x640: (N, Ho, Wo, Cin, Cout, out_f32, act, bn)
PRE_CASES = [(1, 40, 40, 512, 512, False, 1, 0), (3, 80, 80, 512, 256, False, 1, 0), (32, 40, 40, 1024, 512, False, 1, 0),
             (3, 24, 40, 1024, 512, True, 0, 64), (32, 48, 80, 512, 256, False, 1, 16), (1, 48, 80, 512, 256, False, 1, 32),
             (3, 40, 40, 512, 512, True, 0, 128), (1, 24, 40, 512, 512, False, 1, 128), (3, 48, 80, 512, 256, True, 0, 0)]


def pre_inputs(case):
    N, Ho, Wo, Cin, Cout, out_f32, act, bn = case
    g = _gen(N * 1000 + Ho + Cin + Cout + bn)
    x = torch.randn(N, Ho, Wo, Cin, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, 1, 1, Cin, generator=g) * Cin ** -0.5).to(torch.bfloat16)
    b = torch.randn(Cout, generator=g) * 0.1
    pre = torch.randn(N, Ho // 2, Wo // 2, Cout, generator=g)
    return x, w, b, pre


def pre_ref(x, w, b, pre, act, dev, neighbour=False):
    """float64 (z, act(z), sum|x.w| + |b| + |pre|) with z = conv(x) + b + up2(pre); neighbour: pre read one pixel to the right."""
    Ho, Wo = x.shape[1:3]
    iw = (torch.arange(Wo) + (1 if neighbour else 0)).clamp(max=Wo - 1) // 2
    up = pre.to(dev).double()[:, torch.arange(Ho) // 2][:, :, iw]
    xw = _nhwc(F.conv2d(_nchw(x.to(dev).double()), w.to(dev).double().permute(0, 3, 1, 2)))
    xa = _nhwc(F.conv2d(_nchw(x.to(dev).double().abs()), w.to(dev).double().abs().permute(0, 3, 1, 2)))
    z = xw + b.to(dev).double() + up
    mag = xa + b.to(dev).double().abs() + up.abs()
    return z, (silu64(z) if act else z), mag


def pre_bar(z, y, mag, out_f32):
    if out_f32:
        return F32_BAR * mag
    return 2.0 ** -7 * y.abs() + TANH_ERR * z.abs() + F32_BAR * mag


@pytest.mark.gpu
@pytest.mark.parametrize("case", PRE_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3]}to{c[4]}-{'f32' if c[5] else 'bf16'}-bn{c[7]}" for c in PRE_CASES])
def test_cc_conv_pre_addend_matches_float64(case):
    """act(conv(x) + b + up2(pre)) of the fused Upsample -> Concat -> RepNCSPELAN4 first conv, into the lower half of its
    concat buffer; at B = 32 the 128-pixel tiles span several images."""
    N, Ho, Wo, Cin, Cout, out_f32, act, bn = case
    x, w, b, pre = pre_inputs(case)
    dt = torch.float32 if out_f32 else torch.bfloat16
    obuf = _sentinel_buf(N, Ho, Wo, 2 * Cout, dt)
    ops.conv2d(x.cuda(), 0, Cin, w.cuda(), b.cuda(), 1, 1, obuf, 0, Cout, act=act, bn=bn, pre=pre.cuda())
    torch.cuda.synchronize()
    _assert_outside_untouched(obuf, 0, Cout)
    z, y, mag = pre_ref(x, w, b, pre, act, "cuda")
    got = obuf[..., :Cout].double()
    _ratio("conv + pre " + ("f32" if out_f32 else "bf16"), (got - y).abs(), pre_bar(z, y, mag, out_f32), str(case))


# ------------------------------------------------------------------------------------------------ hi x hi segments of the plan
@pytest.mark.gpu
def test_fp32_accurate_plan_keeps_hi_segments_within_48_steps():
    """In YOLOv9-c's fp32-accurate plan every conv runs at least ceil(k^2 Cin / 16 / 48) hi x hi GEMMs, so no tensor-core
    accumulator takes more than 48 k16 steps."""
    from oracle import yolov9 as o
    from clearcam_b200.detection.yolov9 import YOLOv9
    table = {name: (cin, k) for name, cin, cout, k, s, g, act in o.conv_table("c")}
    P = o.synthetic_weights("c", seed=3)
    m = YOLOv9("c", 128, weights=P, precise=True)
    prof = m.profile(o.synthetic_frames(1, 128, 128, seed=3))
    segs = {}
    for op in prof:
        hit = re.match(r"^(.*)\.hi(\d+)$", op["name"])
        if hit:
            segs[hit.group(1)] = segs.get(hit.group(1), 0) + 1
    assert len(segs) > 50
    for key, n in segs.items():
        first = key
        if "+" in key:           # a fused pair ("p.cv1+cv2", "model.22.cv2+cv3.0.0"): the first conv's name
            head, tail = key.split("+", 1)
            first = head + ("." + tail.split(".", 1)[1] if "." in tail else "")
        cin, k = table.get(first + ".conv", table.get(first, (None, None)))
        assert cin is not None, key
        need = math.ceil(k * k * cin / 16 / 48)
        assert n >= need, f"{key}: {n} hi x hi GEMMs for k={k} Cin={cin}, at least {need} keep each within 48 k16 steps"


# ------------------------------------------------------------------------------------------------ CPU: bars and arguments
def test_bars_see_detector_bugs():
    """CPU only: on the GPU tests' own inputs, each typical bug leaves its bar by at least 4x:
    the fp32-accurate conv with any one cross product dropped or with mid and lo swapped in the activation split (coherent
    inputs, every case), finish_f32 with a tanh.approx-sized SiLU error, the pre addend read one pixel to the right (every case
    up to B = 3), and the stem without its channel flip or with its padding shifted by one."""
    worst = {}

    def see(name, diff, bar):
        worst[name] = min(worst.get(name, math.inf), (diff.abs() / bar).max().item())

    # fp32-accurate conv: the kernel sums lo.hi, mid.mid, hi.lo, mid.hi, hi.mid (cross GEMM) and hi.hi (segments)
    for case in PREC_CASES:
        N, H, W, Cin, Cout, k, s, act, use_res = case
        x, w, b, res = prec_inputs(case, "coherent")
        z, y, mag = prec_ref(x, w, b, res, s, act, "cpu")
        xp = dict(zip(("hi", "mid", "lo"), split3(x)))
        wp = dict(zip(("hi", "mid", "lo"), split3(w)))
        conv = lambda a, bb: _nhwc(F.conv2d(_nchw(xp[a].double()), wp[bb].double(), stride=s, padding=k // 2))
        bar = PREC_BAR * mag
        out = lambda zz: (silu64(zz) if act else zz) + (0 if res is None else res.double())
        for a, bb in (("lo", "hi"), ("mid", "mid"), ("hi", "lo"), ("mid", "hi"), ("hi", "mid")):
            see(f"fp32-accurate: {a}.{bb} dropped", out(z - conv(a, bb)) - y, bar)
        see("fp32-accurate: mid and lo swapped", out(z + conv("lo", "mid") - conv("mid", "mid")) - y, bar)
    # finish_f32
    for act, with_res in FIN_CASES:
        if not act:
            continue
        acc, bias, res = finish_inputs(3000, 96, with_res, seed=act + 2 * with_res)
        zz = acc.double() + bias.double()
        r = res[:, 8:].double() if with_res else torch.zeros_like(zz)
        see("finish_f32: tanh.approx-sized SiLU error", silu64(zz, TANH_ERR) - silu64(zz), FIN_BAR * (zz.abs() + r.abs()) + 1e-300)
    # pre addend
    for case in PRE_CASES:
        if case[0] > 3:
            continue
        x, w, b, pre = pre_inputs(case)
        z, y, mag = pre_ref(x, w, b, pre, case[6], "cpu")
        _, y_n, _ = pre_ref(x, w, b, pre, case[6], "cpu", neighbour=True)
        see("pre read at the neighbouring pixel", y_n - y, pre_bar(z, y, mag, case[5]))
    # stems
    for impl, B, H, W, Cout, fdt, odt, out_cs, out_co in STEM_CASES:
        fr, w, b = stem_inputs(B, H, W, Cout, fdt, seed=B + H + W + Cout + impl)
        z, y, mag = stem_ref(fr, w, b, impl)
        bar = stem_bar(z, y, mag, odt == "f32")
        see("stem without the channel flip", stem_ref(fr, w, b, impl, flip=False)[1] - y, bar)
        see("stem padding shifted by one", stem_ref(fr, w, b, impl, shift=1)[1] - y, bar)
    for name, r in sorted(worst.items()):
        print(f"{name}: {r:.1f}x the bar")
    for name, r in worst.items():
        assert r >= 4.0, f"'{name}' moves the result by only {r:.2f}x the bar"


def test_detector_taps_and_cc_conv_reject_bad_arguments():
    """Every check of the taps runs before anything is launched (no GPU needed): the pointers below are never dereferenced."""
    h = lib()
    fake = ctypes.c_void_p(1 << 20)
    odd = ctypes.c_void_p((1 << 20) + 8)
    need = ctypes.c_size_t(0)

    def refused(rc, *words):
        msg = h.cc_last_error().decode()
        assert rc == -1 and all(w_ in msg for w_ in words), (rc, msg, words)

    # cc_pool(op, f32, in, N, H, W, in_cs, in_co, C, out, out_cs, out_co, stream)
    refused(h.cc_pool(4, 0, fake, 1, 8, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "unknown op")
    refused(h.cc_pool(-1, 0, fake, 1, 8, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "unknown op")
    refused(h.cc_pool(0, 2, fake, 1, 8, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "f32")
    refused(h.cc_pool(0, 0, fake, 1, 1, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "at least 2x2")
    refused(h.cc_pool(1, 0, fake, 1, 9, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "even sides")
    refused(h.cc_pool(2, 0, None, 1, 8, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "input is NULL")
    refused(h.cc_pool(2, 0, odd, 1, 8, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "16-byte aligned")
    refused(h.cc_pool(2, 0, fake, 1, 8, 8, 64, 4, 60, fake, 64, 0, None), "cc_pool", "whole vectors of 8")
    refused(h.cc_pool(2, 1, fake, 1, 8, 8, 64, 32, 64, fake, 64, 0, None), "cc_pool", "inside the row")
    refused(h.cc_pool(3, 0, fake, 1, 8, 8, 64, 0, 64, fake, 32, 0, None), "cc_pool", "output", "inside the row")
    refused(h.cc_pool(2, 0, fake, 0, 8, 8, 64, 0, 64, fake, 64, 0, None), "cc_pool", "bad shape")
    # cc_spp3(cat, N, H, W, cs, co, c1, stream): 800 pixels is the limit, c1 a multiple of 64
    refused(h.cc_spp3(fake, 1, 9, 89, 256, 0, 64, None), "cc_spp3", "not supported", "801")
    refused(h.cc_spp3(fake, 1, 20, 20, 128, 0, 32, None), "cc_spp3", "not supported")
    refused(h.cc_spp3(fake, 1, 20, 20, 255, 0, 64, None), "cc_spp3", "whole vectors")
    refused(h.cc_spp3(fake, 70000, 2, 2, 256, 0, 64, None), "cc_spp3", "grid")
    refused(h.cc_spp3(fake, 1, 20, 20, 256, 0, 0, None), "cc_spp3", "c1")
    # cc_cbfuse(f32, nsrc, src[], src_h[], src_w[], src_cs[], src_co[], last, last_cs, last_co, out, out_cs, out_co, N, H, W, C)
    P5, I5 = ctypes.c_void_p * 5, ctypes.c_int * 5
    src, hs, ws, cs, co = P5(*([1 << 20] * 5)), I5(*[10] * 5), I5(*[10] * 5), I5(*[64] * 5), I5(*[0] * 5)
    cbf = lambda f32=0, n=2, src=src, last=fake, out=fake, cs=cs: h.cc_cbfuse(f32, n, src, hs, ws, cs, co, last, 64, 0, out, 64, 0,
                                                                             1, 20, 20, 64, None)
    refused(cbf(n=0), "cc_cbfuse", "nsrc=0")
    refused(cbf(n=6), "cc_cbfuse", "nsrc=6")
    refused(cbf(f32=3), "cc_cbfuse", "f32")
    refused(cbf(src=P5(1 << 20, 0, 0, 0, 0)), "cc_cbfuse", "a source is NULL")
    refused(cbf(cs=I5(64, 60, 64, 64, 64)), "cc_cbfuse", "whole vectors")
    refused(cbf(last=None), "cc_cbfuse", "last is NULL")
    refused(cbf(out=odd), "cc_cbfuse", "output must be 16-byte aligned")
    # cc_split_planes(in, npix, cs, co, C, out) and cc_finish_f32(acc, bias, act, npix, C, out, out_cs, out_co, res, res_cs, res_co)
    refused(h.cc_split_planes(fake, 10, 64, 2, 32, fake, None), "cc_split_planes", "whole vectors of 4")
    refused(h.cc_split_planes(fake, 10, 64, 0, 64, ctypes.c_void_p((1 << 20) + 4), None), "cc_split_planes", "8-byte aligned")
    refused(h.cc_finish_f32(fake, fake, 2, 10, 64, fake, 64, 0, None, 0, 0, None), "cc_finish_f32", "act 2")
    refused(h.cc_finish_f32(fake, odd, 1, 10, 64, fake, 64, 0, None, 0, 0, None), "cc_finish_f32", "d_bias")
    refused(h.cc_finish_f32(fake, fake, 1, 10, 64, fake, 64, 4, None, 0, 0, None), "cc_finish_f32", "output", "inside the row")
    refused(h.cc_finish_f32(fake, fake, 1, 10, 64, fake, 64, 0, fake, 64, 2, None), "cc_finish_f32", "residual")
    # cc_stem(frames, f32, B, H, W, h_w, h_bias, Cout, out, out_cs, out_co, out_f32, impl, ws, ws_bytes, ws_needed, stream)
    wt = torch.zeros(64 * 27)
    stem = lambda f32=0, B=1, H=64, W=64, Cout=64, out=fake, cs=64, co=0, of32=0, impl=1, ws=fake, wsb=1 << 20, hw=wt: h.cc_stem(
        fake, f32, B, H, W, ctypes.c_void_p(hw.data_ptr()) if hw is not None else None, ctypes.c_void_p(wt.data_ptr()), Cout, out,
        cs, co, of32, impl, ws, wsb, ctypes.byref(need), None)
    assert stem(out=None) == 0 and need.value == 6912 + 4096 + 256
    refused(stem(impl=0), "cc_stem", "unknown impl")
    refused(stem(impl=3, out=None), "cc_stem", "unknown impl")
    refused(stem(f32=1), "cc_stem", "stem_tc takes uint8")
    refused(stem(of32=1), "cc_stem", "stem_tc takes uint8")
    refused(stem(Cout=48, cs=48), "cc_stem", "Cout 16, 32 or 64")
    refused(stem(H=63, impl=2), "cc_stem", "bad shape")
    refused(stem(Cout=12, cs=16, impl=2), "cc_stem", "bad shape")
    refused(stem(co=8), "cc_stem", "bad output slice")
    refused(stem(wsb=100), "cc_stem", "too small")
    refused(stem(ws=None), "cc_stem", "too small")
    refused(stem(out=odd), "cc_stem", "16-byte aligned")
    refused(stem(hw=None), "cc_stem", "NULL")
    # cc_conv(op, stream): a 1x1 SiLU conv 64 -> 64 over a 40-wide map with the pre addend, the slices and pre_h / pre_w at the
    # extent its input and stride give, then the fields set by `kw`
    def conv(Hin=40, Cin=64, k=1, s=1, p=fake.value, out_f32=0, **kw):
        Ho, Wo = (Hin - 1) // s + 1, (40 - 1) // s + 1
        op = cc_conv_op(kind=CC_CONV_OP_GEMM, in_=cc_slice(fake.value, Cin, 0, Cin, 1, Hin, 40, 0), w=fake.value, bias=fake.value,
                        out=cc_slice(fake.value, 64, 0, 64, 1, Ho, Wo, out_f32), k=k, stride=s, groups=1, act=1, pre=p,
                        pre_h=Ho // 2, pre_w=Wo // 2)
        for name, v in kw.items():
            setattr(op, name, v)
        return h.cc_conv(ctypes.byref(op), None)
    refused(conv(p=odd.value), "cc_conv:", f"pre={hex(odd.value)} must be 16-byte aligned")
    refused(conv(Hin=41), "cc_conv:", "output 41x40 must have even sides")
    refused(conv(Hin=42, s=2, k=3), "cc_conv:", "output 21x20 must have even sides")
    refused(conv(Cin=24), "cc_conv:", "not supported", "Cin=24")
    refused(conv(s=2), "cc_conv:", "not supported", "k=1 stride=2")
    refused(conv(kind=CC_CONV_OP_NONE), "cc_conv:", "unknown kind 0")
    refused(conv(kind=4), "cc_conv:", "unknown kind 4")
    refused(conv(in_=cc_slice(None, 64, 0, 64, 1, 40, 40, 0)), "cc_conv:", "in.p is NULL")
    refused(conv(w=None), "cc_conv:", "w is NULL")
    refused(conv(out=cc_slice(None, 64, 0, 64, 1, 40, 40, 0)), "cc_conv:", "out.p is NULL")
    refused(conv(out=cc_slice(fake.value, 64, 0, 64, 1, 39, 40, 0)), "cc_conv:", "out is 1x39x40, the output 1x40x40")
    refused(conv(pre_h=19), "cc_conv:", "pre is 19x20, the output's half resolution 20x20")
    refused(conv(act=3, p=None), "cc_conv:", "CC_ACT_PRELU needs", "slope", f"bias={hex(fake.value)}")
    refused(conv(act=3, p=None, slope=fake.value, out_f32=1), "cc_conv:", "CC_ACT_PRELU writes bf16", "out.f32=1")
    refused(conv(kind=CC_CONV_OP_DIRECT), "cc_conv:", "direct kernel takes no pre", f"pre={hex(fake.value)}")
    # cc_conv2d_fp32_accurate(in, N, Hin, Win, in_cs, in_co, Cin, h_w, h_bias, Cout, k, stride, act, res, res_cs, res_co,
    #                         out, out_cs, out_co, ws, ws_bytes, ws_needed, stream)
    wp = torch.zeros(64 * 256 * 9)
    acc = lambda Cin=256, Cout=64, k=3, s=1, act=1, Hin=20, in_cs=256, in_co=0, res=None, res_co=0, out=fake, ws=fake, wsb=1 << 40, hw=wp: \
        h.cc_conv2d_fp32_accurate(fake, 2, Hin, 20, in_cs, in_co, Cin, ctypes.c_void_p(hw.data_ptr()) if hw is not None else None,
                                  None, Cout, k, s, act, res, 64, res_co, out, 64, 0, ws, wsb, ctypes.byref(need), None)
    # the workspace: planes 6 Cin bf16 per input pixel, fp32 partial sums, the five weight planes, the hi segments, the bias
    assert acc(out=None) == 0
    planes, sums = 2 * 20 * 20 * 6 * 256 * 2, 2 * 20 * 20 * 64 * 4
    assert need.value == planes + sums + 64 * 9 * 5 * 256 * 2 + 256 + 4 * 64 * 9 * 64 * 2, need.value   # 3x3 over 256: 4 segments
    refused(acc(k=1, s=2), "cc_conv2d_fp32_accurate", "k=1 stride=2")
    refused(acc(k=5), "cc_conv2d_fp32_accurate", "k=5")
    refused(acc(act=2, out=None), "cc_conv2d_fp32_accurate", "act 2")
    refused(acc(s=2, Hin=21), "cc_conv2d_fp32_accurate", "even sides")
    refused(acc(Cin=24, in_cs=24), "cc_conv2d_fp32_accurate", "multiples of 16")
    refused(acc(Cout=40), "cc_conv2d_fp32_accurate", "multiples of 16")
    refused(acc(in_co=16), "cc_conv2d_fp32_accurate", "bad slice")
    refused(acc(res=fake, res_co=2), "cc_conv2d_fp32_accurate", "bad slice")
    refused(acc(wsb=1000), "cc_conv2d_fp32_accurate", "too small")
    refused(acc(ws=None), "cc_conv2d_fp32_accurate", "too small")
    refused(acc(res=odd), "cc_conv2d_fp32_accurate", "16-byte aligned")
    refused(acc(hw=None), "cc_conv2d_fp32_accurate", "NULL")
