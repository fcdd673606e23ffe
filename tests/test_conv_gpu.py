"""GPU parity of the wgmma implicit-GEMM conv (and the direct conv) against a float64 torch conv2d on the same
bf16-rounded operands.  Reference op: detection/yolov9.py:33-38 (Conv = Conv2d+bias -> SiLU).

fp32 outputs are held to F32_BAR x (sum|x.w| + |bias| + |res|) per element.  bf16 outputs are held to the bar of the stem and
pre-addend tests (tests/test_detector_ops_gpu.py): one bf16 rounding of |y|, the tanh.approx error of SiLU / GELU, and the
fp32 bar.  That bar alone would pass an epilogue that truncates instead of rounding to nearest, so the activation-free bf16
cases with at least 10^4 outputs (CLIP's QKV GEMMs) also check the rounding direction: the mean of
(got - y) sign(y) / ulp_bf16(y) is about 0 when rounding to nearest and -0.5 when truncating.  The inputs are seeded on the
host so that tests/test_clip_ops_gpu.py can show, without a GPU, that these bars see a truncating or doubly rounding store."""
import pytest
import torch
import torch.nn.functional as F

from clearcam_b200 import ops

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, k, s, act, res, out_f32, in_cs, in_co, out_cs, out_co, bn)
CASES = [
    (1, 8, 16, 64, 64, 1, 1, 0, False, False, 64, 0, 64, 0, 0),
    (2, 40, 40, 128, 256, 1, 1, 1, False, False, 128, 0, 256, 0, 0),
    (1, 80, 80, 64, 64, 3, 1, 1, False, False, 64, 0, 64, 0, 0),
    (1, 24, 40, 32, 32, 3, 1, 1, False, False, 32, 0, 32, 0, 0),
    (1, 16, 16, 16, 32, 3, 1, 1, False, False, 16, 0, 32, 0, 0),
    (2, 32, 32, 64, 128, 3, 2, 1, False, False, 64, 0, 128, 0, 0),
    (8, 20, 20, 256, 256, 3, 1, 1, False, False, 256, 0, 256, 0, 0),
    (3, 20, 20, 128, 128, 3, 1, 1, True, False, 256, 64, 512, 128, 0),
    (2, 40, 40, 256, 80, 1, 1, 0, False, True, 256, 0, 80, 0, 0),
    (1, 1, 1000, 1024, 512, 1, 1, 2, False, False, 1024, 0, 512, 0, 0),
    (1, 1, 777, 512, 256, 1, 1, 0, True, True, 512, 0, 256, 0, 0),
    (8, 20, 20, 512, 256, 3, 1, 1, False, False, 512, 0, 256, 0, 128),
    (2, 40, 40, 256, 512, 1, 1, 1, False, False, 256, 0, 512, 0, 256),
    (4, 48, 80, 128, 128, 3, 2, 1, False, False, 256, 128, 128, 0, 0),
    (32, 40, 40, 256, 256, 3, 1, 1, False, False, 256, 0, 256, 0, 0),
    # narrow tiles (BN = 16: one thread of each pair converts the row alone) and odd channel counts
    (2, 40, 40, 32, 32, 3, 1, 1, True, False, 64, 32, 64, 0, 0),
    (2, 20, 20, 64, 16, 1, 1, 0, False, True, 64, 0, 16, 0, 0),
    (2, 20, 20, 64, 96, 3, 1, 1, False, False, 64, 0, 96, 0, 0),
    (3, 33, 21, 48, 16, 3, 1, 1, False, False, 48, 0, 48, 16, 0),
]
# grouped convs (a 16th field: groups) on the direct kernel at the literal-t widths 24 and 48: the t head's g = 4 convs
GROUPED_CASES = [(2, 20, 20, 24, 24, 3, 1, 1, False, False, 24, 0, 24, 0, 0, 4),
                 (1, 40, 40, 48, 48, 3, 1, 1, False, False, 48, 0, 48, 0, 0, 4),
                 (3, 20, 20, 48, 48, 1, 1, 0, False, True, 48, 0, 48, 0, 0, 4),
                 (1, 80, 80, 24, 24, 3, 2, 1, True, False, 48, 24, 48, 24, 0, 4)]
# the CLIP GEMMs as the encoders run them, N = H = 1 and W = token rows (6 x 50, 7 x 77, 3 x 257) at the tower widths:
# QKV (W -> 3W, bf16 out) and mlp fc (W -> 4W, tanh-GELU); out-proj and fc2 are in test_conv_in_place_residual
CLIP_ROWS = (300, 539, 771)
CLIP_WIDTHS = (512, 768, 1024)
# ... and at the row counts of the benchmark's batches, at their own widths: ViT-B/32 images (256 x 50), ViT-L/14 images
# (64 x 257) and 256 text queries (256 x 77) of both towers' text widths
CLIP_BENCH = ((12800, 768), (16448, 1024), (19712, 512), (19712, 768))
CLIP_SHAPES = [(rows, W) for rows in CLIP_ROWS for W in CLIP_WIDTHS] + list(CLIP_BENCH)


def _clip_cases(shapes):
    return [(1, 1, rows, W, m * W, 1, 1, act, False, False, W, 0, m * W, 0, 0) for rows, W in shapes for m, act in ((3, 0), (4, 2))]


# the bench row counts go last, so that the earlier cases keep their positions
CASES += _clip_cases(CLIP_SHAPES[:-len(CLIP_BENCH)]) + GROUPED_CASES + _clip_cases(CLIP_BENCH)

# fp32 outputs against the float64 reference: |got - ref| <= F32_BAR * (sum_k |x_k w_k| + |bias| + |res|) per element,
# the magnitude the fp32 accumulator and the epilogue's fp32 roundings carry.  Measured on an H100: at most 0.045 x 2^-16
# on the CLIP shapes (K up to 4096) and 0.1 x 2^-16 on the K = 64 SiLU convs, so 2^-18 leaves 2.5x headroom.
# The tensor core's fp32 accumulator truncates, so its error grows in proportion to the k16 steps into one accumulator:
# the bar holds per F32_STEPS steps (K = 4096).  Every case here stays within that; a longer K takes
# F32_BAR x steps / F32_STEPS (tests/test_plan_convs_gpu.py: the fp32-accurate mode's cross-product GEMMs, up to 1440 steps).
F32_BAR = 2.0 ** -18
F32_STEPS = 256
F32_REL = 2e-3           # and |got - ref| / max(|ref|, 1): the tighter bar where the sum cancels heavily
TANH_Z = 2.0 ** -12      # tanh.approx.f32 errs by <= 2^-11, so SiLU and tanh-GELU (z/2 (1 + tanh)) err by <= 2^-12 |z|
RN_WINDOW = 0.02         # |mean (got - y) sign(y) / ulp_bf16(y)| of a round-to-nearest store over >= 10^4 outputs
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(_WORST):
        print(f"\nworst {key}: {_WORST[key]:.3f}")


def bf16_bar(z, y, mag, act):
    """Per-element bar of a bf16 output y = [res +] act(z): 2^-7 |y| + 2^-12 |z| (act != 0) + F32_BAR x mag."""
    bar = 2.0 ** -7 * y.abs() + F32_BAR * mag
    return bar + TANH_Z * z.abs() if act else bar


def rn_bias(got, y, noise):
    """(mean of (got - y) sign(y) / ulp_bf16(y), elements used) over the outputs whose fp32-level error bound `noise` is
    below 1/16 of their bf16 ulp (elsewhere the fp32 error, not the store, decides the sign)."""
    ulp = torch.pow(2.0, torch.floor(torch.log2(y.abs())) - 7)
    keep = (y != 0) & (noise < ulp / 16)
    return ((got - y) * torch.sign(y) / ulp)[keep].mean().item(), int(keep.sum().item())


def bf16_trunc(v):
    """v (float64) stored to bf16 the wrong way: rounded to fp32, then truncated toward zero."""
    return (v.float().view(torch.int32) & -65536).view(torch.float32).double()


def ref64(x, w, b, k, s, act, res, groups=1):
    """float64 (z, y = [res +] act(z), sum|x.w| + |b| + |res|) of the conv on the stored (bf16 / fp32) operands."""
    x, w, b = x.double(), w.double(), b.double()
    res = None if res is None else res.double()
    z = _ref(x, w, b, k, s, 0, None, groups)
    y = _ref(x, w, b, k, s, act, res, groups)
    mag = _ref(x.abs(), w.abs(), b.abs(), k, s, 0, None if res is None else res.abs(), groups)
    return z, y, mag


def _check_bf16(got, z, y, mag, act, what):
    assert torch.isfinite(got).all()
    r = ((got.double() - y).abs() / bf16_bar(z, y, mag, act)).max().item()
    _WORST["bf16 |err|/bar"] = max(_WORST.get("bf16 |err|/bar", 0.0), r)
    line = f"{what}: bf16 worst |err|/bar {r:.3f}"
    if act == 0 and y.numel() >= 10 ** 4:
        bias, n = rn_bias(got.double(), y, F32_BAR * mag)
        _WORST["bf16 act-0 |rounding bias|"] = max(_WORST.get("bf16 act-0 |rounding bias|", 0.0), abs(bias))
        line += f", rounding bias {bias:+.4f} ulp over {n} outputs"
        assert n >= 10 ** 4 and abs(bias) <= RN_WINDOW, line
    print(line)
    assert r <= 1.0, line


def conv_inputs(case):
    """Seeded host inputs of a CASES entry: bf16 input buffer, bf16 weights, fp32 bias, residual (output dtype) or None."""
    N, H, W, Cin, Cout, k, s, act, use_res, out_f32, in_cs, in_co, out_cs, out_co, bn = case[:15]
    groups = case[15] if len(case) > 15 else 1
    g = torch.Generator().manual_seed(1234 + N + H + Cin)
    xbuf = torch.randn(N, H, W, in_cs, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin // groups, generator=g) * (2.0 / (k * k * Cin // groups)) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, generator=g) * 0.1
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    odt = torch.float32 if out_f32 else torch.bfloat16
    res = torch.randn(N, Ho, Wo, Cout, generator=g).to(odt) if use_res else None
    return xbuf, w, b, res


def _ref(x, w, b, k, s, act, res, groups=1):
    y = F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), b, stride=s, padding=k // 2, groups=groups)
    if act == 1:
        y = F.silu(y)
    elif act == 2:
        y = F.gelu(y, approximate="tanh")
    y = y.permute(0, 2, 3, 1)
    if res is not None:
        y = y + res
    return y


def _check_f32(got, x, w, b, k, s, act, res, what="", groups=1):
    """fp32 output vs the float64 reference: the Sum|x.w| bar, and the relative 2e-3 bar where that is tighter."""
    res64 = None if res is None else res.double()
    ref = _ref(x.double(), w.double(), b.double(), k, s, act, res64, groups)
    mag = _ref(x.double().abs(), w.double().abs(), b.double().abs(), k, s, 0, None if res is None else res64.abs(), groups)
    err = (got.double() - ref).abs()
    ratio = (err / (F32_BAR * mag)).max().item()
    print(f"{what}: fp32 worst |err|/bar {ratio:.3f}, max rel err {(err / ref.abs().clamp(min=1.0)).max().item():.2e}")
    assert torch.isfinite(got).all()
    assert ratio <= 1.0, f"worst |err|/(F32_BAR * sum|x.w|) {ratio:.3f} (abs {err.max().item()})"
    assert (err / ref.abs().clamp(min=1.0)).max().item() < F32_REL


@pytest.mark.parametrize("impl", [1, 2])
@pytest.mark.parametrize("case", CASES)
def test_conv_matches_torch(case, impl):
    N, H, W, Cin, Cout, k, s, act, use_res, out_f32, in_cs, in_co, out_cs, out_co, bn = case[:15]
    groups = case[15] if len(case) > 15 else 1
    if impl == 2 and N * H * W * Cout * Cin * k * k > 3e10:
        pytest.skip("direct kernel: skip the biggest case")
    if impl == 1 and groups > 1:
        pytest.skip("grouped convs run on the direct kernel only")
    xbuf, w, b, res = (None if t is None else t.cuda() for t in conv_inputs(case))
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    odt = torch.float32 if out_f32 else torch.bfloat16
    dev = "cuda"
    obuf = torch.full((N, Ho, Wo, out_cs), -7.0, device=dev, dtype=odt)
    ops.conv2d(xbuf, in_co, Cin, w, b, k, s, obuf, out_co, Cout, act=act, res=res, res_co=0, groups=groups, impl=impl, bn=bn)
    torch.cuda.synchronize()
    x = xbuf[..., in_co:in_co + Cin].float()
    got = obuf[..., out_co:out_co + Cout].float()
    if out_f32:
        _check_f32(got, x, w.float(), b, k, s, act, res, f"{case} impl {impl}", groups)
    else:
        z, y, mag = ref64(x, w.float(), b, k, s, act, res, groups)
        _check_bf16(got, z, y, mag, act, f"{case} impl {impl}")
    # untouched channels of the wider output buffer keep their sentinel
    if out_cs > Cout:
        mask = torch.ones(out_cs, dtype=torch.bool, device=dev)
        mask[out_co:out_co + Cout] = False
        assert (obuf[..., mask] == -7.0).all()


# (N, H, W, Cin, Cout, k, act, out_f32, bn, out_cs): RepNBottleneck-like convs into the upper half of a 2 x Cout buffer, then
# the CLIP residual stream: out-proj (W -> W) and fc2 (4W -> W) write fp32 in place into the dense [rows, W] stream, at an
# explicit BN = 128 (the tile width of large batches; an explicit bn keeps the grid heuristic from halving it)
RESIDUAL_CASES = [pytest.param(3, 24, 40, 64, Cout, k, 1, f32, 0, 2 * Cout, id=f"{Cout}-{f32}-{k}")
                  for Cout, f32, k in [(32, False, 3), (64, False, 3), (128, False, 1), (16, True, 1), (64, True, 3), (96, False, 1)]]
RESIDUAL_CASES += [pytest.param(1, 1, rows, m * W, W, 1, 0, True, 128, W, id=f"clip-{name}-{rows}x{W}")
                   for m, name in ((1, "out_proj"), (4, "fc2")) for rows, W in CLIP_SHAPES]


def residual_inputs(N, H, W, Cin, Cout, k, out_f32, out_cs):
    """Seeded host inputs of a RESIDUAL_CASES entry: bf16 input, bf16 weights, fp32 bias, the output buffer (= residual)."""
    g = torch.Generator().manual_seed(77 + Cout + Cin + W)
    x = torch.randn(N, H, W, Cin, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin, generator=g) * (2.0 / (k * k * Cin)) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, generator=g) * 0.1
    obuf = torch.randn(N, H, W, out_cs, generator=g).to(torch.float32 if out_f32 else torch.bfloat16)
    return x, w, b, obuf


@pytest.mark.parametrize("N,H,W,Cin,Cout,k,act,out_f32,bn,out_cs", RESIDUAL_CASES)
def test_conv_in_place_residual(N, H, W, Cin, Cout, k, act, out_f32, bn, out_cs):
    """out = act(conv(x)) + out, the RepNBottleneck / transformer residual form: the epilogue reads each residual element
    before it writes the same element, in bf16 and fp32 and at every tile width."""
    x, w, b, obuf = (t.cuda() for t in residual_inputs(N, H, W, Cin, Cout, k, out_f32, out_cs))
    out_co = out_cs - Cout
    before = obuf.clone()
    ops.conv2d(x, 0, Cin, w, b, k, 1, obuf, out_co, Cout, act=act, res=obuf, res_co=out_co, impl=1, bn=bn)
    torch.cuda.synchronize()
    got = obuf[..., out_co:]
    if out_f32:
        _check_f32(got, x.float(), w.float(), b, k, 1, act, before[..., out_co:], f"in place {N}x{H}x{W} {Cin}->{Cout}")
    else:
        z, y, mag = ref64(x.float(), w.float(), b, k, 1, act, before[..., out_co:].float())
        _check_bf16(got.float(), z, y, mag, act, f"in place {N}x{H}x{W} {Cin}->{Cout}")
    assert torch.equal(obuf[..., :out_co], before[..., :out_co])
