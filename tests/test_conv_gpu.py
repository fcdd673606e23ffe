"""GPU parity of the wgmma implicit-GEMM conv (and the direct conv) against a plain fp32 torch conv2d
on the same bf16-rounded operands.  Reference op: detection/yolov9.py:33-38 (Conv = Conv2d+bias -> SiLU)."""
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


def _ref(x, w, b, k, s, act, res):
    y = F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), b, stride=s, padding=k // 2)
    if act == 1:
        y = F.silu(y)
    elif act == 2:
        y = F.gelu(y, approximate="tanh")
    y = y.permute(0, 2, 3, 1)
    if res is not None:
        y = y + res
    return y


@pytest.mark.parametrize("impl", [1, 2])
@pytest.mark.parametrize("case", CASES)
def test_conv_matches_torch(case, impl):
    N, H, W, Cin, Cout, k, s, act, use_res, out_f32, in_cs, in_co, out_cs, out_co, bn = case
    if impl == 2 and N * H * W * Cout * Cin * k * k > 3e10:
        pytest.skip("direct kernel: skip the biggest case")
    g = torch.Generator(device="cuda").manual_seed(1234 + N + H + Cin)
    dev = "cuda"
    xbuf = torch.randn(N, H, W, in_cs, device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin, device=dev, generator=g) * (2.0 / (k * k * Cin)) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, device=dev, generator=g) * 0.1
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    odt = torch.float32 if out_f32 else torch.bfloat16
    obuf = torch.full((N, Ho, Wo, out_cs), -7.0, device=dev, dtype=odt)
    res = torch.randn(N, Ho, Wo, Cout, device=dev, generator=g).to(odt) if use_res else None
    ops.conv2d(xbuf, in_co, Cin, w, b, k, s, obuf, out_co, Cout, act=act, res=res, res_co=0, impl=impl, bn=bn)
    torch.cuda.synchronize()
    x = xbuf[..., in_co:in_co + Cin].float()
    ref = _ref(x, w.float(), b, k, s, act, None if res is None else res.float())
    got = obuf[..., out_co:out_co + Cout].float()
    tol = 2e-2 if not out_f32 else 2e-3
    err = (got - ref).abs()
    scale = ref.abs().clamp(min=1.0)
    assert torch.isfinite(got).all()
    assert (err / scale).max().item() < tol, f"max rel err {(err / scale).max().item()} (abs {err.max().item()})"
    # untouched channels of the wider output buffer keep their sentinel
    if out_cs > Cout:
        mask = torch.ones(out_cs, dtype=torch.bool, device=dev)
        mask[out_co:out_co + Cout] = False
        assert (obuf[..., mask] == -7.0).all()


@pytest.mark.parametrize("Cout,out_f32,k", [(32, False, 3), (64, False, 3), (128, False, 1), (16, True, 1), (64, True, 3), (96, False, 1)])
def test_conv_in_place_residual(Cout, out_f32, k):
    """out = act(conv(x)) + out, the RepNBottleneck / transformer residual form: the epilogue reads each residual element
    before it writes the same element, in bf16 and fp32 and at every tile width."""
    g = torch.Generator(device="cuda").manual_seed(77 + Cout)
    N, H, W, Cin = 3, 24, 40, 64
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, k, k, Cin, device="cuda", generator=g) * (2.0 / (k * k * Cin)) ** 0.5).to(torch.bfloat16)
    b = torch.randn(Cout, device="cuda", generator=g) * 0.1
    odt = torch.float32 if out_f32 else torch.bfloat16
    out_cs, out_co = 2 * Cout, Cout
    obuf = torch.randn(N, H, W, out_cs, device="cuda", generator=g).to(odt)
    before = obuf.clone()
    ops.conv2d(x, 0, Cin, w, b, k, 1, obuf, out_co, Cout, act=1, res=obuf, res_co=out_co, impl=1)
    torch.cuda.synchronize()
    ref = _ref(x.float(), w.float(), b, k, 1, 1, before[..., out_co:].float())
    got = obuf[..., out_co:].float()
    err = ((got - ref).abs() / ref.abs().clamp(min=1.0)).max().item()
    assert err < (2e-3 if out_f32 else 2e-2), err
    assert torch.equal(obuf[..., :out_co], before[..., :out_co])
