"""Convs whose tile plan mixes widths (conv_gemm.cu plan_tiles): the last wave's tiles split along N into narrow tiles, and
the remainder channel block of a Cout that the wide width does not divide.  Each launch must give exactly the output of the
same conv forced to uniform tiles (bn=), pass tests/test_conv_gpu.py's float64 bar, and write every element of its output
slice once and nothing outside it.

Tile counts are 128-pixel tiles x n blocks on 132 SMs; r = tiles mod 132 decides the tail split: s = BN / BNn narrow tiles
per last-wave tile with s r <= 132."""
import pytest
import torch

import test_conv_gpu as tc
from clearcam_b200 import ops

pytestmark = pytest.mark.gpu

NAN = float("nan")

# (id, N, H, W, Cin, Cout, k, s, act, f32, res, out_cs, out_co, uniform bn); act 3 = PReLU; res: None, "sep" (a separate
# residual tensor) or "inplace" (the output slice holds the residual)
CASES = [
    # 133 tiles of 128 (r = 1) -> 132 wide + 8 x 16-wide
    ("r1-128x16", 1, 1, 133 * 128, 64, 128, 1, 1, 1, False, None, 128, 0, 128),
    # 136 tiles (r = 4) -> 132 + 32 x 16-wide, fp32 into the residual in place
    ("r4-128x16-f32-inplace", 1, 1, 136 * 128, 64, 128, 1, 1, 0, True, "inplace", 160, 32, 128),
    # 3x3: 68 images x 2 tiles = 136 (r = 4), SiLU + residual
    ("r4-128x16-3x3-res", 68, 16, 16, 64, 128, 3, 1, 1, False, "sep", 128, 0, 128),
    # 200 tiles (r = 68): no split fits, uniform
    ("r68-128-gelu", 1, 1, 200 * 128, 64, 128, 1, 1, 2, False, None, 192, 64, 128),
    # 263 tiles at BN = 64 (r = 131): uniform
    ("r131-64", 1, 1, 263 * 128, 64, 64, 1, 1, 0, False, None, 64, 0, 64),
    # 3x3 stride 2: 76 images x 2 tiles = 152 (r = 20) -> 132 + 80 x 32-wide
    ("r20-128x32-s2", 76, 32, 32, 64, 128, 3, 2, 1, False, None, 128, 0, 128),
    # 172 tiles (r = 40) -> 132 + 80 x 64-wide, fp32 + residual
    ("r40-128x64-f32-res", 1, 1, 172 * 128, 128, 128, 1, 1, 0, True, "sep", 128, 0, 128),
    # PReLU at BN = 64: 136 tiles (r = 4) -> 132 + 16 x 16-wide
    ("r4-64x16-prelu", 68, 16, 16, 64, 64, 3, 1, 3, False, None, 96, 16, 64),
    # 172 tiles at BN = 64 (r = 40) -> 132 + 80 x 32-wide
    ("r40-64x32", 1, 1, 172 * 128, 64, 64, 1, 1, 1, False, None, 64, 0, 64),
    # BN = 32: 136 tiles (r = 4) -> 132 + 8 x 16-wide, residual in place
    ("r4-32x16-inplace", 68, 16, 16, 32, 32, 3, 1, 1, False, "inplace", 64, 16, 32),
    # remainder blocks: 320 = 128 + 128 + 64 (the detect head's stacked 3x3), 96 = 64 + 32 (stride 2, into a wider buffer)
    # and 48 = 32 + 16 (residual in place); 80 (the class logits, fp32) stays 5 x 16, its 16-wide remainder too narrow
    ("cout320-3x3", 8, 40, 40, 64, 320, 3, 1, 1, False, None, 320, 0, 64),
    ("cout80-f32", 32, 40, 40, 256, 80, 1, 1, 0, True, None, 80, 0, 16),
    ("cout96-s2", 16, 80, 80, 64, 96, 3, 2, 0, False, None, 128, 16, 32),
    ("cout48-inplace", 16, 40, 40, 64, 48, 3, 1, 1, False, "inplace", 64, 8, 16),
]


def _run(case, xbuf, w, bias, slope, res, bn):
    _, N, H, W, Cin, Cout, k, s, act, f32, res_mode, out_cs, out_co, _ = case
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    obuf = torch.full((N, Ho, Wo, out_cs), NAN, device="cuda", dtype=torch.float32 if f32 else torch.bfloat16)
    rbuf, rco = res, 0
    if res_mode == "inplace":
        obuf[..., out_co:out_co + Cout] = res
        rbuf, rco = obuf, out_co
    ops.conv2d(xbuf, 0, Cin, w, bias, k, s, obuf, out_co, Cout, act=act, res=rbuf, res_co=rco, bn=bn, slope=slope)
    torch.cuda.synchronize()
    return obuf


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_mixed_tiles_match_uniform(case):
    _, N, H, W, Cin, Cout, k, s, act, f32, res_mode, out_cs, out_co, bn = case
    g = torch.Generator().manual_seed(7 + Cout + N)
    xbuf = torch.randn(N, H, W, Cin, generator=g).to(torch.bfloat16).cuda()
    w = (torch.randn(Cout, k, k, Cin, generator=g) * (2.0 / (k * k * Cin)) ** 0.5).to(torch.bfloat16).cuda()
    b = torch.randn(Cout, generator=g) * 0.1
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    odt = torch.float32 if f32 else torch.bfloat16
    res = torch.randn(N, Ho, Wo, Cout, generator=g).to(odt).cuda() if res_mode else None
    slope = None
    bias = b.cuda()
    if act == 3:     # PReLU: every border class gets the same bias row, so that the reference is a plain conv
        bias = b.repeat(9, 1).contiguous().cuda()
        slope = (torch.rand(Cout, generator=g) * 0.5).cuda()
    mixed = _run(case, xbuf, w, bias, slope, res, 0)
    uniform = _run(case, xbuf, w, bias, slope, res, bn)
    got = mixed[..., out_co:out_co + Cout]
    assert torch.isfinite(got).all(), "an output element was not written"
    outside = torch.ones(out_cs, dtype=torch.bool, device="cuda")
    outside[out_co:out_co + Cout] = False
    assert torch.isnan(mixed[..., outside]).all(), "a channel outside the output slice was written"
    assert torch.equal(mixed.nan_to_num(0.0), uniform.nan_to_num(0.0)), "mixed tile widths differ from uniform tiles"
    x, wf, resc = xbuf.float().cpu(), w.float().cpu(), None if res is None else res.cpu()
    gotc = got.float().cpu()
    if act == 3:
        z, _, mag = tc.ref64(x, wf, b, k, s, 0, None)
        sl = slope.cpu().double()
        y = torch.where(z > 0, z, sl * z)
        tc._check_bf16(gotc, z, y, mag, 0, case[0])
    elif f32:
        tc._check_f32(gotc, x, wf, b, k, s, act, resc, case[0])
    else:
        z, y, mag = tc.ref64(x, wf, b, k, s, act, resc)
        tc._check_bf16(gotc, z, y, mag, act, case[0])
