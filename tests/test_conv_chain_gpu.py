"""cc_conv2d_chain (a conv with a square 1x1 conv run in its epilogue) against the same two convs as two cc_conv2d calls:
the results must be equal bit for bit.  The shapes are the chains the detector's plans build (layer 1's 3x3/s2 conv -> ELAN
cv1, RepNCSP's last bottleneck cv2 -> cv3 over [x1 | x3], ELAN cv1 -> cv2.0 cv1+cv2 on y1, ELAN cv2.1 -> cv3.0 cv1+cv2 on y2,
the head's cv2.j.1 -> cv2.j.2 logits) at the map sizes of 640x640 and 384x640 inputs, plus maps whose edge tiles are
clipped."""
import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200._lib import CCError

pytestmark = pytest.mark.gpu

# (B, H, W): 160^2 / 80^2 / 40^2 / 20^2 maps of 640x640, 96x160 / 48x80 / 12x20 of 384x640, and clipped edge tiles
MAPS = [(1, 160, 160), (32, 80, 80), (1, 40, 40), (32, 20, 20), (1, 96, 160), (32, 48, 80), (1, 12, 20), (3, 13, 37), (2, 7, 9)]


def _rand(shape, scale, g):
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).cuda()


def _conv_w(cout, k, cin, g):
    return _rand((cout, k, k, cin), 1.0 / (k * k * cin) ** 0.5, g), (torch.randn(cout, generator=g) * 0.1).cuda()


def _standalone_splits(N, H, W, cout2):
    """the standalone 1x1 halves a 128-channel tile when the map has fewer 128-pixel tiles than SMs: no chain then"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return cout2 > 64 and (N * H * W + 127) // 128 < sms


def _maps(b):
    # B = 32 at a 160^2 map of 4b channels is a 26-210 MB tensor: keep the large batches for the smaller maps
    return [m for m in MAPS if m[0] * m[1] * m[2] * b <= 32 * 80 * 80 * 64]


@pytest.mark.parametrize("b", [16, 32, 64])
def test_repncsp_cv2_cv3(b):
    """last bottleneck cv2 (3x3, in-place residual on x1) -> cv3 over [x1 | x3]; x1's final value is dropped"""
    for (N, H, W) in _maps(b):
        g = torch.Generator().manual_seed(1000 * b + H)
        t1 = _rand((N, H, W, 2 * b), 1.0, g)
        t2 = _rand((N, H, W, b), 1.0, g)
        w, bias = _conv_w(b, 3, b, g)
        w2, bias2 = _conv_w(2 * b, 1, 2 * b, g)
        ref1 = t1.clone()
        ops.conv2d(t2, 0, b, w, bias, 3, 1, ref1, 0, b, act=1, res=ref1, res_co=0)
        ref = torch.empty(N, H, W, 2 * b, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(ref1, 0, 2 * b, w2, bias2, 1, 1, ref, 0, 2 * b, act=1)
        got1 = t1.clone()
        got = torch.full_like(ref, float("nan"))
        run = lambda: ops.conv2d_chain(t2, 0, b, w, bias, 3, 1, got1, 0, w2, bias2, 0, got, 0, act2=1, part=got1, part_co=b,
                                       part_C=b, res=got1, res_co=0, store1=False)
        if _standalone_splits(N, H, W, 2 * b):
            with pytest.raises(CCError, match="tile its 128 channels in blocks"):
                run()
            continue
        run()
        torch.cuda.synchronize()
        assert torch.equal(got, ref), (b, N, H, W)
        assert torch.equal(got1, t1), "a dropped first output must not be written"


def test_conv_s2_chain_elan_cv1():
    """layer 1 (3x3 stride 2, 64 -> 128) -> ELAN cv1 (1x1 128 -> 128); layer 1's output is dropped"""
    for (N, H, W) in _maps(4 * 128):
        g = torch.Generator().manual_seed(500 + H)
        x = _rand((N, 2 * H, 2 * W, 64), 1.0, g)
        w, bias = _conv_w(128, 3, 64, g)
        w2, bias2 = _conv_w(128, 1, 128, g)
        y = torch.empty(N, H, W, 128, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(x, 0, 64, w, bias, 3, 2, y, 0, 128, act=1)
        ref = torch.empty(N, H, W, 128, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(y, 0, 128, w2, bias2, 1, 1, ref, 0, 128, act=1)
        got = torch.full_like(ref, float("nan"))
        run = lambda: ops.conv2d_chain(x, 0, 64, w, bias, 3, 2, None, 0, w2, bias2, 0, got, 0, act2=1, store1=False)
        if _standalone_splits(N, H, W, 128):
            with pytest.raises(CCError, match="tile its 128 channels in blocks"):
                run()
            continue
        run()
        torch.cuda.synchronize()
        assert torch.equal(got, ref), (N, H, W)


@pytest.mark.parametrize("b", [16, 32, 64])
def test_elan_cv1_chain_y1(b):
    """ELAN cv1 (1x1 -> cat[0, 4b), kept) -> RepNCSP cv2.0 cv1+cv2 on y1 = cat[2b, 4b), the upper half of the n block"""
    cin = 4 * b
    for (N, H, W) in _maps(4 * b):
        g = torch.Generator().manual_seed(2000 * b + H)
        x = _rand((N, H, W, cin + 16), 1.0, g)
        w, bias = _conv_w(4 * b, 1, cin, g)
        w2, bias2 = _conv_w(2 * b, 1, 2 * b, g)
        ref_cat = torch.zeros(N, H, W, 8 * b, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(x, 16, cin, w, bias, 1, 1, ref_cat, 0, 4 * b, act=1)
        ref = torch.zeros(N, H, W, 2 * b + 32, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(ref_cat, 2 * b, 2 * b, w2, bias2, 1, 1, ref, 16, 2 * b, act=1)
        got_cat = torch.zeros_like(ref_cat)
        got = torch.zeros_like(ref)
        run = lambda: ops.conv2d_chain(x, 16, cin, w, bias, 1, 1, got_cat, 0, w2, bias2, 2 * b, got, 16, act2=1, store1=True)
        if _standalone_splits(N, H, W, 2 * b):
            with pytest.raises(CCError, match="tile its 128 channels in blocks"):
                run()
            continue
        run()
        torch.cuda.synchronize()
        assert torch.equal(got_cat, ref_cat), (b, N, H, W)
        assert torch.equal(got, ref), (b, N, H, W)


@pytest.mark.parametrize("b", [16, 32, 64])
def test_elan_cv21_chain_y2(b):
    """ELAN cv2.1 (3x3 -> cat[4b, 6b), kept) -> RepNCSP cv3.0 cv1+cv2 on y2"""
    for (N, H, W) in _maps(8 * b):
        g = torch.Generator().manual_seed(3000 * b + H)
        r1 = _rand((N, H, W, 2 * b), 1.0, g)
        w, bias = _conv_w(2 * b, 3, 2 * b, g)
        w2, bias2 = _conv_w(2 * b, 1, 2 * b, g)
        ref_cat = torch.zeros(N, H, W, 8 * b, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(r1, 0, 2 * b, w, bias, 3, 1, ref_cat, 4 * b, 2 * b, act=1)
        ref = torch.zeros(N, H, W, 2 * b, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(ref_cat, 4 * b, 2 * b, w2, bias2, 1, 1, ref, 0, 2 * b, act=1)
        got_cat = torch.zeros_like(ref_cat)
        got = torch.zeros_like(ref)
        run = lambda: ops.conv2d_chain(r1, 0, 2 * b, w, bias, 3, 1, got_cat, 4 * b, w2, bias2, 0, got, 0, act2=1, store1=True)
        if _standalone_splits(N, H, W, 2 * b):
            with pytest.raises(CCError, match="tile its 128 channels in blocks"):
                run()
            continue
        run()
        torch.cuda.synchronize()
        assert torch.equal(got_cat, ref_cat), (b, N, H, W)
        assert torch.equal(got, ref), (b, N, H, W)


def test_head_box_logits_fp32():
    """head cv2.j.1 (3x3 64 -> 64) -> cv2.j.2 (1x1 64 -> 64, no activation, fp32 logits); tb is dropped"""
    for (N, H, W) in _maps(64):
        g = torch.Generator().manual_seed(4000 + H)
        t0 = _rand((N, H, W, 64 + 80), 1.0, g)
        w, bias = _conv_w(64, 3, 64, g)
        w2, bias2 = _conv_w(64, 1, 64, g)
        tb = torch.empty(N, H, W, 64, dtype=torch.bfloat16, device="cuda")
        ops.conv2d(t0, 0, 64, w, bias, 3, 1, tb, 0, 64, act=1)
        ref = torch.empty(N, H, W, 64, dtype=torch.float32, device="cuda")
        ops.conv2d(tb, 0, 64, w2, bias2, 1, 1, ref, 0, 64, act=0)
        got = torch.full_like(ref, float("nan"))
        ops.conv2d_chain(t0, 0, 64, w, bias, 3, 1, None, 0, w2, bias2, 0, got, 0, act2=0, store1=False)
        torch.cuda.synchronize()
        assert torch.equal(got, ref), (N, H, W)


def test_rejects_pairs_that_do_not_chain():
    g = torch.Generator().manual_seed(5)
    x = _rand((1, 40, 40, 128), 1.0, g)
    o = torch.zeros(1, 40, 40, 256, dtype=torch.bfloat16, device="cuda")
    o2 = torch.zeros(1, 40, 40, 256, dtype=torch.bfloat16, device="cuda")
    o2f = torch.zeros(1, 40, 40, 128, dtype=torch.float32, device="cuda")
    w64, b64 = _conv_w(64, 3, 128, g)
    w128, b128 = _conv_w(128, 3, 128, g)
    sq = {c: _conv_w(c, 1, c, g) for c in (32, 64, 128, 256)}
    bad = [
        # the 1x1 has more than 128 channels
        dict(w=w128, bias=b128, w2=sq[256], k0=0, o2=o2),
        # on this small map the standalone 1x1 would tile its 128 channels as two 64-channel blocks
        dict(w=w128, bias=b128, w2=sq[128], k0=0, o2=o2),
        # the input run [32, 96) crosses the end of the 64-channel output
        dict(w=w64, bias=b64, w2=sq[64], k0=32, o2=o2),
        # fp32 output of more than 64 channels
        dict(w=w128, bias=b128, w2=sq[128], k0=0, o2=o2f, act2=0),
        # SiLU into an fp32 output
        dict(w=w64, bias=b64, w2=sq[64], k0=0, o2=o2f, act2=1),
        # a partner that is not one staging box wide (64 channels here)
        dict(w=w64, bias=b64, w2=sq[64], k0=0, o2=o2, part=x, part_C=32),
        # a k0 that is not on a k16 step
        dict(w=w64, bias=b64, w2=sq[32], k0=8, o2=o2),
    ]
    for a in bad:
        w2, bias2 = a["w2"]
        with pytest.raises(CCError, match="cc_conv2d_chain"):
            ops.conv2d_chain(x, 0, 128, a["w"], a["bias"], 3, 1, o, 0, w2, bias2, a["k0"], a["o2"], 0, act2=a.get("act2", 1),
                             part=a.get("part"), part_co=0, part_C=a.get("part_C", 0))
    torch.cuda.synchronize()
    assert not o.any() and not o2.any() and not o2f.any(), "a refused chain must launch nothing"


def test_rejects_residual_on_a_128_channel_tile():
    g = torch.Generator().manual_seed(6)
    x = _rand((1, 160, 160, 128), 1.0, g)
    o = torch.zeros(1, 160, 160, 128, dtype=torch.bfloat16, device="cuda")
    o2 = torch.zeros_like(o)
    w, bias = _conv_w(128, 3, 128, g)
    w2, bias2 = _conv_w(128, 1, 128, g)
    with pytest.raises(CCError, match="takes no residual"):
        ops.conv2d_chain(x, 0, 128, w, bias, 3, 1, o, 0, w2, bias2, 0, o2, 0, act2=1, res=o, res_co=0)
    torch.cuda.synchronize()
    assert not o.any() and not o2.any()
