"""The CLIP encoders' kernels outside attention and the GEMMs (vit.cu), called directly through their C-ABI taps and
compared element by element with exact or float64 references:

* patchify, bit-exact: the bf16 patch matrix of the 14x14 / 32x32 / 16x16 patch conv, zeros in the pad columns;
* LayerNorm -> bf16 at every width the kernel is instantiated for, on rows that stress fp32 statistics (a common offset
  10^3 times the spread, one outlier 10^4 times the rest, constant rows, variance near eps), with the ln_post (token 0) and
  ln_final (EOT row index) gathers;
* class token + positional embedding + ln_pre, in place on the fp32 stream;
* the text embedding (exact) and its EOT argmax, with clamped ids;
* the final L2 normalisation, with and without eps;
* both encoders with zero transformer blocks through the public API, which is the plans' own wiring of the kernels above
  and of the patch and projection GEMMs.

LayerNorm bar, per element: |got - y| <= 2^-8 |y| + (1 + 2^-8) D.  2^-8 |y| is the bf16 half-ulp; D bounds the fp32
statistics for the kernel's own order (each lane sums 4 N4 values, then a 5-level shuffle tree; rsqrtf within 2 ulps), derived
per row in float64 by `ln64`.  That bar cannot see an epilogue that truncates instead of rounding, nor a variance divided by
W - 1, so over >= 10^5 gaussian elements the mean of (got - y) sign(y) / ulp_bf16(y) must also lie within +-0.02: rounding to
nearest gives about 0, truncation -0.5.

Each tolerance-based test prints its worst |err|/bar.  `test_bars_see_clip_bugs` shows without a GPU, on the GPU tests' own
inputs (and those of tests/test_conv_gpu.py), that the typical bugs of these kernels leave their bars by at least 4x.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from clearcam_b200 import ops
from clearcam_b200._lib import check, lib
from clearcam_b200.models.objects import _ClipConfig

import test_conv_gpu as tc

SENT = -7.0
U = 2.0 ** -24                 # fp32 unit roundoff
LN_EPS = 1e-5
RN_WINDOW = tc.RN_WINDOW       # +-0.02 ulp: the rounding-direction window
GRID_ROWS = 132 * 4 * 8        # the row kernels run at most 528 CTAs of 8 warps: 4224 rows per grid-stride pass
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(_WORST):
        print(f"\nworst {key}: {_WORST[key]:.3f}")


def _ratio(key, err, bar, what=""):
    r = (err / bar).max().item()
    _WORST[key + " |err|/bar"] = max(_WORST.get(key + " |err|/bar", 0.0), r)
    print(f"{key} {what}: worst |err|/bar {r:.3f}")
    assert math.isfinite(r) and r <= 1.0, f"{key} {what}: worst |err|/bar {r:.3f}"


def _bias(key, got, y, noise, what=""):
    b, n = tc.rn_bias(got, y, noise)
    _WORST[key + " |rounding bias|"] = max(_WORST.get(key + " |rounding bias|", 0.0), abs(b))
    print(f"{key} {what}: rounding bias {b:+.4f} ulp over {n} elements")
    assert n >= 10 ** 5 and abs(b) <= RN_WINDOW, f"{key} {what}: rounding bias {b:+.4f} ulp over {n} elements"


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------ float64 LayerNorm + its bar
def ln64(x, g, b, E=None, eps=LN_EPS, ddof=0, one_pass=False):
    """float64 LayerNorm of rows x (the fp32 values the kernel reads, or float64 values known to within E per row) with
    gamma g and beta b, and D: a bound on the kernel's fp32 output error.

    The kernel's sum of W values runs 4 N4 - 1 sequential adds per lane, one into the accumulator and 5 tree levels, so each
    sum errs by <= ns U sum|.| with ns = 4 N4 + 6.  Mean: dmu = ns U sum|x| / W + U |mu| (+ E).  Variance of x - mu_hat:
    off by <= 2 e mean|x - mu| + e^2 with e = dmu + E, and its sum of squares (2 more roundings per term) by (ns + 4) U;
    + eps rounds once.  rsqrtf errs by <= 2 ulps.  Output (x - mu_hat) rstd g + b: the mean error times rstd |g|, the
    relative rstd error (and 4 roundings) times |x - mu| rstd |g|, and 2 roundings of |y| + |b|.
    ddof / eps / one_pass: the bugs the bars must see (ddof = 1 divides the variance by W - 1; one_pass computes
    E[x^2] - E[x]^2 in fp32)."""
    x64 = x.double()
    g, b = g.double().to(x.device), b.double().to(x.device)
    W = x.shape[-1]
    ns = 4 * (W // 128) + 6
    mu = x64.mean(-1, keepdim=True)
    d = x64 - mu
    var = (d * d).sum(-1, keepdim=True) / (W - ddof)
    if one_pass:
        xf = x.float()
        var = ((xf * xf).sum(-1, keepdim=True) / W - (xf.sum(-1, keepdim=True) / W) ** 2).double().clamp(min=0)
    rstd = 1 / torch.sqrt(var + eps)
    y = d * rstd * g + b
    e = ns * U * x64.abs().sum(-1, keepdim=True) / W + U * mu.abs() + (0 if E is None else E)
    mad = d.abs().mean(-1, keepdim=True)
    dvar = 2 * e * mad + e * e
    dvar = dvar + (ns + 4) * U * (var + dvar) + U * (var + eps)
    t = dvar / (var + eps)
    rel = 0.5 * t / (1 - t).clamp(min=0.5) + 4 * U
    delta = g.abs() * rstd * (e * (1 + rel) + d.abs() * (rel + 4 * U)) + 2 * U * (y.abs() + b.abs())
    return y, delta


def ln_bar(y, delta):
    return 2.0 ** -8 * y.abs() + (1 + 2.0 ** -8) * delta


# row classes, by row index mod 8: 0-3 gaussian, 4 offset 10^3 x the spread, 5 one outlier 10^4 x the rest, 6 constant,
# 7 variance near eps
def ln_inputs(R, W, seed):
    g = _gen(seed)
    kind = torch.arange(R) % 8
    s = torch.exp(0.5 * torch.randn(R, 1, generator=g))
    c = torch.randn(R, 1, generator=g)
    n = torch.randn(R, W, generator=g)
    x = c + s * n
    sign = torch.where(torch.rand(R, 1, generator=g) < 0.5, -1.0, 1.0)
    off = kind == 4
    x[off] = (sign * 1e3 * s + s * n)[off]
    out = kind == 5
    j = torch.randint(0, W, (R,), generator=g)
    xo = s * n
    xo[torch.arange(R), j] = (sign * 1e4 * s)[:, 0]
    x[out] = xo[out]
    x[kind == 6] = (3 * c).expand(R, W)[kind == 6]
    small = kind == 7
    x[small] = (c + 10 ** -2.5 * torch.exp(0.5 * torch.randn(R, 1, generator=g)) * n)[small]
    gamma = 1 + 0.5 * torch.randn(W, generator=g)
    beta = 0.1 * torch.randn(W, generator=g)
    return x.float().contiguous(), gamma, beta, kind


LN_WIDTHS = [128, 256, 384, 512, 640, 768, 1024, 1280, 1536]
LN_ROWS = [1, 7, 9, 1055, 1056, GRID_ROWS, GRID_ROWS + 1, 3 * GRID_ROWS + 1]


def _ln_check(key, got, x, g, b, kind, what):
    y, delta = ln64(x, g, b)
    _ratio(key, (got - y).abs(), ln_bar(y, delta), what)
    gauss = kind.to(x.device) < 4
    if int(gauss.sum()) * x.shape[1] >= 10 ** 5:
        _bias(key, got[gauss], y[gauss], delta[gauss], what)


@pytest.mark.gpu
@pytest.mark.parametrize("W", LN_WIDTHS)
@pytest.mark.parametrize("R", LN_ROWS)
def test_layernorm_bf16_matches_float64(R, W):
    """Every row of an fp32 [R, W] stream -> bf16, at both sides of each grid edge (132 CTAs below 1056 rows, 528 CTAs of
    8 warps and a grid-stride loop above), with a sentinel row after the output."""
    x, g, b, kind = ln_inputs(R, W, seed=R * 31 + W)
    out = torch.full((R + 1, W), SENT, dtype=torch.bfloat16, device="cuda")
    ops.layernorm_bf16(x.cuda(), g.cuda(), b.cuda(), rows=R, out=out)
    torch.cuda.synchronize()
    assert bool((out[R] == SENT).all()), "a row past the output was written"
    _ln_check("layernorm", out[:R].double(), x.cuda(), g.cuda(), b.cuda(), kind, f"{R}x{W}")


# (W, images B, tokens L): ln_post reads token 0 of every image (row_stride = L), past the grid cap at B = 4300
GATHER_CASES = [(1024, 129, 257), (768, 5, 50), (128, 4300, 17), (512, 1, 77)]


@pytest.mark.gpu
@pytest.mark.parametrize("W,B,L", GATHER_CASES)
def test_layernorm_bf16_row_stride(W, B, L):
    """ln_post: output row b is the LayerNorm of row b*L, into dense rows; the other rows are never read (NaN there)."""
    x, g, b, kind = ln_inputs(B, W, seed=B + W + L)
    stream = torch.full((B * L, W), float("nan"))
    stream[::L] = x
    out = torch.full((B + 1, W), SENT, dtype=torch.bfloat16, device="cuda")
    ops.layernorm_bf16(stream.cuda(), g.cuda(), b.cuda(), rows=B, row_stride=L, out=out)
    torch.cuda.synchronize()
    assert bool((out[B] == SENT).all())
    _ln_check("layernorm gather", out[:B].double(), x.cuda(), g.cuda(), b.cuda(), kind, f"stride {L}, {B}x{W}")


# (W, stream rows, gathered rows)
INDEX_CASES = [(768, 77 * 300, 600), (128, 77 * 70, 5000), (1024, 77, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("W,n,R", INDEX_CASES)
def test_layernorm_bf16_row_index(W, n, R):
    """ln_final: output row r is the LayerNorm of row idx[r]; the indices repeat, are unsorted, and include the first and
    last rows of the stream."""
    x, g, b, kind = ln_inputs(n, W, seed=n + W + R)
    idx = torch.randint(0, n, (R,), generator=_gen(R))
    idx[0], idx[-1] = n - 1, 0
    idx[R // 2:R // 2 + 2] = idx[1]
    out = torch.full((R + 1, W), SENT, dtype=torch.bfloat16, device="cuda")
    ops.layernorm_bf16(x.cuda(), g.cuda(), b.cuda(), row_idx=idx.int().cuda(), out=out)
    torch.cuda.synchronize()
    assert bool((out[R] == SENT).all())
    _ln_check("layernorm gather", out[:R].double(), x[idx].cuda(), g.cuda(), b.cuda(), kind[idx], f"index, {R} of {n}x{W}")


# ------------------------------------------------------------------------------------------------ class token + pos + ln_pre
EMB_CASES = [(L, B, W) for L, W in ((50, 768), (257, 1024), (17, 128)) for B in (1, 3, 70)]


def embed_inputs(L, B, W, seed):
    g = _gen(seed)
    x = torch.randn(B * L, W, generator=g)
    x[::L] = float("nan")                    # token 0 is the class token: its input rows must not be read
    cls = torch.randn(W, generator=g)
    pos = torch.randn(L, W, generator=g) + 20 * torch.randn(L, 1, generator=g)
    gamma = 1 + 0.5 * torch.randn(W, generator=g)
    beta = 0.1 * torch.randn(W, generator=g)
    return x, cls, pos, gamma, beta


@pytest.mark.gpu
@pytest.mark.parametrize("L,B,W", EMB_CASES)
def test_embed_ln_pre_matches_float64(L, B, W):
    """In place on the fp32 stream: token 0 := cls, + pos[t] (one fp32 add, so torch's add is the exact input), then
    LayerNorm, within D of float64; every image's token 0 is bit-identical."""
    x, cls, pos, g, b = embed_inputs(L, B, W, seed=L * B + W)
    buf = torch.full((B * L + 1, W), SENT, device="cuda")
    buf[:B * L] = x.cuda()
    ops.clip_embed_ln(buf[:B * L], cls.cuda(), pos.cuda(), g.cuda(), b.cuda(), L)
    torch.cuda.synchronize()
    assert bool((buf[B * L] == SENT).all())
    v = x.clone()
    v[::L] = cls
    v = (v.view(B, L, W) + pos).view(B * L, W)
    got = buf[:B * L].double()
    assert bool(torch.isfinite(got).all())
    y, delta = ln64(v.cuda(), g.cuda(), b.cuda())
    _ratio("embed + ln_pre", (got - y).abs(), delta, f"{B}x{L}x{W}")
    t0 = buf[:B * L].view(B, L, W)[:, 0]
    assert torch.equal(t0, t0[:1].expand(B, W)), "token 0 differs between images"


# ------------------------------------------------------------------------------------------------ patchify (bit-exact)
def patchify_ref(x, p, kpad):
    B, _, S, _ = x.shape
    G = S // p
    P = x.to(torch.bfloat16).view(B, 3, G, p, G, p).permute(0, 2, 4, 1, 3, 5).reshape(B * G * G, 3 * p * p)
    return F.pad(P, (0, kpad - 3 * p * p))


# (S, p, Kpad, B): K = 588 padded to 640 as the plans pad it, and to 592; B = 64 at p = 14 is 20480 B threads of work, past
# the 4224 x 256-thread grid
PATCH_CASES = [(224, 14, 640, 1), (224, 14, 640, 64), (224, 14, 592, 3), (224, 32, 3072, 2), (64, 16, 768, 5), (64, 16, 776, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("S,p,kpad,B", PATCH_CASES)
def test_patchify_bit_exact(S, p, kpad, B):
    """Row b*G^2 + gy*G + gx, column c p^2 + r p + s holds bf16_rn(x[b, c, gy p + r, gx p + s]); zeros in [3p^2, Kpad)."""
    x = torch.randn(B, 3, S, S, generator=_gen(S + p + kpad + B)) * 3
    rows = B * (S // p) ** 2
    out = torch.full((rows + 1, kpad), SENT, dtype=torch.bfloat16, device="cuda")
    ops.patchify(x.cuda(), p, kpad, out=out[:rows])
    torch.cuda.synchronize()
    assert bool((out[rows] == SENT).all())
    assert torch.equal(out[:rows].cpu().view(torch.int16), patchify_ref(x, p, kpad).view(torch.int16))


# ------------------------------------------------------------------------------------------------ text embedding (exact)
EOT = 49407


def text_ids(B, L, vocab, seed):
    """SOT, random tokens, EOT at position b % L, zeros after; then rows with two EOTs, without an EOT, and with ids -1,
    vocab and larger (clamped to the table, but they take part in the argmax as they are)."""
    g = _gen(seed)
    ids = torch.zeros(B, L, dtype=torch.int32)
    for r in range(B):
        e = r % L
        ids[r, :e] = torch.randint(1, 49405, (e,), generator=g, dtype=torch.int32)
        ids[r, 0] = 49406 if e > 0 else ids[r, 0]
        ids[r, e] = EOT
    if B >= 4:
        ids[B - 4, L - 1] = EOT                           # two EOTs: the first wins
        ids[B - 3] = torch.randint(0, 49405, (L,), generator=g, dtype=torch.int32)
        ids[B - 3, 5] = ids[B - 3, 9] = 49405             # no EOT: the first of two equal maxima
        ids[B - 2, :4] = torch.tensor([-1, vocab, 60000, EOT], dtype=torch.int32)
        ids[B - 1, 2] = -5
    return ids


TEXT_CASES = [(1, 77, 128), (100, 77, 768), (70, 77, 512), (7, 16, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,L,W", TEXT_CASES)
def test_text_embed_exact(B, L, W):
    """x = tok[clamp(id, 0, vocab - 1)] + pos[t] bit for bit, eot_row[b] = b L + the first argmax of the raw ids; B L = 7700
    and 5390 rows run past the 4224-row grid."""
    vocab = 49408
    g = _gen(B + L + W)
    tok = torch.randn(vocab, W, generator=g)
    pos = torch.randn(L, W, generator=g) * 0.1
    ids = text_ids(B, L, vocab, seed=B + W)
    x = torch.full((B * L + 1, W), SENT, device="cuda")
    eot = torch.full((B + 1,), -7, dtype=torch.int32, device="cuda")
    ops.text_embed(ids.cuda(), tok.cuda(), pos.cuda(), x=x[:B * L], eot_row=eot[:B])
    torch.cuda.synchronize()
    assert bool((x[B * L] == SENT).all()) and int(eot[B]) == -7
    want = (tok[ids.long().clamp(0, vocab - 1)] + pos).view(B * L, W)
    assert torch.equal(x[:B * L].cpu(), want)
    first = torch.from_numpy(np.argmax(ids.numpy(), axis=1)).int()
    assert torch.equal(eot[:B].cpu(), torch.arange(B, dtype=torch.int32) * L + first)
    if B >= 4:
        assert int(first[B - 4]) == (B - 4) % L < L - 1 and int(first[B - 3]) == 5 and int(first[B - 2]) == 2


# ------------------------------------------------------------------------------------------------ L2 norm
def l2_const(D):
    """Relative bar of the kernel: ceil(D/32) per-lane fused squares, a 5-level tree, IEEE sqrtf (halves the relative error),
    + eps, an IEEE divide and a multiply: (ceil(D/32) + 8) U."""
    return (math.ceil(D / 32) + 8) * U


def l2_inputs(R, D, seed):
    g = _gen(seed)
    x = torch.randn(R, D, generator=g, dtype=torch.float64)
    norms = torch.tensor([1e-6, 1.0, 1e6], dtype=torch.float64)[torch.arange(R) % 3]
    x = (x / x.norm(dim=1, keepdim=True) * norms[:, None]).float()
    zero = R // 2
    x[zero] = 0
    return x, zero


def l2_ref(x, eps):
    x64 = x.double()
    return x64 / (x64.norm(dim=1, keepdim=True) + eps)


L2_CASES = [(D, eps, R) for D in (64, 100, 512, 768, 1024) for eps in (0.0, 1e-8) for R in (5, GRID_ROWS, GRID_ROWS + 1)]
L2_CASES += [(768, 1e-8, 3 * GRID_ROWS + 7), (100, 0.0, 2 * GRID_ROWS + 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("D,eps,R", L2_CASES)
def test_l2norm_matches_float64(D, eps, R):
    """x / (||x|| + eps) within (ceil(D/32) + 8) 2^-24 relative of float64 on rows of norm 1e-6, 1 and 1e6, into rows
    out_stride = D + 12 apart (the gaps keep their sentinel); a zero row gives zeros at eps > 0 and NaN at eps = 0."""
    x, zero = l2_inputs(R, D, seed=D + R + int(eps > 0))
    stride = D + 12
    out = torch.full((R, stride), SENT, device="cuda")
    ops.l2norm(x.cuda(), eps, out=out, out_stride=stride)
    torch.cuda.synchronize()
    assert bool((out[:, D:] == SENT).all()), "the gaps between rows were written"
    got = out[:, :D].double()
    want = l2_ref(x.cuda(), eps)
    if eps > 0:
        assert bool((got[zero] == 0).all())
    else:
        assert bool(torch.isnan(got[zero]).all())
    keep = torch.ones(R, dtype=torch.bool, device="cuda")
    keep[zero] = False
    _ratio("l2norm", (got[keep] - want[keep]).abs(), l2_const(D) * want[keep].abs() + 1e-300, f"D {D} eps {eps} rows {R}")


# ------------------------------------------------------------------------------------------------ zero-block encoders
# width: (image, patch, embed_dim); towers of width W have W / 64 heads, an MLP of 4 W (unused) and no blocks
ZB_ARCHS = {128: (64, 16, 64), 768: (224, 32, 512), 1024: (224, 14, 768)}
ZB_VOCAB, ZB_CTX = 49408, 77
ZB_BATCHES = [1, 2, 5, 128, 129]
ZB_PAD = 24                  # out_row_stride = embed_dim + 24, the gaps keep their sentinel


def zb_geometry(W):
    S, p, D = ZB_ARCHS[W]
    G = S // p
    K = 3 * p * p
    return S, p, D, G * G, 1 + G * G, K, (K + 63) // 64 * 64


def zb_weights(W):
    """Host fp32 weights of a zero-block model.  The positional table carries a common offset 200x the spread, so ln_pre sees
    offset rows, and ln_pre's beta one of 300, so ln_post does too."""
    S, p, D, P, L, K, kpad = zb_geometry(W)
    g = _gen(W)
    return {
        "visual_conv1.weight": torch.randn(W, 3, p, p, generator=g) * K ** -0.5,
        "class_embedding": torch.randn(W, generator=g),
        "positional_embedding": torch.randn(L, W, generator=g) + 200,
        "ln_pre.weight": 1 + 0.3 * torch.randn(W, generator=g),
        "ln_pre.bias": 300 + 0.5 * torch.randn(W, generator=g),
        "ln_post.weight": 1 + 0.3 * torch.randn(W, generator=g),
        "ln_post.bias": 0.2 * torch.randn(W, generator=g),
        "proj": torch.randn(W, D, generator=g) * W ** -0.5,
        "token_embedding.weight": torch.randn(ZB_VOCAB, W, generator=g),
        "positional_embedding_text": 0.5 * torch.randn(ZB_CTX, W, generator=g),
        "ln_final.weight": 1 + 0.3 * torch.randn(W, generator=g),
        "ln_final.bias": 0.2 * torch.randn(W, generator=g),
        "text_projection": torch.randn(W, D, generator=g) * W ** -0.5,
    }


def zb_config(W, v_width=None, t_width=None):
    S, p, D = ZB_ARCHS.get(W, (224, 14, 768))
    vw, tw = v_width or W, t_width or W
    return _ClipConfig(S, p, vw, 0, vw // 64, 4 * vw, D, tw, 0, tw // 64, 4 * tw, ZB_VOCAB, ZB_CTX)


_ZB = {}


@pytest.fixture(scope="module")
def zb_models():
    yield _ZB
    for h, _ in _ZB.values():
        lib().cc_clip_destroy(h)
    _ZB.clear()


def zb_model(models, W):
    if W not in models:
        wts = zb_weights(W)
        arrs = [(k, np.ascontiguousarray(v.numpy())) for k, v in wts.items()]
        names = (ctypes.c_char_p * len(arrs))(*[k.encode() for k, _ in arrs])
        ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for _, a in arrs])
        nums = (ctypes.c_int64 * len(arrs))(*[a.size for _, a in arrs])
        h = ctypes.c_void_p()
        check(lib().cc_clip_create(ctypes.byref(zb_config(W)), len(arrs), names, ptrs, nums, ctypes.byref(h)), "cc_clip_create")
        models[W] = (h, wts)
    return models[W]


def _workspace(h, text, B):
    need = ctypes.c_size_t(0)
    check(lib().cc_clip_workspace_bytes(h, text, B, ctypes.byref(need)), "cc_clip_workspace_bytes")
    ws = torch.zeros(need.value, dtype=torch.uint8, device="cuda")
    check(lib().cc_clip_set_workspace(h, ctypes.c_void_p(ws.data_ptr()), need.value), "cc_clip_set_workspace")
    return ws


def _ws_view(ws, off, n, dtype):
    """n elements of dtype at byte `off` of the workspace; the plans carve it in 1024-byte-aligned pieces in build order."""
    size = torch.empty((), dtype=dtype).element_size()
    return ws[off:off + n * size].view(dtype)


def _align(n):
    return (n + 1023) // 1024 * 1024


def head_ref(x_row, g, b, proj, eps):
    """float64 of LayerNorm(x_row) -> bf16 -> @ bf16(proj) -> / (||.|| + eps), with the bar carried through: h within 2^-8 |h|
    + D (the bf16 store of h is the one rounding that cannot be reproduced), the projection GEMM within 2^-18 sum|h P|, and the
    normalisation: |e_hat/||e_hat|| - e/||e||| <= (be + |o| ||be||) / ||e||, plus the l2norm kernel's own relative bar."""
    h, dh = ln64(x_row, g, b)
    P = proj.to(torch.bfloat16).double().to(x_row.device)
    e = h @ P
    be = (2.0 ** -8 + 2.0 ** -17) * (h.abs() @ P.abs()) + 1.01 * (dh @ P.abs())
    nrm = e.norm(dim=1, keepdim=True) + eps
    o = e / nrm
    bar = 1.01 * (be + o.abs() * be.norm(dim=1, keepdim=True)) / nrm + l2_const(P.shape[1]) * o.abs()
    return o, bar


def _check_out(out, o, bar, D, what):
    assert bool((out[:, D:] == SENT).all()), "the gaps between output rows were written"
    _ratio("zero-block " + what, (out[:, :D].double() - o).abs(), bar)


ZB_CASES = [(W, B) for W in ZB_ARCHS for B in ZB_BATCHES]


@pytest.mark.gpu
@pytest.mark.parametrize("W,B", ZB_CASES)
def test_zero_block_image_encoder(zb_models, W, B):
    """patchify -> patch GEMM (K padded, rows at token 1 of each image, L rows apart) -> cls + pos + ln_pre -> ln_post of
    token 0 -> projection GEMM (M = B) -> l2norm (eps 1e-8).  The patch matrix and the stream after ln_pre are read from the
    caller-owned workspace, where the plan keeps them in its first two pieces."""
    S, p, D, P, L, K, kpad = zb_geometry(W)
    h, wts = zb_model(zb_models, W)
    x = torch.randn(B, 3, S, S, generator=_gen(W + B))
    ws = _workspace(h, 0, B)
    out = torch.full((B, D + ZB_PAD), SENT, device="cuda")
    try:
        xd = x.cuda()
        check(lib().cc_clip_encode_image(h, ctypes.c_void_p(xd.data_ptr()), B, ctypes.c_void_p(out.data_ptr()), D + ZB_PAD, None),
              "cc_clip_encode_image")
        torch.cuda.synchronize()
        patches = _ws_view(ws, 0, B * P * kpad, torch.bfloat16).view(B * P, kpad).clone()
        stream = _ws_view(ws, _align(B * P * kpad * 2), B * L * W, torch.float32).view(B, L, W).clone()
    finally:
        check(lib().cc_clip_set_workspace(h, None, 0), "cc_clip_set_workspace")
    dev = "cuda"
    assert torch.equal(patches.view(torch.int16), patchify_ref(xd, p, kpad).view(torch.int16)), "patch matrix"
    # the stream after ln_pre: token 0 from cls, tokens 1.. from the patch GEMM (fp32, within 2^-18 sum|x.w|) + pos
    Wp = wts["visual_conv1.weight"].reshape(W, K).to(torch.bfloat16).double().to(dev)
    A = patches[:, :K].double()
    emb = (A @ Wp.T).view(B, P, W)
    mag = (A.abs() @ Wp.abs().T).view(B, P, W)
    pos = wts["positional_embedding"].to(dev)
    v = torch.empty(B, L, W, dtype=torch.float64, device=dev)
    v[:, 0] = (wts["class_embedding"].to(dev) + pos[0]).double()
    v[:, 1:] = emb + pos[1:].double()
    E = torch.zeros(B, L, 1, dtype=torch.float64, device=dev)
    E[:, 1:] = (tc.F32_BAR * mag + U * v[:, 1:].abs()).amax(-1, keepdim=True)
    y, delta = ln64(v.view(B * L, W), wts["ln_pre.weight"].to(dev), wts["ln_pre.bias"].to(dev), E=E.view(B * L, 1))
    _ratio("zero-block ln_pre stream", (stream.view(B * L, W).double() - y).abs(), delta, f"W {W} B {B}")
    # ln_post reads token 0 of every image of that stream
    o, bar = head_ref(stream[:, 0], wts["ln_post.weight"].to(dev), wts["ln_post.bias"].to(dev), wts["proj"], 1e-8)
    _check_out(out, o, bar, D, "image")


@pytest.mark.gpu
@pytest.mark.parametrize("W,B", ZB_CASES)
def test_zero_block_text_encoder(zb_models, W, B):
    """tok + pos with the EOT argmax -> ln_final of the EOT row -> text projection (M = B) -> l2norm (eps 0).  The stream
    and the EOT rows are read from the caller-owned workspace (its first two pieces) and must be exact."""
    S, p, D, P, L, K, kpad = zb_geometry(W)
    h, wts = zb_model(zb_models, W)
    ids = text_ids(B, ZB_CTX, ZB_VOCAB, seed=W + B)
    ws = _workspace(h, 1, B)
    out = torch.full((B, D + ZB_PAD), SENT, device="cuda")
    try:
        idd = ids.cuda()
        check(lib().cc_clip_encode_text(h, ctypes.c_void_p(idd.data_ptr()), B, ctypes.c_void_p(out.data_ptr()), D + ZB_PAD, None),
              "cc_clip_encode_text")
        torch.cuda.synchronize()
        stream = _ws_view(ws, 0, B * ZB_CTX * W, torch.float32).view(B * ZB_CTX, W).clone()
        eot = _ws_view(ws, _align(B * ZB_CTX * W * 4), B, torch.int32).clone()
    finally:
        check(lib().cc_clip_set_workspace(h, None, 0), "cc_clip_set_workspace")
    dev = "cuda"
    want = (wts["token_embedding.weight"][ids.long().clamp(0, ZB_VOCAB - 1)] + wts["positional_embedding_text"]).view(-1, W)
    assert torch.equal(stream.cpu(), want)
    first = torch.from_numpy(np.argmax(ids.numpy(), axis=1)).int()
    assert torch.equal(eot.cpu(), torch.arange(B, dtype=torch.int32) * ZB_CTX + first)
    o, bar = head_ref(want[eot.cpu().long()].to(dev), wts["ln_final.weight"].to(dev), wts["ln_final.bias"].to(dev),
                      wts["text_projection"], 0.0)
    _check_out(out, o, bar, D, "text")


# ------------------------------------------------------------------------------------------------ CPU: bars and arguments
def _bf16(v):
    return v.float().to(torch.bfloat16).double()


def _act64(z, act):
    return F.silu(z) if act == 1 else F.gelu(z, approximate="tanh") if act == 2 else z


def test_bars_see_clip_bugs():
    """CPU only: on the GPU tests' own inputs, each typical bug leaves its bar, or the +-0.02 ulp rounding window, by at
    least 4x.  LayerNorm (every width, 4225 rows): a one-pass fp32 variance E[x^2] - E[x]^2 on the offset rows, eps 1e-6 on
    the rows of variance near 1e-5, gamma and beta swapped, a truncating bf16 store; a variance divided by W - 1 is checked at
    W = 128 only: it shrinks every value by 1/(2W), which at wider rows is less than 0.08 ulp of the store and so within 4x of
    the window.  l2norm without eps on the rows of norm 1e-6.  The conv GEMM (tests/test_conv_gpu.py's inputs): a truncating
    bf16 store on the activation-free cases with >= 10^4 outputs, and a residual added after a first bf16 rounding of
    act(z) on every bf16 residual case.  The zero-block image encoder with ln_post reading token 1 instead of token 0."""
    worst = {}

    def see(name, diff, bar):
        worst[name] = min(worst.get(name, math.inf), (diff.abs() / bar).max().item())

    def see_bias(name, got, y, noise):
        worst[name] = min(worst.get(name, math.inf), abs(tc.rn_bias(got, y, noise)[0]) / RN_WINDOW)

    # LayerNorm
    for W in LN_WIDTHS:
        R = GRID_ROWS + 1
        x, g, b, kind = ln_inputs(R, W, seed=R * 31 + W)
        y, delta = ln64(x, g, b)
        bar = ln_bar(y, delta)
        off, small, gauss = kind == 4, kind == 7, kind < 4
        see("layernorm: one-pass fp32 variance (offset rows)", ln64(x[off], g, b, one_pass=True)[0] - y[off], bar[off])
        see("layernorm: eps 1e-6 (variance near 1e-5)", ln64(x[small], g, b, eps=1e-6)[0] - y[small], bar[small])
        see("layernorm: gamma and beta swapped", ln64(x, b, g)[0] - y, bar)
        see_bias("layernorm: truncating bf16 store", tc.bf16_trunc(y[gauss]), y[gauss], delta[gauss])
    for R in (GRID_ROWS + 1, 3 * GRID_ROWS + 1):
        x, g, b, kind = ln_inputs(R, 128, seed=R * 31 + 128)
        gauss = kind < 4
        y, delta = ln64(x[gauss], g, b)
        see_bias("layernorm: variance over W - 1 (W = 128)", _bf16(ln64(x[gauss], g, b, ddof=1)[0]), y, delta)
    # l2norm
    for D, eps, R in L2_CASES:
        if eps == 0:
            continue
        x, zero = l2_inputs(R, D, seed=D + R + 1)
        tiny = (torch.arange(R) % 3 == 0) & (torch.arange(R) != zero)
        want = l2_ref(x[tiny], eps)
        see("l2norm without eps (norm 1e-6)", l2_ref(x[tiny], 0.0) - want, l2_const(D) * want.abs())
    # the conv GEMM's bf16 stores
    for case in tc.CASES:
        N, H, W, Cin, Cout, k, s, act, use_res, out_f32, in_cs, in_co = case[:12]
        groups = case[15] if len(case) > 15 else 1
        act0 = act == 0 and not use_res and N * H * W * Cout >= 10 ** 4
        if out_f32 or not (act0 or use_res):
            continue
        xbuf, w, b, res = tc.conv_inputs(case)
        z, y, mag = tc.ref64(xbuf[..., in_co:in_co + Cin].float(), w.float(), b, k, s, act, res, groups)
        if act0:
            see_bias("conv GEMM: truncating bf16 store (act 0)", tc.bf16_trunc(y), y, tc.F32_BAR * mag)
        else:
            see("conv GEMM: residual added after a bf16 rounding", _bf16(_bf16(_act64(z, act)) + res.double()) - y,
                tc.bf16_bar(z, y, mag, act))
    for p in tc.RESIDUAL_CASES:
        N, H, W, Cin, Cout, k, act, out_f32, bn, out_cs = p.values
        if out_f32:
            continue
        x, w, b, obuf = tc.residual_inputs(N, H, W, Cin, Cout, k, out_f32, out_cs)
        res = obuf[..., out_cs - Cout:].float()
        z, y, mag = tc.ref64(x.float(), w.float(), b, k, 1, act, res)
        see("conv GEMM: residual added after a bf16 rounding", _bf16(_bf16(_act64(z, act)) + res.double()) - y,
            tc.bf16_bar(z, y, mag, act))
    # the zero-block image encoder: ln_post at token 1 (the first patch row) instead of token 0
    for W in ZB_ARCHS:
        S, p, D, P, L, K, kpad = zb_geometry(W)
        wts = zb_weights(W)
        B = 2
        x = torch.randn(B, 3, S, S, generator=_gen(W + B))
        Wp = wts["visual_conv1.weight"].reshape(W, K).to(torch.bfloat16).double()
        emb0 = patchify_ref(x, p, kpad)[:, :K].double().view(B, P, K)[:, 0] @ Wp.T
        pos = wts["positional_embedding"]
        rows = {0: (wts["class_embedding"] + pos[0]).double().expand(B, W), 1: emb0 + pos[1].double()}
        o = {}
        for t, v in rows.items():
            xt = ln64(v, wts["ln_pre.weight"], wts["ln_pre.bias"])[0]
            o[t] = head_ref(xt, wts["ln_post.weight"], wts["ln_post.bias"], wts["proj"], 1e-8)
        see("zero-block image: ln_post reads token 1", o[1][0] - o[0][0], o[0][1])
    for name, r in sorted(worst.items()):
        print(f"{name}: {r:.1f}x the bar")
    for name, r in worst.items():
        assert r >= 4.0, f"'{name}' moves the result by only {r:.2f}x the bar"


def test_clip_taps_reject_bad_arguments():
    """Every check of the CLIP taps, and cc_clip_create's configuration checks, run before anything is launched or any
    device is asked for (no GPU needed): the pointers below are never dereferenced."""
    h = lib()
    fake = ctypes.c_void_p(1 << 20)
    odd = ctypes.c_void_p((1 << 20) + 8)
    odd4 = ctypes.c_void_p((1 << 20) + 4)

    def refused(rc, *words):
        msg = h.cc_last_error().decode()
        assert rc == -1 and all(w_ in msg for w_ in words), (rc, msg, words)

    # cc_patchify(x, B, S, p, Kpad, out, stream)
    pf = lambda x=fake, B=2, S=224, p=14, kpad=640, out=fake: h.cc_patchify(x, B, S, p, kpad, out, None)
    refused(pf(x=None), "cc_patchify", "NULL")
    refused(pf(out=None), "cc_patchify", "NULL")
    refused(pf(out=odd), "cc_patchify", "16-byte aligned")
    refused(pf(S=225), "cc_patchify", "not a multiple of the patch")
    refused(pf(kpad=644), "cc_patchify", "Kpad=644")
    refused(pf(kpad=584), "cc_patchify", "Kpad=584", "588")
    refused(pf(B=-1), "cc_patchify", "bad shape")
    refused(pf(p=0), "cc_patchify", "bad shape")
    # cc_clip_embed_ln(x, cls, pos, gamma, beta, B, L, W, stream)
    el = lambda x=fake, c=fake, pos=fake, g=fake, b=fake, B=2, L=50, W=768: h.cc_clip_embed_ln(x, c, pos, g, b, B, L, W, None)
    for arg in ("x", "c", "pos", "g", "b"):
        refused(el(**{arg: None}), "cc_clip_embed_ln", "NULL")
        refused(el(**{arg: odd}), "cc_clip_embed_ln", "16-byte aligned")
    for W in (896, 1408, 1664, 2048, 100, 0, -128):
        refused(el(W=W), "cc_clip_embed_ln", f"width {W} not supported")
    refused(el(B=-1), "cc_clip_embed_ln", "bad shape")
    refused(el(L=0), "cc_clip_embed_ln", "bad shape")
    refused(el(B=1 << 26, L=257), "cc_clip_embed_ln", "bad shape")
    # cc_layernorm_bf16(x, rows, W, row_stride, row_idx, gamma, beta, out, stream)
    ln = lambda x=fake, rows=4, W=768, stride=1, idx=None, g=fake, b=fake, out=fake: h.cc_layernorm_bf16(x, rows, W, stride, idx, g,
                                                                                                     b, out, None)
    for arg in ("x", "g", "b", "out"):
        refused(ln(**{arg: None}), "cc_layernorm_bf16", "NULL")
    for arg in ("x", "g", "b"):
        refused(ln(**{arg: odd}), "cc_layernorm_bf16", "16-byte aligned")
    refused(ln(out=odd4), "cc_layernorm_bf16", "d_out must be 8-byte aligned")
    for W in (896, 1408, 1792, 64, 0):
        refused(ln(W=W), "cc_layernorm_bf16", f"width {W} not supported")
    refused(ln(rows=-1), "cc_layernorm_bf16", "bad shape")
    refused(ln(stride=-1), "cc_layernorm_bf16", "bad shape")
    # cc_text_embed(ids, tok, pos, B, L, W, vocab, x, eot_row, stream)
    te = lambda ids=fake, tok=fake, pos=fake, B=2, L=77, W=512, vocab=49408, x=fake, eot=fake: h.cc_text_embed(
        ids, tok, pos, B, L, W, vocab, x, eot, None)
    for arg in ("ids", "tok", "pos", "x", "eot"):
        refused(te(**{arg: None}), "cc_text_embed", "NULL")
    for arg in ("tok", "pos", "x"):
        refused(te(**{arg: odd}), "cc_text_embed", "16-byte aligned")
    refused(te(W=510), "cc_text_embed", "bad shape")
    refused(te(vocab=0), "cc_text_embed", "bad shape")
    refused(te(B=-1), "cc_text_embed", "bad shape")
    refused(te(L=0), "cc_text_embed", "bad shape")
    refused(te(B=1 << 25), "cc_text_embed", "bad shape")
    # cc_l2norm(in, rows, D, eps, out, out_stride, stream)
    l2 = lambda i=fake, rows=4, D=512, eps=1e-8, o=fake, stride=512: h.cc_l2norm(i, rows, D, eps, o, stride, None)
    refused(l2(i=None), "cc_l2norm", "NULL")
    refused(l2(o=None), "cc_l2norm", "NULL")
    refused(l2(stride=511), "cc_l2norm", "out_stride 511")
    refused(l2(rows=-1), "cc_l2norm", "bad shape")
    refused(l2(D=0, stride=0), "cc_l2norm", "bad shape")
    refused(l2(eps=-1.0), "cc_l2norm", "eps")
    # cc_clip_create: widths the LayerNorm kernels lack are refused at create, before the device check
    out = ctypes.c_void_p()
    for vw, tw in ((896, 512), (768, 1408), (1664, 768)):
        refused(h.cc_clip_create(ctypes.byref(zb_config(768, v_width=vw, t_width=tw)), 0, None, None, None, ctypes.byref(out)),
                "cc_clip_create", f"widths {vw} / {tw} not supported")
    bad = zb_config(768)
    bad.patch = 0
    refused(h.cc_clip_create(ctypes.byref(bad), 0, None, None, None, ctypes.byref(out)), "cc_clip_create", "unsupported architecture")
    bad = zb_config(768)
    bad.t_heads = 8
    refused(h.cc_clip_create(ctypes.byref(bad), 0, None, None, None, ctypes.byref(out)), "cc_clip_create", "unsupported architecture")
    assert not out.value
