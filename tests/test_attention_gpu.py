"""Both CLIP attention kernels against a float64 reference of the attention itself, called through cc_attention:

* impl 1, `attention_kernel<CAUSAL>` (vit.cu): mma.sync, 16-query x 16-key blocks, a second CTA per (image, head) when
  ceil(L/16) > 10, sequences up to 704 tokens;
* impl 2, `attention_tc_kernel` (attention_tc.cu): wgmma, 64-query x 64-key blocks, sequences up to 384 tokens.

The reference is float64 softmax(q k^T / 8 [+ causal mask]) v of the same bf16 qkv the kernel reads.  Bar, per element:

    |got - ref| <= A_REF * |ref| + B_V * max_j |v_j|       (max over the keys of that image, head and d)

Rounding the output to bf16 costs up to 2^-8 |ref|; rounding P to bf16 before P.V costs up to 2^-8 max |v|.  At
A_REF = B_V = 2^-8 both kernels reached 0.59 of the bar on an H100 (the output rounding alone reaches 0.5 where |ref| is
the column's max |v|), so the bar is 2^-7, for at least 2x margin.  Each test prints its worst error/bar.
`test_bars_see_attention_bugs` proves on the CPU that the bars, on the inputs the GPU tests use, are exceeded at least 4x
by the typical attention bugs: a key dropped at the end, a causal mask off by one, a wrong scale in one head, a query
block never written.
"""
import ctypes

import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200._lib import lib

A_REF = 2.0 ** -7
B_V = 2.0 ** -7
MAX_LEN = {1: 704, 2: 384}
IMPL_NAME = {1: "mma.sync", 2: "wgmma"}
SENTINEL = -7.0

# sequence lengths at and around every 16- and 64-row block edge; 160/161 is where the mma.sync kernel splits a head
# over two CTAs; 384 is the wgmma kernel's limit, 704 the mma.sync kernel's
LS = [1, 2, 15, 16, 17, 33, 50, 63, 64, 65, 77, 127, 128, 129, 160, 161, 192, 193, 256, 257, 320, 383, 384]
LS_MMA_ONLY = [385, 448, 449, 511, 512, 640, 704]
HEADS = [1, 2, 8, 12, 16]

KINDS = ["gaussian", "dominant-first", "dominant-last", "late-max", "large-logits", "large-negative-logits", "v-offset",
         "identical-keys"]
# (name, L, H, causal): the production shapes (ViT-B/32 and ViT-L/14 image and text towers, the tiny test config) and
# block edges: key L-1 alone in its last 16-key block (65, 161, 257) and last 64-key block (65, 257), the kernels' limits
CLASSES = [("image-B32", 50, 12, 0), ("image-L14", 257, 16, 0), ("text-B32", 77, 8, 1), ("text-L14", 77, 12, 1),
           ("tiny-image", 17, 2, 0), ("tiny-text", 77, 2, 1), ("edge-65", 65, 4, 0), ("edge-161-causal", 161, 2, 1),
           ("edge-384", 384, 2, 0), ("edge-384-causal", 384, 2, 1), ("edge-704", 704, 1, 0)]
CLASS_B = 2

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(_WORST):
        print(f"\nworst |err|/bar, {key[0]} kernel, {key[1]}: {_WORST[key]:.3f}")


def make_qkv(kind, B, L, H, seed):
    """bf16 [B*L, 3*H*64] on the CPU.  q, k ~ N(0, 1.6^2) give logits q.k/8 of std ~2.5; channel 0 of q is set to 8 where
    a kind steers the logits, so k[..., 0] adds exactly k[..., 0] to every row's logit of that key."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, L, H, 64, generator=g) * 1.6
    k = torch.randn(B, L, H, 64, generator=g) * 1.6
    v = torch.randn(B, L, H, 64, generator=g)
    if kind in ("dominant-first", "dominant-last", "late-max", "large-logits", "large-negative-logits"):
        q[..., 0] = 8.0
        k[..., 0] = 0.0
    if kind == "dominant-first":
        k[:, 0, :, 0] = 30.0
    elif kind == "dominant-last":
        k[:, L - 1, :, 0] = 30.0
    elif kind == "late-max":          # the row maximum first appears in the last 16-key block: the online softmax rescales
        k[:, (L - 1) // 16 * 16:, :, 0] = 20.0
    elif kind in ("large-logits", "large-negative-logits"):
        sign = 1.0 if kind == "large-logits" else -1.0
        k[..., 0] = sign * (60.0 + 20.0 * torch.rand(B, L, H, generator=g))
    elif kind == "v-offset":
        v = 50.0 + 0.1 * v
    elif kind == "identical-keys":    # every logit of a row equal: the result is the plain mean of the visible v
        k[:] = k[:, :1]
    return torch.stack([q, k, v], 2).reshape(B * L, 3 * H * 64).to(torch.bfloat16)


def reference(qkv, B, L, H, causal, head0_scale=1.0, drop_last=False, causal_shift=0):
    """float64 attention, [B, H, L, 64].  The keyword arguments apply the bugs the bars must see."""
    x = qkv.to(torch.float64).view(B, L, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    s = q @ k.transpose(-1, -2) / 8.0
    s[:, 0] *= head0_scale
    key = torch.arange(L, device=qkv.device)
    masked = torch.zeros(L, L, dtype=torch.bool, device=qkv.device)
    if causal:
        masked |= key[None, :] > key[:, None] + causal_shift
    if drop_last:
        masked[:, L - 1] = True
    return s.masked_fill(masked, float("-inf")).softmax(-1) @ v


def bar(qkv, B, L, H, ref):
    vmax = qkv.to(torch.float64).view(B, L, 3, H, 64)[:, :, 2].abs().amax(1)        # [B, H, 64]
    return A_REF * ref.abs() + B_V * vmax[:, :, None, :]


def as_bhld(ctx, B, L, H):
    return ctx.view(B, L, H, 64).permute(0, 2, 1, 3)


def run(qkv, L, H, causal, impl):
    """One cc_attention call into a ctx buffer with 5 sentinel rows after B*L, which must stay untouched."""
    rows = qkv.shape[0]
    ctx = torch.full((rows + 5, H * 64), SENTINEL, dtype=torch.bfloat16, device="cuda")
    ops.attention(qkv, L, H, causal, impl, ctx=ctx)
    torch.cuda.synchronize()
    assert torch.equal(ctx[rows:], torch.full_like(ctx[rows:], SENTINEL)), "rows after B*L were written"
    return ctx[:rows]


def check(got, qkv, B, L, H, causal, impl, group):
    assert torch.isfinite(got.float()).all()
    ref = reference(qkv, B, L, H, causal)
    b = bar(qkv, B, L, H, ref)
    err = (as_bhld(got, B, L, H).double() - ref).abs()
    ratio = (err / b).max().item()
    key = (IMPL_NAME[impl], group)
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)
    worst = torch.nonzero(err / b == (err / b).max())[0].tolist()
    assert ratio <= 1.0, f"worst |err|/bar {ratio:.3f} at (image, head, row, d) = {worst}"
    return ratio


SWEEP = [(impl, L) for impl in (1, 2) for L in LS] + [(1, L) for L in LS_MMA_ONLY]


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [0, 1], ids=["full", "causal"])
@pytest.mark.parametrize("impl,L", SWEEP, ids=[f"{IMPL_NAME[i]}-L{L}" for i, L in SWEEP])
def test_attention_matches_float64_at_every_tile_edge(impl, L, causal):
    """Gaussian logits at every head count, three images per call.  Each image equals, bit for bit, the same image run
    alone (the wgmma kernel's TMA boxes read the next image's rows past L; only the key < L mask keeps them out), and two
    identical calls give identical outputs."""
    B = 3
    for H in HEADS:
        qkv = make_qkv("gaussian", B, L, H, seed=1000 * L + H).cuda()
        got = run(qkv, L, H, causal, impl)
        r = check(got, qkv, B, L, H, causal, impl, "tile-edge sweep")
        print(f"{IMPL_NAME[impl]} L={L} H={H} causal={causal}: worst |err|/bar {r:.3f}")
        assert torch.equal(run(qkv, L, H, causal, impl), got), "two identical calls differ"
        for b in range(B):
            alone = run(qkv[b * L:(b + 1) * L].contiguous(), L, H, causal, impl)
            assert torch.equal(alone, got[b * L:(b + 1) * L]), f"image {b} differs from the same image run alone (H={H})"


INPUT_CASES = [(impl, c, kind) for c in CLASSES for impl in (1, 2) if c[1] <= MAX_LEN[impl] for kind in KINDS]


@pytest.mark.gpu
@pytest.mark.parametrize("impl,cls,kind", INPUT_CASES, ids=[f"{IMPL_NAME[i]}-{c[0]}-{k}" for i, c, k in INPUT_CASES])
def test_attention_inputs_that_stress_the_softmax(impl, cls, kind):
    """One dominant key (first, last, alone in the last key block), a row maximum that first appears in a late key block,
    logits of magnitude 60-80 of either sign, V with a large common offset, identical keys."""
    name, L, H, causal = cls
    qkv = make_qkv(kind, CLASS_B, L, H, seed=_class_seed(cls, kind)).cuda()
    got = run(qkv, L, H, causal, impl)
    r = check(got, qkv, CLASS_B, L, H, causal, impl, "inputs and production shapes")
    print(f"{IMPL_NAME[impl]} {name} {kind}: worst |err|/bar {r:.3f}")


def _class_seed(cls, kind):
    return 7 + 1000 * cls[1] + 10 * cls[2] + KINDS.index(kind)


def test_bars_see_attention_bugs():
    """CPU only: on the inputs of test_attention_inputs_that_stress_the_softmax, each mutated attention leaves the bar
    by at least 4x on some element of every shape class: the last valid key dropped, the causal mask shifted by one, one
    head's scale x1.1, the last 16-row and the last 64-row query block never written."""
    mutations = {
        "last key dropped": dict(drop_last=True),
        "causal mask shifted by one": dict(causal_shift=1),
        "head 0 scale x1.1": dict(head0_scale=1.1),
    }
    for cls in CLASSES:
        name, L, H, causal = cls
        best = {m: 0.0 for m in list(mutations) + ["16-row block zeroed", "64-row block zeroed"]}
        if not causal:
            del best["causal mask shifted by one"]
        for kind in KINDS:
            qkv = make_qkv(kind, CLASS_B, L, H, seed=_class_seed(cls, kind))
            ref = reference(qkv, CLASS_B, L, H, causal)
            b = bar(qkv, CLASS_B, L, H, ref)
            for m in best:
                if m in mutations:
                    mut = reference(qkv, CLASS_B, L, H, causal, **mutations[m])
                else:
                    mut = ref.clone()
                    rows = 16 if m.startswith("16") else 64
                    mut[:, :, (L - 1) // rows * rows:] = 0.0
                best[m] = max(best[m], ((mut - ref).abs() / b).max().item())
        print(name, {m: round(r, 1) for m, r in best.items()})
        for m, r in best.items():
            assert r >= 4.0, f"{name}: '{m}' moves the result by only {r:.2f}x the bar"


def test_cc_attention_rejects_bad_arguments():
    """Every check runs before anything is launched (no GPU needed): the pointers below are never dereferenced."""
    h = lib()
    fake = ctypes.c_void_p(1 << 20)
    need = ctypes.c_size_t(12345)

    def call(B, L, H, impl, ws=None, ws_bytes=0, ctx=fake, qkv=fake):
        return h.cc_attention(qkv, B, L, H, 0, impl, ws, ws_bytes, ctx, ctypes.byref(need), None)

    # the workspace query: the V^T copy of the wgmma kernel, keys padded to a multiple of 64; none for mma.sync
    assert call(3, 257, 16, 2, ctx=None) == 0 and need.value == 3 * 16 * 64 * 320 * 2
    assert call(3, 257, 16, 1, ctx=None) == 0 and need.value == 0
    assert call(0, 77, 8, 2, ctx=None) == 0 and need.value == 0
    bad = [
        (dict(B=1, L=50, H=12, impl=0), "unknown impl"),
        (dict(B=1, L=50, H=12, impl=3), "unknown impl"),
        (dict(B=1, L=50, H=12, impl=-1), "unknown impl"),
        (dict(B=1, L=0, H=12, impl=1), "bad shape"),
        (dict(B=1, L=-5, H=12, impl=2), "bad shape"),
        (dict(B=1, L=50, H=0, impl=2), "bad shape"),
        (dict(B=-1, L=50, H=12, impl=1), "bad shape"),
        (dict(B=1, L=385, H=2, impl=2), "too long"),
        (dict(B=1, L=705, H=2, impl=1), "too long"),
        (dict(B=4096, L=257, H=16, impl=2), "exceed the grid"),
    ]
    for kw, words in bad:
        for ctx in (fake, None):                                  # refused by the size query too
            rc = call(ctx=ctx, **kw)
            msg = h.cc_last_error().decode()
            assert rc == -1 and words in msg and "cc_attention" in msg, (kw, rc, msg)
    need_257 = 3 * 16 * 64 * 320 * 2
    for kw in (dict(ws=fake, ws_bytes=need_257 - 1), dict(ws=None, ws_bytes=need_257)):
        rc = call(3, 257, 16, 2, **kw)
        msg = h.cc_last_error().decode()
        assert rc == -1 and "workspace" in msg and "too small" in msg, (kw, rc, msg)
    rc = call(3, 257, 16, 2, ws=fake, ws_bytes=need_257, qkv=ctypes.c_void_p((1 << 20) + 2))
    assert rc == -1 and "16-byte aligned" in h.cc_last_error().decode()
    rc = call(3, 257, 16, 2, ws=fake, ws_bytes=need_257, qkv=None)
    assert rc == -1 and "NULL" in h.cc_last_error().decode()
