"""The per-op checks of tests/test_plan_ops_gpu.py see the launches they are there to catch (no GPU needed).

CPU tensors in a small workspace laid out as a plan lays it out, over a batch of B = 7 images that are copies of 3 distinct
ones: an upsample between channel slices of wider buffers, a CBFuse, the three LayerNorm forms (every row, token 0 of each
image, the EOT rows), attention, an L2 norm into rows of a wider output, the postprocess and the decode.  The exact result of
each (the reference, stored as the kernel stores it) passes check_one; each corruption below is flagged by the check named
with it."""
import types

import pytest
import torch

import test_attention_gpu as ta
import test_clip_ops_gpu as tco
import test_detector_ops_gpu as td
import test_plan_ops_gpu as tpo
from oracle import yolov9 as o

B = 7
REPS = tpo.REPS
BF16, F32 = torch.bfloat16, torch.float32


class _Layout:
    """Buffers back to back in one uint8 workspace, 256-byte aligned."""

    def __init__(self):
        self.off, self.g = 0, torch.Generator().manual_seed(13)

    def add(self, N, H, W, cs, dtype, co=0, C=None, ns=0):
        self.off = (self.off + 255) // 256 * 256
        op = tpo.Opnd("ws", self.off, cs, co, cs if C is None else C, N, H, W, dtype, ns)
        self.off += N * (ns or H * W) * cs * dtype.itemsize
        return op

    def workspace(self):
        return torch.zeros((self.off + 255) // 256 * 256, dtype=torch.uint8)

    def fill(self, ws, op, scale=1.0, values=None):
        """REPS distinct images (or `values`, [REPS, H, W, C]) copied over the batch of op."""
        v = values if values is not None else torch.randn((REPS, op.H, op.W, op.C), generator=self.g) * scale
        tpo.oview(ws, op).copy_(v[torch.arange(op.N) % REPS].to(op.dtype))


def _tile(v, n=B):
    return v[torch.arange(n) % v.shape[0]]


def _io(**kw):
    base = dict(causal=0, eps=0.0, conf_thr=0.25, max_det=0, iou_thr=0.45, do_scale=0, act=0, patch=0)
    base.update(kw)
    return types.SimpleNamespace(**base)


def _ctx(**kw):
    c = {"B": B, "L": 0, "input": None, "ids": None, "pitch": {},
         "call_of": lambda kind: "detections" if kind == "postprocess" else "head tap" if kind == "decode" else "embeddings"}
    c.update(kw)
    return c


class Case:
    """One op on the workspace: `exact()` gives (after, call) with the reference written; `check` runs check_one."""

    def __init__(self, kind, ins, outs, io, ctx, ws, write, call=None):
        self.op = tpo.Op(io, kind, kind, ins, outs)
        self.ctx, self.snap, self.write, self.call0 = ctx, ws, write, call or {}

    def exact(self):
        after = self.snap.clone()
        call = {k: v.clone() for k, v in self.call0.items()}
        self.write(after, call)
        return after, call

    def check(self, after, call):
        tpo.check_one(self.op, self.snap, after, self.call0, call, self.ctx, {})


# ------------------------------------------------------------------------------------------------ the cases
def upsample_case():
    lay = _Layout()
    x = lay.add(B, 4, 6, 32, BF16, co=8, C=16)
    y = lay.add(B, 8, 12, 32, BF16, co=8, C=16)
    ws = lay.workspace()
    lay.fill(ws, x._replace(co=0, C=32), 3.0)

    def write(after, call):
        tpo.oview(after, y).copy_(td.ref_pool("upsample2", tpo.oview(after, x).float(), BF16).to(BF16))
    return Case("upsample2", [x], [y], _io(), _ctx(), ws, write)


def cbfuse_case(shift=0):
    lay = _Layout()
    srcs = [lay.add(B, 2, 3, 24, BF16, co=8, C=16), lay.add(B, 4, 6, 16, BF16)]
    last = lay.add(B, 8, 12, 16, BF16)
    out = lay.add(B, 8, 12, 32, BF16, co=16, C=16)
    ws = lay.workspace()
    for s in srcs + [last]:
        lay.fill(ws, s)
    return Case("cbfuse", srcs + [last], [out], _io(), _ctx(), ws,
                lambda after, call: tpo.oview(after, out).copy_(td.ref_cbfuse([tpo.oview(after, s).float() for s in srcs],
                                                                               tpo.oview(after, last).float(), BF16).to(BF16)))


LN_W = 128


def _ln_tables(ws, g, b, gen):
    tpo.oview(ws, g).copy_(1 + 0.5 * torch.randn(1, 1, 1, LN_W, generator=gen))
    tpo.oview(ws, b).copy_(0.1 * torch.randn(1, 1, 1, LN_W, generator=gen))


def _ln_store(rows, g, b, ws, ddof=0):
    return tco.ln64(rows, tpo.oview(ws, g).flatten(), tpo.oview(ws, b).flatten(), ddof=ddof)[0].float().to(BF16)


def layernorm_dense_case(L=512):
    """ln_1 / ln_2: every row of a [B, L, W] stream (L = 512: enough outputs for the rounding-bias check)."""
    lay = _Layout()
    x = lay.add(B, 1, L, LN_W, F32)
    y = lay.add(B, 1, L, LN_W, BF16)
    g, b = lay.add(1, 1, 1, LN_W, F32), lay.add(1, 1, 1, LN_W, F32)
    ws = lay.workspace()
    _ln_tables(ws, g, b, lay.g)
    lay.fill(ws, x, 2.0)
    case = Case("layernorm", [x, g, b], [y], _io(), _ctx(), ws, None)
    case.write = lambda after, call, ddof=0: tpo.oview(after, y).copy_(
        _ln_store(tpo.oview(after, x).reshape(-1, LN_W), g, b, after, ddof).view(B, 1, L, LN_W))
    return case


def layernorm_token0_case(L=5):
    """ln_post: token 0 of each image, rows L apart"""
    lay = _Layout()
    stream = lay.add(B, 1, L, LN_W, F32)
    y = lay.add(B, 1, 1, LN_W, BF16)
    g, b = lay.add(1, 1, 1, LN_W, F32), lay.add(1, 1, 1, LN_W, F32)
    ws = lay.workspace()
    _ln_tables(ws, g, b, lay.g)
    lay.fill(ws, stream, 2.0)
    x = stream._replace(W=1, ns=L)
    case = Case("layernorm", [x, g, b], [y], _io(), _ctx(), ws, None)
    case.write = lambda after, call, tok=0: tpo.oview(after, y).copy_(
        _ln_store(tpo.oview(after, stream)[:, 0, tok], g, b, after).view(B, 1, 1, LN_W))
    return case


def layernorm_eot_case(L=9):
    """ln_final: the EOT rows the token ids place"""
    lay = _Layout()
    stream = lay.add(B, 1, L, LN_W, F32)
    eot = lay.add(B, 1, 1, 1, torch.int32)
    y = lay.add(B, 1, 1, LN_W, BF16)
    g, b = lay.add(1, 1, 1, LN_W, F32), lay.add(1, 1, 1, LN_W, F32)
    ws = lay.workspace()
    _ln_tables(ws, g, b, lay.g)
    lay.fill(ws, stream, 2.0)
    ids = torch.zeros(REPS, L, dtype=torch.int32)
    for r, e in enumerate((2, 5, 8)):
        ids[r, :e] = torch.randint(1, 49000, (e,), generator=lay.g, dtype=torch.int32)
        ids[r, e] = 49407
    ids = _tile(ids)
    rows = tpo._eot(ids)
    tpo.oview(ws, eot).copy_(rows.view(B, 1, 1, 1))
    case = Case("layernorm", [stream, g, b, eot], [y], _io(), _ctx(ids=ids, L=L), ws, None)
    case.write = lambda after, call, d=0: tpo.oview(after, y).copy_(
        _ln_store(tpo.oview(after, stream).reshape(-1, LN_W)[rows.long() + d], g, b, after).view(B, 1, 1, LN_W))
    return case


def attention_case(causal, L=17, H=2):
    lay = _Layout()
    qkv = lay.add(B, 1, L, 3 * H * 64, BF16)
    ctx = lay.add(B, 1, L, H * 64, BF16)
    ws = lay.workspace()
    lay.fill(ws, qkv, 1.5)

    def write(after, call, **bug):
        q = tpo.oview(after, qkv).reshape(B * L, 3 * H * 64)
        ref = ta.reference(q, B, L, H, bug.pop("causal", causal), **bug)
        tpo.oview(after, ctx).copy_(ref.permute(0, 2, 1, 3).reshape(B, 1, L, H * 64).to(BF16))
    return Case("attention", [qkv], [ctx], _io(causal=causal), _ctx(), ws, write)


def l2norm_case(D=64, pad=8):
    """emb rows of norm 1e-6 (where eps matters) into call rows D + pad floats apart"""
    lay = _Layout()
    emb = lay.add(B, 1, 1, D, F32)
    ws = lay.workspace()
    v = torch.randn(REPS, 1, 1, D, generator=lay.g, dtype=torch.float64)
    lay.fill(ws, emb, values=(v / v.norm(dim=-1, keepdim=True) * 1e-6).float())
    out = torch.full((B, D + pad), float("nan"))
    eps = torch.tensor(1e-8, dtype=F32).item()
    call = {"embeddings": tpo._bytes(out)}

    def write(after, call, e=eps):
        rows = call["embeddings"].view(F32).view(B, D + pad)
        rows[:, :D] = tco.l2_ref(tpo.oview(after, emb).reshape(B, D), e).float()
    return Case("l2norm", [emb], [tpo.Opnd("call", 0, D + pad, 0, D, B, 1, 1, F32)], _io(eps=eps), _ctx(pitch={"embeddings": D + pad}),
                ws, write, call)


def postprocess_case(A=64, max_det=20):
    """pred rows with tied confidences (different classes, so both are kept)"""
    lay = _Layout()
    pred = lay.add(B, 1, A, 6, F32)
    ws = lay.workspace()
    g = lay.g
    xy = torch.rand(REPS, A, 2, generator=g) * 300
    wh = torch.rand(REPS, A, 2, generator=g) * 60 + 5
    conf = (torch.rand(REPS, A, generator=g) * 0.7 + 0.26) * (torch.rand(REPS, A, generator=g) < 0.5)
    conf[:, 3] = conf[:, 7] = 0.9
    cls = torch.randint(0, 5, (REPS, A), generator=g).float()
    cls[:, 3], cls[:, 7] = 1, 2
    lay.fill(ws, pred, values=torch.cat([xy, xy + wh, conf[..., None], cls[..., None]], -1).view(REPS, 1, A, 6))
    out = torch.full((B, max_det * 6), float("nan"))
    call = {"detections": tpo._bytes(out)}

    def write(after, call):
        call["detections"].view(F32).view(B, max_det, 6).copy_(o.postprocess_boxes(tpo.oview(after, pred).reshape(B, A, 6), max_det, 0.45))
    return Case("postprocess", [pred], [tpo.Opnd("call", 0, 6, 0, 6, B, 1, max_det, F32)], _io(max_det=max_det), _ctx(), ws, write,
                call)


def decode_case(hw=((4, 4), (2, 2), (1, 1))):
    """the head's fp32 maps, with two equal class logits at every anchor of the first level (first-max-wins matters there)"""
    lay = _Layout()
    box = [lay.add(B, h, w, 64, F32) for h, w in hw]
    cls = [lay.add(B, h, w, 80, F32) for h, w in hw]
    A = sum(h * w for h, w in hw)
    pred = lay.add(B, 1, A, 6, F32)
    ws = lay.workspace()
    for t in box:
        lay.fill(ws, t, 2.0)
    for t in cls:
        lay.fill(ws, t, 2.0)
    c0 = tpo.oview(ws, cls[0])
    c0[..., 7] = c0[..., 3] = 4.0
    raw = torch.full((B, 84 * A), float("nan"))
    call = {"head tap": tpo._bytes(raw)}

    def write(after, call, last_max=False):
        n = REPS          # the reference of the distinct images, copied over the batch
        bx = torch.cat([tpo.oview(after, t)[:n].reshape(n, -1, 64) for t in box], 1).permute(0, 2, 1)
        cl = torch.cat([tpo.oview(after, t)[:n].reshape(n, -1, 80) for t in cls], 1).permute(0, 2, 1)
        dist = (bx.reshape(n, 4, 16, A).softmax(2) * torch.arange(16.0).reshape(1, 1, 16, 1)).sum(2)
        anchors, strides = o.make_anchors(list(hw))
        lt, rb = dist.chunk(2, 1)
        x1y1, x2y2 = anchors.unsqueeze(0) - lt, anchors.unsqueeze(0) + rb
        r = torch.cat([torch.cat([(x1y1 + x2y2) / 2, x2y2 - x1y1], 1) * strides, torch.sigmoid(cl)], 1)
        call["head tap"].view(F32).view(B, 84, A).copy_(_tile(r))
        probs = r[:, 4:].max(1)[0]
        ids = r[:, 4:].argmax(1) if not last_max else 79 - r[:, 4:].flip(1).argmax(1)
        xc, yc, w, h = r[:, 0], r[:, 1], r[:, 2], r[:, 3]
        p = torch.stack([xc - w / 2, yc - h / 2, xc + w / 2, yc + h / 2, torch.where(probs >= 0.25, probs, torch.zeros_like(probs)),
                         ids.float()], -1)
        tpo.oview(after, pred).copy_(_tile(p).view(B, 1, A, 6))
    return Case("decode", box + cls, [pred, tpo.Opnd("call", 0, 1, 0, 1, B, 84, A, F32)], _io(), _ctx(), ws, write, call)


CASES = {"upsample2": upsample_case, "cbfuse": cbfuse_case, "layernorm": layernorm_dense_case, "ln_post": layernorm_token0_case,
         "ln_final": layernorm_eot_case, "attention causal": lambda: attention_case(1), "attention": lambda: attention_case(0),
         "l2norm": l2norm_case, "postprocess": postprocess_case, "decode": decode_case}


@pytest.mark.parametrize("name", list(CASES))
def test_exact_results_pass(name):
    c = CASES[name]()
    c.check(*c.exact())


# ------------------------------------------------------------------------------------------------ the corruptions
def _pixel_shift(c, after, call):
    """images 1 and its copy 4: the upsample written one pixel to the right"""
    y = tpo.oview(after, c.op.outs[0])
    for img in (1, 4):
        y[img] = torch.roll(y[img].clone(), 1, 1)


def _group_shift(c, after, call):
    """the upsample reads the next 8-channel group of its input buffer"""
    x = c.op.ins[0]
    tpo.oview(after, c.op.outs[0]).copy_(td.ref_pool("upsample2", tpo.oview(after, x._replace(co=x.co + 8)).float(), BF16).to(BF16))


def _byte_past(c, after, call):
    """one byte written just past the output slice's last channel, at one pixel"""
    y = c.op.outs[0]
    buf = tpo.oview(after, y._replace(co=0, C=y.cs))
    buf[2, 3, 4, y.co + y.C].view(torch.int16).fill_(1)


def _image_4(c, after, call):
    """one element of image 4 differs from image 1 (a wrong tile in one image)"""
    tpo.oview(after, c.op.outs[0])[4, 1, 2, 3] += 1


def _cbfuse_index(c, after, call):
    """the first source's nearest index one past the right one (clamped at the edge)"""
    srcs = [tpo.oview(after, s).float() for s in c.op.ins[:-1]]
    last = tpo.oview(after, c.op.ins[-1]).float()
    H, W = last.shape[1:3]
    s0 = srcs[0]
    i = (td._nearest_idx(H, s0.shape[1]) + 1).clamp(max=s0.shape[1] - 1)
    j = (td._nearest_idx(W, s0.shape[2]) + 1).clamp(max=s0.shape[2] - 1)
    acc = s0[:, i][:, :, j]
    for s in srcs[1:]:
        acc = acc + s[:, td._nearest_idx(H, s.shape[1])][:, :, td._nearest_idx(W, s.shape[2])]
    tpo.oview(after, c.op.outs[0]).copy_((acc + last).to(BF16))


def _ddof1(c, after, call):
    """the variance divided by W - 1"""
    c.write(after, call, ddof=1)


def _token1(c, after, call):
    c.write(after, call, tok=1)


def _eot_plus(c, after, call):
    c.write(after, call, d=1)


def _eot_minus(c, after, call):
    c.write(after, call, d=-1)


def _no_mask(c, after, call):
    c.write(after, call, causal=0)


def _drop_last(c, after, call):
    c.write(after, call, drop_last=True)


def _no_eps(c, after, call):
    c.write(after, call, e=0.0)


def _gap_write(c, after, call):
    """one float written into the gap after row 2 of the caller's output"""
    call["embeddings"].view(F32).view(B, -1)[2, -1] = 0.0


def _tied_swap(c, after, call):
    """the two tied rows of every image in the other order"""
    d = call["detections"].view(F32).view(B, -1, 6)
    conf = d[0, :, 4]
    k = [int(v) for v in (conf == 0.9).nonzero()[:2, 0]]
    assert len(k) == 2 and not torch.equal(d[:, k[0]], d[:, k[1]])
    d[:, k] = d[:, k[::-1]].clone()


def _last_max(c, after, call):
    c.write(after, call, last_max=True)


CORRUPTIONS = [pytest.param("upsample2", _pixel_shift, r"\(a\) differs", id="upsample-one-pixel-shift"),
               pytest.param("upsample2", _group_shift, r"\(a\) differs", id="upsample-channel-group-shift"),
               pytest.param("upsample2", _byte_past, r"\(d\) byte", id="byte-past-the-output"),
               pytest.param("upsample2", _image_4, r"\(b\) image 4 differs from its copy, image 1", id="image-4-differs"),
               pytest.param("cbfuse", _cbfuse_index, r"\(a\) differs", id="cbfuse-nearest-index-off-by-one"),
               pytest.param("layernorm", _ddof1, r"\(a\) worst \|err\|/bar", id="layernorm-variance-over-w-minus-1"),
               pytest.param("ln_post", _token1, r"\(a\) worst \|err\|/bar", id="ln-post-reads-token-1"),
               pytest.param("ln_final", _eot_plus, r"\(a\) worst \|err\|/bar", id="ln-final-eot-row-plus-1"),
               pytest.param("ln_final", _eot_minus, r"\(a\) worst \|err\|/bar", id="ln-final-eot-row-minus-1"),
               pytest.param("attention causal", _no_mask, r"\(a\) worst \|err\|/bar", id="attention-without-causal-mask"),
               pytest.param("attention", _drop_last, r"\(a\) worst \|err\|/bar", id="attention-drops-last-key"),
               pytest.param("l2norm", _no_eps, r"\(a\) worst \|err\|/bar", id="l2norm-without-eps"),
               pytest.param("l2norm", _gap_write, r"\(d\) byte", id="l2norm-writes-a-row-gap"),
               pytest.param("postprocess", _tied_swap, r"\(a\) differs", id="postprocess-tied-rows-swapped"),
               pytest.param("decode", _last_max, r"\(a\) differs", id="decode-last-max-wins")]


@pytest.mark.parametrize("name,corrupt,flag", CORRUPTIONS)
def test_corruption_is_flagged(name, corrupt, flag):
    c = CASES[name]()
    after, call = c.exact()
    c.check(after, call)
    corrupt(c, after, call)
    with pytest.raises(AssertionError, match=flag):
        c.check(after, call)
