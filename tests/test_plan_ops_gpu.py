"""Every launch of the detector, CLIP and face plans that is not a conv or GEMM, in place, one launch at a time.

tests/test_plan_convs_gpu.py and tests/test_plan_gemms_gpu.py check the conv and GEMM launches of these plans; this file checks
the rest, as the plans wire them: the letterbox, the stems, the pools, SPP, upsample and CBFuse, the fp32-accurate mode's plane
split and finishing pass, the head's decode and postprocess, and CLIP's patchify, embeddings, LayerNorms, attention and L2
norm, and the face embedder's input packing and L2 norm.  Each plan runs op by op (cc_*_run_ops) in a workspace the test owns
and fills with 0xFF bytes.  cc_*_op_io reports what each op reads and writes (include/clearcam_b200.h).  Before each such op
the workspace and the call's output tensors are saved, the op's outputs are filled with NaN (0xFF bytes for the integer ones)
unless an output is also an input, the op runs alone, and:

  (a) images 0..REPS-1 of every output match a reference computed from the operands as stored, with the bars of the kernels'
      direct tests: bit-exact for the pools, SPP, upsample, CBFuse, plane split, face packing, patchify, the text embedding
      and its EOT rows, the letterbox (against the oracle's preprocess) and the postprocess (the oracle's selection and
      scale_boxes, compared as values: a suppressed row is zeros of either sign); the decode bar of tests/test_yolo_gpu.py::test_decode_matches_oracle; float64 references with the bars of
      tests/test_detector_ops_gpu.py (stems, finish_f32), tests/test_clip_ops_gpu.py (LayerNorm, embedding + ln_pre, L2 norm;
      ln_final's rows are the EOT positions of the token ids) and tests/test_attention_gpu.py (attention);
  (b) image b of every output equals image b % REPS bit for bit (the detections, the head tap and the EOT rows, less b L,
      included);
  (c) every output is finite;
  (d) every workspace byte the op changed lies in its reported outputs, and every byte of the call's output tensors outside
      the op's rows keeps what it held (the CLIP embeddings are written out_row_stride = D + 24 floats apart, so the gaps
      between rows must keep their NaN).

The conv and GEMM ops run unchecked here; their reported operands must equal what cc_*_op_conv describes.  Each config checks
that every op is one or the other, and the last test that every kind of non-conv op was reached by some config."""
import collections
import ctypes
import math
import time
from typing import NamedTuple

import numpy as np
import pytest
import torch

from clearcam_b200._lib import (CC_CONV_OP_CHAIN, CC_CONV_OP_NONE, CC_OP_BF16, CC_OP_F32, CC_OP_I32, CC_OP_U8, cc_conv_op, cc_op_io,
                                check, lib, ptr, stream_ptr)

import test_attention_gpu as ta
import test_clip_ops_gpu as tco
import test_conv_gpu as tc
import test_detector_ops_gpu as td
import test_plan_convs_gpu as tp
import test_plan_gemms_gpu as tg

pytestmark = pytest.mark.gpu

REPS = tp.REPS
DTYPES = {CC_OP_U8: torch.uint8, CC_OP_BF16: torch.bfloat16, CC_OP_F32: torch.float32, CC_OP_I32: torch.int32}
FMT_BGR_U8, FMT_BGR_F32, FMT_I420 = 0, 1, 2
CLIP_PAD = 24                     # out_row_stride = embed_dim + 24 floats
POOLS = {"avgpool2_pad": "avg2_pad", "avgmax_pool": "avgmax", "maxpool5": "max5", "upsample2": "upsample2"}
KINDS = {"letterbox", "stem_tc", "stem", "spp3", "cbfuse", "split_planes", "finish_f32", "decode", "postprocess", "patchify",
         "embed_ln_pre", "text_embed", "layernorm", "attention", "l2norm", "face_pack"} | set(POOLS)
CONV_KINDS = {"conv_gemm", "conv_direct"}
_SEEN = collections.defaultdict(set)        # kind -> configs that checked it
_RAN = set()
_REPORT = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nnon-conv kinds checked (kind: configs)")
    for k in sorted(_SEEN):
        print(f"  {k}: {' '.join(sorted(_SEEN[k]))}")
    for line in _REPORT:
        print(line)
    tp._MODELS.clear()
    tg._MODELS.clear()


# ------------------------------------------------------------------------------------------------ operands
class Opnd(NamedTuple):
    """One operand of an op: `where` is "ws" (off: byte offset in the workspace), "call" (the call's own input, output or raw
    tap; off unused) or "const" (off: the device address of a table outside the workspace); then channels per pixel, first
    channel, channels, N, H, W, element dtype and the pixels from one image to the next (0: dense)."""
    where: str
    off: int
    cs: int
    co: int
    C: int
    N: int
    H: int
    W: int
    dtype: torch.dtype
    ns: int = 0


def _opnd(o, ws):
    s, wp = o.s, ws.data_ptr()
    where = "call" if not s.p else "ws" if wp <= s.p < wp + ws.numel() else "const"
    off = 0 if not s.p else s.p - wp if where == "ws" else s.p
    return Opnd(where, off, s.cs, s.co, s.C, s.N, s.H, s.W, DTYPES[o.type], o.ns)


def oview(buf, o):
    """Operand o of the uint8 buffer buf (the workspace, or a call tensor's bytes) as a typed [N, H, W, C] view."""
    es = o.dtype.itemsize
    assert o.off % es == 0 and buf.numel() % es == 0, o
    return buf.view(o.dtype).as_strided((o.N, o.H, o.W, o.C), ((o.ns or o.H * o.W) * o.cs, o.W * o.cs, o.cs, 1), o.off // es + o.co)


def _const(o):
    """A copy of the table at device address o.off (weights, LayerNorm gamma / beta, embedding tables)."""
    assert o.dtype == torch.float32 and o.cs == o.C, o
    return tp._device(o.off, (o.N, o.H, o.W, o.C), torch.float32)


def same_opnd(a, b):
    return (a.where, a.off, a.cs, a.co, a.C) == (b.where, b.off, b.cs, b.co, b.C) and a.where != "call"


def _bytes(t):
    return t.view(-1).view(torch.uint8)


def _first(mask):
    return tuple(int(v) for v in mask.nonzero()[0])


def _bits(t):
    return t if t.dtype in (torch.uint8, torch.int32) else tp.bits(t)


def _equal(tag, got, want):
    """(a), bit-exact: got and want of one dtype."""
    g, w = _bits(got), _bits(want.to(got.dtype))
    if not torch.equal(g, w):
        raise AssertionError(f"{tag}: (a) differs from the reference at {_first(g != w)}: {got[_first(g != w)]} vs "
                             f"{want[_first(g != w)]}")


def _ratio(tag, key, err, bar, worst):
    """(a), against a bar: the worst |err| / bar (a zero bar asks for an exact result)."""
    ratio = torch.where(bar > 0, err / bar.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    r = ratio.max().item()
    worst[key] = max(worst.get(key, 0.0), r)
    assert r <= 1.0, f"{tag}: (a) worst |err|/bar {r:.3f} at {_first(ratio == ratio.max())}"


def check_copies(tag, got, eot_rows=0):
    """(c) and (b) of one output (got: [B, ...], the whole batch).  eot_rows = L: the EOT row indices b L + position."""
    if got.dtype.is_floating_point:
        fin = torch.isfinite(got)
        assert fin.all(), f"{tag}: (c) output not finite at {_first(~fin)}"
    g = _bits(got)
    if eot_rows:
        g = g - torch.arange(g.shape[0], device=g.device, dtype=g.dtype).view(-1, *[1] * (g.dim() - 1)) * eot_rows
    for i in range(REPS, g.shape[0]):
        if not torch.equal(g[i], g[i % REPS]):
            raise AssertionError(f"{tag}: (b) image {i} differs from its copy, image {i % REPS}, at {_first(g[i] != g[i % REPS])}")


def check_stray(tag, before, after, outs):
    """(d): outside the operands `outs`, the buffer `after` holds what `before` held (both uint8)."""
    scratch = after.clone()
    for o in outs:
        oview(scratch, o).copy_(oview(before, o))
    if not torch.equal(scratch, before):
        raise AssertionError(f"{tag}: (d) byte {tp._first_diff(scratch, before)} changed outside the op's outputs")


# ------------------------------------------------------------------------------------------------ references per kind
# Each takes the op (io, the cc_op_io; ins / outs: the input views as stored before the op and the output views after it,
# images 0..n-1 of the batch operands), the plan facts `ctx` and the worst dict, and raises AssertionError on a mismatch.
def ref_pool(op, ins, outs, ctx, worst):
    x = ins[0].float().cpu()
    _equal(op.tag, outs[0].cpu(), td.ref_pool(POOLS[op.kind], x, outs[0].dtype))


def ref_spp3(op, ins, outs, ctx, worst):
    c1 = ins[0].shape[-1]
    p, got = ins[0].float().cpu(), outs[0].cpu()
    for q in range(3):
        p = td.ref_pool("max5", p, torch.bfloat16)
        _equal(op.tag + f" pool {q + 1}", got[..., q * c1:(q + 1) * c1], p)


def ref_cbfuse(op, ins, outs, ctx, worst):
    x = [t.float().cpu() for t in ins]
    _equal(op.tag, outs[0].cpu(), td.ref_cbfuse(x[:-1], x[-1], outs[0].dtype))


def ref_split(op, ins, outs, ctx, worst):
    hi, mid, lo = td.split3(ins[0].cpu())
    _equal(op.tag, outs[0].cpu(), torch.cat([lo, mid, hi, mid, hi, hi], -1))


def ref_finish(op, ins, outs, ctx, worst):
    z = ins[0].double() + ins[1].double().flatten()
    want = td.silu64(z) if op.io.act else z
    r = ins[2].double() if len(ins) > 2 else torch.zeros_like(z)
    _ratio(op.tag, "finish_f32", (outs[0].double() - (want + r)).abs(), td.FIN_BAR * (z.abs() + r.abs()), worst)


def ref_stem(op, ins, outs, ctx, worst):
    Cout = outs[0].shape[-1]
    w = ins[1].reshape(Cout, 3, 3, 3).permute(0, 3, 1, 2).cpu()          # (kh, kw, c) -> PyTorch's (c, kh, kw)
    z, y, mag = td.stem_ref(ins[0].cpu(), w, ins[2].flatten().cpu(), 1 if op.kind == "stem_tc" else 2, dev="cuda")
    f32 = outs[0].dtype == torch.float32
    _ratio(op.tag, f"{op.kind} {'fp32' if f32 else 'bf16'} out", (outs[0].double() - y).abs(), td.stem_bar(z, y, mag, f32), worst)


def ref_letterbox(op, ins, outs, ctx, worst):
    from oracle import yolov9 as o
    from oracle.yuv import i420_to_bgr
    frames = ins[0].cpu()
    if ctx["fmt"] == FMT_I420:
        frames = torch.stack([i420_to_bgr(f[..., 0]) for f in frames])
    want = torch.stack([o.preprocess(f, ctx["res"]) for f in frames])
    got = outs[0].cpu()
    Hr, Wr = want.shape[1:3]
    _equal(op.tag, got[:, :Hr, :Wr], want)
    assert not got[:, Hr:].any() and not got[:, :, Wr:].any(), f"{op.tag}: (a) the net input's last row / column is not zero"


def ref_decode(op, ins, outs, ctx, worst):
    """test_yolo_gpu.py::test_decode_matches_oracle's reference and bars on the stored fp32 maps; pred's boxes are the head
    tap's, as corners."""
    from oracle import yolov9 as o
    n = ins[0].shape[0]
    box, cls = [t.cpu() for t in ins[:3]], [t.cpu() for t in ins[3:]]
    hw = [tuple(t.shape[1:3]) for t in box]
    A = sum(h * w for h, w in hw)
    cat = torch.cat([torch.cat([b, c], -1).reshape(n, -1, 144).permute(0, 2, 1) for b, c in zip(box, cls)], 2)
    bx, cl = cat.split((64, 80), 1)
    dist = (bx.reshape(n, 4, 16, A).softmax(2) * torch.arange(16.0).reshape(1, 1, 16, 1)).sum(2)
    anchors, strides = o.make_anchors(hw)
    lt, rb = dist.chunk(2, 1)
    x1y1, x2y2 = anchors.unsqueeze(0) - lt, anchors.unsqueeze(0) + rb
    want = torch.cat([torch.cat([(x1y1 + x2y2) / 2, x2y2 - x1y1], 1) * strides, torch.sigmoid(cl)], 1)
    raw, pred = outs[1].cpu().reshape(n, 84, A), outs[0].cpu().reshape(n, A, 6)
    _ratio(op.tag + " raw boxes", "decode boxes |err| / 1e-3 px", (raw[:, :4] - want[:, :4]).abs(), torch.full((1,), 1e-3), worst)
    _ratio(op.tag + " raw probs", "decode probs |err| / 2e-6", (raw[:, 4:] - want[:, 4:]).abs(), torch.full((1,), 2e-6), worst)
    probs = raw[:, 4:].max(1)[0]
    _equal(op.tag + " pred class", pred[..., 5], raw[:, 4:].argmax(1).float())
    _equal(op.tag + " pred conf", pred[..., 4], torch.where(probs >= op.io.conf_thr, probs, torch.zeros_like(probs)))
    xc, yc, w, h = want[:, 0], want[:, 1], want[:, 2], want[:, 3]
    corners = torch.stack([xc - w / 2, yc - h / 2, xc + w / 2, yc + h / 2], -1)
    _ratio(op.tag + " pred boxes", "decode boxes |err| / 1e-3 px", (pred[..., :4] - corners).abs(), torch.full((1,), 1e-3), worst)


def ref_postprocess(op, ins, outs, ctx, worst):
    from oracle import yolov9 as o
    n, _, A, _ = ins[0].shape
    boxes = o.postprocess_boxes(ins[0].cpu().reshape(n, A, 6), op.io.max_det, op.io.iou_thr)
    if op.io.do_scale:
        Hf, Wf = ctx["Hf"], ctx["Wf"]
        new_w, new_h, px, py = o.letterbox_params(Hf, Wf, ctx["res"])
        boxes = o.scale_boxes((new_h + 2 * py, new_w + 2 * px), boxes, (Hf, Wf))
    got = outs[0].cpu().reshape(n, op.io.max_det, 6)
    # compared as values, as tests/test_yolo_gpu.py::test_postprocess_bit_exact does: a suppressed row is zeros, which the
    # oracle's boxes * keep leaves as -0.0 where a coordinate was negative
    if not torch.equal(got, boxes):
        raise AssertionError(f"{op.tag}: (a) differs from the reference at {_first(got != boxes)}")


def ref_patchify(op, ins, outs, ctx, worst):
    n, _, Pn, kpad = outs[0].shape
    S = ins[0].shape[2]
    want = tco.patchify_ref(ins[0].cpu().reshape(n, 3, S, S), op.io.patch, kpad)
    _equal(op.tag, outs[0].cpu().reshape(n * Pn, kpad), want)


def _eot(ids):
    """The EOT row of each image: b L + the first position of the largest id (the text encoder's argmax)."""
    n, L = ids.shape
    return torch.arange(n, dtype=torch.int32) * L + torch.from_numpy(np.argmax(ids.cpu().numpy(), axis=1)).int()


def ref_text_embed(op, ins, outs, ctx, worst):
    ids = ins[0].reshape(ins[0].shape[0], -1).cpu()
    tok, pos = ins[1][0, 0], ins[2][0, 0]
    want = tok[ids.long().clamp(0, tok.shape[0] - 1).to(tok.device)] + pos
    _equal(op.tag, outs[0][:, 0], want)
    _equal(op.tag + " EOT rows", outs[1].flatten().cpu(), _eot(ids))


def ref_layernorm(op, ins, outs, ctx, worst):
    W = ins[0].shape[-1]
    x = ins[0].reshape(-1, W)
    if len(ins) > 3:                          # ln_final: the EOT rows, as the token ids place them
        x = x[_eot(ctx["ids"][:ins[0].shape[0]]).long().to(x.device)]
    y, delta = tco.ln64(x, ins[1].flatten(), ins[2].flatten())
    got = outs[0].reshape(-1, W).double()
    _ratio(op.tag, "layernorm", (got - y).abs(), tco.ln_bar(y, delta), worst)
    b, cnt = tc.rn_bias(got, y, delta)           # the store rounds to nearest (a variance over W - 1 shows here only)
    if cnt >= 10 ** 5:
        worst["layernorm |rounding bias|"] = max(worst.get("layernorm |rounding bias|", 0.0), abs(b))
        assert abs(b) <= tco.RN_WINDOW, f"{op.tag}: (a) rounding bias {b:+.4f} ulp over {cnt} outputs"


def ref_embed_ln(op, ins, outs, ctx, worst):
    n, _, L, W = ins[0].shape
    v = ins[0].clone().view(n, L, W)
    v[:, 0] = ins[1].flatten()
    v = (v + ins[2].view(L, W)).view(n * L, W)
    y, delta = tco.ln64(v, ins[3].flatten(), ins[4].flatten())
    _ratio(op.tag, "embed + ln_pre", (outs[0].reshape(n * L, W).double() - y).abs(), delta, worst)


def ref_attention(op, ins, outs, ctx, worst):
    n, _, L, C3 = ins[0].shape
    H = C3 // 192
    qkv = ins[0].reshape(n * L, C3)
    ref = ta.reference(qkv, n, L, H, op.io.causal)
    got = ta.as_bhld(outs[0].reshape(n * L, H * 64), n, L, H).double()
    _ratio(op.tag, f"attention{' causal' if op.io.causal else ''}", (got - ref).abs(), ta.bar(qkv, n, L, H, ref), worst)


def ref_l2norm(op, ins, outs, ctx, worst):
    n, D = ins[0].shape[0], ins[0].shape[-1]
    want = tco.l2_ref(ins[0].reshape(n, D), op.io.eps)
    _ratio(op.tag, "l2norm", (outs[0].reshape(n, D).double() - want).abs(), tco.l2_const(D) * want.abs(), worst)


def ref_face_pack(op, ins, outs, ctx, worst):
    want = torch.zeros(outs[0].shape, dtype=torch.bfloat16)
    want[..., :3] = ins[0].cpu().to(torch.bfloat16)
    _equal(op.tag, outs[0].cpu(), want)


CHECKERS = {"letterbox": ref_letterbox, "stem_tc": ref_stem, "stem": ref_stem, "spp3": ref_spp3, "cbfuse": ref_cbfuse,
            "split_planes": ref_split, "finish_f32": ref_finish, "decode": ref_decode, "postprocess": ref_postprocess,
            "patchify": ref_patchify, "embed_ln_pre": ref_embed_ln, "text_embed": ref_text_embed, "layernorm": ref_layernorm,
            "attention": ref_attention, "l2norm": ref_l2norm, "face_pack": ref_face_pack, **{k: ref_pool for k in POOLS}}
assert set(CHECKERS) == KINDS


# ------------------------------------------------------------------------------------------------ one op, in place
class Op(NamedTuple):
    io: object
    kind: str
    tag: str
    ins: list
    outs: list


def scratch_outputs(op):
    """Outputs that are scratch, not results: the wgmma attention's V^T copy.  Only (d) applies to them."""
    return op.outs[1:] if op.kind == "attention" else []


def check_one(op, snap, ws, call_before, call, ctx, worst):
    """(a)-(d) of one op that ran on ws (held snap before) and the call tensors `call` (held call_before; name -> uint8)."""
    name = ctx["call_of"](op.kind)       # the call tensor this op's p == NULL outputs are rows of
    check_stray(op.tag, snap, ws, [o for o in op.outs if o.where == "ws"])
    for k, buf in call.items():
        check_stray(op.tag + f" ({k})", call_before[k], buf, [o for o in op.outs if o.where == "call" and k == name])

    def view(o, buf, before):
        if o.where == "ws":
            return oview(buf, o)
        if o.where == "const":
            return _const(o)
        if before:                       # the call's input
            return ctx["input"].view(o.N, o.H, o.W, o.C)
        return oview(call[name], o)

    scratch = scratch_outputs(op)
    outs = [view(o, ws, False) for o in op.outs if o not in scratch]
    for o, t in zip([o for o in op.outs if o not in scratch], outs):
        check_copies(op.tag, t, ctx["L"] if op.kind == "text_embed" and o.dtype == torch.int32 else 0)
    n = min(REPS, ctx["B"])
    ins = [view(o, snap, True) for o in op.ins]
    ins = [t if o.where == "const" else t[:n] for o, t in zip(op.ins, ins)]
    CHECKERS[op.kind](op, ins, [t[:n] for t in outs], ctx, worst)


def run_in_place(plan, descs, ios, ws, call, ctx, tag):
    """Every op of the plan one at a time on ws (filled with 0xFF): the non-conv ops checked, the others run.  Returns the
    worst |err|/bar per key and the kinds checked."""
    worst, kinds = {}, collections.Counter()
    ws.fill_(255)
    for buf in call.values():
        buf.fill_(255)
    for i, (d, io) in enumerate(zip(descs, ios)):
        kind, name = io.kind.decode(), io.name.decode()
        assert name == d.name.decode(), (name, d.name)
        ins = [_opnd(io.in_[k], ws) for k in range(io.n_in)]
        outs = [_opnd(io.out[k], ws) for k in range(io.n_out)]
        # a call output's cs is its row width: its rows lie the call's pitch apart
        outs = [o._replace(cs=ctx["pitch"].get(ctx["call_of"](kind), o.cs)) if o.where == "call" else o for o in outs]
        if d.kind != CC_CONV_OP_NONE:
            assert kind in CONV_KINDS, (name, kind)
            check_conv_operands(name, d, ins, outs, ws)
            plan.run(i, i + 1)
            continue
        assert kind in CHECKERS, f"{name}: an op of kind {kind!r} that nothing checks"
        op = Op(io, kind, f"{tag}: op {i} {name} ({kind})", ins, outs)
        snap = ws.clone()
        call_before = {k: v.clone() for k, v in call.items()}
        for o in outs:
            if o in scratch_outputs(op) or any(same_opnd(o, x) for x in ins):
                continue
            if o.where == "ws":
                fill = float("nan") if o.dtype.is_floating_point else 255 if o.dtype == torch.uint8 else -1
                oview(ws, o).fill_(fill)
        plan.run(i, i + 1)
        torch.cuda.synchronize()
        check_one(op, snap, ws, call_before, call, ctx, worst)
        del snap, call_before
        kinds[kind] += 1
    return worst, kinds


def check_conv_operands(name, d, ins, outs, ws):
    """The operand tap of a conv / GEMM op reports what cc_*_op_conv describes: in, [res], [pre], [part]; [out], [out2]."""
    def sl(s, ns=0):
        return (s.p, s.cs, s.co, s.C, s.N, s.H, s.W, s.f32, ns)

    def got(o):
        p = 0 if o.where == "call" else o.off + ws.data_ptr() if o.where == "ws" else o.off
        return (p, o.cs, o.co, o.C, o.N, o.H, o.W, int(o.dtype == torch.float32), o.ns)

    want_in = [sl(d.in_)] + ([sl(d.res, d.out_ns)] if d.res.p else [])
    if d.pre:
        want_in.append((d.pre, d.out.C, 0, d.out.C, d.out.N, d.pre_h, d.pre_w, 1, 0))
    want_in += [sl(d.part)] if d.part.p else []
    chained = d.kind == CC_CONV_OP_CHAIN
    want_out = ([sl(d.out, d.out_ns)] if not chained or d.store1 else []) + ([sl(d.out2)] if chained else [])
    assert [got(o) for o in ins] == want_in, f"{name}: the operand tap's inputs differ from the conv descriptor's"
    assert [got(o) for o in outs] == want_out, f"{name}: the operand tap's outputs differ from the conv descriptor's"


def _taps(op_conv, op_io):
    n = op_conv(0, None)
    check(min(n, 0), "op_conv")
    assert op_io(0, None) == n
    descs, ios = [], []
    for i in range(n):
        d, io = cc_conv_op(), cc_op_io()
        check(min(op_conv(i, ctypes.byref(d)), 0), "op_conv")
        check(min(op_io(i, ctypes.byref(io)), 0), "op_io")
        descs.append(d)
        ios.append(io)
    return descs, ios


def _record(cfg, tag, kinds, worst, n_ops, t0):
    for k in kinds:
        _SEEN[k].add(cfg)
    _RAN.add(cfg)
    line = (f"{tag}: {sum(kinds.values())} of {n_ops} ops checked ({', '.join(f'{k} {v}' for k, v in sorted(kinds.items()))}), "
            f"{time.time() - t0:.1f} s; worst " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))
    _REPORT.append(line)
    print(line)


# ------------------------------------------------------------------------------------------------ the detector plans
#        size res  B   Hf    Wf    fp32-accurate  padded widths  frame format
YOLO_CONFIGS = [pytest.param(*p.values, FMT_BGR_U8, id=p.id) for p in tp.CONFIGS]
YOLO_CONFIGS += [pytest.param("t", 320, 16, 320, 320, False, True, FMT_I420, id="t-b16-320-i420"),
                 pytest.param("t", 320, 16, 240, 426, False, True, FMT_BGR_F32, id="t-b16-240x426-f32")]


class _Yolo:
    def __init__(self, m, fmt, B, Hf, Wf, res, frames, out, raw):
        self.m, self.a, self.fr, self.out, self.raw = m, (fmt, B, Hf, Wf, res), frames, out, raw

    def run(self, first, last):
        check(lib().cc_yolo_run_ops(self.m._h, ptr(self.fr), self.a[0], *self.a[1:], first, last, ptr(self.out), ptr(self.raw),
                                    stream_ptr()), "cc_yolo_run_ops")


def _yolo_frames(fmt, B, Hf, Wf):
    from oracle import yolov9 as o
    if fmt == FMT_I420:
        g = torch.Generator().manual_seed(21)
        base = torch.randint(0, 256, (REPS, Hf * 3 // 2, Wf), generator=g, dtype=torch.uint8)
    else:
        base = o.synthetic_frames(REPS, Hf, Wf, seed=21)
        if fmt == FMT_BGR_F32:
            base = base.float() * torch.rand(base.shape, generator=torch.Generator().manual_seed(22))
    return base[torch.arange(B) % REPS].contiguous().cuda()


@pytest.mark.parametrize("size,res,B,Hf,Wf,precise,pad,fmt", YOLO_CONFIGS)
def test_every_detector_op_in_place(size, res, B, Hf, Wf, precise, pad, fmt):
    t0 = time.time()
    m = tp._model(size, res, precise, pad)
    fr = _yolo_frames(fmt, B, Hf, Wf)
    tag = (f"{size}{'' if pad else '-literal'} res {res} B {B} {Hf}x{Wf} {['bgr24', 'bgr f32', 'i420'][fmt]}"
           f"{' fp32-accurate' if precise else ''}")
    cfg = f"{size}{'' if pad else '-literal'}-b{B}-{Hf}x{Wf}-{['u8', 'f32', 'i420'][fmt]}{'-fp32acc' if precise else ''}"
    L = lib()
    n = ctypes.c_size_t()
    check(L.cc_yolo_workspace_bytes(m._h, fmt, B, Hf, Wf, res, ctypes.byref(n)), "cc_yolo_workspace_bytes")
    ws = torch.empty((n.value + 255) // 256 * 256, dtype=torch.uint8, device="cuda")
    check(L.cc_yolo_set_workspace(m._h, ptr(ws), ws.numel()), "cc_yolo_set_workspace")
    try:
        descs, ios = _taps(lambda i, d: L.cc_yolo_op_conv(m._h, fmt, B, Hf, Wf, res, i, d),
                           lambda i, d: L.cc_yolo_op_io(m._h, fmt, B, Hf, Wf, res, i, d))
        pix = "yuv420p" if fmt == FMT_I420 else "bgr24"
        prof = m.profile(fr, pix_fmt=pix)
        assert [(io.kind.decode(), io.name.decode()) for io in ios] == [(r["kind"], r["name"]) for r in prof]
        A = m.plan_info(B, Hf, Wf, is_f32=fmt == FMT_BGR_F32, pix_fmt=pix)["anchors"]
        out = torch.empty(B, 300, 6, device="cuda")
        raw = torch.empty(B, 84, A, device="cuda")
        call = {"detections": _bytes(out), "head tap": _bytes(raw)}
        ctx = {"B": B, "Hf": Hf, "Wf": Wf, "res": res, "fmt": fmt, "L": 0, "input": fr, "pitch": {},
               "call_of": lambda kind: "detections" if kind == "postprocess" else "head tap"}
        worst, kinds = run_in_place(_Yolo(m, fmt, B, Hf, Wf, res, fr, out, raw), descs, ios, ws, call, ctx, tag)
        n_conv = sum(d.kind != CC_CONV_OP_NONE for d in descs)
        assert sum(kinds.values()) + n_conv == len(prof) and n_conv == sum(r["kind"] in CONV_KINDS for r in prof)
        assert {"decode", "postprocess"} <= set(kinds) and (kinds.keys() & {"stem", "stem_tc"})
    finally:
        torch.cuda.synchronize()
        check(L.cc_yolo_set_workspace(m._h, None, 0), "cc_yolo_set_workspace")
    _record(cfg, tag, kinds, worst, len(descs), t0)


# ------------------------------------------------------------------------------------------------ the CLIP and face plans
class _ClipRun:
    def __init__(self, p, stride):
        self.p, self.stride = p, stride

    def run(self, first, last):
        p = self.p
        check(lib().cc_clip_run_ops(p.m._h, p.text, ptr(p.inp), p.B, first, last, ptr(p.out), self.stride, stream_ptr()),
              "cc_clip_run_ops")


@pytest.mark.parametrize("kind,arch,text,B", tg.CONFIGS)
def test_every_clip_and_face_op_in_place(kind, arch, text, B):
    t0 = time.time()
    p = tg._plan(kind, arch, text, B)
    L = lib()
    if kind == "clip":
        D = p.m.embed_dim
        stride = D + CLIP_PAD
        p.out = torch.empty(B, stride, device="cuda")
        runner = _ClipRun(p, stride)
        taps = (lambda i, d: L.cc_clip_op_conv(p.m._h, p.text, B, i, d), lambda i, d: L.cc_clip_op_io(p.m._h, p.text, B, i, d))
        cfg = f"{arch}-{'text' if text else 'image'}-b{B}"
    else:
        D = stride = 512
        runner = p
        taps = (lambda i, d: L.cc_face_op_conv(p.m._h, B, i, d), lambda i, d: L.cc_face_op_io(p.m._h, B, i, d))
        cfg = f"face-b{B}"
    worst = {}
    with tg._Workspace(p) as ws:
        descs, ios = _taps(*taps)
        if kind == "clip":
            assert [io.name.decode() for io in ios] == p.gemm_names()
        call = {"embeddings": _bytes(p.out)}
        ctx = {"B": B, "L": p.inp.shape[1] if text else 0, "input": p.inp, "ids": p.inp if text else None,
               "pitch": {"embeddings": stride}, "call_of": lambda kind: "embeddings"}
        worst, kinds = run_in_place(runner, descs, ios, ws, call, ctx, p.tag)
        n_conv = sum(d.kind != CC_CONV_OP_NONE for d in descs)
        assert sum(kinds.values()) + n_conv == len(descs)
        if kind == "clip":
            assert n_conv == sum(io.name.decode() in tg.CLIP_GEMMS for io in ios)
        else:
            assert n_conv == tg.FACE_GEMMS and dict(kinds) == {"face_pack": 1, "l2norm": 1}
        nbytes = ws.numel()
    _record(cfg, f"{p.tag} (workspace {nbytes / 2 ** 20:.0f} MiB)", kinds, worst, len(descs), t0)


def test_every_kind_was_reached():
    """Over every config of this file, each kind of non-conv op the plans build was checked at least once.  The plans run
    the wgmma attention kernel at every sequence length they have (50, 77, 257), so the mma.sync kernel is not among them."""
    every = {p.id for p in YOLO_CONFIGS} | {p.id for p in tg.CONFIGS}
    if len(_RAN) < len(every):
        pytest.skip("runs with the whole file")
    assert not KINDS - set(_SEEN), f"kinds no config reached: {sorted(KINDS - set(_SEEN))}"
