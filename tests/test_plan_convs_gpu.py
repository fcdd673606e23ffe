"""Every conv launch of the detector plans, in place, at the shapes the benchmark runs.

Each plan runs op by op on its own buffers (cc_yolo_run_ops) in a workspace the test owns and fills with 0xFF bytes (NaN in
bf16 and fp32).  Before each conv op the whole workspace is saved and the op's output slices are filled with NaN (except a
slice that is also the op's residual); the op then runs alone, and:

  (a) images 0..REPS-1 of its output match a float64 conv of the operands as stored: the saved input, residual and
      pre-activation addend, and the weights and bias read through their device pointers.  The bars are those of
      tests/test_conv_gpu.py (bf16_bar, F32_BAR, the round-to-nearest bias of activation-free bf16 outputs) and, for a conv with
      the fused-upsample addend, that of tests/test_detector_ops_gpu.py::test_cc_conv_pre_addend_matches_float64;
  (b) the batch holds copies of REPS distinct frames, so image b of every output must equal image b % REPS bit for bit: a
      pixel's arithmetic does not depend on which tile or CTA computes it, so a wrong tile anywhere in the batch shows;
  (c) every output is finite;
  (d) every workspace byte the op changed lies in its declared outputs (the first output when stored, the chained output);
  (e) a chained launch: its first conv is checked as in (a) (recomputed unchained when the launch drops it), and the chained
      1x1's output equals the unchained pair (two cc_conv launches over the same channels) bit for bit and is checked as
      in (a) itself.

Then the whole forward: the first cc_yolo_forward call (plain launches, with programmatic dependent launch), the second
(graph capture) and the third (graph replay) each give the bytes of the ops launched one at a time with a device
synchronisation after each; and so do forwards on a zero-filled and a 0xFF-filled
workspace.  The distinct launch configurations each plan selects are printed (kernel instance, tiles, pipeline), so a change
to the conv kernel can see which of them it must keep right."""
import collections
import ctypes
import math
import time
import types
from typing import NamedTuple

import pytest
import torch
import torch.nn.functional as F

from clearcam_b200 import ops
from clearcam_b200._lib import CC_CONV_OP_CHAIN, CC_CONV_OP_DIRECT, CC_CONV_OP_NONE, cc_conv_op, check, lib, ptr, stream_ptr

import test_conv_gpu as tc
import test_detector_ops_gpu as td

pytestmark = pytest.mark.gpu

REPS = 3      # distinct frames per batch: image b is a copy of image b % REPS, at a different offset within its tile group
BF16, F32 = torch.bfloat16, torch.float32
ACT_NAMES = {0: "NONE", 1: "SILU", 2: "GELU_TANH", 3: "PRELU"}
ACT_PRELU = 3


class Slice(NamedTuple):
    """An NHWC slice of the workspace: byte offset of the buffer, channels per pixel, first channel, channels, N, H, W, fp32,
    and the pixels from one image to the next (0: H * W, dense)."""
    off: int
    cs: int
    co: int
    C: int
    N: int
    H: int
    W: int
    f32: int
    ns: int = 0


def sview(ws, s):
    """The slice s of the uint8 workspace ws as a typed [N, H, W, C] view."""
    es = 4 if s.f32 else 2
    assert s.off >= 0 and s.off % es == 0, s
    flat = ws.view(F32 if s.f32 else BF16)
    return flat.as_strided((s.N, s.H, s.W, s.C), ((s.ns or s.H * s.W) * s.cs, s.W * s.cs, s.cs, 1), s.off // es + s.co)


def sbuf(ws, s):
    """The whole buffer s is a slice of: every channel of its pixels."""
    return sview(ws, s._replace(co=0, C=s.cs))


def same_slice(a, b):
    return a is not None and b is not None and (a.off, a.cs, a.co, a.C) == (b.off, b.cs, b.co, b.C)


def bits(t):
    return t.view(torch.int32 if t.dtype == F32 else torch.int16)


def ref64(x, w, b, k, s, groups, act, res=None, pre=None, slope=None):
    """float64 (z, y = [res +] act(z), sum|x.w| + |b| + |pre| + |res|) of a conv, z = conv(x, w) + b [+ up2(pre)].  x: [n, H, W,
    Cin]; w: [Cout, k, k, Cin / groups]; pre: [n, Ho / 2, Wo / 2, Cout] added before the activation (nearest upsampling).
    act = ACT_PRELU: b is the [9, Cout] table indexed by the output pixel's border class, and act(z) = where(z > 0, z,
    slope * z)."""
    xd, wd = x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2)
    z = F.conv2d(xd, wd, None, s, k // 2, 1, groups).permute(0, 2, 3, 1)
    mag = F.conv2d(xd.abs(), wd.abs(), None, s, k // 2, 1, groups).permute(0, 2, 3, 1)
    if b is not None:
        bd = b.double()
        if act == ACT_PRELU:
            from oracle.adaface import class_map
            bd = bd[class_map(*z.shape[1:3]).to(bd.device)]
        z, mag = z + bd, mag + bd.abs()
    if pre is not None:
        Ho, Wo = z.shape[1:3]
        up = pre.double()[:, torch.arange(Ho, device=pre.device) // 2][:, :, torch.arange(Wo, device=pre.device) // 2]
        z, mag = z + up, mag + up.abs()
    if act == ACT_PRELU:
        y = torch.where(z > 0, z, slope.double() * z)
    else:
        y = F.silu(z) if act == 1 else F.gelu(z, approximate="tanh") if act == 2 else z
    if res is not None:
        y, mag = y + res.double(), mag + res.double().abs()
    return z, y, mag


def _first(mask):
    return tuple(int(v) for v in mask.nonzero()[0])


def check_values(tag, got, x, w, b, k, s, groups, act, res, pre, f32, worst, slope=None):
    """(c), (b) and (a) of one output: got [B, Ho, Wo, C] is the whole batch as the op wrote it; x, res and pre are images
    0..REPS-1 of the operands as stored before the op; slope: the PReLU slopes of act = ACT_PRELU."""
    fin = torch.isfinite(got)
    assert fin.all(), f"{tag}: (c) output not finite at {_first(~fin)}"
    gb = bits(got)
    for i in range(REPS, got.shape[0]):
        if not torch.equal(gb[i], gb[i % REPS]):
            raise AssertionError(f"{tag}: (b) image {i} differs from its copy, image {i % REPS}, at "
                                 f"{_first(gb[i] != gb[i % REPS])}")
    n = x.shape[0]
    z, y, mag = ref64(x, w, b, k, s, groups, act, res, pre, slope)
    g = got[:n].double()
    if f32:
        # F32_BAR holds per tc.F32_STEPS k16 steps into one accumulator (see test_conv_gpu.py): the fp32-accurate mode's
        # cross-product GEMMs take up to 1440 (its hi x hi GEMMs, whose products are 2^8 times larger, at most 48)
        steps = k * k * x.shape[-1] // groups // 16
        bar, key = tc.F32_BAR * max(1.0, steps / tc.F32_STEPS) * mag, "fp32 |err|/bar"
    elif pre is not None:
        bar, key = td.pre_bar(z, y, mag, False), "bf16 + pre |err|/bar"
    elif act == ACT_PRELU:
        # the negative side scales z, and so z's fp32 error, by the slope
        bar, key = 2.0 ** -7 * y.abs() + tc.F32_BAR * mag * slope.double().abs().clamp(min=1.0), "PReLU |err|/bar"
    else:
        bar, key = tc.bf16_bar(z, y, mag, act), "bf16 |err|/bar"
    err = (g - y).abs()
    # a zero bar (a padding channel: zero weights and bias) asks for an exact zero
    ratio = torch.where(bar > 0, err / bar.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    r = ratio.max().item()
    worst[key] = max(worst.get(key, 0.0), r)
    assert r <= 1.0, f"{tag}: (a) worst |err|/bar {r:.3f} at {_first(ratio == ratio.max())}"
    if f32:
        rel = err / y.abs().clamp(min=1.0)
        worst["fp32 max |err|/max(|ref|, 1)"] = max(worst.get("fp32 max |err|/max(|ref|, 1)", 0.0), rel.max().item())
        assert rel.max().item() < tc.F32_REL, f"{tag}: (a) relative error {rel.max().item():.2e} at {_first(rel == rel.max())}"
    if not f32 and act == 0:
        rb, cnt = tc.rn_bias(g, y, tc.F32_BAR * mag)
        if cnt >= 10 ** 4:
            worst["bf16 act-0 |rounding bias|"] = max(worst.get("bf16 act-0 |rounding bias|", 0.0), abs(rb))
            assert abs(rb) <= tc.RN_WINDOW, f"{tag}: (a) rounding bias {rb:+.4f} ulp over {cnt} outputs"


def _first_diff(a, b, chunk=1 << 28):
    for lo in range(0, a.numel(), chunk):
        d = a[lo:lo + chunk] != b[lo:lo + chunk]
        if d.any():
            return lo + int(d.nonzero()[0])
    return -1


def check_stray(tag, snap, ws, outs):
    """(d): outside the slices `outs`, the workspace ws holds what it held before the op (snap)."""
    scratch = ws.clone()
    for s in outs:
        sview(scratch, s).copy_(sview(snap, s))
    if not torch.equal(scratch, snap):
        raise AssertionError(f"{tag}: (d) workspace byte {_first_diff(scratch, snap)} changed outside the op's outputs")


def op_outputs(op):
    chained = op.kind == CC_CONV_OP_CHAIN
    return ([op.out] if not chained or op.store1 else []) + ([op.out2] if chained else [])


def images(t, rows):
    """t [1, 1, R, C], the R rows of a row GEMM (a linear as a 1x1 conv), as [R / rows, 1, rows, C]: one image per block of
    `rows` rows.  rows = 0: t as it is."""
    return t if not rows else t.reshape(-1, 1, rows, t.shape[-1])


def check_op(op, snap, ws, worst, rows=0):
    """(a)-(e) of one conv op that ran on ws, whose contents before the op were snap.  rows: the op is a row GEMM whose images
    are blocks of that many rows (see `images`)."""
    tag = op.name
    check_stray(tag, snap, ws, op_outputs(op))
    xs = images(sview(snap, op.in_), rows)
    n = min(REPS, xs.shape[0])
    x = xs[:n]
    res = None if op.res is None else images(sview(snap, op.res), rows)[:n]
    pre = None if op.pre is None else sview(snap, op.pre)[:n]
    if op.kind != CC_CONV_OP_CHAIN:
        check_values(tag, images(sview(ws, op.out), rows), x, op.w, op.bias, op.k, op.stride, op.groups, op.act, res, pre,
                     op.out.f32, worst, op.slope)
        return
    # (e) the same two convs unchained, on the operands as stored: the first into a copy of its buffer
    buf1 = sbuf(snap, op.out).clone()
    rbuf = None
    if op.res is not None:
        rbuf = buf1 if op.res.off == op.out.off else sbuf(snap, op.res).contiguous()
    ops.conv2d(sbuf(snap, op.in_).contiguous(), op.in_.co, op.in_.C, op.w, op.bias, op.k, op.stride, buf1, op.out.co, op.out.C,
               act=op.act, res=rbuf, res_co=0 if op.res is None else op.res.co)
    first = buf1[..., op.out.co:op.out.co + op.out.C]
    if op.store1:
        assert torch.equal(bits(sview(ws, op.out)), bits(first)), f"{tag}: (e) the chained launch's first output differs from cc_conv"
    check_values(tag + " [first conv]", first, x, op.w, op.bias, op.k, op.stride, 1, op.act, res, None, False, worst)
    N2 = op.out2.C
    run = N2 - (op.part.C if op.part is not None else 0)
    x2 = [buf1[..., op.out.co + op.k0:op.out.co + op.k0 + run]] + ([sview(snap, op.part)] if op.part is not None else [])
    x2 = torch.cat(x2, -1).contiguous()
    ref2 = torch.empty(x2.shape[:3] + (N2,), dtype=F32 if op.out2.f32 else BF16, device=x2.device)
    ops.conv2d(x2, 0, N2, op.w2, op.bias2, 1, 1, ref2, 0, N2, act=op.act2)
    got2 = sview(ws, op.out2)
    if not torch.equal(bits(got2), bits(ref2)):
        raise AssertionError(f"{tag}: (e) the chained 1x1 differs from the unchained pair at {_first(bits(got2) != bits(ref2))}")
    check_values(tag + " [chained 1x1]", got2, x2[:n], op.w2, op.bias2, 1, 1, 1, op.act2, None, None, op.out2.f32, worst)


# ------------------------------------------------------------------------------------------------ the plans on the GPU
#        size res  B   Hf    Wf    fp32-accurate  padded widths
CONFIGS = [pytest.param("c", 640, 32, 640, 640, False, True, id="c-b32-640"),
           pytest.param("e", 640, 16, 640, 640, False, True, id="e-b16-640"),
           pytest.param("c", 640, 8, 1080, 1920, False, True, id="c-b8-1080p"),
           pytest.param("t", 320, 16, 320, 320, False, True, id="t-b16-320"),
           pytest.param("t", 320, 16, 320, 320, False, False, id="t-literal-b16-320"),
           pytest.param("s", 256, 2, 192, 256, False, True, id="s-b2-192x256"),
           pytest.param("c", 640, 8, 1080, 1920, True, True, id="c-b8-1080p-fp32acc"),
           pytest.param("t", 320, 16, 320, 320, True, True, id="t-b16-320-fp32acc")]
_WEIGHTS, _MODELS = {}, {}
_COVERAGE = collections.OrderedDict()      # launch configuration -> [ops, plans]
_REPORT = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlaunch configurations (kernel instance | BN BK | tile box w x h x images | s2 | b_res | stages | tiles per CTA"
          " | ops | plans)")
    for key, (n, plans) in _COVERAGE.items():
        print(" | ".join(str(v) for v in key), "|", n, "|", " ".join(sorted(plans)))
    for line in _REPORT:
        print(line)
    _MODELS.clear()


def _model(size, res, precise, pad):
    from oracle import yolov9 as o
    from clearcam_b200.detection.yolov9 import YOLOv9
    key = (size, res, precise, pad)
    if key not in _MODELS:
        if size not in _WEIGHTS:
            _WEIGHTS[size] = o.synthetic_weights(size, seed=21)
        _MODELS[key] = YOLOv9(size, res, weights=_WEIGHTS[size], precise=precise, pad=pad)
    return _MODELS[key]


def _frames(B, Hf, Wf):
    from oracle import yolov9 as o
    return o.synthetic_frames(REPS, Hf, Wf, seed=21)[torch.arange(B) % REPS].contiguous().cuda()


class _Workspace:
    """A caller-owned workspace for the plan of (B, Hf, Wf, res) on model m, handed back to the library on exit."""

    def __init__(self, m, B, Hf, Wf, res):
        self.m, self.shape = m, (B, Hf, Wf, res)

    def __enter__(self):
        n = ctypes.c_size_t()
        check(lib().cc_yolo_workspace_bytes(self.m._h, 0, *self.shape, ctypes.byref(n)), "cc_yolo_workspace_bytes")
        self.ws = torch.empty((n.value + 255) // 256 * 256, dtype=torch.uint8, device="cuda")
        self.adopt()
        return self.ws

    def adopt(self):
        """(Re)hand the workspace over: the handle drops its plans, so the next call builds them again."""
        check(lib().cc_yolo_set_workspace(self.m._h, ptr(self.ws), self.ws.numel()), "cc_yolo_set_workspace")

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        check(lib().cc_yolo_set_workspace(self.m._h, None, 0), "cc_yolo_set_workspace")
        del self.ws


def _descs(m, B, Hf, Wf, res):
    L = lib()
    n = L.cc_yolo_op_conv(m._h, 0, B, Hf, Wf, res, 0, None)
    check(min(n, 0), "cc_yolo_op_conv")
    out = []
    for i in range(n):
        d = cc_conv_op()
        check(min(L.cc_yolo_op_conv(m._h, 0, B, Hf, Wf, res, i, ctypes.byref(d)), 0), "cc_yolo_op_conv")
        out.append(d)
    return out


def _run(m, fr, B, Hf, Wf, res, first, last, out, raw):
    check(lib().cc_yolo_run_ops(m._h, ptr(fr), 0, B, Hf, Wf, res, first, last, ptr(out), ptr(raw), stream_ptr()), "cc_yolo_run_ops")


def _forward(m, fr, B, Hf, Wf, res, out, raw):
    check(lib().cc_yolo_forward(m._h, ptr(fr), 0, B, Hf, Wf, res, ptr(out), ptr(raw), stream_ptr()), "cc_yolo_forward")


def _device(p, shape, dtype):
    """A copy of the device array at address p (weights and biases live outside the workspace)."""
    cai = types.SimpleNamespace(__cuda_array_interface__={"shape": (math.prod(shape),), "typestr": "<f4" if dtype == F32 else "<i2",
                                                          "data": (p, False), "version": 2})
    t = torch.as_tensor(cai, device="cuda")
    return (t if dtype == F32 else t.view(BF16)).view(shape).clone()


def _plan_op(d, ws):
    """The conv op d (a cc_conv_op) with its slices as workspace offsets and its weights copied out."""
    wp, nbytes = ws.data_ptr(), ws.numel()

    def sl(s, ns=0):
        if not s.p:
            return None
        assert wp <= s.p < wp + nbytes, f"{d.name.decode()}: a slice outside the workspace"
        return Slice(s.p - wp, s.cs, s.co, s.C, s.N, s.H, s.W, s.f32, ns)

    Cout = d.out.C
    op = types.SimpleNamespace(kind=d.kind, name=d.name.decode(), in_=sl(d.in_), out=sl(d.out, d.out_ns), res=sl(d.res, d.out_ns),
                               k=d.k, stride=d.stride, groups=d.groups, act=d.act, store1=d.store1, k0=d.k0, act2=d.act2,
                               part=sl(d.part), out2=sl(d.out2), pre=None, w2=None, bias2=None, slope=None)
    op.w = _device(d.w, (Cout, d.k, d.k, d.in_.C // d.groups), BF16)
    op.bias = _device(d.bias, (9, Cout) if d.act == ACT_PRELU else (Cout,), F32) if d.bias else None
    if d.act == ACT_PRELU:
        op.slope = _device(d.slope, (Cout,), F32)
    if d.pre:
        assert wp <= d.pre < wp + nbytes
        op.pre = Slice(d.pre - wp, Cout, 0, Cout, d.out.N, d.pre_h, d.pre_w, 1)
    if d.kind == CC_CONV_OP_CHAIN:
        N2 = d.out2.C
        op.w2 = _device(d.w2, (N2, 1, 1, N2), BF16)
        op.bias2 = _device(d.bias2, (N2,), F32) if d.bias2 else None
    return op


def _launch_key(d):
    if d.kind == CC_CONV_OP_DIRECT:
        return (f"conv_direct_kernel (k {d.k}, s {d.stride}, groups {d.groups}, {'fp32' if d.out.f32 else 'bf16'} out)",) + ("-",) * 6
    inst = f"conv_gemm_kernel<{ACT_NAMES[d.act]}, {'fp32' if d.out.f32 else 'bf16'}, BN {d.BN}"
    if d.kind == CC_CONV_OP_CHAIN:
        inst += f", N2 {d.out2.C}, {ACT_NAMES[d.act2]}, {'fp32' if d.out2.f32 else 'bf16'}"
    return (inst + ">", f"{d.BN} {d.BK}", f"{1 << d.lTW}x{1 << d.lTH}x{1 << d.lTN}", d.s2, d.b_res, d.stages,
            -(-d.num_tiles // d.grid))


@pytest.mark.parametrize("size,res,B,Hf,Wf,precise,pad", CONFIGS)
def test_every_conv_launch_in_place(size, res, B, Hf, Wf, precise, pad):
    t0 = time.time()
    m = _model(size, res, precise, pad)
    fr = _frames(B, Hf, Wf)
    tag = f"{size}{'' if pad else '-literal'} res {res} B {B} {Hf}x{Wf}{' fp32-accurate' if precise else ''}"
    worst = {}
    with _Workspace(m, B, Hf, Wf, res) as ws:
        prof = m.profile(fr)
        descs = _descs(m, B, Hf, Wf, res)
        assert [d.name.decode() for d in descs] == [r["name"] for r in prof]
        for d, r in zip(descs, prof):
            kind = {CC_CONV_OP_NONE: r["kind"], CC_CONV_OP_DIRECT: "conv_direct"}.get(d.kind, "conv_gemm")
            assert kind == r["kind"] and (d.kind != CC_CONV_OP_NONE or kind not in ("conv_gemm", "conv_direct")), (r, d.kind)
        A = m.plan_info(B, Hf, Wf)["anchors"]
        out = torch.empty(B, 300, 6, device="cuda")
        raw = torch.empty(B, 84, A, device="cuda")
        ws.fill_(255)
        checked = 0
        for i, d in enumerate(descs):
            if d.kind == CC_CONV_OP_NONE:
                _run(m, fr, B, Hf, Wf, res, i, i + 1, out, raw)
                continue
            op = _plan_op(d, ws)
            entry = _COVERAGE.setdefault(_launch_key(d), [0, set()])
            entry[0] += 1
            entry[1].add(tag.split(" res")[0] + ("-fp32acc" if precise else ""))
            snap = ws.clone()
            for s in op_outputs(op):
                if not same_slice(s, op.res):
                    sview(ws, s).fill_(float("nan"))
            _run(m, fr, B, Hf, Wf, res, i, i + 1, out, raw)
            torch.cuda.synchronize()
            check_op(op, snap, ws, worst)
            del snap
            checked += 1
        assert checked == sum(r["kind"] in ("conv_gemm", "conv_direct") for r in prof) > 0
        nbytes = ws.numel()
    line = (f"{tag}: {checked} conv ops, workspace {nbytes / 2 ** 20:.0f} MiB, {time.time() - t0:.1f} s; worst "
            + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))
    _REPORT.append(line)
    print(line)


# size res B Hf Wf fp32-accurate
FORWARD_CONFIGS = [pytest.param("c", 640, 32, 640, 640, False, id="c-b32-640"),
                   pytest.param("t", 320, 16, 320, 320, False, id="t-b16-320"),
                   pytest.param("t", 320, 16, 320, 320, True, id="t-b16-320-fp32acc")]


def _same_bits(a, b):
    return torch.equal(a, b) if a.dtype == torch.uint8 else torch.equal(bits(a), bits(b))


@pytest.mark.parametrize("size,res,B,Hf,Wf,precise", FORWARD_CONFIGS)
def test_forward_is_the_ops_and_ignores_stale_workspace(size, res, B, Hf, Wf, precise):
    """Op by op with a device synchronisation after each launch, then three cc_yolo_forward calls with the same frame, out and
    raw pointers (plain launches with programmatic dependent launch, graph capture, graph replay): each gives the output, head
    tap and workspace bytes of the sequence without overlap.  Then forwards on a
    zero-filled and a 0xFF-filled workspace: the same finite output and head tap."""
    t0 = time.time()
    m = _model(size, res, precise, True)
    fr = _frames(B, Hf, Wf)
    A = m.plan_info(B, Hf, Wf)["anchors"]
    out = torch.empty(B, 300, 6, device="cuda")
    raw = torch.empty(B, 84, A, device="cuda")
    W = _Workspace(m, B, Hf, Wf, res)
    with W as ws:
        n = len(_descs(m, B, Hf, Wf, res))
        ws.fill_(255)
        out.fill_(float("nan"))
        raw.fill_(float("nan"))
        for i in range(n):        # one launch at a time: each op starts after the previous one has finished (no overlap)
            _run(m, fr, B, Hf, Wf, res, i, i + 1, out, raw)
            torch.cuda.synchronize()
        want = {"workspace": ws.clone(), "output": out.clone(), "head tap": raw.clone()}
        for call in ("first call (plain launches)", "second call (graph capture)", "third call (graph replay)"):
            out.fill_(float("nan"))
            raw.fill_(float("nan"))
            _forward(m, fr, B, Hf, Wf, res, out, raw)
            torch.cuda.synchronize()
            for name, got in (("workspace", ws), ("output", out), ("head tap", raw)):
                assert _same_bits(got, want[name]), f"{call}: the {name} differs from the op-by-op run"
        del want
        got = []
        for fill in (0, 255):
            ws.fill_(fill)
            W.adopt()
            out.fill_(float("nan"))
            raw.fill_(float("nan"))
            _forward(m, fr, B, Hf, Wf, res, out, raw)
            torch.cuda.synchronize()
            assert torch.isfinite(out).all() and torch.isfinite(raw).all(), f"workspace filled with {fill:#x}: non-finite output"
            got.append((out.clone(), raw.clone()))
        assert _same_bits(got[0][0], got[1][0]) and _same_bits(got[0][1], got[1][1]), \
            "the forward depends on what the workspace held before"
    line = f"whole forward, {size} B {B} {Hf}x{Wf}{' fp32-accurate' if precise else ''}: {n} ops, {time.time() - t0:.1f} s"
    _REPORT.append(line)
    print(line)
