"""Every GEMM launch of the CLIP and face-embedder plans, in place, at the benchmark's and the bucket batch sizes.

The checks are those of tests/test_plan_convs_gpu.py (Slice / sview, check_values, check_stray, check_op); this file only
adapts them to the two plans.  Each plan runs op by op on its own buffers (cc_clip_run_ops, cc_face_run_ops) in a workspace
the test owns and fills with 0xFF bytes.  Before each GEMM op the whole workspace is saved and the op's output is filled with
NaN (unless it is also the op's residual); the op then runs alone, and:

  (a) images 0..REPS-1 of its output match a float64 GEMM / conv of the operands as stored, with the weights, bias, PReLU
      border-class table and slopes read through their device pointers.  A CLIP linear runs over B * L token rows as a 1x1
      conv of N = H = 1; its images are the blocks of L rows (1 row for the pooled projections and the face linear);
  (b) the batch holds copies of REPS distinct inputs, so image b of every output equals image b % REPS bit for bit;
  (c) every output is finite;
  (d) every workspace byte the op changed lies in its output.  The patch embedding writes tokens 1..L-1 of each image of the
      fp32 [B, L, W] residual stream (out_ns = L), so token 0 and every other row of the stream must keep its bytes.

Block 0's subsample shortcut (MaxPool2d(1, 2) as a centre-tap conv with identity weights) must equal the strided input bit
for bit.  Then the whole forward, per network: the ops one at a time with a device synchronisation after each, then one
cc_clip_encode_* / cc_face_embed call with the same pointers gives the same output and workspace bytes (consecutive GEMMs
overlap through programmatic dependent launch there), and forwards on a zero-filled and a 0xFF-filled workspace give the
same finite output.  The distinct launch configurations are printed."""
import collections
import ctypes
import time

import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200._lib import CCError, CC_CONV_OP_GEMM, CC_CONV_OP_NONE, cc_conv_op, check, lib, ptr, stream_ptr

import test_plan_convs_gpu as tp

pytestmark = pytest.mark.gpu

REPS = tp.REPS
CLIP_GEMMS = {"patch_embed", "qkv", "out_proj", "mlp_fc", "mlp_proj", "proj", "text_projection"}
FACE_GEMMS = 1 + 24 * 2 + 4 + 1          # stem, two convs per block, four shortcut convs, the linear
_MODELS = {}
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


# ------------------------------------------------------------------------------------------------ the plans as adapters
class _Plan:
    """One cached plan of a handle: its ops' descriptors, a run of ops [first, last), the whole forward, and the workspace
    calls.  Subclasses set `tag`, `B`, `inp`, `out` and the entry points."""

    def descs(self):
        n = self._op_conv(0, None)
        check(min(n, 0), "op_conv")
        out = []
        for i in range(n):
            d = cc_conv_op()
            check(min(self._op_conv(i, ctypes.byref(d)), 0), "op_conv")
            out.append(d)
        return out

    def rows(self, d):
        """Rows per image of a row GEMM (N = H = 1: a linear over the batch's rows), else 0."""
        return d.in_.W // self.B if d.in_.N == 1 and d.in_.H == 1 else 0


class _Clip(_Plan):
    def __init__(self, m, text, B, inp):
        self.m, self.text, self.B, self.inp = m, int(text), B, inp
        self.out = torch.empty(B, m.embed_dim, device="cuda")
        self.tag = f"{m.arch} {'text' if text else 'image'} B {B}"

    def _op_conv(self, i, out):
        return lib().cc_clip_op_conv(self.m._h, self.text, self.B, i, out)

    def run(self, first, last):
        check(lib().cc_clip_run_ops(self.m._h, self.text, ptr(self.inp), self.B, first, last, ptr(self.out), 0, stream_ptr()),
              "cc_clip_run_ops")

    def forward(self):
        fn = "cc_clip_encode_text" if self.text else "cc_clip_encode_image"
        check(getattr(lib(), fn)(self.m._h, ptr(self.inp), self.B, ptr(self.out), 0, stream_ptr()), fn)

    def ws_bytes(self):
        n = ctypes.c_size_t()
        check(lib().cc_clip_workspace_bytes(self.m._h, self.text, self.B, ctypes.byref(n)), "cc_clip_workspace_bytes")
        return n.value

    def set_ws(self, ws):
        check(lib().cc_clip_set_workspace(self.m._h, ptr(ws), 0 if ws is None else ws.numel()), "cc_clip_set_workspace")

    def gemm_names(self):
        prof, _ = self.m.profile(**({"ids": self.inp} if self.text else {"x": self.inp}))
        return [r["name"] for r in prof]


class _Face(_Plan):
    def __init__(self, m, B, faces):
        self.m, self.B, self.inp = m, B, faces
        self.out = torch.empty(B, 512, device="cuda")
        self.tag = f"AdaFace B {B}"

    def _op_conv(self, i, out):
        return lib().cc_face_op_conv(self.m._h, self.B, i, out)

    def run(self, first, last):
        check(lib().cc_face_run_ops(self.m._h, ptr(self.inp), self.B, first, last, ptr(self.out), stream_ptr()), "cc_face_run_ops")

    def forward(self):
        check(lib().cc_face_embed(self.m._h, ptr(self.inp), self.B, ptr(self.out), 0, stream_ptr()), "cc_face_embed")

    def ws_bytes(self):
        n = ctypes.c_size_t()
        check(lib().cc_face_workspace_bytes(self.m._h, self.B, ctypes.byref(n)), "cc_face_workspace_bytes")
        return n.value

    def set_ws(self, ws):
        check(lib().cc_face_set_workspace(self.m._h, ptr(ws), 0 if ws is None else ws.numel()), "cc_face_set_workspace")


def _clip_model(arch):
    from oracle import clip as oc
    from clearcam_b200.models.objects import OpenCLIP
    if arch not in _MODELS:
        _MODELS.clear()           # one CLIP model at a time: ViT-L/14's weights are 1.7 GB of fp32 on the host
        _MODELS[arch] = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS[arch], seed=7), arch=arch)
    return _MODELS[arch]


def _face_model():
    from oracle import adaface as oa
    from clearcam_b200.models.adaface import ADAFACE
    if "face" not in _MODELS:
        _MODELS["face"] = ADAFACE(oa.synthetic_weights(seed=5))
    return _MODELS["face"]


def _clip_plan(arch, text, B):
    from oracle import clip as oc
    m = _clip_model(arch)
    if text:
        g = torch.Generator().manual_seed(9)
        ids = torch.zeros(REPS, m.ctx, dtype=torch.int32)
        for r, n in enumerate((3, 17, m.ctx - 2)):        # a short, a middle and a full-length prompt
            ids[r, :n + 2] = torch.cat([torch.tensor([49406]), torch.randint(1, 49406, (n,), generator=g), torch.tensor([49407])])
        inp = ids[torch.arange(B) % REPS].contiguous().cuda()
    else:
        inp = oc.synthetic_images(REPS, m.image_size, seed=5)[torch.arange(B) % REPS].contiguous().cuda()
    return _Clip(m, text, B, inp)


def _face_plan(B):
    from oracle import adaface as oa
    return _Face(_face_model(), B, oa.synthetic_faces(REPS, seed=21)[torch.arange(B) % REPS].contiguous().cuda())


class _Workspace:
    """A caller-owned workspace for plan p, handed back to the library on exit."""

    def __init__(self, p):
        self.p = p

    def __enter__(self):
        self.ws = torch.empty((self.p.ws_bytes() + 255) // 256 * 256, dtype=torch.uint8, device="cuda")
        self.adopt()
        return self.ws

    def adopt(self):
        """(Re)hand the workspace over: the handle drops its plans, so the next call builds them again."""
        self.p.set_ws(self.ws)

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.p.set_ws(None)
        del self.ws


# ------------------------------------------------------------------------------------------------ every GEMM, in place
#        plan     arch        text   B
CONFIGS = [pytest.param("clip", "ViT-B/32", False, 256, id="vitb32-image-b256"),
           pytest.param("clip", "ViT-B/32", False, 3, id="vitb32-image-b3"),
           pytest.param("clip", "ViT-B/32", True, 256, id="vitb32-text-b256"),
           pytest.param("clip", "ViT-B/32", True, 1, id="vitb32-text-b1"),
           pytest.param("clip", "ViT-L/14", False, 256, id="vitl14-image-b256"),
           pytest.param("clip", "ViT-L/14", False, 3, id="vitl14-image-b3"),
           pytest.param("clip", "ViT-L/14", True, 256, id="vitl14-text-b256"),
           pytest.param("clip", "ViT-L/14", True, 1, id="vitl14-text-b1"),
           pytest.param("face", None, False, 1, id="face-b1"),
           pytest.param("face", None, False, 12, id="face-b12"),
           pytest.param("face", None, False, 208, id="face-b208"),
           pytest.param("face", None, False, 256, id="face-b256")]


def _plan(kind, arch, text, B):
    return _clip_plan(arch, text, B) if kind == "clip" else _face_plan(B)


@pytest.mark.parametrize("kind,arch,text,B", CONFIGS)
def test_every_gemm_launch_in_place(kind, arch, text, B):
    t0 = time.time()
    p = _plan(kind, arch, text, B)
    worst = {}
    with _Workspace(p) as ws:
        descs = p.descs()
        names = [d.name.decode() for d in descs]
        if kind == "clip":
            assert names == p.gemm_names()
            want = sum(n in CLIP_GEMMS for n in names)
        else:
            want = FACE_GEMMS
        ws.fill_(255)
        checked = 0
        for i, d in enumerate(descs):
            name = names[i]
            if d.kind == CC_CONV_OP_NONE:
                assert name not in CLIP_GEMMS and (kind == "clip" or name in ("pack", "l2norm")), name
                p.run(i, i + 1)
                continue
            op = tp._plan_op(d, ws)
            entry = _COVERAGE.setdefault(tp._launch_key(d), [0, set()])
            entry[0] += 1
            entry[1].add(p.tag.split(" B ")[0])
            snap = ws.clone()
            for s in tp.op_outputs(op):
                if not tp.same_slice(s, op.res):
                    tp.sview(ws, s).fill_(float("nan"))
            p.run(i, i + 1)
            torch.cuda.synchronize()
            tp.check_op(op, snap, ws, worst, p.rows(d))
            if name == "body.0.sc":
                want_sc = tp.sview(snap, op.in_)[:, ::2, ::2]
                assert torch.equal(tp.bits(tp.sview(ws, op.out)), tp.bits(want_sc)), \
                    "body.0.sc: the subsample shortcut differs from the strided input"
            del snap
            checked += 1
        assert checked == want > 0, (checked, want)
        nbytes = ws.numel()
    line = (f"{p.tag}: {checked} GEMM ops, workspace {nbytes / 2 ** 20:.0f} MiB, {time.time() - t0:.1f} s; worst "
            + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))
    _REPORT.append(line)
    print(line)


# ------------------------------------------------------------------------------------------------ whole forwards
FORWARD_CONFIGS = [pytest.param("clip", "ViT-B/32", False, 256, id="vitb32-image-b256"),
                   pytest.param("clip", "ViT-B/32", True, 256, id="vitb32-text-b256"),
                   pytest.param("face", None, False, 208, id="face-b208")]


@pytest.mark.parametrize("kind,arch,text,B", FORWARD_CONFIGS)
def test_forward_is_the_ops_and_ignores_stale_workspace(kind, arch, text, B):
    """Op by op with a device synchronisation after each launch, then one forward with the same input and output pointers:
    the same output and workspace bytes.  Then forwards on a zero-filled and a 0xFF-filled workspace: the same finite
    output."""
    t0 = time.time()
    p = _plan(kind, arch, text, B)
    W = _Workspace(p)
    with W as ws:
        n = len(p.descs())
        ws.fill_(255)
        p.out.fill_(float("nan"))
        for i in range(n):        # one launch at a time: each op starts after the previous one has finished (no overlap)
            p.run(i, i + 1)
            torch.cuda.synchronize()
        want_ws, want_out = ws.clone(), p.out.clone()
        p.out.fill_(float("nan"))
        p.forward()
        torch.cuda.synchronize()
        assert torch.equal(ws, want_ws), f"the forward's workspace differs from the op-by-op run at byte {tp._first_diff(ws, want_ws)}"
        assert torch.equal(tp.bits(p.out), tp.bits(want_out)), "the forward's output differs from the op-by-op run"
        del want_ws
        got = []
        for fill in (0, 255):
            ws.fill_(fill)
            W.adopt()
            p.out.fill_(float("nan"))
            p.forward()
            torch.cuda.synchronize()
            assert torch.isfinite(p.out).all(), f"workspace filled with {fill:#x}: non-finite output"
            got.append(p.out.clone())
        assert torch.equal(tp.bits(got[0]), tp.bits(got[1])), "the forward depends on what the workspace held before"
        assert torch.equal(tp.bits(got[0]), tp.bits(want_out)), "the forward on a fresh workspace differs from the op-by-op run"
    line = f"whole forward, {p.tag}: {n} ops, {time.time() - t0:.1f} s"
    _REPORT.append(line)
    print(line)


# ------------------------------------------------------------------------------------------------ cc_conv with out_ns
def test_cc_conv_pitched_fp32_output_matches_float64():
    """The patch embedding's form through cc_conv: a bf16 [B * Pn, K] GEMM into fp32 tokens 1..L-1 of a [B, L, W] stream
    (one row past the buffer's start, out_ns = L), adding the stream in place as the residual.  Checked against float64;
    token 0 of every image keeps its sentinel.  A pitch shorter than the image is refused."""
    from test_conv_gpu import F32_BAR, F32_REL
    B, Pn, K, W = 5, 49, 3072, 768
    L = Pn + 1
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(B, 1, Pn, K, generator=g)).to(torch.bfloat16).cuda()
    w = (torch.randn(W, 1, 1, K, generator=g) * K ** -0.5).to(torch.bfloat16).cuda()
    stream = torch.randn(B, L, W, generator=g).cuda()
    stream[:, 0] = 1234.5
    before = stream.clone()
    out = stream[:, 1:].unsqueeze(1)                    # [B, 1, Pn, W], images L rows apart
    ops.conv2d(x, 0, K, w, None, 1, 1, out, 0, W, res=out, out_ns=L)
    torch.cuda.synchronize()
    assert torch.equal(stream[:, 0], before[:, 0]), "token 0 changed"
    z, y, mag = tp.ref64(x, w, None, 1, 1, 1, 0, before[:, 1:].unsqueeze(1))
    err = (stream[:, 1:].unsqueeze(1).double() - y).abs()
    assert (err / (F32_BAR * mag)).max().item() <= 1.0
    assert (err / y.abs().clamp(min=1.0)).max().item() < F32_REL
    short = cc_conv_op(kind=CC_CONV_OP_GEMM, in_=ops._slice(x, 0, K), out=ops._slice(out, 0, W), w=ptr(w), k=1, stride=1, groups=1,
                       out_ns=Pn - 1)
    with pytest.raises(CCError, match=r"cc_conv: out_ns=48 pixels per image is less than the output's 1x49"):
        check(lib().cc_conv(ctypes.byref(short), stream_ptr()), "cc_conv")
    assert torch.equal(stream[:, 0], before[:, 0])
