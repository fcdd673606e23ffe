"""The plan cache and the workspace of the detector, CLIP and AdaFace handles (PlanCache in csrc/cc_common.h).

* Eviction: 17 distinct batch sizes over one workspace, so the least recently used plan (B = 1) is dropped by the cache's
  bound and not by a regrown workspace; run again, it gives bit-equal outputs.
* A caller-owned workspace sized by cc_*_workspace_bytes for the largest batch gives the outputs of the library-owned one;
  a larger batch that does not fit raises CCError before anything is launched; NULL returns to the library-owned workspace.
* A workspace that is not 256-byte aligned is refused.
"""
import ctypes

import pytest
import torch

from clearcam_b200._lib import CCError, check, lib, ptr, stream_ptr
from clearcam_b200.detection.yolov9 import YOLOv9
from clearcam_b200.models.adaface import ADAFACE
from clearcam_b200.models.objects import OpenCLIP
from clearcam_b200.pixfmt import CC_FRAME_BGR_U8
from oracle import adaface as oa
from oracle import clip as oc
from oracle import yolov9 as o

pytestmark = pytest.mark.gpu

MAX_PLANS = 16
NB = MAX_PLANS + 1                  # batch sizes 1..NB: one more than the cache holds
H, W, RES = 96, 128, 128            # detector frames and resolution


class Net:
    """One handle, its inputs for batches of 1..NB, and its entry points called directly with exactly B rows."""

    def __init__(self, name, model, x, dim, forward, ws_bytes, set_ws):
        self.name, self.model, self.x, self.dim = name, model, x, dim
        self._forward, self._ws_bytes, self._set_ws = forward, ws_bytes, set_ws

    def run(self, B):
        out = torch.full((B, *self.dim), float("nan"), device="cuda")
        check(self._forward(self.model._h, self.x[:B], B, out), f"{self.name} forward")
        torch.cuda.synchronize()
        return out

    def workspace_bytes(self, B):
        n = ctypes.c_size_t()
        check(self._ws_bytes(self.model._h, B, ctypes.byref(n)), f"{self.name} workspace_bytes")
        return n.value

    def set_workspace(self, p, n):
        return self._set_ws(self.model._h, p, n)


def _yolo():
    base = o.synthetic_frames(4, H, W, seed=3)
    pre = torch.stack([o.preprocess(base[i], RES) for i in range(2)])
    m = YOLOv9("t", RES, weights=o.synthetic_weights("t", seed=3, calib=pre.flip(-1).permute(0, 3, 1, 2).float() / 255))
    L = lib()
    return Net("yolo", m, base[torch.arange(NB) % 4].contiguous().cuda(), (300, 6),
               lambda h, x, B, out: L.cc_yolo_forward(h, ptr(x), CC_FRAME_BGR_U8, B, H, W, RES, ptr(out), None, stream_ptr()),
               lambda h, B, n: L.cc_yolo_workspace_bytes(h, CC_FRAME_BGR_U8, B, H, W, RES, n), L.cc_yolo_set_workspace)


def _clip():
    cfg = oc.CONFIGS["ViT-tiny"]
    m = OpenCLIP(weights=oc.synthetic_weights(cfg, seed=3), arch="ViT-tiny")
    L = lib()
    return Net("clip", m, oc.synthetic_images(NB, cfg.image_size, seed=5).cuda(), (cfg.embed_dim,),
               lambda h, x, B, out: L.cc_clip_encode_image(h, ptr(x), B, ptr(out), 0, stream_ptr()),
               lambda h, B, n: L.cc_clip_workspace_bytes(h, 0, B, n), L.cc_clip_set_workspace)


def _face():
    m = ADAFACE(oa.synthetic_weights(seed=5))
    L = lib()
    return Net("face", m, oa.synthetic_faces(NB, seed=21).cuda(), (512,),
               lambda h, x, B, out: L.cc_face_embed(h, ptr(x), B, ptr(out), 0, stream_ptr()),
               L.cc_face_workspace_bytes, L.cc_face_set_workspace)


@pytest.fixture(scope="module", params=["yolo", "clip", "face"])
def net(request):
    return {"yolo": _yolo, "clip": _clip, "face": _face}[request.param]()


def test_evicted_plan_is_rebuilt_bit_equal(net):
    # Every plan must be built against one workspace generation, or a regrown workspace drops the older plans before the
    # cache is full.  B = NB runs first and sizes the library-owned workspace for all: no smaller batch needs more.
    need = [net.workspace_bytes(B) for B in range(1, NB + 1)]
    assert max(need) == need[-1]
    net.run(NB)
    first = net.run(1)
    assert not first.isnan().any()
    net.run(NB)                             # B = 1 is now the least recently used plan
    for B in range(2, NB):                  # the plan of B = NB - 1 is the 17th: building it drops B = 1's
        net.run(B)
    assert torch.equal(net.run(1), first)


def test_caller_owned_workspace(net):
    sizes = (1, 5, 8)
    want = {B: net.run(B) for B in sizes}
    n = net.workspace_bytes(max(sizes))
    assert n > 0 and net.workspace_bytes(NB) > n
    ws = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert ws.data_ptr() % 256 == 0
    check(net.set_workspace(ptr(ws), n), f"{net.name} set_workspace")
    try:
        for B in sizes:
            assert torch.equal(net.run(B), want[B]), f"B={B} on the caller-owned workspace"
        out = torch.full((NB, *net.dim), float("nan"), device="cuda")
        with pytest.raises(CCError, match="workspace too small"):
            check(net._forward(net.model._h, net.x, NB, out), f"{net.name} forward")
        torch.cuda.synchronize()
        assert out.isnan().all(), "a refused call wrote its output"
    finally:
        check(net.set_workspace(None, 0), f"{net.name} set_workspace(NULL)")
    del ws
    for B in sizes + (NB,):
        got = net.run(B)
        assert not got.isnan().any()
        if B in want:
            assert torch.equal(got, want[B]), f"B={B} back on the library-owned workspace"


def test_misaligned_workspace_is_refused(net):
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    for off in (4, 128):
        assert net.set_workspace(ctypes.c_void_p(ws.data_ptr() + off), ws.numel() - off) != 0
        assert b"256-byte aligned" in lib().cc_last_error()
    assert not net.run(2).isnan().any()     # the refusal left the library-owned workspace in place
