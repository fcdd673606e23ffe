"""yuv420p (I420) frames on the GPU: every path that reads a frame must give, bit for bit, what the bgr24 path gives on
`oracle.yuv.i420_to_bgr(frame)` (cv2's conversion of the same bytes).  Test content is cv2.cvtColor(synthetic BGR,
COLOR_BGR2YUV_I420); the bgr24 side is the oracle's conversion of that YUV, not the original BGR (the round trip is lossy).
Every bar is torch.equal / array_equal."""
import io

import numpy as np
import pytest
import torch

from oracle import yolov9 as o
from oracle.yuv import i420_to_bgr
from clearcam_b200._lib import lib, ptr, stream_ptr
from clearcam_b200.detection.yolov9 import YOLOv9

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")


def _yuv_frames(B, H, W, seed):
    """-> (yuv uint8 [B,H*3/2,W], bgr uint8 [B,H,W,3] = oracle conversion of yuv), CPU tensors."""
    bgr0 = o.synthetic_frames(B, H, W, seed=seed).numpy()
    yuv = np.stack([cv2.cvtColor(np.ascontiguousarray(f), cv2.COLOR_BGR2YUV_I420) for f in bgr0])
    return torch.from_numpy(yuv), torch.from_numpy(i420_to_bgr(yuv))


# ------------------------------------------------------------------------------------------------ letterbox
@pytest.mark.parametrize("shape,res", [((270, 480), 320), ((1080, 1920), 640), ((540, 960), 960), ((334, 518), 256),
                                       ((640, 640), 640)])
def test_letterbox_i420_matches_the_oracle(shape, res):
    yuv, bgr = _yuv_frames(2, shape[0], shape[1], seed=3)
    want = torch.stack([o.preprocess(f, res) for f in bgr])
    m = YOLOv9.__new__(YOLOv9)
    m.res = res
    got = m.preprocess(yuv, pix_fmt="yuv420p").tensor.cpu()
    assert got.shape == want.shape and got.dtype == torch.uint8
    assert torch.equal(got, want)
    one = m.preprocess(yuv[1], pix_fmt="yuv420p").tensor.cpu()          # a single [H*3/2,W] frame
    assert torch.equal(one, want[1])


# ------------------------------------------------------------------------------------------------ detector
_P = {}


def _weights():
    if "c" not in _P:
        fr = o.synthetic_frames(2, 320, 320, seed=9)
        x = torch.stack([o.preprocess(f, 320) for f in fr]).flip(-1).permute(0, 3, 1, 2).float() / 255
        _P["c"] = o.synthetic_weights("c", seed=9, calib=x)
    return _P["c"]


_MODELS = {}


def _model(precise):
    if precise not in _MODELS:
        _MODELS[precise] = YOLOv9("c", 640, weights=_weights(), precise=precise)
    return _MODELS[precise]


@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("H,W", [(1080, 1920), (640, 640)])
def test_detector_i420_equals_bgr_on_the_converted_frames(H, W, precise):
    yuv, bgr = _yuv_frames(4, H, W, seed=11)
    m = _model(precise)
    out_y, raw_y = m.detect_batch(yuv, raw=True, pix_fmt="yuv420p")
    out_b, raw_b = m.detect_batch(bgr, raw=True)
    torch.cuda.synchronize()
    assert torch.equal(raw_y, raw_b)
    assert torch.equal(out_y, out_b)
    assert m.plan_info(4, H, W, pix_fmt="yuv420p")["anchors"] == raw_y.shape[-1]


def test_single_frame_call_and_graph_replay_with_i420():
    yuv, bgr = _yuv_frames(2, 1080, 1920, seed=12)
    m = _model(False)
    want = m(bgr[0].numpy()).numpy()
    for _ in range(3):                       # plain launch, capture, then replay of the captured graph
        got = m(yuv[0], pix_fmt="yuv420p").numpy()
        assert np.array_equal(got, want)
    got = m(yuv[1].numpy(), pix_fmt="yuv420p").numpy()     # same kept buffers, new content
    assert np.array_equal(got, m(bgr[1].numpy()).numpy())
    assert np.array_equal(m(yuv[1].cuda(), pix_fmt="yuv420p").numpy(), m(bgr[1].cuda()).numpy())     # device frame


def test_pipelined_i420_equals_bgr():
    yuv, bgr = _yuv_frames(4, 540, 960, seed=13)
    m = _model(False)
    got = [r.clone() for r in m.detect_pipelined([yuv[:2].pin_memory(), yuv[2:].pin_memory()], pix_fmt="yuv420p")]
    want = [r.clone() for r in m.detect_pipelined([bgr[:2].pin_memory(), bgr[2:].pin_memory()])]
    assert len(got) == 2 and all(torch.equal(a, b) for a, b in zip(got, want))


# ------------------------------------------------------------------------------------------------ crops
_RECTS = [(0, 1, 3, 201, 157), (1, 1719, 881, 1920, 1080), (0, 0, 0, 1920, 1080), (1, 333, 77, 334, 78),
          (0, 1001, 999, 1500, 1080), (1, 0, 1, 113, 700), (0, 1917, 1077, 1920, 1080)]


def test_crops_from_i420_frames_equal_crops_from_the_converted_frames():
    from clearcam_b200.models.objects import ObjectFinder
    yuv, bgr = _yuv_frames(2, 1080, 1920, seed=14)
    of = ObjectFinder()
    got = of.preprocess_device(yuv.cuda(), _RECTS, pix_fmt="yuv420p").tensor
    want = of.preprocess_device(bgr.cuda(), _RECTS).tensor
    assert torch.equal(got, want)
    one = of.preprocess_device(yuv[1], [r[1:] for r in _RECTS], size=37, pix_fmt="yuv420p").tensor      # [H*3/2,W], tail path
    assert torch.equal(one, of.preprocess_device(bgr[1], [r[1:] for r in _RECTS], size=37).tensor)


def test_embed_crops_from_i420_frames():
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    yuv, bgr = _yuv_frames(2, 1080, 1920, seed=15)
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    got = of.embed_crops(yuv.cuda(), _RECTS, pix_fmt="yuv420p").tensor
    want = of.embed_crops(bgr.cuda(), _RECTS).tensor
    assert got.shape == (len(_RECTS), of.model.embed_dim) and torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ ingest
def test_mailboxes_of_mixed_formats_feed_the_batched_detector():
    """Two yuv420p 1080p cameras and one bgr24 720p camera through FrameMailbox -> CameraBatch.step_mailboxes: rows and
    tracker targets equal `step` on the converted BGR frames with fresh trackers."""
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.ingest import FrameMailbox
    m = _model(False)
    boxes = {"y0": FrameMailbox(1080, 1920, pix_fmt="yuv420p"), "y1": FrameMailbox(1080, 1920, pix_fmt="yuv420p"),
             "b": FrameMailbox(720, 1280)}
    cb_yuv, cb_bgr = CameraBatch(m), CameraBatch(m)
    n_dets = 0
    for t in range(3):
        yuv, conv = _yuv_frames(2, 1080, 1920, seed=20 + t)
        b720 = o.synthetic_frames(1, 720, 1280, seed=30 + t)[0]
        for i in range(2):
            assert boxes[f"y{i}"].fill(io.BytesIO(yuv[i].numpy().tobytes()))
        assert boxes["b"].fill(io.BytesIO(b720.numpy().tobytes()))
        got = cb_yuv.step_mailboxes(boxes)
        want = cb_bgr.step({"y0": conv[0].numpy(), "y1": conv[1].numpy(), "b": b720.numpy()})
        assert set(got) == set(want) == {"y0", "y1", "b"}
        assert cb_yuv.cams["y0"].pix_fmt == "yuv420p" and cb_yuv.cams["b"].pix_fmt == "bgr24"
        assert tuple(cb_yuv.device_frame("y1").shape) == (1620, 1920)
        assert torch.equal(cb_yuv.device_frame("y1").cpu(), yuv[1])
        for name in want:
            assert np.array_equal(got[name].rows, want[name].rows), name
            key = lambda tr: (tuple(tr.tlwh), float(tr.score), int(tr.class_id), int(tr.track_id), int(tr.tracklet_len))   # noqa: E731
            assert [key(x) for x in got[name].targets] == [key(x) for x in want[name].targets], name
            assert np.array_equal(got[name].preds, want[name].preds), name
            n_dets += int((got[name].rows[:, 4] > 0).sum())
    assert n_dets > 0


# ------------------------------------------------------------------------------------------------ errors
def test_bad_frames_raise_value_error_in_python():
    from clearcam_b200.models.objects import ObjectFinder
    m = _model(False)
    for f in [torch.zeros(2, 1621, 1920, dtype=torch.uint8), torch.zeros(2, 1620, 1919, dtype=torch.uint8),
              torch.zeros(2, 1620, 1920, dtype=torch.float32), torch.zeros(2, 1080, 1920, 3, dtype=torch.uint8)]:
        with pytest.raises(ValueError):
            m.detect_batch(f.cuda(), pix_fmt="yuv420p")
        with pytest.raises(ValueError):
            ObjectFinder().preprocess_device(f.cuda(), [(0, 0, 0, 8, 8)], pix_fmt="yuv420p")
    with pytest.raises(ValueError):
        m(torch.zeros(1621, 1920, dtype=torch.uint8), pix_fmt="yuv420p")


def test_library_rejects_odd_i420_sizes_and_unknown_formats():
    L = lib()
    m = _model(False)
    buf = torch.zeros(2 * 1622 * 1921, dtype=torch.uint8, device="cuda")
    out = torch.empty(2, 300, 6, device="cuda")
    for fmt, H, W, words in [(2, 1081, 1920, "even"), (2, 1080, 1921, "even"), (7, 1080, 1920, "unknown frame format"),
                             (-1, 1080, 1920, "unknown frame format")]:
        rc = L.cc_yolo_forward(m._h, ptr(buf), fmt, 2, H, W, 640, ptr(out), None, stream_ptr())
        assert rc < 0 and words in L.cc_last_error().decode(), (fmt, H, W)
        rc = L.cc_letterbox(ptr(buf), fmt, 2, H, W, 640, None, None, None, None)
        assert rc < 0 and words in L.cc_last_error().decode(), (fmt, H, W)
    rects = np.array([[0, 0, 0, 8, 8]], np.int32)
    crops = torch.empty(1, 3, 224, 224, device="cuda")
    for fmt, H, W, words in [(2, 1081, 1920, "even"), (2, 1080, 1921, "even"), (3, 1080, 1920, "unknown source format")]:
        rc = L.cc_clip_preprocess(ptr(buf), 1, H, W, rects.ctypes.data, 1, 224, fmt, ptr(crops), stream_ptr())
        assert rc < 0 and words in L.cc_last_error().decode(), (fmt, H, W)
    torch.cuda.synchronize()
