"""yuv420p (I420) frames on the host side: the conversion oracle against OpenCV, the yuv420p mailbox, and CameraBatch's
grouping and validation of mixed-format cameras (with a stand-in detector; the GPU path is in test_yuv_gpu.py)."""
import io
import os

import numpy as np
import pytest
import torch

from clearcam_b200.cameras import CameraBatch
from clearcam_b200.ingest import FrameMailbox
from oracle.yuv import i420_to_bgr, i420_to_rgb

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "yuv420_cv2.npz")


def _even_shapes(n, seed=0):
    rng = np.random.default_rng(seed)
    shapes = [(2, 2), (1080, 1920), (1078, 1918)]
    while len(shapes) < n:
        shapes.append((2 * int(rng.integers(1, 541)), 2 * int(rng.integers(1, 961))))
    return shapes


# ------------------------------------------------------------------------------------------------ the conversion
def test_oracle_is_bit_exact_with_cv2_on_random_planes():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    for h, w in _even_shapes(32):
        yuv = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
        assert np.array_equal(i420_to_bgr(yuv), cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_I420)), (h, w)
        assert np.array_equal(i420_to_rgb(yuv), cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_I420)), (h, w)


def test_oracle_matches_the_stored_cv2_output_including_extreme_planes():
    z = np.load(GOLDEN)
    n = len([k for k in z.files if k.startswith("yuv")])
    assert n >= 5
    for k in range(n):
        yuv, want = z[f"yuv{k}"], z[f"bgr{k}"]
        assert np.array_equal(i420_to_bgr(yuv), want), k
        assert np.array_equal(i420_to_rgb(yuv), want[..., ::-1]), k
        got_t = i420_to_bgr(torch.from_numpy(yuv)[None].repeat(2, 1, 1))          # torch, batched
        assert torch.equal(got_t, torch.from_numpy(want)[None].repeat(2, 1, 1, 1)), k
    ext = z[f"bgr{n - 1}"]
    assert ext.min() == 0 and ext.max() == 255                                     # both saturation ends are exercised


def test_oracle_rejects_odd_sizes():
    with pytest.raises(ValueError):
        i420_to_bgr(np.zeros((4, 6), np.uint8))        # 4 rows: H = 8/3
    with pytest.raises(ValueError):
        i420_to_bgr(np.zeros((6, 5), np.uint8))


# ------------------------------------------------------------------------------------------------ ingest
H, W = 24, 40


def _yuv(k):
    rng = np.random.default_rng(k)
    return rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)


def test_yuv420p_mailbox_reads_whole_frames_from_a_chunked_stream():
    class Dribble(io.RawIOBase):
        def __init__(self, data): self.data, self.pos = data, 0
        def readable(self): return True
        def readinto(self, b):
            n = min(len(b), 333, len(self.data) - self.pos)
            b[:n] = self.data[self.pos:self.pos + n]
            self.pos += n
            return n
    mb = FrameMailbox(H, W, pin=False, pix_fmt="yuv420p")
    assert mb.frame_bytes == H * W * 3 // 2 and mb.pix_fmt == "yuv420p"
    s = Dribble(b"".join(_yuv(k).tobytes() for k in range(3)) + _yuv(3).tobytes()[:100])
    assert mb.fill(s) and mb.frame_num == 0
    n, f = mb.latest()
    assert n == 0 and f.shape == (H * 3 // 2, W) and np.array_equal(f.numpy(), _yuv(0))
    assert mb.fill(s) and mb.fill(s)
    assert np.array_equal(f.numpy(), _yuv(0))                   # the held frame stays intact
    n, g = mb.latest(last_seen=0)
    assert n == 2 and np.array_equal(g.numpy(), _yuv(2))
    assert not mb.fill(s) and mb.frame_num == 2
    assert FrameMailbox(H, W, pin=False).frame_bytes == H * W * 3          # bgr24 stays the default


def test_yuv420p_mailbox_rejects_odd_sizes_and_unknown_formats():
    for h, w in [(25, 40), (24, 41)]:
        with pytest.raises(ValueError):
            FrameMailbox(h, w, pin=False, pix_fmt="yuv420p")
    with pytest.raises(ValueError):
        FrameMailbox(H, W, pin=False, pix_fmt="nv12")


# ------------------------------------------------------------------------------------------------ camera batching
class FakeDetector:
    """Records (shape, pix_fmt) per call and returns one box whose x1 is the batch row's mean byte."""
    def __init__(self):
        self.calls = []

    def detect_batch(self, frames, pix_fmt="bgr24"):
        self.calls.append((tuple(frames.shape), pix_fmt))
        B = frames.shape[0]
        out = torch.zeros(B, 300, 6)
        out[:, 0, 0] = frames.reshape(B, -1).float().mean(1)
        out[:, 0, 2], out[:, 0, 3], out[:, 0, 4] = 200, 200, 0.9
        return out


def test_camera_batch_groups_mixed_formats():
    det = FakeDetector()
    cb = CameraBatch(det)
    for i in range(3):
        cb.add_camera(f"y{i}", pix_fmt="yuv420p")
    frames = {f"y{i}": np.full((H * 3 // 2, W), 10 * i + 1, np.uint8) for i in range(3)}
    frames["b"] = np.full((H, W, 3), 77, np.uint8)                # a bgr24 camera of the same picture size
    frames["y_small"] = np.full((12 * 3 // 2, 20), 5, np.uint8)
    cb.add_camera("y_small", pix_fmt="yuv420p")
    cb.add_camera("b")
    g = CameraBatch.group_by_shape(frames, {n: cb.cams[n].pix_fmt for n in frames})
    assert g == {(H, W, "|u1", "yuv420p"): ["y0", "y1", "y2"], (H, W, "|u1", "bgr24"): ["b"],
                 (12, 20, "|u1", "yuv420p"): ["y_small"]}
    res = cb.step(frames)
    assert sorted(det.calls) == sorted([((4, H * 3 // 2, W), "yuv420p"), ((1, H, W, 3), "bgr24"), ((1, 18, 20), "yuv420p")])
    for name, v in [("y0", 1), ("y1", 11), ("y2", 21), ("b", 77), ("y_small", 5)]:
        assert res[name].rows[0, 0] == v and len(res[name].targets) == 1
    assert tuple(cb.device_frame("y1").shape) == (H * 3 // 2, W) and int(cb.device_frame("y1")[0, 0]) == 11
    assert tuple(cb.device_frame("b").shape) == (H, W, 3)


def test_camera_batch_rejects_frames_that_do_not_match_their_format():
    cb = CameraBatch(FakeDetector())
    cb.add_camera("y", pix_fmt="yuv420p")
    cb.add_camera("b")
    bad = [("y", np.zeros((H, W, 3), np.uint8)),                  # a bgr24 frame on a yuv420p camera
           ("y", np.zeros((H * 3 // 2 + 1, W), np.uint8)),         # odd height (rows not 3 * H/2)
           ("y", np.zeros((H * 3 // 2, W + 1), np.uint8)),         # odd width
           ("y", np.zeros((H * 3 // 2, W), np.float32)),           # not uint8
           ("b", np.zeros((H * 3 // 2, W), np.uint8))]             # a yuv420p frame on a bgr24 camera
    for name, f in bad:
        with pytest.raises(ValueError):
            cb.step({name: f})
    with pytest.raises(ValueError):
        cb.add_camera("z", pix_fmt="rgb24")


def test_step_mailboxes_takes_a_new_cameras_format_from_its_mailbox():
    det = FakeDetector()
    cb = CameraBatch(det)
    boxes = {"y": FrameMailbox(H, W, pin=False, pix_fmt="yuv420p"), "b": FrameMailbox(H, W, pin=False)}
    boxes["y"].fill(io.BytesIO(_yuv(4).tobytes()))
    boxes["b"].fill(io.BytesIO(np.full((H, W, 3), 9, np.uint8).tobytes()))
    res = cb.step_mailboxes(boxes)
    assert cb.cams["y"].pix_fmt == "yuv420p" and cb.cams["b"].pix_fmt == "bgr24"
    assert abs(res["y"].rows[0, 0] - _yuv(4).mean()) < 1e-3 and res["b"].rows[0, 0] == 9
    assert sorted(det.calls) == sorted([((1, H * 3 // 2, W), "yuv420p"), ((1, H, W, 3), "bgr24")])


# ------------------------------------------------------------------------------------------------ Python API checks
def test_detector_and_crop_calls_reject_bad_yuv420p_frames_before_the_library():
    """The shape / dtype checks run before any device work, so they hold on a machine without a GPU too."""
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.models.objects import ObjectFinder
    m = YOLOv9.__new__(YOLOv9)
    m.res = 320
    bad = [np.zeros((2, 25, 40), np.uint8),            # rows not a multiple of 3: odd height
           np.zeros((2, 24, 41), np.uint8),            # odd width
           np.zeros((2, 24, 40), np.float32),          # not uint8
           np.zeros((2, 24, 40, 3), np.uint8)]         # a bgr24 batch
    for f in bad:
        with pytest.raises(ValueError):
            m.detect_batch(f, pix_fmt="yuv420p")
        with pytest.raises(ValueError):
            m.preprocess(f, pix_fmt="yuv420p")
        with pytest.raises(ValueError):
            ObjectFinder().preprocess_device(f, [(0, 0, 0, 4, 4)], pix_fmt="yuv420p")
    with pytest.raises(ValueError):
        m(np.zeros((25, 40), np.uint8), pix_fmt="yuv420p")
    with pytest.raises(ValueError):
        m.detect_batch(np.zeros((2, 24, 40), np.uint8), pix_fmt="i420")
