"""Frames of different shapes and formats in one detector batch, host side: the net-shape key against the oracle's letterbox
arithmetic, and CameraBatch's merging of cameras by net shape with a stand-in detector.  The GPU side is in
test_mixed_batch_gpu.py."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import yolov9 as o
from clearcam_b200._lib import CC_MAX_FRAMES
from clearcam_b200.cameras import CameraBatch
from clearcam_b200.detection.yolov9 import net_shape

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle_net(H, W, res):
    new_w, new_h, px, py = o.letterbox_params(H, W, res)
    return (-(-(new_h + 2 * py) // 32) * 32, -(-(new_w + 2 * px) // 32) * 32)


def test_max_frames_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "clearcam_b200.h")).read()
    assert int(re.search(r"#define CC_MAX_FRAMES (\d+)", hdr).group(1)) == CC_MAX_FRAMES >= 128


def test_net_shape_equals_the_oracle_extent_rounded_up():
    rng = np.random.default_rng(0)
    n = 0
    for res in (320, 640, 960, 1280):
        for _ in range(90):
            H, W = (int(v) for v in rng.integers(64, 4097, 2))
            assert net_shape(H, W, res) == _oracle_net(H, W, res), (H, W, res)
            He, We = H & ~1, W & ~1
            assert net_shape(He, We, res, "yuv420p") == _oracle_net(He, We, res), (He, We, res)
            n += 1
    assert n >= 300
    fleet = [(720, 1280), (1080, 1920), (1440, 2560), (2160, 3840)]
    for fmt in ("bgr24", "yuv420p"):
        assert {net_shape(H, W, 640, fmt) for H, W in fleet} == {(384, 640)}
        assert {net_shape(H, W, 1280, fmt) for H, W in fleet} == {(736, 1280)}
    # reference extents 511 and 512: one net shape, with the zero row below the odd one
    assert [o.letterbox_params(H, 640, 640)[1] + 2 * o.letterbox_params(H, 640, 640)[3] for H in (481, 482)] == [511, 512]
    assert net_shape(481, 640, 640) == net_shape(482, 640, 640) == (512, 640)
    with pytest.raises(ValueError):
        net_shape(481, 640, 640, "yuv420p")


class TableDetector:
    """Stand-in with frame tables: each frame's row 0 encodes its mean value and shape, so results trace to inputs."""
    def __init__(self, res=640):
        self.res, self.calls = res, []

    def net_shape(self, H, W, pix_fmt="bgr24"):
        return net_shape(H, W, self.res, pix_fmt)

    @staticmethod
    def _row(f):
        out = torch.zeros(300, 6)
        m = float(f.float().mean())
        out[0, :4] = torch.tensor([m, f.shape[0], f.shape[1], m + 1])
        out[0, 4], out[0, 5] = 0.9, 2
        return out

    def detect_batch(self, frames, pix_fmt="bgr24"):
        self.calls.append(("batch", tuple(frames.shape), pix_fmt))
        return torch.stack([self._row(f) for f in frames])

    def detect_frames(self, frames, pix_fmts="bgr24"):
        self.calls.append(("frames", [None if f is None else tuple(f.shape) for f in frames], list(pix_fmts)))
        return torch.stack([torch.zeros(300, 6) if f is None else self._row(f) for f in frames])


def _fleet(t):
    """Six uint8 cameras of three shapes and both formats that all letterbox to 384 x 640 at res 640 (small 16:9 frames
    keep the host work light), plus a float32 camera of the same net shape and a camera alone in its own net shape."""
    f = {}
    for i, (H, W) in enumerate([(72, 128), (144, 256), (216, 384)]):
        f[f"b{i}"] = np.full((H, W, 3), 10 * i + t, np.uint8)
        f[f"y{i}"] = np.full((H * 3 // 2, W), 50 + 10 * i + t, np.uint8)
    f["float"] = np.full((72, 128, 3), 120.0 + t, np.float32)
    f["square"] = np.full((64, 64, 3), 200 + t, np.uint8)
    return f


def _batch(det):
    cb = CameraBatch(det)
    for i in range(3):
        cb.add_camera(f"y{i}", pix_fmt="yuv420p")
    return cb


def test_mixed_shapes_and_formats_of_one_net_shape_make_one_detect_frames_call():
    det = TableDetector()
    cb = _batch(det)
    for t in range(3):
        det.calls.clear()
        frames = _fleet(t)
        res = cb.step(frames)
        assert set(res) == set(frames)
        tables = [c for c in det.calls if c[0] == "frames"]
        assert len(tables) == 1
        shapes, fmts = tables[0][1], tables[0][2]
        assert len(shapes) == 8 and shapes[6:] == [None, None]            # 6 cameras padded to the bucket 8
        assert sorted(fmts[:6]) == ["bgr24"] * 3 + ["yuv420p"] * 3
        # float32 frames and the lone square camera keep detect_batch
        assert sorted(c[1] for c in det.calls if c[0] == "batch") == [(1, 64, 64, 3), (1, 72, 128, 3)]
        for name, f in frames.items():
            r = res[name].rows
            assert abs(r[0, 0] - float(f.mean())) < 1e-3 and (r[0, 1], r[0, 2]) == f.shape[:2], name
            assert np.array_equal(cb.device_frame(name).numpy(), f), name
            assert len(res[name].targets) == 1


def test_single_source_groups_still_call_detect_batch():
    det = TableDetector()
    cb = CameraBatch(det)
    frames = {f"c{i}": np.full((72, 128, 3), i, np.uint8) for i in range(3)}
    frames["big"] = np.full((216, 384, 3), 9, np.uint8)     # same net shape as c*, but the group mixes two shapes ...
    res = cb.step(frames)
    assert [c[0] for c in det.calls] == ["frames"]
    det.calls.clear()
    del frames["big"]                                       # ... and without it the group has one source shape
    res = cb.step(frames)
    assert det.calls == [("batch", (4, 72, 128, 3), "bgr24")]
    assert all(abs(res[n].rows[0, 0] - i) < 1e-4 for i, n in enumerate(sorted(frames)))


def test_a_group_larger_than_max_frames_is_split():
    det = TableDetector()
    cb = CameraBatch(det)
    n = CC_MAX_FRAMES + 5
    frames = {f"c{i:03d}": np.full((72, 128, 3) if i % 2 else (144, 256, 3), i % 250, np.uint8) for i in range(n)}
    res = cb.step(frames)
    calls = [c for c in det.calls if c[0] == "frames"]
    assert [len(c[1]) for c in calls] == [CC_MAX_FRAMES, 8]
    assert sum(s is not None for c in calls for s in c[1]) == n
    assert set(res) == set(frames)
    for name, f in frames.items():
        assert abs(res[name].rows[0, 0] - float(f.mean())) < 1e-3, name


def test_models_without_frame_tables_keep_the_per_shape_path():
    class BatchOnly:
        def __init__(self):
            self.inner = TableDetector()
            self.calls = self.inner.calls

        def detect_batch(self, frames, pix_fmt="bgr24"):
            return self.inner.detect_batch(frames, pix_fmt)
    det = BatchOnly()
    assert not hasattr(det, "net_shape")
    cb = _batch(det)
    cb.step(_fleet(0))
    assert all(c[0] == "batch" for c in det.calls) and len(det.calls) == 8
