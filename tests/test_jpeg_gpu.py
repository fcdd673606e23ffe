"""JPEG of frame crops on the GPU: every file must be byte for byte what cv2.imwrite / cv2.imencode writes for the same
crop (and what oracle/jpeg.py computes), for BGR, RGB and I420 frames, one crop or hundreds per call."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import jpeg as oj
from oracle.yuv import i420_to_bgr
from clearcam_b200 import ops
from clearcam_b200._lib import lib, ptr, stream_ptr
from clearcam_b200.pixfmt import CC_FRAME_BGR_U8 as BGR, CC_FRAME_I420_U8 as I420, CC_FRAME_RGB_U8 as RGB

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jpeg_cv2.npz")


def _cv2():
    return pytest.importorskip("cv2")


def _imencode(img, q):
    cv2 = _cv2()
    return cv2.imencode(".jpg", np.ascontiguousarray(img), [cv2.IMWRITE_JPEG_QUALITY, int(q)])[1].tobytes()


def _frames(n, H, W, seed):
    """Smooth gradients + blobs + noise: natural-looking content with long zero runs and busy blocks."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    out = []
    for i in range(n):
        base = np.stack([(xx * (0.1 + 0.05 * c) + yy * (0.07 * (c + 1)) + 40 * i) % 256 for c in range(3)], -1)
        base += rng.normal(0, 6 + 4 * i, (H, W, 3))
        out.append(np.clip(base, 0, 255).astype(np.uint8))
    return np.stack(out)


def _encode_dev(dev, rects, q, fmt=BGR):
    return ops.jpeg_collect(*ops.jpeg_encode_crops_frames(ops.batch_table(dev, fmt), rects, q))


def _encode(frames, rects, q, fmt=BGR):
    return _encode_dev(torch.from_numpy(np.ascontiguousarray(frames)).cuda(), rects, q, fmt)


def test_table_encoder_fixture():
    g = np.load(GOLDEN)
    k = 0
    while f"img{k}" in g:
        for q in g[f"q{k}"]:
            want = g[f"jpg{k}_{q}"].tobytes()
            if f"yuv{k}" in g:
                x1, y1, x2, y2 = (int(v) for v in g[f"rect{k}"])
                got = _encode(g[f"yuv{k}"][None], [(0, x1, y1, x2, y2)], q, I420)[0]
            else:
                img = g[f"img{k}"]
                got = _encode(img[None], [(0, 0, 0, img.shape[1], img.shape[0])], q)[0]
            assert got == want, (k, q)
        k += 1
    assert k >= 17


def test_table_encoder_every_size_up_to_33_in_one_call():
    fr = _frames(2, 70, 70, seed=1)
    rects = [((w + h) % 2, (3 * w) % 5, (7 * h) % 3, (3 * w) % 5 + w, (7 * h) % 3 + h) for w in range(1, 34) for h in range(1, 34)]
    for q in (95, 50):
        got = _encode(fr, rects, q)
        assert len(got) == len(rects) == 33 * 33
        for (f, x1, y1, x2, y2), g in zip(rects, got):
            crop = fr[f, y1:y2, x1:x2]
            assert g == _imencode(crop, q), (x2 - x1, y2 - y1, q)
            if (x2 - x1) % 8 == 1:
                assert g == oj.encode(crop, q)


_RECTS_1080 = [(0, 1, 3, 201, 157), (1, 1719, 881, 1920, 1080), (0, 0, 0, 1920, 1080), (1, 333, 77, 334, 78),
               (0, 1001, 999, 1500, 1080), (1, 0, 1, 113, 700), (0, 1917, 1077, 1920, 1080), (1, 1850, 0, 1920, 61),
               (0, 0, 1000, 97, 1080), (1, 777, 555, 1377, 1155 - 75)]


@pytest.mark.parametrize("q", [95, 85])
def test_table_encoder_source_formats(q):
    cv2 = _cv2()
    bgr = _frames(2, 1080, 1920, seed=2)
    rgb = np.ascontiguousarray(bgr[..., ::-1])
    yuv = np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420) for f in bgr])
    conv = i420_to_bgr(yuv)
    got_b, got_r, got_y = _encode(bgr, _RECTS_1080, q, BGR), _encode(rgb, _RECTS_1080, q, RGB), _encode(yuv, _RECTS_1080, q, I420)
    for i, (f, x1, y1, x2, y2) in enumerate(_RECTS_1080):
        want = _imencode(bgr[f, y1:y2, x1:x2], q)
        assert got_b[i] == want, ("bgr", i)
        assert got_r[i] == want, ("rgb", i)      # cv2 of the swapped image = the BGR crop
        want_y = _imencode(cv2.cvtColor(yuv[f], cv2.COLOR_YUV2BGR_I420)[y1:y2, x1:x2], q)
        assert got_y[i] == want_y, ("i420", i)
        assert np.array_equal(conv[f, y1:y2, x1:x2], cv2.cvtColor(yuv[f], cv2.COLOR_YUV2BGR_I420)[y1:y2, x1:x2])


def test_table_encoder_full_frame_q85_matches_oracle():
    fr = _frames(1, 1080, 1920, seed=3)
    got = _encode(fr, [(0, 0, 0, 1920, 1080)], 85)[0]
    assert got == _imencode(fr[0], 85)
    assert got == oj.encode(fr[0], 85)


def test_table_encoder_many_crops_in_one_call_equal_single_calls():
    fr = _frames(8, 540, 960, seed=4)
    rng = np.random.default_rng(5)
    rects = []
    for _ in range(200):
        w, h = int(rng.integers(1, 400)), int(rng.integers(1, 300))
        x, y = int(rng.integers(0, 960 - w + 1)), int(rng.integers(0, 540 - h + 1))
        rects.append((int(rng.integers(0, 8)), x, y, x + w, y + h))
    got = _encode(fr, rects, 95)
    dev = torch.from_numpy(fr).cuda()
    for i, r in enumerate(rects):
        assert got[i] == _encode_dev(dev, [r], 95)[0], i
        if i % 20 == 0:
            f, x1, y1, x2, y2 = r
            assert got[i] == _imencode(fr[f, y1:y2, x1:x2], 95), i


def test_table_encoder_bytes_past_each_length_stay_untouched_and_noise_fits_the_bound():
    rng = np.random.default_rng(6)
    fr = rng.integers(0, 256, (2, 300, 400, 3), dtype=np.uint8)
    rects = np.array([(0, 0, 0, 400, 300), (1, 7, 9, 240, 263), (0, 399, 299, 400, 300), (1, 100, 100, 133, 117)], np.int32)
    L = lib()
    bounds = np.array([ops.jpeg_bound(r[3] - r[1], r[4] - r[2]) for r in rects], np.int64)
    gap = 64
    offsets = np.ascontiguousarray((np.concatenate([[0], np.cumsum(bounds + gap)[:-1]]) + gap).astype(np.int64))
    cap = int(offsets[-1] + bounds[-1] + gap)
    dev = torch.from_numpy(fr).cuda()
    for q in (100, 0, 95):
        out = torch.full((cap,), 0xA5, dtype=torch.uint8, device="cuda")
        lengths = torch.zeros(len(rects), dtype=torch.int64, device="cuda")
        need = ctypes.c_size_t(0)
        args = (ops.batch_table(dev, BGR), 2, rects.ctypes.data, len(rects), q)
        assert L.cc_jpeg_encode_crops_frames(*args, None, 0, None, None, None, 0, ctypes.byref(need), None) == 0
        ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
        assert L.cc_jpeg_encode_crops_frames(*args, ptr(out), cap, offsets.ctypes.data, ptr(lengths), ptr(ws), need.value, None,
                                             stream_ptr()) == 0
        o, n = out.cpu().numpy(), lengths.cpu().numpy()
        used = np.zeros(cap, bool)
        for k, r in enumerate(rects):
            assert n[k] <= bounds[k]
            got = o[offsets[k]:offsets[k] + n[k]].tobytes()
            assert got == _imencode(fr[r[0], r[2]:r[4], r[1]:r[3]], q), (k, q)
            used[offsets[k]:offsets[k] + n[k]] = True
        assert (o[~used] == 0xA5).all(), q


def test_table_coefficient_tap_equals_the_oracle_blocks():
    cv2 = _cv2()
    fr = _frames(2, 240, 320, seed=7)
    rects = [(0, 0, 0, 320, 240), (1, 3, 5, 40, 22), (1, 311, 231, 320, 240), (0, 17, 1, 18, 2), (1, 100, 50, 250, 200)]
    for q, fmt in ((95, BGR), (10, RGB), (100, I420)):
        src = fr if fmt == BGR else np.ascontiguousarray(fr[..., ::-1]) if fmt == RGB else \
            np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420) for f in fr])
        img = fr if fmt != I420 else i420_to_bgr(src)
        dev = torch.from_numpy(src).cuda()
        got = ops.jpeg_coeffs_frames(ops.batch_table(dev, fmt), rects, q).cpu().numpy()
        want = np.concatenate([oj.blocks(img[f, y1:y2, x1:x2], q) for f, x1, y1, x2, y2 in rects])
        assert got.shape == want.shape and np.array_equal(got, want), (q, fmt)


def _camera_batch_end_to_end(pix_fmt, tmp_path):
    cv2 = _cv2()
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.models.objects import ObjectFinder
    fr = o.synthetic_frames(2, 320, 320, seed=9)
    x = torch.stack([o.preprocess(f, 320) for f in fr]).flip(-1).permute(0, 3, 1, 2).float() / 255
    m = YOLOv9("c", 640, weights=o.synthetic_weights("c", seed=9, calib=x))
    cb = CameraBatch(m)
    H, W = 720, 1280
    bgr = o.synthetic_frames(1, H, W, seed=31)[0].numpy()
    if pix_fmt == "yuv420p":
        frame = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
        cb.add_camera("cam", pix_fmt="yuv420p")
        host = cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_I420)
    else:
        frame, host = bgr, bgr
    res = cb.step({"cam": frame})["cam"]
    rects = [ObjectFinder.crop_rect(r[:4], W, H, min_side=16) for r in res.rows if r[4] > 0]
    rects = [r for r in rects if r is not None][:20] + [(0, 0, W, H), (W - 150, H - 101, W, H)]
    finder = ObjectFinder()
    got = finder.encode_crops(cb.device_frame("cam"), rects, pix_fmt=pix_fmt)
    for i, (x1, y1, x2, y2) in enumerate(rects):
        p = tmp_path / f"{i}.jpg"
        cv2.imwrite(str(p), host[y1:y2, x1:x2])
        q = tmp_path / f"{i}_gpu.jpg"
        q.write_bytes(got[i])
        assert q.read_bytes() == p.read_bytes(), i


def test_camera_batch_to_encode_crops_bgr24(tmp_path):
    _camera_batch_end_to_end("bgr24", tmp_path)


def test_camera_batch_to_encode_crops_yuv420p(tmp_path):
    _camera_batch_end_to_end("yuv420p", tmp_path)
