"""Every camera's object saves in one call on the GPU: the frame-table forms of the JPEG encoder, the crops-decoded tap and
the CLIP preprocess against the uniform entry points on each frame alone and against cv2, ObjectFinder.encode_embed_frames
against the reference's host chain, CameraBatch.save_objects end to end on a mixed fleet, and bad tables."""
import ctypes

import numpy as np
import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200._lib import cc_frame, lib, ptr, stream_ptr

pytestmark = pytest.mark.gpu

# an 8 x 8 grey block whose quality-2 JPEG leaves the range where every libjpeg-turbo IDCT agrees (CC_JPEG_UNSUPPORTED)
Q2_BLOCK = np.array([[62, 255, 30, 78, 236, 18, 248, 80], [0, 198, 25, 35, 232, 126, 208, 117],
                     [110, 0, 145, 246, 148, 6, 187, 90], [218, 226, 255, 53, 0, 243, 23, 217],
                     [255, 254, 36, 91, 8, 110, 150, 21], [227, 47, 93, 44, 239, 10, 0, 1],
                     [128, 143, 3, 166, 255, 17, 7, 35], [255, 26, 255, 43, 177, 35, 230, 159]], np.uint8)
Q2_AT = (40, 24)                # (x, y) of the block in every bgr24 frame of the fleet


def _cv2():
    return pytest.importorskip("cv2")


def _img(h, w, seed, sigma=10):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([(xx * (0.9 + 0.3 * c) + yy * (0.6 + 0.2 * c) + 60 * c) % 256 for c in range(3)], -1)
    return np.clip(base + rng.normal(0, sigma, (h, w, 3)), 0, 255).astype(np.uint8)


FLEET = [((720, 1280), "bgr24"), ((1080, 1920), "yuv420p"), ((1440, 2560), "bgr24"), ((720, 1280), "yuv420p"),
         ((241, 333), "bgr24"), ((1080, 1920), "bgr24")]


def _fleet():
    """-> (device frames, pix_fmts, host BGR pictures): each bgr24 frame carries Q2_BLOCK at Q2_AT."""
    cv2 = _cv2()
    dev, fmts, host = [], [], []
    for i, ((H, W), fmt) in enumerate(FLEET):
        bgr = _img(H, W, 100 + i)
        if fmt == "bgr24":
            x, y = Q2_AT
            bgr[y:y + 8, x:x + 8] = Q2_BLOCK[..., None]
            dev.append(torch.from_numpy(bgr).cuda())
        else:
            yuv = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
            bgr = cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_I420)
            dev.append(torch.from_numpy(yuv).cuda())
        fmts.append(fmt)
        host.append(bgr)
    return dev, fmts, host


def _rects(seed=7, n_random=300):
    """Full frames, 1-pixel crops, crops on every edge and corner, the quality-2 block, and many random crops: more than
    256 in all, so the encoder's call crosses a launch group."""
    rng = np.random.default_rng(seed)
    out = []
    for j, ((H, W), _) in enumerate(FLEET):
        out += [(j, 0, 0, W, H), (j, 0, 0, 1, 1), (j, W - 1, H - 1, W, H), (j, W // 2, H // 3, W // 2 + 1, H // 3 + 1),
                (j, 0, 5, 17, H), (j, W - 33, 0, W, 19), (j, 3, H - 2, W - 5, H), (j, W - 1, 0, W, H), (j, 0, H - 1, W, H)]
        if FLEET[j][1] == "bgr24":
            x, y = Q2_AT
            out += [(j, x, y, x + 8, y + 8)]
    for _ in range(n_random):
        j = int(rng.integers(0, len(FLEET)))
        (H, W), _ = FLEET[j]
        w, h = int(rng.integers(1, min(W, 600) + 1)), int(rng.integers(1, min(H, 600) + 1))
        x, y = int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1))
        out.append((j, x, y, x + w, y + h))
    return np.array(out, np.int32)


def _solo(frames, fmts, j):
    """Frame j alone as a uniform batch of one: (tensor, src_fmt of the uniform entry points)."""
    return frames[j][None], 1 if fmts[j] == "bgr24" else 2


@pytest.fixture(scope="module")
def fleet():
    return _fleet()


def test_table_encoder_equals_the_uniform_encoder_and_cv2(fleet):
    cv2 = _cv2()
    frames, fmts, host = fleet
    rects = _rects()
    assert len(rects) > 256
    for q in (95, 50):
        files = ops.jpeg_encode_crops_frames(frames, fmts, rects, q)
        assert len(files) == len(rects)
        for j in range(len(FLEET)):
            ks = np.flatnonzero(rects[:, 0] == j)
            sub = rects[ks].copy()
            sub[:, 0] = 0
            t, src_fmt = _solo(frames, fmts, j)
            solo = ops.jpeg_encode_crops(t, sub, q, src_fmt)
            for k, f in zip(ks, solo):
                assert files[k] == f, (q, j, k)
        for k, (j, x1, y1, x2, y2) in enumerate(rects):
            want = cv2.imencode(".jpg", np.ascontiguousarray(host[j][y1:y2, x1:x2]), [cv2.IMWRITE_JPEG_QUALITY, q])[1]
            assert files[k] == want.tobytes(), (q, k)


def test_table_encoder_leaves_the_bytes_past_each_length(fleet):
    frames, fmts, _ = fleet
    rects = _rects(seed=8, n_random=40)
    table, sizes = ops.frame_table(frames, fmts)
    bounds = np.array([ops.jpeg_bound(r[3] - r[1], r[4] - r[2]) for r in rects], np.int64)
    offs = np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.int64)
    need = ctypes.c_size_t(0)
    args = (table, len(frames), rects.ctypes.data, len(rects), 95)
    assert lib().cc_jpeg_encode_crops_frames(*args, None, 0, None, None, None, 0, ctypes.byref(need), None) == 0
    out = torch.full((int(bounds.sum()),), 0xA5, dtype=torch.uint8, device="cuda")
    lengths = torch.zeros(len(rects), dtype=torch.int64, device="cuda")
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    assert lib().cc_jpeg_encode_crops_frames(*args, ptr(out), out.numel(), offs.ctypes.data, ptr(lengths), ptr(ws), need.value,
                                             None, stream_ptr()) == 0
    lens, host = lengths.cpu().numpy(), out.cpu().numpy()
    files = ops.jpeg_encode_crops_frames(frames, fmts, rects, 95)
    for k in range(len(rects)):
        assert host[offs[k]:offs[k] + lens[k]].tobytes() == files[k]
        assert (host[offs[k] + lens[k]:offs[k] + bounds[k]] == 0xA5).all(), k


@pytest.mark.parametrize("q", [95, 2])
def test_table_crops_decoded_equal_the_uniform_call(fleet, q):
    cv2 = _cv2()
    frames, fmts, _ = fleet
    rects = _rects(seed=9, n_random=60)
    pix, st = ops.jpeg_crops_decoded_frames(frames, fmts, rects, q)
    pix, st = pix.cpu().numpy(), st.cpu().numpy()
    for j in range(len(FLEET)):
        ks = np.flatnonzero(rects[:, 0] == j)
        sub = rects[ks].copy()
        sub[:, 0] = 0
        t, src_fmt = _solo(frames, fmts, j)
        want, wst = ops.jpeg_crops_decoded(t, sub, q, src_fmt)
        want, wst = want.cpu().numpy(), wst.cpu().numpy()
        for i, k in enumerate(ks):
            assert st[k] == wst[i], (q, j, k)
            if st[k] == ops.JPEG_OK:
                h, w = sub[i, 4] - sub[i, 2], sub[i, 3] - sub[i, 1]
                assert np.array_equal(pix[k, :h, :w], want[i, :h, :w]), (q, j, k)
    if q == 2:
        assert (st == ops.JPEG_UNSUPPORTED).any()
        files = ops.jpeg_encode_crops_frames(frames, fmts, rects, q)
        from oracle import jpeg_decode as od
        for k in np.flatnonzero(st == ops.JPEG_UNSUPPORTED):
            assert od.decode(files[k])[0] == ops.JPEG_UNSUPPORTED
    else:
        assert (st == ops.JPEG_OK).all()
    del cv2


def test_table_clip_preprocess_equals_the_uniform_call(fleet):
    frames, fmts, _ = fleet
    rects = _rects(seed=10, n_random=80)
    assert len(rects) > 64
    table, _ = ops.frame_table(frames, fmts)
    S = 224
    got = torch.full((len(rects) + 1, 3, S, S), 7.0, device="cuda")
    assert lib().cc_clip_preprocess_frames(table, len(frames), rects.ctypes.data, len(rects), S, ptr(got), stream_ptr()) == 0
    assert (got[-1] == 7.0).all()
    for j in range(len(FLEET)):
        ks = np.flatnonzero(rects[:, 0] == j)
        sub = np.ascontiguousarray(rects[ks].copy())
        sub[:, 0] = 0
        t, src_fmt = _solo(frames, fmts, j)
        H, W = FLEET[j][0]
        want = torch.empty(len(sub), 3, S, S, device="cuda")
        assert lib().cc_clip_preprocess(ptr(t), 1, H, W, sub.ctypes.data, len(sub), S, src_fmt, ptr(want), stream_ptr()) == 0
        assert torch.equal(got[torch.from_numpy(ks).cuda()], want), j


def _finder():
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    return of


def _host_chain(of, files):
    """clearcam.py:274-276, 1280-1285: imdecode -> BGR2RGB -> preprocess, stacked and padded to the batch bucket."""
    cv2 = _cv2()
    from clearcam_b200.utils.helpers import batch_bucket
    x = [of.preprocess(cv2.cvtColor(cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB))
         for f in files]
    x = np.stack(x + [np.zeros_like(x[0])] * (batch_bucket(len(x)) - len(x)))
    return of.model.precompute_embedding(x).tensor[:len(files)]


@pytest.mark.parametrize("q", [95, 2])
def test_encode_embed_frames_equals_encode_crops_and_the_host_chain(fleet, q):
    cv2 = _cv2()
    cv2.ipp.setUseIPP(False)
    frames, fmts, _ = fleet
    x, y = Q2_AT
    rects = np.array([(0, 10, 20, 310, 220), (1, 600, 100, 750, 400), (2, 0, 0, 2560, 1440), (3, 1100, 600, 1280, 720),
                      (4, 0, 0, 333, 241), (5, 1700, 900, 1920, 1080), (0, x, y, x + 8, y + 8), (2, 5, 7, 6, 8),
                      (1, 0, 0, 1920, 1080)], np.int32)
    of = _finder()
    files, emb = of.encode_embed_frames(frames, fmts, rects, q)
    for k, (j, *r) in enumerate(rects.tolist()):
        t, _ = _solo(frames, fmts, j)
        assert files[k] == of.encode_crops(t, [(0, *r)], q, pix_fmt=fmts[j])[0], k
    assert torch.equal(emb.tensor, _host_chain(of, files))
    if q == 2:
        _, st = ops.jpeg_crops_decoded_frames(frames, fmts, rects, q)
        assert (st.cpu().numpy() == ops.JPEG_UNSUPPORTED).any()         # the cv2 fallback ran
    of.model = None
    files2, none = of.encode_embed_frames(frames, fmts, rects, q)
    assert files2 == files and none is None


def test_camera_batch_save_objects_end_to_end():
    """A mixed fleet through mailboxes with zones for several steps: each camera's save_objects files are those of
    finder.encode_crops on its device_frame and its embeddings those of the stacked host chain."""
    import io
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.ingest import FrameMailbox
    fleet = {"b180": ((180, 320), "bgr24"), "y180": ((180, 320), "yuv420p"), "b360": ((360, 640), "bgr24"),
             "y360": ((360, 640), "yuv420p"), "b720": ((720, 1280), "bgr24"), "y720": ((720, 1280), "yuv420p")}
    zones = {"y180": ([[0.0, 0.0], [1.0, 0.0], [1.0, 0.6], [0.0, 0.6]], False, False),
             "b360": ([[0.2, 0.2], [0.8, 0.1], [0.7, 0.9]], True, True)}
    xc = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    m = YOLOv9("c", 320, weights=o.synthetic_weights("c", seed=5, calib=xc))
    cb = CameraBatch(m, max_age=100)
    boxes = {n: FrameMailbox(H, W, pix_fmt=fmt) for n, ((H, W), fmt) in fleet.items()}
    for n, ((H, W), fmt) in fleet.items():
        cb.add_camera(n, thresh=0.05, pix_fmt=fmt)
        if n in zones:
            cb.set_zone(n, *zones[n])
    of = _finder()
    n_saves = 0
    for t in range(6):
        for i, n in enumerate(boxes):
            (H, W), fmt = fleet[n]
            f = o.synthetic_frames(1, H, W, seed=40 + i)[0].roll(shifts=(3 * t, 5 * t), dims=(0, 1))
            if fmt == "yuv420p":
                f = torch.cat([f[..., 1].reshape(-1), f[::2, ::2, 0].reshape(-1), f[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)
            assert boxes[n].fill(io.BytesIO(f.numpy().tobytes()))
        res = cb.step_events_mailboxes(boxes, now=1.7e9 + 1.1 * t)
        got = cb.save_objects(res, of)
        assert set(got) == set(res)
        for n, (saves, files, emb) in got.items():
            assert saves is res[n].saves and len(files) == len(saves)
            if not len(saves):
                assert emb is None
                continue
            rects = [(0, *(int(v) for v in s[2:6])) for s in saves]
            assert files == of.encode_crops(cb.device_frame(n)[None], rects, pix_fmt=fleet[n][1]), (t, n)
            assert torch.equal(emb.tensor, _host_chain(of, files)), (t, n)
            n_saves += len(saves)
    assert n_saves > 0


def test_bad_tables_fail_and_leave_the_outputs_untouched(fleet):
    frames, fmts, _ = fleet
    table, _ = ops.frame_table(frames, fmts)
    n = len(frames)
    rects = np.array([(0, 0, 0, 64, 64), (1, 10, 10, 90, 70)], np.int32)
    bad_rows = {
        "NULL frame": lambda t: setattr(t[1], "data", None),
        "float frame": lambda t: setattr(t[1], "fmt", 1),
        "unknown format": lambda t: setattr(t[1], "fmt", 5),
        "odd I420 size": lambda t: setattr(t[1], "h", 1079),
    }
    outside = np.array([(0, 0, 0, 64, 64), (4, 300, 200, 400, 260)], np.int32)   # inside frame 0, outside its own 333 x 241
    S = 32
    for what, spoil in list(bad_rows.items()) + [("rect outside its own frame", None)]:
        t = (cc_frame * n)(*table)
        r = rects
        if spoil is None:
            r = outside
        else:
            spoil(t)
        out = torch.full((2, 3, S, S), 3.0, device="cuda")
        assert lib().cc_clip_preprocess_frames(t, n, r.ctypes.data, 2, S, ptr(out), stream_ptr()) == -1, what
        enc = torch.full((1 << 20,), 0x5A, dtype=torch.uint8, device="cuda")
        lengths = torch.full((2,), -7, dtype=torch.int64, device="cuda")
        ws = torch.empty(1 << 24, dtype=torch.uint8, device="cuda")
        offs = np.array([0, 1 << 19], np.int64)
        assert lib().cc_jpeg_encode_crops_frames(t, n, r.ctypes.data, 2, 95, ptr(enc), enc.numel(), offs.ctypes.data, ptr(lengths),
                                                 ptr(ws), ws.numel(), None, stream_ptr()) == -1, what
        pix = torch.full((2, 128, 128, 3), 0x33, dtype=torch.uint8, device="cuda")
        st = torch.full((2,), 9, dtype=torch.int32, device="cuda")
        assert lib().cc_jpeg_crops_decoded_frames(t, n, r.ctypes.data, 2, 95, ptr(pix), 128, 128, ptr(st), ptr(ws), ws.numel(), None,
                                                  stream_ptr()) == -1, what
        torch.cuda.synchronize()
        assert (out == 3.0).all() and (enc == 0x5A).all() and (lengths == -7).all(), what
        assert (pix == 0x33).all() and (st == 9).all(), what
