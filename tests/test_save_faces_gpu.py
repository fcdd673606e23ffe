"""The faces of the object saves and of uploads on the GPU, on the BlazeFace fixture's weights and a synthetic AdaFace.

* The slot kernels (cc_face_canvas_slots, cc_face_align_slots) on a padded BGR batch equal cc_face_canvas / cc_face_align
  on the contiguous RGB copies, byte for byte: slots of mixed sizes, exact 2x reductions, a 640 long side, 1-pixel-thin
  images, more than one launch of each; bad arguments are refused before anything is written.
* cc_blazeface_first equals numpy's detections[detections[:, 0] != 0][0] on injected rows (-0.0, NaN, no row kept).
* ObjectFinder.encode_embed_faces_frames on bgr24 and yuv420p frames carrying the fixture's face: files and CLIP embeddings
  equal encode_embed_frames, and each person crop's face row, file and embedding equal the reference's host chain
  (imdecode -> RGB -> img_to_face -> imencode, adaface); at quality 2 through the cv2 fallback; CLIP off, face off.
* CameraBatch.save_objects_and_faces on a mixed fleet (bgr24, yuv420p, MJPEG) and on step_video runs.
* ObjectFinder.embed_face_images: 112x112, large, faceless, stored and progressive uploads against run_clip's chain.
"""
import io

import numpy as np
import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200._lib import CCError, cc_face_warp, lib, ptr, stream_ptr
from clearcam_b200.models.blazeface import (align_faces, align_faces_slots, face_canvas, face_canvas_slots, face_geometry,
                                            first_detections)

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

from test_face_detect_gpu import GOLD, _rows  # noqa: E402
from test_object_saves_gpu import Q2_BLOCK  # noqa: E402


@pytest.fixture(scope="module")
def P():
    from oracle import blazeface as bf
    return bf.load_weights(GOLD)


@pytest.fixture(scope="module")
def face_bgr():
    with np.load(GOLD) as z:
        return np.ascontiguousarray(z["firing"][..., ::-1])


@pytest.fixture(scope="module")
def finder(P):
    from oracle import adaface as oa
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    cv2.ipp.setUseIPP(False)
    f = ObjectFinder()
    f.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    f.init_face(weights=oa.synthetic_weights(seed=5), detector={k: v.numpy() for k, v in P.items()})
    return f


def _scaled(face, s):
    return np.ascontiguousarray(cv2.resize(face, (int(256 * s), int(256 * s)), interpolation=cv2.INTER_LINEAR) if s != 1 else face)


def _noise(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


# ------------------------------------------------------------------------------------------------ kernels
def test_slot_kernels_equal_the_contiguous_rgb_copies():
    g = np.random.default_rng(31)
    Hmax, Wmax = 1000, 1300
    sizes = [(1000, 1300), (960, 1280), (480, 640), (640, 480), (640, 640), (1, 640), (640, 1), (2, 900), (333, 129), (97, 300),
             (112, 112), (50, 33)]
    while len(sizes) < 70:
        sizes.append((int(g.integers(40, Hmax + 1)), int(g.integers(40, Wmax + 1))))
    n_slots = 75
    slots = torch.from_numpy(g.integers(0, 256, (n_slots, Hmax, Wmax, 3), dtype=np.uint8)).cuda()   # the padding is not zero
    index = [(7 * b + 3) % n_slots for b in range(len(sizes))]
    rgb = [slots[s, :h, :w].flip(-1).contiguous() for s, (h, w) in zip(index, sizes)]
    got = face_canvas_slots(slots, index, sizes, rows=80)
    assert got.shape[0] == 80 and not got[len(sizes):].any()
    assert torch.equal(got[:len(sizes)], face_canvas(rgb))
    jobs, slot_jobs = [], []
    while len(jobs) < 40:
        b = int(g.integers(0, len(sizes)))
        geo = face_geometry(_rows(g), *sizes[b])
        if geo is None:
            continue
        jobs.append((rgb[b], geo))
        slot_jobs.append((index[b], sizes[b], geo))
    assert torch.equal(align_faces_slots(slots, slot_jobs), align_faces(jobs))


def test_slot_kernels_refuse_bad_arguments_before_launch():
    slots = torch.zeros(2, 64, 96, 3, dtype=torch.uint8, device="cuda")
    out = torch.full((2, 640, 640, 3), 7, dtype=torch.uint8, device="cuda")
    L = lib()

    def canvas(idx, hw, B=None, p=ptr(slots)):
        i, s = np.ascontiguousarray(idx, np.int32), np.ascontiguousarray(hw, np.int32)
        return L.cc_face_canvas_slots(p, 2, 64, 96, i.ctypes.data, s.ctypes.data, len(idx) if B is None else B, ptr(out), stream_ptr())

    assert canvas([0], [(65, 96)]) != 0                  # taller than a slot
    assert canvas([0], [(64, 97)]) != 0                  # wider than a slot
    assert canvas([2], [(64, 96)]) != 0                  # past the last slot
    assert canvas([-1], [(64, 96)]) != 0
    assert canvas([0], [(64, 96)], B=0) != 0
    assert canvas([0], [(64, 96)], p=None) != 0
    assert canvas([0], [(1, 96)]) == 0                      # a 1-pixel-thin image is taken
    ws = (cc_face_warp * 1)()
    ws[0].h, ws[0].w, ws[0].x1, ws[0].y1, ws[0].x2, ws[0].y2, ws[0].rot_w, ws[0].rot_h = 64, 96, 0, 0, 40, 40, 50, 50

    def align(idx, K=1, p=ptr(slots)):
        i = np.ascontiguousarray(idx, np.int32)
        return L.cc_face_align_slots(p, 2, 64, 96, i.ctypes.data, ws, K, ptr(out), stream_ptr())
    assert align([2]) != 0 and align([0], K=0) != 0 and align([0], p=None) != 0
    ws[0].x2 = 97                                        # crop outside its image
    assert align([0]) != 0
    ws[0].x2, ws[0].w = 40, 97                           # image wider than a slot
    assert align([0]) != 0
    torch.cuda.synchronize()
    assert (out[1] == 7).all()


def test_first_detections_equal_numpy():
    g = np.random.default_rng(5)
    B = 131
    d = g.normal(0, 100, (B, 896, 17)).astype(np.float32)
    d[g.random((B, 896, 17)) < 0.05] = np.nan
    d[:, :, 0] = 0
    for b in range(B):
        k = int(g.integers(0, 896))
        kind = b % 5
        d[b, :k, 0] = np.where(g.random(k) < 0.5, -0.0, 0.0)
        if kind == 1:
            d[b, k, 0] = np.nan
        elif kind == 2:
            d[b, k:, 0] = g.normal(0, 10, 896 - k)
        elif kind == 3:
            d[b, k, 0] = -1e-30
        elif kind == 4:
            d[b, 0, 0] = 3.0
    got = first_detections(torch.from_numpy(d).cuda()).cpu().numpy()
    for b in range(B):
        kept = d[b][d[b][:, 0] != 0]
        want = kept[0] if len(kept) else np.zeros(17, np.float32)
        assert np.array_equal(got[b].view(np.int32), want.view(np.int32)), b
    assert (got[::5] == 0).all() and np.isnan(got[1::5, 0]).all()


# ------------------------------------------------------------------------------------------------ the saves
def _host_face(f, file, q):
    """process_latest_face on a thumbnail file: imdecode -> RGB -> img_to_face -> (imencode file, adaface row) or None."""
    img = cv2.cvtColor(cv2.imdecode(np.frombuffer(file, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
    face = f.img_to_face(img)
    if face is None:
        return None
    return cv2.imencode(".jpg", face, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes(), f.adaface(face).tensor[0]


def _check_faces(f, fs, files, person, q):
    """fs equals the host chain on every person file -> the number of faces."""
    rows, want_files, want_emb = [], [], []
    for k in np.flatnonzero(person):
        h = _host_face(f, files[k], q)
        if h is not None:
            rows.append(int(k))
            want_files.append(h[0])
            want_emb.append(h[1])
    assert fs.rows == rows
    assert fs.files == want_files
    assert fs.embeddings.tensor.shape == (len(rows), 512)
    if rows:
        assert torch.equal(fs.embeddings.tensor, torch.stack(want_emb))
    return len(rows)


def _plant(img, face, at, scales):
    """The face at `scales` at the (x, y) offsets `at` -> the rects (x1, y1, x2, y2) they fill.  The fixture's face is
    derived for the whole of BlazeFace's input: a crop of exactly the face keeps it firing through the thumbnail's JPEG
    from a scale of 2 up; smaller scales, and crops with a margin, give no face."""
    rects = []
    for s, (x, y) in zip(scales, at):
        f = _scaled(face, s)
        n = f.shape[0]
        img[y:y + n, x:x + n] = f
        rects.append((x, y, x + n, y + n))
    return rects


@pytest.fixture(scope="module")
def saves_fleet(face_bgr):
    """A bgr24 720p and a yuv420p 1080p frame with the face planted three times each, and the rects: every face as a
    person save and again as a non-person save, noise crops, and the quality-2 block."""
    b = _noise(720, 1280, 1)
    rb = _plant(b, face_bgr, [(100, 100), (700, 150), (1000, 450)], (2, 1, 0.75))
    b[40:48, 24:32] = Q2_BLOCK[..., None]
    y = _noise(1080, 1920, 2)
    ry = _plant(y, face_bgr, [(300, 200), (1000, 300), (1700, 800)], (2, 2.5, 0.75))
    yuv = cv2.cvtColor(y, cv2.COLOR_BGR2YUV_I420)
    frames = [torch.from_numpy(b).cuda(), torch.from_numpy(yuv).cuda()]
    rects, person = [], []
    for j, rs in ((0, rb), (1, ry)):
        for r in rs:
            rects += [(j, *r), (j, *r)]
            person += [True, False]
    rects += [(0, 24, 40, 32, 48), (0, 24, 40, 430, 450), (0, 80, 80, 632, 632), (0, 900, 30, 1200, 300), (1, 10, 600, 400, 1000),
              (1, 0, 0, 1920, 1080)]
    person += [True, True, True, True, False, True]
    return frames, ["bgr24", "yuv420p"], np.array(rects, np.int32), np.array(person)


@pytest.mark.parametrize("q", [95, 2])
def test_encode_embed_faces_frames_equals_the_host_chain(finder, saves_fleet, q):
    frames, fmts, rects, person = saves_fleet
    files, emb, fs = finder.encode_embed_faces_frames(frames, fmts, rects, person, q)
    want_files, want_emb = finder.encode_embed_frames(frames, fmts, rects, q)
    assert files == want_files and torch.equal(emb.tensor, want_emb.tensor)
    n = _check_faces(finder, fs, files, person, q)
    assert not set(fs.rows) & set(np.flatnonzero(~person).tolist())          # non-person crops of the same faces: none
    if q == 95:
        assert n >= 3
    else:
        _, st = ops.jpeg_crops_decoded_frames(ops.frame_table(frames, fmts)[0], rects, q)
        assert (st.cpu().numpy()[person] == ops.JPEG_UNSUPPORTED).any()       # the cv2 fallback ran for a person crop
    clip = finder.model
    try:
        finder.model = None                                                  # CLIP off, face on
        files2, none, fs2 = finder.encode_embed_faces_frames(frames, fmts, rects, person, q)
        assert files2 == files and none is None
        assert fs2.rows == fs.rows and fs2.files == fs.files and torch.equal(fs2.embeddings.tensor, fs.embeddings.tensor)
    finally:
        finder.model = clip
    finder.face = False
    try:
        files3, emb3, off = finder.encode_embed_faces_frames(frames, fmts, rects, person, q)
        assert off is None and files3 == files and torch.equal(emb3.tensor, emb.tensor)
    finally:
        finder.face = True


def test_missing_detector_raises(finder, saves_fleet):
    from clearcam_b200.models.objects import ObjectFinder
    frames, fmts, rects, person = saves_fleet
    f = ObjectFinder()
    f.face, f.adaface = True, finder.adaface
    with pytest.raises(CCError, match="detection is off"):
        f.encode_embed_faces_frames(frames, fmts, rects, person)


def _model():
    from oracle import yolov9 as o
    from clearcam_b200.detection.yolov9 import YOLOv9
    xc = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    return YOLOv9("c", 320, weights=o.synthetic_weights("c", seed=5, calib=xc)), o


def _with_face_saves(ev, rects, seed):
    """The step's own saves plus, per planted face, a person and a non-person save, and a person save of noise."""
    g = np.random.default_rng(seed)
    extra = []
    for r in rects:
        extra += [(int(g.integers(1, 99)), 0, *r), (int(g.integers(1, 99)), 3, *r)]
    extra.append((7, 0, 0, 0, 120, 110))
    return ev._replace(saves=np.concatenate([np.asarray(ev.saves, np.int64).reshape(-1, 6), np.array(extra, np.int64)]))


def _check_saved(cb, finder, res, saved, faces, q=95):
    """saved equals save_objects, describe_saves runs, and every camera's faces equal the host chain on its files."""
    want = cb.save_objects(res, finder, q)
    assert set(saved) == set(want) == set(faces)
    n = 0
    for name, (s, files, emb) in saved.items():
        ws, wf, we = want[name]
        np.testing.assert_array_equal(np.asarray(s), np.asarray(ws))
        assert files == wf and torch.equal(emb.tensor, we.tensor)
        n += _check_faces(finder, faces[name], files, np.asarray(s)[:, -5] == 0, q)
    cb.describe_saves(saved, now=1.7e9)
    return n


def test_camera_batch_fleet_saves_and_faces(finder, face_bgr):
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.ingest import FrameMailbox, JpegMailbox
    m, o = _model()
    cb = CameraBatch(m)
    cams = {"b": ((720, 1280), "bgr24"), "y": ((600, 800), "yuv420p"), "m": ((720, 1080), "mjpeg")}
    boxes = {}
    for n, ((H, W), fmt) in cams.items():
        cb.add_camera(n, thresh=0.05, pix_fmt=fmt)
        boxes[n] = JpegMailbox(H, W, pin=True) if fmt == "mjpeg" else FrameMailbox(H, W, pin=True, pix_fmt=fmt)
    faces_seen = 0
    for t in range(2):
        planted = {}
        for i, (n, ((H, W), fmt)) in enumerate(cams.items()):
            img = np.ascontiguousarray(o.synthetic_frames(1, H, W, seed=60 + i)[0].numpy())
            planted[n] = _plant(img, face_bgr, [(40 + 20 * t, 30), (W - 200, H - 200)], (2, 0.75))
            if fmt == "yuv420p":
                data = cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420).tobytes()
            elif fmt == "mjpeg":
                data = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
            else:
                data = img.tobytes()
            assert boxes[n].fill(io.BytesIO(data))
        res = cb.step_alerts_mailboxes(boxes, now=1.7e9 + t)
        res = {n: _with_face_saves(ev, planted[n], t) for n, ev in res.items()}
        saved, faces = cb.save_objects_and_faces(res, finder)
        faces_seen += _check_saved(cb, finder, res, saved, faces)
    assert faces_seen >= 3
    empty = {n: ev._replace(saves=np.zeros((0, 6), np.int64)) for n, ev in res.items()}
    saved, faces = cb.save_objects_and_faces(empty, finder)
    assert all(faces[n].rows == [] and faces[n].embeddings is None for n in cams)


def test_camera_batch_video_runs_saves_and_faces(finder, face_bgr):
    from clearcam_b200.cameras import CameraBatch
    m, o = _model()
    cb = CameraBatch(m)
    T, H, W = 3, 720, 1280
    imgs, planted = [], []
    for t in range(T):
        img = np.ascontiguousarray(o.synthetic_frames(1, H, W, seed=80 + t)[0].numpy())
        planted.append(_plant(img, face_bgr, [(20 + 30 * t, 40), (W - 200, H - 200)], (2, 0.75)))
        imgs.append(img)
    res = cb.step_video({"v": torch.from_numpy(np.stack(imgs))}, {"v": [1.7e9 + 0.5 * t for t in range(T)]})
    res = {"v": [_with_face_saves(ev, planted[t], t) for t, ev in enumerate(res["v"])]}
    saved, faces = cb.save_objects_and_faces(res, finder)
    s = np.asarray(saved["v"][0])
    assert s.shape[1] == 7 and s.shape[0] == sum(len(ev.saves) for ev in res["v"])
    assert _check_saved(cb, finder, res, saved, faces) >= 2
    for r in faces["v"].rows:                                                # rows index the (m,7) run saves
        f = int(s[r, 0])
        assert s[r, 2] == 0 and any(tuple(s[r, 3:7]) == p for p in planted[f])


# ------------------------------------------------------------------------------------------------ uploads
def test_embed_face_images_equals_run_clip(finder, face_bgr, tmp_path, monkeypatch):
    def jpg(img, **kw):
        params = [cv2.IMWRITE_JPEG_QUALITY, 95] + [v for k, x in kw.items() for v in (getattr(cv2, k), x)]
        return cv2.imencode(".jpg", img, params)[1].tobytes()
    small = jpg(_noise(112, 112, 3))
    big = _scaled(face_bgr, 2)
    mid = _scaled(face_bgr, 2.5)
    framed = _noise(700, 900, 4)
    framed[100:612, 200:712] = big                                                   # the face with a margin: none
    stored = tmp_path / "data" / "cameras" / "cam" / "objects" / "2026-10-19"
    stored.mkdir(parents=True)
    (stored / "1_2_0.jpg").write_bytes(jpg(mid))
    monkeypatch.chdir(tmp_path)
    progressive = jpg(big, IMWRITE_JPEG_PROGRESSIVE=1)
    items = [small, jpg(big), jpg(_noise(300, 400, 6)), "/cam/objects/2026-10-19/1_2_0.jpg", progressive, jpg(framed)]
    assert ops.JpegBatch([progressive]).status[0] != ops.JPEG_OK                       # the cv2 fallback
    emb, rows = finder.embed_face_images(items)
    want = []
    for it in items:
        file = it if isinstance(it, bytes) else (stored / "1_2_0.jpg").read_bytes()
        img = cv2.cvtColor(cv2.imdecode(np.frombuffer(file, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
        face = img if img.shape == (112, 112, 3) else finder.img_to_face(img)            # preprocess_face
        want.append(None if face is None else finder.adaface(face).tensor[0])
    assert [r is None for r in rows] == [w is None for w in want]
    assert rows[0] is not None and rows[2] is None and sum(r is not None for r in rows) >= 3
    assert emb.tensor.shape == (sum(r is not None for r in rows), 512)
    for r, w in zip(rows, want):
        if r is not None:
            assert torch.equal(emb.tensor[r], w)
    assert torch.equal(finder.embed_face_images([small])[0].tensor[0], finder.adaface(finder.preprocess_face(small)).tensor[0])
