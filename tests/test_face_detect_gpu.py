"""BlazeFace on the GPU (csrc/blazeface.cu) against the oracle (oracle/blazeface.py) on the reference's own weights.

* Raw boxes and scores for all 896 anchors at B = 1, 3, 64 and 257 (images of mixed sizes) against a float64 forward: per
  element, the GPU's error may be at most 8 times the fp32 oracle's own error there plus 128 times that error's RMS over
  the tensor.  The GPU sums each 1x1 conv in one sequential fma chain where the CPU convolution blocks its sums; on an
  H100 80GB HBM3 (700 W) its worst error at B = 257 was about 49 times the RMS.
* Each image of a batch is bit-equal to its own B = 1 call.
* Decode, order, suppression and scaling are exact on injected head outputs: ties, all masked, every anchor above 0.85.
* The firing fixture image gives the oracle's detections: the same rows kept, values within the bar.
* Nothing past the outputs is written; argument errors raise before any launch.
* img_to_face: the 640x640 canvas equals cv2.resize + copyMakeBorder; the two warps and the channel swap equal cv2 for
  given detections (clamped crops, eyes at any angle); the firing image gives exactly the cv2 chain's face on the device's
  detections, and on the fp32 oracle's detections the same crop and a face within resampling; `faces_from_images` ->
  `embed_faces` equals `img_to_face` + `adaface` per image.
"""
import ctypes
from pathlib import Path

import numpy as np
import pytest
import torch

from clearcam_b200._lib import CCError, cc_frame, lib, ptr, stream_ptr
from clearcam_b200.models.blazeface import BlazeFace
from clearcam_b200.models.objects import ObjectFinder
from oracle import blazeface as bf

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden" / "blazeface_ref.npz"


@pytest.fixture(scope="module")
def P():
    return bf.load_weights(GOLD)


@pytest.fixture(scope="module")
def det(P):
    return BlazeFace({k: v.numpy() for k, v in P.items()})


@pytest.fixture(scope="module")
def firing():
    with np.load(GOLD) as z:
        return z["firing"]


def _images(B, seed):
    g = np.random.default_rng(seed)
    sizes = [(256, 256), (640, 640), (480, 640), (97, 300), (333, 129), (720, 1280)]
    return [g.integers(0, 256, (*sizes[(i + seed) % len(sizes)], 3), dtype=np.uint8) for i in range(B)]


def _bar_ok(got, o32, o64):
    e32 = (o32.double() - o64).abs()
    bar = 8 * e32 + 128 * e32.pow(2).mean().sqrt()
    err = (got.double().cpu() - o64).abs()
    return bool((err <= bar).all()), float((err / bar).max())


@pytest.mark.parametrize("B", [1, 3, 64, 257])
def test_raw_outputs_against_float64(det, P, B):
    ims = _images(B, B)
    dets, boxes, scores = det.forward(ims)
    x = torch.stack([bf.letterbox(torch.from_numpy(im))[0] for im in ims])
    xn = bf.normalize(x)
    with torch.no_grad():
        r32, c32 = bf.forward(P, xn)
        r64, c64 = bf.forward(P, xn.double(), torch.float64)
    ok_r, wr = _bar_ok(boxes, r32, r64)
    ok_c, wc = _bar_ok(scores, c32, c64)
    assert ok_r and ok_c, f"worst error / bar: boxes {wr:.3f}, scores {wc:.3f}"
    # the decode of the device's own head outputs is exact
    want = torch.stack([bf.unletterbox(bf.postprocess(bf.decode(boxes[i:i + 1].cpu(), scores[i:i + 1].cpu(), P["anchors"])[0]),
                                       *bf.letterbox(torch.from_numpy(ims[i]))[1:]) for i in range(B)])
    assert torch.equal(dets.cpu(), want)


def test_batch_rows_equal_single_calls(det):
    ims = _images(9, 4)
    dets, boxes, scores = det.forward(ims)
    for i, im in enumerate(ims):
        d1, b1, s1 = det.forward([im])
        assert torch.equal(d1[0], dets[i]) and torch.equal(b1[0], boxes[i]) and torch.equal(s1[0], scores[i])


def _oracle_decode(P, r, c, sizes):
    out = []
    for i, (h, w) in enumerate(sizes):
        _, scale, top, left = bf.letterbox(torch.zeros(h, w, 3, dtype=torch.uint8))
        out.append(bf.unletterbox(bf.postprocess(bf.decode(r[i:i + 1], c[i:i + 1], P["anchors"])[0]), scale, top, left))
    return torch.stack(out)


@pytest.mark.parametrize("case", ["ties", "all_masked", "all_above", "random"])
def test_decode_exact_on_injected_heads(det, P, case):
    g = torch.Generator().manual_seed(7)
    B = 5
    r = torch.randn(B, 896, 16, generator=g) * 20
    if case == "ties":
        c = torch.where(torch.rand(B, 896, generator=g) < 0.3, 3.0, -3.0)   # many equal scores above 0.85
        r[:, ::2] = r[:, 1::2]                                               # and pairs of identical boxes
    elif case == "all_masked":
        c = torch.full((B, 896), -1.0)
    elif case == "all_above":
        c = torch.rand(B, 896, generator=g) * 200 + 2                        # clipped at 100 on the way
    else:
        c = torch.randn(B, 896, generator=g) * 4
    sizes = [(640, 640), (480, 640), (97, 300), (256, 256), (1080, 1920)]
    got = det.decode(r, c, sizes).cpu()
    assert torch.equal(got, _oracle_decode(P, r, c, sizes))


def test_firing_image_gives_the_oracles_faces(det, P, firing):
    for img in (firing, np.ascontiguousarray(np.kron(firing, np.ones((2, 2, 1), np.uint8))[:500])):
        want = bf.call(P, img)
        got = det(img).numpy()
        assert got.shape == (896, 17)
        kept = np.flatnonzero(want[:, 0].numpy() != 0)
        assert len(kept) >= 1 and np.array_equal(np.flatnonzero(got[:, 0] != 0), kept)
        assert np.allclose(got[kept], want.numpy()[kept], rtol=1e-4, atol=1e-2)


def test_finder_builds_the_detector(P, firing):
    from oracle import adaface as oa
    f = ObjectFinder()
    f.init_face(weights=oa.synthetic_weights(seed=5), detector={k: v.numpy() for k, v in P.items()})
    assert f.blazeface is not None and f.blazeface(firing).numpy().shape == (896, 17)
    g = ObjectFinder()
    g.init_face(weights=oa.synthetic_weights(seed=5))
    assert g.blazeface is None


def test_sentinels_after_outputs(det):
    ims = [torch.from_numpy(im).cuda() for im in _images(3, 2)]
    B, pad = 3, 4096
    det._workspace(B)
    boxes = torch.full((B * 896 * 16 + pad,), 7.25, device="cuda")
    scores = torch.full((B * 896 + pad,), 7.25, device="cuda")
    dets = torch.full((B * 896 * 17 + pad,), 7.25, device="cuda")
    table = (cc_frame * B)(*[cc_frame(t.data_ptr(), 0, t.shape[0], t.shape[1]) for t in ims])
    assert lib().cc_blazeface_forward(det._h, table, B, ptr(boxes), ptr(scores), ptr(dets), stream_ptr()) == 0
    torch.cuda.synchronize()
    for t, n in ((boxes, B * 896 * 16), (scores, B * 896), (dets, B * 896 * 17)):
        assert bool((t[n:] == 7.25).all())
    want, wb, ws = det.forward(ims)
    assert torch.equal(dets[:B * 896 * 17].view(B, 896, 17), want)


def test_argument_errors(det, P):
    with pytest.raises(ValueError):
        det.forward([np.zeros((10, 10), np.uint8)])
    with pytest.raises(ValueError):
        det.forward([np.zeros((10, 10, 3), np.float32)])
    with pytest.raises(ValueError):
        det.forward([])
    with pytest.raises(CCError):
        det.forward([np.zeros((1, 1000, 3), np.uint8)])                    # resizes to an empty image
    with pytest.raises(ValueError):
        det.decode(torch.zeros(2, 896, 16), torch.zeros(2, 895), [(10, 10)] * 2)
    with pytest.raises(ValueError):
        det.decode(torch.zeros(2, 896, 16), torch.zeros(2, 896), [(10, 10)])
    with pytest.raises(CCError):
        det.decode(torch.zeros(1, 896, 16), torch.zeros(1, 896), [(0, 10)])
    bad = dict(P)
    bad.pop("anchors")
    with pytest.raises(CCError):
        BlazeFace({k: v.numpy() for k, v in bad.items()})
    bad = {k: v.numpy() for k, v in P.items()}
    bad["conv_tiny.bias"] = bad["conv_tiny.bias"][:20]
    with pytest.raises(CCError):
        BlazeFace(bad)
    L = lib()
    img = torch.zeros(64, 64, 3, dtype=torch.uint8, device="cuda")
    out = torch.empty(2 * 896 * 17, device="cuda")
    t1 = (cc_frame * 1)(cc_frame(img.data_ptr(), 2, 64, 64))                 # I420 is not taken
    assert L.cc_blazeface_forward(det._h, t1, 1, ptr(out), ptr(out), ptr(out), stream_ptr()) != 0
    t3 = (cc_frame * 1)(cc_frame(img.data_ptr(), 3, 64, 64))                 # nor RGB, which only the crops take
    assert L.cc_blazeface_forward(det._h, t3, 1, ptr(out), ptr(out), ptr(out), stream_ptr()) != 0
    t0 = (cc_frame * 1)(cc_frame(None, 0, 64, 64))
    assert L.cc_blazeface_forward(det._h, t0, 1, ptr(out), ptr(out), ptr(out), stream_ptr()) != 0
    fresh = BlazeFace({k: v.numpy() for k, v in P.items()})                 # no workspace set
    t2 = (cc_frame * 1)(cc_frame(img.data_ptr(), 0, 64, 64))
    assert L.cc_blazeface_forward(fresh._h, t2, 1, ptr(out), ptr(out), ptr(out), stream_ptr()) != 0
    assert L.cc_blazeface_forward(det._h, t2, 0, ptr(out), ptr(out), ptr(out), stream_ptr()) != 0
    sz = ctypes.c_size_t()
    assert L.cc_blazeface_workspace_bytes(det._h, 0, ctypes.byref(sz)) != 0
    assert L.cc_blazeface_set_workspace(det._h, ctypes.c_void_p(det._ws.data_ptr() + 4), 1024) != 0


# ---- img_to_face on the device: the canvas, the two warps and the channel swap, pixel for pixel with cv2
import cv2  # noqa: E402

from clearcam_b200._lib import cc_face_warp  # noqa: E402
from clearcam_b200.models.blazeface import align_faces, face_canvas, face_geometry  # noqa: E402
from oracle import face_align as fa  # noqa: E402


def test_canvas_equals_cv2():
    g = np.random.default_rng(21)
    sizes = [(720, 1280), (1280, 720), (640, 640), (97, 300), (1080, 1920), (50, 33), (333, 129), (2, 900), (2000, 1999)]
    ims = [g.integers(0, 256, (*s, 3), dtype=np.uint8) for s in sizes]
    got = face_canvas([torch.from_numpy(im).cuda() for im in ims]).cpu().numpy()
    for im, c in zip(ims, got):
        h, w = im.shape[:2]
        s = 640 / max(h, w)
        r = cv2.resize(im, (int(w * s), int(h * s)))
        dw, dh = 640 - r.shape[1], 640 - r.shape[0]
        want = cv2.copyMakeBorder(r, dh // 2, dh - dh // 2, dw // 2, dw - dw // 2, cv2.BORDER_CONSTANT, value=[0, 0, 0])
        assert np.array_equal(c, want), (h, w)


def _rows(g):
    d = np.zeros((896, 17), np.float32)
    cy, cx, s = g.uniform(-40, 680), g.uniform(-40, 680), g.uniform(60, 500)
    d[0, :4] = [cy - s / 2, cx - s / 2, cy + s / 2, cx + s / 2]
    ang = g.uniform(-np.pi, np.pi)                                   # eyes at any angle, including upside down
    r = g.uniform(5, s / 2)
    d[0, 4:8] = [cx - r * np.cos(ang), cy - r * np.sin(ang), cx + r * np.cos(ang), cy + r * np.sin(ang)]
    d[0, 16] = 0.9
    return d


def test_alignment_equals_cv2_for_given_detections():
    g = np.random.default_rng(22)
    jobs, want = [], []
    clamped = 0
    while len(jobs) < 60:
        h, w = (int(v) for v in g.integers(60, 1500, 2))
        geo = face_geometry(_rows(g), h, w)
        if geo is None:
            continue
        img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        x1, y1, x2, y2, rot, nw, nh, tm = geo
        clamped += x1 == 0 or y1 == 0 or x2 == w or y2 == h
        jobs.append((torch.from_numpy(img).cuda(), geo))
        want.append(cv2.cvtColor(cv2.warpAffine(cv2.warpAffine(img[y1:y2, x1:x2], rot, (nw, nh)), tm, (112, 112)), cv2.COLOR_RGB2BGR))
    assert clamped >= 10
    got = align_faces(jobs).cpu().numpy()
    for k in range(len(jobs)):
        assert np.array_equal(got[k], want[k]), k


@pytest.fixture(scope="module")
def face_finder(P):
    from oracle import adaface as oa
    f = ObjectFinder()
    f.init_face(weights=oa.synthetic_weights(seed=5), detector={k: v.numpy() for k, v in P.items()})
    return f


def test_firing_image_gives_the_oracles_face(face_finder, P, firing):
    got = face_finder.img_to_face(firing)
    assert got is not None and got.shape == (112, 112, 3) and got.dtype == np.uint8
    # exact: the cv2-exact oracle chain on the device's own detections
    dev = lambda c: face_finder.blazeface(c).numpy()                          # noqa: E731
    assert np.array_equal(got, fa.img_to_face(dev, firing))
    # the fp32 oracle's own detections differ from the device's in the last bits (within the float64 bar above), so the
    # eye transform moves by a fraction of a pixel: the same crop and rotated size, the same face up to resampling
    orc = lambda c: bf.call(P, c).numpy()                                      # noqa: E731
    g_dev = fa.geometry(dev(fa.canvas(firing)).astype(np.float32), *firing.shape[:2])
    g_orc = fa.geometry(orc(fa.canvas(firing)).astype(np.float32), *firing.shape[:2])
    assert g_dev[:4] == g_orc[:4] and g_dev[5:7] == g_orc[5:7]
    want = fa.img_to_face(orc, firing)
    diff = np.abs(got.astype(int) - want)
    assert diff.mean() < 1.0 and np.mean(diff > 8) < 0.01, (diff.mean(), diff.max(), np.mean(diff > 8))


def test_faces_from_images_then_embed_equals_per_image(face_finder, firing):
    g = np.random.default_rng(23)
    big = np.ascontiguousarray(np.kron(firing, np.ones((5, 5, 1), np.uint8)))               # 1280x1280: the 2x area path
    ims = [firing, g.integers(0, 256, (300, 500, 3), dtype=np.uint8), big, np.ascontiguousarray(firing[:, 20:])]
    faces, rows = face_finder.faces_from_images(ims)
    emb = face_finder.embed_faces(faces).cpu()
    assert rows[0] is not None and faces.shape == (sum(r is not None for r in rows), 112, 112, 3)
    for im, r in zip(ims, rows):
        one = face_finder.img_to_face(im)
        assert (one is None) == (r is None)
        if r is not None:
            assert np.array_equal(faces[r].cpu().numpy(), one)
            assert torch.equal(face_finder.adaface(one).tensor.cpu()[0], emb[r])


def test_alignment_argument_errors(face_finder, det):
    with pytest.raises(CCError, match="detector"):
        ObjectFinder().faces_from_images([np.zeros((10, 10, 3), np.uint8)])
    img = torch.zeros(64, 64, 3, dtype=torch.uint8, device="cuda")
    out = torch.empty(112, 112, 3, dtype=torch.uint8, device="cuda")
    bad = (cc_face_warp * 1)()
    bad[0].src, bad[0].h, bad[0].w = img.data_ptr(), 64, 64
    bad[0].x1, bad[0].y1, bad[0].x2, bad[0].y2, bad[0].rot_w, bad[0].rot_h = 10, 10, 70, 40, 50, 50     # crop past the image
    assert lib().cc_face_align(bad, 1, ptr(out), stream_ptr()) != 0
    assert lib().cc_face_align(bad, 0, ptr(out), stream_ptr()) != 0
    t = (cc_frame * 1)(cc_frame(img.data_ptr(), 2, 64, 64))
    assert lib().cc_face_canvas(t, 1, ptr(out), stream_ptr()) != 0
