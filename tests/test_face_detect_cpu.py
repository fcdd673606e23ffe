"""BlazeFace oracle (oracle/blazeface.py) on the reference's own weights (tests/golden/blazeface_ref.npz): the network
against a torch.nn build, the letterbox geometry, and the decode / suppression / scaling rules the device is held to."""
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import blazeface as bf

GOLD = Path(__file__).parent / "golden" / "blazeface_ref.npz"


@pytest.fixture(scope="module")
def P():
    return bf.load_weights(GOLD)


class _Block(nn.Module):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.stride, self.pad = stride, cout - cin
        self.conv0_tiny = nn.Conv2d(cin, cin, 3, stride, 0 if stride == 2 else 1, groups=cin)
        self.conv1_tiny = nn.Conv2d(cin, cout, 1)

    def forward(self, x):
        h = x
        if self.stride == 2:
            h = nn.functional.pad(x, (0, 2, 0, 2))
            x = nn.functional.max_pool2d(x, 2)
        if self.pad:
            x = nn.functional.pad(x, (0, 0, 0, 0, 0, self.pad))
        return torch.relu(x + self.conv1_tiny(self.conv0_tiny(h)))


class _Net(nn.Module):
    """models/blazeface.py:84-164 as torch.nn modules under the reference's attribute names."""

    def __init__(self):
        super().__init__()
        self.conv_tiny = nn.Conv2d(3, 24, 5, 2)
        self.backbone_tiny = nn.ModuleDict({"list": nn.ModuleList([_Block(*b) for b in bf.BLOCKS])})
        self.final = nn.ModuleDict({"conv0_tiny": nn.Conv2d(96, 96, 3, 2, groups=96), "conv1_tiny": nn.Conv2d(96, 96, 1)})
        for name, c in (("classifier_8", 2), ("classifier_16", 6), ("regressor_8", 32), ("regressor_16", 96)):
            setattr(self, f"{name}_tiny", nn.Conv2d(96, c, 1))

    def forward(self, x):
        b = x.shape[0]
        x = torch.relu(self.conv_tiny(nn.functional.pad(x, (1, 2, 1, 2))))
        for blk in self.backbone_tiny["list"]:
            x = blk(x)
        h = torch.relu(self.final["conv1_tiny"](self.final["conv0_tiny"](nn.functional.pad(x, (0, 2, 0, 2)))))
        c = torch.cat([self.classifier_8_tiny(x).permute(0, 2, 3, 1).reshape(b, -1),
                       self.classifier_16_tiny(h).permute(0, 2, 3, 1).reshape(b, -1)], 1)
        r = torch.cat([self.regressor_8_tiny(x).permute(0, 2, 3, 1).reshape(b, -1, 16),
                       self.regressor_16_tiny(h).permute(0, 2, 3, 1).reshape(b, -1, 16)], 1)
        return r, c


def test_fixture_is_the_reference_file(P):
    with np.load(GOLD) as z:
        stored = sorted(k for k in z.files if k != "firing")
    assert stored == sorted(bf.state_dict_keys()) and len(stored) == 139
    assert sum(v.numel() for v in P.values()) == 139824
    assert P["anchors"].shape == (896, 4)


def test_oracle_equals_torch_nn_build(P):
    net = _Net()
    net.load_state_dict({k: v for k, v in P.items() if k != "anchors"})
    g = torch.Generator().manual_seed(1)
    x = bf.normalize(torch.randint(0, 256, (2, 256, 256, 3), generator=g, dtype=torch.uint8))
    with torch.no_grad():
        r0, c0 = net(x)
        r1, c1 = bf.forward(P, x)
    assert torch.allclose(r0, r1, rtol=0, atol=1e-5) and torch.allclose(c0, c1, rtol=0, atol=1e-5)


def test_firing_image_finds_faces_and_suppresses(P):
    with np.load(GOLD) as z:
        img = z["firing"]
    d = bf.call(P, img)
    kept = d[d[:, 0] != 0]
    assert len(kept) >= 1 and bool((kept[:, 16] >= 0.85).all())
    r, c = bf.forward(P, bf.normalize(torch.from_numpy(img)[None]))
    assert int((bf.sigmoid(c) >= 0.85).sum()) > len(kept)


@pytest.mark.parametrize("h,w", [(256, 256), (640, 640), (480, 640), (1080, 1920), (300, 97), (7, 1000)])
def test_letterbox_geometry(h, w):
    img = torch.zeros(h, w, 3, dtype=torch.uint8)
    x, scale, top, left = bf.letterbox(img)
    assert x.shape == (256, 256, 3)
    assert scale == min(256 / w, 256 / h)
    new_w, new_h = int(w * scale), int(h * scale)
    assert (top, left) == ((256 - new_h) // 2, (256 - new_w) // 2)


def _row(y1, x1, y2, x2, s):
    r = torch.zeros(17)
    r[:4] = torch.tensor([y1, x1, y2, x2])
    r[16] = s
    return r


def test_suppression_counts_suppressed_rows():
    # A suppresses B; B overlaps C but A does not: the reference drops C too, greedy NMS keeps it
    d = torch.zeros(896, 17)
    d[0] = _row(0.0, 0.0, 0.4, 0.4, 0.99)
    d[1] = _row(0.0, 0.15, 0.4, 0.55, 0.95)
    d[2] = _row(0.0, 0.32, 0.4, 0.72, 0.9)
    ref = bf.postprocess(d)
    greedy = bf.postprocess(d, kept_only=True)
    assert ref[0, 16] > 0 and ref[1, 16] == 0 and ref[2, 16] == 0
    assert greedy[2, 16] > 0


def test_ties_go_to_the_lower_anchor_and_zero_boxes_never_suppress():
    d = torch.zeros(896, 17)
    d[5] = _row(0.1, 0.1, 0.2, 0.2, 0.9)
    d[3] = _row(0.5, 0.5, 0.6, 0.6, 0.9)
    d[7] = _row(0.0, 0.0, 0.0, 0.0, 0.9)          # a zero box: IoU 0/0 = NaN compares false
    out = bf.postprocess(d)
    assert torch.equal(out[0], d[3]) and torch.equal(out[1], d[5]) and out[2, 16] == 0.9


def test_keypoints_keep_their_pads():
    d = torch.zeros(896, 17)
    d[0] = _row(0.2, 0.3, 0.4, 0.5, 0.9)
    d[0, 4:16] = 0.25
    got = bf.unletterbox(d, 256 / 640, 64, 0)
    mut = bf.unletterbox(d, 256 / 640, 64, 0, pad_keypoints=True)
    assert not torch.equal(got, mut)
    s = torch.tensor(256 / 640, dtype=torch.float32)
    assert got[0, 5] == (torch.tensor(0.25) * 256) / s and got[0, 0] == (torch.tensor(0.2) * 256 - 64) / s


def test_masked_rows_are_zero(P):
    r = torch.zeros(1, 896, 16)
    c = torch.full((1, 896), -5.0)
    c[0, 10] = 5.0
    d = bf.decode(r, c, P["anchors"])
    assert int((d[0, :, 16] != 0).sum()) == 1 and bool((d[0, torch.arange(896) != 10] == 0).all())


# ---- img_to_face's image arithmetic (oracle/face_align.py) against cv2 itself
import cv2  # noqa: E402

from clearcam_b200.models.blazeface import face_geometry  # noqa: E402
from oracle import face_align as fa  # noqa: E402

CV2 = Path(__file__).parent / "golden" / "face_align_cv2.npz"


def test_resize_and_warp_equal_the_cv2_fixture():
    with np.load(CV2) as z:
        n = sum(1 for k in z.files if k.endswith("_out")) // 2
        for i in range(n):
            dw, dh = (int(v) for v in z[f"rs{i}_size"])
            assert np.array_equal(fa.resize_linear(z[f"rs{i}_in"], dw, dh), z[f"rs{i}_out"]), f"resize case {i}"
            W, H = (int(v) for v in z[f"wa{i}_size"])
            assert np.array_equal(fa.warp_affine(z[f"wa{i}_in"], z[f"wa{i}_M"], (W, H)), z[f"wa{i}_out"]), f"warp case {i}"


def test_resize_equals_cv2_on_fresh_cases():
    g = np.random.default_rng(11)
    for i in range(520):
        h, w = (int(v) for v in g.integers(1, 400, 2))
        if i % 10 == 0:
            h, w = 2 * h, 2 * w                                  # cv2 takes the INTER_AREA path for an exact 2x
        img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if i % 2:
            s = 640 / max(h, w)
            dw, dh = max(1, int(w * s)), max(1, int(h * s))
        else:
            dw, dh = (w // 2, h // 2) if i % 10 == 0 else (int(v) for v in g.integers(1, 300, 2))
        assert np.array_equal(fa.resize_linear(img, dw, dh), cv2.resize(img, (dw, dh))), (h, w, dw, dh)


def test_warp_equals_cv2_on_fresh_cases():
    g = np.random.default_rng(12)
    for i in range(520):
        h, w = (int(v) for v in g.integers(1, 120, 2))
        img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        M = cv2.getRotationMatrix2D((w / 2, h / 2), float(g.uniform(-180, 180)), float(g.uniform(0.1, 5)))
        M[:, 2] += g.uniform(-30, 30, 2)
        if i % 3 == 0:
            M = M.astype(np.float32).astype(np.float64)          # the float32 transform_mat of img_to_face
        W, H = (int(v) for v in g.integers(1, 130, 2))
        assert np.array_equal(fa.warp_affine(img, M, (W, H)), cv2.warpAffine(img, M, (W, H))), i


def _random_rows(g, n=896):
    d = np.zeros((n, 17), np.float32)
    k = int(g.integers(0, 4))
    for j in range(k):
        cy, cx, s = g.uniform(-50, 690), g.uniform(-50, 690), g.uniform(5, 400)
        d[j, :4] = [cy - s / 2, cx - s / 2, cy + s / 2, cx + s / 2]
        d[j, 4:16] = np.repeat([[cx, cy]], 6, 0).ravel() + g.normal(0, s / 4, 12)
        d[j, 16] = g.uniform(0.85, 1)
    return d


def test_geometry_equals_the_reference_lines():
    g = np.random.default_rng(13)
    seen = 0
    for _ in range(400):
        h, w = (int(v) for v in g.integers(40, 2000, 2))
        d = _random_rows(g)
        a = fa.geometry(d.copy(), h, w, rotation=cv2.getRotationMatrix2D)
        b = face_geometry(d.copy(), h, w)
        c = fa.geometry(d.copy(), h, w)
        assert (a is None) == (b is None) == (c is None)
        if a is not None:
            seen += 1
            for u, v, t in zip(a, b, c):
                assert np.array_equal(np.asarray(u), np.asarray(v)) and np.array_equal(np.asarray(u), np.asarray(t))
    assert seen > 50


def test_alignment_mutations_change_the_answer(P):
    g = np.random.default_rng(14)
    rounded = 0
    for _ in range(200):
        h, w = (int(v) for v in g.integers(40, 2000, 2))
        d = _random_rows(g)
        a, b = fa.geometry(d.copy(), h, w), fa.geometry(d.copy(), h, w, rounded_crop=True)
        if a is not None and b is not None and a[:4] != b[:4]:
            rounded += 1
    assert rounded > 0
    with np.load(GOLD) as z:
        img = z["firing"]
    det = lambda c: bf.call(P, c).numpy()                                # noqa: E731
    face = fa.img_to_face(det, img)
    assert face is not None and face.shape == (112, 112, 3)
    geo = fa.geometry(det(fa.canvas(img)).astype(np.float32), *img.shape[:2])
    assert not np.array_equal(fa.align(img, geo, swap=False), face)
    # the whole chain with cv2 in place of the restated arithmetic gives the same face
    canvas = cv2.copyMakeBorder(cv2.resize(img, (640, 640)), 0, 0, 0, 0, cv2.BORDER_CONSTANT, value=[0, 0, 0])
    x1, y1, x2, y2, rot, nw, nh, tm = face_geometry(det(canvas).astype(np.float32), *img.shape[:2])
    ref = cv2.cvtColor(cv2.warpAffine(cv2.warpAffine(img[y1:y2, x1:x2], rot, (nw, nh)), tm, (112, 112)), cv2.COLOR_RGB2BGR)
    assert np.array_equal(ref, face)
