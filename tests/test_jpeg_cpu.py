"""oracle/jpeg.py against cv2.imencode, byte for byte, and the argument checks of the JPEG entry points (no GPU needed).

The oracle is what the GPU encoder is held to, so it is pinned here on a broad case set: every size up to 33 x 33, sizes
around the 8 / 16 block edges, random sizes up to 400, noise, natural crops, flat and checkerboard images, every quality
class, and crops of I420 frames at odd offsets.  Counts from the oracle show that the set reaches the rare paths, and
each of the usual mistakes changes the bytes of at least one case."""
import ctypes
import os

import numpy as np
import pytest

from oracle import jpeg as oj
from oracle.yuv import i420_to_bgr

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jpeg_cv2.npz")
QUALITIES = [0, 1, 10, 50, 75, 85, 95, 100]


def _golden_cases():
    g = np.load(GOLDEN)
    k, out = 0, []
    while f"img{k}" in g:
        out.append((g[f"img{k}"], [int(q) for q in g[f"q{k}"]], {int(q): g[f"jpg{k}_{q}"].tobytes() for q in g[f"q{k}"]}))
        k += 1
    return out


def _cases():
    """-> list of (name, BGR image, quality)"""
    rng = np.random.default_rng(2024)
    out = []
    nat = [img for img, _, _ in _golden_cases()[:10]]      # natural crops of MOT16-03 frames
    for w in range(1, 34):
        for h in range(1, 34):
            q = QUALITIES[(w * 7 + h) % len(QUALITIES)]
            src = nat[(w + h) % len(nat)]
            img = src[:h, :w] if src.shape[0] >= h and src.shape[1] >= w else rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            if (w * h) % 3 == 0:
                img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            out.append((f"size{w}x{h}", img, q))
    for i, base in enumerate((8, 16, 32, 48, 64, 96, 128)):
        for dw in (-1, 0, 1):
            for dh in (-1, 0, 1):
                w, h = base + dw, base + 2 * dh
                img = nat[(i + dw + dh) % len(nat)]
                img = img[:h, :w] if img.shape[0] >= h and img.shape[1] >= w else rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
                out.append((f"edge{w}x{h}", img, QUALITIES[(i + dw + 3 * dh) % len(QUALITIES)]))
    for i in range(24):
        w, h = (int(v) for v in rng.integers(1, 401, 2))
        yy, xx = np.mgrid[0:h, 0:w]
        img = np.stack([(xx * (1 + c) + yy * (3 - c)) % 256 for c in range(3)], -1) + rng.normal(0, 8, (h, w, 3))
        out.append((f"random{w}x{h}", np.clip(img, 0, 255).astype(np.uint8), QUALITIES[i % len(QUALITIES)]))
    for q in QUALITIES:
        out.append((f"noise-q{q}", rng.integers(0, 256, (47, 61, 3), dtype=np.uint8), q))
        out.append((f"solid-q{q}", np.full((37, 45, 3), (17, 130, 244), np.uint8), q))
        chk = ((np.indices((64, 72)).sum(0) // 8) % 2 * 255).astype(np.uint8)
        out.append((f"checker8-q{q}", np.repeat(chk[..., None], 3, 2), q))
        chk = ((np.indices((50, 51)).sum(0) // 3) % 2 * 255).astype(np.uint8)
        out.append((f"checker3-q{q}", np.stack([chk, 255 - chk, chk], -1), q))
    for i, img in enumerate(nat):
        out.append((f"natural{i}", img, QUALITIES[(i * 3) % len(QUALITIES)]))
    # crops of I420 frames (what a yuv420p camera's frame is, converted as cv2 does) at odd offsets and at the edges
    yuv = rng.integers(0, 256, (120 * 3 // 2, 160), dtype=np.uint8)
    yuv[:120] = (np.add.outer(np.arange(120), np.arange(160)) % 256).astype(np.uint8)
    bgr = i420_to_bgr(yuv)
    for i, (x1, y1, x2, y2) in enumerate([(1, 1, 40, 30), (3, 5, 160, 120), (0, 0, 17, 33), (151, 101, 160, 120),
                                          (77, 13, 131, 100), (9, 0, 10, 1)]):
        out.append((f"i420-{x1},{y1}", bgr[y1:y2, x1:x2], QUALITIES[(i + 5) % len(QUALITIES)]))
    return out


CASES = _cases()


def test_case_set_is_large():
    assert len(CASES) >= 300


@pytest.mark.parametrize("part", range(8))
def test_oracle_equals_cv2(part):
    cv2 = pytest.importorskip("cv2")
    for name, img, q in CASES[part::8]:
        want = cv2.imencode(".jpg", np.ascontiguousarray(img), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
        assert oj.encode(img, q) == want, (name, q)


def test_quality_clamp_and_bound():
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(3).integers(0, 256, (40, 40, 3), dtype=np.uint8)
    enc = lambda q: cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()   # noqa: E731
    assert enc(0) == enc(1) == oj.encode(img, 0)
    assert enc(101) == enc(100)
    assert len(oj.headers(40, 40, 95)) == oj.HEADER_BYTES
    for q in (100, 1):
        assert len(oj.encode(img, q)) <= oj.bound(40, 40)


def test_oracle_equals_the_golden_file():
    n = 0
    for img, qs, want in _golden_cases():
        for q in qs:
            assert oj.encode(img, q) == want[q], q
            n += 1
    assert n >= 50


def test_case_set_reaches_the_rare_paths():
    stats = {}
    for _, img, q in CASES:
        oj.encode(img, q, stats=stats)
    assert stats["zrl"] > 0                      # runs of 16+ zeros before a nonzero coefficient
    assert stats["ff"] > 0                       # 0xFF bytes that need stuffing
    assert stats["max_dc_cat"] >= 10             # DC differences of 10+ bits
    assert stats["right_dummies"] > 0 and stats["bottom_dummies"] > 0
    assert stats["even_h_chroma_pad"] > 0        # H even, not a multiple of 16: the chroma rows replicated after downsampling


@pytest.mark.parametrize("variant", [{"pad16_rows": True}, {"dummy_dc": False}, {"cols_after": True}, {"stuffing": False}])
def test_each_usual_mistake_changes_some_bytes(variant):
    changed = [name for name, img, q in CASES if oj.encode(img, q, **dict(variant)) != oj.encode(img, q)]
    assert changed, variant


# ------------------------------------------------------------------------------------------------ argument checks
def test_jpeg_entry_points_reject_bad_arguments():
    """Every check runs before anything is launched: the device pointers below are never dereferenced."""
    from clearcam_b200._lib import lib
    h = lib()
    fake = ctypes.c_void_p(1 << 20)
    b = ctypes.c_int64(0)
    need = ctypes.c_size_t(0)

    def refused(rc, *words):
        msg = h.cc_last_error().decode()
        assert rc == -1 and all(w in msg for w in words), (rc, msg, words)

    assert h.cc_jpeg_bound(100, 100, ctypes.byref(b)) == 0 and b.value == oj.bound(100, 100)
    refused(h.cc_jpeg_bound(0, 5, ctypes.byref(b)), "cc_jpeg_bound", "bad size")
    refused(h.cc_jpeg_bound(65536, 5, ctypes.byref(b)), "cc_jpeg_bound", "bad size")
    refused(h.cc_jpeg_bound(5, 5, None), "cc_jpeg_bound", "NULL")

    rects = np.array([[0, 0, 0, 100, 80], [1, 10, 10, 50, 50]], np.int32)
    bounds = [oj.bound(100, 80), oj.bound(40, 40)]
    offs = np.array([0, bounds[0]], np.int64)
    cap = sum(bounds)

    def enc(frames=fake, n=2, H=240, W=320, fmt=1, r=rects, K=2, q=95, out=fake, cap=cap, offsets=offs, lengths=fake, ws=fake,
            wsb=1 << 30, need=ctypes.byref(need)):
        return h.cc_jpeg_encode_crops(frames, n, H, W, fmt, None if r is None else r.ctypes.data, K, q, out, cap,
                                      None if offsets is None else offsets.ctypes.data, lengths, ws, wsb, need, None)

    assert enc(out=None) == 0 and need.value > 0
    refused(enc(frames=None), "cc_jpeg_encode_crops", "null pointer")
    refused(enc(r=None), "cc_jpeg_encode_crops", "null pointer")
    refused(enc(n=0), "cc_jpeg_encode_crops", "bad sizes")
    refused(enc(fmt=3), "cc_jpeg_encode_crops", "unknown source format 3")
    refused(enc(fmt=-1), "cc_jpeg_encode_crops", "unknown source format")
    refused(enc(fmt=2, H=241), "cc_jpeg_encode_crops", "even height and width")
    refused(enc(fmt=2, W=321), "cc_jpeg_encode_crops", "even height and width")
    refused(enc(q=-1), "cc_jpeg_encode_crops", "quality -1")
    refused(enc(q=101), "cc_jpeg_encode_crops", "quality 101")
    refused(enc(r=np.array([[0, 5, 5, 5, 9], [1, 10, 10, 50, 50]], np.int32)), "rect 0", "empty or outside")
    refused(enc(r=np.array([[0, 0, 0, 100, 80], [1, 10, 10, 321, 50]], np.int32)), "rect 1", "empty or outside")
    refused(enc(r=np.array([[0, 0, 0, 100, 80], [2, 10, 10, 50, 50]], np.int32)), "rect 1", "frame 2")
    refused(enc(offsets=None), "out_offsets and d_lengths")
    refused(enc(lengths=None), "out_offsets and d_lengths")
    refused(enc(wsb=need.value - 1), "workspace of", "too small")
    refused(enc(ws=None), "too small")
    refused(enc(ws=ctypes.c_void_p((1 << 20) + 16)), "256-byte aligned")
    refused(enc(lengths=ctypes.c_void_p((1 << 20) + 4)), "8-byte aligned")
    refused(enc(cap=cap - 1), "crop 1", "exceeds the output capacity")
    refused(enc(offsets=np.array([0, bounds[0] - 1], np.int64)), "crops 0 and 1 overlap")
    refused(enc(offsets=np.array([bounds[1] + 1, 0], np.int64)), "crop 0", "exceeds")
    refused(enc(offsets=np.array([-1, bounds[0]], np.int64)), "crop 0", "exceeds")
    assert enc(offsets=np.array([bounds[1], 0], np.int64), cap=cap, out=None) == 0      # query ignores the offsets

    def coef(fmt=1, H=240, q=95, d=fake, nb=ctypes.byref(b)):
        return h.cc_jpeg_coeffs(fake, 2, H, 320, fmt, rects.ctypes.data, 2, q, d, nb, None)

    assert coef(d=None) == 0
    g = [oj.geometry(100, 80), oj.geometry(40, 40)]
    assert b.value == sum(6 * x["mw"] * x["mh"] for x in g)
    refused(coef(fmt=7), "cc_jpeg_coeffs", "unknown source format 7")
    refused(coef(fmt=2, H=239), "cc_jpeg_coeffs", "even height")
    refused(coef(q=200), "cc_jpeg_coeffs", "quality 200")
    refused(coef(d=ctypes.c_void_p((1 << 20) + 2)), "cc_jpeg_coeffs", "4-byte aligned")
