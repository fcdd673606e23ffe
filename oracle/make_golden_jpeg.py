"""Writes tests/golden/jpeg_cv2.npz: images and the bytes cv2.imencode(".jpg") gives for them, so the tests pin
oracle/jpeg.py and the GPU encoder to cv2 without needing cv2 or the video.

    python oracle/make_golden_jpeg.py [path/to/MOT16-03.mp4]

Contents, per case k: "img{k}" uint8 BGR [h,w,3], "q{k}" int32 [n] qualities, "jpg{k}_{q}" uint8 = cv2's bytes.  Cases:
crops of natural content cut from MOT16-03 frames (the reference's test video) at assorted sizes and offsets, solid and
checkerboard images, noise, and crops of I420 frames: for those, "yuv{k}" uint8 [H*3/2,W] and "rect{k}" int32 (x1, y1,
x2, y2) are stored too, and img{k} is the crop of cv2.cvtColor(yuv, COLOR_YUV2BGR_I420)."""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "jpeg_cv2.npz")
VIDEO = "/root/reference/test/videos/MOT16-03.mp4"

# (frame, x1, y1, w, h): people, street and the frame edges of the 960x540 video
NATURAL = [(0, 350, 200, 100, 100), (0, 1, 3, 131, 97), (0, 710, 360, 250, 180), (0, 333, 77, 48, 64),
           (150, 450, 250, 160, 120), (150, 0, 0, 17, 23), (150, 927, 507, 33, 33), (300, 600, 150, 200, 150),
           (300, 320, 289, 33, 250), (300, 501, 251, 96, 200)]
QUALITIES = [50, 85, 95]


def frames(path, idx):
    cap = cv2.VideoCapture(path)
    out, i = {}, 0
    while len(out) < len(idx):
        ok, f = cap.read()
        if not ok:
            raise RuntimeError(f"{path}: ended at frame {i}")
        if i in idx:
            out[i] = f
        i += 1
    return out


def cases(path):
    fr = frames(path, sorted({c[0] for c in NATURAL}))
    out = []
    for f, x, y, w, h in NATURAL:
        out.append({"img": fr[f][y:y + h, x:x + w]})
    rng = np.random.default_rng(8)
    out.append({"img": np.full((24, 40, 3), (30, 200, 90), np.uint8)})
    chk = ((np.indices((40, 42)).sum(0) // 4) % 2 * 255).astype(np.uint8)
    out.append({"img": np.repeat(chk[..., None], 3, 2)})
    out.append({"img": rng.integers(0, 256, (31, 29, 3), dtype=np.uint8), "q": [10, 95, 100]})
    # I420: a natural 112 x 160 region as yuv420p, crops at odd offsets and touching each edge
    yuv = cv2.cvtColor(np.ascontiguousarray(fr[0][250:362, 400:560]), cv2.COLOR_BGR2YUV_I420)
    bgr = cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_I420)
    for x1, y1, x2, y2 in [(1, 3, 100, 80), (0, 0, 160, 112), (77, 51, 160, 112), (5, 0, 38, 17)]:
        out.append({"img": bgr[y1:y2, x1:x2], "yuv": yuv, "rect": np.array([x1, y1, x2, y2], np.int32)})
    return out


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else VIDEO
    data = {}
    for k, c in enumerate(cases(path)):
        img = np.ascontiguousarray(c["img"])
        qs = c.get("q", QUALITIES)
        data[f"img{k}"] = img
        data[f"q{k}"] = np.array(qs, np.int32)
        for q in qs:
            data[f"jpg{k}_{q}"] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].reshape(-1)
        if "yuv" in c:
            data[f"yuv{k}"], data[f"rect{k}"] = c["yuv"], c["rect"]
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes, cv2", cv2.__version__, sum(1 for k in data if k.startswith("img")), "cases")


if __name__ == "__main__":
    main()
