"""Writes tests/golden/jpeg_decode_cv2.npz: JPEG files of every variant the device decoder takes, a few it leaves to the host,
and cv2.imdecode(file, IMREAD_COLOR) of each.

    python oracle/make_golden_jpeg_decode.py

Keys: file{k} (uint8 bytes), want{k} (BGR uint8 [h, w, 3], absent where cv2 returns None), status{k} (oracle.jpeg_decode
status), name{k}.  Content: seeded gradients with noise, small sizes so the fixture stays well under 1 MB."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import jpeg as oj  # noqa: E402
from oracle import jpeg_decode as od  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "jpeg_decode_cv2.npz")


def image(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([(xx * (1.5 + c) + yy * (2.0 - 0.5 * c) + 50 * c) % 256 for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)


def cases():
    import cv2
    S = {444: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, 422: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
         440: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, 420: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
    out = []
    sizes = [(1, 1), (7, 5), (16, 16), (17, 31), (33, 47), (61, 40), (90, 123)]
    k = 0
    for samp in (420, 422, 440, 444, "grey"):
        for (h, w) in sizes:
            k += 1
            img = image(h, w, k)
            q = (95, 75, 30, 100, 5, 85, 60)[k % 7]
            p = [cv2.IMWRITE_JPEG_QUALITY, q]
            if samp != "grey":
                p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, S[samp]]
            if k % 3 == 0:
                p += [cv2.IMWRITE_JPEG_RST_INTERVAL, (1, 3, 7)[k % 9 // 3]]
            if k % 4 == 0:
                p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
            if k % 5 == 0:
                p += [cv2.IMWRITE_JPEG_LUMA_QUALITY, 40, cv2.IMWRITE_JPEG_CHROMA_QUALITY, 90]
            src = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if samp == "grey" else img
            out.append((f"{samp}_{w}x{h}_q{q}", cv2.imencode(".jpg", src, p)[1].tobytes()))
    out.append(("project_encoder_45x29", oj.encode(image(29, 45, 99), 95)))
    img = image(40, 56, 100)
    out.append(("progressive", cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()))
    base = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
    exif = b"Exif\x00\x00" + b"MM\x00\x2a\x00\x00\x00\x08" + b"\x00\x01" + b"\x01\x12\x00\x03\x00\x00\x00\x01\x00\x06\x00\x00" + b"\x00" * 4
    out.append(("exif_orientation_6", base[:2] + b"\xff\xe1" + (len(exif) + 2).to_bytes(2, "big") + exif + base[2:]))
    out.append(("truncated_scan", base[:len(base) * 2 // 3]))
    return out


def main():
    import cv2
    data = {}
    for k, (name, f) in enumerate(cases()):
        data[f"file{k}"] = np.frombuffer(f, np.uint8)
        want = cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)
        if want is not None:
            data[f"want{k}"] = want
        data[f"status{k}"] = np.array(od.decode(f)[0])
        data[f"name{k}"] = np.array(name)
    np.savez_compressed(OUT, **data)
    print(OUT, os.path.getsize(OUT), "bytes,", sum(1 for key in data if key.startswith("file")), "files")


if __name__ == "__main__":
    main()
