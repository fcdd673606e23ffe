"""Writes tests/golden/yuv420_cv2.npz: small I420 frames and OpenCV's conversion of them, so the CPU tests pin
oracle/yuv.py to cv2 without needing cv2.

    python oracle/make_golden_yuv.py

Contents: for each case k, "yuv{k}" uint8 [H*3/2, W] and "bgr{k}" = cv2.cvtColor(yuv, COLOR_YUV2BGR_I420).  Cases: random
planes at a few even sizes, and planes at the extremes of the conversion (Y < 16, Y = 255, U / V at 0 and 255 in every
combination), which exercise the clamp at 0, the saturation at 255 and the arithmetic shift of negative sums."""
import os

import cv2
import numpy as np

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "yuv420_cv2.npz")


def cases():
    rng = np.random.default_rng(420)
    out = [rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8) for h, w in [(2, 2), (4, 6), (22, 30), (36, 64)]]
    # extremes: every (Y, U, V) in {0, 8, 15, 16, 17, 128, 235, 240, 254, 255} x {0, 1, 127, 128, 129, 254, 255}^2,
    # one 2x2 block per combination (chroma is shared by the block)
    ys, cs = [0, 8, 15, 16, 17, 128, 235, 240, 254, 255], [0, 1, 127, 128, 129, 254, 255]
    combos = [(y, u, v) for y in ys for u in cs for v in cs]
    nb = len(combos)                     # blocks along one row of a 2-row frame
    H, W = 2, 2 * nb
    Y = np.repeat(np.array([c[0] for c in combos], np.uint8), 2)[None].repeat(2, 0)
    U = np.array([c[1] for c in combos], np.uint8)[None]
    V = np.array([c[2] for c in combos], np.uint8)[None]
    out.append(np.concatenate([Y.reshape(-1), U.reshape(-1), V.reshape(-1)]).reshape(H * 3 // 2, W))
    return out


def main():
    data = {}
    for k, yuv in enumerate(cases()):
        data[f"yuv{k}"] = yuv
        data[f"bgr{k}"] = cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_I420)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, "cv2", cv2.__version__, {k: v.shape for k, v in data.items()})


if __name__ == "__main__":
    main()
