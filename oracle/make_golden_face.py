"""Writes tests/golden/face_align_cv2.npz (cv2.resize INTER_LINEAR and cv2.warpAffine outputs made by the installed cv2 for
seeded random sizes, angles and scales: the fixture oracle/face_align.py is held to) and tests/golden/blazeface_ref.npz: the reference's BlazeFace weights and 896 anchors (models/blazeface.safetensors,
139,824 floats), and `firing`, a 256x256x3 uint8 image on which those weights find faces.

No face photo comes with the reference, so the image is derived: gradient ascent with the oracle on the raw scores of
three neighbouring anchors of the 8x8 grid (its large boxes, so that img_to_face keeps the face), from a fixed seed, then rounded to uint8.  The
script checks that the stored image, run through oracle.blazeface.call, keeps at least one row at score >= 0.85 and
suppresses at least one.

    python oracle/make_golden_face.py /path/to/reference/models/blazeface.safetensors
"""
import cv2
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import blazeface as bf  # noqa: E402

TARGETS = (512 + 6 * (3 * 8 + 3), 512 + 6 * (3 * 8 + 3) + 1, 512 + 6 * (3 * 8 + 4))


def firing_image(P, seed=0, steps=300):
    g = torch.Generator().manual_seed(seed)
    z = (torch.rand(1, 3, 256, 256, generator=g) * 0.2 - 0.1).requires_grad_(True)
    opt = torch.optim.Adam([z], lr=0.05)
    for _ in range(steps):
        _, c = bf.forward(P, torch.tanh(z))
        loss = -c[0, list(TARGETS)].clamp(max=4.0).sum()
        opt.zero_grad()
        loss.backward()
        opt.step()
    u = ((torch.tanh(z) + 1) * 127.5).round().clamp(0, 255).to(torch.uint8)
    return u[0].permute(1, 2, 0).contiguous().detach()


def cv2_cases(seed=0, n=40):
    """n resize and n warp cases on small images: inputs, parameters and cv2's outputs."""
    g = np.random.default_rng(seed)
    out = {}
    for i in range(n):
        h, w = (int(v) for v in g.integers(2, 48, 2))
        img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        dw, dh = (int(v) for v in g.integers(1, 64, 2))
        if i % 8 == 0:
            dw, dh = max(1, w // 2), max(1, h // 2)
            img = img[:2 * dh, :2 * dw].copy()
        out[f"rs{i}_in"], out[f"rs{i}_size"] = img, np.array([dw, dh])
        out[f"rs{i}_out"] = cv2.resize(img, (dw, dh))
        h, w = (int(v) for v in g.integers(2, 48, 2))
        img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        M = cv2.getRotationMatrix2D((w / 2, h / 2), float(g.uniform(-180, 180)), float(g.uniform(0.2, 4)))
        M[:, 2] += g.uniform(-10, 10, 2)
        if i % 4 == 0:
            M = M.astype(np.float32).astype(np.float64)
        size = np.array([int(v) for v in g.integers(1, 64, 2)])
        out[f"wa{i}_in"], out[f"wa{i}_M"], out[f"wa{i}_size"] = img, M, size
        out[f"wa{i}_out"] = cv2.warpAffine(img, M, (int(size[0]), int(size[1])))
    return out


def main(src):
    np.savez_compressed(ROOT / "tests" / "golden" / "face_align_cv2.npz", **cv2_cases())
    P = bf.load_weights(src)
    img = firing_image(P)
    d = bf.call(P, img)
    r, c = bf.forward(P, bf.normalize(img[None]))
    n_above = int((bf.sigmoid(c) >= bf.MIN_SCORE).sum())
    n_kept = int((d[:, 0] != 0).sum())
    print(f"anchors >= 0.85: {n_above}, kept after suppression: {n_kept}")
    assert n_kept >= 1 and n_above > n_kept
    out = {k: v.numpy() for k, v in P.items()}
    out["firing"] = img.numpy()
    np.savez_compressed(ROOT / "tests" / "golden" / "blazeface_ref.npz", **out)


if __name__ == "__main__":
    main(sys.argv[1])
