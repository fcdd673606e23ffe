"""Faces of the object saves for a fleet: one `CameraBatch.save_objects_and_faces` call against `save_objects` plus the
per-save host chain the reference runs on each person thumbnail (process_latest_face, clearcam.py:272-279, 1228-1241).

    python tools/face_save_fleet.py [--steps 20] [--warmup 3] [--arch ViT-B/32] [--out results.json]

16 seeded cameras at mixed resolutions and formats (bgr24 and yuv420p at 480p, 720p and 1080p), the BlazeFace fixture's
`firing` face (tests/golden/blazeface_ref.npz) at twice its size planted in six of the 720p and 1080p ones, a synthetic
YOLOv9-c at res 320 stepping them, and per camera and step the step's own saves plus injected ones: a person save of
exactly the face (where planted), a person save of background and a non-person save.  Per step, after --warmup untimed steps:
  device  `save_objects_and_faces(results, finder)`: thumbnails, CLIP, and the faces of the person saves in one call;
  host    `save_objects(results, finder)`, then per person save imdecode -> RGB -> img_to_face -> imencode -> adaface.
Both are timed with host clocks around work that ends in a device synchronise; the faces of the two are checked equal
every step.  CLIP and AdaFace weights are synthetic (the same kernels and shapes as the real ones).  The card's name and
power limit are read in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CAMS = [((480, 640), "bgr24"), ((720, 1280), "yuv420p"), ((1080, 1920), "bgr24"), ((720, 1280), "bgr24"),
        ((1080, 1920), "yuv420p"), ((480, 640), "yuv420p"), ((720, 1280), "bgr24"), ((1080, 1920), "bgr24")] * 2


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def host_faces(finder, files, person, quality):
    """The reference's chain on each person thumbnail -> (rows, files, embeddings as one host array)."""
    import cv2
    rows, out, emb = [], [], []
    for k in np.flatnonzero(person):
        img = cv2.cvtColor(cv2.imdecode(np.frombuffer(files[k], np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
        face = finder.img_to_face(img)
        if face is None:
            continue
        rows.append(int(k))
        out.append(cv2.imencode(".jpg", face, [cv2.IMWRITE_JPEG_QUALITY, quality])[1].tobytes())
        emb.append(finder.adaface(face).numpy()[0])
    return rows, out, np.array(emb, np.float32).reshape(-1, 512)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--arch", default="ViT-B/32")
    ap.add_argument("--out")
    args = ap.parse_args()
    import cv2
    cv2.ipp.setUseIPP(False)
    from oracle import adaface as oa
    from oracle import clip as oc
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    torch.cuda.set_device(0)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "blazeface_ref.npz"))
    face = cv2.resize(np.ascontiguousarray(gold["firing"][..., ::-1]), (512, 512))
    finder = ObjectFinder()
    finder.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS[args.arch], seed=3), arch=args.arch)
    finder.init_face(weights=oa.synthetic_weights(seed=5), detector={k: gold[k] for k in gold.files if k != "firing"})
    xc = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    cb = CameraBatch(YOLOv9("c", 320, weights=o.synthetic_weights("c", seed=5, calib=xc)))
    for i, (_, fmt) in enumerate(CAMS):
        cb.add_camera(i, thresh=0.05, pix_fmt=fmt)
    g = np.random.default_rng(0)
    t_dev, t_host, n_saves, n_person, n_faces = [], [], 0, 0, 0
    for step in range(args.warmup + args.steps):
        frames, extra = {}, {}
        for i, ((H, W), fmt) in enumerate(CAMS):
            img = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
            rows = [(1, 0, 0, H // 2, W // 4, H), (2, 2, W // 2, 0, W, H // 2)]
            if i % 2 == 0 and H >= 720:                # the fixture's face fires when a save is exactly it, at 2x or more
                x, y = int(g.integers(0, (W - 512) // 2)) * 2, int(g.integers(0, (H - 512) // 2)) * 2
                img[y:y + 512, x:x + 512] = face
                rows.append((3, 0, x, y, x + 512, y + 512))
            extra[i] = np.array(rows, np.int64)
            frames[i] = cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420) if fmt == "yuv420p" else img
        res = cb.step_events(frames, now=1.7e9 + step)
        res = {i: ev._replace(saves=np.concatenate([np.asarray(ev.saves, np.int64).reshape(-1, 6), extra[i]])) for i, ev in res.items()}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        saved, faces = cb.save_objects_and_faces(res, finder)
        for fs in faces.values():
            if fs.embeddings is not None:
                fs.embeddings.tensor.cpu()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        want = cb.save_objects(res, finder)
        host = {i: host_faces(finder, want[i][1], np.asarray(want[i][0])[:, 1] == 0, 95) for i in want}
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        for i in want:
            rows, files, emb = host[i]
            fs = faces[i]
            assert saved[i][1] == want[i][1] and fs.rows == rows and fs.files == files, (step, i)
            assert np.array_equal(fs.embeddings.tensor.cpu().numpy().reshape(-1, 512), emb), (step, i)
        if step >= args.warmup:
            t_dev.append(t1 - t0)
            t_host.append(t2 - t1)
            n_saves += sum(len(s[1]) for s in saved.values())
            n_person += sum(int((np.asarray(s[0])[:, 1] == 0).sum()) for s in saved.values())
            n_faces += sum(len(f.rows) for f in faces.values())
    c = card()
    dev, hst = 1e3 * float(np.median(t_dev)), 1e3 * float(np.median(t_host))
    res = {"card": c, "cameras": len(CAMS), "steps": args.steps, "saves_per_step": n_saves / args.steps,
           "person_saves_per_step": n_person / args.steps, "faces_per_step": n_faces / args.steps,
           "one_call_ms_median": dev, "save_objects_plus_host_chain_ms_median": hst, "speedup": hst / dev}
    print("card:", c)
    print(f"{len(CAMS)} cameras, {res['saves_per_step']:.1f} saves / {res['person_saves_per_step']:.1f} person saves / "
          f"{res['faces_per_step']:.1f} faces per step over {args.steps} steps")
    print(f"save_objects_and_faces {dev:8.2f} ms   save_objects + per-save host chain {hst:8.2f} ms   x{hst / dev:.1f}  (medians)")
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
