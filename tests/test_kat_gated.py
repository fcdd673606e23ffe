"""Known-answer tests that need data this repository cannot ship; each one runs by itself as soon as the data is there.

  * CLIP: the reference's real ViT-L/14 weights (models/objects.py:91 downloads CLIP-ViT-L-14-laion2B-s32B-b82K.safetensors)
    under $CLEARCAM_B200_WEIGHTS -> test/test_clip.py's 0.330654 and the embeddings stored in test/clip_images/embeddings.pkl
    (fixtures: tests/golden/clip_kat.npz from oracle/make_golden_clip_kat.py), for the CPU oracle and for the CUDA path.
  * Detector + tracker: the reference's test/videos/MOT16-03.mp4 (11 MB) at $CLEARCAM_B200_MOT_VIDEO
    -> test/run_mot.py's 156 distinct moving person tracks through the CUDA detector (YOLOv9-t weights recovered from the
    reference's iOS bundle, tests/golden/yolov9t_mot16.npz) and the C++ tracker.
Until then CLIP numerics stay "parity unpinned" (DESIGN.md §2)."""
import os
from pathlib import Path

import numpy as np
import pytest
import torch

GOLD = Path(__file__).parent / "golden"
W_NAME = "CLIP-ViT-L-14-laion2B-s32B-b82K.safetensors"
W_PATH = Path(os.environ.get("CLEARCAM_B200_WEIGHTS", "/nonexistent")) / W_NAME
VIDEO = next((p for p in (os.environ.get("CLEARCAM_B200_MOT_VIDEO", ""), str(Path(__file__).parent.parent / "tmp_mot16.mp4"))
              if p and os.path.exists(p)), None)
needs_clip_weights = pytest.mark.skipif(not W_PATH.exists(), reason=f"real CLIP weights not found at {W_PATH}")
needs_video = pytest.mark.skipif(VIDEO is None, reason="MOT16-03.mp4 not available (set $CLEARCAM_B200_MOT_VIDEO)")


def _kat():
    import cv2
    z = np.load(GOLD / "clip_kat.npz")
    imgs = {n: cv2.imdecode(z[f"{n}_jpg"], cv2.IMREAD_COLOR) for n in ("f40", "micra")}      # BGR, as cv2.imread gives
    return z, imgs


@needs_clip_weights
def test_oracle_reproduces_the_references_clip_known_answer():
    """oracle/clip.py with the real weights: test/test_clip.py:6-12 (note: that test feeds the BGR image unswapped)."""
    from safetensors.torch import load_file
    from oracle import clip as oc
    from clearcam_b200.utils.clip_tokenizer import SimpleTokenizer
    z, imgs = _kat()
    P = {k: v.float() for k, v in load_file(str(W_PATH)).items()}
    cfg = oc.CONFIGS["ViT-L/14"]
    with torch.no_grad():
        e = oc.encode_image(cfg, P, torch.from_numpy(oc.preprocess(imgs["f40"]))[None])
        t = oc.encode_text_ids(cfg, P, oc.pad_tokens([SimpleTokenizer().encode(str(z["query"]))]))
    assert abs(float(t[0] @ e[0]) - float(z["known_answer"])) < 2e-4          # fp32 vs fp32, different summation order
    for n in ("f40", "micra"):                                                   # stored by the pipeline: RGB (clearcam.py:275)
        import cv2
        with torch.no_grad():
            e = oc.encode_image(cfg, P, torch.from_numpy(oc.preprocess(cv2.cvtColor(imgs[n], cv2.COLOR_BGR2RGB)))[None])[0]
        assert float(e @ torch.from_numpy(z[f"emb_{n}"])) >= 0.9995, n


@pytest.mark.gpu
@needs_clip_weights
def test_cuda_path_reproduces_the_references_clip_known_answer():
    import cv2
    from clearcam_b200.models.objects import ObjectFinder
    z, imgs = _kat()
    f = ObjectFinder()
    f.init_clip(weights=str(W_PATH), arch="ViT-L/14")
    emb = f.model.precompute_embedding(f.preprocess(imgs["f40"])[None]).numpy()
    txt = f.model._encode_text(str(z["query"]), realize=True)
    assert abs(float(txt @ emb[0]) - float(z["known_answer"])) < 3e-3           # bf16 GEMM operands: cosine >= 0.999 bar
    for n in ("f40", "micra"):
        e = f.model.precompute_embedding(f.preprocess(cv2.cvtColor(imgs[n], cv2.COLOR_BGR2RGB))[None]).numpy()[0]
        assert float(e @ z[f"emb_{n}"]) >= 0.999, n
    # and the search built on them: the stored vectors as the index, "ferrari f40" must rank f40.jpg first
    f.image_embeddings = {"/data/cameras/c/objects/2026-01-01/1_1_2.jpg": z["emb_f40"][None], "/data/cameras/c/objects/2026-01-01/2_2_2.jpg": z["emb_micra"][None]}
    assert f.search("ferrari f40", top_k=1)[0][0].endswith("1_1_2.jpg")


@pytest.mark.gpu
@needs_video
@pytest.mark.parametrize("precise", [True, False], ids=["fp32-accurate", "default-bf16"])
def test_mot16_known_answer_through_the_cuda_detector(precise):
    """test/run_mot.py:14-51: YOLOv9-t at res 960 on all 1501 frames -> OCSort(max_age=60).update(pred, 0.25) -> distinct
    moving person tracks == 156.  The fixtures were recorded by a detector revision without the BGR->RGB swap (SURVEY D10),
    so the frames are fed channel-reversed (the CUDA path always swaps)."""
    import cv2
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.ocsort_tracker import ocsort
    z = np.load(GOLD / "yolov9t_mot16.npz")
    P = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}
    m = YOLOv9("t", 960, weights=P, precise=precise)
    trk = ocsort.OCSort(max_age=60)
    cap = cv2.VideoCapture(VIDEO)
    ppl, n, batch = set(), 0, []

    def flush():
        real = len(batch)
        while len(batch) < 16:                                                               # one plan: pad the last batch,
            batch.append(batch[-1])
        out = m.detect_batch(torch.from_numpy(np.stack(batch)).float()).cpu().numpy()      # run_mot.py:33 casts to float32
        for pred in out[:real]:                                                              # ... and drop the padded rows
            for x in trk.update(pred, 0.25):
                if x.tracklet_len < 1 or x.speed < 2.5:
                    continue
                if x.class_id == 0:
                    ppl.add(x.track_id)
        batch.clear()
    while True:
        ret, im = cap.read()
        if not ret:
            break
        batch.append(np.ascontiguousarray(im[..., ::-1]))
        n += 1
        if len(batch) == 16:
            flush()
    if batch:
        flush()
    assert n == 1501
    if precise:
        assert len(ppl) == 156, len(ppl)
    else:
        assert abs(len(ppl) - 156) <= 4, len(ppl)      # bf16 storage moves a few borderline tracks (the bf16-mirror oracle gives 155)
