"""GPU parity of the CLIP encoders against the CPU oracle (oracle/clip.py).

Bar (north star): embedding cosine >= 0.999 vs the fp32 oracle.  Because synthetic-weight embeddings of different
inputs are themselves fairly close, two stronger checks are added: the pairwise-cosine matrix of the batch must
match the oracle's within 5e-3, and the batch-mean-centred embeddings must still have cosine >= 0.99."""
import numpy as np
import pytest
import torch

from oracle import clip as oc
from clearcam_b200.models.objects import OpenCLIP, ObjectFinder, search_scores

pytestmark = pytest.mark.gpu

PROMPTS = ["ferrari f40", "text here", "a photo of a cat", "person riding a bicycle at night", "white van with ladder on roof",
           "delivery driver carrying a box", "dog"]


def _check(got: torch.Tensor, want: torch.Tensor, pairwise: float = 5e-3):
    cos = (got * want).sum(-1) / (got.norm(dim=-1) * want.norm(dim=-1))
    assert cos.min() >= 0.999, f"cosine {cos.min()}"
    assert (got.norm(dim=-1) - 1).abs().max() < 1e-4
    if got.shape[0] > 2:
        assert ((got @ got.T) - (want @ want.T)).abs().max() < pairwise
        gc, wc = got - got.mean(0, keepdim=True), want - want.mean(0, keepdim=True)
        cosc = (gc * wc).sum(-1) / (gc.norm(dim=-1) * wc.norm(dim=-1))
        assert cosc.min() >= 0.99, f"centred cosine {cosc.min()}"


@pytest.mark.parametrize("arch,B", [("ViT-tiny", 5), ("ViT-B/32", 6), ("ViT-B/32", 1), ("ViT-L/14", 3)])
def test_image_encoder(arch, B):
    cfg = oc.CONFIGS[arch]
    P = oc.synthetic_weights(cfg, seed=3)
    x = oc.synthetic_images(B, cfg.image_size, seed=5)
    with torch.no_grad():
        want = oc.encode_image(cfg, P, x)
    m = OpenCLIP(weights=P, arch=arch)
    got = m.precompute_embedding(x).tensor.cpu()
    assert got.shape == (B, cfg.embed_dim)
    _check(got, want)


@pytest.mark.parametrize("arch", ["ViT-tiny", "ViT-B/32", "ViT-L/14"])
def test_text_encoder(arch):
    cfg = oc.CONFIGS[arch]
    P = oc.synthetic_weights(cfg, seed=4)
    m = OpenCLIP(weights=P, arch=arch)
    ids = torch.tensor([m.tokenize(q) for q in PROMPTS])
    with torch.no_grad():
        want = oc.encode_text_ids(cfg, P, ids.long())
    got = m.encode_text_batch(PROMPTS).tensor.cpu()
    _check(got, want)
    one = m._encode_text("ferrari f40", realize=True)               # reference signature (models/objects.py:135)
    assert one.shape == (cfg.embed_dim,) and np.allclose(one, got[0].numpy(), atol=1e-5)


@pytest.mark.parametrize("arch", ["ViT-tiny", "ViT-B/32"])
def test_text_encoder_at_every_eot_position(arch):
    """One row per EOT position 1..76; the last row is a full 77-token prompt with no padding.  Token ids 1000-40000 keep
    the EOT (49407) the row's argmax.  Covers text_embed_kernel's EOT argmax, the ln_final row gather and the causal
    attention rows past 64 (the second 64-row query block) end to end."""
    cfg = oc.CONFIGS[arch]
    P = oc.synthetic_weights(cfg, seed=4)
    g = torch.Generator().manual_seed(9)
    ids = torch.zeros(cfg.ctx - 1, cfg.ctx, dtype=torch.long)
    for r, eot in enumerate(range(1, cfg.ctx)):
        ids[r, 0] = 49406
        ids[r, 1:eot] = torch.randint(1000, 40000, (eot - 1,), generator=g)
        ids[r, eot] = 49407
    assert (ids.argmax(-1) == torch.arange(1, cfg.ctx)).all()
    with torch.no_grad():
        want = oc.encode_text_ids(cfg, P, ids)
    m = OpenCLIP(weights=P, arch=arch)
    got = m.encode_token_ids(ids).tensor.cpu()
    # ViT-tiny's 128-wide tower: the oracle with its activations and weights rounded to bf16 where this path stores bf16
    # (and exact arithmetic otherwise) already moves the pairwise-cosine matrix of these 76 rows by 0.0049-0.0060 (seeds
    # 9-12), so 5e-3 would only measure bf16 storage there; the 512-wide ViT-B/32 tower moves by <= 0.0016.
    _check(got, want, pairwise=1e-2 if arch == "ViT-tiny" else 5e-3)


def test_search_matches_reference_semantics(tmp_path):
    g = torch.Generator().manual_seed(0)
    N, D = 300, 512
    index = torch.nn.functional.normalize(torch.randn(N, D, generator=g), dim=-1)
    q = torch.nn.functional.normalize(torch.randn(3, D, generator=g), dim=-1)
    got = search_scores(index, q).cpu()
    assert (got - q @ index.T).abs().max() < 1e-5
    # ObjectFinder.search: best score per object id, descending, top_k (models/objects.py:356-390)
    f = ObjectFinder(base_path=str(tmp_path))
    f.image_embeddings = {f"/x/cameras/cam{i % 2}/objects/2026-01-01/{1000 + i}_{i % 40}_0.jpg": index[i:i + 1].numpy() for i in range(N)}
    res = f.search(top_k=10, text_embedding=q[0].numpy())
    sims = (index @ q[0]).numpy()
    best = {}
    for i, p in enumerate(f.image_embeddings):
        oid = str(i % 40)
        if oid not in best or sims[i] > best[oid][1]:
            best[oid] = (p, float(sims[i]))
    want = sorted(best.values(), key=lambda t: -t[1])[:10]
    assert [p for p, _ in res] == [p for p, _ in want]
    assert np.allclose([s for _, s in res], [s for _, s in want], atol=1e-5)
    assert all("/cameras/cam1/" in p for p, _ in f.search(top_k=50, text_embedding=q[0].numpy(), cam_name="cam1"))


def _reference_search(emb, qv, top_k, cam_name=None, timestamp=None):
    """models/objects.py:356-390 restated on the host (scores by the oracle's plain dot product)."""
    import os
    from clearcam_b200.models.objects import event_img_info
    sims = []
    for path, e in emb.items():
        if e is None:
            continue
        similarity = float(oc.search_scores(torch.from_numpy(np.asarray(e, np.float32).reshape(1, -1)), torch.from_numpy(qv))[0])
        norm = path.replace("\\", "/")
        if cam_name and f"/cameras/{cam_name}/" not in norm:
            continue
        if timestamp and f"/objects/{timestamp}/" not in norm and "/objects/video/" not in norm:
            continue
        filename = os.path.basename(path)
        if filename.lower().endswith(".jpg"):
            oid = event_img_info(filename.split(".jpg")[0])["object_id"] if "_" in filename else None
            sims.append((path, similarity, oid))
    if any(s_[2] for s_ in sims):
        best = {}
        for path, score, oid in sims:
            if oid is not None and (oid not in best or score > best[oid][1]):
                best[oid] = (path, score)
        results = list(best.values()) + [(p_, s_) for p_, s_, oid in sims if oid is None]
    else:
        results = [(p_, s_) for p_, s_, _ in sims]
    results.sort(key=lambda x: x[1], reverse=True)
    return results[:top_k]


def test_device_topk_search_equals_the_reference_loop(tmp_path):
    """cc_search_topk (scores + best-per-object-id + top-k on the device) against the reference's Python loop on an index
    with every kind of row: several cameras and dates, the shared 'video' folder, rows without an object id, non-jpg rows,
    a replaced embedding, and more requested results than matches."""
    g = torch.Generator().manual_seed(3)
    N, D = 700, 512
    index = torch.nn.functional.normalize(torch.randn(N, D, generator=g), dim=-1).numpy()
    qs = torch.nn.functional.normalize(torch.randn(4, D, generator=g), dim=-1).numpy()
    emb = {}
    for i in range(N):
        cam, date = f"cam{i % 3}", ("video" if i % 11 == 0 else f"2026-01-0{1 + i % 4}")
        name = f"{1000 + i}_{i % 57}_{i % 5}.jpg" if i % 7 else (f"snap{i}.jpg" if i % 2 else f"{1000 + i}_{i % 57}_0.png")
        emb[f"/data/cameras/{cam}/objects/{date}/{name}"] = index[i:i + 1]
    emb["/data/cameras/cam0/objects/2026-01-01/none.jpg"] = None
    f = ObjectFinder(base_path=str(tmp_path))
    f.image_embeddings = emb
    cases = [dict(top_k=10), dict(top_k=25, cam_name="cam1"), dict(top_k=10, timestamp="2026-01-02"),
             dict(top_k=400, cam_name="cam2", timestamp="2026-01-03"), dict(top_k=5, cam_name="nope"), dict(top_k=1000)]
    for qv in qs[:2]:
        for kw in cases:
            got, want = f.search(text_embedding=qv, **kw), _reference_search(emb, qv, **kw)
            assert [p_ for p_, _ in got] == [p_ for p_, _ in want], kw
            assert np.allclose([s_ for _, s_ in got], [s_ for _, s_ in want], atol=1e-5)
    # no row with an object id among the candidates -> every row stands for itself (:377)
    f2 = ObjectFinder(base_path=str(tmp_path))
    f2.image_embeddings = {f"/data/cameras/cam0/objects/video/frame{i}.jpg": index[i:i + 1] for i in range(50)}
    got, want = f2.search(text_embedding=qs[2], top_k=20), _reference_search(f2.image_embeddings, qs[2], 20)
    assert [p_ for p_, _ in got] == [p_ for p_, _ in want]
    # an embedding replaced under an existing path is picked up (the device index is fingerprinted by value identity)
    key = next(iter(f2.image_embeddings))
    f2.image_embeddings[key] = qs[3:4].copy()
    assert f2.search(text_embedding=qs[3], top_k=1)[0][0] == key


# ------------------------------------------------------------------------------------------------ crop -> CLIP input
def test_device_crop_preprocess_bit_exact():
    """cc_clip_preprocess == crop + cvtColor + ObjectFinder.preprocess with OpenCV's bicubic (oracle pinned to cv2)."""
    from pathlib import Path
    from oracle import clip_preprocess as cp
    g = np.load(Path(__file__).parent / "golden" / "clip_preprocess.npz")
    of = ObjectFinder()
    got = of.preprocess_device(g["frame"], g["rects"]).tensor.cpu().numpy()
    want = np.stack([np.transpose((r.astype(np.float32) / 255.0 - 0.5) / 0.5, (2, 0, 1)) for r in g["resized"]])
    np.testing.assert_array_equal(got, want)                                 # cv2's own output, committed
    # several frames, > 64 rects (two launches), up- and down-scaling, 1-pixel-wide and full-frame crops, RGB input
    rng = np.random.default_rng(5)
    frames = rng.integers(0, 256, (3, 270, 480, 3), dtype=np.uint8)
    rects = [(0, 0, 0, 480, 270), (1, 5, 7, 6, 200), (2, 100, 40, 324, 264), (2, 0, 269, 480, 270)]
    for _ in range(70):
        x1, y1 = int(rng.integers(0, 470)), int(rng.integers(0, 260))
        rects.append((int(rng.integers(0, 3)), x1, y1, int(rng.integers(x1 + 1, 481)), int(rng.integers(y1 + 1, 271))))
    for bgr in (True, False):
        got = of.preprocess_device(torch.from_numpy(frames).cuda(), rects, bgr=bgr).tensor.cpu().numpy()
        for k, (f, x1, y1, x2, y2) in enumerate(rects):
            crop = frames[f, y1:y2, x1:x2, ::-1] if bgr else frames[f, y1:y2, x1:x2]
            np.testing.assert_array_equal(got[k], cp.normalize(cp.resize_cubic_u8(np.ascontiguousarray(crop), 224, 224)), err_msg=str(rects[k]))
    got = of.preprocess_device(frames[0], [(10, 10, 200, 150)], size=37).tensor.cpu().numpy()      # tail columns: integer form
    np.testing.assert_array_equal(got[0], cp.normalize(cp.resize_cubic_u8(np.ascontiguousarray(frames[0, 10:150, 10:200, ::-1]), 37, 37)))
    with pytest.raises(Exception):
        of.preprocess_device(frames, [(0, 10, 10, 500, 100)])               # outside the frame: refused, not clamped


def test_embed_crops_end_to_end():
    from pathlib import Path
    from oracle import clip_preprocess as cp
    g = np.load(Path(__file__).parent / "golden" / "clip_preprocess.npz")
    cfg = oc.CONFIGS["ViT-B/32"]
    P = oc.synthetic_weights(cfg, seed=3)
    of = ObjectFinder()
    of.model = OpenCLIP(weights=P, arch="ViT-B/32")
    got = of.embed_crops(g["frame"], g["rects"]).tensor.cpu()
    with torch.no_grad():
        want = oc.encode_image(cfg, P, torch.from_numpy(cp.preprocess_crops(g["frame"], g["rects"])))
    _check(got, want)
