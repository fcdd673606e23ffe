"""The AdaFace IR-50 embedder on the GPU (csrc/adaface.cu, the ACT_PRELU conv epilogue) against the CPU oracle.

* The ACT_PRELU epilogue against float64 at 112², 56², 28², 14² and 7²: Cout 64..512, strides 1 and 2, slopes negative, zero
  and above 1, a distinct bias per border class, B = 1 and 5.
* `embed_faces` against the fp32 oracle (oracle/adaface.py `forward`) at B = 1, 3, 64 and 200 on synthetic weights.  The bar
  is the bf16 mirror's own deviation from the fp32 oracle on the same faces (`forward_folded(bf16=True)`, which rounds
  where the GPU path stores bf16): the GPU may deviate at most twice as much.  On an H100 80GB HBM3 (700 W), on the first 8
  of these faces: max |mirror - fp32| = 1.7e-3 and max |GPU - fp32| = 1.9e-3 per element of the unit-norm embedding
  (tools/face_fleet.py prints both).
* Each face of a batch is bit-equal to its own B = 1 call; the per-block taps follow the mirror.
* `adaface(img)` equals the reference's call form, including the channel quirk of 112² uploads (preprocess_face returns RGB).
* `search(is_face=True)` equals the reference's search loop on the host, alternated with image searches.
* Argument errors raise before any launch.
"""

import cv2
import numpy as np
import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200._lib import CCError, lib, ptr, stream_ptr
from clearcam_b200.models import adaface as ca
from clearcam_b200.models.objects import ObjectFinder, event_img_info
from oracle import adaface as oa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    return oa.synthetic_weights(seed=5)


@pytest.fixture(scope="module")
def finder(weights):
    f = ObjectFinder()
    f.init_face(weights=weights)
    return f


@pytest.fixture(scope="module")
def distinct():
    return oa.synthetic_faces(16, seed=21)


@pytest.fixture(scope="module")
def oracle_rows(weights, distinct):
    with torch.no_grad():
        fp32 = oa.forward(weights, distinct)
        mirror = oa.forward_folded(ca.fold_state_dict(weights), distinct, bf16=True)
    return fp32, mirror


# ---- the ACT_PRELU epilogue
PRELU_CASES = [   # (side, Cin, Cout, stride, B)
    (112, 16, 64, 1, 1), (112, 64, 64, 2, 5), (56, 64, 128, 1, 5), (56, 64, 128, 2, 1), (28, 128, 256, 1, 1),
    (28, 128, 128, 2, 5), (14, 256, 256, 1, 5), (14, 256, 512, 2, 1), (7, 512, 512, 1, 5), (7, 512, 512, 1, 1),
]


@pytest.mark.parametrize("side,cin,cout,stride,B", PRELU_CASES)
def test_prelu_epilogue_vs_float64(side, cin, cout, stride, B):
    g = torch.Generator().manual_seed(side * 1000 + cout + stride + B)
    x = (torch.randn(B, side, side, cin, generator=g)).to(torch.bfloat16)
    w = (torch.randn(cout, 3, 3, cin, generator=g) * (2.0 / (9 * cin)) ** 0.5).to(torch.bfloat16)
    cls = torch.randn(9, cout, generator=g) + torch.arange(9).view(9, 1) * 0.25       # every border class its own bias
    slope = torch.cat([torch.tensor([-0.5, 0.0, 1.75]), torch.rand(cout - 3, generator=g) * 0.4])
    Ho = side // stride
    out = torch.full((B, Ho, Ho, cout), float("nan"), dtype=torch.bfloat16, device="cuda")
    ops.conv2d(x.cuda(), 0, cin, w.cuda(), cls.cuda(), 3, stride, out, 0, cout, act=3, slope=slope.cuda())
    torch.cuda.synchronize()
    y = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2), stride=stride, padding=1)
    y = y + cls.double()[oa.class_map(Ho, Ho)].permute(2, 0, 1)[None]
    want = torch.where(y > 0, y, slope.double().view(1, -1, 1, 1) * y).permute(0, 2, 3, 1)
    got = out.cpu().double()
    err = (got - want).abs()
    # the bf16 store's half ulp (<= 2^-8 |x|) plus the fp32 accumulation over up to 4608 products (~1e-5 at |x| ~ 4)
    tol = 2 ** -8 * want.abs() + 1e-4
    assert torch.isfinite(got).all()
    assert (err <= tol).all(), f"max err {err.max().item()}"
    # the border rows / columns carry their own class bias (a wrong class would be off by >= 0.25 before PReLU)
    assert (err[:, 0] <= tol[:, 0]).all() and (err[:, :, -1] <= tol[:, :, -1]).all()


# ---- the network
def _tile(distinct, B):
    idx = torch.arange(B) % distinct.shape[0]
    return distinct[idx], idx


@pytest.mark.parametrize("B", [1, 3, 64, 200])
def test_embed_faces_vs_oracle(finder, distinct, oracle_rows, B):
    fp32, mirror = oracle_rows
    faces, idx = _tile(distinct, B)
    got = finder.embed_faces(faces).cpu()
    assert got.shape == (B, 512) and torch.isfinite(got).all()
    bar = (mirror - fp32)[idx].abs().max().item()
    dev = (got - fp32[idx]).abs().max().item()
    assert dev <= 2 * bar, f"GPU deviates {dev:.3e} from the fp32 oracle; the bf16 mirror {bar:.3e}"
    cos = (got * fp32[idx]).sum(-1)
    assert cos.min() > 0.999
    assert ((got.norm(dim=-1) - 1).abs() < 1e-5).all()


def test_batch_rows_equal_single_calls(finder, distinct):
    faces = torch.cat([distinct, oa.synthetic_faces(48, seed=99)])           # 64 distinct faces
    batch = finder.embed_faces(faces.cuda())
    for b in list(range(0, 64, 7)) + [63]:
        one = finder.adaface(faces[b].numpy()).tensor
        assert torch.equal(one[0], batch[b]), f"face {b}"
    # a batch that is not a bucket size pads, and its rows are still the single calls'
    part = finder.embed_faces(faces[:13])
    assert torch.equal(part, batch[:13])


def test_layer_taps_follow_mirror(finder, weights, distinct):
    faces = distinct[:2]
    with torch.no_grad():
        _, taps = oa.forward_folded(ca.fold_state_dict(weights), faces, bf16=True, taps=True)
    for layer in (0, 1, 4, 8, 22, 24, 25):
        got = finder.adaface.layer_output(faces, layer).cpu()
        want = taps[layer]
        want = want.permute(0, 2, 3, 1) if want.dim() == 4 else want.view(got.shape)
        assert got.shape == want.shape, layer
        rel = (got - want).abs().max() / want.abs().max()
        assert rel < 0.03, f"layer {layer}: relative deviation {rel.item():.3e}"


def test_adaface_call_form_and_upload_quirk(finder, weights, distinct):
    bgr = distinct[3].numpy()                                   # a saved face is BGR (img_to_face, objects.py:263-354)
    got = finder.adaface(bgr)
    assert got.numpy().shape == (1, 512)
    with torch.no_grad():
        want_saved = oa.forward(weights, torch.from_numpy(bgr)[None])
        # run_clip: an uploaded 112x112 file comes back RGB from preprocess_face and is embedded as is (channels swapped)
        ok, png = cv2.imencode(".png", bgr)
        rgb = finder.preprocess_face(png.tobytes())
        want_upload = oa.forward(weights, torch.from_numpy(np.ascontiguousarray(rgb))[None])
    up = finder.adaface(rgb).numpy()
    assert np.abs(got.numpy() - want_saved.numpy()).max() < 5e-3
    assert np.abs(up - want_upload.numpy()).max() < 5e-3
    assert np.abs(up - got.numpy()).max() > 1e-2                # the quirk is kept, not fixed


def _reference_search(embeddings, q, top_k, cam_name, timestamp):
    """ObjectFinder.search of the reference (models/objects.py:356-390) on the host, verbatim."""
    import os
    all_similarities = []
    for path, img_embedding in embeddings.items():
        if img_embedding is None:
            continue
        normalized_path = path.replace("\\", "/")
        if cam_name and f"/cameras/{cam_name}/" not in normalized_path:
            continue
        if timestamp and f"/objects/{timestamp}/" not in normalized_path and "/objects/video/" not in normalized_path:
            continue
        similarity = (img_embedding @ q.T).item()
        filename = os.path.basename(path)
        if filename.lower().endswith((".jpg")):
            object_id = event_img_info(filename.split(".jpg")[0])["object_id"] if "_" in filename else None
            all_similarities.append((path, similarity, object_id))
    if any(item[2] for item in all_similarities):
        best_per_id = {}
        for path, score, object_id in all_similarities:
            if object_id is not None:
                if object_id not in best_per_id or score > best_per_id[object_id][1]:
                    best_per_id[object_id] = (path, score)
        items_without_id = [(path, score) for path, score, object_id in all_similarities if object_id is None]
        results = list(best_per_id.values()) + items_without_id
    else:
        results = [(path, score) for path, score, _ in all_similarities]
    results.sort(key=lambda x: x[1], reverse=True)
    return results[:top_k]


def test_face_search_matches_reference_loop(finder):
    faces = oa.synthetic_faces(40, seed=8)
    emb = finder.embed_faces(faces).cpu().numpy()
    rng = np.random.default_rng(1)
    f = ObjectFinder()
    for i in range(40):
        cam = ["front", "back"][i % 2]
        date = ["2026-10-16", "2026-10-17", "video"][i % 3]
        name = f"{1700000000 + i}_{rng.integers(0, 9)}_0.jpg" if i % 5 else f"{1700000000 + i}.jpg"
        f.face_embeddings[f"data/cameras/{cam}/objects/{date}/{name}"] = emb[i:i + 1]          # stored as (1,512), :1236-1239
    f.face_embeddings["data/cameras/front/objects/2026-10-17/notes.png"] = emb[0:1]
    clip_dim = 64
    for i in range(30):
        f.image_embeddings[f"data/cameras/front/objects/2026-10-17/{i}_{i % 4}_2.jpg"] = rng.standard_normal((1, clip_dim)).astype(np.float32)
    qs = [emb[5:6], emb[17:18]]
    for rep in range(2):                                       # alternate face and image searches over the two device indexes
        for q in qs:
            for cam, ts in [(None, None), ("front", None), (None, "2026-10-17"), ("back", "2026-10-16")]:
                got = f.search(None, 10, cam, ts, q, is_face=True)
                want = _reference_search(f.face_embeddings, q, 10, cam, ts)
                assert [p for p, _ in got] == [p for p, _ in want], (cam, ts)
                assert np.allclose([s for _, s in got], [s for _, s in want], atol=1e-5)
        tq = rng.standard_normal((1, clip_dim)).astype(np.float32)
        got = f.search(None, 5, None, None, tq)
        want = _reference_search(f.image_embeddings, tq, 5, None, None)
        assert [p for p, _ in got] == [p for p, _ in want]
        f.face_embeddings[f"data/cameras/back/objects/video/{1800000000 + rep}_77_0.jpg"] = emb[5:6] * 0.5   # the index follows


def test_argument_errors_before_launch(finder):
    L = lib()
    h = finder.adaface._h
    faces = oa.synthetic_faces(2, seed=1).cuda()
    out = torch.full((2, 512), 7.0, device="cuda")
    for args in [(h, ptr(faces), 0, ptr(out), 512), (h, None, 2, ptr(out), 512), (h, ptr(faces), 2, None, 512),
                 (h, ptr(faces), 2, ptr(out), 100), (None, ptr(faces), 2, ptr(out), 512)]:
        assert L.cc_face_embed(*args, stream_ptr()) != 0
    torch.cuda.synchronize()
    assert (out == 7.0).all()
    assert L.cc_face_layer_output(h, ptr(faces), 2, 26, ptr(out), None, None, None, stream_ptr()) != 0
    with pytest.raises(ValueError):
        finder.embed_faces(faces[..., :2])
    with pytest.raises(ValueError):
        finder.embed_faces(faces.float())
    with pytest.raises(ValueError):
        finder.adaface(faces)
    x = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(64, 3, 3, 64, dtype=torch.bfloat16, device="cuda")
    o = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(CCError, match="cc_conv2d_prelu"):
        ops.conv2d(x, 0, 64, w, torch.zeros(9, 64, device="cuda"), 3, 1, o, 0, 64, act=3, slope=None)
    with pytest.raises(CCError):
        ca.ADAFACE({k: v for k, v in oa.synthetic_weights(0).items() if k != "linear.bias"})
    off = ObjectFinder()
    with pytest.raises(CCError, match="init_face"):
        off.embed_faces(faces)
