"""JPEG decoding on the GPU: every decoded image must be pixel for pixel what cv2.imdecode(buf, IMREAD_COLOR) returns, for
the fixture, every size up to 33 x 33, every sampling mode, restart intervals, optimised tables and hundreds of files per
call; files the device leaves to the host are reported, not guessed; the crop -> JPEG -> pixels chain and the CLIP entry
points equal the reference's host chain."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import jpeg_decode as od
from clearcam_b200 import ops
from clearcam_b200._lib import cc_jpeg_dest, lib, ptr, stream_ptr
from clearcam_b200.pixfmt import CC_FRAME_BGR_U8 as BGR, CC_FRAME_I420_U8 as I420, CC_FRAME_RGB_U8 as RGB

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jpeg_decode_cv2.npz")


def _cv2():
    return pytest.importorskip("cv2")


def _img(h, w, seed, sigma=10):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([(xx * (0.9 + 0.3 * c) + yy * (0.6 + 0.2 * c) + 60 * c) % 256 for c in range(3)], -1)
    return np.clip(base + rng.normal(0, sigma, (h, w, 3)), 0, 255).astype(np.uint8)


def _enc(img, q=95, samp=420, rst=0, opt=False):
    cv2 = _cv2()
    S = {444: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, 422: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
         440: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, 420: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
    p = [cv2.IMWRITE_JPEG_QUALITY, q]
    if samp == "grey":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, S[samp]]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if opt:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    return cv2.imencode(".jpg", img, p)[1].tobytes()


def _imdecode(f):
    cv2 = _cv2()
    return cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)


def _check_all(files, sentinel=True):
    """Decode in one call into a sentinel-filled batch; every OK image equals cv2, every other byte is untouched."""
    b = ops.JpegBatch(files)
    ok = b.status == ops.JPEG_OK
    hmax = max([int(h) for h in b.sizes[:, 1]] + [1])
    wmax = max([int(w) for w in b.sizes[:, 0]] + [1])
    out = torch.full((len(files), hmax, wmax, 3), 0xA5, dtype=torch.uint8, device="cuda")
    out, st = b.decode(out)
    o, st = out.cpu().numpy(), st.cpu().numpy()
    written = np.zeros(o.shape[:3], bool)
    for k, f in enumerate(files):
        if st[k] == ops.JPEG_OK:
            w, h = b.sizes[k]
            want = _imdecode(f)
            assert np.array_equal(o[k, :h, :w], want), (k, w, h)
            written[k, :h, :w] = True
    if sentinel:
        assert (o[~written] == 0xA5).all()
    return st


def test_fixture():
    g = np.load(GOLDEN)
    files, want_status = [], []
    k = 0
    while f"file{k}" in g:
        files.append(g[f"file{k}"].tobytes())
        want_status.append(int(g[f"status{k}"]))
        k += 1
    st = _check_all(files)
    assert list(st) == want_status
    out, sizes, _ = ops.jpeg_decode(files)
    o = out.cpu().numpy()
    for k, f in enumerate(files):
        if want_status[k] == 0:
            w, h = sizes[k]
            assert np.array_equal(o[k, :h, :w], g[f"want{k}"]), k


def test_every_size_up_to_33_in_one_call():
    files = []
    modes = (420, 422, 440, 444, "grey")
    for w in range(1, 34):
        for h in range(1, 34):
            i = w * 34 + h
            files.append(_enc(_img(h, w, i), (95, 50, 10, 100)[i % 4], modes[i % 5], rst=(0, 1, 3)[i % 3], opt=i % 7 == 0))
    st = _check_all(files)
    assert (st == 0).all()


@pytest.mark.parametrize("rst", [0, 7])
def test_1080p_q85(rst):
    f = _enc(_img(1080, 1920, 3, sigma=6), 85, 420, rst=rst)
    assert (_check_all([f]) == 0).all()


def test_200_mixed_files_in_one_call_equal_single_calls():
    rng = np.random.default_rng(7)
    files = []
    for i in range(200):
        h, w = int(rng.integers(1, 400)), int(rng.integers(1, 500))
        files.append(_enc(_img(h, w, 100 + i), int(rng.integers(1, 101)), (420, 422, 440, 444, "grey")[i % 5],
                          rst=int(rng.choice([0, 0, 1, 5, 13])), opt=bool(i % 3 == 0)))
    assert (_check_all(files) == 0).all()
    out, sizes, _ = ops.jpeg_decode(files)
    for i in range(0, 200, 23):
        one, _, _ = ops.jpeg_decode([files[i]])
        w, h = sizes[i]
        assert torch.equal(one[0, :h, :w], out[i, :h, :w]), i


def test_unsupported_and_corrupt_are_reported_and_do_not_disturb_the_others():
    cv2 = _cv2()
    img = _img(64, 80, 9)
    good = [_enc(img, 90), _enc(_img(33, 17, 10), 70, 444), _enc(_img(50, 50, 11), 30, "grey", rst=2)]
    prog = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    base = good[0]
    truncated = base[:len(base) // 2]
    st_, info = od.parse(base)
    off, ln = info["scan"]
    invalid = bytearray(base)
    invalid[off + ln // 3: off + ln // 3 + 8] = b"\xff\x00" * 4          # all-ones: no code of any table
    bad_rst = bytearray(_enc(img, 90, rst=1))
    i = bytes(bad_rst).find(b"\xff\xd3")
    bad_rst[i + 1] = 0xD5
    files = [good[0], prog, truncated, good[1], bytes(invalid), b"not a jpeg", bytes(bad_rst), good[2]]
    st = _check_all(files)
    assert list(st) == [0, 1, 2, 0, 2, 2, 2, 0]
    for f, s in zip(files, st):
        assert od.decode(f)[0] == s


def test_decode_coefficient_tap_equals_the_table_encoders_coefficients():
    cv2 = _cv2()
    fr = _img(240, 320, 12)
    rects = [(0, 0, 0, 320, 240), (0, 3, 5, 40, 22), (0, 311, 231, 320, 240), (0, 17, 1, 18, 2), (0, 100, 50, 250, 200)]
    dev = torch.from_numpy(fr[None]).cuda()
    table = ops.batch_table(dev, BGR)
    for q in (95, 20):
        files = ops.jpeg_collect(*ops.jpeg_encode_crops_frames(table, rects, q))
        got, st = ops.jpeg_decode_coeffs(files)
        assert (st.cpu().numpy() == 0).all()
        assert torch.equal(got, ops.jpeg_coeffs_frames(table, rects, q)), q
        assert np.array_equal(got.cpu().numpy(), np.concatenate([od.coeffs(f) for f in files]))
    del cv2


_RECTS = [(0, 1, 3, 201, 157), (1, 1719, 881, 1920, 1080), (0, 0, 0, 1920, 1080), (1, 333, 77, 334, 78), (0, 5, 5, 7, 6),
          (1, 0, 1, 113, 700), (0, 1917, 1077, 1920, 1080), (1, 1850, 0, 1920, 61)]


@pytest.mark.parametrize("q", [95, 60, 2])
def test_table_crops_decoded_equal_imdecode_of_table_encoder(q):
    cv2 = _cv2()
    bgr = np.stack([_img(1080, 1920, 20), _img(1080, 1920, 21)])
    rgb = np.ascontiguousarray(bgr[..., ::-1])
    yuv = np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420) for f in bgr])
    for src, fmt in ((bgr, BGR), (rgb, RGB), (yuv, I420)):
        dev = torch.from_numpy(src).cuda()
        table = ops.batch_table(dev, fmt)
        files = ops.jpeg_collect(*ops.jpeg_encode_crops_frames(table, _RECTS, q))
        pix, st = ops.jpeg_crops_decoded_frames(table, _RECTS, q)
        pix, st = pix.cpu().numpy(), st.cpu().numpy()
        for k, (f, x1, y1, x2, y2) in enumerate(_RECTS):
            # a crop is left to cv2 exactly where the decoder of its file would leave it (the IDCT range check)
            assert st[k] == od.decode(files[k])[0], (fmt, k)
            if st[k] == 0:
                assert np.array_equal(pix[k, :y2 - y1, :x2 - x1], _imdecode(files[k])), (fmt, k)


def test_table_crops_decoded_200_in_one_call():
    fr = np.stack([_img(540, 960, 30 + i) for i in range(4)])
    rng = np.random.default_rng(31)
    rects = []
    for _ in range(200):
        w, h = int(rng.integers(1, 300)), int(rng.integers(1, 200))
        x, y = int(rng.integers(0, 960 - w + 1)), int(rng.integers(0, 540 - h + 1))
        rects.append((int(rng.integers(0, 4)), x, y, x + w, y + h))
    dev = torch.from_numpy(fr).cuda()
    table = ops.batch_table(dev, BGR)
    files = ops.jpeg_collect(*ops.jpeg_encode_crops_frames(table, rects, 95))
    pix, st = ops.jpeg_crops_decoded_frames(table, rects, 95)
    assert (st.cpu().numpy() == 0).all()
    pix = pix.cpu().numpy()
    for k, (f, x1, y1, x2, y2) in enumerate(rects):
        assert np.array_equal(pix[k, :y2 - y1, :x2 - x1], _imdecode(files[k])), k


def _finder():
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    return of


def test_encode_embed_crops_equals_the_host_chain():
    cv2 = _cv2()
    from clearcam_b200.utils.helpers import batch_bucket
    cv2.ipp.setUseIPP(False)
    of = _finder()
    bgr = np.stack([_img(720, 1280, 40)])
    yuv = np.stack([cv2.cvtColor(bgr[0], cv2.COLOR_BGR2YUV_I420)])
    rects = [(0, 10, 20, 310, 220), (0, 600, 100, 750, 400), (0, 0, 0, 1280, 720), (0, 1100, 600, 1280, 720)]
    for frames, pix_fmt in ((bgr, "bgr24"), (yuv, "yuv420p")):
        files, emb = of.encode_embed_crops(torch.from_numpy(frames).cuda(), rects, pix_fmt=pix_fmt)
        assert files == of.encode_crops(torch.from_numpy(frames).cuda(), rects, pix_fmt=pix_fmt)
        x = [of.preprocess(cv2.cvtColor(_imdecode(f), cv2.COLOR_BGR2RGB)) for f in files]       # clearcam.py:274-276, 1280-1285
        x = np.stack(x + [np.zeros_like(x[0])] * (batch_bucket(len(x)) - len(x)))
        want = of.model.precompute_embedding(x).tensor[:len(files)]
        assert torch.equal(emb.tensor, want), pix_fmt


def test_embed_images_equals_preprocess_clip(tmp_path, monkeypatch):
    cv2 = _cv2()
    from clearcam_b200.utils.helpers import batch_bucket
    cv2.ipp.setUseIPP(False)
    of = _finder()
    img = _img(120, 90, 50)
    prog = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    good = _enc(_img(200, 300, 51), 95)
    st_, info = od.parse(good)
    off, ln = info["scan"]
    corrupt = bytearray(good)
    corrupt[off + ln // 2: off + ln // 2 + 8] = b"\xff\x00" * 4
    monkeypatch.chdir(tmp_path)
    (tmp_path / "data" / "cameras" / "cam" / "objects").mkdir(parents=True)
    (tmp_path / "data" / "cameras" / "cam" / "objects" / "a.jpg").write_bytes(_enc(_img(77, 133, 52), 85, 444))
    items = [good, "/cam/objects/a.jpg", prog, bytes(corrupt), _enc(_img(31, 20, 53), 50, "grey")]
    got = of.embed_images(items).tensor
    x = [of.preprocess_clip(it)[0] for it in items]
    x = np.stack(x + [np.zeros_like(x[0])] * (batch_bucket(len(x)) - len(x)))
    assert torch.equal(got, of.model.precompute_embedding(x).tensor[:len(items)])
    with pytest.raises(cv2.error):
        of.embed_images([good, b"not a jpeg"])
    with pytest.raises(cv2.error):
        of.embed_images(["/cam/objects/missing.jpg"])


def test_decode_and_crops_decoded_tables_refuse_bad_arguments_before_any_launch():
    L = lib()
    f = _enc(_img(20, 30, 60), 90)
    b = ops.JpegBatch([f])
    d_data, h_table, d_table = b._ptrs()
    out = torch.zeros(1, 20, 30, 3, dtype=torch.uint8, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    need = ctypes.c_size_t(0)
    assert L.cc_jpeg_decode_frames(d_data, h_table, d_table, 1, None, None, None, None, 0, ctypes.byref(need), None) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")

    def args(H=20, W=30, data=d_data, coef=None, ws_bytes=need.value):     # slot 0 of an H x W batch
        dest = (cc_jpeg_dest * 1)(cc_jpeg_dest(out.data_ptr(), 3 * W, H, W))
        return [data, h_table, d_table, 1, dest, ptr(st), coef, ptr(ws), ws_bytes, None, stream_ptr()]
    assert L.cc_jpeg_decode_frames(*args()) == 0
    assert L.cc_jpeg_decode_frames(*args(H=19)) == -1                # the image does not fit the batch
    assert L.cc_jpeg_decode_frames(*args(ws_bytes=need.value - 1)) == -1          # workspace too small
    assert L.cc_jpeg_decode_frames(*args(data=None)) == -1
    assert L.cc_jpeg_decode_frames(*args(W=0)) == -1
    assert L.cc_jpeg_decode_frames(*args(coef=ctypes.c_void_p(ws.data_ptr() + 8))) == -1     # coefficient tap not 16-byte aligned
    with pytest.raises(ValueError):
        b.decode(hmax=19)
    data = np.frombuffer(f, np.uint8).copy()
    assert L.cc_jpeg_parse(data.ctypes.data, len(f) - 1, np.array([0], np.int64).ctypes.data,
                           np.array([len(f)], np.int64).ctypes.data, 1, ctypes.c_void_p(b.host.data_ptr() + b.table_off),
                           np.zeros(2, np.int32).ctypes.data, np.zeros(1, np.int32).ctypes.data,
                           np.zeros(1, np.int64).ctypes.data) == -1   # file outside the data
    dev = torch.from_numpy(_img(40, 40, 61)[None]).cuda()
    t = ops.batch_table(dev, BGR)
    r = np.array([(0, 0, 0, 40, 40)], np.int32)
    assert L.cc_jpeg_crops_decoded_frames(t, 1, r.ctypes.data, 1, 95, ptr(out), 20, 30, ptr(st), ptr(ws), 1 << 30, None,
                                          stream_ptr()) == -1        # the crop does not fit the batch
    big = torch.zeros(1, 40, 40, 3, dtype=torch.uint8, device="cuda")
    assert L.cc_jpeg_crops_decoded_frames(t, 1, r.ctypes.data, 1, 95, ptr(big), 40, 40, None, ptr(ws), 1 << 30, None,
                                          stream_ptr()) == -1        # no status array
    t7 = ops.batch_table(dev, 7)
    assert L.cc_jpeg_crops_decoded_frames(t7, 1, r.ctypes.data, 1, 95, None, 0, 0, None, None, 0, ctypes.byref(need),
                                          None) == -1                # unknown source format
    torch.cuda.synchronize()
    assert st.cpu().item() == 0
