"""Motion-JPEG cameras on the GPU: cc_jpeg_decode_frames writes cv2.imdecode of every file into its destination and
nothing else; the coefficient tap of large files without restart markers equals the oracle's; an MJPEG fleet through
JpegMailbox -> step_alerts_mailboxes -> save_objects -> describe_saves equals a twin CameraBatch fed the cv2-decoded
frames as bgr24, through parse-time and device-time fallbacks, a dropped frame and a resolution change; step_video runs
of JPEG files equal step_video of their cv2 pictures."""
import ctypes
import io
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200._lib import cc_jpeg_dest, lib, ptr, stream_ptr
from clearcam_b200.alerts import Alert
from clearcam_b200.ingest import FrameMailbox, JpegMailbox, with_default_tables

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
cv2 = pytest.importorskip("cv2")


def _img(h, w, seed, sigma=8):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([(xx * (0.9 + 0.3 * c) + yy * (0.6 + 0.2 * c) + 60 * c) % 256 for c in range(3)], -1)
    return np.clip(base + rng.normal(0, sigma, (h, w, 3)), 0, 255).astype(np.uint8)


def _enc(img, q=85, samp=420, rst=0, prog=False):
    S = {444: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, 422: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
         420: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
    p = [cv2.IMWRITE_JPEG_QUALITY, q]
    if samp == "grey":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, S[samp]]
    p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst] if rst else []
    p += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1] if prog else []
    return cv2.imencode(".jpg", img, p)[1].tobytes()


def _strip(f):
    """f without its DHT segments (what a Motion-JPEG camera sends)."""
    out, pos = bytearray(f[:2]), 2
    while True:
        m, n = f[pos + 1], int.from_bytes(f[pos + 2:pos + 4], "big")
        if m != 0xC4:
            out += f[pos:pos + 2 + n]
        pos += 2 + n
        if m == 0xDA:
            return bytes(out) + f[pos:]


def _imdecode(f):
    return cv2.imdecode(np.frombuffer(bytes(f), np.uint8), cv2.IMREAD_COLOR)


def test_decode_frames_into_pitched_rows_and_buffers_touches_nothing_else():
    rng = np.random.default_rng(3)
    files = []
    for i in range(150):                                              # K > 128: two reconstruction launches
        h, w = int(rng.integers(1, 120)), int(rng.integers(1, 160))
        files.append(_enc(_img(h, w, i), int(rng.integers(20, 100)), (420, 422, 444, "grey")[i % 4], rst=(0, 1, 4)[i % 3]))
    good = _enc(_img(100, 150, 7), 90)
    files[7] = good[:len(good) * 2 // 3]                              # a truncated scan: parsed, then corrupt on the device
    dec = ops.JpegDecoder()
    sizes, status = dec.stage(files)
    assert status[7] == ops.JPEG_OK
    Hm, Wm = int(sizes[:, 1].max()), int(sizes[:, 0].max())
    batch = torch.full((75, Hm + 2, Wm + 3, 3), 0xA5, dtype=torch.uint8, device="cuda")   # pitched rows of one batch
    own = [torch.full((int(h) + 1, int(w) + 1, 3), 0x5A, dtype=torch.uint8, device="cuda") for w, h in sizes[75:]]
    dests = [batch[k, :int(sizes[k, 1]), :int(sizes[k, 0])] for k in range(75)] + \
            [own[j][:int(sizes[75 + j, 1]), :int(sizes[75 + j, 0])] for j in range(75)]
    st = dec.decode(dests)
    torch.cuda.synchronize()
    st = st.numpy().copy()
    assert st[7] == ops.JPEG_CORRUPT and (np.delete(st, 7) == ops.JPEG_OK).all()
    ref, _, _ = ops.jpeg_decode(files)
    ref = ref.cpu().numpy()
    b = batch.cpu().numpy()
    written = np.zeros(b.shape[:3], bool)
    for k in range(150):
        w, h = sizes[k]
        got = dests[k].cpu().numpy()
        if k == 7:
            assert (got == (0xA5 if k < 75 else 0x5A)).all()          # left as it was
            continue
        np.testing.assert_array_equal(got, _imdecode(files[k]))
        np.testing.assert_array_equal(got, ref[k, :h, :w])
        if k < 75:
            written[k, :h, :w] = True
        else:
            o = own[k - 75].cpu().numpy()
            assert (o[h:] == 0x5A).all() and (o[:, w:] == 0x5A).all()
    assert (b[~written] == 0xA5).all()


def test_decode_frames_refuses_bad_destinations_before_launch():
    f = _enc(_img(20, 30, 60), 90)
    dec = ops.JpegDecoder()
    dec.stage([f, f])
    out = torch.full((2, 20, 30, 3), 7, dtype=torch.uint8, device="cuda")
    dec.decode([out[0], out[1]])
    torch.cuda.synchronize()
    base = dec._dev.data_ptr()
    args = (ctypes.c_void_p(base), ctypes.c_void_p(dec._host.data_ptr() + dec._table_off), ctypes.c_void_p(base + dec._table_off), 2)
    L = lib()
    big = torch.full((40, 40, 3), 9, dtype=torch.uint8, device="cuda")

    def call(*d):
        outs = (cc_jpeg_dest * 2)(*d)
        return L.cc_jpeg_decode_frames(*args, outs, ptr(dec._st_dev), None, ptr(dec._ws), dec._ws.numel(), None, stream_ptr())
    ok = cc_jpeg_dest(out[0].data_ptr(), 90, 20, 30), cc_jpeg_dest(out[1].data_ptr(), 90, 20, 30)
    assert call(*ok) == 0
    assert call(ok[0], cc_jpeg_dest(big.data_ptr(), 120, 21, 30)) == -1              # not the image's size
    assert call(ok[0], cc_jpeg_dest(big.data_ptr(), 89, 20, 30)) == -1               # pitch below 3 w
    assert call(ok[0], cc_jpeg_dest(out[0].data_ptr() + 90 * 19, 90, 20, 30)) == -1  # overlaps the first
    assert call(ok[0], cc_jpeg_dest(None, 90, 20, 30)) == -1
    assert L.cc_jpeg_decode_frames(*args, (cc_jpeg_dest * 2)(*ok), ptr(dec._st_dev), None, ptr(dec._ws), 1, None, stream_ptr()) == -1
    out.fill_(3)
    big.fill_(3)
    for bad in ((ok[0], cc_jpeg_dest(big.data_ptr(), 120, 21, 30)), (ok[0], cc_jpeg_dest(big.data_ptr(), 89, 20, 30))):
        assert call(*bad) == -1
    torch.cuda.synchronize()
    assert (out == 3).all() and (big == 3).all()                     # a refused call launched nothing


@pytest.mark.parametrize("hw", [(1080, 1920), (2160, 3840)])
def test_dc_values_of_large_files_without_restart_markers_equal_the_oracle(hw):
    from oracle import jpeg_decode as od
    for samp in (420, 422):
        f = _enc(_img(*hw, 70, sigma=6), 85, samp)
        got, st = ops.jpeg_decode_coeffs([f])
        assert int(st.cpu()[0]) == 0
        assert np.array_equal(got.cpu().numpy(), od.coeffs(f))
        _, _, st = ops.jpeg_decode([_strip(f)])                       # no tables: left to the host, as before
        assert int(st.cpu()[0]) == ops.JPEG_UNSUPPORTED
        dec = ops.JpegDecoder()
        dst = torch.empty(hw + (3,), dtype=torch.uint8, device="cuda")
        dec.stage([with_default_tables(_strip(f))])
        s = dec.decode([dst])
        torch.cuda.synchronize()
        assert int(s[0]) == 0
        np.testing.assert_array_equal(dst.cpu().numpy(), _imdecode(_strip(f)))


def _finder():
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS["ViT-B/32"], seed=3), arch="ViT-B/32")
    return of


def _model():
    sys.path.insert(0, str(ROOT))
    from oracle import yolov9 as o
    from clearcam_b200.detection.yolov9 import YOLOv9
    xc = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    return YOLOv9("c", 320, weights=o.synthetic_weights("c", seed=5, calib=xc)), o


def _yuv(f):
    return cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420)


class _Bytes:
    """A mailbox that publishes one given JPEG file (a file a JpegMailbox would not publish, stepped beside the others)."""
    pix_fmt = "mjpeg"

    def __init__(self, f, num):
        self.f, self.num = f, num

    def latest(self, last_seen=-1):
        return self.num, self.f


def test_mjpeg_fleet_through_mailboxes_equals_bgr24_of_imdecode(monkeypatch):
    from clearcam_b200.cameras import CameraBatch
    statuses = []
    decode = ops.JpegDecoder.decode

    def record(self, dests, stream=None):                              # read after the step's status wait
        st = decode(self, dests, stream)
        statuses.append(st)
        return st
    monkeypatch.setattr(ops.JpegDecoder, "decode", record)
    m, o = _model()
    of = _finder()
    # name: (H, W), format, sampling, tables, restart interval
    cams = {"m720": ((720, 1280), "mjpeg", 422, False, 0), "m1080": ((1080, 1920), "mjpeg", 420, True, 120),
            "m1440": ((1440, 2560), "mjpeg", 422, True, 0), "m2160": ((2160, 3840), "mjpeg", 420, False, 240),
            "b1080": ((1080, 1920), "bgr24", 0, 0, 0), "y720": ((720, 1280), "yuv420p", 0, 0, 0)}
    al = {"default": Alert.make(max=1, classes=[0, 1, 2, 3, 5, 7]), "any": Alert.make(max=2, window=3, zone=False),
          "thing": Alert.make(desc="a thing", threshold=-1.0)}
    mj, twin = CameraBatch(m), CameraBatch(m)
    for n, (_, fmt, *_r) in cams.items():
        for cb, f in ((mj, fmt), (twin, "yuv420p" if fmt == "yuv420p" else "bgr24")):
            cb.add_camera(n, thresh=0.05, pix_fmt=f)
            cb.set_zone(n, [[0.0, 0.0], [0.7, 0.0], [0.7, 1.0], [0.0, 1.0]], False, True)
            cb.set_alerts(n, al, of)
    base = {n: o.synthetic_frames(1, H, W, seed=90 + i)[0].numpy() for i, (n, ((H, W), *_r)) in enumerate(cams.items())}
    boxes = {n: JpegMailbox(*cams[n][0], pin=True) if cams[n][1] == "mjpeg" else FrameMailbox(*cams[n][0], pin=True, pix_fmt=cams[n][1])
             for n in cams}
    T0, fired, saves, drops = 1.7e9, 0, 0, {}
    for t in range(20):
        now = T0 + 3.0 * t
        want_in, mb_in = {}, {}
        for n, ((H, W), fmt, samp, tables, rst) in cams.items():
            img = np.ascontiguousarray(np.roll(base[n], (5 * t, 7 * t), (0, 1)))
            if fmt != "mjpeg":
                want_in[n] = _yuv(img) if fmt == "yuv420p" else img
                assert boxes[n].fill(io.BytesIO(want_in[n].tobytes()))
                mb_in[n] = boxes[n]
                continue
            if n == "m2160" and t >= 13:                              # a resolution change
                img = np.ascontiguousarray(img[::2, ::2])
            f = _enc(img, 85, samp, rst=rst // (2 if n == "m2160" and t >= 13 else 1))
            f = f if tables else _strip(f)
            if n == "m720" and t == 7:
                f = _enc(img, 85, 422, prog=True)                     # parse-time fallback
            if n == "m1080" and t == 9:                               # an invalid code: device-time fallback
                from oracle import jpeg_decode as od
                off, ln = od.parse(f)[1]["scan"]
                f = f[:off + ln // 2] + b"\xff\x00" * 4 + f[off + ln // 2 + 8:]
            if n == "m1440" and t == 11:
                f = b"\xff\xd8\xff\xdb\x00\x03" + b"\x00" * 64        # the parse and cv2 reject it: dropped
            if n == "m720" and t == 11:
                f = f[:len(f) * 2 // 3]                               # parsed, then the device and cv2 reject it: dropped
            if (n, t) in (("m1080", 9), ("m1440", 11), ("m720", 11)):
                mb_in[n] = _Bytes(with_default_tables(f), -2 - t)     # a JpegMailbox publishes whole files only
            else:
                assert boxes[n].fill(io.BytesIO(f))
                mb_in[n] = boxes[n]
            d = _imdecode(f)
            if d is not None:
                want_in[n] = d
            else:
                drops[n] = drops.get(n, 0) + 1
        res = mj.step_alerts_mailboxes(mb_in, now=now)
        st = statuses[-1].numpy().tolist()
        assert len(st) == 4 and st.count(ops.JPEG_OK) == 4 - (t in (7, 9)) - 2 * (t == 11), (t, st)
        if t == 7:
            assert ops.JPEG_UNSUPPORTED in st                          # the progressive frame, from the parse
        if t in (9, 11):
            assert ops.JPEG_CORRUPT in st                              # found on the device
        want = twin.step_alerts(want_in, now=now)
        assert sorted(res) == sorted(want)
        for n in want:
            np.testing.assert_array_equal(res[n].rows, want[n].rows)
            for u, v in zip(res[n][1:4], want[n][1:4]):
                np.testing.assert_array_equal(u, v)
            assert res[n].fired == want[n].fired
            fired += len(res[n].fired)
            assert torch.equal(mj.device_frame(n), twin.device_frame(n)), (n, t)
        s1, s2 = mj.save_objects(res, of), twin.save_objects(want, of)
        for n in want:
            np.testing.assert_array_equal(np.asarray(s1[n][0]), np.asarray(s2[n][0]))
            assert s1[n][1] == s2[n][1]
            if s2[n][2] is not None:
                assert torch.equal(s1[n][2].tensor, s2[n][2].tensor)
            saves += len(s1[n][1])
        assert mj.describe_saves(s1, now=now) == twin.describe_saves(s2, now=now)
    assert mj.dropped_frames == drops == {"m720": 1, "m1440": 1}
    assert len(statuses) == 20
    assert fired > 0 and saves > 0


@pytest.mark.parametrize("T", [1, 7, 32])
def test_step_video_mjpeg_runs_equal_bgr24_runs(T):
    from clearcam_b200.cameras import CameraBatch
    m, o = _model()
    vid, twin = CameraBatch(m), CameraBatch(m)
    vid.add_camera("v", thresh=0.05, pix_fmt="mjpeg")
    twin.add_camera("v", thresh=0.05)
    base = o.synthetic_frames(1, 360, 640, seed=11)[0].numpy()
    files = [_strip(_enc(np.ascontiguousarray(np.roll(base, (3 * t, 5 * t), (0, 1))), 85, 422, rst=40 * (t % 2)))
             for t in range(T)]
    clocks = {"v": [1.7e9 + 0.5 * t for t in range(T)]}
    got = vid.step_video({"v": files}, clocks)["v"]
    want = twin.step_video({"v": torch.from_numpy(np.stack([_imdecode(f) for f in files]))}, clocks)["v"]
    for g, w in zip(got, want):
        for u, v in zip(g[:4], w[:4]):
            np.testing.assert_array_equal(u, v)
        assert g.fired == w.fired
    for f in range(T):
        assert torch.equal(vid.device_frame(("v", f)), twin.device_frame(("v", f)))
