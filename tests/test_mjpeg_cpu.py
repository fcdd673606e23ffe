"""Motion-JPEG cameras without a GPU: the splitter cuts a stream of concatenated JPEG files back into the exact files
whatever the read sizes; the inserted Annex K tables are cv2's own DHT segments and make the decode equal cv2.imdecode of
the stripped frame; JpegMailbox, PipeReader and VideoReader carry whole files; CameraBatch on host rows treats an MJPEG
camera as a bgr24 camera fed cv2.imdecode of its frames."""
import io
import os
import threading
import time

import numpy as np
import pytest
import torch

from clearcam_b200._lib import declared_symbols
from clearcam_b200.alerts import Alert
from clearcam_b200.cameras import CameraBatch
from clearcam_b200.ingest import (JpegMailbox, MjpegSplitter, PipeReader, TABLE_ROOM, VideoReader, default_tables,
                                  with_default_tables)

cv2 = pytest.importorskip("cv2")


def _img(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([(xx * (0.9 + 0.3 * c) + yy * (0.6 + 0.2 * c) + 60 * c) % 256 for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 8, (h, w, 3)), 0, 255).astype(np.uint8)


def _enc(img, q=85, samp=420, rst=0, opt=False, prog=False):
    S = {444: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, 422: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
         420: cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420}
    p = [cv2.IMWRITE_JPEG_QUALITY, q]
    if samp == "grey":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, S[samp]]
    p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst] if rst else []
    p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1] if opt else []
    p += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1] if prog else []
    return cv2.imencode(".jpg", img, p)[1].tobytes()


def _segments(f):
    """[(marker, segment bytes)] up to and including the first SOS header, then the rest."""
    out, pos = [], 2
    while True:
        m, n = f[pos + 1], int.from_bytes(f[pos + 2:pos + 4], "big")
        out.append((m, f[pos:pos + 2 + n]))
        pos += 2 + n
        if m == 0xDA:
            return out, f[pos:]


def _strip(f, keep=()):
    """f without its DHT tables, except those whose (class, slot) is in keep."""
    segs, rest = _segments(f)
    body = b""
    for m, s in segs:
        if m == 0xC4:
            i, kept = 4, b""
            while i < len(s):
                n = 17 + sum(s[i + 1:i + 17])
                if (s[i] >> 4, s[i] & 15) in keep:
                    kept += s[i:i + n]
                i += n
            if kept:
                body += b"\xff\xc4" + (2 + len(kept)).to_bytes(2, "big") + kept
        else:
            body += s
    return f[:2] + body + rest


def _exif_with_thumbnail(f, thumb):
    """f with an APP1 Exif segment carrying a whole JPEG file (SOI ... EOI) inside."""
    payload = b"Exif\0\0MM\0*\0\0\0\x08\0\0" + thumb
    return f[:2] + b"\xff\xe1" + (2 + len(payload)).to_bytes(2, "big") + payload + f[2:]


def _files():
    a = _enc(_img(40, 56, 1), 90, 444)
    b = _enc(_img(33, 47, 2), 75, 422, rst=2)
    c = _enc(_img(64, 80, 3), 85, 420, rst=1)
    c = c[:2] + b"\xff\xfe\0\x07hello" + c[2:]                        # a COM segment
    d = _enc(_img(24, 24, 4), 60, "grey")
    e = _exif_with_thumbnail(_enc(_img(50, 30, 5), 80), _enc(_img(8, 8, 6), 50))
    p = _enc(_img(36, 52, 7), 80, prog=True)
    segs, rest = _segments(_enc(_img(20, 28, 8), 70))
    fill = rest.replace(b"\xff\xd9", b"\xff\xff\xff\xd9")            # fill bytes before EOI
    g = _enc(_img(20, 28, 8), 70)[:-len(rest)] + fill
    return [a, b, c, d, e, p, g, _strip(a)]


class _Reads(io.RawIOBase):
    """A pipe that hands out `step` bytes per read."""

    def __init__(self, data, step):
        self.b, self.step = io.BytesIO(data), step

    def readable(self):
        return True

    def readinto(self, buf):
        d = self.b.read(min(len(buf), self.step))
        buf[:len(d)] = d
        return len(d)


def _split(data, step, cap=1 << 16):
    sp, out, buf = MjpegSplitter(), [], np.empty(cap, np.uint8)
    s = _Reads(data, step)
    while True:
        n = sp.read(s, buf)
        if not n:
            return out, sp.dropped
        out.append(buf[:n].tobytes())


def test_splitter_gives_back_the_exact_files_for_every_read_size():
    files = _files()
    data = b"garbage\xff\xd8\x00" + files[0] + b"\x00\xffjunk"
    for f in files[1:]:
        data += f + b"\x13\x37"
    data += files[2][:len(files[2]) // 2]                             # a truncated last frame
    assert all(cv2.imdecode(np.frombuffer(f, np.uint8), 1) is not None for f in files[:-1])
    for step in list(range(1, 40)) + [97, 1000, 4096, len(data)]:
        got, dropped = _split(data, step)
        assert got == files and dropped == 0, step


def test_splitter_drops_an_oversize_frame_and_keeps_the_next():
    small, big = _enc(_img(16, 16, 9), 80), _enc(_img(200, 200, 10), 95)
    for step in (1, 7, 500, 1 << 20):
        got, dropped = _split(small + big + small + big, step, cap=len(big) - 1)
        assert got == [small, small] and dropped == 2, step


def test_inserted_tables_are_cv2s_dht_segments():
    f = _enc(_img(32, 48, 11), 85, 420)
    segs, _ = _segments(f)
    dht = b"".join(s for m, s in segs if m == 0xC4)
    at, seg = default_tables(_strip(f))
    assert seg == dht and len(dht) == TABLE_ROOM
    assert with_default_tables(_strip(f))[at:at + len(seg)] == dht
    assert with_default_tables(f) == f                                # tables present: byte-identical


@pytest.mark.parametrize("samp", [420, 422, 444, "grey"])
def test_stripped_frames_decode_as_cv2_decodes_them(samp):
    from oracle import jpeg_decode as od
    for opt in (False, True):
        for keep in ((), ((0, 0), (1, 0))):                           # no tables; only slot 1 missing
            f = _strip(_enc(_img(30, 44, 12), 80, samp, rst=3 if opt else 0, opt=opt), keep)
            want = cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)
            st, got = od.decode(with_default_tables(f))[:2]
            # optimised codes read with the standard tables: cv2 may warn and fill, the decoder refuses (left to cv2)
            assert st == 0 or opt, (samp, opt, keep)
            if st == 0:
                np.testing.assert_array_equal(got, want)
            assert od.decode(f)[0] != 0 or samp == "grey" and keep   # without tables the oracle still refuses


def test_jpeg_mailbox_latest_and_held_slots_under_a_concurrent_writer():
    files = [_enc(_img(24, 32, 20 + k), 80) for k in range(40)]
    mb = JpegMailbox(24, 32, pin=False)
    stream = _Reads(b"".join(files), 333)
    assert mb.pix_fmt == "mjpeg" and mb.capacity == 24 * 32 * 3 + TABLE_ROOM

    def write():
        while mb.fill(stream):
            time.sleep(0.001)
    t = threading.Thread(target=write)
    t.start()
    last, seen = -1, []
    while t.is_alive() or mb.latest(last) is not None:
        got = mb.latest(last)
        if got is None:
            time.sleep(0.0005)
            continue
        last, view = got
        held = view.numpy().tobytes()
        time.sleep(0.002)                                             # the writer keeps going; the held view must not change
        assert view.numpy().tobytes() == held == files[last]
        seen.append(last)
    t.join()
    assert seen == sorted(set(seen)) and seen[-1] == len(files) - 1


def test_pipe_reader_restarts_a_stalled_mjpeg_stream():
    opened = []

    def open_stream():
        r, w = os.pipe()
        k0 = 10 * len(opened)
        opened.append(w)

        def feed():
            try:
                with os.fdopen(w, "wb") as out:
                    for k in range(k0, k0 + 3):
                        out.write(_enc(np.full((16, 16, 3), k, np.uint8), 90))
                        out.flush()
                        time.sleep(0.01)
                    out.write(b"\xff\xd8\xff\xe0\x00")                 # stalls mid-frame; EOF follows
            except (BrokenPipeError, OSError):
                pass
        threading.Thread(target=feed, daemon=True).start()
        return os.fdopen(r, "rb")

    mb = JpegMailbox(16, 16, pin=False)
    rd = PipeReader(mb, open_stream, max_fail=2, retry_sleep=0.01)
    rd.start()
    seen, last, t0 = [], -1, time.time()
    while time.time() - t0 < 10 and not (rd.restarts >= 1 and len(seen) >= 4):
        got = mb.latest(last)
        if got is None:
            time.sleep(0.002)
            continue
        last, f = got
        seen.append(int(cv2.imdecode(f.numpy(), 1)[0, 0, 0]))
    rd.stop()
    rd.join()
    assert rd.restarts >= 1 and len(opened) >= 2
    assert any(v >= 10 for v in seen) and any(v < 10 for v in seen) and seen == sorted(seen)


@pytest.mark.parametrize("every", [1, 2, 3])
def test_video_reader_mjpeg_runs_in_order_with_positions(every):
    files = [_strip(_enc(_img(20, 24, 30 + k), 80, 422)) for k in range(17)]
    got, pos = [], []
    for frames, p in VideoReader(_Reads(b"".join(files) + files[0][:50], 97), 20, 24, "mjpeg", run=4, every=every, pin=False):
        assert isinstance(frames, list) and 1 <= len(frames) <= 4 and len(frames) == len(p)
        got += [f.numpy().tobytes() for f in frames]
        pos += p.tolist()
    keep = list(range(every - 1, len(files), every))
    assert pos == [i + 1 for i in keep]
    assert got == [with_default_tables(files[i]) for i in keep]


class _HostModel:
    """A stand-in detector with host rows whose boxes follow the frame's mean pixel."""

    def detect_batch(self, frames, pix_fmt="bgr24"):
        out = np.zeros((frames.shape[0], 300, 6), np.float32)
        for b in range(frames.shape[0]):
            s = float(frames[b].float().mean()) * 37 % 120                # jumps: new objects appear
            for i in range(4):
                x, y = 10 + 50 * i + s, 12 + 20 * i + s
                out[b, i] = [x, y, x + 50 + 5 * i, y + 70, 0.9 - 0.1 * i, i % 3]
        return torch.from_numpy(out)


def test_camera_batch_mjpeg_on_host_rows_equals_bgr24_of_imdecode():
    al = {"d": Alert.make(max=1, classes=[0, 1, 2]), "z": Alert.make(max=2, window=3, zone=False)}
    mj, bgr = CameraBatch(_HostModel()), CameraBatch(_HostModel())
    for cb, fmt in ((mj, "mjpeg"), (bgr, "bgr24")):
        for n in ("a", "b"):
            cb.add_camera(n, thresh=0.3, pix_fmt=fmt)
            cb.set_zone(n, [[0.0, 0.0], [0.7, 0.0], [0.7, 1.0], [0.0, 1.0]], False, True)
            cb.set_alerts(n, al)
    clock, fired = 1.7e9, 0
    for t in range(16):
        files = {"a": _strip(_enc(_img(240, 320, 40 + t), 80, 422)), "b": _enc(_img(180, 336, 60 + t), 85, 420, rst=1)}
        if t == 5:
            files["b"] = b"\xff\xd8 not a jpeg"
        got = mj.step_alerts(files, now=clock)
        dec = {n: cv2.imdecode(np.frombuffer(f, np.uint8), 1) for n, f in files.items()}
        want = bgr.step_alerts({n: d for n, d in dec.items() if d is not None}, now=clock)
        assert sorted(got) == sorted(want)
        for n in want:
            for u, v in zip(got[n][:4], want[n][:4]):
                np.testing.assert_array_equal(u, v)
            assert got[n].fired == want[n].fired
            fired += len(got[n].fired)
            np.testing.assert_array_equal(mj.device_frame(n).numpy(), dec[n])
        clock += 1.0
    assert fired > 0 and mj.dropped_frames == {"b": 1}
    runs = [_enc(_img(64, 64, 80 + f), 80) for f in range(3)]
    got = mj.step_video({"a": runs}, {"a": [clock + f for f in range(3)]})
    want = bgr.step_video({"a": [cv2.imdecode(np.frombuffer(f, np.uint8), 1) for f in runs]}, {"a": [clock + f for f in range(3)]})
    for g, w in zip(got["a"], want["a"]):
        for u, v in zip(g[:4], w[:4]):
            np.testing.assert_array_equal(u, v)


def test_camera_batch_mjpeg_argument_errors_before_the_detector():
    class _Never:
        def detect_batch(self, frames, pix_fmt="bgr24"):
            raise AssertionError("the detector must not run")
    cb = CameraBatch(_Never())
    with pytest.raises(ValueError, match="pix_fmt"):
        cb.add_camera("x", pix_fmt="h264")
    cb.add_camera("a", pix_fmt="mjpeg")
    cb.add_camera("b")
    with pytest.raises(ValueError, match="one JPEG file"):
        cb.step({"a": np.zeros((4, 4, 3), np.uint8)})
    with pytest.raises(ValueError, match="must be an array"):
        cb.step({"b": _enc(_img(8, 8, 1))})
    with pytest.raises(ValueError, match="not a JPEG file"):
        cb.step_video({"a": [b"nope"]}, {"a": [0.0]})


def test_decode_frames_entry_point_is_declared():
    assert "cc_jpeg_decode_frames" in declared_symbols()
