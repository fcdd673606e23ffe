"""Recorded videos without a GPU: VideoReader keeps every frame in order (every=1) or the second of each pair (every=2,
as grab() + read()), reports cv2's CAP_PROP_POS_FRAMES, gives a short last run and drops a partial last frame;
CameraBatch.step_video on host rows equals successive step_alerts calls with the same clocks; save_objects and
describe_saves take its results; the run entry points are exported."""
import io

import numpy as np
import pytest
import torch

from clearcam_b200._lib import CC_MAX_FRAMES, declared_symbols
from clearcam_b200.alerts import Alert
from clearcam_b200.cameras import CameraBatch
from clearcam_b200.ingest import VideoReader


class _Chunked(io.RawIOBase):
    """A pipe that hands out at most 1000 bytes per read."""

    def __init__(self, data):
        self.b = io.BytesIO(data)

    def readable(self):
        return True

    def readinto(self, buf):
        d = self.b.read(min(len(buf), 1000))
        buf[:len(d)] = d
        return len(d)


def _video(n, H, W, fmt="bgr24"):
    shape = (H, W, 3) if fmt == "bgr24" else (H * 3 // 2, W)
    return [np.random.default_rng(i).integers(0, 255, shape, dtype=np.uint8) for i in range(n)]


@pytest.mark.parametrize("every", [1, 2, 3])
@pytest.mark.parametrize("fmt", ["bgr24", "yuv420p"])
def test_video_reader_every_frame_in_order_with_positions(every, fmt):
    H, W, n, run = 6, 8, 23, 4
    fr = _video(n, H, W, fmt)
    data = b"".join(f.tobytes() for f in fr) + b"\x07" * 5            # a partial last frame
    got, pos = [], []
    for frames, p in VideoReader(_Chunked(data), H, W, fmt, run=run, every=every, pin=False):
        assert frames.shape[1:] == fr[0].shape and 1 <= len(frames) <= run
        got += [f.numpy().copy() for f in frames]
        pos += p.tolist()
    keep = list(range(every - 1, n, every))                           # grab() x (every-1), then read()
    assert pos == [i + 1 for i in keep]                               # cv2's CAP_PROP_POS_FRAMES after each read
    assert len(got) == len(keep)
    for g, i in zip(got, keep):
        np.testing.assert_array_equal(g, fr[i])


def test_video_reader_short_last_run_and_empty_stream():
    fr = _video(10, 4, 4)
    runs = [len(f) for f, _ in VideoReader(io.BytesIO(b"".join(f.tobytes() for f in fr)), 4, 4, run=4, every=1, pin=False)]
    assert runs == [4, 4, 2]
    assert list(VideoReader(io.BytesIO(b""), 4, 4, pin=False)) == []
    with pytest.raises(ValueError):
        VideoReader(io.BytesIO(b""), 4, 4, run=0, pin=False)


class _Failing(io.RawIOBase):
    """A pipe whose reads fail after `good` bytes."""

    def __init__(self, data, good):
        self.b, self.good = io.BytesIO(data), good

    def readable(self):
        return True

    def readinto(self, buf):
        if self.b.tell() >= self.good:
            raise OSError("read failed")
        d = self.b.read(min(len(buf), self.good - self.b.tell()))
        buf[:len(d)] = d
        return len(d)


def test_video_reader_raises_a_read_error_and_closes_early():
    fr = _video(10, 4, 4)
    data = b"".join(f.tobytes() for f in fr)
    r = VideoReader(_Failing(data, 5 * 48 + 7), 4, 4, run=2, every=1, pin=False)
    got = []
    with pytest.raises(OSError, match="read failed"):
        for f, _ in r:
            got.append(len(f))
    assert got == [2, 2]                                              # the runs read before the error
    with VideoReader(io.BytesIO(data * 50), 4, 4, run=2, every=1, pin=False) as r:
        next(r)                                                       # stop after one run: the thread ends on close
    assert not r._thread.is_alive()


class _HostModel:
    """A stand-in detector with host rows: boxes that move with the frame's first pixel."""

    def detect_batch(self, frames, pix_fmt="bgr24"):
        out = np.zeros((frames.shape[0], 300, 6), np.float32)
        for b in range(frames.shape[0]):
            s = float(frames[b, 0, 0, 0] if frames.dim() == 4 else frames[b, 0, 0])
            for i in range(5):
                x, y = 20 + 90 * i + 9 * s, 15 + 40 * i + 4 * s
                out[b, i] = [x, y, x + 120 + 10 * i, y + 150, 0.9 - 0.05 * i, i % 3]
        return torch.from_numpy(out)


class _Finder:
    """encode_embed_frames on the host: a file per crop naming its frame's first pixel and rectangle, an embedding per crop."""

    def encode_embed_frames(self, frames, pix_fmts, rects, quality=95):
        files = [f"{int(frames[r[0]].reshape(-1)[0])}:{r[1]},{r[2]},{r[3]},{r[4]}".encode() for r in rects]
        emb = np.stack([np.cos(np.arange(8) * (1 + int(frames[r[0]].reshape(-1)[0]) + r[1])) for r in rects]).astype(np.float32)
        return files, _Emb(torch.from_numpy(emb))


class _Emb:
    def __init__(self, t):
        self.tensor = t


def _frames(T, H, W, t0, fmt="bgr24"):
    if fmt == "bgr24":
        return torch.stack([torch.full((H, W, 3), t0 + t, dtype=torch.uint8) for t in range(T)])
    return torch.stack([torch.full((H * 3 // 2, W), t0 + t, dtype=torch.uint8) for t in range(T)])


def test_step_video_on_host_rows_equals_successive_step_alerts():
    """Two videos (bgr24 and yuv420p) with zones and alerts, runs of 5, 1 and 7 frames, then a step_alerts on the same
    cameras: every frame's rows, preds, flags, saves and fired ids equal step_alerts frame by frame on a second batch;
    save_objects cuts each save from its own frame; describe_saves matches each frame at its own clock."""
    cams = {"a": ((240, 320), "bgr24"), "b": ((240, 320), "yuv420p")}
    al = {"d": Alert.make(max=1, classes=[0, 1, 2]), "z": Alert.make(max=2, window=3, zone=False),
          "t": Alert.make(desc="x", threshold=-10.0)}
    desc = np.ones((1, 8), np.float32)
    video, single = CameraBatch(_HostModel()), CameraBatch(_HostModel())
    for cb in (video, single):
        cb._desc["x"] = desc[0]
        for n, (_, fmt) in cams.items():
            cb.add_camera(n, thresh=0.3, pix_fmt=fmt)
            cb.set_zone(n, [[0.0, 0.0], [0.6, 0.0], [0.6, 1.0], [0.0, 1.0]], False, True)
            cb.set_alerts(n, al)
    t0, clock, fired, saves, hits = 0, 1.7e9, 0, 0, 0
    for T in (5, 1, 7):
        frames = {n: _frames(T, H, W, t0 + 3 * i, fmt) for i, (n, ((H, W), fmt)) in enumerate(cams.items())}
        clocks = {n: [clock + 1.5 * f for f in range(T)] for n in cams}
        res = video.step_video(frames, clocks)
        saved = video.save_objects(res, _Finder())
        desc_hits = video.describe_saves(saved, now=clocks)
        for n in cams:
            assert len(res[n]) == T
            rows7, files, emb = saved[n]
            want_saves, want_files, want_hits, k = [], [], [], 0
            for f in range(T):
                one = single.step_alerts({n: frames[n][f]}, now=clocks[n][f])[n]
                for u, v in zip(res[n][f][:4], one[:4]):
                    np.testing.assert_array_equal(u, v)
                assert res[n][f].fired == one.fired
                fired += len(one.fired)
                sv = single.save_objects({n: one}, _Finder())
                want_saves += [np.concatenate([[f], s]) for s in np.asarray(sv[n][0])]
                want_files += sv[n][1]
                want_hits += [(k + s, a, v) for s, a, v in single.describe_saves(sv, now=clocks[n][f])[n]]
                k += len(sv[n][1])
            np.testing.assert_array_equal(rows7, np.array(want_saves, np.int64).reshape(-1, 7))
            assert files == want_files
            assert desc_hits[n] == want_hits
            saves += len(files)
            hits += len(want_hits)
        clock += 1.5 * T
        t0 += T
    assert fired > 0 and saves > 0 and hits > 0
    # the same cameras step once more, frame by frame: one state
    one = {n: single.step_alerts({n: _frames(1, H, W, t0, fmt)[0]}, now=clock)[n] for n, ((H, W), fmt) in cams.items()}
    got = video.step_alerts({n: _frames(1, H, W, t0, fmt)[0] for n, ((H, W), fmt) in cams.items()}, now=clock)
    for n in cams:
        for u, v in zip(got[n][1:4], one[n][1:4]):
            np.testing.assert_array_equal(u, v)
        np.testing.assert_array_equal(video.object_counts(n), single.object_counts(n))


def test_step_video_argument_errors_before_the_detector():
    class _Never:
        def detect_batch(self, frames, pix_fmt="bgr24"):
            raise AssertionError("the detector must not run")
    cb = CameraBatch(_Never())
    cb.add_camera("a")
    f = _frames(3, 8, 8, 0)
    with pytest.raises(ValueError, match="one finite clock per frame"):
        cb.step_video({"a": f}, {"a": [0.0, 1.0]})
    with pytest.raises(ValueError, match="one finite clock per frame"):
        cb.step_video({"a": f}, {"a": [0.0, float("nan"), 1.0]})
    with pytest.raises(ValueError, match="frames"):
        cb.step_video({"a": _frames(CC_MAX_FRAMES + 1, 2, 2, 0)}, {"a": [0.0] * (CC_MAX_FRAMES + 1)})
    with pytest.raises(ValueError, match="one local time per frame"):
        cb.step_video({"a": f}, {"a": [0.0, 1.0, 2.0]}, local={"a": [(0.0, 0)]})


def test_run_entry_points_are_declared():
    for name in ("cc_ocsort_gpu_update_runs", "cc_ocsort_gpu_events_runs", "cc_ocsort_gpu_alerts_runs", "cc_ocsort_gpu_describe_runs"):
        assert name in declared_symbols()
