"""Every camera's object saves in one call, host side: CameraBatch.save_objects with a stand-in finder, the Python checks
of a frame table of crops (all before any library call), and the argument checks of the table entry points of the JPEG
encoder, the crops-decoded tap and the CLIP preprocess.  The GPU side is in test_object_saves_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import jpeg as oj
from clearcam_b200 import ops
from clearcam_b200.cameras import CameraBatch, CameraEvents
from clearcam_b200.detection.yolov9 import DeviceResult

from test_mixed_batch_cpu import TableDetector, _batch, _fleet


class StandInFinder:
    """Records each encode_embed_frames call; file k names its frame's first value and its rect, embedding k is k."""
    def __init__(self):
        self.calls = []

    def encode_embed_frames(self, frames, pix_fmts, rects, quality=95):
        self.calls.append((list(frames), list(pix_fmts), np.array(rects), quality))
        files = [f"{int(frames[r[0]].flatten()[0])}:{tuple(int(v) for v in r[1:])}".encode() for r in rects]
        return files, DeviceResult(torch.arange(len(rects), dtype=torch.float32)[:, None].repeat(1, 4))


def _saves(rows):
    return np.array(rows, np.int64).reshape(-1, 6)


def _events(saves):
    return CameraEvents(np.zeros((300, 6), np.float32), np.zeros((0, 7)), np.zeros(0, np.uint8), saves)


def _stepped():
    cb = _batch(TableDetector())
    frames = _fleet(0)
    cb.step(frames)
    return cb, frames


def test_a_mixed_fleet_saves_in_one_call_split_back_in_saves_order():
    cb, frames = _stepped()
    saves = {"b0": _saves([[7, 2, 1, 2, 30, 40], [3, 0, 0, 0, 128, 72]]),
             "y2": _saves([[1, 1, 10, 20, 110, 120]]),
             "square": _saves([[9, 5, 4, 4, 60, 60], [2, 5, 0, 0, 1, 1], [4, 5, 63, 63, 64, 64]]),
             "b1": _saves([]), "y0": _saves([])}
    results = {name: _events(s) for name, s in saves.items()}
    finder = StandInFinder()
    out = cb.save_objects(results, finder, quality=80)
    assert len(finder.calls) == 1
    fr, fmts, rects, q = finder.calls[0]
    assert q == 80 and len(fr) == 3 and rects.shape == (6, 5) and rects.dtype == np.int32
    cams = ["b0", "y2", "square"]                                    # cameras with saves, in results order
    for j, name in enumerate(cams):
        assert fr[j] is cb.device_frame(name) or torch.equal(fr[j], cb.device_frame(name))
        assert fmts[j] == cb.cams[name].pix_fmt
    assert fmts == ["bgr24", "yuv420p", "bgr24"]
    assert rects[:, 0].tolist() == [0, 0, 1, 2, 2, 2]
    assert (rects[:, 1:] == np.concatenate([saves[n][:, 2:6] for n in cams])).all()
    assert set(out) == set(results)
    k = 0
    for name in cams:
        s, files, emb = out[name]
        assert s is saves[name] and len(files) == len(s) and emb.tensor.shape == (len(s), 4)
        for i, row in enumerate(s):
            value = int(np.asarray(frames[name]).flatten()[0])
            assert files[i] == f"{value}:{tuple(int(v) for v in row[2:6])}".encode()
            assert emb.tensor[i, 0].item() == k
            k += 1
    for name in ("b1", "y0"):
        s, files, emb = out[name]
        assert s is saves[name] and files == [] and emb is None


def test_a_step_without_saves_makes_no_call():
    cb, _ = _stepped()
    finder = StandInFinder()
    results = {name: _events(_saves([])) for name in ("b0", "y1", "float")}
    out = cb.save_objects(results, finder)
    assert finder.calls == [] and all(out[n][1] == [] and out[n][2] is None for n in results)
    assert cb.save_objects({}, finder) == {} and finder.calls == []


def test_embeddings_none_pass_through():
    cb, _ = _stepped()

    class NoClip(StandInFinder):
        def encode_embed_frames(self, frames, pix_fmts, rects, quality=95):
            return super().encode_embed_frames(frames, pix_fmts, rects, quality)[0], None
    out = cb.save_objects({"b2": _events(_saves([[1, 0, 0, 0, 10, 10]]))}, NoClip())
    assert len(out["b2"][1]) == 1 and out["b2"][2] is None


# ------------------------------------------------------------------------------------------------ Python table checks
class _FakeCuda(torch.Tensor):
    """A host tensor that reports itself as a CUDA tensor: the table checks read only its metadata."""
    @property
    def is_cuda(self):
        return True


def _dev(shape, dtype=torch.uint8):
    return torch.zeros(shape, dtype=dtype).as_subclass(_FakeCuda)


@pytest.fixture
def no_library(monkeypatch):
    calls = []

    def refuse():
        calls.append(1)
        raise AssertionError("the library was called")
    monkeypatch.setattr(ops, "lib", refuse)
    yield calls
    assert calls == []


def test_table_checks_raise_before_any_library_call(no_library):
    from clearcam_b200.models.objects import ObjectFinder
    big, small = _dev((64, 96, 3)), _dev((24 * 3 // 2, 32))
    table, sizes = ops.frame_table([big, small], ["bgr24", "yuv420p"])
    assert sizes == [(64, 96), (24, 32)] and [table[i].fmt for i in range(2)] == [0, 2]
    assert [(table[i].h, table[i].w) for i in range(2)] == [(64, 96), (24, 32)]
    ops.table_rects([(0, 0, 0, 96, 64), (1, 31, 23, 32, 24)], sizes)
    of = ObjectFinder()
    bad = {
        "float32 frame": ([_dev((64, 96, 3), torch.float32), small], ["bgr24", "yuv420p"], [(0, 0, 0, 8, 8)]),
        "odd I420 size": ([big, _dev((25 * 3 // 2 + 1, 33))], ["bgr24", "yuv420p"], [(1, 0, 0, 8, 8)]),
        "odd I420 width": ([big, _dev((24 * 3 // 2, 33))], ["bgr24", "yuv420p"], [(1, 0, 0, 8, 8)]),
        "rect outside its own frame": ([big, small], ["bgr24", "yuv420p"], [(0, 0, 0, 8, 8), (1, 30, 10, 60, 20)]),
        "rect below its own frame": ([big, small], ["bgr24", "yuv420p"], [(1, 0, 20, 8, 25)]),
        "frame index outside the table": ([big, small], ["bgr24", "yuv420p"], [(2, 0, 0, 8, 8)]),
        "empty rect": ([big, small], ["bgr24", "yuv420p"], [(0, 5, 5, 5, 9)]),
        "more formats than frames": ([big, small], ["bgr24", "yuv420p", "bgr24"], [(0, 0, 0, 8, 8)]),
        "fewer formats than frames": ([big, small], ["bgr24"], [(0, 0, 0, 8, 8)]),
        "unknown format": ([big, small], ["bgr24", "rgb24"], [(0, 0, 0, 8, 8)]),
        "host frame": ([torch.zeros(64, 96, 3, dtype=torch.uint8), small], ["bgr24", "yuv420p"], [(0, 0, 0, 8, 8)]),
        "padding row": ([big, None], ["bgr24", "bgr24"], [(0, 0, 0, 8, 8)]),
        "bgr24 shape": ([_dev((64, 96)), small], ["bgr24", "yuv420p"], [(0, 0, 0, 8, 8)]),
    }
    for what, (frames, fmts, rects) in bad.items():
        with pytest.raises(ValueError):
            of.encode_embed_frames(frames, fmts, rects)
            pytest.fail(what)
        with pytest.raises(ValueError):
            ops.table_rects(rects, ops.frame_table(frames, fmts)[1])
    with pytest.raises(ValueError):
        of.encode_embed_frames([big], "bgr24", [(0, 0, 0, 8, 8)], quality=101)


def test_detector_frame_table_keeps_its_checks():
    from clearcam_b200.detection.yolov9 import frame_table
    from clearcam_b200._lib import CC_MAX_FRAMES
    f = _dev((72, 128, 3))
    table, net = frame_table([f, None], ["bgr24", "bgr24"], 640)
    assert net == (384, 640) and table[1].data is None
    for frames, fmts in (([f], ["bgr24", "bgr24"]), ([None, None], "bgr24"), ([f] * (CC_MAX_FRAMES + 1), "bgr24"),
                         ([f, _dev((64, 64, 3))], "bgr24"), ([_dev((72, 128, 3), torch.float32)], "bgr24")):
        with pytest.raises(ValueError):
            frame_table(frames, fmts, 640)


# ------------------------------------------------------------------------------------------------ C-ABI argument checks
def test_crop_tables_reject_bad_arguments_and_take_rgb():
    """Every check runs before anything is launched: the device pointers below are never dereferenced."""
    from clearcam_b200._lib import cc_frame, lib
    h = lib()
    fake = 1 << 20
    need = ctypes.c_size_t(0)

    def refused(rc, *words):
        msg = h.cc_last_error().decode()
        assert rc == -1 and all(w in msg for w in words), (rc, msg, words)

    good = [cc_frame(fake, 0, 240, 320), cc_frame(fake + (1 << 24), 2, 480, 640), cc_frame(fake + (1 << 25), 0, 33, 17)]
    rects = np.array([[0, 0, 0, 320, 240], [1, 100, 200, 640, 480], [2, 0, 0, 17, 33], [1, 0, 0, 1, 1]], np.int32)
    bounds = [oj.bound(r[3] - r[1], r[4] - r[2]) for r in rects]
    offs = np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.int64)
    cap = int(sum(bounds))

    def table(rows):
        return (cc_frame * max(len(rows), 1))(*rows)

    def enc(frames=good, n=None, r=rects, K=None, q=95, out=fake, cap=cap, offsets=offs, lengths=fake, ws=fake, wsb=1 << 30,
            need=ctypes.byref(need)):
        return h.cc_jpeg_encode_crops_frames(None if frames is None else table(frames), len(frames or []) if n is None else n,
                                             None if r is None else r.ctypes.data, len(r) if K is None and r is not None else K or 0,
                                             q, out, cap, None if offsets is None else offsets.ctypes.data, lengths, ws, wsb,
                                             need, None)

    def dec(frames=good, r=rects, q=95, out=None, H=0, W=0, st=None, ws=None, wsb=0, need=ctypes.byref(need)):
        return h.cc_jpeg_crops_decoded_frames(table(frames), len(frames), r.ctypes.data, len(r), q, out, H, W, st, ws, wsb, need,
                                              None)

    def pre(frames=good, r=rects, size=224, out=fake):
        return h.cc_clip_preprocess_frames(table(frames), len(frames), r.ctypes.data, len(r), size, out, None)

    assert enc(out=None) == 0 and need.value > 0
    assert dec() == 0 and need.value > 0
    rgb = [cc_frame(f.data, 3 if f.fmt == 0 else f.fmt, f.h, f.w) for f in good]      # CC_FRAME_RGB_U8: the crops take it
    assert enc(frames=rgb, out=None) == 0 and dec(frames=rgb) == 0
    odd_i420 = [good[0], cc_frame(fake, 2, 481, 640), good[2]]
    cases = [
        (dict(frames=[good[0], cc_frame(None, 0, 480, 640), good[2]]), ["frame 1 is NULL"]),
        (dict(frames=[good[0], cc_frame(fake, 1, 480, 640), good[2]]), ["frame 1 has format 1"]),
        (dict(frames=[good[0], cc_frame(fake, 4, 480, 640), good[2]]), ["frame 1 has format 4"]),
        (dict(frames=odd_i420), ["frame 1", "even height and width"]),
        (dict(frames=[good[0], cc_frame(fake, 2, 480, 639), good[2]]), ["frame 1", "even height and width"]),
        (dict(frames=[good[0], good[1], cc_frame(fake, 0, 0, 17)]), ["frame 2 has a bad size"]),
        (dict(r=np.array([[0, 0, 0, 320, 241]], np.int32)), ["rect 0", "outside its 320x240 frame"]),
        # inside the 640 x 480 frame 1 of the table, outside its own 320 x 240 frame 0
        (dict(r=np.array([[1, 0, 0, 8, 8], [0, 300, 200, 400, 300]], np.int32)), ["rect 1", "outside its 320x240 frame"]),
        (dict(r=np.array([[2, 0, 0, 18, 33]], np.int32)), ["rect 0", "outside its 17x33 frame"]),
        (dict(r=np.array([[3, 0, 0, 8, 8]], np.int32)), ["rect 0 names frame 3 of a 3-frame table"]),
        (dict(r=np.array([[-1, 0, 0, 8, 8]], np.int32)), ["rect 0 names frame -1"]),
        (dict(r=np.array([[0, 5, 5, 5, 9]], np.int32)), ["rect 0", "empty or outside"]),
    ]
    for kw, words in cases:
        refused(enc(**kw), "cc_jpeg_encode_crops_frames", *words)
        refused(dec(**kw), "cc_jpeg_crops_decoded_frames", *words)
        refused(pre(**kw), "cc_clip_preprocess_frames", *words)
    refused(enc(frames=None, n=2), "cc_jpeg_encode_crops_frames", "null pointer")
    refused(enc(r=None, K=2), "cc_jpeg_encode_crops_frames", "null pointer")
    refused(enc(frames=[], n=0, r=rects[:0]), "cc_jpeg_encode_crops_frames", "bad sizes")
    refused(enc(q=-1), "cc_jpeg_encode_crops_frames", "quality -1")
    refused(dec(q=101), "cc_jpeg_crops_decoded_frames", "quality 101")
    refused(enc(offsets=None), "out_offsets and d_lengths")
    refused(enc(wsb=1), "workspace of", "too small")
    refused(enc(cap=cap - 1), "crop 3", "exceeds the output capacity")
    refused(enc(offsets=np.array([0, bounds[0] - 1, offs[2], offs[3]], np.int64)), "crops 0 and 1 overlap")
    refused(dec(out=fake, H=240, W=100, st=fake, ws=fake, wsb=1 << 30), "cc_jpeg_crops_decoded_frames", "does not fit")
    refused(dec(out=fake, H=480, W=640, st=None, ws=fake, wsb=1 << 30), "d_status must not be NULL")
    refused(pre(size=0), "cc_clip_preprocess_frames", "bad size 0")
    refused(pre(out=None), "cc_clip_preprocess_frames", "null pointer")
    big = np.array([[0, 0, 0, 320, 240]], np.int32)
    refused(enc(frames=[cc_frame(fake, 0, 70000, 70000)], r=np.array([[0, 0, 0, 65536, 8]], np.int32)), "larger than 65535")
    assert enc(r=big, out=None) == 0
    # RGB frames are for the crops only: the letterbox and the face canvas refuse them before any device query
    oh, ow = ctypes.c_int(), ctypes.c_int()
    refused(h.cc_letterbox_frames((cc_frame * 1)(rgb[0]), 1, 640, None, ctypes.byref(oh), ctypes.byref(ow), None),
            "cc_letterbox_frames", "frame 0 has format 3")
    assert h.cc_letterbox_frames((cc_frame * 1)(good[0]), 1, 640, None, ctypes.byref(oh), ctypes.byref(ow), None) == 0
    refused(h.cc_face_canvas((cc_frame * 1)(rgb[0]), 1, fake, None), "cc_face_canvas", "format 3")
