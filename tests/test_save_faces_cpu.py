"""The faces of the object saves, host side: CameraBatch.save_objects_and_faces with a stand-in finder (person selection,
rows mapped back per camera and per run frame, no call without saves), ObjectFinder's checks before any library call, and
the argument checks of the slot face kernels and cc_blazeface_first.  The GPU side is in test_save_faces_gpu.py."""
import numpy as np
import pytest
import torch

from clearcam_b200 import ops
from clearcam_b200.cameras import CameraBatch
from clearcam_b200.detection.yolov9 import DeviceResult
from clearcam_b200.models.objects import FaceSaves, ObjectFinder

from test_mixed_batch_cpu import TableDetector, _batch, _fleet
from test_object_saves_cpu import StandInFinder, _dev, _events, _saves


class FaceFinder(StandInFinder):
    """Records each encode_embed_faces_frames call; every person rect whose x1 is odd has a face, face j's embedding is
    100 + j."""
    face = True

    def __init__(self):
        super().__init__()
        self.face_calls = []

    def encode_embed_faces_frames(self, frames, pix_fmts, rects, person, quality=95):
        self.face_calls.append(np.array(person))
        files, emb = self.encode_embed_frames(frames, pix_fmts, rects, quality)
        rows = [k for k, (p, r) in enumerate(zip(person, rects)) if p and r[1] % 2]
        return files, emb, FaceSaves(rows, [b"face%d" % k for k in rows],
                                     DeviceResult(100 + torch.arange(len(rows), dtype=torch.float32)[:, None].repeat(1, 3)))


def _stepped():
    cb = _batch(TableDetector())
    cb.step(_fleet(0))
    return cb


def test_person_saves_give_faces_mapped_back_per_camera():
    cb = _stepped()
    saves = {"b0": _saves([[7, 0, 1, 2, 30, 40], [3, 2, 3, 0, 128, 72], [4, 0, 5, 0, 60, 60]]),
             "y2": _saves([[1, 1, 11, 20, 110, 120]]),
             "square": _saves([[9, 0, 4, 4, 60, 60], [2, 0, 1, 0, 9, 9], [4, 5, 63, 63, 64, 64]]),
             "b1": _saves([])}
    results = {name: _events(s) for name, s in saves.items()}
    finder = FaceFinder()
    saved, faces = cb.save_objects_and_faces(results, finder, quality=80)
    assert len(finder.calls) == 1 and len(finder.face_calls) == 1
    assert finder.calls[0][3] == 80
    assert finder.face_calls[0].tolist() == [True, False, True, False, True, True, False]     # class 0 = person ("_0.jpg")
    want = cb.save_objects(results, StandInFinder())
    assert set(saved) == set(want) == set(faces)
    for n in want:
        assert saved[n][0] is want[n][0] and saved[n][1] == want[n][1]
        assert (saved[n][2] is None) == (want[n][2] is None)
        if want[n][2] is not None:
            assert torch.equal(saved[n][2].tensor, want[n][2].tensor)
    # global face rows 0 (b0 save 0), 2 (b0 save 2), 5 (square save 1); square save 0 has an even x1: no face
    assert faces["b0"].rows == [0, 2] and faces["b0"].files == [b"face0", b"face2"]
    assert faces["b0"].embeddings.tensor[:, 0].tolist() == [100, 101]
    assert faces["y2"].rows == [] and faces["y2"].files == [] and faces["y2"].embeddings.tensor.shape[0] == 0
    assert faces["square"].rows == [1] and faces["square"].files == [b"face5"]
    assert faces["square"].embeddings.tensor[:, 0].tolist() == [102]
    assert faces["b1"] == FaceSaves([], [], None)


def test_run_rows_index_the_run_saves():
    from test_video_cpu import _HostModel, _frames
    cb = CameraBatch(_HostModel())
    cb.add_camera("v", thresh=0.3)
    res = cb.step_video({"v": _frames(3, 240, 320, 0)}, {"v": [1.7e9, 1.7e9 + 1, 1.7e9 + 2]})["v"]
    run = [res[0]._replace(saves=_saves([[1, 0, 3, 0, 20, 20]])), res[1]._replace(saves=_saves([])),
           res[2]._replace(saves=_saves([[2, 1, 5, 5, 30, 30], [3, 0, 7, 1, 40, 40], [4, 0, 2, 2, 10, 10]]))]
    finder = FaceFinder()
    saved, faces = cb.save_objects_and_faces({"v": run}, finder)
    s = saved["v"][0]
    assert s.shape == (4, 7) and s[:, 0].tolist() == [0, 2, 2, 2]
    assert finder.face_calls[0].tolist() == [True, False, True, True]
    assert faces["v"].rows == [0, 2]                           # run frame 0 save 0 and run frame 2 save 1 of the (m,7) rows
    assert faces["v"].files == [b"face0", b"face2"] and faces["v"].embeddings.tensor[:, 0].tolist() == [100, 101]
    assert saved["v"][1][0].startswith(b"0:") and saved["v"][1][2].startswith(b"2:")      # each save from its own frame


def test_no_saves_no_call_and_face_off():
    cb = _stepped()
    finder = FaceFinder()
    results = {name: _events(_saves([])) for name in ("b0", "y1")}
    saved, faces = cb.save_objects_and_faces(results, finder)
    assert finder.calls == [] and finder.face_calls == []
    assert faces == {"b0": FaceSaves([], [], None), "y1": FaceSaves([], [], None)}
    assert cb.save_objects_and_faces({}, finder) == ({}, {})

    class FaceOff(FaceFinder):
        face = False

        def encode_embed_faces_frames(self, frames, pix_fmts, rects, person, quality=95):
            return super().encode_embed_faces_frames(frames, pix_fmts, rects, person, quality)[:2] + (None,)
    off = FaceOff()
    saved, faces = cb.save_objects_and_faces({"b0": _events(_saves([[1, 0, 1, 0, 10, 10]]))}, off)
    assert faces == {"b0": None} and len(saved["b0"][1]) == 1
    assert cb.save_objects_and_faces(results, off)[1] == {"b0": None, "y1": None}


@pytest.fixture
def no_library(monkeypatch):
    from clearcam_b200.models import blazeface, objects
    calls = []

    def refuse():
        calls.append(1)
        raise AssertionError("the library was called")
    for mod in (ops, objects, blazeface):
        monkeypatch.setattr(mod, "lib", refuse)
    yield calls
    assert calls == []


def test_finder_checks_before_any_library_call(no_library):
    big = _dev((64, 96, 3))
    of = ObjectFinder()
    of.face = True                                              # a face leg without a detector
    with pytest.raises(Exception, match="detection is off"):
        of.encode_embed_faces_frames([big], "bgr24", [(0, 0, 0, 8, 8)], [True])
    of.face = False
    for rects, person, q in (([(0, 0, 0, 8, 8)], [True, False], 95),        # one flag per rect
                             ([(0, 0, 0, 97, 8)], [True], 95),               # rect outside its frame
                             ([(0, 0, 0, 8, 8)], [True], 101)):              # quality
        with pytest.raises(ValueError):
            of.encode_embed_faces_frames([big], "bgr24", rects, person, q)
    with pytest.raises(Exception, match="face embedder is off"):
        ObjectFinder().embed_face_images([b"\xff\xd8"])


def test_slot_kernels_and_first_refuse_bad_arguments():
    """Every check runs before anything is launched: the device pointers below are never dereferenced."""
    from clearcam_b200._lib import cc_face_warp, lib
    h = lib()
    fake = 1 << 20

    def refused(rc, *words):
        msg = h.cc_last_error().decode()
        assert rc == -1 and all(w in msg for w in words), (rc, msg, words)

    def canvas(idx=(0,), hw=((64, 96),), B=None, slots=fake, n=2, H=64, W=96, out=fake):
        i, s = np.ascontiguousarray(idx, np.int32), np.ascontiguousarray(hw, np.int32)
        return h.cc_face_canvas_slots(slots, n, H, W, i.ctypes.data, s.ctypes.data, len(idx) if B is None else B, out, None)

    refused(canvas(hw=((65, 96),)), "cc_face_canvas_slots", "does not fit")
    refused(canvas(hw=((64, 97),)), "does not fit")
    refused(canvas(hw=((0, 96),)), "does not fit")
    refused(canvas(idx=(2,)), "image 0 names slot 2 of 2")
    refused(canvas(idx=(-1,)), "slot -1")
    refused(canvas(B=0), "bad argument")
    refused(canvas(slots=None), "bad argument")
    refused(canvas(out=None), "bad argument")
    refused(canvas(n=0), "bad argument")
    refused(canvas(H=2000, W=2000, hw=((1, 1000),)), "resizes to nothing")
    w = (cc_face_warp * 1)()
    w[0].h, w[0].w, w[0].x1, w[0].y1, w[0].x2, w[0].y2, w[0].rot_w, w[0].rot_h = 64, 96, 0, 0, 40, 40, 50, 50

    def align(idx=(0,), K=1, slots=fake, faces=w):
        i = np.ascontiguousarray(idx, np.int32)
        return h.cc_face_align_slots(slots, 2, 64, 96, i.ctypes.data, faces, K, fake, None)
    refused(align(idx=(2,)), "cc_face_align_slots", "slot 2 of 2")
    refused(align(K=0), "bad argument")
    refused(align(slots=None), "bad argument")
    refused(align(faces=None), "faces is NULL")
    w[0].x2 = 97
    refused(align(), "face 0", "crop")
    w[0].x2, w[0].w = 40, 97
    refused(align(), "does not fit")
    refused(h.cc_blazeface_first(None, 2, fake, None), "cc_blazeface_first")
    refused(h.cc_blazeface_first(fake, 0, fake, None), "cc_blazeface_first")
    refused(h.cc_blazeface_first(fake, 2, None, None), "cc_blazeface_first")
