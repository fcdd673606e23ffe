"""Frames of different shapes and formats in one detector call, on the GPU: the table-driven letterbox against cc_letterbox,
detect_frames rows bit for bit against detect_batch of uniform batches, graph replay across changing tables, CameraBatch
end to end, and the error paths."""
import ctypes
import io

import numpy as np
import pytest
import torch

from oracle import yolov9 as o
from oracle import yuv as oy
from clearcam_b200._lib import CC_MAX_FRAMES, cc_frame, lib, ptr, stream_ptr
from clearcam_b200.detection.yolov9 import YOLOv9, frame_table

pytestmark = pytest.mark.gpu

RES = 320
# frames that all letterbox to 192 x 320 at res 320: three 16:9 resolutions in both formats, and an identity frame
MIXED = [((180, 320), "bgr24"), ((360, 640), "bgr24"), ((720, 1280), "bgr24"), ((360, 640), "yuv420p"),
         ((720, 1280), "yuv420p"), ((192, 320), "bgr24")]
# reference extents 255 and 256: one net shape (256 x 320), the odd one with a zero row below it
ODD_PAIR = [((241, 320), "bgr24"), ((242, 320), "bgr24")]


def _i420(H, W, seed):
    """A structured yuv420p frame [H*3/2,W]: the planes of a synthetic BGR frame."""
    f = o.synthetic_frames(1, H, W, seed=seed)[0]
    return torch.cat([f[..., 1].reshape(-1), f[::2, ::2, 0].reshape(-1), f[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)


def _frame(shape, fmt, seed):
    H, W = shape
    return (o.synthetic_frames(1, H, W, seed=seed)[0] if fmt == "bgr24" else _i420(H, W, seed)).cuda()


def _bgr_host(f, fmt):
    return f.cpu() if fmt == "bgr24" else oy.i420_to_bgr(f.cpu())


_MODELS = {}


def _model(size, precise=False):
    if (size, precise) not in _MODELS:
        fr = o.synthetic_frames(2, 192, 320, seed=5)
        x = fr.flip(-1).permute(0, 3, 1, 2).float() / 255
        _MODELS[(size, precise)] = YOLOv9(size, RES, weights=o.synthetic_weights(size, seed=5, calib=x), precise=precise)
    return _MODELS[(size, precise)]


# ------------------------------------------------------------------------------------------------ letterbox tap
def _letterbox_frames(frames, fmts, res, rows_after=1):
    table, (nh, nw) = frame_table(frames, fmts, res)
    B = len(frames)
    buf = torch.full((B + rows_after, nh, nw, 3), 0xAB, dtype=torch.uint8, device="cuda")
    oh, ow = ctypes.c_int(), ctypes.c_int()
    rc = lib().cc_letterbox_frames(ctypes.cast(table, ctypes.c_void_p), B, res, ptr(buf), ctypes.byref(oh), ctypes.byref(ow),
                                   stream_ptr())
    assert rc == 0, lib().cc_last_error()
    assert (oh.value, ow.value) == (nh, nw)
    return buf.cpu()


def _single_letterbox(f, fmt, res, nh, nw):
    m = YOLOv9.__new__(YOLOv9)
    m.res = res
    one = m.preprocess(f, pix_fmt=fmt).tensor.cpu()
    want = torch.zeros(nh, nw, 3, dtype=torch.uint8)
    want[:one.shape[0], :one.shape[1]] = one
    return want


@pytest.mark.parametrize("res,cases", [
    (640, [((720, 1280), "bgr24"), ((1080, 1920), "bgr24"), ((1440, 2560), "bgr24"), ((2160, 3840), "bgr24"),
           ((720, 1280), "yuv420p"), ((1080, 1920), "yuv420p"), ((2160, 3840), "yuv420p"), ((384, 640), "bgr24"), None]),
    (640, [((481, 640), "bgr24"), None, ((482, 640), "bgr24")]),
])
def test_letterbox_frames_equals_cc_letterbox_per_frame(res, cases):
    frames = [None if c is None else _frame(c[0], c[1], seed=i) for i, c in enumerate(cases)]
    fmts = ["bgr24" if c is None else c[1] for c in cases]
    got = _letterbox_frames(frames, fmts, res)
    B, nh, nw = len(cases), got.shape[1], got.shape[2]
    for i, (f, fmt) in enumerate(zip(frames, fmts)):
        if f is None:
            assert int(got[i].max()) == 0, f"padding row {i} is not zero"
        else:
            assert torch.equal(got[i], _single_letterbox(f, fmt, res, nh, nw)), (i, cases[i])
    assert bool((got[B] == 0xAB).all()), "a byte after the batch was written"


# ------------------------------------------------------------------------------------------------ detector rows
def _uniform_row(m, f, fmt, B, i, raw):
    """Row i of detect_batch over B copies of frame f (f at row i): what a mixed call must reproduce for f at row i."""
    batch = torch.stack([f] * B)
    out, r = m.detect_batch(batch, raw=True, pix_fmt=fmt)
    return out[i], r[i]


@pytest.mark.parametrize("size,precise", [("t", False), ("c", False), ("t", True), ("c", True)])
def test_detect_frames_rows_equal_uniform_batches_bitwise(size, precise):
    m = _model(size, precise)
    for cases in (MIXED + [None], ODD_PAIR):
        frames = [None if c is None else _frame(c[0], c[1], seed=10 + i) for i, c in enumerate(cases)]
        fmts = ["bgr24" if c is None else c[1] for c in cases]
        out, raw = m.detect_frames(frames, pix_fmts=fmts, raw=True)
        B = len(frames)
        for i, (f, fmt) in enumerate(zip(frames, fmts)):
            if f is None:
                continue
            want, want_raw = _uniform_row(m, f, fmt, B, i, raw=True)
            assert torch.equal(out[i], want), (size, precise, cases[i])
            assert torch.equal(raw[i], want_raw), (size, precise, cases[i])
        assert int((out[..., 4] > 0).sum()) > 0


def test_graph_replay_follows_every_table():
    m = _model("c")
    frames = [_frame(c[0], c[1], seed=20 + i) for i, c in enumerate(MIXED)]
    fmts = [c[1] for c in MIXED]
    B = len(frames)
    want = [m.detect_batch(torch.stack([f] * B), pix_fmt=fmt)[0] for f, fmt in zip(frames, fmts)]
    perm = [4, 2, 0, 5, 1, 3]
    subset = [0, None, 3, None, 5, None]
    calls = [list(range(B))] * 3 + [perm, perm, subset, subset, list(range(B)), perm]
    for k, order in enumerate(calls):
        fr = [None if j is None else frames[j] for j in order]
        fm = ["bgr24" if j is None else fmts[j] for j in order]
        out = m.detect_frames(fr, pix_fmts=fm)
        for i, j in enumerate(order):
            if j is not None:
                assert torch.equal(out[i], want[j]), f"call {k}: row {i} (frame {j}) differs"


# ------------------------------------------------------------------------------------------------ CameraBatch
def _match(ref, got):
    A, Bq = ref[ref[:, 4] > 0], got[got[:, 4] > 0]
    if len(A) == 0:
        return 1.0
    if len(Bq) == 0:
        return 0.0
    d = (A[:, None, :4] - Bq[None, :, :4]).abs().max(-1)[0] + (A[:, None, 5] != Bq[None, :, 5]) * 1e6
    dc = (A[:, None, 4] - Bq[None, :, 4]).abs()
    return float(((d < 3.0) & (dc < 0.05)).any(1).float().mean())


class _Counting:
    """Counts the detector library calls a CameraBatch makes."""
    def __init__(self, m):
        self.m, self.calls = m, []

    def __getattr__(self, k):
        return getattr(self.m, k)

    def detect_batch(self, *a, **kw):
        self.calls.append("detect_batch")
        return self.m.detect_batch(*a, **kw)

    def detect_frames(self, *a, **kw):
        self.calls.append("detect_frames")
        return self.m.detect_frames(*a, **kw)


CAMS = {"b180": ((180, 320), "bgr24"), "y180": ((180, 320), "yuv420p"), "b360": ((360, 640), "bgr24"),
        "y360": ((360, 640), "yuv420p"), "b720": ((720, 1280), "bgr24"), "y720": ((720, 1280), "yuv420p")}


def _run_fleet(m, steps):
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.ingest import FrameMailbox
    det = _Counting(m)
    cb = CameraBatch(det)
    boxes = {n: FrameMailbox(H, W, pix_fmt=fmt) for n, ((H, W), fmt) in CAMS.items()}
    history = []
    for t in range(steps):
        frames = {n: _frame(s, fmt, seed=40 + 7 * t + i).cpu() for i, (n, (s, fmt)) in enumerate(CAMS.items())}
        for n, f in frames.items():
            assert boxes[n].fill(io.BytesIO(f.numpy().tobytes()))
        det.calls.clear()
        res = cb.step_mailboxes(boxes)
        assert det.calls == ["detect_frames"], det.calls
        assert set(res) == set(CAMS)
        history.append((frames, res, {n: cb.device_frame(n).clone() for n in CAMS}))
    return history


def test_camera_batch_merges_a_mixed_fleet_into_one_call():
    from clearcam_b200.models.objects import ObjectFinder
    from clearcam_b200.ocsort_tracker import ocsort
    m = _model("t")
    solo = {n: ocsort.OCSort(max_age=100) for n in CAMS}
    finder = ObjectFinder()
    n_dets = 0
    for frames, res, dev in _run_fleet(m, 3):
        for n, f in frames.items():
            fmt = CAMS[n][1]
            assert torch.equal(dev[n].cpu(), f), n
            single = m(f.numpy(), pix_fmt=fmt).numpy()
            got = res[n].rows
            assert np.array_equal(got, single) or _match(torch.from_numpy(single), torch.from_numpy(got)) >= 0.9, n
            exp = solo[n].update(got, 0.5)
            assert [int(x.track_id) for x in exp] == [int(x.track_id) for x in res[n].targets], n
            n_dets += int((got[:, 4] > 0).sum())
            H, W = CAMS[n][0]
            rects = [(0, 0, W, H), (W // 4, H // 4, W // 2 + 3, H // 2 + 5)]
            assert finder.encode_crops(dev[n], rects, pix_fmt=fmt) == finder.encode_crops(f.cuda(), rects, pix_fmt=fmt), n
    assert n_dets > 0


def test_camera_batch_mixed_fleet_meets_the_oracle_per_camera():
    """fp32-accurate mode: every camera's rows against oracle.detect of its (converted) frame at the north-star bar."""
    m = _model("t", precise=True)
    P = o.synthetic_weights("t", seed=5, calib=o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255)
    (frames, res, _), = _run_fleet(m, 1)
    n_rows = 0
    for n, f in frames.items():
        want = o.detect("t", P, _bgr_host(f, CAMS[n][1])[None], RES)[0]
        got = torch.from_numpy(res[n].rows)
        A, G = want[want[:, 4] > 0], got[got[:, 4] > 0]
        n_rows += len(A)
        if len(A) == len(G) and len(A) and bool((A[:, 5] == G[:, 5]).all()):
            assert float((A[:, :4] - G[:, :4]).abs().max()) <= 0.25 and float((A[:, 4] - G[:, 4]).abs().max()) <= 1e-3, n
        else:
            assert _match(want, got) >= 0.95 and abs(len(A) - len(G)) <= 1, (n, len(A), len(G))
    assert n_rows > 0


# ------------------------------------------------------------------------------------------------ errors
def test_bad_tables_fail_and_leave_the_output_untouched():
    m = _model("t")
    b180, b360 = _frame((180, 320), "bgr24", 1), _frame((360, 640), "bgr24", 2)
    square = _frame((320, 320), "bgr24", 3)
    f32 = torch.zeros(180, 320, 3, dtype=torch.float32, device="cuda")
    odd = torch.zeros(181 * 3 // 2, 320, dtype=torch.uint8, device="cuda")
    bad = {
        "mixed net shapes": [cc_frame(b180.data_ptr(), 0, 180, 320), cc_frame(square.data_ptr(), 0, 320, 320)],
        "float32 frame": [cc_frame(b180.data_ptr(), 0, 180, 320), cc_frame(f32.data_ptr(), 1, 180, 320)],
        "odd I420 side": [cc_frame(b360.data_ptr(), 0, 360, 640), cc_frame(odd.data_ptr(), 2, 181, 320)],
        "too many frames": [cc_frame(b180.data_ptr(), 0, 180, 320)] * (CC_MAX_FRAMES + 1),
        "only padding": [cc_frame(None, 0, 0, 0)] * 2,
    }
    for what, rows in bad.items():
        B = len(rows)
        table = (cc_frame * B)(*rows)
        out = torch.full((B, 300, 6), -7.0, device="cuda")
        rc = lib().cc_yolo_forward_frames(m._h, ctypes.cast(table, ctypes.c_void_p), B, RES, ptr(out), None, stream_ptr())
        torch.cuda.synchronize()
        assert rc != 0 and lib().cc_last_error(), what
        assert bool((out == -7.0).all()), f"{what}: d_out was written"
    for frames, fmts in [([b180, square], "bgr24"), ([b180, f32], "bgr24"), ([b180.cpu()], "bgr24"),
                         ([b360, b180[None]], "bgr24"), ([b180] * (CC_MAX_FRAMES + 1), "bgr24"), ([None, None], "bgr24"),
                         ([b180, b180], ["bgr24"]), ([b180], "nv12")]:
        with pytest.raises(ValueError):
            m.detect_frames(frames, pix_fmts=fmts)
