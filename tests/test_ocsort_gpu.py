"""The device tracker (csrc/ocsort_gpu.cu, `DeviceTrackers`) against the host tracker (csrc/ocsort.cu, `OCSort`): every
frame's nine output columns array-equal, track ids included, on every golden sequence and argument set the host tracker
is pinned to (tests/test_ocsort_cpu.py), on 128 cameras in one launch, through slot growth and through every error."""
import ctypes
import io
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from clearcam_b200._lib import CCError, cc_track_job, check, lib
from clearcam_b200.ocsort_tracker import ocsort

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).parent / "golden"
sys.path.insert(0, str(Path(__file__).parent.parent / "oracle"))


def _as_rows(tracks):
    return np.array([[*t.tlwh, t.score, t.class_id, t.track_id, t.tracklet_len, t.speed] for t in tracks], np.float64).reshape(-1, 9)


def _sequences():
    """(name, frames [F,300,6], det_thresh, OCSort kwargs, golden (rows, offsets) or None) of every pinned sequence."""
    from make_golden_ocsort import RANDOM_SEEDS, random_scene_args
    out = []
    g = np.load(GOLD / "ocsort_mot16.npz")
    out.append(("mot16", g["frames"], float(g["det_thresh"]), dict(max_age=int(g["max_age"])), (g["rows"], g["offsets"])))
    s = np.load(GOLD / "ocsort_synth.npz")
    for sc in "abc":
        a = s[f"{sc}_args"]
        out.append((f"synth_{sc}", s[f"{sc}_frames"], float(a[0]),
                    dict(max_age=int(a[1]), min_hits=int(a[2]), iou_threshold=float(a[3]), delta_t=int(a[4]), inertia=float(a[5]),
                         use_byte=bool(a[6])), (s[f"{sc}_rows"], s[f"{sc}_offsets"])))
    st = np.load(GOLD / "ocsort_street.npz")
    for v in "ab":
        a = st[f"{v}_args"]
        out.append((f"street_{v}", st["frames"], float(a[0]), dict(max_age=int(a[1]), use_byte=bool(a[2])), None))
    for seed in RANDOM_SEEDS:
        kw, thr, frames = random_scene_args(seed)
        out.append((f"random_{seed}", np.asarray(frames, np.float32), thr, kw, None))
    return out


SEQS = _sequences()


def _replay(frames, thr, kw, gold=None, capacity=64):
    dev = ocsort.DeviceTrackers(slots=4, capacity=capacity)
    dev.add("c", **kw)
    host = ocsort.OCSort(**kw)
    rows = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    for i in range(len(frames)):
        exp = _as_rows(host.update(frames[i], thr))
        [got] = dev.update([("c", rows[i], thr)])
        np.testing.assert_array_equal(_as_rows(got), exp, err_msg=f"frame {i}")
        if gold is not None:
            g = gold[0][gold[1][i]:gold[1][i + 1]]
            np.testing.assert_allclose(_as_rows(got), g, rtol=1e-5, atol=1e-9, err_msg=f"frame {i} against the golden")
    assert dev.num_tracks("c") == len(host)
    return dev


@pytest.mark.parametrize("seq", SEQS, ids=[s[0] for s in SEQS])
def test_sequence_equals_host_tracker(seq):
    name, frames, thr, kw, gold = seq
    _replay(frames, thr, kw, gold)


def test_growth_from_capacity_8():
    """A slot that starts with room for 8 tracks on a scene that reaches hundreds of live tracks."""
    g = np.load(GOLD / "ocsort_street.npz")
    frames = g["frames"][:400]
    dev = _replay(frames, 0.5, dict(max_age=100), capacity=8)
    assert dev._cap["c"] >= 100


def test_128_cameras_in_one_launch():
    """Each camera gets one sequence with its own arguments and start; some skip frames, one is reset and one is freed and
    re-added mid-run; rows come from two separate tensors in one job table.  Each equals its own host tracker."""
    B, F = 128, 90                                                     # the random scenes have 100 frames
    dev = ocsort.DeviceTrackers(slots=256, capacity=16)
    host, cams = {}, []
    for b in range(B):
        name, frames, thr, kw, _ = SEQS[b % len(SEQS)]
        start = (7 * b) % (len(frames) - F + 1)
        cams.append((b, frames[start:start + F], thr, kw))
        dev.add(b, **kw)
        host[b] = ocsort.OCSort(**kw)
    even = torch.from_numpy(np.stack([c[1] for c in cams[0::2]], 1).copy()).cuda()     # [F, 64, 300, 6]
    odd = torch.from_numpy(np.stack([c[1] for c in cams[1::2]], 1).copy()).cuda()
    for f in range(F):
        if f == 30:
            dev.reset(5)
            host[5] = ocsort.OCSort(**cams[5][3])
        if f == 40:
            dev.remove(9)
            del host[9]
        if f == 50:
            dev.add(9, **cams[9][3])
            host[9] = ocsort.OCSort(**cams[9][3])
        jobs = []
        for b, frames, thr, kw in cams:
            if b not in host or (b % 7 == 3 and f % 4 == 1):
                continue
            jobs.append((b, (even if b % 2 == 0 else odd)[f, b // 2], thr))
        got = dev.update(jobs)
        for (b, _, thr), g in zip(jobs, got):
            np.testing.assert_array_equal(_as_rows(g), _as_rows(host[b].update(cams[b][1][f], thr)), err_msg=f"camera {b} frame {f}")


def test_known_answer_156_people_tracks():
    """The reference's run_mot.py statistic on the oracle detections (tests/test_oracle_cpu.py) through DeviceTrackers."""
    g = np.load(GOLD / "mot16_oracle_dets.npz")
    dets = torch.from_numpy(g["dets"]).cuda()
    dev = ocsort.DeviceTrackers(slots=1)
    dev.add("mot", max_age=60)
    ppl = set()
    for i in range(dets.shape[0]):
        for x in dev.update([("mot", dets[i], 0.25)])[0]:
            if x.tracklet_len >= 1 and x.speed >= 2.5 and x.class_id == 0:
                ppl.add(x.track_id)
    assert len(ppl) == int(g["expected"]) == 156


def _raw_update(dev, jobs, B, cap):
    out = torch.full((B, cap, 9), -7.0, dtype=torch.float64, device="cuda")
    cs = torch.full((2, B), -9, dtype=torch.int32, device="cuda")
    table = (cc_track_job * B)(*[cc_track_job(r.data_ptr(), r.shape[0], dev._slot[c], t, 0) for c, r, t in jobs])
    check(lib().cc_ocsort_gpu_update(dev._h, table, B, out.data_ptr(), cap, cs[0].data_ptr(), cs[1].data_ptr(), None), "update")
    torch.cuda.synchronize()
    return out.cpu().numpy(), cs.cpu().numpy()


def test_errors():
    s = np.load(GOLD / "ocsort_synth.npz")
    frames = s["a_frames"]
    dev = ocsort.DeviceTrackers(slots=4)
    host = {c: ocsort.OCSort(max_age=20) for c in "abc"}
    for c in "abc":
        dev.add(c, max_age=20)
    rows = torch.from_numpy(frames).cuda()
    for f in range(20):
        got = dev.update([(c, rows[f], 0.25) for c in "abc"])
        for c, g in zip("abc", got):
            np.testing.assert_array_equal(_as_rows(g), _as_rows(host[c].update(frames[f], 0.25)))
    # class ids: out of range, non-integer, on a row above the threshold and on one in the BYTE band -> that camera's state
    # untouched, its neighbours stepped and their targets returned with the error
    for score, bad in [(0.9, 80.0), (0.9, -1.0), (0.9, 2.5), (0.9, float("nan")), (0.15, 80.0), (0.15, 2.5)]:
        r = rows[20].clone()
        r[0, 4], r[0, 5] = score, bad
        with pytest.raises(CCError, match="camera 'b'") as ei:
            dev.update([("a", rows[20], 0.25), ("b", r, 0.25)])
        assert ei.value.results[1] is None
        np.testing.assert_array_equal(_as_rows(ei.value.results[0]), _as_rows(host["a"].update(frames[20], 0.25)))
        out, cs = _raw_update(dev, [("a", rows[20], 0.25), ("b", r, 0.25)], 2, 1024)
        assert cs[1, 1] == 2 and cs[0, 1] == 0 and (out[1] == -7.0).all()
        n = cs[0, 0]
        np.testing.assert_array_equal(out[0, :n], _as_rows(host["a"].update(frames[20], 0.25)))   # ... and again here
        assert (out[0, n:] == -7.0).all()
    for f in range(21, 40):                     # b's next valid frames still match its host tracker
        [g] = dev.update([("b", rows[f], 0.25)])
        np.testing.assert_array_equal(_as_rows(g), _as_rows(host["b"].update(frames[f], 0.25)))
    # output overflow: applied, count reported, nothing written past the capacity, as the host's error
    out, cs = _raw_update(dev, [("c", rows[20], 0.25)], 1, 1)
    hout = np.empty((1, 9))
    n_host = ctypes.c_int()
    rc = lib().cc_ocsort_update(host["c"]._h, np.ascontiguousarray(frames[20]).ctypes.data, 300, 0.25, hout.ctypes.data, 1,
                                ctypes.byref(n_host))
    assert n_host.value > 1 and rc != 0                     # the frame does overflow a one-row output
    assert cs[1, 0] == 3 and cs[0, 0] == n_host.value
    np.testing.assert_array_equal(out[0, :1], hout)
    for f in range(21, 40):
        [g] = dev.update([("c", rows[f], 0.25)])
        np.testing.assert_array_equal(_as_rows(g), _as_rows(host["c"].update(frames[f], 0.25)))
    # bad slot, repeated slot, null pointers, too many rows, delta_t above the bound
    out = torch.zeros((2, 8, 9), dtype=torch.float64, device="cuda")
    cs = torch.zeros((2, 2), dtype=torch.int32, device="cuda")
    J = cc_track_job
    for table, B in [((J * 1)(J(rows[0].data_ptr(), 300, 3, 0.25, 0)), 1),          # slot 3 not configured
                     ((J * 1)(J(rows[0].data_ptr(), 300, 99, 0.25, 0)), 1),
                     ((J * 2)(J(rows[0].data_ptr(), 300, 0, 0.25, 0), J(rows[1].data_ptr(), 300, 0, 0.25, 0)), 2),
                     ((J * 1)(J(None, 300, 0, 0.25, 0)), 1),
                     ((J * 1)(J(rows[0].data_ptr(), 1025, 0, 0.25, 0)), 1)]:
        assert lib().cc_ocsort_gpu_update(dev._h, table, B, out.data_ptr(), 8, cs[0].data_ptr(), cs[1].data_ptr(), None) != 0
        assert lib().cc_last_error()
    t1 = (J * 1)(J(rows[0].data_ptr(), 300, 0, 0.25, 0))
    assert lib().cc_ocsort_gpu_update(dev._h, t1, 1, None, 8, cs[0].data_ptr(), cs[1].data_ptr(), None) != 0
    assert lib().cc_ocsort_gpu_update(dev._h, None, 1, out.data_ptr(), 8, cs[0].data_ptr(), cs[1].data_ptr(), None) != 0
    assert lib().cc_ocsort_gpu_update(None, t1, 1, out.data_ptr(), 8, cs[0].data_ptr(), cs[1].data_ptr(), None) != 0
    assert lib().cc_ocsort_gpu_configure(dev._h, 3, 30, 3, 0.3, 9, 0.2, 0, 8, None) != 0           # delta_t 9 > bound 8
    assert lib().cc_ocsort_gpu_configure(dev._h, 4, 30, 3, 0.3, 3, 0.2, 0, 8, None) != 0           # slot out of range
    assert lib().cc_ocsort_gpu_grow(dev._h, 3, 64, None) != 0                                      # slot not configured
    with pytest.raises(KeyError):
        dev.update([("zz", rows[0], 0.25)])
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ CameraBatch
RES = 320
# frames that all letterbox to 192 x 320 at res 320, in both formats: one merged detector call per step
FLEET = {"b180": ((180, 320), "bgr24"), "y180": ((180, 320), "yuv420p"), "b360": ((360, 640), "bgr24"),
         "y360": ((360, 640), "yuv420p"), "b720": ((720, 1280), "bgr24"), "y720": ((720, 1280), "yuv420p")}


def _fleet_frame(shape, fmt, seed):
    from oracle import yolov9 as o
    H, W = shape
    f = o.synthetic_frames(1, H, W, seed=seed)[0]
    if fmt == "bgr24":
        return f
    return torch.cat([f[..., 1].reshape(-1), f[::2, ::2, 0].reshape(-1), f[::2, ::2, 2].reshape(-1)]).reshape(H * 3 // 2, W)


def test_camera_batch_mailboxes_track_on_the_device_as_solo_host_trackers():
    """CameraBatch.step_mailboxes over a mixed fleet (three resolutions, bgr24 and yuv420p, one merged detector call) for
    16 steps: every camera's rows, all nine columns of its targets and its preds equal a solo OCSort(max_age=100) stepped
    on the same rows.  Frames hold still for 4 steps at a time, so tracks live past min_hits and then die.  One camera's
    tracker is reset mid-run; another camera is removed and re-added later (a fresh tracker)."""
    from oracle import yolov9 as o
    from clearcam_b200.cameras import CameraBatch
    from clearcam_b200.detection.yolov9 import YOLOv9
    from clearcam_b200.ingest import FrameMailbox
    x = o.synthetic_frames(2, 192, 320, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    m = YOLOv9("t", RES, weights=o.synthetic_weights("t", seed=5, calib=x))
    cb = CameraBatch(m, max_age=100)
    boxes = {n: FrameMailbox(H, W, pix_fmt=fmt) for n, ((H, W), fmt) in FLEET.items()}
    solo = {n: ocsort.OCSort(max_age=100) for n in FLEET}
    emitted = later = 0
    for t in range(16):
        if t == 5:
            cb.reset_tracker("b360")
            solo["b360"] = ocsort.OCSort(max_age=100)
        if t == 7:
            cb.remove_camera("y720")
            del boxes["y720"], solo["y720"]
        if t == 10:
            boxes["y720"] = FrameMailbox(720, 1280, pix_fmt="yuv420p")
            solo["y720"] = ocsort.OCSort(max_age=100)
        for i, n in enumerate(boxes):
            assert boxes[n].fill(io.BytesIO(_fleet_frame(*FLEET[n], seed=40 + i + 100 * (t // 4)).numpy().tobytes()))
        res = cb.step_mailboxes(boxes)
        assert set(res) == set(boxes) and cb._dev_trk is not None
        for n, r in res.items():
            exp = solo[n].update(r.rows, 0.5)
            np.testing.assert_array_equal(_as_rows(r.targets), _as_rows(exp), err_msg=f"step {t} camera {n}")
            keep = [x for x in exp if x.tracklet_len >= 1]
            preds = np.array([[x.tlwh[0], x.tlwh[1], x.tlwh[0] + x.tlwh[2], x.tlwh[1] + x.tlwh[3], x.score, x.class_id, x.track_id]
                              for x in keep], np.float64).reshape(-1, 7)
            np.testing.assert_array_equal(r.preds, preds, err_msg=f"step {t} camera {n}")
            emitted += len(exp)
            later += len(keep) if t % 4 == 3 else 0
    assert emitted > 0 and later > 0           # targets past min_hits, with ages and speeds, were compared
