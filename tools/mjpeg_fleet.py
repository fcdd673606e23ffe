"""MJPEG cameras: frames decoded on the GPU by CameraBatch's decode stage, against the same JPEG frames decoded by
cv2.imdecode on host threads and stepped as bgr24 from pinned memory.

    python tools/mjpeg_fleet.py [--steps 200] [--runs 3] [--out FILE]

(b) is a proxy for the ffmpeg decode to bgr24 that MJPEG cameras otherwise need, not a measurement of ffmpeg.  Fleets:
8 x 1080p, 32 x 1080p, and 8 each of 720p / 1080p / 1440p / 2160p.  Frames are seeded synthetic content (gradients and
noise, shifted every frame; 4 distinct frames per camera, cycled), q85, 4:2:0 and 4:2:2 alternating by camera, without
Huffman tables, every second camera with a restart interval of one MCU row.  Synthetic content does not have a real
camera's entropy statistics.  Detector: YOLOv9-c at 640 with seeded synthetic weights; step_alerts with a zone and two
alerts per camera.

First checks, per fleet, that 3 steps of (a) and (b) give equal rows, preds, flags, saves, fired ids and device frames.
Then alternates (a) and (b) `runs` times, `steps` steps each, and reports frames/s; then, from one torch.profiler pass of
20 steps of (a), the device time per step of every decode kernel and of the host-to-device copies; the wall time per
step of the decode stage from the copy to the end of the status wait (and cv2 fallbacks, none here); and per frame on
the host: splitting the byte stream as read from a pipe in reads of at most 64 KB (MjpegSplitter), gathering and parsing (JpegDecoder.stage with the table inserts),
against cv2.imdecode on one thread; and bytes over PCIe per frame.  Prints the card's name and power limit first."""
import argparse
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from clearcam_b200 import ops  # noqa: E402
from clearcam_b200.alerts import Alert  # noqa: E402
from clearcam_b200.cameras import CameraBatch  # noqa: E402
from clearcam_b200.ingest import MjpegSplitter, with_default_tables  # noqa: E402

FLEETS = {"8x1080p": [(1080, 1920)] * 8, "32x1080p": [(1080, 1920)] * 32,
          "8x720p+8x1080p+8x1440p+8x2160p": [(720, 1280)] * 8 + [(1080, 1920)] * 8 + [(1440, 2560)] * 8 + [(2160, 3840)] * 8}
NF = 4


def _strip(f):
    out, pos = bytearray(f[:2]), 2
    while True:
        m, n = f[pos + 1], int.from_bytes(f[pos + 2:pos + 4], "big")
        if m != 0xC4:
            out += f[pos:pos + 2 + n]
        pos += 2 + n
        if m == 0xDA:
            return bytes(out) + f[pos:]


def camera_files(i, H, W):
    rng = np.random.default_rng(100 + i)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    base = np.clip(np.stack([(xx * (0.5 + 0.2 * c) + yy * (0.3 + 0.1 * c) + 50 * c + 20 * i) % 256 for c in range(3)], -1)
                   + rng.normal(0, 6, (H, W, 3)), 0, 255).astype(np.uint8)
    samp = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420 if i % 2 == 0 else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422
    p = [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp]
    p += [cv2.IMWRITE_JPEG_RST_INTERVAL, (W + 15) // 16] if i % 4 >= 2 else []
    return [_strip(cv2.imencode(".jpg", np.ascontiguousarray(np.roll(base, (9 * f, 13 * f), (0, 1))), p)[1].tobytes())
            for f in range(NF)]


def pinned(b):
    t = torch.empty(len(b), dtype=torch.uint8, pin_memory=True)
    t.numpy()[:] = np.frombuffer(b, np.uint8)
    return t


def make_batch(model, names, fmt):
    cb = CameraBatch(model)
    for n in names:
        cb.add_camera(n, thresh=0.25, pix_fmt=fmt)
        cb.set_zone(n, [[0.0, 0.0], [0.7, 0.0], [0.7, 1.0], [0.0, 1.0]], False, True)
        cb.set_alerts(n, {"d": Alert.make(max=1, classes=[0, 2]), "z": Alert.make(max=2, window=3, zone=False)})
    return cb


class Pipe(io.RawIOBase):
    """A byte stream read as from an ffmpeg pipe: at most 64 KB per read (the Linux pipe buffer)."""

    def __init__(self, data):
        self.b = io.BytesIO(data)

    def readable(self):
        return True

    def readinto(self, buf):
        d = self.b.read(min(len(buf), 1 << 16))
        buf[:len(d)] = d
        return len(d)


class HostDecode:
    """(b): cv2.imdecode on host threads into pinned bgr24 buffers."""

    def __init__(self, names, shapes):
        self.bufs = {n: torch.empty((H, W, 3), dtype=torch.uint8, pin_memory=True) for n, (H, W) in zip(names, shapes)}
        self.pool = ThreadPoolExecutor(os.cpu_count() or 4)

    def __call__(self, files):
        def one(item):
            n, f = item
            np.copyto(self.bufs[n].numpy(), cv2.imdecode(f.numpy(), cv2.IMREAD_COLOR))
        list(self.pool.map(one, files.items()))
        return self.bufs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    cv2.setNumThreads(1)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(card, flush=True)
    from oracle import yolov9 as o
    from clearcam_b200.detection.yolov9 import YOLOv9
    xc = o.synthetic_frames(2, 384, 640, seed=5).flip(-1).permute(0, 3, 1, 2).float() / 255
    model = YOLOv9("c", 640, weights=o.synthetic_weights("c", seed=5, calib=xc))
    report = {"card": card, "steps": a.steps, "runs": a.runs, "fleets": {}}
    for fleet, shapes in FLEETS.items():
        names = [f"cam{i}" for i in range(len(shapes))]
        files = {n: [pinned(f) for f in camera_files(i, H, W)] for i, (n, (H, W)) in enumerate(zip(names, shapes))}
        dev_b, host_b = make_batch(model, names, "mjpeg"), make_batch(model, names, "bgr24")
        host = HostDecode(names, shapes)
        T0 = 1.7e9

        def step_a(t):
            return dev_b.step_alerts({n: files[n][t % NF] for n in names}, now=T0 + t)

        def step_b(t):
            return host_b.step_alerts(host({n: files[n][t % NF] for n in names}), now=T0 + t)

        for t in range(3):                                  # equal outputs first
            ra, rb = step_a(t), step_b(t)
            assert sorted(ra) == sorted(rb)
            for n in names:
                for u, v in zip(ra[n][:4], rb[n][:4]):
                    assert np.array_equal(u, v), (fleet, n, t)
                assert ra[n].fired == rb[n].fired
                assert torch.equal(dev_b.device_frame(n), host_b.device_frame(n)), (fleet, n)
        stage_s = []
        dec = CameraBatch._decode_jpeg

        def timed(self, *args):
            t0 = time.perf_counter()
            r = dec(self, *args)
            stage_s.append(time.perf_counter() - t0)
            return r
        CameraBatch._decode_jpeg = timed
        rates = {"a_device_decode": [], "b_host_cv2": []}
        t = 3
        for _ in range(a.runs):
            for key, fn in (("a_device_decode", step_a), ("b_host_cv2", step_b)):
                for _ in range(10):
                    fn(t)
                    t += 1
                stage_s.clear()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    fn(t)
                    t += 1
                dt = time.perf_counter() - t0
                rates[key].append(round(len(names) * a.steps / dt, 1))
                if key == "a_device_decode":
                    stage = sorted(stage_s)
        CameraBatch._decode_jpeg = dec
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                step_a(t)
                t += 1
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type.name != "CUDA":
                continue
            if "jdec_" in e.name:
                name = e.name.split("jdec_")[1].split("(")[0].split("ENS")[0]
            elif "Memcpy HtoD" in e.name:
                name = "memcpy HtoD (all cameras' uploads)"
            else:
                continue
            kern[name] = kern.get(name, 0.0) + e.device_time_total / 20
        # host costs per frame
        stream = b"".join(bytes(files[n][f].numpy()) for f in range(NF) for n in names)
        sp, buf, s = MjpegSplitter(), np.empty(max(H * W * 3 for H, W in shapes), np.uint8), Pipe(stream)
        t0 = time.perf_counter()
        nsplit = 0
        while sp.read(s, buf):
            nsplit += 1
        split_us = (time.perf_counter() - t0) / nsplit * 1e6
        jd = ops.JpegDecoder()
        from clearcam_b200.ingest import default_tables
        step_files = [files[n][0].numpy() for n in names]
        t0 = time.perf_counter()
        for _ in range(10):
            ins = [default_tables(f) for f in step_files]
            jd.stage(step_files, [i if i[1] else None for i in ins])
        gather_us = (time.perf_counter() - t0) / (10 * len(names)) * 1e6
        t0 = time.perf_counter()
        for f in step_files:
            cv2.imdecode(f, cv2.IMREAD_COLOR)
        imdecode_us = (time.perf_counter() - t0) / len(names) * 1e6
        jpeg_bytes = float(np.mean([len(with_default_tables(bytes(f.numpy()))) for n in names for f in files[n]]))
        raw_bytes = float(np.mean([H * W * 3 for H, W in shapes]))
        r = {"cameras": len(names), "frames_per_s": rates,
             "decode_kernels_us_per_step": {k: round(v, 1) for k, v in sorted(kern.items())},
             "decode_stage_ms_per_step (queue, status wait, fallbacks)": {"p50": round(stage[len(stage) // 2] * 1e3, 3),
                                                                          "p90": round(stage[len(stage) * 9 // 10] * 1e3, 3)},
             "host_us_per_frame": {"split": round(split_us, 1), "gather+tables+parse": round(gather_us, 1),
                                   "cv2.imdecode 1 thread": round(imdecode_us, 1)},
             "pcie_bytes_per_frame": {"mjpeg": round(jpeg_bytes), "bgr24": round(raw_bytes)}}
        report["fleets"][fleet] = r
        print(json.dumps({fleet: r}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
