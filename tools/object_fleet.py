"""What saving and embedding every camera's objects in one call buys over one call per camera.

    python tools/object_fleet.py [--steps 100] [--runs 3] [--archs ViT-B/32 ViT-L/14] [--parent-lib PATH] [--out FILE]

Prints the card's name and power limit, then, for each CLIP architecture (synthetic weights) and each fleet:
  * a: 8 cameras each of 720p, 1080p, 1440p and 2160p, alternately bgr24 and yuv420p (32 cameras);
  * c: 32 x 1080p bgr24;
  * 8 x 1080p bgr24;
a seeded sequence of steps in which a seeded subset of cameras (about half) has 1 to 3 object saves of 100-600 px sides.
It first checks, over the first steps, that `CameraBatch.save_objects`'s way (one `encode_embed_frames` call) gives the
same files as the per-camera `encode_embed_crops` loop, and reports how far the embeddings are apart (bit-equal, or the
largest difference).  Then it alternates the two ways in `runs` runs of `steps` steps each and records, per step, the
device time between CUDA events around the step's calls and the wall time of the step (ending in a synchronise).

With --parent-lib (a libclearcam_b200.so built from the parent commit) it also re-times the uniform crop workloads of
tools/jpeg_crops.py and tools/jpeg_decode.py (64 crops of 150-600 px from 8 1080p frames, bgr24 and yuv420p, quality 95)
and the uniform cc_clip_preprocess of the same crops, on the parent library and on this tree's, alternated in fresh
processes, because the crop kernels changed.  One JSON line at the end."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

FLEETS = {
    "a_mixed32": [((720, 1280), "bgr24"), ((1080, 1920), "yuv420p"), ((1440, 2560), "bgr24"), ((2160, 3840), "yuv420p"),
                  ((720, 1280), "yuv420p"), ((1080, 1920), "bgr24"), ((1440, 2560), "yuv420p"), ((2160, 3840), "bgr24")] * 4,
    "c_32x1080p": [((1080, 1920), "bgr24")] * 32,
    "8x1080p": [((1080, 1920), "bgr24")] * 8,
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({ex!r})", "max_sm_clock": "unknown"}


def device_frames(fleet, seed=0):
    """Seeded frames made on the device: smooth gradients plus noise, in each camera's format."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for i, ((H, W), fmt) in enumerate(fleet):
        rows = H if fmt == "bgr24" else H * 3 // 2
        yy = torch.arange(rows, device="cuda", dtype=torch.float32)[:, None]
        xx = torch.arange(W, device="cuda", dtype=torch.float32)[None, :]
        base = (xx * 0.31 + yy * 0.17 + 23 * i) % 256
        if fmt == "bgr24":
            base = torch.stack([(base + 60 * c) % 256 for c in range(3)], -1)
        noise = torch.randn(base.shape, generator=g, device="cuda") * 6
        out.append((base + noise).clamp(0, 255).to(torch.uint8).contiguous())
    return out


def step_saves(fleet, n_steps, seed=1):
    """Per step: {camera index: int32 [k,4] rects} for a seeded subset of the cameras, 1-3 saves of 100-600 px sides."""
    rng = np.random.default_rng(seed)
    steps = []
    for _ in range(n_steps):
        cams = np.flatnonzero(rng.random(len(fleet)) < 0.5)
        s = {}
        for c in cams:
            (H, W), _ = fleet[c]
            rows = []
            for _ in range(int(rng.integers(1, 4))):
                w, h = int(rng.integers(100, min(600, W) + 1)), int(rng.integers(100, min(600, H) + 1))
                x, y = int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1))
                rows.append((x, y, x + w, y + h))
            s[int(c)] = np.array(rows, np.int32)
        steps.append(s)
    return steps


def loop_way(of, frames, fleet, saves):
    return {c: of.encode_embed_crops(frames[c][None], [(0, *r) for r in rects.tolist()], pix_fmt=fleet[c][1])
            for c, rects in saves.items()}


def table_way(of, frames, fleet, saves):
    cams = list(saves)
    if not cams:
        return {}
    rects = np.concatenate([np.concatenate([np.full((len(saves[c]), 1), j, np.int32), saves[c]], 1) for j, c in enumerate(cams)])
    files, emb = of.encode_embed_frames([frames[c] for c in cams], [fleet[c][1] for c in cams], rects)
    out, k = {}, 0
    for c in cams:
        n = len(saves[c])
        out[c] = (files[k:k + n], emb.tensor[k:k + n])
        k += n
    return out


def compare(of, frames, fleet, steps):
    """Files must be equal; embeddings: bit-equal count and the largest absolute difference."""
    equal_emb, n, worst = 0, 0, 0.0
    for s in steps:
        a, b = loop_way(of, frames, fleet, s), table_way(of, frames, fleet, s)
        assert set(a) == set(b)
        for c in a:
            fa, ea = a[c][0], a[c][1].tensor
            fb, eb = b[c]
            assert fa == fb, f"camera {c}: files differ"
            for i in range(len(fa)):
                n += 1
                equal_emb += bool(torch.equal(ea[i], eb[i]))
                worst = max(worst, float((ea[i] - eb[i]).abs().max()))
    return {"crops_checked": n, "embeddings_bit_equal": equal_emb, "max_abs_embedding_diff": worst}


def timed_run(way, of, frames, fleet, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms, wall_ms, calls = [], [], 0
    for s in steps:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        way(of, frames, fleet, s)
        e1.record()
        torch.cuda.synchronize()
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        dev_ms.append(e0.elapsed_time(e1))
        calls += len(s) if way is loop_way else int(bool(s))
    return {"device_ms_per_step": round(statistics.mean(dev_ms), 3), "wall_ms_per_step": round(statistics.mean(wall_ms), 3),
            "calls_per_step": round(calls / len(steps), 2)}


def fleet_bench(arch, steps_n, runs):
    from oracle import clip as oc
    from clearcam_b200.models.objects import ObjectFinder, OpenCLIP
    of = ObjectFinder()
    of.model = OpenCLIP(weights=oc.synthetic_weights(oc.CONFIGS[arch], seed=3), arch=arch)
    out = {}
    for name, fleet in FLEETS.items():
        frames = device_frames(fleet)
        steps = step_saves(fleet, steps_n)
        check = compare(of, frames, fleet, steps[:5])
        for s in steps[:10]:                                   # warm every batch bucket the window uses
            loop_way(of, frames, fleet, s)
            table_way(of, frames, fleet, s)
        rows = {"loop": [], "table": []}
        for _ in range(runs):
            for way, key in ((loop_way, "loop"), (table_way, "table")):
                rows[key].append(timed_run(way, of, frames, fleet, steps))
        out[name] = {"check": check, "saves_per_step": round(sum(sum(len(v) for v in s.values()) for s in steps) / len(steps), 2),
                     **rows}
        print(arch, name, json.dumps(out[name]), flush=True)
    return out


# ---- the uniform crop workloads (run in a fresh process per library)
def uniform_workloads(calls=50):
    import ctypes
    from tools.jpeg_crops import Call, crop_rects, device_ms, frames
    from tools.jpeg_decode import Chain
    from clearcam_b200._lib import lib, ptr
    import cv2
    fr = frames()
    rects = crop_rects()
    bgr = torch.from_numpy(fr).cuda()
    yuv = torch.from_numpy(np.stack([cv2.cvtColor(f, cv2.COLOR_BGR2YUV_I420) for f in fr])).cuda()
    res = {}
    for name, dev, fmt in (("bgr24", bgr, 1), ("yuv420p", yuv, 2)):
        res[f"encode_{name}_ms"] = device_ms(Call(dev, rects, 95, fmt), calls)
    res["crops_decoded_bgr24_ms"] = device_ms(Chain(bgr, rects, 95), calls)
    H, W = fr.shape[1], fr.shape[2]
    r = np.ascontiguousarray(rects, np.int32)
    out = torch.empty(len(r), 3, 224, 224, device="cuda")
    for name, dev, fmt in (("bgr24", bgr, 1), ("yuv420p", yuv, 2)):
        def pre(dev=dev, fmt=fmt):
            s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            assert lib().cc_clip_preprocess(ptr(dev), dev.shape[0], H, W, r.ctypes.data, len(r), 224, fmt, ptr(out), s) == 0
        res[f"clip_preprocess_{name}_ms"] = device_ms(pre, calls)
    return {k: round(v, 4) for k, v in res.items()}


def uniform_ab(parent_lib, reps):
    rows = {"parent": [], "this": []}
    for _ in range(reps):
        for key in ("parent", "this"):
            env = dict(os.environ)
            env.pop("CC_LIB", None)
            if key == "parent":
                env["CC_LIB"] = parent_lib
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--uniform-only"], env=env, capture_output=True,
                               text=True, cwd=ROOT)
            if p.returncode != 0:
                raise RuntimeError(p.stderr[-3000:])
            rows[key].append(json.loads(p.stdout.strip().splitlines()[-1]))
            print(key, rows[key][-1], flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--archs", nargs="+", default=["ViT-B/32", "ViT-L/14"])
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--uniform-only", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    if a.uniform_only:
        print(json.dumps(uniform_workloads()))
        return
    result = {"card": card()}
    print(json.dumps(result["card"]), flush=True)
    if a.parent_lib:
        result["uniform_crops"] = uniform_ab(a.parent_lib, a.runs)
    for arch in a.archs:
        result[arch] = fleet_bench(arch, a.steps, a.runs)
    line = json.dumps(result)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
