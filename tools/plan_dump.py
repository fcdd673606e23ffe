"""What the detector and CLIP plans of this build are made of, as text two builds can be diffed on (CC_LIB selects the
library, as in tools/ab.py): per op its kind, name, algorithmic FLOPs and bytes; the plan facts; and a SHA-256 of what a
forward returns on seeded frames.  A host-side change to how convs are described must leave every line as it was.

usage:  python tools/plan_dump.py OUT.txt
Covers the sizes bench.py runs (c at B=32 and e at B=16, 640x640; c on 1080p frames), small t / s / m plans, the default
and the fp32-accurate mode, a frame-table call over frames of two shapes, and both CLIP towers (ViT-B/32, ViT-L/14)."""
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import clip as oc  # noqa: E402
from oracle import yolov9 as o  # noqa: E402
from clearcam_b200.detection.yolov9 import YOLOv9  # noqa: E402
from clearcam_b200.models.objects import OpenCLIP  # noqa: E402

#        size res  B   H     W     modes (False: bf16 storage, True: fp32-accurate)
CASES = [("c", 640, 32, 640, 640, (False,)), ("e", 640, 16, 640, 640, (False,)), ("c", 640, 8, 1080, 1920, (False, True)),
         ("t", 320, 16, 320, 320, (False, True)), ("s", 256, 2, 192, 256, (False, True)), ("m", 320, 16, 320, 320, (False,))]


def sha(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def main():
    out = open(sys.argv[1], "w")
    say = lambda *a: print(*a, file=out, flush=True)     # noqa: E731
    for size, res, B, H, W, modes in CASES:
        base = o.synthetic_frames(4, H, W, seed=21)
        fr = base[torch.arange(B) % 4].contiguous().cuda()
        pre = torch.stack([o.preprocess(base[i], res) for i in range(2)])
        P = o.synthetic_weights(size, seed=21, calib=pre.flip(-1).permute(0, 3, 1, 2).float() / 255)
        for precise in modes:
            m = YOLOv9(size, res, weights=P, precise=precise)
            tag = f"yolo {size} res{res} B{B} {H}x{W} {'fp32-accurate' if precise else 'bf16'}"
            say(tag, "plan", sorted(m.plan_info(B, H, W).items()))
            for r in m.profile(fr):
                say(tag, r["kind"], r["name"], repr(r["flops"]), repr(r["bytes"]))
            det, raw = m.detect_batch(fr, raw=True)
            say(tag, "outputs", sha(det, raw))
            if size == "c" and H == 1080 and not precise:       # frame-table plan: bgr24 1080p and yuv420p 720p share a net shape
                yuv = o.synthetic_frames(1, 1080, 1280, seed=5)[0, :, :, 0].contiguous().cuda()      # [720*3/2, 1280]
                frames, fmts = [fr[0], yuv, None, fr[1]], ["bgr24", "yuv420p", "bgr24", "bgr24"]
                if m.net_shape(1080, 1920) == m.net_shape(720, 1280, "yuv420p"):
                    det, raw = m.detect_frames(frames, fmts, raw=True)
                    say(tag, "frame-table outputs", sha(det, raw))
            del m
    for arch, B in (("ViT-B/32", 256), ("ViT-L/14", 64)):
        cfg = oc.CONFIGS[arch]
        cm = OpenCLIP(weights=oc.synthetic_weights(cfg, seed=3), arch=arch)
        x = oc.synthetic_images(8, cfg.image_size, seed=5)[torch.arange(B) % 8].cuda()
        g = torch.Generator().manual_seed(1)
        ids = oc.pad_tokens([torch.randint(1000, 40000, (int(n),), generator=g).tolist() for n in torch.randint(3, 20, (32,), generator=g)]).int().cuda()
        for tower, kw in (("image", {"x": x}), ("text", {"ids": ids})):
            ops, total = cm.profile(**kw)
            say("clip", arch, tower, "total flops", repr(total))
            for r in ops:
                say("clip", arch, tower, r["name"], repr(r["flops"]))
        say("clip", arch, "outputs", sha(cm.precompute_embedding(x).tensor, cm.encode_token_ids(ids).tensor))
        del cm
    out.close()


if __name__ == "__main__":
    main()
