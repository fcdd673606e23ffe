"""What the detector, CLIP and face plans of this build are made of, as text two builds can be diffed on (CC_LIB selects the
library, as in tools/ab.py): per op its kind, name, algorithmic FLOPs and bytes; the detector trace's kind, name and FLOPs per
op; every op's conv descriptor (cc_*_op_conv: each non-pointer field, and whether each pointer is NULL) and operands
(cc_*_op_io, likewise; the lines of an older build without that tap are missing, the others unchanged); the plan facts; and
a SHA-256 of what a forward returns on seeded frames.  A host-side change to how plans are built or run must leave every
line as it was.

usage:  python tools/plan_dump.py OUT.txt
Covers the sizes bench.py runs (c at B=32 and e at B=16, 640x640; c on 1080p frames), small t / s / m plans, the default
and the fp32-accurate mode, a frame-table call over frames of two shapes, both CLIP towers (ViT-B/32, ViT-L/14), AdaFace
embeddings on synthetic weights and BlazeFace detections on the reference's weights (tests/golden/blazeface_ref.npz)."""
import ctypes
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import adaface as oa  # noqa: E402
from oracle import blazeface as obf  # noqa: E402
from oracle import clip as oc  # noqa: E402
from oracle import yolov9 as o  # noqa: E402
from clearcam_b200._lib import cc_conv_op, cc_op_io, check, lib  # noqa: E402
from clearcam_b200.detection.yolov9 import YOLOv9  # noqa: E402
from clearcam_b200.models.adaface import ADAFACE  # noqa: E402
from clearcam_b200.models.blazeface import BlazeFace  # noqa: E402
from clearcam_b200.models.objects import OpenCLIP  # noqa: E402
from clearcam_b200.utils.helpers import batch_bucket  # noqa: E402

#        size res  B   H     W     modes (False: bf16 storage, True: fp32-accurate)
CASES = [("c", 640, 32, 640, 640, (False,)), ("e", 640, 16, 640, 640, (False,)), ("c", 640, 8, 1080, 1920, (False, True)),
         ("t", 320, 16, 320, 320, (False, True)), ("s", 256, 2, 192, 256, (False, True)), ("m", 320, 16, 320, 320, (False,))]


def sha(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def fields(s):
    """A ctypes struct as text: every non-pointer field's value, and for a pointer only whether it is NULL."""
    out = []
    for name, typ in s._fields_:
        v = getattr(s, name)
        if isinstance(v, ctypes.Structure):
            out.append(f"{name}({fields(v)})")
        elif typ is ctypes.c_void_p:
            out.append(f"{name}={'NULL' if v is None else 'set'}")
        else:
            out.append(f"{name}={v.decode() if isinstance(v, bytes) else v}")
    return " ".join(out)


def op_convs(say, tag, op_conv):
    """Every op's cc_conv_op of a plan; op_conv(i, out) is the cc_*_op_conv call with the plan's arguments bound."""
    n = op_conv(0, None)
    check(min(n, 0), "op_conv")
    for i in range(n):
        d = cc_conv_op()
        check(min(op_conv(i, ctypes.byref(d)), 0), "op_conv")
        say(tag, "conv", i, fields(d))


def io_fields(d):
    """A cc_op_io as text: its scalars, then the n_in / n_out operands it reports (the unused slots left out)."""
    head = " ".join(f"{n}={getattr(d, n).decode() if n in ('kind', 'name') else getattr(d, n)}" for n, _ in d._fields_
                    if n not in ("in_", "out"))
    return " ".join([head] + [f"in{k}({fields(d.in_[k])})" for k in range(d.n_in)] + [f"out{k}({fields(d.out[k])})" for k in range(d.n_out)])


def op_ios(say, tag, op_io):
    """Every op's cc_op_io of a plan; op_io(i, out) is the cc_*_op_io call with the plan's arguments bound (nothing from a
    build without the tap)."""
    try:
        n = op_io(0, None)
    except AttributeError:
        return
    check(min(n, 0), "op_io")
    for i in range(n):
        d = cc_op_io()
        check(min(op_io(i, ctypes.byref(d)), 0), "op_io")
        say(tag, "io", i, io_fields(d))


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
            for r in m.trace(fr):
                say(tag, "trace", r["kind"], r["name"], repr(r["flops"]))
            op_convs(say, tag, lambda i, d: lib().cc_yolo_op_conv(m._h, 0, B, H, W, m.res, i, d))
            op_ios(say, tag, lambda i, d: lib().cc_yolo_op_io(m._h, 0, B, H, W, m.res, i, d))
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
            nb = B if tower == "image" else ids.shape[0]
            op_convs(say, f"clip {arch} {tower} B{nb}",
                     lambda i, d: lib().cc_clip_op_conv(cm._h, int(tower == "text"), nb, i, d))
            op_ios(say, f"clip {arch} {tower} B{nb}", lambda i, d: lib().cc_clip_op_io(cm._h, int(tower == "text"), nb, i, d))
        say("clip", arch, "outputs", sha(cm.precompute_embedding(x).tensor, cm.encode_token_ids(ids).tensor))
        del cm
    fm = ADAFACE(oa.synthetic_weights(seed=5))
    for B in (1, 3, 16, 64, 200):
        say("adaface", f"B{B}", "outputs", sha(fm.embed(oa.synthetic_faces(B, seed=B))))
        op_convs(say, f"adaface B{batch_bucket(B)}", lambda i, d: lib().cc_face_op_conv(fm._h, batch_bucket(B), i, d))
        op_ios(say, f"adaface B{batch_bucket(B)}", lambda i, d: lib().cc_face_op_io(fm._h, batch_bucket(B), i, d))
    del fm
    det = BlazeFace({k: v.numpy() for k, v in obf.load_weights(os.path.join(ROOT, "tests", "golden", "blazeface_ref.npz")).items()})
    sizes = [(256, 256), (640, 640), (480, 640), (97, 300), (333, 129), (720, 1280), (1080, 1920)]
    for B in (1, 7, 64):
        g = np.random.default_rng(B)
        ims = [g.integers(0, 256, (*sizes[i % len(sizes)], 3), dtype=np.uint8) for i in range(B)]
        say("blazeface", f"B{B}", "outputs", sha(*det.forward(ims)))
    del det
    out.close()


if __name__ == "__main__":
    main()
