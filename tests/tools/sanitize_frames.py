"""Small frame-table forwards for compute-sanitizer (memcheck / racecheck): YOLOv9-c at res 256, one cc_yolo_forward_frames
call over a table of bgr24 frames of two shapes, a yuv420p frame and a padding row, all with the net shape 192 x 256 (table
letterbox, the graph-replayed middle of the plan, per-image postprocess), with the head tap, in the default and the
fp32-accurate mode; then the cc_letterbox_frames tap on the same table.
usage: compute-sanitizer --tool memcheck python tests/tools/sanitize_frames.py"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from oracle import yolov9 as o
from clearcam_b200._lib import check, lib, ptr, stream_ptr
from clearcam_b200.detection.yolov9 import YOLOv9, frame_table

fr = o.synthetic_frames(2, 192, 256, seed=11)
x = fr.flip(-1).permute(0, 3, 1, 2).float() / 255
P = o.synthetic_weights("c", seed=11, calib=x)
small = o.synthetic_frames(1, 96, 128, seed=12)[0].cuda()
yuv = torch.randint(0, 256, (288 * 3 // 2, 384), dtype=torch.uint8, generator=torch.Generator().manual_seed(1)).cuda()
table = [fr[0].cuda(), small, None, yuv, fr[1].cuda()]
fmts = ["bgr24", "bgr24", "bgr24", "yuv420p", "bgr24"]
for precise in (False, True):
    m = YOLOv9("c", 256, weights=P, precise=precise)
    for _ in range(3):                       # plain launches, then graph capture, then replay
        out, raw = m.detect_frames(table, pix_fmts=fmts, raw=True)
    torch.cuda.synchronize()
    print("frame table", "fp32-accurate" if precise else "default", int((out[..., 4] > 0).sum()))
    del m
ct, (nh, nw) = frame_table(table, fmts, 256)
lb = torch.empty(len(table), nh, nw, 3, dtype=torch.uint8, device="cuda")
oh, ow = ctypes.c_int(), ctypes.c_int()
check(lib().cc_letterbox_frames(ctypes.cast(ct, ctypes.c_void_p), len(table), 256, ptr(lb), ctypes.byref(oh), ctypes.byref(ow),
                                stream_ptr()), "cc_letterbox_frames")
torch.cuda.synchronize()
print("letterbox table", tuple(lb.shape), int(lb[2].max()))
