"""Frame pixel formats, by ffmpeg's `-pix_fmt` names.

  * "bgr24"    HWC BGR uint8 [H,W,3] per frame (what clearcam.py:349-371 asks ffmpeg for); float32 frames are also bgr24
               here (test/run_mot.py:33).  The default everywhere.
  * "yuv420p"  planar YUV 4:2:0 uint8 [H*3/2,W] per frame: the Y plane (H rows), then U and V ((H/2) x (W/2) each),
               contiguous.  H and W must be even.  What a camera's H.264/HEVC decodes to, half the bytes of bgr24; the
               GPU converts it exactly as cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_I420) does.
  * "mjpeg"    a camera input format only (`CameraBatch.add_camera`, `ingest.JpegMailbox`, `ingest.VideoReader`): each
               frame is one JPEG file (`-c:v copy -f mjpeg`).  The camera's device frame is the bgr24 [H,W,3] picture
               cv2.imdecode gives for it, decoded on the GPU where it can be; the detector and the object crops see that
               bgr24 frame.

The format of a frame is always passed explicitly (`pix_fmt=`), never inferred from its shape."""
from typing import Sequence, Tuple

BGR24, YUV420P, MJPEG = "bgr24", "yuv420p", "mjpeg"
PIX_FMTS = (BGR24, YUV420P)
CAMERA_PIX_FMTS = PIX_FMTS + (MJPEG,)

# frame_fmt codes of the C-ABI (include/clearcam_b200.h)
CC_FRAME_BGR_U8, CC_FRAME_BGR_F32, CC_FRAME_I420_U8 = 0, 1, 2


def check_pix_fmt(pix_fmt) -> str:
    if pix_fmt not in PIX_FMTS:
        raise ValueError(f"pix_fmt must be one of {PIX_FMTS}, got {pix_fmt!r}")
    return pix_fmt


def check_camera_pix_fmt(pix_fmt) -> str:
    if pix_fmt not in CAMERA_PIX_FMTS:
        raise ValueError(f"pix_fmt must be one of {CAMERA_PIX_FMTS}, got {pix_fmt!r}")
    return pix_fmt


def yuv420p_rows(height: int, width: int) -> int:
    """Rows of the [H*3/2, W] buffer of one yuv420p frame of height x width pixels."""
    if height <= 0 or width <= 0 or height % 2 or width % 2:
        raise ValueError(f"a yuv420p frame needs an even height and width, got {height}x{width}")
    return height * 3 // 2


def yuv420p_size(shape: Sequence[int]) -> Tuple[int, int]:
    """(H, W) in pixels of a yuv420p buffer whose last two dimensions are [H*3/2, W]."""
    if len(shape) < 2:
        raise ValueError(f"a yuv420p frame is [H*3/2, W], got shape {tuple(shape)}")
    rows, w = int(shape[-2]), int(shape[-1])
    if rows % 3 or w % 2 or rows <= 0 or w <= 0:           # rows = 3 * (H/2): divisible by 3 exactly when H is even
        raise ValueError(f"a yuv420p frame is [H*3/2, W] with H and W even, got shape {tuple(shape)}")
    return rows * 2 // 3, w
