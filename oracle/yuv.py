"""I420 (ffmpeg yuv420p) -> BGR / RGB exactly as OpenCV's cv2.cvtColor(COLOR_YUV2BGR_I420 / COLOR_YUV2RGB_I420) computes it.

A frame is a uint8 [H*3/2, W] buffer: the Y plane H x W, then U (H/2) x (W/2), then V, contiguous; H and W even.  Each 2x2
block shares one U and one V sample (nearest chroma).  BT.601 limited range in 20-bit fixed point:

    u = U-128, v = V-128, y = max(0, Y-16) * 1220542, half = 1 << 19
    B = sat8((y + half + 2116026*u) >> 20)
    G = sat8((y + half - 852492*v - 409993*u) >> 20)
    R = sat8((y + half + 1673527*v) >> 20)

int32 holds every intermediate; >> is an arithmetic shift (floor) of the negative sums, then the clamp.  This is not
ffmpeg's swscale arithmetic: a frame piped as bgr24 can differ from the conversion here by a grey level or so.  Pinned
against cv2 in tests/test_yuv_cpu.py and tests/golden/yuv420_cv2.npz (oracle/make_golden_yuv.py)."""
import numpy as np
import torch


def _planes(yuv: torch.Tensor):
    rows, W = yuv.shape[-2], yuv.shape[-1]
    if yuv.dtype != torch.uint8 or rows % 3 or W % 2:
        raise ValueError(f"an I420 frame is uint8 [H*3/2, W] with H and W even, got {yuv.dtype} {tuple(yuv.shape)}")
    H = rows * 2 // 3
    lead = yuv.shape[:-2]
    flat = yuv.reshape(*lead, rows * W)
    n = H * W
    Y = flat[..., :n].reshape(*lead, H, W)
    U = flat[..., n:n + n // 4].reshape(*lead, H // 2, W // 2)
    V = flat[..., n + n // 4:].reshape(*lead, H // 2, W // 2)
    up = lambda c: c.repeat_interleave(2, -2).repeat_interleave(2, -1)          # noqa: E731  nearest chroma
    return Y.to(torch.int32), up(U).to(torch.int32) - 128, up(V).to(torch.int32) - 128


def i420_to_bgr(yuv):
    """[..., H*3/2, W] uint8 (numpy or torch) -> [..., H, W, 3] uint8 BGR of the same kind."""
    is_np = isinstance(yuv, np.ndarray)
    t = torch.from_numpy(np.ascontiguousarray(yuv)) if is_np else yuv.cpu().contiguous()
    Y, u, v = _planes(t)
    y = (Y - 16).clamp_min(0) * 1220542 + (1 << 19)
    b = (y + 2116026 * u) >> 20
    g = (y - 852492 * v - 409993 * u) >> 20
    r = (y + 1673527 * v) >> 20
    out = torch.stack([b, g, r], -1).clamp(0, 255).to(torch.uint8)
    return out.numpy() if is_np else out


def i420_to_rgb(yuv):
    """[..., H*3/2, W] uint8 (numpy or torch) -> [..., H, W, 3] uint8 RGB of the same kind."""
    bgr = i420_to_bgr(yuv)
    return np.ascontiguousarray(bgr[..., ::-1]) if isinstance(bgr, np.ndarray) else bgr.flip(-1)
