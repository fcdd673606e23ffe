"""Thin Python wrappers over the kernel-level C-ABI ops (used by the parity tests and the graphs)."""
import ctypes

import torch

from ._lib import CC_CONV_OP_CHAIN, CC_CONV_OP_DIRECT, CC_CONV_OP_GEMM, cc_conv_op, cc_slice, lib, check, ptr, stream_ptr


def conv2d(xbuf, in_co, Cin, w, bias, k, stride, obuf, out_co, Cout, act=0, res=None, res_co=0, groups=1, impl=1, bn=0,
           stream=None, slope=None, pre=None, out_ns=0):
    """xbuf: [N,H,W,in_cs] bf16 CUDA; w: [Cout,k,k,Cin/groups] bf16; obuf: [N,Ho,Wo,out_cs] bf16|fp32.  impl 1 = the wgmma
    kernel, 2 = the direct kernel.  act = 3 (CC_ACT_PRELU): bias is the fp32 [9,Cout] border-class table and slope the fp32
    [Cout] PReLU slopes, bf16 out.  pre: the fp32 [N,Ho/2,Wo/2,Cout] addend before the activation.  out_ns: pixels per image
    in obuf's and res's buffers (0 = dense); obuf and res are then [N,Ho,Wo,cs] views with an image stride of out_ns * cs
    elements, e.g. x.view(N, L, cs)[:, 1:].unsqueeze(1) for tokens 1.. of an L-token stream."""
    assert impl in (1, 2), "impl 1 = wgmma, 2 = direct"
    assert pre is None or (pre.dtype == torch.float32 and pre.is_contiguous() and pre.dim() == 4)
    return _conv(CC_CONV_OP_GEMM if impl == 1 else CC_CONV_OP_DIRECT, xbuf, in_co, Cin, w, bias, k, stride, obuf, out_co, Cout,
                 act, res, res_co, stream, groups=groups, BN=bn, slope=ptr(slope), pre=ptr(pre),
                 pre_h=0 if pre is None else pre.shape[1], pre_w=0 if pre is None else pre.shape[2], out_ns=out_ns)


def conv2d_chain(xbuf, in_co, Cin, w, bias, k, stride, obuf, out_co, w2, bias2, k0, o2buf, out2_co, act2=1, part=None,
                 part_co=0, part_C=0, res=None, res_co=0, store1=True, stream=None):
    """A SiLU conv of w (bf16 [Cout,k,k,Cin]) into obuf[..., out_co:] and, in its epilogue, the square 1x1 conv w2 (bf16
    [Cout2,1,1,Cout2]) over [its output channels k0.. | part[..., part_co:part_co + part_C]] into o2buf[..., out2_co:] (bf16 with
    act2 = 1 SiLU, or fp32 with act2 = 0).  store1=False drops the first output (obuf may be None)."""
    assert w2.is_contiguous()
    _conv(CC_CONV_OP_CHAIN, xbuf, in_co, Cin, w, bias, k, stride, obuf, out_co, w.shape[0], 1, res, res_co, stream, w2=ptr(w2),
          bias2=ptr(bias2), act2=act2, k0=k0, part=_slice(part, part_co, part_C), out2=_slice(o2buf, out2_co, w2.shape[0]),
          store1=int(store1))
    return o2buf


def _slice(t, co, C):
    """Channels [co, co + C) of the NHWC tensor t as a cc_slice (t None: no buffer)."""
    if t is None:
        return cc_slice(None, 0, co, C)
    N, H, W, cs = t.shape
    return cc_slice(t.data_ptr(), cs, co, C, N, H, W, int(t.dtype == torch.float32))


def _dense_or_pitched(t, ns):
    """t is contiguous, or (ns > 0) a [N,H,W,cs] view whose images are ns pixels apart and dense within."""
    if t is None or ns == 0:
        return t is None or t.is_contiguous()
    N, H, W, cs = t.shape
    return t.stride()[1:] == (W * cs, cs, 1) and (N == 1 or t.stride(0) == ns * cs)


def _conv(kind, xbuf, in_co, Cin, w, bias, k, stride, obuf, out_co, Cout, act, res, res_co, stream, **fields):
    """One cc_conv launch of the given kind; `fields` sets the rest of the cc_conv_op."""
    assert xbuf.is_cuda and xbuf.dtype == torch.bfloat16 and xbuf.is_contiguous()
    ns = fields.get("out_ns", 0)
    assert w.dtype == torch.bfloat16 and w.is_contiguous() and _dense_or_pitched(obuf, ns) and (ns == 0 or _dense_or_pitched(res, ns))
    op = cc_conv_op(kind=kind, in_=_slice(xbuf, in_co, Cin), out=_slice(obuf, out_co, Cout), res=_slice(res, res_co, Cout),
                    w=ptr(w), bias=ptr(bias), k=k, stride=stride, act=act, **{"groups": 1, **fields})
    check(lib().cc_conv(ctypes.byref(op), stream_ptr(stream)), "cc_conv")
    return obuf


def attention(qkv, L, H, causal, impl, ctx=None, stream=None):
    """qkv: [B*L, 3*H*64] bf16 CUDA (Q | K | V rows of B sequences of L tokens) -> ctx [B*L, H*64] bf16, the attention of
    each (sequence, head).  impl: 1 = mma.sync kernel, 2 = wgmma kernel.  ctx may have more rows than B*L; only the first
    B*L are written."""
    assert qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape[-1] == 3 * H * 64
    assert qkv.shape[0] % L == 0
    B = qkv.shape[0] // L
    need = ctypes.c_size_t(0)
    check(lib().cc_attention(ptr(qkv), B, L, H, causal, impl, None, 0, None, ctypes.byref(need), None), "cc_attention")
    ws = torch.empty(need.value, dtype=torch.uint8, device=qkv.device) if need.value else None
    if ctx is None:
        ctx = torch.empty(B * L, H * 64, dtype=torch.bfloat16, device=qkv.device)
    assert ctx.dtype == torch.bfloat16 and ctx.is_contiguous() and ctx.shape[0] >= B * L and ctx.shape[-1] == H * 64
    check(lib().cc_attention(ptr(qkv), B, L, H, causal, impl, ptr(ws), need.value, ptr(ctx), None, stream_ptr(stream)),
          "cc_attention")
    return ctx


# ---- the detector's non-GEMM kernels and its fp32-accurate conv, as the plan runs them (include/clearcam_b200.h)
POOL_OPS = {"avg2_pad": 0, "avgmax": 1, "max5": 2, "upsample2": 3}


def _nhwc(t):
    assert t.is_cuda and t.dtype in (torch.bfloat16, torch.float32) and t.is_contiguous() and t.dim() == 4
    return t.shape


def pool(op, xbuf, in_co, C, obuf, out_co, stream=None):
    """op in POOL_OPS on channels [in_co, in_co + C) of xbuf [N,H,W,in_cs] into [out_co, out_co + C) of obuf
    [N,Ho,Wo,out_cs]; both bf16 or both fp32."""
    N, H, W, in_cs = _nhwc(xbuf)
    _nhwc(obuf)
    assert obuf.dtype == xbuf.dtype
    check(lib().cc_pool(POOL_OPS[op], int(xbuf.dtype == torch.float32), ptr(xbuf), N, H, W, in_cs, in_co, C, ptr(obuf),
                        obuf.shape[-1], out_co, stream_ptr(stream)), "cc_pool")
    return obuf


def spp3(cat, co, c1, stream=None):
    """The three cascaded 5x5 max pools of SPPELAN in place in the bf16 concat buffer cat [N,H,W,cs]."""
    N, H, W, cs = _nhwc(cat)
    check(lib().cc_spp3(ptr(cat), N, H, W, cs, co, c1, stream_ptr(stream)), "cc_spp3")
    return cat


def cbfuse(srcs, last, out, C, stream=None):
    """srcs: list of (buf [N,h,w,cs], co); last, out: (buf [N,H,W,cs], co).  out = sum of nearest-resized sources + last."""
    n = len(srcs)
    bufs = [s for s, _ in srcs]
    for b in bufs + [last[0], out[0]]:
        _nhwc(b)
    N, H, W, _ = out[0].shape
    arr = lambda vals, t=ctypes.c_int: (t * max(n, 1))(*vals)
    check(lib().cc_cbfuse(int(out[0].dtype == torch.float32), n, arr([b.data_ptr() for b in bufs], ctypes.c_void_p),
                          arr([b.shape[1] for b in bufs]), arr([b.shape[2] for b in bufs]), arr([b.shape[3] for b in bufs]),
                          arr([co for _, co in srcs]), ptr(last[0]), last[0].shape[-1], last[1], ptr(out[0]), out[0].shape[-1],
                          out[1], N, H, W, C, stream_ptr(stream)), "cc_cbfuse")
    return out[0]


def split_planes(x, co, C, stream=None):
    """x: fp32 [npix, cs] CUDA -> bf16 [npix, 6C] planes lo | mid | hi | mid | hi | hi of channels [co, co + C)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
    out = torch.empty(x.shape[0], 6 * C, dtype=torch.bfloat16, device=x.device)
    check(lib().cc_split_planes(ptr(x), x.shape[0], x.shape[1], co, C, ptr(out), stream_ptr(stream)), "cc_split_planes")
    return out


def finish_f32(acc, bias, act, out, out_co, res=None, res_co=0, stream=None):
    """out[:, out_co:out_co+C] = [res[:, res_co:res_co+C] +] act(acc + bias); acc fp32 [npix, C], out / res fp32 [npix, cs]."""
    npix, C = acc.shape
    check(lib().cc_finish_f32(ptr(acc), ptr(bias), act, npix, C, ptr(out), out.shape[-1], out_co, ptr(res),
                              0 if res is None else res.shape[-1], res_co, stream_ptr(stream)), "cc_finish_f32")
    return out


def stem(frames, w, b, obuf, out_co, impl, stream=None):
    """frames: [B,H,W,3] BGR uint8 | float32 CUDA; w: fp32 [Cout,3,3,3] and b: fp32 [Cout] on the host (PyTorch layout);
    obuf: [B,H/2,W/2,cs] bf16 | fp32.  impl 1 = stem_tc, 2 = stem_kernel."""
    B, H, W, _ = frames.shape
    assert frames.is_cuda and frames.is_contiguous() and frames.dtype in (torch.uint8, torch.float32)
    w, b = w.detach().float().contiguous().cpu(), b.detach().float().contiguous().cpu()
    Cout = w.shape[0]
    args = (ptr(frames), int(frames.dtype == torch.float32), B, H, W, ptr(w), ptr(b), Cout)
    need = ctypes.c_size_t(0)
    check(lib().cc_stem(*args, None, obuf.shape[-1], out_co, int(obuf.dtype == torch.float32), impl, None, 0,
                        ctypes.byref(need), None), "cc_stem")
    ws = torch.empty(need.value, dtype=torch.uint8, device=frames.device)
    check(lib().cc_stem(*args, ptr(obuf), obuf.shape[-1], out_co, int(obuf.dtype == torch.float32), impl, ptr(ws), need.value,
                        None, stream_ptr(stream)), "cc_stem")
    return obuf


def conv2d_fp32_accurate(xbuf, in_co, Cin, w, bias, stride, act, obuf, out_co, res=None, res_co=0, stream=None):
    """One conv of the detector's fp32-accurate mode.  xbuf / obuf / res: fp32 NHWC CUDA; w: fp32 [Cout,Cin,k,k] and bias
    fp32 [Cout] (or None) on the host, split into bf16 planes exactly as the detector splits its weights."""
    N, H, W, in_cs = _nhwc(xbuf)
    w = w.detach().float().contiguous().cpu()
    bias = None if bias is None else bias.detach().float().contiguous().cpu()
    Cout, k = w.shape[0], w.shape[-1]
    args = (ptr(xbuf), N, H, W, in_cs, in_co, Cin, ptr(w), ptr(bias), Cout, k, stride, act, ptr(res),
            0 if res is None else res.shape[-1], res_co)
    need = ctypes.c_size_t(0)
    check(lib().cc_conv2d_fp32_accurate(*args, None, obuf.shape[-1], out_co, None, 0, ctypes.byref(need), None),
          "cc_conv2d_fp32_accurate")
    ws = torch.empty(need.value, dtype=torch.uint8, device=xbuf.device)
    check(lib().cc_conv2d_fp32_accurate(*args, ptr(obuf), obuf.shape[-1], out_co, ptr(ws), need.value, None,
                                        stream_ptr(stream)), "cc_conv2d_fp32_accurate")
    return obuf


# ---- the CLIP encoders' row kernels, as the plans run them (include/clearcam_b200.h)
def _f32_cuda(*ts):
    for t in ts:
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()


def patchify(x, p, kpad, out=None, stream=None):
    """x: fp32 [B,3,S,S] CUDA -> bf16 [B*(S/p)^2, kpad] patch matrix (zeros past 3p^2)."""
    _f32_cuda(x)
    B, _, S, _ = x.shape
    if out is None:
        out = torch.empty(B * (S // p) ** 2, kpad, dtype=torch.bfloat16, device=x.device)
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape[-1] == kpad
    check(lib().cc_patchify(ptr(x), B, S, p, kpad, ptr(out), stream_ptr(stream)), "cc_patchify")
    return out


def clip_embed_ln(x, cls, pos, gamma, beta, L, stream=None):
    """In place on x fp32 [B*L, W]: token 0 := cls, + pos[t], then ln_pre with gamma / beta."""
    _f32_cuda(x, cls, pos, gamma, beta)
    W = x.shape[-1]
    assert x.shape[0] % L == 0 and pos.numel() == L * W
    check(lib().cc_clip_embed_ln(ptr(x), ptr(cls), ptr(pos), ptr(gamma), ptr(beta), x.shape[0] // L, L, W, stream_ptr(stream)),
          "cc_clip_embed_ln")
    return x


def layernorm_bf16(x, gamma, beta, rows=None, row_stride=1, row_idx=None, out=None, stream=None):
    """x fp32 [n, W] -> bf16 [rows, W]: LayerNorm of rows r * row_stride, or of rows row_idx[r] (int32 CUDA) when given."""
    _f32_cuda(x, gamma, beta)
    W = x.shape[-1]
    if rows is None:
        rows = row_idx.numel() if row_idx is not None else (x.shape[0] + row_stride - 1) // max(row_stride, 1)
    if row_idx is not None:
        assert row_idx.is_cuda and row_idx.dtype == torch.int32 and row_idx.numel() >= rows
    if out is None:
        out = torch.empty(rows, W, dtype=torch.bfloat16, device=x.device)
    assert out.dtype == torch.bfloat16 and out.is_contiguous()
    check(lib().cc_layernorm_bf16(ptr(x), rows, W, row_stride, ptr(row_idx), ptr(gamma), ptr(beta), ptr(out), stream_ptr(stream)),
          "cc_layernorm_bf16")
    return out


def text_embed(ids, tok, pos, x=None, eot_row=None, stream=None):
    """ids int32 [B, L] CUDA -> (x fp32 [B*L, W] = tok[clamp(id)] + pos[t], eot_row int32 [B] = b*L + first argmax of ids)."""
    assert ids.is_cuda and ids.dtype == torch.int32 and ids.is_contiguous()
    _f32_cuda(tok, pos)
    B, L = ids.shape
    vocab, W = tok.shape
    if x is None:
        x = torch.empty(B * L, W, device=ids.device)
    if eot_row is None:
        eot_row = torch.empty(B, dtype=torch.int32, device=ids.device)
    _f32_cuda(x)
    check(lib().cc_text_embed(ptr(ids), ptr(tok), ptr(pos), B, L, W, vocab, ptr(x), ptr(eot_row), stream_ptr(stream)),
          "cc_text_embed")
    return x, eot_row


def l2norm(x, eps, out=None, out_stride=None, stream=None):
    """x fp32 [rows, D] -> out rows r * out_stride .. + D: x / (||x|| + eps)."""
    _f32_cuda(x)
    rows, D = x.shape
    if out is None:
        out = torch.empty(rows, D, device=x.device)
    out_stride = out.stride(0) if out_stride is None else out_stride
    check(lib().cc_l2norm(ptr(x), rows, D, eps, ptr(out), out_stride, stream_ptr(stream)), "cc_l2norm")
    return out


# ---- frame tables: device frames of different shapes and formats in one call
def frame_table(frames, pix_fmts, padding=False):
    """Validate a list of device frames with per-frame formats -> (ctypes cc_frame array, [(H, W) or None per frame]).
    frames: contiguous uint8 CUDA tensors, [H,W,3] for "bgr24" or [H*3/2,W] for "yuv420p" (H, W even); with `padding`, None
    is a padding row.  pix_fmts: one format for all, or one per frame.  Raises ValueError; calls nothing in the library."""
    from ._lib import cc_frame
    from .pixfmt import BGR24, CC_FRAME_BGR_U8, CC_FRAME_I420_U8, check_pix_fmt, yuv420p_size
    frames = list(frames)
    B = len(frames)
    fmts = [pix_fmts] * B if isinstance(pix_fmts, str) else list(pix_fmts)
    if len(fmts) != B:
        raise ValueError(f"{B} frames but {len(fmts)} pixel formats")
    table = (cc_frame * B)()
    sizes = []
    for i, (f, fmt) in enumerate(zip(frames, fmts)):
        check_pix_fmt(fmt)
        if f is None and padding:
            sizes.append(None)
            continue
        if not isinstance(f, torch.Tensor) or not f.is_cuda or f.dtype != torch.uint8 or not f.is_contiguous():
            raise ValueError(f"frame {i}: expected a contiguous uint8 CUDA tensor, got "
                             f"{type(f).__name__} {getattr(f, 'dtype', '')} {tuple(getattr(f, 'shape', ()))}")
        if fmt == BGR24:
            if f.dim() != 3 or f.shape[2] != 3:
                raise ValueError(f"frame {i}: a bgr24 frame is [H,W,3], got {tuple(f.shape)}")
            H, W = int(f.shape[0]), int(f.shape[1])
        else:
            if f.dim() != 2:
                raise ValueError(f"frame {i}: a yuv420p frame is [H*3/2,W], got {tuple(f.shape)}")
            H, W = yuv420p_size(f.shape)
        sizes.append((H, W))
        table[i] = cc_frame(f.data_ptr(), CC_FRAME_BGR_U8 if fmt == BGR24 else CC_FRAME_I420_U8, H, W)
    return table, sizes


# the numpy layout of one cc_frame row (include/clearcam_b200.h): pointer, format, height, width
_FRAME_ROW = {"names": ["data", "fmt", "h", "w"], "formats": ["<u8", "<i4", "<i4", "<i4"], "offsets": [0, 8, 12, 16],
              "itemsize": 24}
# ... and of one cc_jpeg_dest: pointer, row pitch, height, width
_DEST_ROW = {"names": ["data", "pitch", "h", "w"], "formats": ["<u8", "<i8", "<i4", "<i4"], "offsets": [0, 8, 16, 20],
             "itemsize": 24}


def batch_table(frames, fmt):
    """The frame table of a contiguous uint8 CUDA batch of n frames of one format (a CC_FRAME_* code): [n,H,W,3] for
    CC_FRAME_BGR_U8 / CC_FRAME_RGB_U8, [n,H*3/2,W] for CC_FRAME_I420_U8 -> ctypes cc_frame [n], row i at the batch's
    pointer + i frames.  The library checks the rows (and the rects against them) when a call reads the table."""
    import numpy as np
    from ._lib import cc_frame
    from .pixfmt import CC_FRAME_I420_U8
    assert frames.is_cuda and frames.dtype == torch.uint8 and frames.is_contiguous()
    n, rows, W = frames.shape[:3]
    t = np.zeros(n, _FRAME_ROW)                         # filled as one array: a fraction of the cost of n ctypes rows
    t["data"] = frames.data_ptr() + frames.stride(0) * np.arange(n, dtype=np.uint64)
    t["fmt"], t["h"], t["w"] = fmt, rows * 2 // 3 if fmt == CC_FRAME_I420_U8 else rows, W
    return (cc_frame * n).from_buffer(t)


def _rects_i32(rects):
    import numpy as np
    return np.ascontiguousarray(np.asarray(rects, np.int32).reshape(-1, 5))


def table_rects(rects, sizes):
    """rects: K rows (frame, x1, y1, x2, y2) against a frame table's sizes -> contiguous int32 [K,5]; ValueError for a
    frame index outside the table or a rect that is empty or leaves its own frame."""
    import numpy as np
    r = _rects_i32(rects)
    for k, (f, x1, y1, x2, y2) in enumerate(r.tolist()):
        if not 0 <= f < len(sizes) or sizes[f] is None:
            raise ValueError(f"rect {k} names frame {f} of a {len(sizes)}-frame table")
        H, W = sizes[f]
        if not (0 <= x1 < x2 <= W and 0 <= y1 < y2 <= H):
            raise ValueError(f"rect {k} ({x1},{y1}-{x2},{y2}) is empty or outside its frame {f} ({W}x{H})")
    return np.ascontiguousarray(r)


# ---- JPEG of frame crops (object thumbnails), byte-identical to cv2.imwrite.  table: a frame_table or batch_table;
# rects: K rows (frame index into the table, x1, y1, x2, y2)
def jpeg_bound(w, h):
    """Worst-case bytes of one encoded w x h crop."""
    b = ctypes.c_int64(0)
    check(lib().cc_jpeg_bound(int(w), int(h), ctypes.byref(b)), "cc_jpeg_bound")
    return b.value


def jpeg_encode_crops_frames(table, rects, quality=95, stream=None):
    """Queue the encoding of K crops -> (out, device lengths, offsets); nothing waits.  The crops go into one device
    buffer at offsets given by the prefix sum of their bounds; `jpeg_collect` brings the files back, file k being the one
    cv2.imwrite writes for crop k at `quality`."""
    import numpy as np
    r = _rects_i32(rects)
    K = len(r)
    args = (table, len(table), r.ctypes.data, K, int(quality))
    bounds = np.array([jpeg_bound(x2 - x1, y2 - y1) if x2 > x1 and y2 > y1 else 0 for _, x1, y1, x2, y2 in r], np.int64)
    offsets = np.ascontiguousarray(np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.int64))
    need = ctypes.c_size_t(0)
    check(lib().cc_jpeg_encode_crops_frames(*args, None, 0, None, None, None, 0, ctypes.byref(need), None),
          "cc_jpeg_encode_crops_frames")
    out = torch.empty(int(bounds.sum()), dtype=torch.uint8, device="cuda")
    lengths = torch.empty(K, dtype=torch.int64, device="cuda")
    ws = torch.empty(max(need.value, 1), dtype=torch.uint8, device="cuda")
    check(lib().cc_jpeg_encode_crops_frames(*args, ptr(out), out.numel(), offsets.ctypes.data, ptr(lengths), ptr(ws), need.value,
                                            None, stream_ptr(stream)), "cc_jpeg_encode_crops_frames")
    return out, lengths, offsets


def jpeg_collect(out, lengths, offsets, lens=None):
    """The files of `jpeg_encode_crops_frames`' (out, lengths, offsets) as a list of K `bytes`: the used bytes of every crop
    gathered into one device run, one copy to the host.  lens: the lengths already on the host, or None to fetch them
    (a second host wait)."""
    lens = lengths.cpu().numpy() if lens is None else lens
    return jpeg_split(jpeg_gather(out, lengths, offsets, lens).cpu().numpy(), lens)


def jpeg_gather(out, lengths, offsets, lens):
    """Queue the gather of the used bytes of every crop (lens: the lengths on the host) into one device run; nothing
    waits.  `jpeg_split` cuts its host copy into the files."""
    dev = out.device
    total = int(lens.sum())
    starts = torch.cumsum(lengths, 0) - lengths
    idx = torch.arange(total, device=dev) + torch.repeat_interleave(torch.from_numpy(offsets).to(dev) - starts, lengths,
                                                                     output_size=total)
    return out[idx]


def jpeg_split(flat, lens):
    """The host copy of a `jpeg_gather` run (uint8 numpy) -> the list of files."""
    import numpy as np
    flat = flat.tobytes()
    ends = np.cumsum(lens)
    return [flat[e - l:e] for e, l in zip(ends, lens)]


def read_together(*tensors):
    """Device tensors -> numpy copies of each, through one device-to-host copy (one host wait)."""
    flat = torch.cat([t.contiguous().reshape(-1).view(torch.uint8) for t in tensors]).cpu().numpy()
    out, o = [], 0
    for t in tensors:
        n = t.numel() * t.element_size()
        out.append(flat[o:o + n].copy().view(torch.empty(0, dtype=t.dtype).numpy().dtype).reshape(t.shape))
        o += n
    return out


def jpeg_coeffs_frames(table, rects, quality=95, stream=None):
    """The quantised coefficients of every block of every crop: int16 CUDA [n_blocks, 64], zigzag order, crop by crop, MCU
    by MCU (Y0 Y1 Y2 Y3 Cb Cr), dummy blocks included (oracle.jpeg.blocks of each crop, concatenated)."""
    r = _rects_i32(rects)
    nb = ctypes.c_int64(0)
    args = (table, len(table), r.ctypes.data, len(r), int(quality))
    check(lib().cc_jpeg_coeffs_frames(*args, None, ctypes.byref(nb), None), "cc_jpeg_coeffs_frames")
    coef = torch.empty(nb.value, 64, dtype=torch.int16, device="cuda")
    check(lib().cc_jpeg_coeffs_frames(*args, ptr(coef), ctypes.byref(nb), stream_ptr(stream)), "cc_jpeg_coeffs_frames")
    return coef


def jpeg_crops_decoded_frames(table, rects, quality=95, out=None, stream=None):
    """-> (uint8 CUDA [K, Hmax, Wmax, 3], device int32 status [K]): where the status is JPEG_OK, crop k's slot holds, in its
    h x w corner, the pixels cv2.imdecode gives for the file jpeg_encode_crops_frames writes for it; JPEG_UNSUPPORTED
    (coefficients outside the range where every libjpeg-turbo IDCT agrees) leaves the slot unwritten, for the caller to
    decode that file with cv2.  Nothing waits."""
    r = _rects_i32(rects)
    K = len(r)
    if out is None:
        hmax = max([int(y2 - y1) for _, _, y1, _, y2 in r] + [1])
        wmax = max([int(x2 - x1) for _, x1, _, x2, _ in r] + [1])
        out = torch.zeros(K, hmax, wmax, 3, dtype=torch.uint8, device="cuda")
    args = (table, len(table), r.ctypes.data, K, int(quality))
    need = ctypes.c_size_t(0)
    check(lib().cc_jpeg_crops_decoded_frames(*args, None, 0, 0, None, None, 0, ctypes.byref(need), None),
          "cc_jpeg_crops_decoded_frames")
    ws = torch.empty(max(need.value, 256), dtype=torch.uint8, device=out.device)
    status = torch.empty(max(K, 1), dtype=torch.int32, device=out.device)
    check(lib().cc_jpeg_crops_decoded_frames(*args, ptr(out), out.shape[1], out.shape[2], ptr(status), ptr(ws), ws.numel(), None,
                                             stream_ptr(stream)), "cc_jpeg_crops_decoded_frames")
    return out, status[:K]


# ---- JPEG files -> BGR pixels, pixel for pixel cv2.imdecode(buf, IMREAD_COLOR)
JPEG_OK, JPEG_UNSUPPORTED, JPEG_CORRUPT = 0, 1, 2


class JpegBatch:
    """K files parsed on the host and copied to the device once: the files' bytes and the parse table share one pinned
    buffer and one host-to-device copy."""

    def __init__(self, files, device="cuda"):
        import numpy as np
        files = [bytes(f) for f in files]
        self.K = K = len(files)
        lengths = np.array([len(f) for f in files], np.int64)
        offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64) if K else np.zeros(0, np.int64)
        nbytes = int(lengths.sum())
        tb = int(lib().cc_jpeg_table_bytes())
        self.table_off = (nbytes + 255) & ~255
        host = torch.empty(self.table_off + K * tb, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
        h = host.numpy()
        if K:
            h[:nbytes] = np.frombuffer(b"".join(files), np.uint8)
        self.sizes = np.zeros((K, 2), np.int32)
        self.status = np.zeros(K, np.int32)
        self.blocks = np.zeros(K, np.int64)
        base = host.data_ptr()
        check(lib().cc_jpeg_parse(ctypes.c_void_p(base), nbytes, offsets.ctypes.data, lengths.ctypes.data, K,
                                  ctypes.c_void_p(base + self.table_off), self.sizes.ctypes.data, self.status.ctypes.data,
                                  self.blocks.ctypes.data), "cc_jpeg_parse")
        self.host = host
        self.dev = host.to(device, non_blocking=True)

    def _ptrs(self):
        return (ctypes.c_void_p(self.dev.data_ptr()), ctypes.c_void_p(self.host.data_ptr() + self.table_off),
                ctypes.c_void_p(self.dev.data_ptr() + self.table_off))

    def decode(self, out=None, hmax=None, wmax=None, coef=None, stream=None):
        """-> (out uint8 CUDA [K, Hmax, Wmax, 3], device int32 status [K]).  Image k fills out[k, :h, :w] when its status
        is JPEG_OK; nothing else of `out` is written."""
        ok = self.status == JPEG_OK
        if out is None:
            hmax = hmax or max([int(v) for v in self.sizes[ok, 1]] + [1])
            wmax = wmax or max([int(v) for v in self.sizes[ok, 0]] + [1])
            out = torch.zeros(self.K, hmax, wmax, 3, dtype=torch.uint8, device=self.dev.device)
        status = torch.empty(max(self.K, 1), dtype=torch.int32, device=self.dev.device)
        args = (*self._ptrs(), self.K)
        need = ctypes.c_size_t(0)
        check(lib().cc_jpeg_decode_frames(*args, None, None, ptr(coef), None, 0, ctypes.byref(need), None), "cc_jpeg_decode_frames")
        ws = torch.empty(max(need.value, 256), dtype=torch.uint8, device=self.dev.device)
        check(lib().cc_jpeg_decode_frames(*args, self.dests(out), ptr(status), ptr(coef), ptr(ws), ws.numel(), None,
                                          stream_ptr(stream)), "cc_jpeg_decode_frames")
        return out, status[:self.K]

    def dests(self, out):
        """The decode destinations of a padded batch out uint8 CUDA [>= K, Hmax, Wmax, 3]: image k (parse status OK) to
        the h x w corner of slot k.  ValueError when an image does not fit its slot."""
        import numpy as np
        from ._lib import cc_jpeg_dest
        assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.dim() == 4 and out.shape[0] >= self.K
        K, (w, h) = self.K, self.sizes.T
        ok = self.status == JPEG_OK                     # the other files' rows stay zero: the library does not read them
        big = np.flatnonzero(ok & ((h > out.shape[1]) | (w > out.shape[2])))
        if len(big):
            k = big[0]
            raise ValueError(f"image {k} ({w[k]}x{h[k]}) does not fit the {out.shape[2]}x{out.shape[1]} batch")
        d = np.zeros(max(K, 1), _DEST_ROW)              # filled as one array, like batch_table
        d["data"][:K] = np.where(ok, out.data_ptr() + out.stride(0) * np.arange(K, dtype=np.uint64), 0)
        d["pitch"][:K], d["h"][:K], d["w"][:K] = out.stride(1), h, w
        return (cc_jpeg_dest * len(d)).from_buffer(d)


class JpegDecoder:
    """A reusable decode context for JPEG files that go to caller-given device destinations (cc_jpeg_decode_frames), e.g.
    the frames of MJPEG cameras.  It owns a pinned staging buffer (the files' bytes, then the parse table), its device
    copy, the device workspace and the statuses; each grows when a call needs more and is otherwise reused, so the steady
    state allocates nothing.  One call sequence per batch: `stage` (host: gather and parse) -> `decode` (queued: one
    host-to-device copy, the decode, the statuses back to pinned memory).  The staging buffer is rewritten by the next
    `stage`, so the caller waits for the stream between batches."""

    def __init__(self, device="cuda"):
        import numpy as np
        self.device = torch.device(device)
        self._pin = self.device.type == "cuda"
        self._tb = int(lib().cc_jpeg_table_bytes())
        self._host = torch.empty(0, dtype=torch.uint8)
        self._dev = self._ws = None
        self._st_dev = self._st_host = None
        self.K = 0
        self.sizes = np.zeros((0, 2), np.int32)
        self.status = np.zeros(0, np.int32)
        self._nbytes = 0

    @staticmethod
    def _grow(t, n, **kw):
        if t is not None and t.numel() >= n:
            return t
        return torch.empty(max(n, 256, 0 if t is None else t.numel() * 3 // 2), dtype=kw.pop("dtype", torch.uint8), **kw)

    def stage(self, files, inserts=None):
        """files: K JPEG files (bytes-like, or uint8 CPU tensors / arrays); inserts: None, or per file None or (offset,
        bytes) to insert at that offset while gathering (ingest.default_tables).  Gathers them into the staging buffer
        and parses them -> (sizes int32 [K,2] width, height; parse status int32 [K]), valid until the next `stage`."""
        import numpy as np
        arrs = []
        for f in files:
            if isinstance(f, torch.Tensor):
                arrs.append(f.reshape(-1).numpy())
            else:
                arrs.append(f if isinstance(f, np.ndarray) else np.frombuffer(f, np.uint8))
        inserts = inserts or [None] * len(arrs)
        lengths = np.array([len(a) + (len(i[1]) if i else 0) for a, i in zip(arrs, inserts)], np.int64)
        K = self.K = len(arrs)
        offsets = np.zeros(K, np.int64)
        if K:
            offsets[1:] = np.cumsum(lengths)[:-1]
        nbytes = int(lengths.sum())
        self._table_off = (nbytes + 255) & ~255
        self._nbytes = self._table_off + K * self._tb
        self._host = self._grow(self._host, self._nbytes, pin_memory=self._pin)
        h = self._host.numpy()
        for a, ins, o in zip(arrs, inserts, offsets.tolist()):
            if ins:
                at, seg = ins
                h[o:o + at] = a[:at]
                h[o + at:o + at + len(seg)] = np.frombuffer(seg, np.uint8)
                h[o + at + len(seg):o + len(a) + len(seg)] = a[at:]
            else:
                h[o:o + len(a)] = a
        self.sizes = np.zeros((K, 2), np.int32)
        self.status = np.zeros(K, np.int32)
        blocks = np.zeros(K, np.int64)
        base = self._host.data_ptr()
        check(lib().cc_jpeg_parse(ctypes.c_void_p(base), nbytes, offsets.ctypes.data, lengths.ctypes.data, K,
                                  ctypes.c_void_p(base + self._table_off), self.sizes.ctypes.data, self.status.ctypes.data,
                                  blocks.ctypes.data), "cc_jpeg_parse")
        self._files = (offsets, lengths)
        return self.sizes, self.status

    def file(self, k) -> memoryview:
        """The bytes of staged file k as parsed (default tables inserted)."""
        o, n = (int(x[k]) for x in self._files)
        return memoryview(self._host.numpy()[o:o + n])

    def decode(self, dests, stream=None) -> torch.Tensor:
        """Queue the decode of the staged files: dests[k] is a device uint8 [h,w,3] tensor whose rows are contiguous
        (a frame buffer, or a row of a batch), or None for a file the parse did not accept.  -> pinned int32 [K] statuses,
        filled when the stream reaches this point (JPEG_OK: dests[k] holds cv2.imdecode of file k; otherwise dests[k] is
        as it was)."""
        from ._lib import cc_jpeg_dest
        K = self.K
        outs = (cc_jpeg_dest * max(K, 1))()
        for k, d in enumerate(dests):
            if d is None:
                continue
            assert d.is_cuda and d.dtype == torch.uint8 and d.dim() == 3 and d.shape[2] == 3 and d.stride(2) == 1 \
                and d.stride(1) == 3, "a destination is a device uint8 [h, w, 3] tensor with contiguous rows"
            outs[k] = cc_jpeg_dest(d.data_ptr(), d.stride(0), d.shape[0], d.shape[1])
        self._dev = self._grow(self._dev, self._nbytes, device=self.device)
        self._st_dev = self._grow(self._st_dev, K, dtype=torch.int32, device=self.device)
        self._st_host = self._grow(self._st_host, K, dtype=torch.int32, pin_memory=self._pin)
        base = self._dev.data_ptr()
        h_table = ctypes.c_void_p(self._host.data_ptr() + self._table_off)
        args = (ctypes.c_void_p(base), h_table, ctypes.c_void_p(base + self._table_off), K)
        need = ctypes.c_size_t(0)
        check(lib().cc_jpeg_decode_frames(*args, None, None, None, None, 0, ctypes.byref(need), None), "cc_jpeg_decode_frames")
        self._ws = self._grow(self._ws, need.value, device=self.device)
        self._dev[:self._nbytes].copy_(self._host[:self._nbytes], non_blocking=True)
        check(lib().cc_jpeg_decode_frames(*args, outs, ptr(self._st_dev), None, ptr(self._ws), self._ws.numel(), None,
                                          stream_ptr(stream)), "cc_jpeg_decode_frames")
        st = self._st_host[:K]
        st.copy_(self._st_dev[:K], non_blocking=True)
        return st


def jpeg_decode(files, out=None, stream=None):
    """files: list of `bytes` -> (out uint8 CUDA [K, Hmax, Wmax, 3] BGR, sizes int32 numpy [K, 2] (width, height), device int32
    status [K]).  Where status is JPEG_OK, out[k, :h, :w] is exactly cv2.imdecode(file, IMREAD_COLOR); JPEG_UNSUPPORTED and
    JPEG_CORRUPT images are not written (the caller decodes those with cv2)."""
    b = JpegBatch(files)
    o, st = b.decode(out, stream=stream)
    return o, b.sizes, st


def jpeg_decode_coeffs(files, stream=None):
    """The dequantisation input of every file the host parse accepts: int16 CUDA [n_blocks, 64], zigzag order, block by
    block in scan order, file after file (the coefficient tap), and the device status."""
    b = JpegBatch(files)
    coef = torch.zeros(max(int(b.blocks.sum()), 1), 64, dtype=torch.int16, device=b.dev.device)
    _, st = b.decode(coef=coef, stream=stream)
    return coef[:int(b.blocks.sum())], st
