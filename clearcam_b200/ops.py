"""Thin Python wrappers over the kernel-level C-ABI ops (used by the parity tests and the graphs)."""
import ctypes

import torch

from ._lib import lib, check, ptr, stream_ptr


def conv2d(xbuf, in_co, Cin, w, bias, k, stride, obuf, out_co, Cout, act=0, res=None, res_co=0, groups=1, impl=0, bn=0,
           stream=None):
    """xbuf: [N,H,W,in_cs] bf16 CUDA; w: [Cout,k,k,Cin/groups] bf16; obuf: [N,Ho,Wo,out_cs] bf16|fp32."""
    assert xbuf.is_cuda and xbuf.dtype == torch.bfloat16 and xbuf.is_contiguous()
    assert w.dtype == torch.bfloat16 and w.is_contiguous() and obuf.is_contiguous()
    N, H, W, in_cs = xbuf.shape
    out_cs = obuf.shape[-1]
    out_f32 = 1 if obuf.dtype == torch.float32 else 0
    rc = lib().cc_conv2d(ptr(xbuf), N, H, W, in_cs, in_co, Cin, ptr(w), ptr(bias), Cout, k, stride, groups, ptr(obuf),
                         out_cs, out_co, out_f32, act, ptr(res), 0 if res is None else res.shape[-1], res_co, impl, bn,
                         stream_ptr(stream))
    check(rc, "cc_conv2d")
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
