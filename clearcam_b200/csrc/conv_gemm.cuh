// Implicit-GEMM convolution / linear layer on Hopper warpgroup MMA (wgmma, sm_90a), host-side descriptors.
//
// One kernel serves every GEMM-shaped op on the hot path:
//   * YOLOv9 `Conv` = nn.Conv2d(bias) -> SiLU          (reference detection/yolov9.py:33-38), k in {1,3}, s in {1,2}
//   * bare nn.Conv2d head/CBLinear convs (no act)       (detection/yolov9.py:173,186,224)
//   * RepNBottleneck residual  x + cv2(cv1(x))          (detection/yolov9.py:82-89)  -> residual fused in epilogue
//   * CLIP linears: QKV / out-proj / MLP (+tanh-GELU)   (models/objects.py:107-127,157-179)
//   * AdaFace conv -> BN -> PReLU, shortcuts, linear   (models/adaface.py:45-57,84-92) -> ACT_PRELU epilogue (csrc/adaface.cu)
// Activations are NHWC bf16 (a channel *slice* of a wider buffer is addressed in place, so Tensor.cat /
// chunk in the reference cost nothing here); weights are [Cout][kh][kw][Cin] bf16 (K-major); accumulation fp32
// in registers; bias + activation + residual in the epilogue.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "ops.cuh"

namespace cc {

enum Act : int32_t { ACT_NONE = 0, ACT_SILU = 1, ACT_GELU_TANH = 2, ACT_PRELU = 3 };

struct GemmParams {
  CUtensorMap tmA;  // 5-D view of the NHWC activation (see conv_gemm.cu)
  CUtensorMap tmB;  // 2-D [Cout][Ktot] weights
  CUtensorMap tmO;  // 4-D output slice [N][H][W][Cout] (epilogue TMA stores)
  CUtensorMap tmR;  // 4-D residual slice, same boxes (when res != nullptr)
  int32_t tap[9][4];  // per filter tap: delta on dims 0..3 of the A view
  int32_t num_taps, chunks_per_tap, BK, BN;
  int32_t n_blocks;                   // Cout / BN
  int32_t tiles_w, tiles_h, tiles_n;  // M tiles per dimension
  int32_t lTW, lTH, lTN;              // log2 of the 128-pixel tile box
  int32_t s2;                         // 1: stride-2 "pixel pair" view (dims C2,W/2,2,H/2,N)
  int32_t W, H, N;                    // OUTPUT spatial dims / batch
  int32_t stages;
  int32_t num_tiles;
  // epilogue
  void* out;
  int32_t out_cs, out_co, out_f32;    // channel stride of the out buffer, channel offset, fp32 output flag
  const float* bias;                  // [Cout] or nullptr; ACT_PRELU: [9][Cout], row = the output pixel's border class
  int32_t act;
  const void* res;                    // residual (same dtype as out) or nullptr; may be the output slice itself (in place)
  int32_t res_cs, res_co;
  int32_t cout;
  int32_t out_ns;                     // pixels per image in the out/residual buffers (default H*W)
  int32_t b_res;                      // weights of the (single) N block stay resident in smem for the whole kernel
  // tile index -> (n block, w, h, n) without integer division: q = (umulhi(mul, x) + x) >> shift
  uint32_t fd_nb[2], fd_tw[2], fd_twh[2];
  const float* pre;                   // optional fp32 [N][H/2][W/2][Cout]: added BEFORE the activation at (n, h/2, w/2) — a 1x1 conv over
  int32_t pre_h, pre_w;               //   concat(upsample(a), b) is computed as conv_b(b) + upsample(conv_a(a)) (see yolo.cu)
  unsigned long long* trace;          // optional device timeline slots [8] (globaltimer ns): first CTA entry, dependency released, last CTA exit,
                                      // and of CTA 0: first operands landed, -, first accumulator complete, last epilogue done, exit
  // chained 1x1 conv (conv_gemm_chain_build; ch_n2 == 0: none): the bf16 tiles of n block ch_nb, once in the consumer's
  // staging, are the A operand of a square 1x1 conv of ch_n2 channels whose output goes to tmO2
  CUtensorMap tmW2;                   // 2-D [Cout2][Cin2] weights of the 1x1, box = its standalone BK x Cout2
  CUtensorMap tmP;                    // 4-D partner slice appended to the 1x1's input (one staging box wide; ch_part)
  CUtensorMap tmO2;                   // 4-D output slice of the 1x1
  int32_t ch_n2, ch_nb, ch_k0;        // 1x1 channels, chaining n block, first staging channel of the 1x1's input run
  int32_t ch_part, ch_store1;         // partner box present; the first output is still stored
  int32_t ch_bk2;                     // K block of the 1x1's weights in smem (the standalone launch's BK)
  int32_t ch_stage;                   // bytes of one consumer's staging region (staging + partner box, or the 1x1's output tile)
  int32_t act2, out2_f32;
  const float* bias2;                 // [Cout2] or nullptr
  const float* slope;                 // ACT_PRELU: [Cout] negative-side slopes
};

// One conv / linear as the host describes it.  The slices carry pointer, row pitch, channel offset and width; the output
// extent follows from the input's and the stride (conv_out), so the N / H / W of `out` and `res` are not read.
struct ConvDesc {
  TSlice in;                               // bf16 input slice; N, H, W: stored input dims (even for stride 2)
  const void* w;                           // bf16 [Cout][k*k*Cin]
  const float* bias;                       // ACT_PRELU: fp32 [9][Cout] (see GemmParams::bias), bf16 output only
  const float* slope;                      // ACT_PRELU: fp32 [Cout]
  int k, stride;                           // k in {1,3}; pad = k/2; stride in {1,2}
  TSlice out;                              // output slice, C = Cout, bf16 or fp32 (f32); p == nullptr: none (a chain that drops it)
  int act;
  TSlice res;                              // residual slice (same dtype as out), p == nullptr: none
  int bn_override;                         // 0 = heuristic
  int out_ns;                              // 0 = Hout*Wout; else pixels per image in the out/residual buffers
  const float* pre; int pre_h, pre_w;      // optional half-resolution fp32 pre-activation addend (see GemmParams::pre)
};
// The one place a ConvDesc is made; bn_override, out_ns and pre start at 0 and are set by the few callers that use them.
inline ConvDesc conv_desc(const TSlice& in, const void* w, const float* bias, int k, int stride, const TSlice& out, int act,
                          const TSlice* res = nullptr) {
  ConvDesc d{};
  d.in = in; d.w = w; d.bias = bias; d.k = k; d.stride = stride; d.out = out; d.act = act;
  if (res) d.res = *res;
  return d;
}
// Output extent of the convs the GEMM kernel runs (pad = k/2, even input sides for stride 2)
inline int conv_out(int n, int stride) { return stride == 2 ? n / 2 : n; }
// The same conv for the direct kernel (conv_direct.cu), which also takes grouped convs and odd extents
DirectConvParams direct_conv_params(const ConvDesc& d, int groups);

// A square 1x1 conv run in the epilogue of the conv it reads (conv_gemm_chain_build): its input is the channel run
// [k0, k0 + out.C - part.C) of that conv's output, followed by an optional partner slice of part.C channels
struct ChainDesc {
  const void* w;                           // bf16 [Cout][Cout], Cout = out.C
  const float* bias;
  int act, k0;
  TSlice part;                             // partner slice (bf16, same pixels as the output), p == nullptr: none
  TSlice out;                              // bf16 or fp32 (f32) output slice
  bool store1;                             // also store the first conv's output (ConvDesc::out)
};

struct GemmLaunch {
  GemmParams p;
  int grid, smem_bytes;
  double flops;       // 2*M*N*K algorithmic
  double bytes;       // algorithmic HBM bytes: input slice once + output once (+ residual) + weights once
};

// Returns 0 on success; <0 and sets cc_last_error otherwise.
int conv_gemm_build(const ConvDesc& d, int num_sms, GemmLaunch* out);
// The conv d with the 1x1 c in its epilogue: bit-identical to two conv_gemm_build launches.  Fails with CC_ERR_INVALID
// (nothing built) when the pair does not chain: see the conditions in conv_gemm.cu.
int conv_gemm_chain_build(const ConvDesc& d, const ChainDesc& c, int num_sms, GemmLaunch* out);
int conv_gemm_launch(const GemmLaunch& L, cudaStream_t stream);
bool conv_gemm_supported(const ConvDesc& d);

}  // namespace cc
