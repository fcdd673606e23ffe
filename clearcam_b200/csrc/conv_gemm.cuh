// Implicit-GEMM convolution / linear layer on Hopper warpgroup MMA (wgmma, sm_90a), host-side descriptors.
//
// One kernel serves every GEMM-shaped op on the hot path:
//   * YOLOv9 `Conv` = nn.Conv2d(bias) -> SiLU          (reference detection/yolov9.py:33-38), k in {1,3}, s in {1,2}
//   * bare nn.Conv2d head/CBLinear convs (no act)       (detection/yolov9.py:173,186,224)
//   * RepNBottleneck residual  x + cv2(cv1(x))          (detection/yolov9.py:82-89)  -> residual fused in epilogue
//   * CLIP linears: QKV / out-proj / MLP (+tanh-GELU)   (models/objects.py:107-127,157-179)
// Activations are NHWC bf16 (a channel *slice* of a wider buffer is addressed in place, so Tensor.cat /
// chunk in the reference cost nothing here); weights are [Cout][kh][kw][Cin] bf16 (K-major); accumulation fp32
// in registers; bias + activation + residual in the epilogue.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cc {

enum Act : int32_t { ACT_NONE = 0, ACT_SILU = 1, ACT_GELU_TANH = 2, ACT_SILU_EXACT = 3 };

struct GemmParams {
  CUtensorMap tmA;  // 5-D view of the NHWC activation (see conv_gemm.cu)
  CUtensorMap tmB;  // 2-D [Cout][Ktot] weights
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
  const float* bias;                  // [Cout] or nullptr
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
};

struct ConvDesc {
  const void* in; int in_cs, in_co, Cin;   // input buffer: channels per pixel, slice offset, slice width
  int N, Hin, Win;                         // stored input dims (even for stride 2)
  int k, stride;                           // k in {1,3}; pad = k/2; stride in {1,2}
  const void* w;                           // bf16 [Cout][k*k*Cin]
  const float* bias;
  void* out; int out_cs, out_co, Cout, out_f32;
  int act;
  const void* res; int res_cs, res_co;
  int bn_override;                         // 0 = heuristic
  int out_ns;                              // 0 = Hout*Wout; else pixels per image in the out/residual buffers
  const float* pre; int pre_h, pre_w;      // optional half-resolution fp32 pre-activation addend (see GemmParams::pre)
};

struct GemmLaunch {
  GemmParams p;
  int grid, smem_bytes;
  double flops;       // 2*M*N*K algorithmic
  double bytes;       // algorithmic HBM bytes: input slice once + output once (+ residual) + weights once
};

// Returns 0 on success; <0 and sets cc_last_error otherwise.
int conv_gemm_build(const ConvDesc& d, int num_sms, GemmLaunch* out);
int conv_gemm_launch(const GemmLaunch& L, cudaStream_t stream);
bool conv_gemm_supported(const ConvDesc& d);

}  // namespace cc
