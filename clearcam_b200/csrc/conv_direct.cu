// Direct (CUDA-core) NHWC convolution: the generic path for shapes the wgmma kernel does not take
// (channel counts that are not multiples of 16 — YOLOv9-t/-s/-m widths such as 24/48/90 —, true grouped
// convs, odd spatial sizes with stride 2) and the stem.  fp32 accumulate, same epilogue semantics as
// conv_gemm (bias -> act -> +residual).  Reference: detection/yolov9.py:33-38 (Conv), :171-194 (head convs).
#include "ops.cuh"
#include "conv_gemm.cuh"
#include "cc_common.h"
#include <cuda_bf16.h>

namespace cc {

__device__ __forceinline__ float act_apply_d(float x, int act) {
  if (act == 1) return x / (1.0f + __expf(-x));
  if (act == 2) {
    const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
    return 0.5f * x * (1.0f + tanhf(u));
  }
  return x;
}

// one thread = one output pixel x 4 consecutive output channels
__global__ void conv_direct_kernel(DirectConvParams p) {
  const int cq = (p.Cout + 3) / 4;
  const long long total = static_cast<long long>(p.N) * p.Hout * p.Wout * cq;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(idx % cq) * 4;
    long long pix = idx / cq;
    const int ox = static_cast<int>(pix % p.Wout);
    const int oy = static_cast<int>((pix / p.Wout) % p.Hout);
    const int n = static_cast<int>(pix / (static_cast<long long>(p.Wout) * p.Hout));
    const int cpg_out = p.Cout / p.groups, cpg_in = p.Cin / p.groups;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < 4; ++j) {
      const int co = c4 + j;
      if (co >= p.Cout) break;
      const int g = co / cpg_out;
      const __nv_bfloat16* wrow = p.w + static_cast<long long>(co) * p.k * p.k * cpg_in;
      float a = 0.f;
      for (int r = 0; r < p.k; ++r) {
        const int iy = oy * p.stride + r - p.pad;
        if (iy < 0 || iy >= p.Hin) continue;
        for (int s = 0; s < p.k; ++s) {
          const int ix = ox * p.stride + s - p.pad;
          if (ix < 0 || ix >= p.Win) continue;
          const __nv_bfloat16* ip =
              p.in + ((static_cast<long long>(n) * p.Hbuf + iy) * p.Wbuf + ix) * p.in_cs + p.in_co + g * cpg_in;
          const __nv_bfloat16* wp = wrow + (r * p.k + s) * cpg_in;
          for (int c = 0; c < cpg_in; ++c) a = fmaf(__bfloat162float(ip[c]), __bfloat162float(wp[c]), a);
        }
      }
      acc[j] = a;
    }
    const long long opix = (static_cast<long long>(n) * p.Hout + oy) * p.Wout + ox;
    for (int j = 0; j < 4; ++j) {
      const int co = c4 + j;
      if (co >= p.Cout) break;
      float x = acc[j] + (p.bias ? p.bias[co] : 0.f);
      x = act_apply_d(x, p.act);
      if (p.res) {
        if (p.out_f32) x += reinterpret_cast<const float*>(p.res)[opix * p.res_cs + p.res_co + co];
        else x += __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.res)[opix * p.res_cs + p.res_co + co]);
      }
      if (p.out_f32) reinterpret_cast<float*>(p.out)[opix * p.out_cs + p.out_co + co] = x;
      else reinterpret_cast<__nv_bfloat16*>(p.out)[opix * p.out_cs + p.out_co + co] = __float2bfloat16_rn(x);
    }
  }
}

DirectConvParams direct_conv_params(const ConvDesc& d, int groups) {
  DirectConvParams p{};
  p.in = d.in.p; p.in_cs = d.in.cs; p.in_co = d.in.co; p.Cin = d.in.C;
  p.N = d.in.N; p.Hin = d.in.H; p.Win = d.in.W; p.Hbuf = d.in.H; p.Wbuf = d.in.W;
  p.k = d.k; p.stride = d.stride; p.pad = d.k / 2; p.groups = groups;
  p.w = static_cast<const __nv_bfloat16*>(d.w); p.bias = d.bias;
  p.out = d.out.p; p.out_cs = d.out.cs; p.out_co = d.out.co; p.Cout = d.out.C; p.out_f32 = d.out.f32;
  p.Hout = (p.Hin + 2 * p.pad - p.k) / p.stride + 1;   // the general form: conv_out() only holds for the GEMM kernel's shapes
  p.Wout = (p.Win + 2 * p.pad - p.k) / p.stride + 1;
  p.act = d.act; p.res = d.res.p; p.res_cs = d.res.cs; p.res_co = d.res.co;
  return p;
}

int conv_direct_launch(const DirectConvParams& p, cudaStream_t stream) {
  CC_REQUIRE(p.groups >= 1 && p.Cin % p.groups == 0 && p.Cout % p.groups == 0, "conv_direct: bad groups");
  const long long total = static_cast<long long>(p.N) * p.Hout * p.Wout * ((p.Cout + 3) / 4);
  if (total == 0) return CC_OK;
  const int threads = 128;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > 132 * 64) blocks = 132 * 64;
  conv_direct_kernel<<<static_cast<int>(blocks), threads, 0, stream>>>(p);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // namespace cc
