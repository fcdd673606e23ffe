// C-ABI entry points (include/clearcam_b200.h).
#include "clearcam_b200.h"
#include "cc_common.h"
#include "conv_gemm.cuh"
#include "ops.cuh"

using namespace cc;

extern "C" {

int cc_version(void) { return CC_ABI_VERSION; }
const char* cc_last_error(void) { return last_error(); }
int cc_device_check(void) {
  const int n = device_sm_count();
  if (n <= 0) set_error("no sm_90 (H100) CUDA device available");
  return n;
}

int cc_conv2d(const void* d_in, int N, int Hin, int Win, int in_cs, int in_co, int Cin, const void* d_w,
              const float* d_bias, int Cout, int k, int stride, int groups, void* d_out, int out_cs, int out_co,
              int out_f32, int act, const void* d_res, int res_cs, int res_co, int impl, int bn, void* stream) {
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_conv2d: no sm_90 (H100) device");
  ConvDesc d{};
  d.in = d_in; d.in_cs = in_cs; d.in_co = in_co; d.Cin = Cin;
  d.N = N; d.Hin = Hin; d.Win = Win; d.k = k; d.stride = stride;
  d.w = d_w; d.bias = d_bias;
  d.out = d_out; d.out_cs = out_cs; d.out_co = out_co; d.Cout = Cout; d.out_f32 = out_f32;
  d.act = act; d.res = d_res; d.res_cs = res_cs; d.res_co = res_co; d.bn_override = bn;
  const bool gemm_ok = groups == 1 && conv_gemm_supported(d);
  CC_REQUIRE(impl != 1 || gemm_ok, "cc_conv2d: shape not supported by the wgmma path");
  if (impl != 2 && gemm_ok) {
    GemmLaunch L;
    int rc = conv_gemm_build(d, sms, &L);
    if (rc) return rc;
    return conv_gemm_launch(L, static_cast<cudaStream_t>(stream));
  }
  DirectConvParams p{};
  p.in = static_cast<const __nv_bfloat16*>(d_in); p.in_cs = in_cs; p.in_co = in_co; p.Cin = Cin;
  p.N = N; p.Hin = Hin; p.Win = Win; p.Hbuf = Hin; p.Wbuf = Win;
  p.k = k; p.stride = stride; p.pad = k / 2; p.groups = groups;
  p.w = static_cast<const __nv_bfloat16*>(d_w); p.bias = d_bias;
  p.out = d_out; p.out_cs = out_cs; p.out_co = out_co; p.Cout = Cout; p.out_f32 = out_f32;
  p.Hout = (Hin + 2 * p.pad - k) / stride + 1;
  p.Wout = (Win + 2 * p.pad - k) / stride + 1;
  p.act = act; p.res = d_res; p.res_cs = res_cs; p.res_co = res_co;
  return conv_direct_launch(p, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
