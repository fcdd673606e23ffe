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
  const TSlice res = nhwc_slice(d_res, res_cs, res_co, Cout, out_f32);
  ConvDesc d = conv_desc(nhwc_slice(d_in, in_cs, in_co, Cin, 0, N, Hin, Win), d_w, d_bias, k, stride,
                         nhwc_slice(d_out, out_cs, out_co, Cout, out_f32), act, d_res ? &res : nullptr);
  d.bn_override = bn;
  const bool gemm_ok = groups == 1 && conv_gemm_supported(d);
  CC_REQUIRE(impl != 1 || gemm_ok, "cc_conv2d: shape not supported by the wgmma path");
  if (impl != 2 && gemm_ok) {
    GemmLaunch L;
    int rc = conv_gemm_build(d, sms, &L);
    if (rc) return rc;
    return conv_gemm_launch(L, static_cast<cudaStream_t>(stream));
  }
  return conv_direct_launch(direct_conv_params(d, groups), static_cast<cudaStream_t>(stream));
}

int cc_conv2d_chain(const void* d_in, int N, int Hin, int Win, int in_cs, int in_co, int Cin, const void* d_w, const float* d_bias,
                    int Cout, int k, int stride, void* d_out, int out_cs, int out_co, int store1, const void* d_res, int res_cs,
                    int res_co, const void* d_w2, const float* d_bias2, int Cout2, int act2, int k0, const void* d_part, int part_cs,
                    int part_co, int part_C, void* d_out2, int out2_cs, int out2_co, int out2_f32, void* stream) {
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_conv2d_chain: no sm_90 (H100) device");
  CC_REQUIRE(d_in && (d_out || !store1) && d_w2 && d_out2 && (!d_part || part_C > 0), "cc_conv2d_chain: NULL argument");
  CC_REQUIRE(!d_part || (part_co >= 0 && part_co + part_C <= part_cs), "cc_conv2d_chain: partner slice outside its row");
  const TSlice res = nhwc_slice(d_res, res_cs, res_co, Cout);
  const ConvDesc d = conv_desc(nhwc_slice(d_in, in_cs, in_co, Cin, 0, N, Hin, Win), d_w, d_bias, k, stride,
                               nhwc_slice(d_out, out_cs, out_co, Cout), CC_ACT_SILU, d_res ? &res : nullptr);
  ChainDesc c{};
  c.w = d_w2; c.bias = d_bias2; c.act = act2; c.k0 = k0;
  if (d_part) c.part = nhwc_slice(d_part, part_cs, part_co, part_C);
  c.out = nhwc_slice(d_out2, out2_cs, out2_co, Cout2, out2_f32);
  c.store1 = store1 != 0;
  CC_REQUIRE(out2_co >= 0 && out2_co + Cout2 <= out2_cs, "cc_conv2d_chain: second output slice outside its row");
  GemmLaunch L;
  if (int rc = conv_gemm_chain_build(d, c, sms, &L)) return rc;
  return conv_gemm_launch(L, static_cast<cudaStream_t>(stream));
}

int cc_conv2d_prelu(const void* d_in, int N, int Hin, int Win, int in_cs, int in_co, int Cin, const void* d_w, const float* d_bias_cls,
                    const float* d_slope, int Cout, int k, int stride, void* d_out, int out_cs, int out_co, const void* d_res,
                    int res_cs, int res_co, int bn, void* stream) {
  CC_REQUIRE(d_in && d_w && d_bias_cls && d_slope && d_out, "cc_conv2d_prelu: d_in, d_w, d_bias_cls, d_slope and d_out must not be NULL");
  CC_REQUIRE(N >= 1 && Hin >= 1 && Win >= 1, "cc_conv2d_prelu: bad shape N=%d Hin=%d Win=%d", N, Hin, Win);
  const TSlice res = nhwc_slice(d_res, res_cs, res_co, Cout);
  ConvDesc d = conv_desc(nhwc_slice(d_in, in_cs, in_co, Cin, 0, N, Hin, Win), d_w, d_bias_cls, k, stride,
                         nhwc_slice(d_out, out_cs, out_co, Cout), ACT_PRELU, d_res ? &res : nullptr);
  d.slope = d_slope;
  d.bn_override = bn;
  CC_REQUIRE(conv_gemm_supported(d), "cc_conv2d_prelu: shape not supported by the wgmma conv (Cin=%d Cout=%d k=%d stride=%d)", Cin, Cout, k, stride);
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_conv2d_prelu: no sm_90 (H100) device");
  GemmLaunch L;
  if (int rc = conv_gemm_build(d, sms, &L)) return rc;
  return conv_gemm_launch(L, static_cast<cudaStream_t>(stream));
}

int cc_attention(const void* d_qkv, int B, int L, int H, int causal, int impl, void* d_ws, size_t ws_bytes, void* d_ctx,
                 size_t* ws_needed, void* stream) {
  CC_REQUIRE(impl == 1 || impl == 2, "cc_attention: unknown impl %d (1 = mma.sync, 2 = wgmma)", impl);
  CC_REQUIRE(B >= 0 && L >= 1 && H >= 1, "cc_attention: bad shape B=%d L=%d H=%d", B, L, H);
  const int max_len = impl == 1 ? attention_max_len() : attention_tc_max_len();
  CC_REQUIRE(L <= max_len, "cc_attention: sequence length %d too long for impl %d (at most %d)", L, impl, max_len);
  // one CTA row per (image, head): gridDim.x for the mma.sync kernel, gridDim.y (at most 65535) for the wgmma kernel
  CC_REQUIRE(static_cast<long long>(B) * H <= (impl == 1 ? 0x7fffffffLL : 65535LL),
             "cc_attention: B*H = %lld (image, head) pairs exceed the grid of impl %d", static_cast<long long>(B) * H, impl);
  const size_t need = impl == 2 ? attention_tc_workspace_bytes(B, L, H) : 0;
  if (ws_needed) *ws_needed = need;
  if (!d_ctx) return CC_OK;   // workspace size query
  CC_REQUIRE(d_qkv != nullptr, "cc_attention: d_qkv is NULL");
  CC_REQUIRE(ws_bytes >= need && (need == 0 || d_ws != nullptr), "cc_attention: workspace of %zu bytes too small (%zu needed)",
             d_ws ? ws_bytes : size_t(0), need);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_ws) & 15) == 0,
             "cc_attention: d_qkv and d_ws must be 16-byte aligned");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* qkv = static_cast<const __nv_bfloat16*>(d_qkv);
  __nv_bfloat16* ctx = static_cast<__nv_bfloat16*>(d_ctx);
  return impl == 1 ? attention_launch(qkv, ctx, B, L, H, causal ? 1 : 0, st)
                   : attention_tc_launch(qkv, ctx, static_cast<__nv_bfloat16*>(d_ws), B, L, H, causal ? 1 : 0, st);
}

}  // extern "C"

// An NHWC slice argument of the detector taps: non-NULL, 16-byte aligned, cs / co / C in whole vectors of `vec` channels
// and the slice inside the row.
static int slice_arg(const char* who, const char* what, const void* p, int N, int H, int W, int cs, int co, int C, int f32, int vec,
                     TSlice* t) {
  CC_REQUIRE(p != nullptr, "%s: %s is NULL", who, what);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0, "%s: %s must be 16-byte aligned", who, what);
  CC_REQUIRE(N >= 1 && H >= 1 && W >= 1 && C >= 1, "%s: %s has a bad shape N=%d H=%d W=%d C=%d", who, what, N, H, W, C);
  CC_REQUIRE(C % vec == 0 && co % vec == 0 && cs % vec == 0 && co >= 0 && co + C <= cs,
             "%s: %s slice cs=%d co=%d C=%d must be whole vectors of %d channels inside the row", who, what, cs, co, C, vec);
  *t = nhwc_slice(p, cs, co, C, f32, N, H, W);
  return CC_OK;
}

extern "C" {

int cc_pool(int op, int f32, const void* d_in, int N, int H, int W, int in_cs, int in_co, int C, void* d_out, int out_cs, int out_co,
            void* stream) {
  CC_REQUIRE(op >= CC_POOL_AVG2_PAD && op <= CC_POOL_UPSAMPLE2, "cc_pool: unknown op %d", op);
  CC_REQUIRE(f32 == 0 || f32 == 1, "cc_pool: f32 is 0 (bf16) or 1 (fp32), got %d", f32);
  CC_REQUIRE(op == CC_POOL_MAX5 || op == CC_POOL_UPSAMPLE2 || (H >= 2 && W >= 2), "cc_pool: op %d needs a map of at least 2x2", op);
  CC_REQUIRE(op != CC_POOL_AVGMAX || (H % 2 == 0 && W % 2 == 0), "cc_pool: avgmax needs even sides, got %dx%d", H, W);
  const int Ho = op == CC_POOL_AVGMAX ? H / 2 : op == CC_POOL_UPSAMPLE2 ? 2 * H : H;
  const int Wo = op == CC_POOL_AVGMAX ? W / 2 : op == CC_POOL_UPSAMPLE2 ? 2 * W : W;
  TSlice in, out;
  if (int rc = slice_arg("cc_pool", "input", d_in, N, H, W, in_cs, in_co, C, f32, 8, &in)) return rc;
  if (int rc = slice_arg("cc_pool", "output", d_out, N, Ho, Wo, out_cs, out_co, C, f32, 8, &out)) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (op) {
    case CC_POOL_AVG2_PAD: return avgpool2_pad_launch(in, out, st);
    case CC_POOL_AVGMAX: return avgmax_pool_launch(in, out, st);
    case CC_POOL_MAX5: return maxpool5_launch(in, out, st);
    default: return upsample2_launch(in, out, st);
  }
}

int cc_spp3(void* d_cat, int N, int H, int W, int cs, int co, int c1, void* stream) {
  CC_REQUIRE(c1 >= 1, "cc_spp3: c1=%d", c1);
  TSlice cat;
  if (int rc = slice_arg("cc_spp3", "concat buffer", d_cat, N, H, W, cs, co, 4 * c1, 0, 8, &cat)) return rc;
  CC_REQUIRE(N <= 65535, "cc_spp3: N=%d exceeds the grid", N);
  CC_REQUIRE(spp3_supported(cat, c1), "cc_spp3: not supported for H*W=%d, c1=%d (c1 a multiple of 64, at most 800 pixels)", H * W, c1);
  return spp3_launch(cat, c1, static_cast<cudaStream_t>(stream));
}

int cc_cbfuse(int f32, int nsrc, const void* const* d_src, const int* src_h, const int* src_w, const int* src_cs, const int* src_co,
              const void* d_last, int last_cs, int last_co, void* d_out, int out_cs, int out_co, int N, int H, int W, int C,
              void* stream) {
  CC_REQUIRE(f32 == 0 || f32 == 1, "cc_cbfuse: f32 is 0 (bf16) or 1 (fp32), got %d", f32);
  CC_REQUIRE(nsrc >= 1 && nsrc <= 5, "cc_cbfuse: nsrc=%d (1 to 5 sources)", nsrc);
  CC_REQUIRE(d_src && src_h && src_w && src_cs && src_co, "cc_cbfuse: a NULL source array");
  CBFuseParams p{};
  p.nsrc = nsrc;
  for (int k = 0; k < nsrc; ++k)
    if (int rc = slice_arg("cc_cbfuse", "a source", d_src[k], N, src_h[k], src_w[k], src_cs[k], src_co[k], C, f32, 8, &p.src[k])) return rc;
  if (int rc = slice_arg("cc_cbfuse", "last", d_last, N, H, W, last_cs, last_co, C, f32, 8, &p.last)) return rc;
  if (int rc = slice_arg("cc_cbfuse", "output", d_out, N, H, W, out_cs, out_co, C, f32, 8, &p.out)) return rc;
  return cbfuse_launch(p, static_cast<cudaStream_t>(stream));
}

int cc_split_planes(const float* d_in, int npix, int cs, int co, int C, void* d_out, void* stream) {
  TSlice in;
  if (int rc = slice_arg("cc_split_planes", "input", d_in, npix, 1, 1, cs, co, C, 1, 4, &in)) return rc;
  CC_REQUIRE(d_out != nullptr && (reinterpret_cast<uintptr_t>(d_out) & 7) == 0, "cc_split_planes: d_out must be 8-byte aligned");
  return split_planes_launch(in, static_cast<__nv_bfloat16*>(d_out), static_cast<cudaStream_t>(stream));
}

int cc_finish_f32(const float* d_acc, const float* d_bias, int act, int npix, int C, float* d_out, int out_cs, int out_co,
                  const float* d_res, int res_cs, int res_co, void* stream) {
  CC_REQUIRE(act == CC_ACT_NONE || act == CC_ACT_SILU, "cc_finish_f32: act %d (0 none, 1 SiLU)", act);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_bias) & 15) == 0, "cc_finish_f32: d_bias must be 16-byte aligned");
  FinishParams p{};
  TSlice t;
  if (int rc = slice_arg("cc_finish_f32", "acc", d_acc, npix, 1, 1, C, 0, C, 1, 4, &t)) return rc;
  if (int rc = slice_arg("cc_finish_f32", "output", d_out, npix, 1, 1, out_cs, out_co, C, 1, 4, &t)) return rc;
  if (d_res)
    if (int rc = slice_arg("cc_finish_f32", "residual", d_res, npix, 1, 1, res_cs, res_co, C, 1, 4, &t)) return rc;
  p.acc = d_acc; p.bias = d_bias; p.act = act; p.npix = npix; p.C = C;
  p.out = d_out; p.out_cs = out_cs; p.out_co = out_co;
  p.res = d_res; p.res_cs = res_cs; p.res_co = res_co;
  return finish_f32_launch(p, static_cast<cudaStream_t>(stream));
}

int cc_conv2d_pre(const void* d_in, int N, int Hin, int Win, int in_cs, int in_co, int Cin, const void* d_w, const float* d_bias,
                  int Cout, int k, int stride, void* d_out, int out_cs, int out_co, int out_f32, int act, const float* d_pre, int bn,
                  void* stream) {
  CC_REQUIRE(d_in && d_w && d_out && d_pre, "cc_conv2d_pre: d_in, d_w, d_out and d_pre must not be NULL");
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_pre) & 15) == 0, "cc_conv2d_pre: d_pre must be 16-byte aligned");
  CC_REQUIRE(N >= 1 && Hin >= 1 && Win >= 1 && (stride == 1 || stride == 2), "cc_conv2d_pre: bad shape N=%d Hin=%d Win=%d stride=%d", N, Hin, Win, stride);
  const int Ho = conv_out(Hin, stride), Wo = conv_out(Win, stride);
  CC_REQUIRE(Ho % 2 == 0 && Wo % 2 == 0, "cc_conv2d_pre: the output %dx%d must have even sides (pre is its half-resolution map)", Ho, Wo);
  ConvDesc d = conv_desc(nhwc_slice(d_in, in_cs, in_co, Cin, 0, N, Hin, Win), d_w, d_bias, k, stride,
                         nhwc_slice(d_out, out_cs, out_co, Cout, out_f32), act);
  d.bn_override = bn;
  d.pre = d_pre; d.pre_h = Ho / 2; d.pre_w = Wo / 2;
  CC_REQUIRE(conv_gemm_supported(d), "cc_conv2d_pre: shape not supported by the wgmma conv (Cin=%d Cout=%d k=%d stride=%d)", Cin, Cout, k, stride);
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_conv2d_pre: no sm_90 (H100) device");
  GemmLaunch L;
  if (int rc = conv_gemm_build(d, sms, &L)) return rc;
  return conv_gemm_launch(L, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

// ---- the CLIP encoders' row kernels (vit.cu) as the plans run them
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int ln_width_arg(const char* who, int W) {
  CC_REQUIRE(layernorm_width_supported(W), "%s: width %d not supported (128 x 1, 2, 3, 4, 5, 6, 8, 10 or 12)", who, W);
  return CC_OK;
}

extern "C" {

int cc_patchify(const float* d_x, int B, int S, int p, int Kpad, void* d_out, void* stream) {
  CC_REQUIRE(d_x && d_out, "cc_patchify: d_x and d_out must not be NULL");
  CC_REQUIRE(aligned16(d_out), "cc_patchify: d_out must be 16-byte aligned");
  CC_REQUIRE(B >= 0 && S >= 1 && p >= 1, "cc_patchify: bad shape B=%d S=%d p=%d", B, S, p);
  CC_REQUIRE(S % p == 0, "cc_patchify: image side %d is not a multiple of the patch %d", S, p);
  CC_REQUIRE(Kpad % 8 == 0 && Kpad >= 3 * p * p, "cc_patchify: Kpad=%d must be a multiple of 8 and at least 3p^2 = %d", Kpad,
             3 * p * p);
  if (B == 0) return CC_OK;
  return patchify_launch(d_x, static_cast<__nv_bfloat16*>(d_out), B, S, p, Kpad, static_cast<cudaStream_t>(stream));
}

int cc_clip_embed_ln(float* d_x, const float* d_cls, const float* d_pos, const float* d_gamma, const float* d_beta, int B, int L, int W,
                     void* stream) {
  CC_REQUIRE(d_x && d_cls && d_pos && d_gamma && d_beta, "cc_clip_embed_ln: a NULL pointer");
  CC_REQUIRE(aligned16(d_x) && aligned16(d_cls) && aligned16(d_pos) && aligned16(d_gamma) && aligned16(d_beta),
             "cc_clip_embed_ln: every pointer must be 16-byte aligned");
  CC_REQUIRE(B >= 0 && L >= 1 && static_cast<long long>(B) * L <= 0x7fffffffLL, "cc_clip_embed_ln: bad shape B=%d L=%d", B, L);
  if (int rc = ln_width_arg("cc_clip_embed_ln", W)) return rc;
  if (B == 0) return CC_OK;
  return embed_ln_pre_launch(d_x, d_cls, d_pos, d_gamma, d_beta, B * L, L, W, static_cast<cudaStream_t>(stream));
}

int cc_layernorm_bf16(const float* d_x, int rows, int W, long long row_stride, const int32_t* d_row_idx, const float* d_gamma,
                      const float* d_beta, void* d_out, void* stream) {
  CC_REQUIRE(d_x && d_gamma && d_beta && d_out, "cc_layernorm_bf16: d_x, d_gamma, d_beta and d_out must not be NULL");
  CC_REQUIRE(aligned16(d_x) && aligned16(d_gamma) && aligned16(d_beta), "cc_layernorm_bf16: d_x, d_gamma and d_beta must be 16-byte aligned");
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_out) & 7) == 0, "cc_layernorm_bf16: d_out must be 8-byte aligned");
  CC_REQUIRE(rows >= 0 && row_stride >= 0, "cc_layernorm_bf16: bad shape rows=%d row_stride=%lld", rows, row_stride);
  if (int rc = ln_width_arg("cc_layernorm_bf16", W)) return rc;
  return layernorm_bf16_launch(d_x, static_cast<__nv_bfloat16*>(d_out), d_gamma, d_beta, rows, W, row_stride, d_row_idx,
                               static_cast<cudaStream_t>(stream));
}

int cc_text_embed(const int32_t* d_ids, const float* d_tok, const float* d_pos, int B, int L, int W, int vocab, float* d_x,
                  int32_t* d_eot_row, void* stream) {
  CC_REQUIRE(d_ids && d_tok && d_pos && d_x && d_eot_row, "cc_text_embed: a NULL pointer");
  CC_REQUIRE(aligned16(d_tok) && aligned16(d_pos) && aligned16(d_x), "cc_text_embed: d_tok, d_pos and d_x must be 16-byte aligned");
  CC_REQUIRE(B >= 0 && L >= 1 && W >= 4 && W % 4 == 0 && vocab >= 1 && static_cast<long long>(B) * L <= 0x7fffffffLL,
             "cc_text_embed: bad shape B=%d L=%d W=%d vocab=%d (W a multiple of 4)", B, L, W, vocab);
  if (B == 0) return CC_OK;
  return text_embed_launch(d_ids, d_tok, d_pos, d_x, d_eot_row, B, L, W, vocab, static_cast<cudaStream_t>(stream));
}

int cc_l2norm(const float* d_in, int rows, int D, float eps, float* d_out, long long out_stride, void* stream) {
  CC_REQUIRE(d_in && d_out, "cc_l2norm: d_in and d_out must not be NULL");
  CC_REQUIRE(rows >= 0 && D >= 1, "cc_l2norm: bad shape rows=%d D=%d", rows, D);
  CC_REQUIRE(out_stride >= D, "cc_l2norm: out_stride %lld is shorter than a row of %d", out_stride, D);
  CC_REQUIRE(eps >= 0.f, "cc_l2norm: eps must be >= 0");
  return l2norm_launch(d_in, d_out, rows, D, out_stride, eps, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
