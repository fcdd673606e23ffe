// C-ABI entry points (include/clearcam_b200.h).
#include <utility>
#include "clearcam_b200.h"
#include "cc_common.h"
#include "conv_gemm.cuh"
#include "ops.cuh"

using namespace cc;

// ---- one conv launch: the public cc_conv_op and the descriptors the conv kernels are built from, both ways
static TSlice conv_slice(const cc_slice& s) { return nhwc_slice(s.p, s.cs, s.co, s.C, s.f32, s.N, s.H, s.W); }

static cc_slice op_slice(const TSlice& t, int N, int H, int W) {
  cc_slice s{};
  s.p = t.p; s.cs = t.cs; s.co = t.co; s.C = t.C; s.N = N; s.H = H; s.W = W; s.f32 = t.f32;
  return s;
}

namespace cc {

ConvDesc conv_desc_of(const cc_conv_op& o, ChainDesc* c) {
  const TSlice res = conv_slice(o.res);
  ConvDesc d = conv_desc(conv_slice(o.in), o.w, o.bias, o.k, o.stride, conv_slice(o.out), o.act, o.res.p ? &res : nullptr);
  d.slope = o.slope;
  d.bn_override = o.BN;
  d.out_ns = o.out_ns;
  d.pre = o.pre; d.pre_h = o.pre_h; d.pre_w = o.pre_w;
  *c = ChainDesc{};
  if (o.kind == CC_CONV_OP_CHAIN) {
    c->w = o.w2; c->bias = o.bias2; c->act = o.act2; c->k0 = o.k0;
    if (o.part.p) c->part = conv_slice(o.part);
    c->out = conv_slice(o.out2);
    c->store1 = o.store1 != 0;
  }
  return d;
}

cc_conv_op conv_op_of(const ConvDesc& d, const ChainDesc& c, const GemmLaunch& L) {
  const GemmParams& g = L.p;
  const int N = d.in.N, Ho = conv_out(d.in.H, d.stride), Wo = conv_out(d.in.W, d.stride);
  cc_conv_op o{};
  o.kind = c.out.p ? CC_CONV_OP_CHAIN : CC_CONV_OP_GEMM;
  o.in = op_slice(d.in, N, d.in.H, d.in.W);
  o.out = op_slice(d.out, N, Ho, Wo);
  if (d.res.p) o.res = op_slice(d.res, N, Ho, Wo);
  o.w = d.w; o.bias = d.bias; o.k = d.k; o.stride = d.stride; o.groups = 1; o.act = d.act; o.slope = d.slope;
  o.pre = d.pre; o.pre_h = d.pre_h; o.pre_w = d.pre_w;
  o.out_ns = d.out_ns;
  if (c.out.p) {
    o.w2 = c.w; o.bias2 = c.bias; o.act2 = c.act; o.k0 = c.k0;
    if (c.part.p) o.part = op_slice(c.part, N, Ho, Wo);
    o.out2 = op_slice(c.out, N, Ho, Wo);
    o.store1 = c.store1 ? 1 : 0;
  }
  o.BN = g.BN; o.BK = g.BK; o.lTW = g.lTW; o.lTH = g.lTH; o.lTN = g.lTN; o.s2 = g.s2; o.stages = g.stages; o.b_res = g.b_res;
  o.grid = L.grid; o.num_tiles = g.num_tiles; o.BNn = g.BNn; o.narrow_tiles = g.num_tiles - g.num_wide;
  return o;
}

cc_conv_op conv_op_of(const DirectConvParams& p) {
  cc_conv_op o{};
  o.kind = CC_CONV_OP_DIRECT;
  o.in = op_slice(nhwc_slice(p.in, p.in_cs, p.in_co, p.Cin), p.N, p.Hin, p.Win);
  o.out = op_slice(nhwc_slice(p.out, p.out_cs, p.out_co, p.Cout, p.out_f32), p.N, p.Hout, p.Wout);
  if (p.res) o.res = op_slice(nhwc_slice(p.res, p.res_cs, p.res_co, p.Cout, p.out_f32), p.N, p.Hout, p.Wout);
  o.w = p.w; o.bias = p.bias; o.k = p.k; o.stride = p.stride; o.groups = p.groups; o.act = p.act;
  return o;
}

}  // namespace cc

extern "C" {

int cc_version(void) { return CC_ABI_VERSION; }
const char* cc_last_error(void) { return last_error(); }
int cc_device_check(void) {
  const int n = device_sm_count();
  if (n <= 0) set_error("no sm_90 (H100) CUDA device available");
  return n;
}

int cc_conv(const cc_conv_op* op, void* stream) {
  CC_REQUIRE(op != nullptr, "cc_conv: op is NULL");
  const cc_conv_op& o = *op;
  const bool chain = o.kind == CC_CONV_OP_CHAIN, direct = o.kind == CC_CONV_OP_DIRECT;
  CC_REQUIRE(o.kind == CC_CONV_OP_GEMM || chain || direct, "cc_conv: unknown kind %d (%d GEMM, %d CHAIN, %d DIRECT)", o.kind,
             CC_CONV_OP_GEMM, CC_CONV_OP_CHAIN, CC_CONV_OP_DIRECT);
  CC_REQUIRE(o.in.p != nullptr, "cc_conv: in.p is NULL");
  CC_REQUIRE(o.w != nullptr, "cc_conv: w is NULL");
  CC_REQUIRE(o.out.p != nullptr || (chain && !o.store1), "cc_conv: out.p is NULL (only a CHAIN with store1 = 0 drops its output)");
  CC_REQUIRE(!chain || (o.w2 && o.out2.p), "cc_conv: a CHAIN needs w2 and out2.p (w2=%p out2.p=%p)", o.w2, o.out2.p);
  CC_REQUIRE(o.in.N >= 1 && o.in.H >= 1 && o.in.W >= 1 && o.in.C >= 1 && o.out.C >= 1 && (o.k == 1 || o.k == 3) &&
             (o.stride == 1 || o.stride == 2),
             "cc_conv: bad shape N=%d H=%d W=%d Cin=%d Cout=%d k=%d stride=%d (k 1 or 3, stride 1 or 2)", o.in.N, o.in.H, o.in.W,
             o.in.C, o.out.C, o.k, o.stride);
  CC_REQUIRE(!o.in.f32 && (!o.res.p || o.res.f32 == o.out.f32), "cc_conv: in is bf16 and res has out's dtype (in.f32=%d res.f32=%d "
             "out.f32=%d)", o.in.f32, o.res.f32, o.out.f32);
  // pad = k/2 with k odd: the direct kernel's extent, and conv_out() of every shape the wgmma kernel takes
  const int N = o.in.N, Ho = (o.in.H - 1) / o.stride + 1, Wo = (o.in.W - 1) / o.stride + 1;
  const std::pair<const char*, const cc_slice*> outs[] = {{"out", &o.out}, {"res", &o.res}, {"part", &o.part}, {"out2", &o.out2}};
  for (const auto& [what, s] : outs) {
    if (!s->p) continue;
    CC_REQUIRE(s->N == N && s->H == Ho && s->W == Wo, "cc_conv: %s is %dx%dx%d, the output %dx%dx%d (N x H x W)", what, s->N, s->H,
               s->W, N, Ho, Wo);
    CC_REQUIRE(s->C > 0 && s->co >= 0 && s->co + s->C <= s->cs, "cc_conv: %s slice cs=%d co=%d C=%d outside its row", what, s->cs,
               s->co, s->C);
  }
  if (o.out_ns != 0) {
    CC_REQUIRE(o.kind == CC_CONV_OP_GEMM, "cc_conv: out_ns=%d needs kind GEMM, got %d", o.out_ns, o.kind);
    CC_REQUIRE(o.out_ns >= Ho * Wo, "cc_conv: out_ns=%d pixels per image is less than the output's %dx%d", o.out_ns, Ho, Wo);
  }
  if (o.pre) {
    CC_REQUIRE((reinterpret_cast<uintptr_t>(o.pre) & 15) == 0, "cc_conv: pre=%p must be 16-byte aligned", o.pre);
    CC_REQUIRE(Ho % 2 == 0 && Wo % 2 == 0, "cc_conv: the output %dx%d must have even sides (pre is its half-resolution map)", Ho, Wo);
    CC_REQUIRE(o.pre_h == Ho / 2 && o.pre_w == Wo / 2, "cc_conv: pre is %dx%d, the output's half resolution %dx%d", o.pre_h, o.pre_w,
               Ho / 2, Wo / 2);
  }
  if (o.act == CC_ACT_PRELU) {
    CC_REQUIRE(o.bias && o.slope, "cc_conv: CC_ACT_PRELU needs its [9][Cout] bias table and slope (bias=%p slope=%p)", o.bias, o.slope);
    CC_REQUIRE(!o.out.f32, "cc_conv: CC_ACT_PRELU writes bf16, got out.f32=%d", o.out.f32);
  }
  ChainDesc c;
  const ConvDesc d = conv_desc_of(o, &c);
  if (direct) {
    CC_REQUIRE(!o.pre && o.act != CC_ACT_PRELU && !o.out2.p, "cc_conv: the direct kernel takes no pre, PReLU or chained output "
               "(pre=%p act=%d out2.p=%p)", o.pre, o.act, o.out2.p);
  } else {
    CC_REQUIRE(o.groups == 1, "cc_conv: the wgmma kernel takes groups = 1, got %d", o.groups);
    CC_REQUIRE(conv_gemm_supported(d), "cc_conv: shape not supported by the wgmma conv (Cin=%d in_cs=%d in_co=%d Cout=%d k=%d "
               "stride=%d H=%d W=%d)", o.in.C, o.in.cs, o.in.co, o.out.C, o.k, o.stride, o.in.H, o.in.W);
  }
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_conv: no sm_90 (H100) device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (direct) return conv_direct_launch(direct_conv_params(d, o.groups), st);
  GemmLaunch L;
  if (int rc = chain ? conv_gemm_chain_build(d, c, sms, &L) : conv_gemm_build(d, sms, &L)) return rc;
  return conv_gemm_launch(L, st);
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
