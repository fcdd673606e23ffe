// CLIP (OpenCLIP ViT) image + text encoders as static op lists over the sm_90a kernels.
//
// Replaces in the reference: OpenCLIP.precompute_embedding (models/objects.py:94-133), encode_text (:145-186) and the
// weight container OpenCLIP.__init__ (:22-92).  Parametric in the architecture (the reference hard-codes
// ViT-L/14; BASELINE.json's metric names ViT-B/32).
//
// Data layout: the residual stream is fp32 [B*L, W] (kept in fp32 across all blocks so the final cosine does not
// depend on bf16 round-off accumulation); every GEMM operand is bf16 (LayerNorm writes bf16, the QKV / MLP-fc
// epilogues write bf16), the out-proj and MLP-proj GEMMs add the fp32 residual in their epilogue in place.
// Per block: LN -> QKV GEMM(+bias) -> attention -> out-proj GEMM(+bias,+residual) -> LN -> fc GEMM(+bias,+GELU-tanh)
// -> proj GEMM(+bias,+residual).  All GEMMs run on the wgmma kernel of conv_gemm.cu.
#include "clearcam_b200.h"
#include "cc_common.h"
#include "conv_gemm.cuh"
#include "ops.cuh"
#include "plan.h"

namespace cc {

struct Tower { int width, layers, heads, mlp, tokens; };
struct BlockW {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  __nv_bfloat16 *w_in, *w_out, *w_fc, *w_proj;
  float *b_in, *b_out, *b_fc, *b_proj;
};

struct ClipPlan {
  int B = 0; bool text = false;
  std::vector<PlanOp> ops;
  size_t alloc_bytes = 0;      // bytes of the handle's shared workspace this plan addresses
  double flops = 0;
};

struct ClipModel {
  cc_clip_config cfg{};
  Tower v{}, t{};
  int kpad = 0, sms = 0;
  DeviceWeights weights;
  // image tower
  __nv_bfloat16* patch_w = nullptr; float *cls = nullptr, *pos = nullptr, *lnpre_g = nullptr, *lnpre_b = nullptr,
                 *lnpost_g = nullptr, *lnpost_b = nullptr;
  __nv_bfloat16* projT = nullptr;
  std::vector<BlockW> vb, tb;
  // text tower
  float *tok = nullptr, *pos_t = nullptr, *lnf_g = nullptr, *lnf_b = nullptr;
  __nv_bfloat16* tprojT = nullptr;
  PlanCache<std::string, ClipPlan> plans{"clip"};   // activation workspace shared by all plans (size of the largest)

  // [rows][cols] fp32 -> bf16 [rows][cols_pad] (zero padded) ; transpose=true reads the source as [cols][rows]
  int up_bf16(const std::string& name, int rows, int cols, int cols_pad, bool transpose, __nv_bfloat16** d) {
    const float* h;
    int rc = weights.host.get(name, static_cast<long long>(rows) * cols, &h);
    if (rc) return rc;
    std::vector<__nv_bfloat16> w(static_cast<size_t>(rows) * cols_pad, __float2bfloat16_rn(0.f));
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < cols; ++c)
        w[static_cast<size_t>(r) * cols_pad + c] =
            __float2bfloat16_rn(transpose ? h[static_cast<size_t>(c) * rows + r] : h[static_cast<size_t>(r) * cols + c]);
    return weights.upload(w, d);
  }
  int load_blocks(const std::string& prefix, const Tower& tw, const char* outw, const char* outb, std::vector<BlockW>* dst) {
    const int W = tw.width, M = tw.mlp;
    for (int i = 0; i < tw.layers; ++i) {
      const std::string p = prefix + "." + std::to_string(i);
      BlockW b{};
      int rc = 0;
      if ((rc = weights.up_f32(p + ".ln_1.weight", W, &b.ln1_g))) return rc;
      if ((rc = weights.up_f32(p + ".ln_1.bias", W, &b.ln1_b))) return rc;
      if ((rc = weights.up_f32(p + ".ln_2.weight", W, &b.ln2_g))) return rc;
      if ((rc = weights.up_f32(p + ".ln_2.bias", W, &b.ln2_b))) return rc;
      if ((rc = up_bf16(p + ".in_proj_weight", 3 * W, W, W, false, &b.w_in))) return rc;
      if ((rc = weights.up_f32(p + ".in_proj_bias", 3 * W, &b.b_in))) return rc;
      if ((rc = up_bf16(p + outw, W, W, W, false, &b.w_out))) return rc;
      if ((rc = weights.up_f32(p + outb, W, &b.b_out))) return rc;
      if ((rc = up_bf16(p + ".mlp_c_fc.weight", M, W, W, false, &b.w_fc))) return rc;
      if ((rc = weights.up_f32(p + ".mlp_c_fc.bias", M, &b.b_fc))) return rc;
      if ((rc = up_bf16(p + ".mlp_c_proj.weight", W, M, M, false, &b.w_proj))) return rc;
      if ((rc = weights.up_f32(p + ".mlp_c_proj.bias", W, &b.b_proj))) return rc;
      dst->push_back(b);
    }
    return CC_OK;
  }
};

struct PlanBuilder {
  ClipModel& M; ClipPlan& P; int rc = CC_OK;
  Bump bump;                   // workspace carving; bump.dry = measuring pass (descriptors are not built)
  PlanBuilder(ClipModel& m, ClipPlan& p) : M(m), P(p) {}
  void* dalloc(size_t bytes) {
    if (rc) return nullptr;
    void* d = bump.take(bytes);
    P.alloc_bytes = bump.off;
    return d;
  }
  void push(PlanOp op) {
    P.flops += op.flops;
    P.ops.push_back(std::move(op));
  }
  // out[M,N] = act(A[M,K] . Wt[N,K]^T + bias) (+res)
  void gemm(const char* name, const __nv_bfloat16* A, int lda, int Mrows, int K, const __nv_bfloat16* Wt, const float* bias,
            int N, void* out, int ldc, bool f32, int act, const void* res, int n_img = 1, int rows_per_img = 0, int out_ns = 0) {
    if (rc) return;
    if (bump.dry) return;
    const TSlice o = nhwc_slice(out, ldc, 0, N, f32 ? 1 : 0), r = nhwc_slice(res, ldc, 0, N, f32 ? 1 : 0);
    ConvDesc d = conv_desc(nhwc_slice(A, lda, 0, K, 0, n_img, 1, rows_per_img ? rows_per_img : Mrows), Wt, bias, 1, 1, o, act, res ? &r : nullptr);
    d.out_ns = out_ns;
    GemmLaunch L;
    rc = conv_gemm_build(d, M.sms, &L);
    if (rc) return;
    push(gemm_op(name, d, ChainDesc{}, L));
  }
  // LayerNorm of `rows` fp32 rows of x (row_stride rows apart, or the rows row_idx names) into bf16; x is a stream of B images
  // of L rows
  void layernorm(const char* name, const float* x, __nv_bfloat16* out, const float* g, const float* b, int rows, int W,
                 long long row_stride, const int* row_idx, int B, int L) {
    const int per = rows / B;   // output rows per image
    cc_op_io io = op_io({row_idx || row_stride == 1 ? operand(x, CC_OP_F32, B, 1, L, W) : operand(x, CC_OP_F32, B, 1, 1, W, 0, 0, L),
                         operand(g, CC_OP_F32, 1, 1, 1, W), operand(b, CC_OP_F32, 1, 1, 1, W)},
                        {operand(out, CC_OP_BF16, B, 1, per, W)});
    if (row_idx) io.in[io.n_in++] = operand(row_idx, CC_OP_I32, B, 1, 1, 1);
    push(plan_op(name, "layernorm", io, [=](const PlanIO&, cudaStream_t st) {
      return layernorm_bf16_launch(x, out, g, b, rows, W, row_stride, row_idx, st);
    }));
  }
  // the embeddings, L2-normalised into the call's output rows
  void l2norm(const float* emb, int B, int D, float eps) {
    cc_op_io io = op_io({operand(emb, CC_OP_F32, B, 1, 1, D)}, {operand(nullptr, CC_OP_F32, B, 1, 1, D)});
    io.eps = eps;
    push(plan_op("l2norm", "l2norm", io, [=](const PlanIO& io, cudaStream_t st) {
      return l2norm_launch(emb, io.out, B, D, io.out_stride, eps, st);
    }));
  }
  void blocks(const Tower& tw, const std::vector<BlockW>& bw, int B, float* x, bool causal) {
    const int W = tw.width, L = tw.tokens, rows = B * L;
    __nv_bfloat16* h = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(rows) * W * 2));
    __nv_bfloat16* qkv = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(rows) * 3 * W * 2));
    __nv_bfloat16* ctx = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(rows) * W * 2));
    __nv_bfloat16* hid = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(rows) * tw.mlp * 2));
    __nv_bfloat16* vt = attention_tc_supported(L) ? static_cast<__nv_bfloat16*>(dalloc(attention_tc_workspace_bytes(B, L, tw.heads))) : nullptr;
    for (int i = 0; i < tw.layers && !rc; ++i) {
      const BlockW& b = bw[i];
      layernorm("ln_1", x, h, b.ln1_g, b.ln1_b, rows, W, 1, nullptr, B, L);
      gemm("qkv", h, W, rows, W, b.w_in, b.b_in, 3 * W, qkv, 3 * W, false, CC_ACT_NONE, nullptr);
      const int heads = tw.heads, c = causal ? 1 : 0;
      cc_op_io io = op_io({operand(qkv, CC_OP_BF16, B, 1, L, 3 * W)}, {operand(ctx, CC_OP_BF16, B, 1, L, W)});
      if (vt) io.out[io.n_out++] = operand(vt, CC_OP_BF16, B, heads * 64, (L + 63) / 64 * 64, 1);
      io.causal = c;
      push(plan_op("attention", "attention", io, [=](const PlanIO&, cudaStream_t st) {
        return vt ? attention_tc_launch(qkv, ctx, vt, B, L, heads, c, st) : attention_launch(qkv, ctx, B, L, heads, c, st);
      }, 4.0 * B * tw.heads * double(L) * L * 64));
      gemm("out_proj", ctx, W, rows, W, b.w_out, b.b_out, W, x, W, true, CC_ACT_NONE, x);
      layernorm("ln_2", x, h, b.ln2_g, b.ln2_b, rows, W, 1, nullptr, B, L);
      gemm("mlp_fc", h, W, rows, W, b.w_fc, b.b_fc, tw.mlp, hid, tw.mlp, false, CC_ACT_GELU_TANH, nullptr);
      gemm("mlp_proj", hid, tw.mlp, rows, tw.mlp, b.w_proj, b.b_proj, W, x, W, true, CC_ACT_NONE, x);
    }
  }
  int build_image(int B) {
    const Tower& tw = M.v;
    const int W = tw.width, L = tw.tokens, Pn = L - 1, S = M.cfg.image_size, p = M.cfg.patch, D = M.cfg.embed_dim;
    __nv_bfloat16* patches = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(B) * Pn * M.kpad * 2));
    float* x = static_cast<float*>(dalloc(static_cast<size_t>(B) * L * W * 4));
    const int kpad = M.kpad;
    cc_op_io pio = op_io({operand(nullptr, CC_OP_F32, B, 3 * S, S, 1)}, {operand(patches, CC_OP_BF16, B, 1, Pn, kpad)});
    pio.patch = p;
    push(plan_op("patchify", "patchify", pio, [=](const PlanIO& io, cudaStream_t st) {
      return patchify_launch(static_cast<const float*>(io.in), patches, B, S, p, kpad, st);
    }));
    // conv14x14/s14 (no bias) == GEMM over patches; rows land at token 1.. of each image (out_ns = L, +1 row offset)
    gemm("patch_embed", patches, M.kpad, B * Pn, M.kpad, M.patch_w, nullptr, W, x + W, W, true, CC_ACT_NONE, nullptr, B, Pn, L);
    const float *cls = M.cls, *pos = M.pos, *g = M.lnpre_g, *b = M.lnpre_b;
    const cc_op_io eio = op_io({operand(x, CC_OP_F32, B, 1, L, W), operand(cls, CC_OP_F32, 1, 1, 1, W), operand(pos, CC_OP_F32, 1, 1, L, W),
                                operand(g, CC_OP_F32, 1, 1, 1, W), operand(b, CC_OP_F32, 1, 1, 1, W)},
                               {operand(x, CC_OP_F32, B, 1, L, W)});
    push(plan_op("cls+pos+ln_pre", "embed_ln_pre", eio, [=](const PlanIO&, cudaStream_t st) {
      return embed_ln_pre_launch(x, cls, pos, g, b, B * L, L, W, st);
    }));
    blocks(tw, M.vb, B, x, false);
    __nv_bfloat16* pooled = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(B) * W * 2));
    float* emb = static_cast<float*>(dalloc(static_cast<size_t>(B) * D * 4));
    layernorm("ln_post(token 0)", x, pooled, M.lnpost_g, M.lnpost_b, B, W, L, nullptr, B, L);
    gemm("proj", pooled, W, B, W, M.projT, nullptr, D, emb, D, true, CC_ACT_NONE, nullptr);
    l2norm(emb, B, D, 1e-8f);
    return rc;
  }
  int build_text(int B) {
    const Tower& tw = M.t;
    const int W = tw.width, L = tw.tokens, D = M.cfg.embed_dim;
    float* x = static_cast<float*>(dalloc(static_cast<size_t>(B) * L * W * 4));
    int* eot = static_cast<int*>(dalloc(static_cast<size_t>(B) * 4));
    const float *tok = M.tok, *pos = M.pos_t;
    const int vocab = M.cfg.vocab;
    const cc_op_io tio = op_io({operand(nullptr, CC_OP_I32, B, 1, L, 1), operand(tok, CC_OP_F32, 1, 1, vocab, W), operand(pos, CC_OP_F32, 1, 1, L, W)},
                               {operand(x, CC_OP_F32, B, 1, L, W), operand(eot, CC_OP_I32, B, 1, 1, 1)});
    push(plan_op("tok+pos", "text_embed", tio, [=](const PlanIO& io, cudaStream_t st) {
      return text_embed_launch(static_cast<const int*>(io.in), tok, pos, x, eot, B, L, W, vocab, st);
    }));
    blocks(tw, M.tb, B, x, true);
    __nv_bfloat16* pooled = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(B) * W * 2));
    float* emb = static_cast<float*>(dalloc(static_cast<size_t>(B) * D * 4));
    layernorm("ln_final(EOT row)", x, pooled, M.lnf_g, M.lnf_b, B, W, 0, eot, B, L);
    gemm("text_projection", pooled, W, B, W, M.tprojT, nullptr, D, emb, D, true, CC_ACT_NONE, nullptr);
    l2norm(emb, B, D, 0.f);
    return rc;
  }
};

}  // namespace cc

using namespace cc;

struct cc_clip { ClipModel m; };

extern "C" {

int cc_clip_create(const cc_clip_config* cfg, int n_tensors, const char* const* names, const float* const* h_data,
                   const int64_t* numels, cc_clip** out) {
  CC_REQUIRE(cfg && out, "cc_clip_create: null argument");
  // the configuration first: a CPU-only caller sees the same refusal
  CC_REQUIRE(cfg->patch >= 1 && cfg->image_size >= cfg->patch && cfg->image_size % cfg->patch == 0 && cfg->v_layers >= 0 &&
                 cfg->t_layers >= 0 && cfg->v_width == cfg->v_heads * 64 && cfg->t_width == cfg->t_heads * 64 &&
                 cfg->embed_dim >= 16 && cfg->embed_dim % 16 == 0 && cfg->v_mlp >= 16 && cfg->v_mlp % 16 == 0 &&
                 cfg->t_mlp >= 16 && cfg->t_mlp % 16 == 0 && cfg->vocab >= 1 && cfg->ctx >= 1,
             "cc_clip_create: unsupported architecture (need width = 64*heads, image size a multiple of the patch)");
  CC_REQUIRE(layernorm_width_supported(cfg->v_width) && layernorm_width_supported(cfg->t_width),
             "cc_clip_create: widths %d / %d not supported by the LayerNorm kernels (128 x 1, 2, 3, 4, 5, 6, 8, 10 or 12)",
             cfg->v_width, cfg->t_width);
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_clip_create: no sm_90 (H100) device");
  std::unique_ptr<cc_clip> h(new cc_clip());
  ClipModel& M = h->m;
  M.cfg = *cfg; M.sms = sms;
  const int G = cfg->image_size / cfg->patch;
  M.v = Tower{cfg->v_width, cfg->v_layers, cfg->v_heads, cfg->v_mlp, 1 + G * G};
  M.t = Tower{cfg->t_width, cfg->t_layers, cfg->t_heads, cfg->t_mlp, cfg->ctx};
  const int K = 3 * cfg->patch * cfg->patch;
  M.kpad = (K + 63) / 64 * 64;
  const int W = M.v.width, Wt = M.t.width, D = cfg->embed_dim;
  int rc = 0;
  if ((rc = M.weights.host.fill("cc_clip_create", n_tensors, names, h_data, numels))) return rc;
  if ((rc = M.up_bf16("visual_conv1.weight", W, K, M.kpad, false, &M.patch_w))) return rc;
  if ((rc = M.weights.up_f32("class_embedding", W, &M.cls))) return rc;
  if ((rc = M.weights.up_f32("positional_embedding", static_cast<long long>(M.v.tokens) * W, &M.pos))) return rc;
  if ((rc = M.weights.up_f32("ln_pre.weight", W, &M.lnpre_g))) return rc;
  if ((rc = M.weights.up_f32("ln_pre.bias", W, &M.lnpre_b))) return rc;
  if ((rc = M.weights.up_f32("ln_post.weight", W, &M.lnpost_g))) return rc;
  if ((rc = M.weights.up_f32("ln_post.bias", W, &M.lnpost_b))) return rc;
  if ((rc = M.up_bf16("proj", D, W, W, true, &M.projT))) return rc;          // stored (W, D) -> [D][W]
  if ((rc = M.load_blocks("resblocks_img", M.v, ".out_proj_weight", ".out_proj_bias", &M.vb))) return rc;
  if ((rc = M.weights.up_f32("token_embedding.weight", static_cast<long long>(cfg->vocab) * Wt, &M.tok))) return rc;
  if ((rc = M.weights.up_f32("positional_embedding_text", static_cast<long long>(cfg->ctx) * Wt, &M.pos_t))) return rc;
  if ((rc = M.weights.up_f32("ln_final.weight", Wt, &M.lnf_g))) return rc;
  if ((rc = M.weights.up_f32("ln_final.bias", Wt, &M.lnf_b))) return rc;
  if ((rc = M.up_bf16("text_projection", D, Wt, Wt, true, &M.tprojT))) return rc;
  if ((rc = M.load_blocks("resblocks", M.t, ".attn_out_proj_weight", ".attn_out_proj_bias", &M.tb))) return rc;
  M.weights.host.clear();
  *out = h.release();
  return CC_OK;
}

int cc_clip_destroy(cc_clip* h) {
  delete h;
  return CC_OK;
}

static int clip_plan_bytes(cc_clip* h, bool text, int B, size_t* bytes) {
  ClipPlan tmp;
  tmp.B = B; tmp.text = text;
  PlanBuilder dry(h->m, tmp);
  dry.bump.dry = true;
  int rc = text ? dry.build_text(B) : dry.build_image(B);
  if (rc) return rc;
  *bytes = dry.bump.off + 1024;
  return CC_OK;
}
static int clip_plan(cc_clip* h, bool text, int B, ClipPlan** out) {
  return h->m.plans.get(
      std::string(text ? "t" : "i") + std::to_string(B), [&](size_t* bytes) { return clip_plan_bytes(h, text, B, bytes); },
      [&](ClipPlan& P, uint8_t* base, size_t* used) {
        P.B = B; P.text = text;
        PlanBuilder b(h->m, P);
        b.bump.base = base;
        const int rc = text ? b.build_text(B) : b.build_image(B);
        *used = b.bump.off;
        return rc;
      },
      out);
}

int cc_clip_workspace_bytes(cc_clip* h, int text, int B, size_t* bytes) {
  CC_REQUIRE(h && bytes && B > 0, "cc_clip_workspace_bytes: bad argument");
  return clip_plan_bytes(h, text != 0, B, bytes);
}

int cc_clip_set_workspace(cc_clip* h, void* d_workspace, size_t bytes) {
  if (int rc = check_workspace("cc_clip_set_workspace", h, d_workspace)) return rc;
  return h->m.plans.adopt(d_workspace, bytes);
}

int cc_clip_encode_image(cc_clip* h, const float* d_x, int B, float* d_out, long long out_row_stride, void* stream) {
  CC_REQUIRE(h && d_x && d_out && B > 0, "cc_clip_encode_image: bad argument");
  ClipPlan* P = nullptr;
  int rc = clip_plan(h, false, B, &P);
  if (rc) return rc;
  return run_ops(P->ops, PlanIO{d_x, d_out, out_row_stride > 0 ? out_row_stride : h->m.cfg.embed_dim}, static_cast<cudaStream_t>(stream));
}

int cc_clip_encode_text(cc_clip* h, const int32_t* d_ids, int B, float* d_out, long long out_row_stride, void* stream) {
  CC_REQUIRE(h && d_ids && d_out && B > 0, "cc_clip_encode_text: bad argument");
  ClipPlan* P = nullptr;
  int rc = clip_plan(h, true, B, &P);
  if (rc) return rc;
  return run_ops(P->ops, PlanIO{d_ids, d_out, out_row_stride > 0 ? out_row_stride : h->m.cfg.embed_dim}, static_cast<cudaStream_t>(stream));
}

int cc_clip_profile(cc_clip* h, int text, const void* d_in, int B, float* d_out, int cap, float* ms, double* flops,
                    const char** names, int* n_ops, double* total_flops, void* stream) {
  CC_REQUIRE(h && d_in && d_out, "cc_clip_profile: bad argument");
  ClipPlan* P = nullptr;
  int rc = clip_plan(h, text != 0, B, &P);
  if (rc) return rc;
  rc = profile_ops(P->ops, PlanIO{d_in, d_out, h->m.cfg.embed_dim}, static_cast<cudaStream_t>(stream), cap, ms, flops, nullptr, nullptr,
                   names);
  if (n_ops) *n_ops = static_cast<int>(P->ops.size());
  if (total_flops) *total_flops = P->flops;
  return rc;
}

// conv op taps: what each GEMM launch of the cached plan computes, and the plan run one range of ops at a time
int cc_clip_op_conv(cc_clip* h, int text, int B, int i, cc_conv_op* out) {
  CC_REQUIRE(h && B > 0, "cc_clip_op_conv: bad argument");
  ClipPlan* P = nullptr;
  if (int rc = clip_plan(h, text != 0, B, &P)) return rc;
  return op_conv_tap("cc_clip_op_conv", P->ops, i, out);
}

int cc_clip_op_io(cc_clip* h, int text, int B, int i, cc_op_io* out) {
  CC_REQUIRE(h && B > 0, "cc_clip_op_io: bad argument");
  ClipPlan* P = nullptr;
  if (int rc = clip_plan(h, text != 0, B, &P)) return rc;
  return op_io_tap("cc_clip_op_io", P->ops, i, out);
}

int cc_clip_run_ops(cc_clip* h, int text, const void* d_in, int B, int first, int last, float* d_out, long long out_row_stride,
                    void* stream) {
  CC_REQUIRE(h && d_in && d_out && B > 0, "cc_clip_run_ops: bad argument");
  ClipPlan* P = nullptr;
  if (int rc = clip_plan(h, text != 0, B, &P)) return rc;
  if (int rc = check_range("cc_clip_run_ops", first, last, static_cast<int>(P->ops.size()))) return rc;
  return run_ops(P->ops, PlanIO{d_in, d_out, out_row_stride > 0 ? out_row_stride : h->m.cfg.embed_dim}, static_cast<cudaStream_t>(stream),
                 first, last);
}

int cc_search_scores(const float* d_index, int N, int D, const float* d_q, int Q, float* d_scores, void* stream) {
  CC_REQUIRE(d_index && d_q && d_scores && N >= 0 && D > 0 && Q > 0, "cc_search_scores: bad argument");
  return search_scores_launch(d_index, d_q, d_scores, N, D, Q, static_cast<cudaStream_t>(stream));
}

int cc_search_topk(const float* d_index, int N, int D, const float* d_q, const int32_t* d_group, const uint8_t* d_mask, int G, int k,
                   void* d_workspace, int32_t* d_rows, float* d_scores, void* stream) {
  CC_REQUIRE(d_index && d_q && d_group && d_workspace && d_rows && d_scores && N >= 0 && D > 0 && G >= 0 && k > 0,
             "cc_search_topk: bad argument");
  return search_topk_launch(d_index, d_q, d_group, d_mask, static_cast<unsigned long long*>(d_workspace), N, D, G, k, d_rows, d_scores,
                            static_cast<cudaStream_t>(stream));
}

}  // extern "C"
