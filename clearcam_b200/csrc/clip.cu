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
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace cc {

struct Tower { int width, layers, heads, mlp, tokens; };
struct BlockW {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  __nv_bfloat16 *w_in, *w_out, *w_fc, *w_proj;
  float *b_in, *b_out, *b_fc, *b_proj;
};

struct VOp {
  enum Kind { PATCHIFY, GEMM, EMBED_LN, LN, ATTN, TEXT_EMBED, L2NORM } kind;
  GemmLaunch gemm;
  // generic slots
  const float* f0 = nullptr; const float* f1 = nullptr; const float* f2 = nullptr; const float* f3 = nullptr;
  float* fo = nullptr;
  __nv_bfloat16* bo = nullptr; const __nv_bfloat16* bi = nullptr; __nv_bfloat16* bw = nullptr;
  const int* idx = nullptr; int* io = nullptr;
  int i0 = 0, i1 = 0, i2 = 0, i3 = 0, i4 = 0;
  long long l0 = 0;
  float eps = 0.f;
  const char* name = "";
  double flops = 0;
};

struct ClipPlan {
  int B = 0; bool text = false;
  std::vector<VOp> ops;
  size_t alloc_bytes = 0;      // bytes of the handle's shared workspace this plan addresses
  uint64_t gen = 0, last_use = 0;
  double flops = 0;
};

struct ClipModel {
  cc_clip_config cfg{};
  Tower v{}, t{};
  int kpad = 0, sms = 0;
  std::map<std::string, std::pair<const float*, long long>> host;
  std::vector<void*> allocs;
  // image tower
  __nv_bfloat16* patch_w = nullptr; float *cls = nullptr, *pos = nullptr, *lnpre_g = nullptr, *lnpre_b = nullptr,
                 *lnpost_g = nullptr, *lnpost_b = nullptr;
  __nv_bfloat16* projT = nullptr;
  std::vector<BlockW> vb, tb;
  // text tower
  float *tok = nullptr, *pos_t = nullptr, *lnf_g = nullptr, *lnf_b = nullptr;
  __nv_bfloat16* tprojT = nullptr;
  std::map<std::string, std::unique_ptr<ClipPlan>> plans;   // bounded, least recently used goes first
  Arena arena;                 // activation workspace shared by all plans (size of the largest)
  uint64_t tick = 0;
  ~ClipModel() { plans.clear(); for (void* p : allocs) cudaFree(p); }

  int get(const std::string& name, long long n, const float** out) {
    auto it = host.find(name);
    CC_REQUIRE(it != host.end(), "clip: missing weight '%s'", name.c_str());
    CC_REQUIRE(it->second.second == n, "clip: '%s' has %lld elements, expected %lld", name.c_str(), it->second.second, n);
    *out = it->second.first;
    return CC_OK;
  }
  int up(const void* h, size_t bytes, void** d) {
    CC_CHECK_CUDA(cudaMalloc(d, bytes));
    allocs.push_back(*d);
    CC_CHECK_CUDA(cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice));
    return CC_OK;
  }
  int up_f32(const std::string& name, long long n, float** d) {
    const float* h;
    int rc = get(name, n, &h);
    if (rc) return rc;
    return up(h, n * 4, reinterpret_cast<void**>(d));
  }
  // [rows][cols] fp32 -> bf16 [rows][cols_pad] (zero padded) ; transpose=true reads the source as [cols][rows]
  int up_bf16(const std::string& name, int rows, int cols, int cols_pad, bool transpose, __nv_bfloat16** d) {
    const float* h;
    int rc = get(name, static_cast<long long>(rows) * cols, &h);
    if (rc) return rc;
    std::vector<__nv_bfloat16> w(static_cast<size_t>(rows) * cols_pad, __float2bfloat16_rn(0.f));
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < cols; ++c)
        w[static_cast<size_t>(r) * cols_pad + c] =
            __float2bfloat16_rn(transpose ? h[static_cast<size_t>(c) * rows + r] : h[static_cast<size_t>(r) * cols + c]);
    return up(w.data(), w.size() * 2, reinterpret_cast<void**>(d));
  }
  int load_blocks(const std::string& prefix, const Tower& tw, const char* outw, const char* outb, std::vector<BlockW>* dst) {
    const int W = tw.width, M = tw.mlp;
    for (int i = 0; i < tw.layers; ++i) {
      const std::string p = prefix + "." + std::to_string(i);
      BlockW b{};
      int rc = 0;
      if ((rc = up_f32(p + ".ln_1.weight", W, &b.ln1_g))) return rc;
      if ((rc = up_f32(p + ".ln_1.bias", W, &b.ln1_b))) return rc;
      if ((rc = up_f32(p + ".ln_2.weight", W, &b.ln2_g))) return rc;
      if ((rc = up_f32(p + ".ln_2.bias", W, &b.ln2_b))) return rc;
      if ((rc = up_bf16(p + ".in_proj_weight", 3 * W, W, W, false, &b.w_in))) return rc;
      if ((rc = up_f32(p + ".in_proj_bias", 3 * W, &b.b_in))) return rc;
      if ((rc = up_bf16(p + outw, W, W, W, false, &b.w_out))) return rc;
      if ((rc = up_f32(p + outb, W, &b.b_out))) return rc;
      if ((rc = up_bf16(p + ".mlp_c_fc.weight", M, W, W, false, &b.w_fc))) return rc;
      if ((rc = up_f32(p + ".mlp_c_fc.bias", M, &b.b_fc))) return rc;
      if ((rc = up_bf16(p + ".mlp_c_proj.weight", W, M, M, false, &b.w_proj))) return rc;
      if ((rc = up_f32(p + ".mlp_c_proj.bias", W, &b.b_proj))) return rc;
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
  // out[M,N] = act(A[M,K] . Wt[N,K]^T + bias) (+res)
  void gemm(const char* name, const __nv_bfloat16* A, int lda, int Mrows, int K, const __nv_bfloat16* Wt, const float* bias,
            int N, void* out, int ldc, bool f32, int act, const void* res, int n_img = 1, int rows_per_img = 0, int out_ns = 0) {
    if (rc) return;
    ConvDesc d{};
    d.in = A; d.in_cs = lda; d.in_co = 0; d.Cin = K;
    d.N = n_img; d.Hin = 1; d.Win = rows_per_img ? rows_per_img : Mrows;
    d.k = 1; d.stride = 1; d.w = Wt; d.bias = bias;
    d.out = out; d.out_cs = ldc; d.out_co = 0; d.Cout = N; d.out_f32 = f32 ? 1 : 0; d.act = act;
    d.res = res; d.res_cs = ldc; d.res_co = 0; d.out_ns = out_ns;
    if (bump.dry) return;
    VOp op; op.kind = VOp::GEMM; op.name = name;
    rc = conv_gemm_build(d, M.sms, &op.gemm);
    if (rc) return;
    op.flops = op.gemm.flops;
    P.flops += op.flops;
    P.ops.push_back(op);
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
      { VOp op; op.kind = VOp::LN; op.name = "ln_1"; op.f0 = x; op.bo = h; op.f1 = b.ln1_g; op.f2 = b.ln1_b; op.i0 = rows; op.i1 = W; op.l0 = 1; P.ops.push_back(op); }
      gemm("qkv", h, W, rows, W, b.w_in, b.b_in, 3 * W, qkv, 3 * W, false, CC_ACT_NONE, nullptr);
      { VOp op; op.kind = VOp::ATTN; op.name = "attention"; op.bi = qkv; op.bo = ctx; op.bw = vt; op.i0 = B; op.i1 = L; op.i2 = tw.heads; op.i3 = causal ? 1 : 0;
        op.flops = 4.0 * B * tw.heads * double(L) * L * 64; P.flops += op.flops; P.ops.push_back(op); }
      gemm("out_proj", ctx, W, rows, W, b.w_out, b.b_out, W, x, W, true, CC_ACT_NONE, x);
      { VOp op; op.kind = VOp::LN; op.name = "ln_2"; op.f0 = x; op.bo = h; op.f1 = b.ln2_g; op.f2 = b.ln2_b; op.i0 = rows; op.i1 = W; op.l0 = 1; P.ops.push_back(op); }
      gemm("mlp_fc", h, W, rows, W, b.w_fc, b.b_fc, tw.mlp, hid, tw.mlp, false, CC_ACT_GELU_TANH, nullptr);
      gemm("mlp_proj", hid, tw.mlp, rows, tw.mlp, b.w_proj, b.b_proj, W, x, W, true, CC_ACT_NONE, x);
    }
  }
  int build_image(int B) {
    const Tower& tw = M.v;
    const int W = tw.width, L = tw.tokens, Pn = L - 1, S = M.cfg.image_size, p = M.cfg.patch, D = M.cfg.embed_dim;
    __nv_bfloat16* patches = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(B) * Pn * M.kpad * 2));
    float* x = static_cast<float*>(dalloc(static_cast<size_t>(B) * L * W * 4));
    { VOp op; op.kind = VOp::PATCHIFY; op.name = "patchify"; op.bo = patches; op.i0 = B; op.i1 = S; op.i2 = p; op.i3 = M.kpad; P.ops.push_back(op); }
    // conv14x14/s14 (no bias) == GEMM over patches; rows land at token 1.. of each image (out_ns = L, +1 row offset)
    gemm("patch_embed", patches, M.kpad, B * Pn, M.kpad, M.patch_w, nullptr, W, x + W, W, true, CC_ACT_NONE, nullptr, B, Pn, L);
    { VOp op; op.kind = VOp::EMBED_LN; op.name = "cls+pos+ln_pre"; op.fo = x; op.f0 = M.cls; op.f1 = M.pos; op.f2 = M.lnpre_g; op.f3 = M.lnpre_b;
      op.i0 = B * L; op.i1 = L; op.i2 = W; P.ops.push_back(op); }
    blocks(tw, M.vb, B, x, false);
    __nv_bfloat16* pooled = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(B) * W * 2));
    float* emb = static_cast<float*>(dalloc(static_cast<size_t>(B) * D * 4));
    { VOp op; op.kind = VOp::LN; op.name = "ln_post(token 0)"; op.f0 = x; op.bo = pooled; op.f1 = M.lnpost_g; op.f2 = M.lnpost_b; op.i0 = B; op.i1 = W; op.l0 = L; P.ops.push_back(op); }
    gemm("proj", pooled, W, B, W, M.projT, nullptr, D, emb, D, true, CC_ACT_NONE, nullptr);
    { VOp op; op.kind = VOp::L2NORM; op.name = "l2norm"; op.f0 = emb; op.i0 = B; op.i1 = D; op.eps = 1e-8f; P.ops.push_back(op); }
    return rc;
  }
  int build_text(int B) {
    const Tower& tw = M.t;
    const int W = tw.width, L = tw.tokens, D = M.cfg.embed_dim;
    float* x = static_cast<float*>(dalloc(static_cast<size_t>(B) * L * W * 4));
    int* eot = static_cast<int*>(dalloc(static_cast<size_t>(B) * 4));
    { VOp op; op.kind = VOp::TEXT_EMBED; op.name = "tok+pos"; op.f0 = M.tok; op.f1 = M.pos_t; op.fo = x; op.io = eot; op.i0 = B; op.i1 = L; op.i2 = W; op.i3 = M.cfg.vocab; P.ops.push_back(op); }
    blocks(tw, M.tb, B, x, true);
    __nv_bfloat16* pooled = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(B) * W * 2));
    float* emb = static_cast<float*>(dalloc(static_cast<size_t>(B) * D * 4));
    { VOp op; op.kind = VOp::LN; op.name = "ln_final(EOT row)"; op.f0 = x; op.bo = pooled; op.f1 = M.lnf_g; op.f2 = M.lnf_b; op.i0 = B; op.i1 = W; op.idx = eot; P.ops.push_back(op); }
    gemm("text_projection", pooled, W, B, W, M.tprojT, nullptr, D, emb, D, true, CC_ACT_NONE, nullptr);
    { VOp op; op.kind = VOp::L2NORM; op.name = "l2norm"; op.f0 = emb; op.i0 = B; op.i1 = D; op.eps = 0.f; P.ops.push_back(op); }
    return rc;
  }
};

static int run_plan(ClipPlan& P, const void* d_in, float* d_out, long long out_stride, cudaStream_t st,
                    std::vector<cudaEvent_t>* ev = nullptr) {
  size_t oi = 0;
  for (VOp& op : P.ops) {
    int rc = CC_OK;
    if (ev) cudaEventRecord((*ev)[oi++], st);
    switch (op.kind) {
      case VOp::PATCHIFY: rc = patchify_launch(static_cast<const float*>(d_in), op.bo, op.i0, op.i1, op.i2, op.i3, st); break;
      case VOp::GEMM: rc = conv_gemm_launch(op.gemm, st); break;
      case VOp::EMBED_LN: rc = embed_ln_pre_launch(op.fo, op.f0, op.f1, op.f2, op.f3, op.i0, op.i1, op.i2, st); break;
      case VOp::LN: rc = layernorm_bf16_launch(op.f0, op.bo, op.f1, op.f2, op.i0, op.i1, op.l0, op.idx, st); break;
      case VOp::ATTN:
        rc = op.bw ? attention_tc_launch(op.bi, op.bo, op.bw, op.i0, op.i1, op.i2, op.i3, st)
                   : attention_launch(op.bi, op.bo, op.i0, op.i1, op.i2, op.i3, st);
        break;
      case VOp::TEXT_EMBED: rc = text_embed_launch(static_cast<const int*>(d_in), op.f0, op.f1, op.fo, op.io, op.i0, op.i1, op.i2, op.i3, st); break;
      case VOp::L2NORM: rc = l2norm_launch(op.f0, d_out, op.i0, op.i1, out_stride, op.eps, st); break;
    }
    if (rc) return rc;
  }
  if (ev) cudaEventRecord((*ev)[oi], st);
  return CC_OK;
}

}  // namespace cc

using namespace cc;

struct cc_clip { ClipModel m; };

extern "C" {

int cc_clip_create(const cc_clip_config* cfg, int n_tensors, const char* const* names, const float* const* h_data,
                   const int64_t* numels, cc_clip** out) {
  CC_REQUIRE(cfg && out, "cc_clip_create: null argument");
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_clip_create: no sm_90 (H100) device");
  CC_REQUIRE(cfg->image_size % cfg->patch == 0 && cfg->v_width % 128 == 0 && cfg->t_width % 128 == 0 &&
                 cfg->v_width == cfg->v_heads * 64 && cfg->t_width == cfg->t_heads * 64 && cfg->embed_dim % 16 == 0 &&
                 cfg->v_mlp % 16 == 0 && cfg->t_mlp % 16 == 0,
             "cc_clip_create: unsupported architecture (need width = 64*heads, widths multiple of 128)");
  std::unique_ptr<cc_clip> h(new cc_clip());
  ClipModel& M = h->m;
  M.cfg = *cfg; M.sms = sms;
  const int G = cfg->image_size / cfg->patch;
  M.v = Tower{cfg->v_width, cfg->v_layers, cfg->v_heads, cfg->v_mlp, 1 + G * G};
  M.t = Tower{cfg->t_width, cfg->t_layers, cfg->t_heads, cfg->t_mlp, cfg->ctx};
  const int K = 3 * cfg->patch * cfg->patch;
  M.kpad = (K + 63) / 64 * 64;
  for (int i = 0; i < n_tensors; ++i) M.host[names[i]] = {h_data[i], static_cast<long long>(numels[i])};
  const int W = M.v.width, Wt = M.t.width, D = cfg->embed_dim;
  int rc = 0;
  if ((rc = M.up_bf16("visual_conv1.weight", W, K, M.kpad, false, &M.patch_w))) return rc;
  if ((rc = M.up_f32("class_embedding", W, &M.cls))) return rc;
  if ((rc = M.up_f32("positional_embedding", static_cast<long long>(M.v.tokens) * W, &M.pos))) return rc;
  if ((rc = M.up_f32("ln_pre.weight", W, &M.lnpre_g))) return rc;
  if ((rc = M.up_f32("ln_pre.bias", W, &M.lnpre_b))) return rc;
  if ((rc = M.up_f32("ln_post.weight", W, &M.lnpost_g))) return rc;
  if ((rc = M.up_f32("ln_post.bias", W, &M.lnpost_b))) return rc;
  if ((rc = M.up_bf16("proj", D, W, W, true, &M.projT))) return rc;          // stored (W, D) -> [D][W]
  if ((rc = M.load_blocks("resblocks_img", M.v, ".out_proj_weight", ".out_proj_bias", &M.vb))) return rc;
  if ((rc = M.up_f32("token_embedding.weight", static_cast<long long>(cfg->vocab) * Wt, &M.tok))) return rc;
  if ((rc = M.up_f32("positional_embedding_text", static_cast<long long>(cfg->ctx) * Wt, &M.pos_t))) return rc;
  if ((rc = M.up_f32("ln_final.weight", Wt, &M.lnf_g))) return rc;
  if ((rc = M.up_f32("ln_final.bias", Wt, &M.lnf_b))) return rc;
  if ((rc = M.up_bf16("text_projection", D, Wt, Wt, true, &M.tprojT))) return rc;
  if ((rc = M.load_blocks("resblocks", M.t, ".attn_out_proj_weight", ".attn_out_proj_bias", &M.tb))) return rc;
  M.host.clear();
  *out = h.release();
  return CC_OK;
}

int cc_clip_destroy(cc_clip* h) {
  delete h;
  return CC_OK;
}

static constexpr size_t kMaxClipPlans = 16;

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
  ClipModel& M = h->m;
  const std::string key = std::string(text ? "t" : "i") + std::to_string(B);
  auto it = M.plans.find(key);
  if (it != M.plans.end() && it->second->gen == M.arena.gen) {
    it->second->last_use = ++M.tick;
    *out = it->second.get();
    return CC_OK;
  }
  size_t bytes = 0;
  int rc = clip_plan_bytes(h, text, B, &bytes);
  if (rc) return rc;
  if ((rc = M.arena.reserve(bytes))) return rc;
  for (auto p = M.plans.begin(); p != M.plans.end();)
    p = (p->second->gen != M.arena.gen) ? M.plans.erase(p) : std::next(p);
  std::unique_ptr<ClipPlan> P(new ClipPlan());
  P->B = B; P->text = text;
  PlanBuilder b(M, *P);
  b.bump.base = static_cast<uint8_t*>(M.arena.base);
  rc = text ? b.build_text(B) : b.build_image(B);
  if (rc) return rc;
  CC_REQUIRE(b.bump.off <= M.arena.cap, "clip plan: workspace overrun (%zu > %zu)", b.bump.off, M.arena.cap);
  P->gen = M.arena.gen;
  P->last_use = ++M.tick;
  if (M.plans.size() >= kMaxClipPlans) {
    auto lru = M.plans.begin();
    for (auto p = M.plans.begin(); p != M.plans.end(); ++p)
      if (p->second->last_use < lru->second->last_use) lru = p;
    M.plans.erase(lru);
  }
  *out = (M.plans[key] = std::move(P)).get();
  return CC_OK;
}

int cc_clip_workspace_bytes(cc_clip* h, int text, int B, size_t* bytes) {
  CC_REQUIRE(h && bytes && B > 0, "cc_clip_workspace_bytes: bad argument");
  return clip_plan_bytes(h, text != 0, B, bytes);
}

int cc_clip_set_workspace(cc_clip* h, void* d_workspace, size_t bytes) {
  CC_REQUIRE(h, "cc_clip_set_workspace: null handle");
  CC_REQUIRE(d_workspace == nullptr || (reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0,
             "cc_clip_set_workspace: the workspace must be 256-byte aligned");
  h->m.plans.clear();
  return h->m.arena.adopt(d_workspace, bytes);
}

int cc_clip_encode_image(cc_clip* h, const float* d_x, int B, float* d_out, long long out_row_stride, void* stream) {
  CC_REQUIRE(h && d_x && d_out && B > 0, "cc_clip_encode_image: bad argument");
  ClipPlan* P = nullptr;
  int rc = clip_plan(h, false, B, &P);
  if (rc) return rc;
  return run_plan(*P, d_x, d_out, out_row_stride > 0 ? out_row_stride : h->m.cfg.embed_dim, static_cast<cudaStream_t>(stream));
}

int cc_clip_encode_text(cc_clip* h, const int32_t* d_ids, int B, float* d_out, long long out_row_stride, void* stream) {
  CC_REQUIRE(h && d_ids && d_out && B > 0, "cc_clip_encode_text: bad argument");
  ClipPlan* P = nullptr;
  int rc = clip_plan(h, true, B, &P);
  if (rc) return rc;
  return run_plan(*P, d_ids, d_out, out_row_stride > 0 ? out_row_stride : h->m.cfg.embed_dim, static_cast<cudaStream_t>(stream));
}

int cc_clip_profile(cc_clip* h, int text, const void* d_in, int B, float* d_out, int cap, float* ms, double* flops,
                    const char** names, int* n_ops, double* total_flops, void* stream) {
  CC_REQUIRE(h && d_in && d_out, "cc_clip_profile: bad argument");
  ClipPlan* P = nullptr;
  int rc = clip_plan(h, text != 0, B, &P);
  if (rc) return rc;
  const size_t n = P->ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) CC_CHECK_CUDA(cudaEventCreate(&e));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = run_plan(*P, d_in, d_out, h->m.cfg.embed_dim, st, &ev);
  if (!rc) {
    CC_CHECK_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n && static_cast<int>(i) < cap; ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, ev[i], ev[i + 1]);
      if (ms) ms[i] = t;
      if (flops) flops[i] = P->ops[i].flops;
      if (names) names[i] = P->ops[i].name;
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  if (n_ops) *n_ops = static_cast<int>(n);
  if (total_flops) *total_flops = P->flops;
  return rc;
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
