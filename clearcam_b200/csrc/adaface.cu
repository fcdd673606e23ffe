// AdaFace IR-50 face embedder as a static op list over the wgmma conv GEMM.
//
// Replaces in the reference: class ADAFACE (models/adaface.py:63-96) with its 24 BasicBlockIR_tiny blocks (:24-57).  The
// host (clearcam_b200/models/adaface.py `fold_state_dict`) folds every BatchNorm and the input normalisation into the convs
// and the linear in float64; this file only repacks the folded tensors to bf16 and runs them.
//
// Data layout: NHWC bf16 activations; per image 112x112 -> 56 -> 28 -> 14 -> 7 pixels, 64..512 channels.
//   pack      uint8 [B,112,112,3] -> bf16 [B,112,112,16] raw 0..255 (exact in bf16), channels 3..15 zero; the channel flip
//             and the /127.5 - 1 of the reference's input (:81) are in the stem's weights and border-class bias table
//   stem      conv0 -> bn0 -> PReLU (:84-86): one ACT_PRELU conv
//   block i   t = PReLU(res_layer1(conv_layer0(res_layer0(x))))      one ACT_PRELU conv (res_layer0 folded exactly: the
//                                                                     border-class table carries its shift over in-bounds taps)
//             x' = res_layer2(conv_layer1(t)) + shortcut(x)          the shortcut is x itself (stride 1, same width: the
//                                                                     residual is added in place), or a 1x1 stride-s conv
//                                                                     (+BN) run first into the output buffer, which conv_layer1
//                                                                     then adds in place.  The GEMM runs stride-2 convs as
//                                                                     3x3, so a 1x1 stride-2 shortcut is a 3x3 whose only
//                                                                     nonzero tap is the centre (exact); block 0's MaxPool2d(1,
//                                                                     2) subsample is that conv with identity weights
//   linear    bn -> flatten (NCHW) -> linear -> bn2 (:89-92): one GEMM over the NHWC 7x7x512 map with permuted columns, fp32
//   l2norm    x / sqrt(sum x^2), no epsilon (:93-95)
#include "clearcam_b200.h"
#include "cc_common.h"
#include "conv_gemm.cuh"
#include "ops.cuh"
#include "plan.h"

namespace cc {

static constexpr int kFaceSide = 112, kFacePackC = 16, kFaceDim = 512, kFaceBlocks = 24;
// (in channels, depth, stride) of the 24 blocks: models/adaface.py:61 `sizes`
static constexpr int kFaceSizes[kFaceBlocks][3] = {
    {64, 64, 2},    {64, 64, 1},    {64, 64, 1},    {64, 128, 2},   {128, 128, 1}, {128, 128, 1}, {128, 128, 1}, {128, 256, 2},
    {256, 256, 1},  {256, 256, 1},  {256, 256, 1},  {256, 256, 1},  {256, 256, 1}, {256, 256, 1}, {256, 256, 1}, {256, 256, 1},
    {256, 256, 1},  {256, 256, 1},  {256, 256, 1},  {256, 256, 1},  {256, 256, 1}, {256, 512, 2}, {512, 512, 1}, {512, 512, 1}};

__global__ void face_pack_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* __restrict__ out, long long npix) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < npix;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint8_t* s = in + 3 * i;
    __align__(16) __nv_bfloat16 v[kFacePackC];
#pragma unroll
    for (int c = 0; c < kFacePackC; ++c) v[c] = __float2bfloat16_rn(c < 3 ? static_cast<float>(s[c]) : 0.f);
    uint4* d = reinterpret_cast<uint4*>(out + kFacePackC * i);
    d[0] = reinterpret_cast<const uint4*>(v)[0];
    d[1] = reinterpret_cast<const uint4*>(v)[1];
  }
}

struct FaceBlockW {
  __nv_bfloat16 *w0 = nullptr, *w1 = nullptr, *wsc = nullptr;   // wsc == nullptr: identity shortcut at stride 1
  float *cls0 = nullptr, *slope0 = nullptr, *b1 = nullptr, *bsc = nullptr;
};

struct FaceLayer { TSlice out; size_t last_op; };   // a layer's output and the op that completes it

struct FacePlan {
  int B = 0;
  std::vector<PlanOp> ops;   // pack, stem, body.<i>.c0 | sc | c1, linear, l2norm
  std::vector<FaceLayer> layers;     // 0: stem, 1..24: blocks, 25: the linear's output before the L2 norm
};

struct FaceModel {
  int sms = 0;
  DeviceWeights weights;
  __nv_bfloat16* stem_w = nullptr; float *stem_cls = nullptr, *stem_slope = nullptr;
  FaceBlockW blk[kFaceBlocks];
  __nv_bfloat16* lin_w = nullptr; float* lin_b = nullptr;
  PlanCache<int, FacePlan> plans{"face"};   // by batch size
  // [cout][taps][cin] fp32 -> bf16 [cout][3][3][cin_pad]; taps = 1 puts the tap at the centre of the 3x3
  int up_conv(const std::string& name, int cout, int taps, int cin, int cin_pad, __nv_bfloat16** d) {
    const float* h;
    if (int rc = weights.host.get(name, static_cast<long long>(cout) * taps * cin, &h)) return rc;
    std::vector<__nv_bfloat16> w(static_cast<size_t>(cout) * 9 * cin_pad, __float2bfloat16_rn(0.f));
    for (int o = 0; o < cout; ++o)
      for (int t = 0; t < taps; ++t)
        for (int c = 0; c < cin; ++c)
          w[(static_cast<size_t>(o) * 9 + (taps == 1 ? 4 : t)) * cin_pad + c] =
              __float2bfloat16_rn(h[(static_cast<size_t>(o) * taps + t) * cin + c]);
    return weights.upload(w, d);
  }
};

struct FacePlanBuilder {
  FaceModel& M; FacePlan& P; int rc = CC_OK;
  Bump bump;
  FacePlanBuilder(FaceModel& m, FacePlan& p) : M(m), P(p) {}
  void* dalloc(size_t bytes) { return bump.take(bytes); }
  void gemm(const std::string& name, const ConvDesc& d) {
    if (rc || bump.dry) return;
    GemmLaunch L;
    rc = conv_gemm_build(d, M.sms, &L);
    if (rc) return;
    P.ops.push_back(gemm_op(name, d, ChainDesc{}, L));
  }
  void conv(const std::string& name, const TSlice& in, const __nv_bfloat16* w, const float* bias, const float* slope, int stride,
            const TSlice& out, int act, const TSlice* res) {
    ConvDesc d = conv_desc(in, w, bias, 3, stride, out, act, res);
    d.slope = slope;
    gemm(name, d);
  }
  void layer(const TSlice& out) { P.layers.push_back(FaceLayer{out, P.ops.size() - 1}); }
  int build(int B) {
    const size_t big = static_cast<size_t>(B) * kFaceSide * kFaceSide * 64 * 2;
    __nv_bfloat16* packed = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(B) * kFaceSide * kFaceSide * kFacePackC * 2));
    __nv_bfloat16* X = static_cast<__nv_bfloat16*>(dalloc(big));
    __nv_bfloat16* T = static_cast<__nv_bfloat16*>(dalloc(big));
    __nv_bfloat16* S = static_cast<__nv_bfloat16*>(dalloc(big));
    float* feat = static_cast<float*>(dalloc(static_cast<size_t>(B) * kFaceDim * 4));
    if (bump.dry) return CC_OK;
    P.ops.push_back(plan_op("pack", "face_pack",
                            op_io({operand(nullptr, CC_OP_U8, B, kFaceSide, kFaceSide, 3)},
                                  {operand(packed, CC_OP_BF16, B, kFaceSide, kFaceSide, kFacePackC)}),
                            [packed, B](const PlanIO& io, cudaStream_t st) {
      const long long npix = static_cast<long long>(B) * kFaceSide * kFaceSide;
      const long long blocks = (npix + 255) / 256;
      face_pack_kernel<<<blocks < 132 * 16 ? static_cast<int>(blocks) : 132 * 16, 256, 0, st>>>(static_cast<const uint8_t*>(io.in),
                                                                                              packed, npix);
      CC_CHECK_CUDA(cudaGetLastError());
      return CC_OK;
    }));
    int H = kFaceSide;
    conv("stem", nhwc_slice(packed, kFacePackC, 0, kFacePackC, 0, B, H, H), M.stem_w, M.stem_cls, M.stem_slope, 1,
         nhwc_slice(X, 64, 0, 64), ACT_PRELU, nullptr);
    layer(nhwc_slice(X, 64, 0, 64, 0, B, H, H));
    for (int i = 0; i < kFaceBlocks && !rc; ++i) {
      const int cin = kFaceSizes[i][0], D = kFaceSizes[i][1], s = kFaceSizes[i][2], Ho = H / s;
      const FaceBlockW& b = M.blk[i];
      const std::string name = "body." + std::to_string(i);
      conv(name + ".c0", nhwc_slice(X, cin, 0, cin, 0, B, H, H), b.w0, b.cls0, b.slope0, 1, nhwc_slice(T, D, 0, D), ACT_PRELU, nullptr);
      if (!b.wsc) {          // identity shortcut: conv_layer1 adds x in place
        const TSlice o = nhwc_slice(X, D, 0, D);
        conv(name + ".c1", nhwc_slice(T, D, 0, D, 0, B, H, H), b.w1, b.b1, nullptr, 1, o, ACT_NONE, &o);
      } else {               // shortcut conv into S, then conv_layer1 adds onto it in place
        const TSlice o = nhwc_slice(S, D, 0, D);
        conv(name + ".sc", nhwc_slice(X, cin, 0, cin, 0, B, H, H), b.wsc, b.bsc, nullptr, s, o, ACT_NONE, nullptr);
        conv(name + ".c1", nhwc_slice(T, D, 0, D, 0, B, H, H), b.w1, b.b1, nullptr, s, o, ACT_NONE, &o);
        std::swap(X, S);
      }
      H = Ho;
      layer(nhwc_slice(X, D, 0, D, 0, B, H, H));
    }
    if (rc) return rc;
    {  // bn -> flatten -> linear -> bn2: [B, 7*7*512] . W^T + b, fp32
      const int K = H * H * kFaceDim;
      const TSlice o = nhwc_slice(feat, kFaceDim, 0, kFaceDim, 1);
      ConvDesc d = conv_desc(nhwc_slice(X, K, 0, K, 0, 1, 1, B), M.lin_w, M.lin_b, 1, 1, o, ACT_NONE);
      // 512 outputs in 16 n blocks of 32: at small B the 25.7 MB of weights are streamed by 16 x ceil(B / 128) CTAs
      d.bn_override = 32;
      gemm("linear", d);
      if (rc) return rc;
      layer(nhwc_slice(feat, kFaceDim, 0, kFaceDim, 1, B, 1, 1));
    }
    P.ops.push_back(plan_op("l2norm", "l2norm", op_io({operand(feat, CC_OP_F32, B, 1, 1, kFaceDim)}, {operand(nullptr, CC_OP_F32, B, 1, 1, kFaceDim)}),
                            [feat, B](const PlanIO& io, cudaStream_t st) {
      return l2norm_launch(feat, io.out, B, kFaceDim, io.out_stride, 0.f, st);
    }));
    return rc;
  }
};

}  // namespace cc

using namespace cc;

struct cc_face { FaceModel m; };

// workspace bytes the plan of batch B addresses (measuring pass of the builder: no device work)
static int face_plan_bytes(cc_face* h, int B, size_t* bytes) {
  FacePlan tmp;
  FacePlanBuilder dry(h->m, tmp);
  dry.bump.dry = true;
  if (int rc = dry.build(B)) return rc;
  *bytes = dry.bump.off + 1024;
  return CC_OK;
}
static int face_plan(cc_face* h, int B, FacePlan** out) {
  return h->m.plans.get(
      B, [&](size_t* bytes) { return face_plan_bytes(h, B, bytes); },
      [&](FacePlan& P, uint8_t* base, size_t* used) {
        P.B = B;
        FacePlanBuilder b(h->m, P);
        b.bump.base = base;
        const int rc = b.build(B);
        *used = b.bump.off;
        return rc;
      },
      out);
}

extern "C" {

int cc_face_create(int n_tensors, const char* const* names, const float* const* h_data, const int64_t* numels, cc_face** out) {
  CC_REQUIRE(out, "cc_face_create: null argument");
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_face_create: no sm_90 (H100) device");
  std::unique_ptr<cc_face> h(new cc_face());
  FaceModel& M = h->m;
  M.sms = sms;
  int rc = 0;
  if ((rc = M.weights.host.fill("cc_face_create", n_tensors, names, h_data, numels))) return rc;
  if ((rc = M.up_conv("stem.w", 64, 9, 3, kFacePackC, &M.stem_w))) return rc;
  if ((rc = M.weights.up_f32("stem.cls", 9 * 64, &M.stem_cls))) return rc;
  if ((rc = M.weights.up_f32("stem.slope", 64, &M.stem_slope))) return rc;
  for (int i = 0; i < kFaceBlocks; ++i) {
    const int cin = kFaceSizes[i][0], D = kFaceSizes[i][1];
    const bool proj = cin != D || kFaceSizes[i][2] != 1;
    const std::string p = "body." + std::to_string(i);
    FaceBlockW& b = M.blk[i];
    if ((rc = M.up_conv(p + ".c0.w", D, 9, cin, cin, &b.w0))) return rc;
    if ((rc = M.weights.up_f32(p + ".c0.cls", 9 * D, &b.cls0))) return rc;
    if ((rc = M.weights.up_f32(p + ".c0.slope", D, &b.slope0))) return rc;
    if ((rc = M.up_conv(p + ".c1.w", D, 9, D, D, &b.w1))) return rc;
    if ((rc = M.weights.up_f32(p + ".c1.b", D, &b.b1))) return rc;
    if (proj) {
      if ((rc = M.up_conv(p + ".sc.w", D, 1, cin, cin, &b.wsc))) return rc;
      if ((rc = M.weights.up_f32(p + ".sc.b", D, &b.bsc))) return rc;
    }
  }
  const int K = 7 * 7 * kFaceDim;
  {
    const float* w;
    if ((rc = M.weights.host.get("linear.w", static_cast<long long>(kFaceDim) * K, &w))) return rc;
    std::vector<__nv_bfloat16> wb(static_cast<size_t>(kFaceDim) * K);
    for (size_t i = 0; i < wb.size(); ++i) wb[i] = __float2bfloat16_rn(w[i]);
    if ((rc = M.weights.upload(wb, &M.lin_w))) return rc;
  }
  if ((rc = M.weights.up_f32("linear.b", kFaceDim, &M.lin_b))) return rc;
  M.weights.host.clear();
  *out = h.release();
  return CC_OK;
}

int cc_face_destroy(cc_face* h) {
  delete h;
  return CC_OK;
}

int cc_face_workspace_bytes(cc_face* h, int B, size_t* bytes) {
  CC_REQUIRE(h && bytes && B > 0, "cc_face_workspace_bytes: bad argument");
  return face_plan_bytes(h, B, bytes);
}

int cc_face_set_workspace(cc_face* h, void* d_workspace, size_t bytes) {
  if (int rc = check_workspace("cc_face_set_workspace", h, d_workspace)) return rc;
  return h->m.plans.adopt(d_workspace, bytes);
}

int cc_face_embed(cc_face* h, const uint8_t* d_faces, int B, float* d_out, long long out_row_stride, void* stream) {
  CC_REQUIRE(h && d_faces && d_out && B > 0, "cc_face_embed: bad argument");
  CC_REQUIRE(out_row_stride == 0 || out_row_stride >= kFaceDim, "cc_face_embed: out_row_stride %lld is shorter than a row of %d",
             out_row_stride, kFaceDim);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_out) & 3) == 0, "cc_face_embed: d_out must be 4-byte aligned");
  FacePlan* P = nullptr;
  if (int rc = face_plan(h, B, &P)) return rc;
  return run_ops(P->ops, PlanIO{d_faces, d_out, out_row_stride > 0 ? out_row_stride : kFaceDim}, static_cast<cudaStream_t>(stream));
}

int cc_face_layer_output(cc_face* h, const uint8_t* d_faces, int B, int layer, float* d_dst, int* C, int* H, int* W, void* stream) {
  CC_REQUIRE(h && B > 0, "cc_face_layer_output: bad argument");
  CC_REQUIRE(layer >= 0 && layer <= kFaceBlocks + 1, "cc_face_layer_output: bad layer %d (0 stem, 1..24 blocks, 25 linear)", layer);
  FacePlan* P = nullptr;
  if (int rc = face_plan(h, B, &P)) return rc;
  const TSlice& t = P->layers[layer].out;
  if (C) *C = t.C;
  if (H) *H = t.H;
  if (W) *W = t.W;
  if (!d_dst) return CC_OK;
  CC_REQUIRE(d_faces, "cc_face_layer_output: d_faces is NULL");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = run_ops(P->ops, PlanIO{d_faces, nullptr, kFaceDim}, st, 0, P->layers[layer].last_op + 1)) return rc;
  return slice_to_f32_launch(t, d_dst, st);
}

// conv op taps: what each GEMM launch of the cached plan computes, and the plan run one range of ops at a time
int cc_face_op_conv(cc_face* h, int B, int i, cc_conv_op* out) {
  CC_REQUIRE(h && B > 0, "cc_face_op_conv: bad argument");
  FacePlan* P = nullptr;
  if (int rc = face_plan(h, B, &P)) return rc;
  return op_conv_tap("cc_face_op_conv", P->ops, i, out);
}

int cc_face_op_io(cc_face* h, int B, int i, cc_op_io* out) {
  CC_REQUIRE(h && B > 0, "cc_face_op_io: bad argument");
  FacePlan* P = nullptr;
  if (int rc = face_plan(h, B, &P)) return rc;
  return op_io_tap("cc_face_op_io", P->ops, i, out);
}

int cc_face_run_ops(cc_face* h, const uint8_t* d_faces, int B, int first, int last, float* d_out, void* stream) {
  CC_REQUIRE(h && d_faces && d_out && B > 0, "cc_face_run_ops: bad argument");
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_out) & 3) == 0, "cc_face_run_ops: d_out must be 4-byte aligned");
  FacePlan* P = nullptr;
  if (int rc = face_plan(h, B, &P)) return rc;
  if (int rc = check_range("cc_face_run_ops", first, last, static_cast<int>(P->ops.size()))) return rc;
  return run_ops(P->ops, PlanIO{d_faces, d_out, kFaceDim}, static_cast<cudaStream_t>(stream), first, last);
}

}  // extern "C"
