// YOLOv9 (t/s/c/e) forward as a static op list over the sm_90a kernels.
//
// What it replaces in the reference: YOLOv9.__init__ graph (detection/yolov9.py:299-371), YOLOv9.__call__
// (:375-388: preprocess -> BGR flip -> /255 -> layer routing by m.f -> postprocess -> scale_boxes) and the
// TinyJit capture of jit_infer (utils/helpers.py:214-221: here a cached "plan" per input shape).
//
// Design (GPU-first, not a translation):
//  * a plan = flat vector of kernel launches with every tensor map / pointer resolved at build time;
//  * Tensor.cat / chunk / split never move data: producers write straight into channel slices of the
//    consumer's concat buffer (NHWC, channel stride = buffer width);
//  * RepNCSP.cv1 and .cv2 (two 1x1 convs on the same input) run as ONE GEMM with concatenated output channels,
//    likewise the first 3x3 of the box and class branches of each detect scale;
//  * grouped (g=4) head convs become block-diagonal dense weights so they ride the tensor-core kernel too;
//  * RepNBottleneck's residual is fused in the conv epilogue (in place);
//  * head logits stay fp32; everything else is bf16 storage with fp32 accumulation.
#include "clearcam_b200.h"
#include "cc_common.h"
#include "conv_gemm.cuh"
#include "ops.cuh"
#include "plan.h"
#include <cmath>

namespace cc {

// ------------------------------------------------------------------------------------------------ spec
// Own restatement of the reference layer tables (detection/yolov9.py:299-371, SIZES :461-464).
enum LOp { L_CONV, L_ELAN1, L_ELAN4, L_ADOWN, L_ACONV, L_SPPELAN, L_UPSAMPLE, L_CONCAT, L_SILENCE, L_CBLINEAR, L_CBFUSE, L_DETECT };
struct Layer {
  LOp op;
  std::vector<int> f;          // sources (-1 = previous)
  int a = 0, b = 0, c = 0, n = 0, k = 0, s = 0;   // op-specific ints
  std::vector<int> list;       // c2s (cblinear) / idx (cbfuse) / chs (detect)
};

static Layer mk(LOp op, std::vector<int> f = {-1}) { Layer l; l.op = op; l.f = std::move(f); return l; }
static Layer conv_l(int cin, int cout, int k, int s, std::vector<int> f = {-1}) {
  Layer l = mk(L_CONV, std::move(f)); l.a = cin; l.b = cout; l.k = k; l.s = s; return l;
}
static Layer elan4_l(int a, int b, int c, int n) { Layer l = mk(L_ELAN4); l.a = a; l.b = b; l.c = c; l.n = n; return l; }
static Layer adown_l(int ch) { Layer l = mk(L_ADOWN); l.a = ch; return l; }
static Layer aconv_l(int cin, int cout) { Layer l = mk(L_ACONV); l.a = cin; l.b = cout; return l; }
static Layer cbl_l(int cin, std::vector<int> c2s, int f) { Layer l = mk(L_CBLINEAR, {f}); l.a = cin; l.list = std::move(c2s); return l; }
static Layer cbf_l(std::vector<int> f, std::vector<int> idx) { Layer l = mk(L_CBFUSE, std::move(f)); l.list = std::move(idx); return l; }

static bool build_spec(const std::string& size, std::vector<Layer>* out) {
  std::vector<Layer>& L = *out;
  static const std::map<std::string, std::vector<int>> SZ = {
      {"t", {16, 64, 96, 24, 128, 256, 224, 160, 48, 144, 192, 80, 32, 16, 3, 96, 32, 64, 128, 64, 64, 128}},
      {"s", {32, 128, 192, 48, 256, 512, 448, 320, 96, 288, 384, 128, 64, 32, 3, 192, 64, 64, 128, 128, 128, 256}},
      {"m", {32, 240, 360, 90, 480, 960, 840, 600, 184, 544, 720, 240, 128, 60, 1, 360, 120, 64, 128, 240, 240, 480}},
      {"c", {64, 256, 512, 128, 256, 1024, 1024, 1024, 128, 768, 1024, 256, 128, 64, 1, 256, 128, 128, 256, 128, 512, 512}},
      // zero-padded equivalents of t and m (every width a multiple of 16): same graphs, weights scattered into the padded
      // layout by the host (clearcam_b200/detection/padding.py; the function computed is unchanged, tests/test_oracle_cpu.py)
      {"t@16", {16, 64, 96, 32, 128, 256, 224, 160, 48, 144, 192, 96, 32, 16, 3, 96, 32, 64, 128, 64, 64, 128}},
      {"m@16", {32, 240, 384, 96, 480, 960, 864, 624, 192, 576, 720, 240, 128, 64, 1, 384, 128, 64, 128, 240, 240, 480}}};
  if (size == "e") {
    L.push_back(mk(L_SILENCE));
    L.push_back(conv_l(3, 64, 3, 2));
    L.push_back(conv_l(64, 128, 3, 2));
    L.push_back(elan4_l(128, 32, 256, 2));
    L.push_back(adown_l(128));
    L.push_back(elan4_l(256, 64, 512, 2));
    L.push_back(adown_l(256));
    L.push_back(elan4_l(512, 128, 1024, 2));
    L.push_back(adown_l(512));
    L.push_back(elan4_l(1024, 128, 1024, 2));
    L.push_back(cbl_l(64, {64}, 1));
    L.push_back(cbl_l(256, {64, 128}, 3));
    L.push_back(cbl_l(512, {64, 128, 256}, 5));
    L.push_back(cbl_l(1024, {64, 128, 256, 512}, 7));
    L.push_back(cbl_l(1024, {64, 128, 256, 512, 1024}, 9));
    L.push_back(conv_l(3, 64, 3, 2, {0}));
    L.push_back(cbf_l({10, 11, 12, 13, 14, -1}, {0, 0, 0, 0, 0}));
    L.push_back(conv_l(64, 128, 3, 2));
    L.push_back(cbf_l({11, 12, 13, 14, -1}, {1, 1, 1, 1}));
    L.push_back(elan4_l(128, 32, 256, 2));
    L.push_back(adown_l(128));
    L.push_back(cbf_l({12, 13, 14, -1}, {2, 2, 2}));
    L.push_back(elan4_l(256, 64, 512, 2));
    L.push_back(adown_l(256));
    L.push_back(cbf_l({13, 14, -1}, {3, 3}));
    L.push_back(elan4_l(512, 128, 1024, 2));
    L.push_back(adown_l(512));
    L.push_back(cbf_l({14, -1}, {4}));
    L.push_back(elan4_l(1024, 128, 1024, 2));
    { Layer l = mk(L_SPPELAN, {28}); l.a = 1024; l.b = 256; l.c = 512; L.push_back(l); }
    L.push_back(mk(L_UPSAMPLE));
    L.push_back(mk(L_CONCAT, {-1, 25}));
    L.push_back(elan4_l(1536, 128, 512, 2));
    L.push_back(mk(L_UPSAMPLE));
    L.push_back(mk(L_CONCAT, {-1, 22}));
    L.push_back(elan4_l(1024, 64, 256, 2));
    L.push_back(adown_l(128));
    L.push_back(mk(L_CONCAT, {-1, 32}));
    L.push_back(elan4_l(768, 128, 512, 2));
    L.push_back(adown_l(256));
    L.push_back(mk(L_CONCAT, {-1, 29}));
    L.push_back(elan4_l(1024, 256, 512, 2));
    { Layer l = mk(L_DETECT, {35, 38, 41}); l.list = {256, 512, 512}; l.a = 256; L.push_back(l); }
    return true;
  }
  auto it = SZ.find(size);
  if (it == SZ.end()) return false;
  const std::vector<int>& z = it->second;
  const int a = z[0], b = z[1], c = z[2], d = z[3], e = z[4], f = z[5], g = z[6], h = z[7], i = z[8], j = z[9], k = z[10],
            l = z[11], m = z[12], n = z[13], p = z[14], q = z[15], r = z[16], s = z[17], t = z[18], u = z[19], v = z[20],
            w = z[21];
  const std::string base = size.substr(0, size.find('@'));
  const bool small = base == "t" || base == "s";
  const bool isc = size == "c";
  L.push_back(conv_l(3, a, 3, 2));
  L.push_back(conv_l(a, a * 2, 3, 2));
  if (small) { Layer x = mk(L_ELAN1); x.a = a * 2; x.b = m; x.c = a; x.n = b; L.push_back(x); }
  else L.push_back(elan4_l(s, 32, t, p));
  L.push_back(isc ? adown_l(128) : aconv_l(m, u));
  L.push_back(elan4_l(b, n, v, p));
  L.push_back(isc ? adown_l(256) : aconv_l(b, q));
  L.push_back(elan4_l(c, d, c, p));
  L.push_back(isc ? adown_l(256) : aconv_l(q, e));
  L.push_back(elan4_l(w, r, w, p));
  { Layer x = mk(L_SPPELAN); x.a = w; x.b = b; x.c = w; (void)f; L.push_back(x); }
  L.push_back(mk(L_UPSAMPLE));
  L.push_back(mk(L_CONCAT, {-1, 6}));
  L.push_back(elan4_l(g, d, c, p));
  L.push_back(mk(L_UPSAMPLE));
  L.push_back(mk(L_CONCAT, {-1, 4}));
  L.push_back(elan4_l(h, n, b, p));
  L.push_back(isc ? adown_l(128) : aconv_l(v, i));
  L.push_back(mk(L_CONCAT, {-1, 12}));
  L.push_back(elan4_l(j, d, c, p));
  L.push_back(isc ? adown_l(256) : aconv_l(q, b));
  L.push_back(mk(L_CONCAT, {-1, 9}));
  L.push_back(elan4_l(k, r, w, p));
  { Layer x = mk(L_DETECT, {15, 18, 21}); x.list = {b, c, w}; x.a = l; L.push_back(x); }
  return true;
}

// ------------------------------------------------------------------------------------------------ weights
struct ConvW {           // device-resident, kernel layout
  __nv_bfloat16* w = nullptr;   // [Cout][k][k][Cin_eff]  (Cin_eff = Cin when dense, Cin/groups when grouped)
  float* wf32 = nullptr;        // stem only: fp32 [Cout][3][3][3]
  __nv_bfloat16* wtc = nullptr; // stem only: bf16 [Cout][32] = w/255 in (r,s,c) order, zero padded (tensor-core uint8 path)
  // fp32-accurate mode: the fp32 weight is split w = hi + mid + lo (three bf16).  w5: [Cout][k][k][5][Cin] = planes
  // hi|mid|lo|hi|mid (the five cross products below 2^-8 of the result, against the activation planes lo|mid|hi|mid|hi);
  // whi[i]: [Cout][k][k][seg_c[i]] = the hi plane of input-channel segment i (the hi x hi products, one GEMM per segment so
  // that no tensor-core accumulator takes more than 48 MMA steps: hi_segments)
  __nv_bfloat16* w5 = nullptr;
  std::vector<__nv_bfloat16*> whi;
  std::vector<int> seg_off, seg_c;
  float* bias = nullptr;
  int cin = 0, cout = 0, k = 0, groups = 1;   // groups == 1 -> dense (possibly block-diagonal expansion)
};

static __nv_bfloat16 f2bf(float x) { return __float2bfloat16_rn(x); }

// ---- weight packing, shared by the plan builder and the kernel-level taps (cc_stem, cc_conv2d_fp32_accurate)
// stem: PyTorch [Cout][3][3][3] fp32 -> wf [Cout][27] fp32 with the taps in (r, s, RGB) order (stem_kernel)
static void stem_weights_rsc(const float* w, int cout, float* wf) {
  for (int co = 0; co < cout; ++co)
    for (int ci = 0; ci < 3; ++ci)
      for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s) wf[(static_cast<size_t>(co) * 9 + r * 3 + s) * 3 + ci] = w[((static_cast<size_t>(co) * 3 + ci) * 3 + r) * 3 + s];
}
// ... and the tensor-core stem's operand: bf16(w / 255) [Cout][32], K = 27 taps zero padded to 32 (raw pixels are exact in bf16)
static std::vector<__nv_bfloat16> stem_tc_weights(const float* wf, int cout) {
  std::vector<__nv_bfloat16> wt(static_cast<size_t>(cout) * 32, f2bf(0.f));
  for (int co = 0; co < cout; ++co)
    for (int kk = 0; kk < 27; ++kk) wt[static_cast<size_t>(co) * 32 + kk] = f2bf(wf[static_cast<size_t>(co) * 27 + kk] / 255.0f);
  return wt;
}

// fp32-accurate mode: the input-channel segments of the hi x hi products, one GEMM each.  The tensor core's fp32 accumulation
// truncates and its bias grows with the number of MMA steps into one accumulator (tests/tools/diag_tc_accum.py), so no segment
// takes more than 48 k16 steps (seg_c * k * k / 16 <= 48).  Widths are multiples of 64 when Cin allows (the kernel's widest
// k-block), else of 16, and as even as that allows.
static constexpr int kMaxHiSteps = 48;
static void hi_segments(int cin, int k, std::vector<int>* seg_off, std::vector<int>* seg_c) {
  const int unit = cin % 64 == 0 ? 64 : 16;
  int max_c = kMaxHiSteps * 16 / (k * k) / unit * unit;
  if (max_c < unit) max_c = unit;
  const int nseg = (cin + max_c - 1) / max_c;
  const int sc = ((cin + nseg - 1) / nseg + unit - 1) / unit * unit;
  seg_off->clear(); seg_c->clear();
  for (int off = 0; off < cin; off += sc) { seg_off->push_back(off); seg_c->push_back(std::min(sc, cin - off)); }
}
// Split fp32 weights wf [rows = Cout*k*k][cin] into w = hi + mid + lo (three bf16).  w5: [rows][5][cin] = planes hi|mid|lo|hi|mid
// (the five cross products below 2^-8 of the result, against the activation planes lo|mid|hi|mid|hi); whi[i]: [rows][seg_c[i]] =
// the hi plane of input-channel segment i.
static void split_weight_planes(const float* wf, size_t rows, int cin, const std::vector<int>& seg_off, const std::vector<int>& seg_c,
                                std::vector<__nv_bfloat16>* w5, std::vector<std::vector<__nv_bfloat16>>* whi) {
  w5->assign(rows * 5 * cin, f2bf(0.f));
  std::vector<__nv_bfloat16> hi_plane(rows * cin);
  for (size_t row = 0; row < rows; ++row)
    for (int ci = 0; ci < cin; ++ci) {
      const float v = wf[row * cin + ci];
      const __nv_bfloat16 hi = f2bf(v);
      const float r1 = v - __bfloat162float(hi);
      const __nv_bfloat16 mid = f2bf(r1);
      const __nv_bfloat16 lo = f2bf(r1 - __bfloat162float(mid));
      __nv_bfloat16* d5 = w5->data() + row * 5 * cin + ci;
      d5[0] = hi; d5[cin] = mid; d5[2 * cin] = lo; d5[3 * cin] = hi; d5[4 * cin] = mid;
      hi_plane[row * cin + ci] = hi;
    }
  whi->assign(seg_off.size(), {});
  for (size_t sgi = 0; sgi < seg_off.size(); ++sgi) {
    const int off = seg_off[sgi], sc = seg_c[sgi];
    std::vector<__nv_bfloat16>& ws = (*whi)[sgi];
    ws.resize(rows * sc);
    for (size_t row = 0; row < rows; ++row)
      for (int c = 0; c < sc; ++c) ws[row * sc + c] = hi_plane[row * cin + off + c];
  }
}

// ---- letterbox geometry of one Hf x Wf frame at `res` (detection/yolov9.py:390-404, scale_boxes :406-421), shared by the plan
// builder, cc_letterbox, the frame-table path and cc_yolo_net_shape
struct LbGeom {
  int new_h = 0, new_w = 0, py = 0, px = 0;   // resized extent, pads
  int Hr = 0, Wr = 0;                         // the reference's letterboxed extent
  int H = 0, W = 0;                           // the net input: Hr x Wr rounded up to a multiple of 32
  float sx = 0.f, sy = 0.f;                   // float(Wf / new_w), float(Hf / new_h), computed in double
  PostScale scale{};                          // scale_boxes back to the frame
};
static LbGeom letterbox_geom(int Hf, int Wf, int res) {
  LbGeom g;
  const double r = std::min(double(res) / Hf, double(res) / Wf);
  g.new_w = int(std::nearbyint(Wf * r)); g.new_h = int(std::nearbyint(Hf * r));
  const double dw = double(((res - g.new_w) % 32 + 32) % 32) / 2, dh = double(((res - g.new_h) % 32 + 32) % 32) / 2;
  g.px = int(std::nearbyint(dw - 0.1)); g.py = int(std::nearbyint(dh - 0.1));
  // The reference pads int(round(d - 0.1)) on BOTH sides, so when (res - new) % 32 is odd its net input is one pixel short of
  // a multiple of 32 (SURVEY App. A5) — and it keeps going: a 3x3/s2/p1 conv over 2k-1 rows gives the same k output rows as
  // over 2k rows whose last row is zero.  So the net input buffer is rounded up to the multiple of 32 with that zero row /
  // column (the letterbox kernel pads with zeros anyway): identical arithmetic, even dims for the TMA views.  scale_boxes
  // still sees the reference's odd extent (Hr, Wr).
  g.Hr = g.new_h + 2 * g.py; g.Wr = g.new_w + 2 * g.px;
  g.H = (g.Hr + 31) / 32 * 32; g.W = (g.Wr + 31) / 32 * 32;
  g.sx = float(double(Wf) / double(g.new_w)); g.sy = float(double(Hf) / double(g.new_h));
  const double gain = std::min(double(g.Hr) / Hf, double(g.Wr) / Wf);   // the reference's img1_shape (detection/yolov9.py:406-416)
  g.scale.gain = float(gain);
  g.scale.pad_x = float((g.Wr - Wf * gain) / 2); g.scale.pad_y = float((g.Hr - Hf * gain) / 2);
  g.scale.clip_w = float(Wf); g.scale.clip_h = float(Hf);
  return g;
}
// the detector runs a frame only when its letterboxed extent is within one pixel of a multiple of 32 (res a multiple of 32)
static int require_net(const LbGeom& g, int Hf, int Wf, int res) {
  CC_REQUIRE(g.H > 0 && g.W > 0 && g.H - g.Hr <= 1 && g.W - g.Wr <= 1,
             "yolo: letterboxed input %dx%d is not within one pixel of a multiple of 32 (frame %dx%d, res %d)", g.Hr, g.Wr, Hf, Wf, res);
  return CC_OK;
}

// A tensor of the plan: a slice, or the input frames (`image`, no buffer of the plan's own)
struct T : TSlice { bool image = false; T() : TSlice{} {} };

struct YoloPlan {
  int B = 0, Hf = 0, Wf = 0, res = 0, fmt = 0, H = 0, W = 0, A = 0;    // fmt: CC_FRAME_* of the frames
  int Hr = 0, Wr = 0;          // the reference's letterboxed extent (H, W are it rounded up to a multiple of 32)
  // frame-table plan (cc_yolo_forward_frames): Hf x Wf is the net shape itself, the frames come with every call.  Its op list
  // has no letterbox (launched by the caller with the call's table into lb_out) and ends with the postprocess (launched with
  // the call's per-image scales); in between it is the op list of a uniform plan of the net shape.
  bool table = false;
  std::vector<PlanOp> ops;
  PostParams post{};          // the postprocess op's parameters (a frame-table call launches it with per-image scales)
  size_t alloc_bytes = 0;      // bytes of the handle's shared workspace this plan addresses
  float* pred = nullptr;   // [B,A,6]
  float* raw = nullptr;    // [B,84,A] (allocated lazily when a tap is requested)
  void* lb_out = nullptr;  // letterboxed BGR frames (float32 for float frames, else uint8) or nullptr when identity
  double conv_flops = 0;
  int n_launch = 0;
  std::vector<T> layer_outs;   // per spec layer (parity taps)
  // CUDA graph of the whole launch list (the analogue of the reference's TinyJit capture, utils/helpers.py:214-221).  Kernel
  // arguments are baked into a graph, so it is captured once the caller has passed the same (frames, out, raw) pointers twice
  // in a row — the steady state of a camera loop that reuses its buffers — and replayed while they stay the same.
  cudaGraphExec_t gexec = nullptr;
  const void* g_frames = nullptr; float* g_out = nullptr; float* g_raw = nullptr;      // pointers the graph was captured with
  const void* l_frames = nullptr; float* l_out = nullptr; float* l_raw = nullptr;      // pointers of the previous call
  bool ran = false;            // a previous call exists (a frame-table plan passes null frames / out pointers every time)
  ~YoloPlan() { if (gexec) cudaGraphExecDestroy(gexec); }
};

struct YoloModel {
  std::string size;
  std::vector<Layer> spec;
  DeviceWeights weights;
  std::map<std::string, ConvW> convs;
  PlanCache<std::string, YoloPlan> plans{"yolo"};   // activation workspace shared by all plans (size of the largest)
  int sms = 0;
  cudaStream_t cap_stream = nullptr;   // private stream the graphs are captured on (the caller's may be the legacy default stream)
  // fp32-accurate mode (CC_YOLO_FP32_ACCURATE): activations are stored in fp32 and every conv runs on the same wgmma kernel
  // over a 3-way bf16 split of both operands (six plane products, fp32 accumulation): the result carries fp32-level error
  // instead of bf16's 2^-9, at ~6x the tensor work and 2x the activation bytes.  The mode the 1e-3 parity bar is checked in.
  bool precise = false;
  // the plans' CUDA graph execs go before the capture stream and the workspace
  ~YoloModel() { plans.plans.clear(); if (cap_stream) cudaStreamDestroy(cap_stream); }

  // Load conv `name` (PyTorch layout [Cout][Cin/g][k][k]) -> [Cout][k][k][Cin] bf16, optionally expanding groups
  // to block-diagonal dense, optionally stacking a second conv's output channels under it (fused 1x1 pair).
  // ci_begin / ci_total: load only input channels [ci_begin, ci_begin + cin) of a conv stored with ci_total input channels (the
  // two halves of a 1x1 conv over a concat); with_bias = false leaves the bias zero (it is applied once, by the other half)
  int load_conv(const std::string& key, const std::vector<std::string>& names, int cin, const std::vector<int>& couts,
                int k, int groups, bool dense, bool stem = false, int ci_begin = 0, int ci_total = 0, bool with_bias = true) {
    if (convs.count(key)) return CC_OK;
    if (ci_total == 0) ci_total = cin;
    int cout_total = 0;
    for (int c : couts) cout_total += c;
    const int cin_g = cin / groups;
    const int cin_eff = dense ? cin : cin_g;
    std::vector<__nv_bfloat16> w(static_cast<size_t>(cout_total) * k * k * cin_eff, f2bf(0.f));
    std::vector<float> wf, bias(cout_total);
    if (stem) wf.resize(static_cast<size_t>(cout_total) * 27);
    else if (precise) wf.assign(w.size(), 0.f);   // fp32-accurate mode: w's layout in fp32 (split into bf16 planes below)
    int co_base = 0;
    for (size_t t = 0; t < names.size(); ++t) {
      const int cout = couts[t];
      const int src_cin_g = ci_total / groups;
      const float *src, *bsrc;
      int rc;
      if ((rc = weights.host.get(names[t] + ".weight", static_cast<long long>(cout) * src_cin_g * k * k, &src)) ||
          (rc = weights.host.get(names[t] + ".bias", cout, &bsrc)))
        return rc;
      CC_REQUIRE(ci_total == cin || groups == 1, "yolo: '%s': an input-channel sub-range of a grouped conv", names[t].c_str());
      const int cpg_out = cout / groups;
      if (stem) {
        CC_REQUIRE(k == 3 && cin == 3 && groups == 1 && ci_total == 3, "yolo: stem '%s' is not a 3x3 conv over 3 channels", names[t].c_str());
        stem_weights_rsc(src, cout, &wf[static_cast<size_t>(co_base) * 27]);
      }
      for (int co = 0; co < cout; ++co) {
        const int g = co / cpg_out;
        for (int ci = 0; ci < cin_g && !stem; ++ci)
          for (int r = 0; r < k; ++r)
            for (int s = 0; s < k; ++s) {
              const float v = src[((static_cast<size_t>(co) * src_cin_g + ci_begin + ci) * k + r) * k + s];
              const int ci_eff = dense ? g * cin_g + ci : ci;
              const size_t o = ((static_cast<size_t>(co_base + co) * k + r) * k + s) * cin_eff + ci_eff;
              w[o] = f2bf(v);
              if (precise) wf[o] = v;
            }
        bias[co_base + co] = with_bias ? bsrc[co] : 0.f;
      }
      co_base += cout;
    }
    ConvW cw;
    cw.cin = cin; cw.cout = cout_total; cw.k = k; cw.groups = dense ? 1 : groups;
    int rc;
    if (stem) {
      if ((rc = weights.upload(wf, &cw.wf32))) return rc;
      if ((rc = weights.upload(stem_tc_weights(wf.data(), cout_total), &cw.wtc))) return rc;
    }
    else if (!precise) { if ((rc = weights.upload(w, &cw.w))) return rc; }
    else {
      hi_segments(cin_eff, k, &cw.seg_off, &cw.seg_c);
      std::vector<__nv_bfloat16> w5;
      std::vector<std::vector<__nv_bfloat16>> whi;
      split_weight_planes(wf.data(), static_cast<size_t>(cout_total) * k * k, cin_eff, cw.seg_off, cw.seg_c, &w5, &whi);
      if ((rc = weights.upload(w5, &cw.w5))) return rc;
      for (const std::vector<__nv_bfloat16>& ws : whi) {
        __nv_bfloat16* dptr = nullptr;
        if ((rc = weights.upload(ws, &dptr))) return rc;
        cw.whi.push_back(dptr);
      }
    }
    if ((rc = weights.upload(bias, &cw.bias))) return rc;
    convs[key] = cw;
    return CC_OK;
  }
};

static bool tc_ok(int cin, int cout) { return cin % 16 == 0 && cout % 16 == 0; }
// algorithmic HBM bytes of a slice, for the bytes a memory-bound op reports (inputs once + outputs once)
static double slice_bytes(const TSlice& t) { return double(t.N) * t.H * t.W * t.C * (t.f32 ? 4 : 2); }

// The fp32-accurate conv as ops, shared by the plan builder and cc_conv2d_fp32_accurate: fp32 slice -> six bf16 planes
// [lo|mid|hi|mid|hi|hi] in `scratch`; then on the same wgmma conv kernel, all with fp32 output into the dense partial-sum buffer
// `accbuf`: one GEMM per input-channel segment of the hi x hi products (hi plane at channel offset 5C), accumulated with the
// in-place fp32 residual of the epilogue (one round-to-nearest add), one GEMM for the five cross products (planes 0..4 against
// the weight planes hi|mid|lo|hi|mid); a last pass applies bias, the exact SiLU and the residual and writes the output slice.
static int precise_conv_ops(const std::string& key, const ConvW& cw, const TSlice& in, int stride, int act, __nv_bfloat16* scratch,
                            float* accbuf, const TSlice& out, const TSlice* res, int sms, std::vector<PlanOp>* ops, double* conv_flops) {
  ops->push_back(plan_op(key + ".split", "split_planes", op_io({operand(in)}, {operand(scratch, CC_OP_BF16, in.N, in.H, in.W, 6 * in.C)}),
                         [in, scratch](const PlanIO&, cudaStream_t st) {
    return split_planes_launch(in, scratch, st);
  }));
  const int Ho = conv_out(in.H, stride), Wo = conv_out(in.W, stride);
  const int nseg = static_cast<int>(cw.seg_off.size());
  const TSlice acc = dense_f32(accbuf, cw.cout);
  for (int g = 0; g <= nseg; ++g) {
    const TSlice planes = g < nseg ? nhwc_slice(scratch, 6 * in.C, 5 * in.C + cw.seg_off[g], cw.seg_c[g], 0, in.N, in.H, in.W)
                                   : nhwc_slice(scratch, 6 * in.C, 0, 5 * in.C, 0, in.N, in.H, in.W);
    const ConvDesc d = conv_desc(planes, g < nseg ? cw.whi[g] : cw.w5, nullptr, cw.k, stride, acc, CC_ACT_NONE, g > 0 ? &acc : nullptr);
    GemmLaunch L;
    if (int rc = conv_gemm_build(d, sms, &L)) return rc;
    L.flops = g == 0 ? 2.0 * in.N * Ho * Wo * double(cw.cout) * cw.k * cw.k * cw.cin : 0.0;   // algorithmic FLOPs once
    *conv_flops += L.flops;
    ops->push_back(gemm_op(key + (g < nseg ? ".hi" + std::to_string(g) : ".cross"), d, ChainDesc{}, L));
  }
  FinishParams f{};
  f.acc = accbuf; f.bias = cw.bias; f.act = act; f.npix = static_cast<long long>(in.N) * Ho * Wo; f.C = cw.cout;
  f.out = reinterpret_cast<float*>(out.p); f.out_cs = out.cs; f.out_co = out.co;
  if (res) { f.res = reinterpret_cast<const float*>(res->p); f.res_cs = res->cs; f.res_co = res->co; }
  cc_op_io io = op_io({operand(accbuf, CC_OP_F32, in.N, Ho, Wo, cw.cout), operand(cw.bias, CC_OP_F32, 1, 1, 1, cw.cout)},
                      {operand(out, in.N, Ho, Wo)});
  if (res) io.in[io.n_in++] = operand(*res, in.N, Ho, Wo);
  io.act = act;
  ops->push_back(plan_op(key, "finish_f32", io, [f](const PlanIO&, cudaStream_t st) { return finish_f32_launch(f, st); }));
  return CC_OK;
}
// The two first convs of a detect-head scale read the same input and are fused into one conv of 64 + d output channels —
// unless that sum only tiles in narrow blocks (the conv kernel tiles Cout by its largest divisor that is a multiple of 16
// and at most 256: 64 + 240 = 304 = 16 x 19 would run 19 blocks of 16, measured 7 ms of a 14 ms YOLOv9-m step).
static bool head_fuse_ok(int d) {
  const int c = 64 + d;
  for (int bn = (c < 256 ? c : 256) & ~15; bn >= 64; bn -= 16)
    if (c % bn == 0) return true;
  return false;
}

// ------------------------------------------------------------------------------------------------ plan builder
struct Builder {
  YoloModel& M;
  YoloPlan& P;
  int rc = CC_OK;
  std::vector<T> outs;                      // per layer output (tuple outputs: see cbl)
  std::vector<std::vector<T>> cbl_chunks;   // per layer: CBLinear chunks
  struct Place { int concat; int co; };
  std::map<int, Place> place;               // layer -> slice of a concat buffer
  std::map<int, T> concat_buf;              // concat layer -> buffer
  std::vector<int> outC;                    // inferred channels per layer
  // a Conv layer whose only reader is the next layer's ELAN cv1: its conv is queued there, chained with that cv1
  struct Deferred { std::string key; T in, out; int stride = 1, layer = -1; } deferred;
  std::vector<int> folded;                  // layers whose output a chained launch never stored

  Bump bump;                                // workspace carving; bump.dry = measuring pass (no launches are built)
  size_t scratch_bytes = 0;                 // fp32-accurate mode: size of the plane-split scratch (from the measuring pass)
  size_t max_scratch = 0;                   //   ... largest split any conv of this plan needs
  __nv_bfloat16* scratch = nullptr;
  size_t acc_bytes = 0, max_acc = 0;        //   ... and the fp32 partial-sum buffer of the split accumulation
  float* accbuf = nullptr;

  Builder(YoloModel& m, YoloPlan& p) : M(m), P(p) {}

  void* dalloc(size_t bytes) {
    if (rc) return nullptr;
    void* d = bump.take(bytes);
    P.alloc_bytes = bump.off;
    return d;
  }
  T talloc(int C, int H, int W) {
    T t; t.cs = C; t.co = 0; t.C = C; t.N = P.B; t.H = H; t.W = W; t.f32 = M.precise;
    t.p = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(P.B) * H * W * C * (M.precise ? 4 : 2)));
    return t;
  }
  static T slice(const T& t, int co, int C) { T s = t; s.co = t.co + co; s.C = C; return s; }

  // conv: in -> out slice, a tensor of the plan or a dense fp32 map (dense_f32)
  void conv(const std::string& key, const TSlice& in, const TSlice& out, int stride, int act, const TSlice* res = nullptr,
            const float* pre = nullptr, int pre_h = 0, int pre_w = 0) {
    if (rc) return;
    auto it = M.convs.find(key);
    if (it == M.convs.end()) { set_error("yolo plan: conv '%s' not loaded", key.c_str()); rc = CC_ERR_STATE; return; }
    const ConvW& cw = it->second;
    if (cw.cin != in.C) { set_error("yolo plan: conv '%s' expects Cin=%d, got %d", key.c_str(), cw.cin, in.C); rc = CC_ERR_INVALID; return; }
    if (cw.cout != out.C) { set_error("yolo plan: conv '%s' writes Cout=%d, its output has %d", key.c_str(), cw.cout, out.C); rc = CC_ERR_INVALID; return; }
    if (M.precise) {
      if (!(cw.groups == 1 && tc_ok(cw.cin, cw.cout))) {
        set_error("yolo plan: conv '%s' (%d->%d, groups %d) has no tensor-core form; the fp32-accurate mode needs one", key.c_str(), cw.cin, cw.cout, cw.groups);
        rc = CC_ERR_INVALID;
        return;
      }
      const size_t need = static_cast<size_t>(P.B) * in.H * in.W * 6 * in.C * 2;
      if (need > max_scratch) max_scratch = need;
      const size_t need_acc = static_cast<size_t>(P.B) * conv_out(in.H, stride) * conv_out(in.W, stride) * cw.cout * 4;
      if (need_acc > max_acc) max_acc = need_acc;
    }
    if (bump.dry) return;
    if (M.precise) {
      rc = precise_conv_ops(key, cw, in, stride, act, scratch, accbuf, out, res, M.sms, &P.ops, &P.conv_flops);
      return;
    }
    ConvDesc d = conv_desc(in, cw.w, cw.bias, cw.k, stride, out, act, res);
    d.pre = pre; d.pre_h = pre_h; d.pre_w = pre_w;
    if (cw.groups == 1 && tc_ok(cw.cin, cw.cout)) {
      GemmLaunch L;
      rc = conv_gemm_build(d, M.sms, &L);
      if (rc) return;
      P.conv_flops += L.flops;
      P.ops.push_back(gemm_op(key, d, ChainDesc{}, L));
    } else {   // the direct kernel's FLOPs count in conv_flops; its op reports none
      const DirectConvParams p = direct_conv_params(d, cw.groups);
      P.conv_flops += 2.0 * P.B * p.Hout * p.Wout * cw.cout * (cw.cin / cw.groups) * cw.k * cw.k;
      const cc_conv_op c = conv_op_of(p);
      PlanOp op = plan_op(key, "conv_direct", conv_io(c), [p](const PlanIO&, cudaStream_t st) { return conv_direct_launch(p, st); });
      op.conv = c;
      P.ops.push_back(std::move(op));
    }
  }
  // conv key1 (in -> out1) followed by the 1x1 conv key2 over in2, a slice of out1's buffer that starts inside out1 and may
  // run past its end (the partner: channels another conv wrote), into out2 (a tensor or a dense fp32 map).  One chained
  // launch (conv_gemm_chain_build) when the pair chains, and then out1 is written only when keep1; else the two convs.
  // Returns whether the pair was chained.
  bool conv_pair(const std::string& key1, const TSlice& in, const TSlice& out1, int stride, const TSlice* res, const std::string& key2,
                 const TSlice& in2, const TSlice& out2, int act2, bool keep1) {
    if (rc) return false;
    auto i1 = M.convs.find(key1), i2 = M.convs.find(key2);
    if (!bump.dry && !M.precise && i1 != M.convs.end() && i2 != M.convs.end()) {
      const ConvW& c1 = i1->second;
      const ConvW& c2 = i2->second;
      const int part_c = in2.co + in2.C - (out1.co + out1.C);
      if (c1.groups == 1 && tc_ok(c1.cin, c1.cout) && c1.cin == in.C && c1.cout == out1.C && c2.groups == 1 && c2.k == 1 &&
          c2.cin == in2.C && c2.cout == c2.cin && c2.cout == out2.C && in2.p == out1.p && in2.cs == out1.cs && in2.co >= out1.co &&
          in2.co < out1.co + out1.C) {
        const ConvDesc d = conv_desc(in, c1.w, c1.bias, c1.k, stride, out1, CC_ACT_SILU, res);
        ChainDesc c{};
        c.w = c2.w; c.bias = c2.bias; c.act = act2; c.k0 = in2.co - out1.co;
        if (part_c > 0) c.part = nhwc_slice(in2.p, in2.cs, out1.co + out1.C, part_c);
        c.out = out2;
        c.store1 = keep1;
        GemmLaunch L;
        if (conv_gemm_chain_build(d, c, M.sms, &L) == CC_OK) {
          P.conv_flops += L.flops;
          P.ops.push_back(gemm_op(key1 + "+" + key2, d, c, L));
          return true;
        }
      }
    }
    conv(key1, in, out1, stride, CC_ACT_SILU, res);   // the pair does not chain here (shape, tile width, smem, fp32 mode)
    conv(key2, in2, out2, 1, act2);
    return false;
  }
  // a pool or upsample kernel from slice `in` to slice `out`
  void simple(const char* kind, int (*launch)(const TSlice&, const TSlice&, cudaStream_t), const TSlice& in, const TSlice& out,
              const char* name) {
    if (rc || bump.dry) return;
    P.ops.push_back(plan_op(name, kind, op_io({operand(in)}, {operand(out)}), [launch, in, out](const PlanIO&, cudaStream_t st) { return launch(in, out, st); }, 0,
                            slice_bytes(in) + slice_bytes(out)));
  }

  // destination of layer i's output: a slice of a later concat buffer, or a fresh buffer
  T out_for(int i, int C, int H, int W) {
    auto it = place.find(i);
    if (it == place.end()) return talloc(C, H, W);
    const int ci = it->second.concat;
    if (!concat_buf.count(ci)) concat_buf[ci] = talloc(outC[ci], H, W);
    return slice(concat_buf[ci], it->second.co, C);
  }

  // RepNCSP (detection/yolov9.py:92-105) on `x` (2b channels) -> fresh 2b-channel tensor.  t1 = [x1 | x3] = cv1+cv2(x); the
  // caller may already have queued that conv (chained onto x's producer) into `t1_done`.  The last bottleneck's cv2 and cv3
  // over [x1 | x3] run as one chained launch where they can (x1's final value is then never stored).
  T repncsp(const std::string& pfx, const T& x, int b, int n, const T* t1_done = nullptr) {
    T t1 = t1_done ? *t1_done : talloc(2 * b, x.H, x.W);    // [x1 | x3]
    if (!t1_done) conv(pfx + ".cv1+cv2", x, t1, 1, CC_ACT_SILU);
    T x1 = slice(t1, 0, b);
    T o = talloc(2 * b, x.H, x.W);
    if (n == 0) conv(pfx + ".cv3", t1, o, 1, CC_ACT_SILU);
    for (int i = 0; i < n; ++i) {
      T t2 = talloc(b, x.H, x.W);
      conv(pfx + ".m." + std::to_string(i) + ".cv1", x1, t2, 1, CC_ACT_SILU);
      if (i + 1 < n) conv(pfx + ".m." + std::to_string(i) + ".cv2", t2, x1, 1, CC_ACT_SILU, &x1);   // x + cv2(cv1(x)), in place
      else conv_pair(pfx + ".m." + std::to_string(i) + ".cv2", t2, x1, 1, &x1, pfx + ".cv3", t1, o, CC_ACT_SILU, false);
    }
    return o;
  }


  int build();
};

static int layer_out_channels(const Layer& l, const std::vector<int>& outC, int idx) {
  auto src = [&](int f) { return f == -1 ? outC[idx - 1] : outC[f]; };
  switch (l.op) {
    case L_CONV: return l.b;
    case L_ELAN1: return l.b;
    case L_ELAN4: return l.c;
    case L_ADOWN: return 2 * l.a;
    case L_ACONV: return l.b;
    case L_SPPELAN: return l.c;
    case L_UPSAMPLE: return src(l.f[0]);
    case L_CONCAT: return src(l.f[0]) + src(l.f[1]);
    case L_SILENCE: return 3;
    case L_CBLINEAR: { int s = 0; for (int c : l.list) s += c; return s; }
    case L_CBFUSE: return src(l.f.back());
    case L_DETECT: return 0;
  }
  return 0;
}

// Upsample -> Concat(-1, skip) -> RepNCSPELAN4: the block's first conv is a 1x1 over concat(upsample(a), b), and a 1x1 conv
// commutes with nearest upsampling: silu(W [up(a); b] + bias) = silu(up(W_a a) + W_b b + bias).  So W_a runs at HALF resolution
// (a quarter of its FLOPs) into a small fp32 map, and the full-resolution conv over b alone adds it before the activation by
// addressing (GemmParams::pre): the upsample kernel, the concat buffer and half of the conv's input traffic disappear
// (detection/yolov9.py:285-292, :107-125; layers 10-12 and 13-15 of t/s/m/c, 30-32 and 33-35 of e).
static bool fuse_up_concat(const std::vector<Layer>& S, const std::vector<int>& outC, int i, bool precise, int* c_up = nullptr) {
  if (precise || i < 3) return false;
  const Layer& e = S[i];
  if (e.op != L_ELAN4 || e.f.size() != 1 || e.f[0] != -1) return false;
  const Layer& c = S[i - 1];
  if (c.op != L_CONCAT || c.f[0] != -1 || S[i - 2].op != L_UPSAMPLE || S[i - 2].f[0] != -1) return false;
  const int cu = outC[i - 2], cskip = outC[i - 1] - cu;
  if (cu % 16 || cskip % 16 || cu <= 0 || cskip <= 0 || (4 * e.b) % 16) return false;
  if (c_up) *c_up = cu;
  return true;
}

// Conv layer i feeds only the next layer, an ELAN4 whose cv1 reads it whole (not the fused Upsample -> Concat form): the conv
// can run with that cv1 chained in its epilogue and its own output never stored.
static bool conv_feeds_only_elan(const std::vector<Layer>& S, const std::vector<int>& outC, int i, bool precise) {
  const int nl = static_cast<int>(S.size());
  if (i + 1 >= nl || S[i + 1].op != L_ELAN4 || S[i + 1].f.size() != 1 || S[i + 1].f[0] != -1) return false;
  if (fuse_up_concat(S, outC, i + 1, precise)) return false;
  for (int j = 0; j < nl; ++j)
    for (int f : S[j].f)
      if (j != i + 1 && (f == -1 ? j - 1 : f) == i) return false;
  return true;
}

int Builder::build() {
  const std::vector<Layer>& S = M.spec;
  const int nl = static_cast<int>(S.size());
  outC.assign(nl, 0);
  for (int i = 0; i < nl; ++i) outC[i] = layer_out_channels(S[i], outC, i);
  // concat placement: each source of a Concat writes directly into the concat buffer
  for (int i = 0; i < nl; ++i)
    if (S[i].op == L_CONCAT) {
      const int a = S[i].f[0] == -1 ? i - 1 : S[i].f[0], b = S[i].f[1] == -1 ? i - 1 : S[i].f[1];
      if (i + 1 < nl && fuse_up_concat(S, outC, i + 1, M.precise)) continue;   // never materialised
      if (!place.count(a) && !place.count(b) && S[a].op != L_SILENCE && S[b].op != L_SILENCE) {
        place[a] = {i, 0};
        place[b] = {i, outC[a]};
      }
    }

  // ---- preprocess (detection/yolov9.py:390-404)
  LbGeom g;                       // a frame-table plan has no frame geometry of its own (the postprocess gets it per call)
  if (P.table) {
    P.H = P.Hr = P.Hf; P.W = P.Wr = P.Wf;
  } else {
    g = letterbox_geom(P.Hf, P.Wf, P.res);
    if (int e = require_net(g, P.Hf, P.Wf, P.res)) return e;
    P.H = g.H; P.W = g.W; P.Hr = g.Hr; P.Wr = g.Wr;
  }
  const void* net_in = nullptr;   // filled per run when identity (frames pointer) -> patched in run()
  const bool f32 = P.fmt == CC_FRAME_BGR_F32;
  // the stems read HWC BGR: I420 frames always go through the letterbox, which converts them (an identity resize included);
  // a frame-table plan always letterboxes into lb_out (its frames are not one tensor)
  const bool identity = g.new_w == P.Wf && g.new_h == P.Hf && g.px == 0 && g.py == 0 && P.H == g.Hr && P.W == g.Wr;
  if (P.table || P.fmt == CC_FRAME_I420_U8 || !identity) {
    const size_t es = f32 ? 4 : 1;
    P.lb_out = dalloc(static_cast<size_t>(P.B) * P.H * P.W * 3 * es);
    net_in = P.lb_out;
    if (!bump.dry && !P.table) {
      LetterboxParams lb{};
      lb.in = nullptr; lb.out = P.lb_out; lb.fmt = P.fmt;
      lb.B = P.B; lb.Hin = P.Hf; lb.Win = P.Wf; lb.Hr = g.new_h; lb.Wr = g.new_w;
      lb.pad_y = g.py; lb.pad_x = g.px; lb.Hout = P.H; lb.Wout = P.W;
      lb.sx = g.sx; lb.sy = g.sy;
      const double in_px = lb.fmt == CC_FRAME_BGR_F32 ? 12.0 : lb.fmt == CC_FRAME_I420_U8 ? 1.5 : 3.0;   // bytes per pixel
      const double bytes = double(lb.B) * (double(lb.Hin) * lb.Win * in_px + double(lb.Hout) * lb.Wout * 3 * (lb.fmt == CC_FRAME_BGR_F32 ? 4 : 1));
      const int in_type = lb.fmt == CC_FRAME_BGR_F32 ? CC_OP_F32 : CC_OP_U8;
      const cc_operand frames = lb.fmt == CC_FRAME_I420_U8 ? operand(nullptr, CC_OP_U8, lb.B, lb.Hin * 3 / 2, lb.Win, 1)
                                                           : operand(nullptr, in_type, lb.B, lb.Hin, lb.Win, 3);
      P.ops.push_back(plan_op("letterbox", "letterbox", op_io({frames}, {operand(lb.out, in_type, lb.B, lb.Hout, lb.Wout, 3)}), [lb](const PlanIO& io, cudaStream_t st) {
        LetterboxParams q = lb;
        q.in = io.in;
        return letterbox_launch(q, st);
      }, 0, bytes));
    }
  }

  if (M.precise && !bump.dry) {
    scratch = static_cast<__nv_bfloat16*>(dalloc(scratch_bytes));
    accbuf = static_cast<float*>(dalloc(acc_bytes));
  }

  outs.assign(nl, T{});
  cbl_chunks.assign(nl, {});
  T image; image.image = true; image.C = 3; image.H = P.H; image.W = P.W;
  for (int i = 0; i < nl && !rc; ++i) {
    const Layer& l = S[i];
    const std::string pfx = "model." + std::to_string(i);
    auto src = [&](int f) -> const T& { return f == -1 ? outs[i - 1] : outs[f]; };
    T in = (i == 0) ? image : src(l.f[0]);
    T out;
    switch (l.op) {
      case L_SILENCE: out = image; break;
      case L_CONV: {
        if (in.image) {
          CC_REQUIRE(l.a == 3 && l.k == 3 && l.s == 2, "yolo: unexpected image conv");
          out = out_for(i, l.b, in.H / 2, in.W / 2);
          const ConvW& cw = M.convs[pfx];
          if (bump.dry) break;
          // the stems read the letterbox's output, or the call's frames (net_in == nullptr)
          const cc_op_io stem_io = op_io({operand(net_in, f32 ? CC_OP_F32 : CC_OP_U8, P.B, P.H, P.W, 3),
                                          operand(cw.wf32, CC_OP_F32, 1, 1, cw.cout, 27), operand(cw.bias, CC_OP_F32, 1, 1, 1, cw.cout)},
                                         {operand(out)});
          if (!f32 && !M.precise && (cw.cout == 16 || cw.cout == 32 || cw.cout == 64)) {
            // uint8 frames: raw pixel values are exact in bf16, weights bf16(w/255); stem_tc_kernel gathers the A tile from
            // the frame itself
            StemTcParams tc;
            rc = stem_tc_build(P.B, P.H, P.W, cw.wtc, cw.bias, cw.cout, out, &tc);
            if (rc) break;
            const double flops = 2.0 * P.B * (P.H / 2) * (P.W / 2) * cw.cout * 27;
            P.conv_flops += flops;
            P.ops.push_back(plan_op(pfx, "stem_tc", stem_io, [tc, net_in](const PlanIO& io, cudaStream_t st) {
              return stem_tc_launch(tc, static_cast<const uint8_t*>(net_in ? net_in : io.in), st);
            }, flops, double(tc.B) * tc.H * tc.W * 3 + double(tc.Mrows) * tc.Cout * 2));
            break;
          }
          // the CUDA-core stem's FLOPs count in conv_flops; its op reports none
          StemParams sp{};
          sp.in = net_in; sp.is_f32 = f32; sp.B = P.B; sp.H = P.H; sp.W = P.W;
          sp.w = cw.wf32; sp.bias = cw.bias; sp.Cout = cw.cout; sp.out = out;
          P.conv_flops += 2.0 * P.B * (P.H / 2) * (P.W / 2) * cw.cout * 27;
          P.ops.push_back(plan_op(pfx, "stem", stem_io, [sp](const PlanIO& io, cudaStream_t st) {
            StemParams q = sp;
            if (!q.in) q.in = io.in;
            return stem_launch(q, st);
          }));
        } else {
          out = out_for(i, l.b, conv_out(in.H, l.s), conv_out(in.W, l.s));
          if (!place.count(i) && conv_feeds_only_elan(S, outC, i, M.precise)) deferred = {pfx, in, out, l.s, i};
          else conv(pfx, in, out, l.s, CC_ACT_SILU);
        }
        break;
      }
      case L_ELAN1: {
        // detection/yolov9.py:65-80: cv1 -> chunk2 -> cv2 -> cv3 -> cat4 -> cv4
        const int ch1 = l.b, ch2 = l.c, ch3 = l.n;
        T cat = talloc(ch3, in.H, in.W);
        conv(pfx + ".cv1", in, slice(cat, 0, ch1), 1, CC_ACT_SILU);
        conv(pfx + ".cv2", slice(cat, ch1 / 2, ch2), slice(cat, ch1, ch2), 1, CC_ACT_SILU);
        conv(pfx + ".cv3", slice(cat, ch1, ch2), slice(cat, ch1 + ch2, ch2), 1, CC_ACT_SILU);
        out = out_for(i, ch1, in.H, in.W);
        conv(pfx + ".cv4", cat, out, 1, CC_ACT_SILU);
        break;
      }
      case L_ELAN4: {
        // detection/yolov9.py:107-125
        const int b = l.b;
        T cat = talloc(8 * b, in.H, in.W);
        T t1 = talloc(2 * b, in.H, in.W);                  // RepNCSP cv2.0's [x1 | x3]
        if (fuse_up_concat(S, outC, i, M.precise)) {
          const T& lo = outs[i - 3];                       // the Upsample layer's source
          const T& hi = src(S[i - 1].f[1]);                // the Concat's second source
          float* part = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * lo.H * lo.W * 4 * b * 4));
          conv(pfx + ".cv1.lo", lo, dense_f32(part, 4 * b), 1, CC_ACT_NONE);
          conv(pfx + ".cv1.hi", hi, slice(cat, 0, 4 * b), 1, CC_ACT_SILU, nullptr, part, lo.H, lo.W);
          if (!rc && !bump.dry && P.ops.size() >= 2) {
            // algorithmic FLOPs: the pair replaces ONE 1x1 conv over all input channels at full resolution (what the reference
            // computes and SURVEY 8(d) counts); booked on the full-resolution launch, the half-resolution one carries none
            PlanOp& op_hi = P.ops[P.ops.size() - 1];
            PlanOp& op_lo = P.ops[P.ops.size() - 2];
            const double full = 2.0 * P.B * in.H * in.W * double(4 * b) * in.C;
            P.conv_flops += full - op_hi.flops - op_lo.flops;
            op_hi.flops = full;
            op_lo.flops = 0.0;
          }
          conv(pfx + ".cv2.0.cv1+cv2", slice(cat, 2 * b, 2 * b), t1, 1, CC_ACT_SILU);
        } else if (deferred.layer == i - 1) {   // the previous Conv with cv1 chained in its epilogue; its output is not stored
          if (conv_pair(deferred.key, deferred.in, deferred.out, deferred.stride, nullptr, pfx + ".cv1", in, slice(cat, 0, 4 * b),
                        CC_ACT_SILU, false))
            folded.push_back(i - 1);
          deferred.layer = -1;
          conv(pfx + ".cv2.0.cv1+cv2", slice(cat, 2 * b, 2 * b), t1, 1, CC_ACT_SILU);
        } else {   // cv1 -> cat[0, 4b) (kept: cv4 reads it) chained with cv2.0's cv1+cv2 on y1 = cat[2b, 4b)
          conv_pair(pfx + ".cv1", in, slice(cat, 0, 4 * b), 1, nullptr, pfx + ".cv2.0.cv1+cv2", slice(cat, 2 * b, 2 * b), t1, CC_ACT_SILU,
                    true);
        }
        T r1 = repncsp(pfx + ".cv2.0", slice(cat, 2 * b, 2 * b), b, l.n, &t1);
        // cv2.1 -> y2 = cat[4b, 6b) (kept) chained with cv3.0's cv1+cv2 on y2
        T t1b = talloc(2 * b, in.H, in.W);
        conv_pair(pfx + ".cv2.1", r1, slice(cat, 4 * b, 2 * b), 1, nullptr, pfx + ".cv3.0.cv1+cv2", slice(cat, 4 * b, 2 * b), t1b,
                  CC_ACT_SILU, true);
        T r2 = repncsp(pfx + ".cv3.0", slice(cat, 4 * b, 2 * b), b, l.n, &t1b);
        conv(pfx + ".cv3.1", r2, slice(cat, 6 * b, 2 * b), 1, CC_ACT_SILU);
        out = out_for(i, l.c, in.H, in.W);
        conv(pfx + ".cv4", cat, out, 1, CC_ACT_SILU);
        break;
      }
      case L_ADOWN: {
        // detection/yolov9.py:40-52
        const int ch = l.a;
        CC_REQUIRE(in.C == 2 * ch, "yolo: ADown(%d) fed %d channels", ch, in.C);
        T t1 = talloc(ch, in.H, in.W);
        simple("avgpool2_pad", avgpool2_pad_launch, slice(in, 0, ch), t1, "adown.avg");
        out = out_for(i, 2 * ch, in.H / 2, in.W / 2);
        conv(pfx + ".cv1", t1, slice(out, 0, ch), 2, CC_ACT_SILU);
        T t2 = talloc(ch, in.H / 2, in.W / 2);
        simple("avgmax_pool", avgmax_pool_launch, slice(in, ch, ch), t2, "adown.avgmax");
        conv(pfx + ".cv2", t2, slice(out, ch, ch), 1, CC_ACT_SILU);
        break;
      }
      case L_ACONV: {
        // detection/yolov9.py:54-63
        T t1 = talloc(in.C, in.H, in.W);
        simple("avgpool2_pad", avgpool2_pad_launch, in, t1, "aconv.avg");
        out = out_for(i, l.b, in.H / 2, in.W / 2);
        conv(pfx + ".cv1", t1, out, 2, CC_ACT_SILU);
        break;
      }
      case L_SPPELAN: {
        // detection/yolov9.py:134-149
        const int c1 = l.b;
        T cat = talloc(4 * c1, in.H, in.W);
        conv(pfx + ".cv1", in, slice(cat, 0, c1), 1, CC_ACT_SILU);
        if (spp3_supported(cat, c1)) {
          if (!rc && !bump.dry)
            P.ops.push_back(plan_op("spp.max5x3", "spp3", op_io({operand(slice(cat, 0, c1))}, {operand(slice(cat, c1, 3 * c1))}), [cat, c1](const PlanIO&, cudaStream_t st) { return spp3_launch(cat, c1, st); }, 0,
                                    4.0 * cat.N * cat.H * cat.W * c1 * 2));
        } else {
          for (int q = 0; q < 3; ++q) simple("maxpool5", maxpool5_launch, slice(cat, q * c1, c1), slice(cat, (q + 1) * c1, c1), "spp.max5");
        }
        out = out_for(i, l.c, in.H, in.W);
        conv(pfx + ".cv5", cat, out, 1, CC_ACT_SILU);
        break;
      }
      case L_UPSAMPLE: {
        if (i + 2 < nl && fuse_up_concat(S, outC, i + 2, M.precise)) {     // folded into the consumer's first conv: shape only
          out = T{}; out.C = in.C; out.H = in.H * 2; out.W = in.W * 2;
          break;
        }
        out = out_for(i, in.C, in.H * 2, in.W * 2);
        simple("upsample2", upsample2_launch, in, out, "upsample");
        break;
      }
      case L_CONCAT: {
        if (i + 1 < nl && fuse_up_concat(S, outC, i + 1, M.precise)) {     // shape only (see fuse_up_concat)
          const T& skip = src(l.f[1]);
          out = T{}; out.C = outC[i]; out.H = skip.H; out.W = skip.W;
          break;
        }
        if (concat_buf.count(i)) { out = concat_buf[i]; break; }
        // fallback (a source was already placed elsewhere): explicit copy through 1:1 "upsample"-free path not needed
        // for the reference graphs; refuse rather than silently mis-route.
        CC_REQUIRE(false, "yolo: concat %d has no placement", i);
        break;
      }
      case L_CBLINEAR: {
        // detection/yolov9.py:222-228: bare 1x1 conv, split into chunks
        out = talloc(outC[i], in.H, in.W);
        conv(pfx + ".conv", in, out, 1, CC_ACT_NONE);
        int co = 0;
        for (int c : l.list) { cbl_chunks[i].push_back(slice(out, co, c)); co += c; }
        break;
      }
      case L_CBFUSE: {
        // detection/yolov9.py:230-245
        const T& last = src(l.f.back());
        out = out_for(i, last.C, last.H, last.W);
        if (bump.dry) break;
        CBFuseParams cbf{};
        cbf.nsrc = static_cast<int>(l.f.size()) - 1;
        for (int q = 0; q < cbf.nsrc; ++q) {
          const T& ch = cbl_chunks[l.f[q]][l.list[q]];
          CC_REQUIRE(ch.C == last.C, "yolo: CBFuse chunk has %d channels, target %d", ch.C, last.C);
          cbf.src[q] = ch;
        }
        cbf.last = last; cbf.out = out;
        double bytes = slice_bytes(cbf.last) + slice_bytes(cbf.out);
        for (int q = 0; q < cbf.nsrc; ++q) bytes += slice_bytes(cbf.src[q]);
        cc_op_io io = op_io({}, {operand(cbf.out)});
        for (int q = 0; q < cbf.nsrc; ++q) io.in[io.n_in++] = operand(cbf.src[q]);
        io.in[io.n_in++] = operand(cbf.last);
        P.ops.push_back(plan_op(pfx, "cbfuse", io, [cbf](const PlanIO&, cudaStream_t st) { return cbfuse_launch(cbf, st); }, 0, bytes));
        break;
      }
      case L_DETECT: {
        // detection/yolov9.py:157-220 + postprocess :439-458 + scale_boxes :406-421
        const int d = l.a;
        DecodeParams dec{};
        int A = 0;
        for (int q = 0; q < 3; ++q) {
          const T& x = src(l.f[q]);
          const std::string hp = pfx;
          const std::string sq = std::to_string(q);
          T t0 = talloc(64 + d, x.H, x.W);                     // [box branch 64 | class branch d]
          if (head_fuse_ok(d)) {
            conv(hp + ".cv2+cv3." + sq + ".0", x, t0, 1, CC_ACT_SILU);
          } else {
            conv(hp + ".cv2." + sq + ".0", x, slice(t0, 0, 64), 1, CC_ACT_SILU);
            conv(hp + ".cv3." + sq + ".0", x, slice(t0, 64, d), 1, CC_ACT_SILU);
          }
          T tb = talloc(64, x.H, x.W), tc = talloc(d, x.H, x.W);
          float* bl = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * x.H * x.W * 64 * 4));
          float* cl = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * x.H * x.W * 80 * 4));
          // box branch: cv2.j.1 chained with its 1x1 logits cv2.j.2 (tb is then never stored)
          conv_pair(hp + ".cv2." + sq + ".1", slice(t0, 0, 64), tb, 1, nullptr, hp + ".cv2." + sq + ".2", tb, dense_f32(bl, 64), CC_ACT_NONE, false);
          conv(hp + ".cv3." + sq + ".1", slice(t0, 64, d), tc, 1, CC_ACT_SILU);
          conv(hp + ".cv3." + sq + ".2", tc, dense_f32(cl, 80), 1, CC_ACT_NONE);
          dec.box[q] = bl; dec.cls[q] = cl; dec.h[q] = x.H; dec.w[q] = x.W;
          dec.stride[q] = float(P.H / x.H);
          A += x.H * x.W;
        }
        P.A = A;
        P.pred = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * A * 6 * 4));
        dec.B = P.B; dec.A = A; dec.conf_thr = 0.25f; dec.pred = P.pred; dec.raw = nullptr;
        if (bump.dry) break;
        cc_op_io dio = op_io({}, {operand(P.pred, CC_OP_F32, P.B, 1, A, 6), operand(nullptr, CC_OP_F32, P.B, 84, A, 1)});
        for (int q = 0; q < 3; ++q) dio.in[dio.n_in++] = operand(dec.box[q], CC_OP_F32, P.B, dec.h[q], dec.w[q], 64);
        for (int q = 0; q < 3; ++q) dio.in[dio.n_in++] = operand(dec.cls[q], CC_OP_F32, P.B, dec.h[q], dec.w[q], 80);
        dio.conf_thr = dec.conf_thr;
        P.ops.push_back(plan_op("decode", "decode", dio, [dec](const PlanIO& io, cudaStream_t st) {
          DecodeParams q = dec;
          q.raw = io.raw;
          return decode_launch(q, st);
        }, 0, double(dec.B) * dec.A * ((64 + 80) * 4 + 6 * 4)));
        PostParams& post = P.post;
        post = PostParams{};
        post.pred = P.pred; post.B = P.B; post.A = A; post.max_det = 300; post.iou_thr = 0.45f;
        post.scale = g.scale; post.do_scale = 1;
        post.out = nullptr;
        cc_op_io pio = op_io({operand(P.pred, CC_OP_F32, P.B, 1, A, 6)}, {operand(nullptr, CC_OP_F32, P.B, 1, post.max_det, 6)});
        pio.max_det = post.max_det; pio.iou_thr = post.iou_thr; pio.do_scale = post.do_scale;
        pio.pad_x = post.scale.pad_x; pio.pad_y = post.scale.pad_y; pio.gain = post.scale.gain;
        pio.clip_w = post.scale.clip_w; pio.clip_h = post.scale.clip_h;
        P.ops.push_back(plan_op("postprocess", "postprocess", pio, [post](const PlanIO& io, cudaStream_t st) {
          PostParams q = post;
          q.out = io.out;
          return postprocess_launch(q, st);
        }));
        break;
      }
    }
    outs[i] = out;
  }
  P.n_launch = static_cast<int>(P.ops.size());
  P.layer_outs = outs;
  for (int f : folded) P.layer_outs[f].p = nullptr;   // reported as a folded layer (a shape, no tensor)
  return rc;
}

}  // namespace cc

using namespace cc;

struct cc_yolo { YoloModel m; };

extern "C" {

int cc_yolo_create(const char* size, int n_tensors, const char* const* names, const float* const* h_data,
                   const int64_t* numels, cc_yolo** out) {
  return cc_yolo_create_ex(size, 0, n_tensors, names, h_data, numels, out);
}

int cc_yolo_create_ex(const char* size, int flags, int n_tensors, const char* const* names, const float* const* h_data,
                      const int64_t* numels, cc_yolo** out) {
  CC_REQUIRE(size && out, "cc_yolo_create: null argument");
  CC_REQUIRE((flags & ~CC_YOLO_FP32_ACCURATE) == 0, "cc_yolo_create_ex: unknown flags 0x%x", flags);
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_yolo_create: no sm_90 (H100) device");
  std::unique_ptr<cc_yolo> h(new cc_yolo());
  YoloModel& M = h->m;
  M.size = size;
  M.sms = sms;
  M.precise = (flags & CC_YOLO_FP32_ACCURATE) != 0;
  CC_REQUIRE(build_spec(M.size, &M.spec), "cc_yolo_create: unknown size '%s' (t|s|m|c|e)", size);
  int rc = M.weights.host.fill("cc_yolo_create", n_tensors, names, h_data, numels);
  auto L = [&](const std::string& key, std::vector<std::string> nm, int cin, std::vector<int> couts, int k, int g = 1,
               bool stem = false, int ci_begin = 0, int ci_total = 0, bool with_bias = true) {
    if (rc) return;
    int ct = 0;
    for (int c : couts) ct += c;
    const bool dense = tc_ok(cin, ct);   // grouped convs ride the tensor-core kernel as block-diagonal dense
    rc = M.load_conv(key, nm, cin, couts, k, g, dense || g == 1, stem, ci_begin, ci_total, with_bias);
  };
  std::vector<int> outC(M.spec.size(), 0);
  for (size_t i = 0; i < M.spec.size(); ++i) outC[i] = layer_out_channels(M.spec[i], outC, static_cast<int>(i));
  auto repncsp = [&](const std::string& p, int a, int b, int n) {
    L(p + ".cv1+cv2", {p + ".cv1.conv", p + ".cv2.conv"}, a, {b, b}, 1);
    L(p + ".cv3", {p + ".cv3.conv"}, a, {a}, 1);
    for (int i = 0; i < n; ++i) {
      const std::string q = p + ".m." + std::to_string(i);
      L(q + ".cv1", {q + ".cv1.conv"}, b, {b}, 3);
      L(q + ".cv2", {q + ".cv2.conv"}, b, {b}, 3);
    }
  };
  for (size_t i = 0; i < M.spec.size() && !rc; ++i) {
    const Layer& l = M.spec[i];
    const std::string p = "model." + std::to_string(i);
    switch (l.op) {
      case L_CONV: L(p, {p + ".conv"}, l.a, {l.b}, l.k, 1, l.a == 3); break;
      case L_ELAN1:
        L(p + ".cv1", {p + ".cv1.conv"}, l.a, {l.b}, 1);
        L(p + ".cv2", {p + ".cv2.conv"}, l.c, {l.c}, 3);
        L(p + ".cv3", {p + ".cv3.conv"}, l.c, {l.c}, 3);
        L(p + ".cv4", {p + ".cv4.conv"}, l.n, {l.b}, 1);
        break;
      case L_ELAN4: {
        int c_up = 0;
        if (fuse_up_concat(M.spec, outC, static_cast<int>(i), M.precise, &c_up)) {   // the two input-channel halves of cv1
          L(p + ".cv1.lo", {p + ".cv1.conv"}, c_up, {4 * l.b}, 1, 1, false, 0, l.a, false);
          L(p + ".cv1.hi", {p + ".cv1.conv"}, l.a - c_up, {4 * l.b}, 1, 1, false, c_up, l.a, true);
        } else {
          L(p + ".cv1", {p + ".cv1.conv"}, l.a, {4 * l.b}, 1);
        }
        repncsp(p + ".cv2.0", 2 * l.b, l.b, l.n);
        L(p + ".cv2.1", {p + ".cv2.1.conv"}, 2 * l.b, {2 * l.b}, 3);
        repncsp(p + ".cv3.0", 2 * l.b, l.b, l.n);
        L(p + ".cv3.1", {p + ".cv3.1.conv"}, 2 * l.b, {2 * l.b}, 3);
        L(p + ".cv4", {p + ".cv4.conv"}, 8 * l.b, {l.c}, 1);
        break;
      }
      case L_ADOWN:
        L(p + ".cv1", {p + ".cv1.conv"}, l.a, {l.a}, 3);
        L(p + ".cv2", {p + ".cv2.conv"}, l.a, {l.a}, 1);
        break;
      case L_ACONV: L(p + ".cv1", {p + ".cv1.conv"}, l.a, {l.b}, 3); break;
      case L_SPPELAN:
        L(p + ".cv1", {p + ".cv1.conv"}, l.a, {l.b}, 1);
        L(p + ".cv5", {p + ".cv5.conv"}, 4 * l.b, {l.c}, 1);
        break;
      case L_CBLINEAR: {
        int s = 0;
        for (int c : l.list) s += c;
        L(p + ".conv", {p + ".conv"}, l.a, {s}, 1);
        break;
      }
      case L_DETECT:
        for (int q = 0; q < 3; ++q) {
          const std::string sq = std::to_string(q);
          if (head_fuse_ok(l.a)) {
            L(p + ".cv2+cv3." + sq + ".0", {p + ".cv2." + sq + ".0.conv", p + ".cv3." + sq + ".0.conv"}, l.list[q], {64, l.a}, 3);
          } else {
            L(p + ".cv2." + sq + ".0", {p + ".cv2." + sq + ".0.conv"}, l.list[q], {64}, 3);
            L(p + ".cv3." + sq + ".0", {p + ".cv3." + sq + ".0.conv"}, l.list[q], {l.a}, 3);
          }
          L(p + ".cv2." + sq + ".1", {p + ".cv2." + sq + ".1.conv"}, 64, {64}, 3, 4);
          L(p + ".cv2." + sq + ".2", {p + ".cv2." + sq + ".2"}, 64, {64}, 1, 4);
          L(p + ".cv3." + sq + ".1", {p + ".cv3." + sq + ".1.conv"}, l.a, {l.a}, 3);
          L(p + ".cv3." + sq + ".2", {p + ".cv3." + sq + ".2"}, l.a, {80}, 1);
        }
        break;
      default: break;
    }
  }
  M.weights.host.clear();
  if (rc) return rc;
  *out = h.release();
  return CC_OK;
}

int cc_yolo_destroy(cc_yolo* h) {
  delete h;
  return CC_OK;
}

// frame_fmt is a CC_FRAME_* code; I420 needs even sides (4:2:0 chroma covers 2x2 blocks)
static int check_frame_fmt(const char* who, int fmt, int Hf, int Wf) {
  CC_REQUIRE(fmt == CC_FRAME_BGR_U8 || fmt == CC_FRAME_BGR_F32 || fmt == CC_FRAME_I420_U8,
             "%s: unknown frame format %d (0 = BGR uint8, 1 = BGR float32, 2 = I420)", who, fmt);
  CC_REQUIRE(fmt != CC_FRAME_I420_U8 || (Hf % 2 == 0 && Wf % 2 == 0),
             "%s: an I420 frame needs an even height and width, got %dx%d", who, Hf, Wf);
  return CC_OK;
}

// table: a frame-table plan (Hf x Wf = the net shape, fmt = CC_FRAME_BGR_U8: what its letterbox writes)
static std::string plan_key(int fmt, int B, int Hf, int Wf, int res, bool table) {
  char key[96];
  snprintf(key, sizeof(key), "%s%d,%d,%d,%d,%d", table ? "table:" : "", fmt, B, Hf, Wf, res);
  return key;
}
// workspace bytes a plan of this shape addresses (measuring pass of the builder: no device work)
static int plan_bytes(cc_yolo* h, int fmt, int B, int Hf, int Wf, int res, size_t* bytes, size_t* scratch = nullptr, size_t* accb = nullptr,
                      bool table = false) {
  YoloPlan tmp;
  tmp.B = B; tmp.Hf = Hf; tmp.Wf = Wf; tmp.res = res; tmp.fmt = fmt; tmp.table = table;
  Builder dry(h->m, tmp);
  dry.bump.dry = true;
  int rc = dry.build();
  if (rc) return rc;
  *bytes = dry.bump.off + dry.max_scratch + dry.max_acc + 8192;
  if (scratch) *scratch = dry.max_scratch;
  if (accb) *accb = dry.max_acc;
  return CC_OK;
}
static int get_plan(cc_yolo* h, int fmt, int B, int Hf, int Wf, int res, YoloPlan** out, bool table = false) {
  size_t scratch = 0, accb = 0;   // the measuring pass's fp32-accurate buffer sizes, carved by the real build
  return h->m.plans.get(
      plan_key(fmt, B, Hf, Wf, res, table),
      [&](size_t* bytes) { return plan_bytes(h, fmt, B, Hf, Wf, res, bytes, &scratch, &accb, table); },
      [&](YoloPlan& P, uint8_t* base, size_t* used) {
        P.B = B; P.Hf = Hf; P.Wf = Wf; P.res = res; P.fmt = fmt; P.table = table;
        Builder bld(h->m, P);
        bld.bump.base = base;
        bld.scratch_bytes = scratch;
        bld.acc_bytes = accb;
        const int rc = bld.build();
        *used = bld.bump.off;
        return rc;
      },
      out);
}

int cc_yolo_workspace_bytes(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, size_t* bytes) {
  CC_REQUIRE(h && bytes && B > 0 && Hf > 0 && Wf > 0 && res > 0, "cc_yolo_workspace_bytes: bad argument");
  if (int rc = check_frame_fmt("cc_yolo_workspace_bytes", frame_fmt, Hf, Wf)) return rc;
  return plan_bytes(h, frame_fmt, B, Hf, Wf, res, bytes);
}

int cc_yolo_set_workspace(cc_yolo* h, void* d_workspace, size_t bytes) {
  if (int rc = check_workspace("cc_yolo_set_workspace", h, d_workspace)) return rc;
  return h->m.plans.adopt(d_workspace, bytes);
}

// What a detector call supplies to its plan's ops
static PlanIO frames_io(const void* d_frames, float* d_out, float* d_raw) {
  PlanIO io;
  io.in = d_frames; io.out = d_out; io.raw = d_raw;
  return io;
}

// Runs ops [first, last) of the plan on `st`: from its CUDA graph once the caller has passed the same (frames, out, raw)
// pointers twice in a row, else launch by launch.
static int run_graphed(cc_yolo* h, YoloPlan* P, const void* d_frames, float* d_out, float* d_raw, cudaStream_t st, size_t first = 0,
                       size_t last = SIZE_MAX) {
  if (P->gexec && P->g_frames == d_frames && P->g_out == d_out && P->g_raw == d_raw) {
    CC_CHECK_CUDA(cudaGraphLaunch(P->gexec, st));
    return CC_OK;
  }
  const bool stable = P->ran && P->l_frames == d_frames && P->l_out == d_out && P->l_raw == d_raw;
  P->l_frames = d_frames; P->l_out = d_out; P->l_raw = d_raw; P->ran = true;
  const PlanIO io = frames_io(d_frames, d_out, d_raw);
  if (stable) {
    // second call in a row with these pointers: capture the launch list (on a private stream: nothing executes) and replay
    if (!h->m.cap_stream) CC_CHECK_CUDA(cudaStreamCreateWithFlags(&h->m.cap_stream, cudaStreamNonBlocking));
    if (P->gexec) { cudaGraphExecDestroy(P->gexec); P->gexec = nullptr; }
    cudaGraph_t g = nullptr;
    bool ok = cudaStreamBeginCapture(h->m.cap_stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    if (ok) {
      const int rc = run_ops(P->ops, io, h->m.cap_stream, first, last);
      ok = cudaStreamEndCapture(h->m.cap_stream, &g) == cudaSuccess && rc == CC_OK && g != nullptr;
    }
    if (ok) ok = cudaGraphInstantiate(&P->gexec, g, 0) == cudaSuccess;
    if (g) cudaGraphDestroy(g);
    if (ok) {
      P->g_frames = d_frames; P->g_out = d_out; P->g_raw = d_raw;
      CC_CHECK_CUDA(cudaGraphLaunch(P->gexec, st));
      return CC_OK;
    }
    cudaGetLastError();            // capture is an optimisation: fall through to plain launches
    P->gexec = nullptr;
  }
  return run_ops(P->ops, io, st, first, last);
}

int cc_yolo_forward(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, float* d_out,
                    float* d_raw, void* stream) {
  CC_REQUIRE(h && d_frames && d_out && B > 0 && Hf > 0 && Wf > 0 && res > 0, "cc_yolo_forward: bad argument");
  if (int rc = check_frame_fmt("cc_yolo_forward", frame_fmt, Hf, Wf)) return rc;
  YoloPlan* P = nullptr;
  int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P);
  if (rc) return rc;
  return run_graphed(h, P, d_frames, d_out, d_raw, static_cast<cudaStream_t>(stream));
}

// ---- frame tables: every frame's geometry, the shared net shape, and the letterbox table of a call
static int table_geometry(const char* who, const cc_frame* frames, int B, int res, std::vector<LbGeom>* geo, int* net_h, int* net_w) {
  CC_REQUIRE(frames && B >= 1 && B <= CC_MAX_FRAMES && res > 0, "%s: bad argument (B=%d must be in [1, %d], res %d)", who, B,
             CC_MAX_FRAMES, res);
  geo->assign(B, LbGeom{});
  int H = 0, W = 0, first = -1;
  for (int b = 0; b < B; ++b) {
    const cc_frame& f = frames[b];
    if (!f.data) continue;
    CC_REQUIRE(f.fmt == CC_FRAME_BGR_U8 || f.fmt == CC_FRAME_I420_U8,
               "%s: frame %d has format %d; a frame table takes CC_FRAME_BGR_U8 (0) or CC_FRAME_I420_U8 (2) frames", who, b, f.fmt);
    CC_REQUIRE(f.h > 0 && f.w > 0, "%s: frame %d is %dx%d", who, b, f.h, f.w);
    if (int rc = check_frame_fmt(who, f.fmt, f.h, f.w)) return rc;
    const LbGeom g = letterbox_geom(f.h, f.w, res);
    if (int rc = require_net(g, f.h, f.w, res)) return rc;
    if (first < 0) { first = b; H = g.H; W = g.W; }
    CC_REQUIRE(g.H == H && g.W == W, "%s: frame %d (%dx%d) has net shape %dx%d, frame %d has %dx%d: one call takes one net shape",
               who, b, f.h, f.w, g.H, g.W, first, H, W);
    (*geo)[b] = g;
  }
  CC_REQUIRE(first >= 0, "%s: every one of the %d frames is a padding row", who, B);
  *net_h = H; *net_w = W;
  return CC_OK;
}
static void table_letterbox(const cc_frame* frames, int B, const std::vector<LbGeom>& geo, int H, int W, void* out, LetterboxTable* t) {
  t->out = out; t->B = B; t->Hout = H; t->Wout = W; t->out_f32 = 0;
  for (int b = 0; b < B; ++b) {
    const LbGeom& g = geo[b];
    LetterboxFrame& f = t->f[b];
    f = LetterboxFrame{};
    f.in = frames[b].data;
    if (!f.in) continue;
    f.fmt = frames[b].fmt; f.Hin = frames[b].h; f.Win = frames[b].w; f.Hr = g.new_h; f.Wr = g.new_w;
    f.pad_y = g.py; f.pad_x = g.px; f.sx = g.sx; f.sy = g.sy;
  }
}

int cc_yolo_net_shape(int frame_fmt, int Hf, int Wf, int res, int* net_h, int* net_w) {
  CC_REQUIRE(Hf > 0 && Wf > 0 && res > 0 && net_h && net_w, "cc_yolo_net_shape: bad argument (%dx%d, res %d)", Hf, Wf, res);
  if (int rc = check_frame_fmt("cc_yolo_net_shape", frame_fmt, Hf, Wf)) return rc;
  const LbGeom g = letterbox_geom(Hf, Wf, res);
  if (int rc = require_net(g, Hf, Wf, res)) return rc;
  *net_h = g.H; *net_w = g.W;
  return CC_OK;
}

int cc_yolo_workspace_bytes_frames(cc_yolo* h, const cc_frame* frames, int B, int res, size_t* bytes) {
  CC_REQUIRE(h && bytes, "cc_yolo_workspace_bytes_frames: bad argument");
  std::vector<LbGeom> geo;
  int H = 0, W = 0;
  if (int rc = table_geometry("cc_yolo_workspace_bytes_frames", frames, B, res, &geo, &H, &W)) return rc;
  return plan_bytes(h, CC_FRAME_BGR_U8, B, H, W, res, bytes, nullptr, nullptr, true);
}

int cc_yolo_forward_frames(cc_yolo* h, const cc_frame* frames, int B, int res, float* d_out, float* d_raw, void* stream) {
  CC_REQUIRE(h && d_out, "cc_yolo_forward_frames: bad argument");
  std::vector<LbGeom> geo;
  int H = 0, W = 0;
  if (int rc = table_geometry("cc_yolo_forward_frames", frames, B, res, &geo, &H, &W)) return rc;
  YoloPlan* P = nullptr;
  if (int rc = get_plan(h, CC_FRAME_BGR_U8, B, H, W, res, &P, true)) return rc;
  CC_REQUIRE(!P->ops.empty() && P->post.pred && P->lb_out, "cc_yolo_forward_frames: plan without postprocess");
  LetterboxTable t;
  table_letterbox(frames, B, geo, H, W, P->lb_out, &t);
  std::vector<PostScale> scales(B);
  for (int b = 0; b < B; ++b)
    if (frames[b].data) scales[b] = geo[b].scale;
    else scales[b] = PostScale{0.f, 0.f, 1.f, 0.f, 0.f};     // a padding row: boxes clipped to 0
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  // the letterbox and the postprocess take this call's tables as kernel parameters; the ops between them read and write only
  // the workspace (and d_raw), so their graph does not depend on the table
  if (int rc = letterbox_frames_launch(t, st)) return rc;
  if (int rc = run_graphed(h, P, nullptr, nullptr, d_raw, st, 0, P->ops.size() - 1)) return rc;
  PostParams q = P->post;
  q.out = d_out;
  return postprocess_launch(q, st, scales.data());
}

int cc_yolo_plan_info(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int* net_h, int* net_w, int* anchors,
                      int* launches, double* conv_flops, double* act_bytes) {
  CC_REQUIRE(h, "cc_yolo_plan_info: null handle");
  YoloPlan* P = nullptr;
  if (int rc = check_frame_fmt("cc_yolo_plan_info", frame_fmt, Hf, Wf)) return rc;
  int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P);
  if (rc) return rc;
  if (net_h) *net_h = P->H;
  if (net_w) *net_w = P->W;
  if (anchors) *anchors = P->A;
  if (launches) *launches = P->n_launch;
  if (conv_flops) *conv_flops = P->conv_flops;
  if (act_bytes) *act_bytes = double(P->alloc_bytes);
  return CC_OK;
}

/* Per-op device timing of one forward (CUDA events between launches on `stream`; synchronises at the end).
 * Fills up to `cap` entries: ms[i], flops[i] (algorithmic, 0 for non-conv ops) and a name pointer valid for the
 * life of the process.  Returns the op count through n_ops. */
int cc_yolo_profile(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, float* d_out, int cap,
                    float* ms, double* flops, double* bytes, const char** kinds, const char** names, int* n_ops, void* stream) {
  CC_REQUIRE(h && d_frames && d_out, "cc_yolo_profile: bad argument");
  YoloPlan* P = nullptr;
  if (int rc = check_frame_fmt("cc_yolo_profile", frame_fmt, Hf, Wf)) return rc;
  int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P);
  if (rc) return rc;
  rc = profile_ops(P->ops, frames_io(d_frames, d_out, nullptr), static_cast<cudaStream_t>(stream), cap, ms, flops, bytes, kinds, names);
  if (n_ops) *n_ops = static_cast<int>(P->ops.size());
  return rc;
}

/* In-situ device timeline of one forward (no events between the launches, so programmatic dependent launch overlaps
 * as in production): for every conv_gemm op, globaltimer ns of (first CTA entered, grid dependency released, last CTA
 * exited, then five stamps of CTA 0: first operands landed, all MMAs issued, first accumulator complete, last epilogue group
 * done, exit); zeros for the other ops.  host_ns: [12 * cap].  Synchronises at the end. */
int cc_yolo_trace(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, float* d_out, int cap,
                  unsigned long long* host_ns, const char** kinds, const char** names, double* flops, int* n_ops, void* stream) {
  CC_REQUIRE(h && d_frames && d_out && host_ns, "cc_yolo_trace: bad argument");
  YoloPlan* P = nullptr;
  if (int rc = check_frame_fmt("cc_yolo_trace", frame_fmt, Hf, Wf)) return rc;
  int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P);
  if (rc) return rc;
  const size_t n = P->ops.size();
  unsigned long long* d_trace = nullptr;
  CC_CHECK_CUDA(cudaMalloc(&d_trace, n * 12 * sizeof(unsigned long long)));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(d_trace, 0, n * 12 * sizeof(unsigned long long), st);
  PlanIO io = frames_io(d_frames, d_out, nullptr);
  io.trace = d_trace;
  rc = run_ops(P->ops, io, st);
  if (!rc) {
    cudaError_t e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) {
      const size_t m = n < static_cast<size_t>(cap) ? n : static_cast<size_t>(cap);
      e = cudaMemcpy(host_ns, d_trace, m * 12 * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
      for (size_t i = 0; i < m; ++i) {
        const PlanOp& op = P->ops[i];
        const bool gemm = op.conv.kind == CC_CONV_OP_GEMM || op.conv.kind == CC_CONV_OP_CHAIN;
        if (kinds) kinds[i] = op.kind;
        if (names) names[i] = op.name;
        if (flops) flops[i] = gemm ? op.flops : 0.0;
      }
    }
    if (e != cudaSuccess) { set_error("cc_yolo_trace: %s", cudaGetErrorString(e)); rc = CC_ERR_CUDA; }
  }
  cudaFree(d_trace);
  if (n_ops) *n_ops = static_cast<int>(n);
  return rc;
}

// conv op taps: what each conv launch of the cached plan computes, and the plan run one range of ops at a time
int cc_yolo_op_conv(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int i, cc_conv_op* out) {
  CC_REQUIRE(h, "cc_yolo_op_conv: null handle");
  if (int rc = check_frame_fmt("cc_yolo_op_conv", frame_fmt, Hf, Wf)) return rc;
  YoloPlan* P = nullptr;
  if (int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P)) return rc;
  return op_conv_tap("cc_yolo_op_conv", P->ops, i, out);
}

int cc_yolo_op_io(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int i, cc_op_io* out) {
  CC_REQUIRE(h, "cc_yolo_op_io: null handle");
  if (int rc = check_frame_fmt("cc_yolo_op_io", frame_fmt, Hf, Wf)) return rc;
  YoloPlan* P = nullptr;
  if (int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P)) return rc;
  return op_io_tap("cc_yolo_op_io", P->ops, i, out);
}

int cc_yolo_run_ops(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, int first, int last,
                    float* d_out, float* d_raw, void* stream) {
  CC_REQUIRE(h && d_frames && d_out, "cc_yolo_run_ops: bad argument");
  if (int rc = check_frame_fmt("cc_yolo_run_ops", frame_fmt, Hf, Wf)) return rc;
  YoloPlan* P = nullptr;
  if (int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P)) return rc;
  if (int rc = check_range("cc_yolo_run_ops", first, last, static_cast<int>(P->ops.size()))) return rc;
  return run_ops(P->ops, frames_io(d_frames, d_out, d_raw), static_cast<cudaStream_t>(stream), first, last);
}

// parity tap: copy the output of spec layer `layer` of the cached plan (after a forward) to dense fp32 NHWC
int cc_yolo_layer_output(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int layer, float* d_dst, int* C,
                         int* H, int* W, void* stream) {
  CC_REQUIRE(h, "cc_yolo_layer_output: null handle");
  YoloPlan* P = nullptr;
  if (int rc = check_frame_fmt("cc_yolo_layer_output", frame_fmt, Hf, Wf)) return rc;
  int rc = get_plan(h, frame_fmt, B, Hf, Wf, res, &P);
  if (rc) return rc;
  CC_REQUIRE(layer >= 0 && layer < static_cast<int>(P->layer_outs.size()), "cc_yolo_layer_output: bad layer %d", layer);
  const T& t = P->layer_outs[layer];
  if (C) *C = (t.image || !t.p) ? 0 : t.C;      // layers folded into their consumer have a shape but no tensor
  if (H) *H = t.H;
  if (W) *W = t.W;
  if (!d_dst || t.image || !t.p) return CC_OK;
  return slice_to_f32_launch(t, d_dst, static_cast<cudaStream_t>(stream));
}

// kernel-level taps for the parity tests
int cc_detect_postprocess(const float* d_pred, int B, int A, int max_det, float iou_thr, int do_scale, float pad_x,
                          float pad_y, float gain, float clip_w, float clip_h, float* d_out, void* stream) {
  PostParams p{};
  p.pred = d_pred; p.B = B; p.A = A; p.max_det = max_det; p.iou_thr = iou_thr;
  p.do_scale = do_scale; p.scale = PostScale{pad_x, pad_y, gain, clip_w, clip_h};
  p.out = d_out;
  return postprocess_launch(p, static_cast<cudaStream_t>(stream));
}

int cc_detect_pred_from_raw(const float* d_raw, int B, int n_classes, int A, float conf_thr, float* d_pred, void* stream) {
  return pred_from_raw_launch(d_raw, B, A, n_classes, conf_thr, d_pred, static_cast<cudaStream_t>(stream));
}

int cc_detect_decode(const float* const* d_box, const float* const* d_cls, const int* hs, const int* ws, int B,
                     float conf_thr, float* d_pred, float* d_raw, void* stream) {
  DecodeParams p{};
  int A = 0;
  const float strides[3] = {8.f, 16.f, 32.f};
  for (int q = 0; q < 3; ++q) {
    p.box[q] = d_box[q]; p.cls[q] = d_cls[q]; p.h[q] = hs[q]; p.w[q] = ws[q]; p.stride[q] = strides[q];
    A += hs[q] * ws[q];
  }
  p.B = B; p.A = A; p.conf_thr = conf_thr; p.pred = d_pred; p.raw = d_raw;
  return decode_launch(p, static_cast<cudaStream_t>(stream));
}

int cc_letterbox(const void* d_in, int frame_fmt, int B, int Hin, int Win, int res, void* d_out, int* out_h, int* out_w,
                 void* stream) {
  if (int rc = check_frame_fmt("cc_letterbox", frame_fmt, Hin, Win)) return rc;
  const LbGeom g = letterbox_geom(Hin, Win, res);
  if (out_h) *out_h = g.Hr;
  if (out_w) *out_w = g.Wr;
  if (!d_out) return CC_OK;   // size query
  LetterboxParams p{};
  p.in = d_in; p.out = d_out; p.fmt = frame_fmt; p.B = B; p.Hin = Hin; p.Win = Win; p.Hr = g.new_h; p.Wr = g.new_w;
  p.pad_y = g.py; p.pad_x = g.px; p.Hout = g.Hr; p.Wout = g.Wr;
  p.sx = g.sx; p.sy = g.sy;
  return letterbox_launch(p, static_cast<cudaStream_t>(stream));
}

int cc_letterbox_frames(const cc_frame* frames, int B, int res, void* d_out, int* net_h, int* net_w, void* stream) {
  std::vector<LbGeom> geo;
  int H = 0, W = 0;
  if (int rc = table_geometry("cc_letterbox_frames", frames, B, res, &geo, &H, &W)) return rc;
  if (net_h) *net_h = H;
  if (net_w) *net_w = W;
  if (!d_out) return CC_OK;   // size query
  LetterboxTable t;
  table_letterbox(frames, B, geo, H, W, d_out, &t);
  return letterbox_frames_launch(t, static_cast<cudaStream_t>(stream));
}

static size_t al256(size_t b) { return (b + 255) & ~size_t(255); }
static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int cc_stem(const void* d_frames, int frame_f32, int B, int H, int W, const float* h_w, const float* h_bias, int Cout, void* d_out,
            int out_cs, int out_co, int out_f32, int impl, void* d_ws, size_t ws_bytes, size_t* ws_needed, void* stream) {
  CC_REQUIRE(impl == 1 || impl == 2, "cc_stem: unknown impl %d (1 = stem_tc, 2 = stem_kernel)", impl);
  CC_REQUIRE((frame_f32 == 0 || frame_f32 == 1) && (out_f32 == 0 || out_f32 == 1), "cc_stem: frame_f32 and out_f32 are 0 or 1");
  CC_REQUIRE(B >= 1 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0 && Cout >= 8 && Cout % 8 == 0,
             "cc_stem: bad shape B=%d H=%d W=%d Cout=%d (even frame sides, Cout a multiple of 8)", B, H, W, Cout);
  CC_REQUIRE(impl == 2 || (!frame_f32 && !out_f32 && (Cout == 16 || Cout == 32 || Cout == 64)),
             "cc_stem: stem_tc takes uint8 frames and writes bf16, Cout 16, 32 or 64");
  CC_REQUIRE(out_co >= 0 && out_co % 8 == 0 && out_cs % 8 == 0 && out_co + Cout <= out_cs,
             "cc_stem: bad output slice cs=%d co=%d for Cout=%d (multiples of 8 channels)", out_cs, out_co, Cout);
  const size_t need = al256(size_t(Cout) * 27 * 4) + al256(size_t(Cout) * 32 * 2) + al256(size_t(Cout) * 4);
  if (ws_needed) *ws_needed = need;
  if (!d_out) return CC_OK;   // workspace size query
  CC_REQUIRE(d_frames && h_w && h_bias, "cc_stem: d_frames, h_w and h_bias must not be NULL");
  CC_REQUIRE(ws_bytes >= need && d_ws, "cc_stem: workspace of %zu bytes too small (%zu needed)", d_ws ? ws_bytes : size_t(0), need);
  CC_REQUIRE(al16(d_out) && al16(d_ws) && (!frame_f32 || (reinterpret_cast<uintptr_t>(d_frames) & 3) == 0),
             "cc_stem: d_out and d_ws must be 16-byte aligned, float frames 4-byte aligned");
  std::vector<float> wf(static_cast<size_t>(Cout) * 27);
  stem_weights_rsc(h_w, Cout, wf.data());
  const std::vector<__nv_bfloat16> wt = stem_tc_weights(wf.data(), Cout);
  uint8_t* ws = static_cast<uint8_t*>(d_ws);
  float* dwf = reinterpret_cast<float*>(ws);
  __nv_bfloat16* dwt = reinterpret_cast<__nv_bfloat16*>(ws + al256(wf.size() * 4));
  float* db = reinterpret_cast<float*>(ws + al256(wf.size() * 4) + al256(wt.size() * 2));
  const TSlice out = nhwc_slice(d_out, out_cs, out_co, Cout, out_f32, B, H / 2, W / 2);
  StemTcParams tc{};
  if (impl == 1)
    if (int rc = stem_tc_build(B, H, W, dwt, db, Cout, out, &tc)) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CC_CHECK_CUDA(cudaMemcpyAsync(dwf, wf.data(), wf.size() * 4, cudaMemcpyHostToDevice, st));
  CC_CHECK_CUDA(cudaMemcpyAsync(dwt, wt.data(), wt.size() * 2, cudaMemcpyHostToDevice, st));
  CC_CHECK_CUDA(cudaMemcpyAsync(db, h_bias, size_t(Cout) * 4, cudaMemcpyHostToDevice, st));
  if (impl == 1) return stem_tc_launch(tc, static_cast<const uint8_t*>(d_frames), st);
  StemParams p{};
  p.in = d_frames; p.is_f32 = frame_f32; p.B = B; p.H = H; p.W = W; p.w = dwf; p.bias = db; p.Cout = Cout; p.out = out;
  return stem_launch(p, st);
}

int cc_conv2d_fp32_accurate(const float* d_in, int N, int Hin, int Win, int in_cs, int in_co, int Cin, const float* h_w,
                            const float* h_bias, int Cout, int k, int stride, int act, const float* d_res, int res_cs, int res_co,
                            float* d_out, int out_cs, int out_co, void* d_ws, size_t ws_bytes, size_t* ws_needed, void* stream) {
  CC_REQUIRE((k == 1 && stride == 1) || (k == 3 && (stride == 1 || stride == 2)),
             "cc_conv2d_fp32_accurate: k=%d stride=%d (k 1 with stride 1, or k 3 with stride 1 or 2)", k, stride);
  CC_REQUIRE(act == CC_ACT_NONE || act == CC_ACT_SILU, "cc_conv2d_fp32_accurate: act %d (0 none, 1 SiLU)", act);
  CC_REQUIRE(N >= 1 && Hin >= 1 && Win >= 1 && (stride == 1 || (Hin % 2 == 0 && Win % 2 == 0)),
             "cc_conv2d_fp32_accurate: bad shape N=%d Hin=%d Win=%d (even sides for stride 2)", N, Hin, Win);
  CC_REQUIRE(Cin >= 16 && Cin % 16 == 0 && Cout >= 16 && Cout % 16 == 0,
             "cc_conv2d_fp32_accurate: Cin=%d Cout=%d (multiples of 16)", Cin, Cout);
  CC_REQUIRE(in_co >= 0 && in_co % 4 == 0 && in_cs % 4 == 0 && in_co + Cin <= in_cs && out_co >= 0 && out_co % 4 == 0 &&
                 out_cs % 4 == 0 && out_co + Cout <= out_cs && (!d_res || (res_co >= 0 && res_co % 4 == 0 && res_cs % 4 == 0 && res_co + Cout <= res_cs)),
             "cc_conv2d_fp32_accurate: bad slice (cs, co multiples of 4 channels, the slice inside the row)");
  const int Ho = conv_out(Hin, stride), Wo = conv_out(Win, stride);
  std::vector<int> seg_off, seg_c;
  hi_segments(Cin, k, &seg_off, &seg_c);
  const size_t rows = static_cast<size_t>(Cout) * k * k;
  const size_t planes_b = al256(static_cast<size_t>(N) * Hin * Win * 6 * Cin * 2), acc_b = al256(static_cast<size_t>(N) * Ho * Wo * Cout * 4);
  const size_t w5_b = al256(rows * 5 * Cin * 2), bias_b = al256(size_t(Cout) * 4);
  size_t need = planes_b + acc_b + w5_b + bias_b;
  for (int c : seg_c) need += al256(rows * c * 2);
  if (ws_needed) *ws_needed = need;
  if (!d_out) return CC_OK;   // workspace size query
  CC_REQUIRE(d_in && h_w, "cc_conv2d_fp32_accurate: d_in and h_w must not be NULL");
  CC_REQUIRE(ws_bytes >= need && d_ws, "cc_conv2d_fp32_accurate: workspace of %zu bytes too small (%zu needed)", d_ws ? ws_bytes : size_t(0), need);
  CC_REQUIRE(al16(d_in) && al16(d_out) && al16(d_res) && al16(d_ws), "cc_conv2d_fp32_accurate: device pointers must be 16-byte aligned");
  const int sms = device_sm_count();
  CC_REQUIRE(sms > 0, "cc_conv2d_fp32_accurate: no sm_90 (H100) device");
  // PyTorch [Cout][Cin][k][k] -> the kernel layout [Cout][k][k][Cin], then the planes exactly as the plan's weights
  std::vector<float> wf(rows * Cin);
  for (int co = 0; co < Cout; ++co)
    for (int ci = 0; ci < Cin; ++ci)
      for (int r = 0; r < k; ++r)
        for (int s = 0; s < k; ++s) wf[((static_cast<size_t>(co) * k + r) * k + s) * Cin + ci] = h_w[((static_cast<size_t>(co) * Cin + ci) * k + r) * k + s];
  std::vector<__nv_bfloat16> w5;
  std::vector<std::vector<__nv_bfloat16>> whi;
  split_weight_planes(wf.data(), rows, Cin, seg_off, seg_c, &w5, &whi);
  uint8_t* ws = static_cast<uint8_t*>(d_ws);
  __nv_bfloat16* planes = reinterpret_cast<__nv_bfloat16*>(ws);  ws += planes_b;
  float* acc = reinterpret_cast<float*>(ws);                     ws += acc_b;
  ConvW cw;
  cw.cin = Cin; cw.cout = Cout; cw.k = k; cw.groups = 1; cw.seg_off = seg_off; cw.seg_c = seg_c;
  cw.w5 = reinterpret_cast<__nv_bfloat16*>(ws);                  ws += w5_b;
  cw.bias = h_bias ? reinterpret_cast<float*>(ws) : nullptr;     ws += bias_b;
  for (size_t i = 0; i < seg_c.size(); ++i) { cw.whi.push_back(reinterpret_cast<__nv_bfloat16*>(ws)); ws += al256(rows * seg_c[i] * 2); }
  const TSlice in = nhwc_slice(d_in, in_cs, in_co, Cin, 1, N, Hin, Win), res = nhwc_slice(d_res, res_cs, res_co, Cout, 1);
  std::vector<PlanOp> ops;
  double flops = 0;
  if (int rc = precise_conv_ops("conv", cw, in, stride, act, planes, acc, nhwc_slice(d_out, out_cs, out_co, Cout, 1), d_res ? &res : nullptr, sms,
                                &ops, &flops))
    return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CC_CHECK_CUDA(cudaMemcpyAsync(cw.w5, w5.data(), w5.size() * 2, cudaMemcpyHostToDevice, st));
  if (h_bias) CC_CHECK_CUDA(cudaMemcpyAsync(cw.bias, h_bias, size_t(Cout) * 4, cudaMemcpyHostToDevice, st));
  for (size_t i = 0; i < whi.size(); ++i)
    CC_CHECK_CUDA(cudaMemcpyAsync(cw.whi[i], whi[i].data(), whi[i].size() * 2, cudaMemcpyHostToDevice, st));
  return run_ops(ops, PlanIO{}, st);
}

}  // extern "C"
