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
#include <cmath>
#include <cstdlib>
#include <map>
#include <memory>
#include <string>
#include <vector>

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
struct HostT { const float* p; long long n; };
struct ConvW {           // device-resident, kernel layout
  __nv_bfloat16* w = nullptr;   // [Cout][k][k][Cin_eff]  (Cin_eff = Cin when dense, Cin/groups when grouped)
  float* wf32 = nullptr;        // stem only: fp32 [Cout][3][3][3]
  __nv_bfloat16* wtc = nullptr; // stem only: bf16 [Cout][32] = w/255 in (r,s,c) order, zero padded (tensor-core uint8 path)
  // fp32-accurate mode: the fp32 weight is split w = hi + mid + lo (three bf16).  w5: [Cout][k][k][5][Cin] = planes
  // hi|mid|lo|hi|mid (the five cross products below 2^-8 of the result, against the activation planes lo|mid|hi|mid|hi);
  // whi[i]: [Cout][k][k][seg_c[i]] = the hi plane of input-channel segment i (the hi x hi products, one GEMM per segment so
  // that no tensor-core accumulator takes more than ~48 MMA steps: the tensor core's fp32 accumulation truncates, and its bias
  // grows with the number of steps into one accumulator — tests/tools/diag_tc_accum.py)
  __nv_bfloat16* w5 = nullptr;
  std::vector<__nv_bfloat16*> whi;
  std::vector<int> seg_off, seg_c;
  float* bias = nullptr;
  int cin = 0, cout = 0, k = 0, groups = 1;   // groups == 1 -> dense (possibly block-diagonal expansion)
};

static __nv_bfloat16 f2bf(float x) { return __float2bfloat16_rn(x); }

struct T { __nv_bfloat16* p = nullptr; int cs = 0, co = 0, C = 0, H = 0, W = 0; bool image = false; bool f32 = false; };   // f32: p is really float*

struct Op {
  enum Kind { GEMM, DIRECT, AVGPAD, AVGMAX, MAXPOOL5, UPSAMPLE, CBFUSE, LETTERBOX, STEM, STEM_IM2COL, STEM_TC, DECODE, POST, SPLIT, FINISH, SPP3 } kind;
  GemmLaunch gemm;
  DirectConvParams direct;
  TSlice s_in, s_out;
  CBFuseParams cbf;
  LetterboxParams lb;
  StemParams stem;
  StemTcParams stem_tc;
  FinishParams fin;
  double flops = 0;          // algorithmic FLOPs of a non-GEMM conv op (stem)
  DecodeParams dec;
  PostParams post;
  std::string name;
};

struct YoloPlan {
  int B = 0, Hf = 0, Wf = 0, res = 0, is_f32 = 0, H = 0, W = 0, A = 0;
  int Hr = 0, Wr = 0;          // the reference's letterboxed extent (H, W are it rounded up to a multiple of 32)
  std::vector<Op> ops;
  size_t alloc_bytes = 0;      // bytes of the handle's shared workspace this plan addresses
  uint64_t gen = 0;            // workspace generation the pointers / TMA descriptors were built against
  uint64_t last_use = 0;       // LRU stamp
  float* pred = nullptr;   // [B,A,6]
  float* raw = nullptr;    // [B,84,A] (allocated lazily when a tap is requested)
  void* lb_out = nullptr;  // letterboxed frames (same dtype as input) or nullptr when identity
  double conv_flops = 0;
  int n_launch = 0;
  std::vector<T> layer_outs;   // per spec layer (parity taps)
  // CUDA graph of the whole launch list (the analogue of the reference's TinyJit capture, utils/helpers.py:214-221).  Kernel
  // arguments are baked into a graph, so it is captured once the caller has passed the same (frames, out, raw) pointers twice
  // in a row — the steady state of a camera loop that reuses its buffers — and replayed while they stay the same.
  cudaGraphExec_t gexec = nullptr;
  const void* g_frames = nullptr; float* g_out = nullptr; float* g_raw = nullptr;      // pointers the graph was captured with
  const void* l_frames = nullptr; float* l_out = nullptr; float* l_raw = nullptr;      // pointers of the previous call
  ~YoloPlan() { if (gexec) cudaGraphExecDestroy(gexec); }
};

struct YoloModel {
  std::string size;
  std::vector<Layer> spec;
  std::map<std::string, HostT> host;     // borrowed pointers, valid only during create
  std::map<std::string, ConvW> convs;
  std::vector<void*> allocs;
  std::map<std::string, std::unique_ptr<YoloPlan>> plans;   // bounded (kMaxPlans, least recently used goes first)
  Arena arena;                 // activation workspace shared by all plans (size of the largest)
  uint64_t tick = 0;
  int sms = 0;
  cudaStream_t cap_stream = nullptr;   // private stream the graphs are captured on (the caller's may be the legacy default stream)
  // fp32-accurate mode (CC_YOLO_FP32_ACCURATE): activations are stored in fp32 and every conv runs on the same wgmma kernel
  // over a 3-way bf16 split of both operands (six plane products, fp32 accumulation): the result carries fp32-level error
  // instead of bf16's 2^-9, at ~6x the tensor work and 2x the activation bytes.  The mode the 1e-3 parity bar is checked in.
  bool precise = false;
  ~YoloModel() { plans.clear(); if (cap_stream) cudaStreamDestroy(cap_stream); for (void* p : allocs) cudaFree(p); }

  int upload(const void* h, size_t bytes, void** d) {
    CC_CHECK_CUDA(cudaMalloc(d, bytes));
    allocs.push_back(*d);
    CC_CHECK_CUDA(cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice));
    return CC_OK;
  }

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
    int co_base = 0;
    for (size_t t = 0; t < names.size(); ++t) {
      auto iw = host.find(names[t] + ".weight"), ib = host.find(names[t] + ".bias");
      CC_REQUIRE(iw != host.end() && ib != host.end(), "yolo: missing weight '%s'", names[t].c_str());
      const int cout = couts[t];
      const int src_cin_g = ci_total / groups;
      CC_REQUIRE(iw->second.n == static_cast<long long>(cout) * src_cin_g * k * k && ib->second.n == cout,
                 "yolo: '%s' has %lld weight / %lld bias elements, expected %lld / %d", names[t].c_str(), iw->second.n,
                 ib->second.n, static_cast<long long>(cout) * src_cin_g * k * k, cout);
      CC_REQUIRE(ci_total == cin || groups == 1, "yolo: '%s': an input-channel sub-range of a grouped conv", names[t].c_str());
      const float* src = iw->second.p;
      const int cpg_out = cout / groups;
      for (int co = 0; co < cout; ++co) {
        const int g = co / cpg_out;
        for (int ci = 0; ci < cin_g; ++ci)
          for (int r = 0; r < k; ++r)
            for (int s = 0; s < k; ++s) {
              const float v = src[((static_cast<size_t>(co) * src_cin_g + ci_begin + ci) * k + r) * k + s];
              const int ci_eff = dense ? g * cin_g + ci : ci;
              if (stem) wf[(static_cast<size_t>(co_base + co) * 9 + r * 3 + s) * 3 + ci] = v;
              else w[((static_cast<size_t>(co_base + co) * k + r) * k + s) * cin_eff + ci_eff] = f2bf(v);
            }
        bias[co_base + co] = with_bias ? ib->second.p[co] : 0.f;
      }
      co_base += cout;
    }
    ConvW cw;
    cw.cin = cin; cw.cout = cout_total; cw.k = k; cw.groups = dense ? 1 : groups;
    int rc;
    if (stem) {
      if ((rc = upload(wf.data(), wf.size() * 4, reinterpret_cast<void**>(&cw.wf32)))) return rc;
      std::vector<__nv_bfloat16> wt(static_cast<size_t>(cout_total) * 32, f2bf(0.f));
      for (int co = 0; co < cout_total; ++co)
        for (int kk = 0; kk < 27; ++kk) wt[static_cast<size_t>(co) * 32 + kk] = f2bf(wf[static_cast<size_t>(co) * 27 + kk] / 255.0f);
      if ((rc = upload(wt.data(), wt.size() * 2, reinterpret_cast<void**>(&cw.wtc)))) return rc;
    }
    else if (!precise) { if ((rc = upload(w.data(), w.size() * 2, reinterpret_cast<void**>(&cw.w)))) return rc; }
    else {
      // the fp32 weights again (w above is already rounded = the hi plane)
      {
        const int steps = cin_eff * k * k / 16;
        const int nseg = (steps + 47) / 48;
        const int unit = cin_eff % 64 == 0 ? 64 : 16;
        int sc = ((cin_eff + nseg - 1) / nseg + unit - 1) / unit * unit;
        for (int off = 0; off < cin_eff; off += sc) { cw.seg_off.push_back(off); cw.seg_c.push_back(std::min(sc, cin_eff - off)); }
      }
      std::vector<__nv_bfloat16> w5(w.size() * 5, f2bf(0.f));
      int cb = 0;
      for (size_t t = 0; t < names.size(); ++t) {
        const float* src = host.find(names[t] + ".weight")->second.p;
        const int cout = couts[t], cpg_out = cout / groups;
        for (int co = 0; co < cout; ++co) {
          const int g = co / cpg_out;
          for (int ci = 0; ci < cin_g; ++ci)
            for (int r = 0; r < k; ++r)
              for (int s2 = 0; s2 < k; ++s2) {
                const float v = src[((static_cast<size_t>(co) * cin_g + ci) * k + r) * k + s2];
                const __nv_bfloat16 hi = f2bf(v);
                const float r1 = v - __bfloat162float(hi);
                const __nv_bfloat16 mid = f2bf(r1);
                const __nv_bfloat16 lo = f2bf(r1 - __bfloat162float(mid));
                const int ci_eff = dense ? g * cin_g + ci : ci;
                __nv_bfloat16* d5 = &w5[(((static_cast<size_t>(cb + co) * k + r) * k + s2) * 5) * cin_eff + ci_eff];
                d5[0] = hi; d5[cin_eff] = mid; d5[2 * cin_eff] = lo; d5[3 * cin_eff] = hi; d5[4 * cin_eff] = mid;
              }
        }
        cb += cout;
      }
      if ((rc = upload(w5.data(), w5.size() * 2, reinterpret_cast<void**>(&cw.w5)))) return rc;
      for (size_t sgi = 0; sgi < cw.seg_off.size(); ++sgi) {
        const int off = cw.seg_off[sgi], sc = cw.seg_c[sgi];
        std::vector<__nv_bfloat16> ws(static_cast<size_t>(cout_total) * k * k * sc);
        for (size_t row = 0; row < static_cast<size_t>(cout_total) * k * k; ++row)
          for (int c = 0; c < sc; ++c) ws[row * sc + c] = w[row * cin_eff + off + c];
        __nv_bfloat16* dptr = nullptr;
        if ((rc = upload(ws.data(), ws.size() * 2, reinterpret_cast<void**>(&dptr)))) return rc;
        cw.whi.push_back(dptr);
      }
    }
    if ((rc = upload(bias.data(), bias.size() * 4, reinterpret_cast<void**>(&cw.bias)))) return rc;
    convs[key] = cw;
    return CC_OK;
  }
};

static bool tc_ok(int cin, int cout) { return cin % 16 == 0 && cout % 16 == 0; }
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
    T t; t.cs = C; t.co = 0; t.C = C; t.H = H; t.W = W; t.f32 = M.precise;
    t.p = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(P.B) * H * W * C * (M.precise ? 4 : 2)));
    return t;
  }
  static T slice(const T& t, int co, int C) { T s = t; s.co = t.co + co; s.C = C; return s; }
  TSlice ts(const T& t) const { TSlice s; s.p = t.p; s.cs = t.cs; s.co = t.co; s.C = t.C; s.N = P.B; s.H = t.H; s.W = t.W; s.f32 = t.f32 ? 1 : 0; return s; }

  // conv: in -> out slice (out.H/W must already be the conv's output extent)
  void conv(const std::string& key, const T& in, const T& out, int stride, int act, const T* res = nullptr,
            float* out_f32 = nullptr, const float* pre = nullptr, int pre_h = 0, int pre_w = 0) {
    if (rc) return;
    auto it = M.convs.find(key);
    if (it == M.convs.end()) { set_error("yolo plan: conv '%s' not loaded", key.c_str()); rc = CC_ERR_STATE; return; }
    const ConvW& cw = it->second;
    if (cw.cin != in.C) { set_error("yolo plan: conv '%s' expects Cin=%d, got %d", key.c_str(), cw.cin, in.C); rc = CC_ERR_INVALID; return; }
    if (M.precise) {
      if (!(cw.groups == 1 && tc_ok(cw.cin, cw.cout))) {
        set_error("yolo plan: conv '%s' (%d->%d, groups %d) has no tensor-core form; the fp32-accurate mode needs one", key.c_str(), cw.cin, cw.cout, cw.groups);
        rc = CC_ERR_INVALID;
        return;
      }
      const size_t need = static_cast<size_t>(P.B) * in.H * in.W * 6 * in.C * 2;
      if (need > max_scratch) max_scratch = need;
      const size_t need_acc = static_cast<size_t>(P.B) * (stride == 2 ? in.H / 2 : in.H) * (stride == 2 ? in.W / 2 : in.W) * cw.cout * 4;
      if (need_acc > max_acc) max_acc = need_acc;
    }
    if (bump.dry) return;
    Op op;
    op.name = key;
    if (M.precise) {
      // fp32 slice -> six bf16 planes [lo|mid|hi|mid|hi|hi] in the scratch; then on the same wgmma conv kernel, all with fp32
      // output into one dense partial-sum buffer: one GEMM per input-channel segment of the hi x hi products (hi plane at
      // channel offset 5C), accumulated with the in-place fp32 residual of the epilogue (one round-to-nearest add), one GEMM
      // for the five cross products (planes 0..4 against the weight planes hi|mid|lo|hi|mid); a last pass applies bias, the
      // exact SiLU and the residual and writes the output slice.
      Op sp; sp.kind = Op::SPLIT; sp.name = key + ".split"; sp.s_in = ts(in); sp.s_out = TSlice{}; sp.s_out.p = scratch;
      P.ops.push_back(std::move(sp));
      const int Ho = stride == 2 ? in.H / 2 : in.H, Wo = stride == 2 ? in.W / 2 : in.W;
      const int nseg = static_cast<int>(cw.seg_off.size());
      for (int g = 0; g <= nseg; ++g) {
        ConvDesc d{};
        d.in = scratch; d.in_cs = 6 * in.C;
        if (g < nseg) { d.in_co = 5 * in.C + cw.seg_off[g]; d.Cin = cw.seg_c[g]; d.w = cw.whi[g]; }
        else { d.in_co = 0; d.Cin = 5 * in.C; d.w = cw.w5; }
        d.N = P.B; d.Hin = in.H; d.Win = in.W; d.k = cw.k; d.stride = stride;
        d.bias = nullptr;
        d.out = accbuf; d.out_cs = cw.cout; d.out_co = 0; d.out_f32 = 1;
        d.Cout = cw.cout; d.act = CC_ACT_NONE;
        if (g > 0) { d.res = accbuf; d.res_cs = cw.cout; d.res_co = 0; }
        Op gop; gop.kind = Op::GEMM; gop.name = key + (g < nseg ? ".hi" + std::to_string(g) : ".cross");
        rc = conv_gemm_build(d, M.sms, &gop.gemm);
        if (rc) return;
        gop.gemm.flops = g == 0 ? 2.0 * P.B * Ho * Wo * double(cw.cout) * cw.k * cw.k * cw.cin : 0.0;   // algorithmic FLOPs once
        P.conv_flops += gop.gemm.flops;
        P.ops.push_back(std::move(gop));
      }
      op.kind = Op::FINISH;
      FinishParams& f = op.fin;
      f = FinishParams{};
      f.acc = accbuf; f.bias = cw.bias; f.act = act; f.npix = static_cast<long long>(P.B) * Ho * Wo; f.C = cw.cout;
      if (out_f32) { f.out = out_f32; f.out_cs = cw.cout; f.out_co = 0; }
      else { f.out = reinterpret_cast<float*>(out.p); f.out_cs = out.cs; f.out_co = out.co; }
      if (res) { f.res = reinterpret_cast<const float*>(res->p); f.res_cs = res->cs; f.res_co = res->co; }
    } else if (cw.groups == 1 && tc_ok(cw.cin, cw.cout)) {
      ConvDesc d{};
      d.in = in.p; d.in_cs = in.cs; d.in_co = in.co; d.Cin = in.C;
      d.N = P.B; d.Hin = in.H; d.Win = in.W; d.k = cw.k; d.stride = stride;
      d.w = cw.w; d.bias = cw.bias;
      if (out_f32) { d.out = out_f32; d.out_cs = cw.cout; d.out_co = 0; d.out_f32 = 1; }
      else { d.out = out.p; d.out_cs = out.cs; d.out_co = out.co; d.out_f32 = 0; }
      d.Cout = cw.cout; d.act = act;
      if (res) { d.res = res->p; d.res_cs = res->cs; d.res_co = res->co; }
      d.pre = pre; d.pre_h = pre_h; d.pre_w = pre_w;
      op.kind = Op::GEMM;
      rc = conv_gemm_build(d, M.sms, &op.gemm);
      if (rc) return;
      P.conv_flops += op.gemm.flops;
    } else {
      DirectConvParams& q = op.direct;
      q = DirectConvParams{};
      q.in = in.p; q.in_cs = in.cs; q.in_co = in.co; q.Cin = in.C;
      q.N = P.B; q.Hin = in.H; q.Win = in.W; q.Hbuf = in.H; q.Wbuf = in.W;
      q.k = cw.k; q.stride = stride; q.pad = cw.k / 2; q.groups = cw.groups;
      q.w = cw.w; q.bias = cw.bias;
      if (out_f32) { q.out = out_f32; q.out_cs = cw.cout; q.out_co = 0; q.out_f32 = 1; }
      else { q.out = out.p; q.out_cs = out.cs; q.out_co = out.co; q.out_f32 = 0; }
      q.Cout = cw.cout;
      q.Hout = stride == 2 ? in.H / 2 : in.H; q.Wout = stride == 2 ? in.W / 2 : in.W;
      q.act = act;
      if (res) { q.res = res->p; q.res_cs = res->cs; q.res_co = res->co; }
      op.kind = Op::DIRECT;
      P.conv_flops += 2.0 * P.B * q.Hout * q.Wout * cw.cout * (cw.cin / cw.groups) * cw.k * cw.k;
    }
    P.ops.push_back(std::move(op));
  }
  void simple(Op::Kind kind, const T& in, const T& out, const char* name) {
    if (rc || bump.dry) return;
    Op op; op.kind = kind; op.s_in = ts(in); op.s_out = ts(out); op.name = name;
    P.ops.push_back(std::move(op));
  }

  // destination of layer i's output: a slice of a later concat buffer, or a fresh buffer
  T out_for(int i, int C, int H, int W) {
    auto it = place.find(i);
    if (it == place.end()) return talloc(C, H, W);
    const int ci = it->second.concat;
    if (!concat_buf.count(ci)) concat_buf[ci] = talloc(outC[ci], H, W);
    return slice(concat_buf[ci], it->second.co, C);
  }

  // RepNCSP (detection/yolov9.py:92-105) on `x` (2b channels) -> fresh 2b-channel tensor
  T repncsp(const std::string& pfx, const T& x, int b, int n) {
    T t1 = talloc(2 * b, x.H, x.W);                         // [x1 | x3]
    conv(pfx + ".cv1+cv2", x, t1, 1, CC_ACT_SILU);
    T x1 = slice(t1, 0, b);
    for (int i = 0; i < n; ++i) {
      T t2 = talloc(b, x.H, x.W);
      conv(pfx + ".m." + std::to_string(i) + ".cv1", x1, t2, 1, CC_ACT_SILU);
      conv(pfx + ".m." + std::to_string(i) + ".cv2", t2, x1, 1, CC_ACT_SILU, &x1);   // x + cv2(cv1(x)), in place
    }
    T o = talloc(2 * b, x.H, x.W);
    conv(pfx + ".cv3", t1, o, 1, CC_ACT_SILU);
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
  static const int env = getenv("CC_FUSE_UP") ? atoi(getenv("CC_FUSE_UP")) : 1;
  if (!env || precise || i < 3) return false;
  const Layer& e = S[i];
  if (e.op != L_ELAN4 || e.f.size() != 1 || e.f[0] != -1) return false;
  const Layer& c = S[i - 1];
  if (c.op != L_CONCAT || c.f[0] != -1 || S[i - 2].op != L_UPSAMPLE || S[i - 2].f[0] != -1) return false;
  const int cu = outC[i - 2], cskip = outC[i - 1] - cu;
  if (cu % 16 || cskip % 16 || cu <= 0 || cskip <= 0 || (4 * e.b) % 16) return false;
  if (c_up) *c_up = cu;
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
  const double r = std::min(double(P.res) / P.Hf, double(P.res) / P.Wf);
  const int new_w = int(std::nearbyint(P.Wf * r)), new_h = int(std::nearbyint(P.Hf * r));
  double dw = double((P.res - new_w) % 32), dh = double((P.res - new_h) % 32);
  if (dw < 0) dw += 32;
  if (dh < 0) dh += 32;
  dw /= 2; dh /= 2;
  const int px = int(std::nearbyint(dw - 0.1)), py = int(std::nearbyint(dh - 0.1));
  // The reference pads int(round(d - 0.1)) on BOTH sides, so when (res - new) % 32 is odd its net input is one pixel short of
  // a multiple of 32 (SURVEY App. A5) — and it keeps going: a 3x3/s2/p1 conv over 2k-1 rows gives the same k output rows as
  // over 2k rows whose last row is zero.  So the net input buffer is rounded up to the multiple of 32 with that zero row /
  // column (the letterbox kernel pads with zeros anyway): identical arithmetic, even dims for the TMA views.  scale_boxes
  // still sees the reference's odd extent (Hr, Wr below).
  const int Hr = new_h + 2 * py, Wr = new_w + 2 * px;
  P.H = (Hr + 31) / 32 * 32; P.W = (Wr + 31) / 32 * 32;
  P.Hr = Hr; P.Wr = Wr;
  CC_REQUIRE(P.H > 0 && P.W > 0 && P.H - Hr <= 1 && P.W - Wr <= 1,
             "yolo: letterboxed input %dx%d is not within one pixel of a multiple of 32 (frame %dx%d, res %d)", Hr, Wr, P.Hf, P.Wf, P.res);
  const void* net_in = nullptr;   // filled per run when identity (frames pointer) -> patched in run()
  if (!(new_w == P.Wf && new_h == P.Hf && px == 0 && py == 0 && P.H == Hr && P.W == Wr)) {
    const size_t es = P.is_f32 ? 4 : 1;
    P.lb_out = dalloc(static_cast<size_t>(P.B) * P.H * P.W * 3 * es);
    net_in = P.lb_out;
    if (!bump.dry) {
    Op op; op.kind = Op::LETTERBOX; op.name = "letterbox";
    op.lb = LetterboxParams{};
    op.lb.in = nullptr; op.lb.out = P.lb_out; op.lb.is_f32 = P.is_f32;
    op.lb.B = P.B; op.lb.Hin = P.Hf; op.lb.Win = P.Wf; op.lb.Hr = new_h; op.lb.Wr = new_w;
    op.lb.pad_y = py; op.lb.pad_x = px; op.lb.Hout = P.H; op.lb.Wout = P.W;
    op.lb.sx = float(double(P.Wf) / double(new_w)); op.lb.sy = float(double(P.Hf) / double(new_h));
    P.ops.push_back(std::move(op));
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
          static const int stem_tc_env = getenv("CC_STEM_TC") ? atoi(getenv("CC_STEM_TC")) : 1;
          if (!P.is_f32 && stem_tc_env && cw.cout % 16 == 0 && !M.precise) {
            // uint8 frames: raw pixel values are exact in bf16, weights bf16(w/255).  Default (CC_STEM_TC=1): stem_tc_kernel
            // gathers the A tile from the frame itself; CC_STEM_TC=2: the earlier im2col to [B*Ho*Wo, 32] + conv_gemm
            const long long Mrows = static_cast<long long>(P.B) * (P.H / 2) * (P.W / 2);
            if (stem_tc_env == 1 && (cw.cout == 16 || cw.cout == 32 || cw.cout == 64)) {
              if (bump.dry) break;
              Op op; op.kind = Op::STEM_TC; op.name = pfx; op.stem = StemParams{}; op.stem.in = net_in;
              rc = stem_tc_build(P.B, P.H, P.W, cw.wtc, cw.bias, cw.cout, ts(out), &op.stem_tc);
              if (rc) break;
              op.flops = 2.0 * Mrows * cw.cout * 27;
              P.conv_flops += op.flops;
              P.ops.push_back(std::move(op));
              break;
            }
            __nv_bfloat16* cols = static_cast<__nv_bfloat16*>(dalloc(static_cast<size_t>(Mrows) * 32 * 2));
            if (bump.dry) break;
            { Op op; op.kind = Op::STEM_IM2COL; op.name = pfx + ".im2col"; op.stem = StemParams{};
              op.stem.in = net_in; op.stem.B = P.B; op.stem.H = P.H; op.stem.W = P.W;
              op.s_out.p = cols; P.ops.push_back(std::move(op)); }
            ConvDesc d{};
            d.in = cols; d.in_cs = 32; d.in_co = 0; d.Cin = 32;
            d.N = 1; d.Hin = 1; d.Win = static_cast<int>(Mrows); d.k = 1; d.stride = 1;
            d.w = cw.wtc; d.bias = cw.bias;
            d.out = out.p; d.out_cs = out.cs; d.out_co = out.co; d.Cout = cw.cout; d.out_f32 = 0; d.act = CC_ACT_SILU;
            Op op; op.kind = Op::GEMM; op.name = pfx;
            rc = conv_gemm_build(d, M.sms, &op.gemm);
            if (rc) break;
            op.gemm.flops = 2.0 * Mrows * cw.cout * 27;
            P.conv_flops += op.gemm.flops;
            P.ops.push_back(std::move(op));
            break;
          }
          if (bump.dry) break;
          Op op; op.kind = Op::STEM; op.name = pfx;
          op.stem = StemParams{};
          op.stem.in = net_in; op.stem.is_f32 = P.is_f32; op.stem.B = P.B; op.stem.H = P.H; op.stem.W = P.W;
          op.stem.w = cw.wf32; op.stem.bias = cw.bias; op.stem.Cout = cw.cout; op.stem.out = ts(out);
          P.conv_flops += 2.0 * P.B * (P.H / 2) * (P.W / 2) * cw.cout * 27;
          P.ops.push_back(std::move(op));
        } else {
          out = out_for(i, l.b, l.s == 2 ? in.H / 2 : in.H, l.s == 2 ? in.W / 2 : in.W);
          conv(pfx, in, out, l.s, CC_ACT_SILU);
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
        if (fuse_up_concat(S, outC, i, M.precise)) {
          const T& lo = outs[i - 3];                       // the Upsample layer's source
          const T& hi = src(S[i - 1].f[1]);                // the Concat's second source
          float* part = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * lo.H * lo.W * 4 * b * 4));
          T dummy;
          conv(pfx + ".cv1.lo", lo, dummy, 1, CC_ACT_NONE, nullptr, part);
          conv(pfx + ".cv1.hi", hi, slice(cat, 0, 4 * b), 1, CC_ACT_SILU, nullptr, nullptr, part, lo.H, lo.W);
          if (!rc && !bump.dry && P.ops.size() >= 2) {
            // algorithmic FLOPs: the pair replaces ONE 1x1 conv over all input channels at full resolution (what the reference
            // computes and SURVEY 8(d) counts); booked on the full-resolution launch, the half-resolution one carries none
            GemmLaunch& g_hi = P.ops[P.ops.size() - 1].gemm;
            GemmLaunch& g_lo = P.ops[P.ops.size() - 2].gemm;
            const double full = 2.0 * P.B * in.H * in.W * double(4 * b) * in.C;
            P.conv_flops += full - g_hi.flops - g_lo.flops;
            g_hi.flops = full;
            g_lo.flops = 0.0;
          }
        } else {
          conv(pfx + ".cv1", in, slice(cat, 0, 4 * b), 1, CC_ACT_SILU);
        }
        T r1 = repncsp(pfx + ".cv2.0", slice(cat, 2 * b, 2 * b), b, l.n);
        conv(pfx + ".cv2.1", r1, slice(cat, 4 * b, 2 * b), 1, CC_ACT_SILU);
        T r2 = repncsp(pfx + ".cv3.0", slice(cat, 4 * b, 2 * b), b, l.n);
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
        simple(Op::AVGPAD, slice(in, 0, ch), t1, "adown.avg");
        out = out_for(i, 2 * ch, in.H / 2, in.W / 2);
        conv(pfx + ".cv1", t1, slice(out, 0, ch), 2, CC_ACT_SILU);
        T t2 = talloc(ch, in.H / 2, in.W / 2);
        simple(Op::AVGMAX, slice(in, ch, ch), t2, "adown.avgmax");
        conv(pfx + ".cv2", t2, slice(out, ch, ch), 1, CC_ACT_SILU);
        break;
      }
      case L_ACONV: {
        // detection/yolov9.py:54-63
        T t1 = talloc(in.C, in.H, in.W);
        simple(Op::AVGPAD, in, t1, "aconv.avg");
        out = out_for(i, l.b, in.H / 2, in.W / 2);
        conv(pfx + ".cv1", t1, out, 2, CC_ACT_SILU);
        break;
      }
      case L_SPPELAN: {
        // detection/yolov9.py:134-149
        const int c1 = l.b;
        T cat = talloc(4 * c1, in.H, in.W);
        conv(pfx + ".cv1", in, slice(cat, 0, c1), 1, CC_ACT_SILU);
        static const int spp3_env = getenv("CC_SPP3") ? atoi(getenv("CC_SPP3")) : 1;
        if (spp3_env && spp3_supported(ts(cat), c1)) {
          if (!rc && !bump.dry) { Op op; op.kind = Op::SPP3; op.s_in = ts(cat); op.s_out = ts(cat); op.s_out.C = c1; op.name = "spp.max5x3"; P.ops.push_back(std::move(op)); }
        } else {
          for (int q = 0; q < 3; ++q) simple(Op::MAXPOOL5, slice(cat, q * c1, c1), slice(cat, (q + 1) * c1, c1), "spp.max5");
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
        simple(Op::UPSAMPLE, in, out, "upsample");
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
        Op op; op.kind = Op::CBFUSE; op.name = pfx;
        op.cbf = CBFuseParams{};
        op.cbf.nsrc = static_cast<int>(l.f.size()) - 1;
        for (int q = 0; q < op.cbf.nsrc; ++q) {
          const T& ch = cbl_chunks[l.f[q]][l.list[q]];
          CC_REQUIRE(ch.C == last.C, "yolo: CBFuse chunk has %d channels, target %d", ch.C, last.C);
          op.cbf.src[q] = ts(ch);
        }
        op.cbf.last = ts(last); op.cbf.out = ts(out);
        P.ops.push_back(std::move(op));
        break;
      }
      case L_DETECT: {
        // detection/yolov9.py:157-220 + postprocess :439-458 + scale_boxes :406-421
        const int d = l.a;
        Op dec; dec.kind = Op::DECODE; dec.name = "decode";
        dec.dec = DecodeParams{};
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
          conv(hp + ".cv2." + sq + ".1", slice(t0, 0, 64), tb, 1, CC_ACT_SILU);
          conv(hp + ".cv3." + sq + ".1", slice(t0, 64, d), tc, 1, CC_ACT_SILU);
          float* bl = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * x.H * x.W * 64 * 4));
          float* cl = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * x.H * x.W * 80 * 4));
          T dummy;
          conv(hp + ".cv2." + sq + ".2", tb, dummy, 1, CC_ACT_NONE, nullptr, bl);
          conv(hp + ".cv3." + sq + ".2", tc, dummy, 1, CC_ACT_NONE, nullptr, cl);
          dec.dec.box[q] = bl; dec.dec.cls[q] = cl; dec.dec.h[q] = x.H; dec.dec.w[q] = x.W;
          dec.dec.stride[q] = float(P.H / x.H);
          A += x.H * x.W;
        }
        P.A = A;
        P.pred = static_cast<float*>(dalloc(static_cast<size_t>(P.B) * A * 6 * 4));
        dec.dec.B = P.B; dec.dec.A = A; dec.dec.conf_thr = 0.25f; dec.dec.pred = P.pred; dec.dec.raw = nullptr;
        if (bump.dry) break;
        P.ops.push_back(std::move(dec));
        Op po; po.kind = Op::POST; po.name = "postprocess";
        po.post = PostParams{};
        po.post.pred = P.pred; po.post.B = P.B; po.post.A = A; po.post.max_det = 300; po.post.iou_thr = 0.45f;
        const int Hr = P.Hr, Wr = P.Wr;               // the reference's img1_shape (detection/yolov9.py:406-416)
        const double gain = std::min(double(Hr) / P.Hf, double(Wr) / P.Wf);
        po.post.gain = float(gain);
        po.post.pad_x = float((Wr - P.Wf * gain) / 2); po.post.pad_y = float((Hr - P.Hf * gain) / 2);
        po.post.clip_w = float(P.Wf); po.post.clip_h = float(P.Hf); po.post.do_scale = 1;
        po.post.out = nullptr;
        P.ops.push_back(std::move(po));
        break;
      }
    }
    outs[i] = out;
  }
  P.n_launch = static_cast<int>(P.ops.size());
  P.layer_outs = outs;
  return rc;
}

static int plan_run(YoloPlan& P, const void* d_frames, float* d_out, float* d_raw, cudaStream_t st,
                    std::vector<cudaEvent_t>* ev = nullptr, unsigned long long* d_trace = nullptr) {
  size_t oi = 0, ti = 0;
  for (Op& op : P.ops) {
    int rc = CC_OK;
    if (ev) cudaEventRecord((*ev)[oi++], st);
    switch (op.kind) {
      case Op::GEMM:
        if (d_trace) { GemmLaunch g = op.gemm; g.p.trace = d_trace + 12 * ti; rc = conv_gemm_launch(g, st); }
        else rc = conv_gemm_launch(op.gemm, st);
        break;
      case Op::DIRECT: rc = conv_direct_launch(op.direct, st); break;
      case Op::AVGPAD: rc = avgpool2_pad_launch(op.s_in, op.s_out, st); break;
      case Op::AVGMAX: rc = avgmax_pool_launch(op.s_in, op.s_out, st); break;
      case Op::MAXPOOL5: rc = maxpool5_launch(op.s_in, op.s_out, st); break;
      case Op::UPSAMPLE: rc = upsample2_launch(op.s_in, op.s_out, st); break;
      case Op::SPP3: rc = spp3_launch(op.s_in, op.s_out.C, st); break;
      case Op::CBFUSE: rc = cbfuse_launch(op.cbf, st); break;
      case Op::LETTERBOX: { LetterboxParams q = op.lb; q.in = d_frames; rc = letterbox_launch(q, st); break; }
      case Op::STEM: { StemParams q = op.stem; if (!q.in) q.in = d_frames; rc = stem_launch(q, st); break; }
      case Op::STEM_IM2COL:
        rc = stem_im2col_launch(static_cast<const uint8_t*>(op.stem.in ? op.stem.in : d_frames), op.s_out.p, op.stem.B, op.stem.H,
                                op.stem.W, st);
        break;
      case Op::STEM_TC:
        rc = stem_tc_launch(op.stem_tc, static_cast<const uint8_t*>(op.stem.in ? op.stem.in : d_frames), st);
        break;
      case Op::DECODE: { DecodeParams q = op.dec; q.raw = d_raw; rc = decode_launch(q, st); break; }
      case Op::POST: { PostParams q = op.post; q.out = d_out; rc = postprocess_launch(q, st); break; }
      case Op::SPLIT: rc = split_planes_launch(op.s_in, op.s_out.p, st); break;
      case Op::FINISH: rc = finish_f32_launch(op.fin, st); break;
    }
    if (rc) return rc;
    ++ti;
  }
  if (ev) cudaEventRecord((*ev)[oi], st);
  return CC_OK;
}

// algorithmic HBM bytes of a memory-bound op (inputs once + outputs once), for the achieved-GB/s figures of the bench line
static double op_bytes(const Op& op) {
  auto sl = [](const TSlice& t) { return double(t.N) * t.H * t.W * t.C * (t.f32 ? 4 : 2); };
  switch (op.kind) {
    case Op::AVGPAD: case Op::AVGMAX: case Op::MAXPOOL5: case Op::UPSAMPLE: return sl(op.s_in) + sl(op.s_out);
    case Op::SPP3: return 4.0 * op.s_in.N * op.s_in.H * op.s_in.W * op.s_out.C * 2;
    case Op::CBFUSE: { double b = sl(op.cbf.last) + sl(op.cbf.out); for (int k = 0; k < op.cbf.nsrc; ++k) b += sl(op.cbf.src[k]); return b; }
    case Op::STEM_TC: return double(op.stem_tc.B) * op.stem_tc.H * op.stem_tc.W * 3 + double(op.stem_tc.Mrows) * op.stem_tc.Cout * 2;
    case Op::LETTERBOX: return double(op.lb.B) * (double(op.lb.Hin) * op.lb.Win + double(op.lb.Hout) * op.lb.Wout) * 3 * (op.lb.is_f32 ? 4 : 1);
    case Op::DECODE: return double(op.dec.B) * op.dec.A * ((64 + 80) * 4 + 6 * 4);
    default: return 0.0;
  }
}

static const char* op_kind_name(Op::Kind k) {
  switch (k) {
    case Op::GEMM: return "conv_gemm"; case Op::DIRECT: return "conv_direct"; case Op::AVGPAD: return "avgpool2_pad";
    case Op::AVGMAX: return "avgmax_pool"; case Op::MAXPOOL5: return "maxpool5"; case Op::UPSAMPLE: return "upsample2";
    case Op::CBFUSE: return "cbfuse"; case Op::LETTERBOX: return "letterbox"; case Op::STEM: return "stem"; case Op::STEM_IM2COL: return "stem_im2col"; case Op::STEM_TC: return "stem_tc";
    case Op::DECODE: return "decode"; case Op::POST: return "postprocess"; case Op::SPLIT: return "split_planes"; case Op::FINISH: return "finish_f32"; case Op::SPP3: return "spp3";
  }
  return "?";
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
  for (int i = 0; i < n_tensors; ++i) M.host[names[i]] = HostT{h_data[i], static_cast<long long>(numels[i])};

  int rc = CC_OK;
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
  M.host.clear();
  if (rc) return rc;
  *out = h.release();
  return CC_OK;
}

int cc_yolo_destroy(cc_yolo* h) {
  delete h;
  return CC_OK;
}

static constexpr size_t kMaxPlans = 16;   // cached plans per handle (host metadata only: plans own no device memory)

static std::string plan_key(int is_f32, int B, int Hf, int Wf, int res) {
  char key[96];
  snprintf(key, sizeof(key), "%d,%d,%d,%d,%d", is_f32, B, Hf, Wf, res);
  return key;
}
// workspace bytes a plan of this shape addresses (measuring pass of the builder: no device work)
static int plan_bytes(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, size_t* bytes, size_t* scratch = nullptr, size_t* accb = nullptr) {
  YoloPlan tmp;
  tmp.B = B; tmp.Hf = Hf; tmp.Wf = Wf; tmp.res = res; tmp.is_f32 = is_f32;
  Builder dry(h->m, tmp);
  dry.bump.dry = true;
  int rc = dry.build();
  if (rc) return rc;
  *bytes = dry.bump.off + dry.max_scratch + dry.max_acc + 8192;
  if (scratch) *scratch = dry.max_scratch;
  if (accb) *accb = dry.max_acc;
  return CC_OK;
}
static int get_plan(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, YoloPlan** out) {
  YoloModel& M = h->m;
  const std::string key = plan_key(is_f32, B, Hf, Wf, res);
  auto it = M.plans.find(key);
  if (it != M.plans.end() && it->second->gen == M.arena.gen) {
    it->second->last_use = ++M.tick;
    *out = it->second.get();
    return CC_OK;
  }
  size_t bytes = 0, scratch = 0, accb = 0;
  int rc = plan_bytes(h, is_f32, B, Hf, Wf, res, &bytes, &scratch, &accb);
  if (rc) return rc;
  if ((rc = M.arena.reserve(bytes))) return rc;
  // plans built against an older workspace are stale (they are rebuilt on their next use)
  for (auto p = M.plans.begin(); p != M.plans.end();)
    p = (p->second->gen != M.arena.gen) ? M.plans.erase(p) : std::next(p);
  std::unique_ptr<YoloPlan> P(new YoloPlan());
  P->B = B; P->Hf = Hf; P->Wf = Wf; P->res = res; P->is_f32 = is_f32;
  Builder bld(M, *P);
  bld.bump.base = static_cast<uint8_t*>(M.arena.base);
  bld.scratch_bytes = scratch;
  bld.acc_bytes = accb;
  rc = bld.build();
  if (rc) return rc;
  CC_REQUIRE(bld.bump.off <= M.arena.cap, "yolo plan: workspace overrun (%zu > %zu)", bld.bump.off, M.arena.cap);
  P->gen = M.arena.gen;
  P->last_use = ++M.tick;
  if (M.plans.size() >= kMaxPlans) {
    auto lru = M.plans.begin();
    for (auto p = M.plans.begin(); p != M.plans.end(); ++p)
      if (p->second->last_use < lru->second->last_use) lru = p;
    M.plans.erase(lru);
  }
  *out = (M.plans[key] = std::move(P)).get();
  return CC_OK;
}

int cc_yolo_workspace_bytes(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, size_t* bytes) {
  CC_REQUIRE(h && bytes && B > 0 && Hf > 0 && Wf > 0 && res > 0, "cc_yolo_workspace_bytes: bad argument");
  return plan_bytes(h, is_f32, B, Hf, Wf, res, bytes);
}

int cc_yolo_set_workspace(cc_yolo* h, void* d_workspace, size_t bytes) {
  CC_REQUIRE(h, "cc_yolo_set_workspace: null handle");
  CC_REQUIRE(d_workspace == nullptr || (reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0,
             "cc_yolo_set_workspace: the workspace must be 256-byte aligned");
  h->m.plans.clear();
  return h->m.arena.adopt(d_workspace, bytes);
}

int cc_yolo_forward(cc_yolo* h, const void* d_frames, int is_f32, int B, int Hf, int Wf, int res, float* d_out,
                    float* d_raw, void* stream) {
  CC_REQUIRE(h && d_frames && d_out && B > 0 && Hf > 0 && Wf > 0 && res > 0, "cc_yolo_forward: bad argument");
  YoloPlan* P = nullptr;
  int rc = get_plan(h, is_f32, B, Hf, Wf, res, &P);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static const int graph_env = getenv("CC_GRAPH") ? atoi(getenv("CC_GRAPH")) : 1;
  if (graph_env) {
    if (P->gexec && P->g_frames == d_frames && P->g_out == d_out && P->g_raw == d_raw) {
      CC_CHECK_CUDA(cudaGraphLaunch(P->gexec, st));
      return CC_OK;
    }
    const bool stable = P->l_frames == d_frames && P->l_out == d_out && P->l_raw == d_raw;
    P->l_frames = d_frames; P->l_out = d_out; P->l_raw = d_raw;
    if (stable) {
      // second call in a row with these pointers: capture the launch list (on a private stream: nothing executes) and replay
      if (!h->m.cap_stream) CC_CHECK_CUDA(cudaStreamCreateWithFlags(&h->m.cap_stream, cudaStreamNonBlocking));
      if (P->gexec) { cudaGraphExecDestroy(P->gexec); P->gexec = nullptr; }
      cudaGraph_t g = nullptr;
      bool ok = cudaStreamBeginCapture(h->m.cap_stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
      if (ok) {
        rc = plan_run(*P, d_frames, d_out, d_raw, h->m.cap_stream);
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
  }
  return plan_run(*P, d_frames, d_out, d_raw, st);
}

int cc_yolo_plan_info(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, int* net_h, int* net_w, int* anchors,
                      int* launches, double* conv_flops, double* act_bytes) {
  CC_REQUIRE(h, "cc_yolo_plan_info: null handle");
  YoloPlan* P = nullptr;
  int rc = get_plan(h, is_f32, B, Hf, Wf, res, &P);
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
 * life of the handle.  Returns the op count through n_ops. */
int cc_yolo_profile(cc_yolo* h, const void* d_frames, int is_f32, int B, int Hf, int Wf, int res, float* d_out, int cap,
                    float* ms, double* flops, double* bytes, const char** kinds, const char** names, int* n_ops, void* stream) {
  CC_REQUIRE(h && d_frames && d_out, "cc_yolo_profile: bad argument");
  YoloPlan* P = nullptr;
  int rc = get_plan(h, is_f32, B, Hf, Wf, res, &P);
  if (rc) return rc;
  const size_t n = P->ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) CC_CHECK_CUDA(cudaEventCreate(&e));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = plan_run(*P, d_frames, d_out, nullptr, st, &ev);
  if (!rc) {
    CC_CHECK_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n && static_cast<int>(i) < cap; ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, ev[i], ev[i + 1]);
      if (ms) ms[i] = t;
      if (flops) flops[i] = P->ops[i].kind == Op::GEMM ? P->ops[i].gemm.flops : P->ops[i].flops;
      if (bytes) bytes[i] = P->ops[i].kind == Op::GEMM ? P->ops[i].gemm.bytes : op_bytes(P->ops[i]);
      if (kinds) kinds[i] = op_kind_name(P->ops[i].kind);
      if (names) names[i] = P->ops[i].name.c_str();
    }
  }
  for (auto& e : ev) cudaEventDestroy(e);
  if (n_ops) *n_ops = static_cast<int>(n);
  return rc;
}

/* In-situ device timeline of one forward (no events between the launches, so programmatic dependent launch overlaps
 * as in production): for every conv_gemm op, globaltimer ns of (first CTA entered, grid dependency released, last CTA
 * exited, then five stamps of CTA 0: first operands landed, all MMAs issued, first accumulator complete, last epilogue group
 * done, exit); zeros for the other ops.  host_ns: [12 * cap].  Synchronises at the end. */
int cc_yolo_trace(cc_yolo* h, const void* d_frames, int is_f32, int B, int Hf, int Wf, int res, float* d_out, int cap,
                  unsigned long long* host_ns, const char** kinds, const char** names, double* flops, int* n_ops, void* stream) {
  CC_REQUIRE(h && d_frames && d_out && host_ns, "cc_yolo_trace: bad argument");
  YoloPlan* P = nullptr;
  int rc = get_plan(h, is_f32, B, Hf, Wf, res, &P);
  if (rc) return rc;
  const size_t n = P->ops.size();
  unsigned long long* d_trace = nullptr;
  CC_CHECK_CUDA(cudaMalloc(&d_trace, n * 12 * sizeof(unsigned long long)));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(d_trace, 0, n * 12 * sizeof(unsigned long long), st);
  rc = plan_run(*P, d_frames, d_out, nullptr, st, nullptr, d_trace);
  if (!rc) {
    cudaError_t e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) {
      const size_t m = n < static_cast<size_t>(cap) ? n : static_cast<size_t>(cap);
      e = cudaMemcpy(host_ns, d_trace, m * 12 * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
      for (size_t i = 0; i < m; ++i) {
        if (kinds) kinds[i] = op_kind_name(P->ops[i].kind);
        if (names) names[i] = P->ops[i].name.c_str();
        if (flops) flops[i] = P->ops[i].kind == Op::GEMM ? P->ops[i].gemm.flops : 0.0;
      }
    }
    if (e != cudaSuccess) { set_error("cc_yolo_trace: %s", cudaGetErrorString(e)); rc = CC_ERR_CUDA; }
  }
  cudaFree(d_trace);
  if (n_ops) *n_ops = static_cast<int>(n);
  return rc;
}

// parity tap: copy the output of spec layer `layer` of the cached plan (after a forward) to dense fp32 NHWC
__global__ void tap_kernel(const __nv_bfloat16* src, int f32, int cs, int co, int C, long long npix, float* dst) {
  const long long total = npix * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = i / C;
    const int c = static_cast<int>(i % C);
    dst[i] = f32 ? reinterpret_cast<const float*>(src)[pix * cs + co + c] : __bfloat162float(src[pix * cs + co + c]);
  }
}

int cc_yolo_layer_output(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, int layer, float* d_dst, int* C,
                         int* H, int* W, void* stream) {
  CC_REQUIRE(h, "cc_yolo_layer_output: null handle");
  YoloPlan* P = nullptr;
  int rc = get_plan(h, is_f32, B, Hf, Wf, res, &P);
  if (rc) return rc;
  CC_REQUIRE(layer >= 0 && layer < static_cast<int>(P->layer_outs.size()), "cc_yolo_layer_output: bad layer %d", layer);
  const T& t = P->layer_outs[layer];
  if (C) *C = (t.image || !t.p) ? 0 : t.C;      // layers folded into their consumer have a shape but no tensor
  if (H) *H = t.H;
  if (W) *W = t.W;
  if (!d_dst || t.image || !t.p) return CC_OK;
  const long long npix = static_cast<long long>(B) * t.H * t.W;
  tap_kernel<<<132 * 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(t.p, t.f32 ? 1 : 0, t.cs, t.co, t.C, npix, d_dst);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// kernel-level taps for the parity tests
int cc_detect_postprocess(const float* d_pred, int B, int A, int max_det, float iou_thr, int do_scale, float pad_x,
                          float pad_y, float gain, float clip_w, float clip_h, float* d_out, void* stream) {
  PostParams p{};
  p.pred = d_pred; p.B = B; p.A = A; p.max_det = max_det; p.iou_thr = iou_thr;
  p.do_scale = do_scale; p.pad_x = pad_x; p.pad_y = pad_y; p.gain = gain; p.clip_w = clip_w; p.clip_h = clip_h;
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

int cc_letterbox(const void* d_in, int is_f32, int B, int Hin, int Win, int res, void* d_out, int* out_h, int* out_w,
                 void* stream) {
  const double r = std::min(double(res) / Hin, double(res) / Win);
  const int new_w = int(std::nearbyint(Win * r)), new_h = int(std::nearbyint(Hin * r));
  double dw = double(((res - new_w) % 32 + 32) % 32) / 2, dh = double(((res - new_h) % 32 + 32) % 32) / 2;
  const int px = int(std::nearbyint(dw - 0.1)), py = int(std::nearbyint(dh - 0.1));
  if (out_h) *out_h = new_h + 2 * py;
  if (out_w) *out_w = new_w + 2 * px;
  if (!d_out) return CC_OK;   // size query
  LetterboxParams p{};
  p.in = d_in; p.out = d_out; p.is_f32 = is_f32; p.B = B; p.Hin = Hin; p.Win = Win; p.Hr = new_h; p.Wr = new_w;
  p.pad_y = py; p.pad_x = px; p.Hout = new_h + 2 * py; p.Wout = new_w + 2 * px;
  p.sx = float(double(Win) / double(new_w)); p.sy = float(double(Hin) / double(new_h));
  return letterbox_launch(p, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
