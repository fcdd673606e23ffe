// BlazeFace face detector, fp32 on CUDA cores.
//
// Replaces in the reference: class BlazeFace (models/blazeface.py:62-232) with its BlazeBlocks (:5-30) and FinalBlazeBlock
// (:43-60).  The score threshold (0.85) and the suppression (IoU 0.3) are decided on fp32 logits, so nothing runs in bf16.
//
// One forward of B images of any sizes:
//   letterbox  pool.cu's letterbox kernel (the tinygrad linear resize of utils/helpers.resize, uint8 arithmetic) to
//              256x256, centred zero pads (:155-165)                                          uint8 [B,256,256,3]
//   stem       /127.5 - 1, pad (1,2), conv 5x5 s2 3->24, ReLU (:137-140)                      fp32 NHWC [B,128,128,24]
//   blocks     31 BlazeBlocks, one fused kernel each: depthwise 3x3 (stride 1 pad 1, or stride 2 with the (0,2) pad),
//              pointwise 1x1, shortcut (x, or its 2x2 max pool, zero-padded to the new width), add, ReLU; an 8x8 output
//              tile with its input halo in shared memory                                      ... [B,16,16,96]
//   final      the same kernel without the shortcut (FinalBlazeBlock)                         fp32 NHWC [B,8,8,96]
//   heads      the four 1x1 head convs, written in the [B,896,16] / [B,896] anchor layout of the permute + reshape + cat
//   decode     one CTA per image: _decode_boxes, clip + sigmoid + 0.85 mask, the score order, the one-shot suppression and
//              the *256 / pads / scale tail of __call__                                       fp32 [B,896,17]
#include "clearcam_b200.h"
#include "cc_common.h"
#include "ops.cuh"

namespace cc {

static constexpr int kSide = 256, kAnchors = 896, kCoords = 16, kDet = 17, kBlocks = 31, kTile = 8;
static constexpr float kMinScore = 0.85f, kIouThr = 0.3f, kScoreClip = 100.f;
// (in channels, out channels, stride) of backbone_tiny.list.0 .. 30 (models/blazeface.py:98-127)
__host__ __device__ constexpr int block_cin(int i) { return i < 16 ? 24 : i < 24 ? 48 : 96; }
__host__ __device__ constexpr int block_cout(int i) { return i < 15 ? 24 : i < 23 ? 48 : 96; }
__host__ __device__ constexpr int block_stride(int i) { return (i == 7 || i == 15 || i == 23) ? 2 : 1; }

// ------------------------------------------------------------------------------------------------ stem
// one thread per output pixel, all 24 channels; weights [24][3][5][5] + bias in shared memory
__global__ void __launch_bounds__(128) blaze_stem_kernel(const uint8_t* __restrict__ in, const float* __restrict__ w,
                                                         const float* __restrict__ bias, float* __restrict__ out) {
  __shared__ float sw[24 * 75 + 24];
  for (int i = threadIdx.x; i < 24 * 75 + 24; i += blockDim.x) sw[i] = i < 24 * 75 ? w[i] : bias[i - 24 * 75];
  __syncthreads();
  const int n = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= 128 * 128) return;
  const int oy = p / 128, ox = p % 128;
  const uint8_t* img = in + static_cast<long long>(n) * kSide * kSide * 3;
  float acc[24];
#pragma unroll
  for (int o = 0; o < 24; ++o) acc[o] = sw[24 * 75 + o];
  for (int ky = 0; ky < 5; ++ky) {
    const int y = 2 * oy + ky - 1;                 // pad (1, 2): top 1, bottom 2
    if (y < 0 || y >= kSide) continue;
    for (int kx = 0; kx < 5; ++kx) {
      const int x = 2 * ox + kx - 1;
      if (x < 0 || x >= kSide) continue;
      const uint8_t* px = img + (y * kSide + x) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = __fsub_rn(__fdiv_rn(static_cast<float>(px[c]), 127.5f), 1.f);
#pragma unroll
        for (int o = 0; o < 24; ++o) acc[o] = fmaf(sw[o * 75 + c * 25 + ky * 5 + kx], v, acc[o]);
      }
    }
  }
  float4* dst = reinterpret_cast<float4*>(out + (static_cast<long long>(n) * 128 * 128 + p) * 24);
#pragma unroll
  for (int q = 0; q < 6; ++q)
    dst[q] = make_float4(fmaxf(acc[4 * q], 0.f), fmaxf(acc[4 * q + 1], 0.f), fmaxf(acc[4 * q + 2], 0.f), fmaxf(acc[4 * q + 3], 0.f));
}

// ------------------------------------------------------------------------------------------------ BlazeBlock
struct BlockArgs {
  const float* in; float* out;
  const float *dw, *dwb, *pw, *pwb;   // depthwise [Cin][9], [Cin]; pointwise transposed at create time to [Cin][Cout], [Cout]
  int H, W, Cin, Cout, stride, shortcut;
};

static size_t block_smem(int cin, int cout, int stride) {
  const int R = stride == 1 ? kTile + 2 : 2 * kTile + 1;
  return (static_cast<size_t>(R) * R * cin + kTile * kTile * cin + static_cast<size_t>(cin) * cout) * 4;
}

// CTA = one 8x8 output tile of one image.  Shared memory: the input tile with its halo [R][R][Cin] (zeros outside the map),
// the depthwise output [64][Cin] and the pointwise weights [Cin][Cout] (a straight copy: consecutive output channels sit in
// consecutive banks for the pointwise loop).
__global__ void __launch_bounds__(256) blaze_block_kernel(const BlockArgs a) {
  extern __shared__ float smem[];
  const int s = a.stride, R = s == 1 ? kTile + 2 : 2 * kTile + 1, Cin = a.Cin, Cout = a.Cout;
  const int Ho = a.H / s, Wo = a.W / s;
  float* s_in = smem;
  float* s_mid = s_in + R * R * Cin;
  float* s_w = s_mid + kTile * kTile * Cin;
  const int n = blockIdx.z, oy0 = blockIdx.y * kTile, ox0 = blockIdx.x * kTile;
  const int iy0 = s == 1 ? oy0 - 1 : 2 * oy0, ix0 = s == 1 ? ox0 - 1 : 2 * ox0;
  const float* img = a.in + static_cast<long long>(n) * a.H * a.W * Cin;
  for (int i = threadIdx.x; i < R * R * Cin; i += blockDim.x) {
    const int q = i / Cin, c = i - q * Cin;
    const int y = iy0 + q / R, x = ix0 + q % R;
    s_in[i] = (y >= 0 && y < a.H && x >= 0 && x < a.W) ? __ldg(img + (static_cast<long long>(y) * a.W + x) * Cin + c) : 0.f;
  }
  for (int i = threadIdx.x; i < Cin * Cout; i += blockDim.x) s_w[i] = __ldg(a.pw + i);
  __syncthreads();
  for (int i = threadIdx.x; i < kTile * kTile * Cin; i += blockDim.x) {
    const int p = i / Cin, c = i - p * Cin, py = p / kTile, px = p % kTile;
    float acc = __ldg(a.dwb + c);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) acc = fmaf(__ldg(a.dw + c * 9 + ky * 3 + kx), s_in[((py * s + ky) * R + px * s + kx) * Cin + c], acc);
    s_mid[i] = acc;
  }
  __syncthreads();
  float* dst = a.out + static_cast<long long>(n) * Ho * Wo * Cout;
  for (int i = threadIdx.x; i < kTile * kTile * Cout; i += blockDim.x) {
    const int p = i / Cout, o = i - p * Cout, py = p / kTile, px = p % kTile;
    const float* m = s_mid + p * Cin;
    float acc = __ldg(a.pwb + o);
    for (int c = 0; c < Cin; ++c) acc = fmaf(s_w[c * Cout + o], m[c], acc);
    if (a.shortcut && o < Cin) {               // channels >= Cin of the shortcut are the zero channel pad
      if (s == 1) {
        acc += s_in[((py + 1) * R + px + 1) * Cin + o];
      } else {
        const float* q = s_in + ((2 * py) * R + 2 * px) * Cin + o;
        acc += fmaxf(fmaxf(q[0], q[Cin]), fmaxf(q[R * Cin], q[(R + 1) * Cin]));
      }
    }
    dst[(static_cast<long long>(oy0 + py) * Wo + ox0 + px) * Cout + o] = fmaxf(acc, 0.f);
  }
}

static int block_launch(const BlockArgs& a, int B, cudaStream_t st) {
  const size_t smem = block_smem(a.Cin, a.Cout, a.stride);
  const dim3 grid(a.W / a.stride / kTile, a.H / a.stride / kTile, B);
  blaze_block_kernel<<<grid, 256, smem, st>>>(a);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ heads
// one thread per (image, anchor, column): columns 0..15 the regressor, 16 the classifier.  Anchors 0..511 are the 16x16 map
// with 2 anchors per pixel, 512..895 the 8x8 map with 6 per pixel (the permute(0,2,3,1) + reshape of :143-160).
struct HeadArgs {
  const float *x16, *h8;
  const float *c8w, *c8b, *c16w, *c16b, *r8w, *r8b, *r16w, *r16b;
  float *boxes, *scores;
  int B;
};

__global__ void __launch_bounds__(256) blaze_heads_kernel(const HeadArgs a) {
  const long long total = static_cast<long long>(a.B) * kAnchors * kDet;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(i % kDet);
    const long long na = i / kDet;
    const int n = static_cast<int>(na / kAnchors), an = static_cast<int>(na % kAnchors);
    const float *f, *w, *b;
    int row;
    if (an < 512) {
      const int pix = an >> 1, k = an & 1;
      f = a.x16 + (static_cast<long long>(n) * 256 + pix) * 96;
      if (j < kCoords) { w = a.r8w; b = a.r8b; row = k * kCoords + j; } else { w = a.c8w; b = a.c8b; row = k; }
    } else {
      const int pix = (an - 512) / 6, k = (an - 512) % 6;
      f = a.h8 + (static_cast<long long>(n) * 64 + pix) * 96;
      if (j < kCoords) { w = a.r16w; b = a.r16b; row = k * kCoords + j; } else { w = a.c16w; b = a.c16b; row = k; }
    }
    const float4* f4 = reinterpret_cast<const float4*>(f);
    const float4* w4 = reinterpret_cast<const float4*>(w + row * 96);
    float acc = __ldg(b + row);
#pragma unroll 4
    for (int q = 0; q < 24; ++q) {
      const float4 u = __ldg(f4 + q), v = __ldg(w4 + q);
      acc = fmaf(v.x, u.x, acc); acc = fmaf(v.y, u.y, acc); acc = fmaf(v.z, u.z, acc); acc = fmaf(v.w, u.w, acc);
    }
    if (j < kCoords) a.boxes[na * kCoords + j] = acc; else a.scores[na] = acc;
  }
}

// ------------------------------------------------------------------------------------------------ decode + suppression
struct DecodeImage { float scale; float top, left; };
static constexpr size_t kDecodeSmem = static_cast<size_t>(kAnchors) * kDet * 4;   // the decoded rows, set up in cc_blazeface_create
struct DecodeTable { DecodeImage im[CC_MAX_FRAMES]; };

__device__ __forceinline__ unsigned long long score_key(float score, int idx) {
  // score >= 0: its bits order like the value; ties go to the smaller anchor index
  return (static_cast<unsigned long long>(__float_as_uint(score)) << 32) | (0xFFFFFFFFu - static_cast<unsigned>(idx));
}

// One CTA per image.  The decoded rows live in shared memory [896][17]; every row's place in the order is the number of
// keys above its own (896 keys, so a count is cheaper than a sort).  Row j of the order is suppressed when any earlier row
// (masked and suppressed ones included, as the reference's triu + column sum does) has IoU > 0.3 with it.
__global__ void __launch_bounds__(1024) blaze_decode_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                            const float* __restrict__ anchors, float* __restrict__ out,
                                                            const __grid_constant__ DecodeTable t) {
  extern __shared__ float s_rows[];                               // [896][17]
  __shared__ unsigned long long s_key[kAnchors];
  __shared__ short s_order[kAnchors];
  const int n = blockIdx.x;
  const float* rb = boxes + static_cast<long long>(n) * kAnchors * kCoords;
  const float* rs = scores + static_cast<long long>(n) * kAnchors;
  for (int i = threadIdx.x; i < kAnchors; i += blockDim.x) {
    const float ax = __ldg(anchors + 4 * i), ay = __ldg(anchors + 4 * i + 1), aw = __ldg(anchors + 4 * i + 2), ah = __ldg(anchors + 4 * i + 3);
    const float* r = rb + i * kCoords;
    const float c = fminf(fmaxf(__ldg(rs + i), -kScoreClip), kScoreClip);
    const float score = static_cast<float>(1.0 / (1.0 + exp(-static_cast<double>(c))));
    const float m = score >= kMinScore ? 1.f : 0.f;
    const float xc = __fadd_rn(__fmul_rn(__fdiv_rn(__ldg(r), 256.f), aw), ax);
    const float yc = __fadd_rn(__fmul_rn(__fdiv_rn(__ldg(r + 1), 256.f), ah), ay);
    const float w = __fmul_rn(__fdiv_rn(__ldg(r + 2), 256.f), aw);
    const float h = __fmul_rn(__fdiv_rn(__ldg(r + 3), 256.f), ah);
    float* row = s_rows + i * kDet;
    row[0] = __fmul_rn(__fsub_rn(yc, __fdiv_rn(h, 2.f)), m);
    row[1] = __fmul_rn(__fsub_rn(xc, __fdiv_rn(w, 2.f)), m);
    row[2] = __fmul_rn(__fadd_rn(yc, __fdiv_rn(h, 2.f)), m);
    row[3] = __fmul_rn(__fadd_rn(xc, __fdiv_rn(w, 2.f)), m);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      row[4 + 2 * k] = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(__ldg(r + 4 + 2 * k), 256.f), aw), ax), m);
      row[5 + 2 * k] = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(__ldg(r + 5 + 2 * k), 256.f), ah), ay), m);
    }
    row[16] = __fmul_rn(score, m);
    s_key[i] = score_key(row[16], i);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kAnchors; i += blockDim.x) {
    const unsigned long long k = s_key[i];
    int rank = 0;
    for (int q = 0; q < kAnchors; ++q) rank += s_key[q] > k;
    s_order[rank] = static_cast<short>(i);
  }
  __syncthreads();
  const DecodeImage& g = t.im[n];
  float* o = out + static_cast<long long>(n) * kAnchors * kDet;
  for (int j = threadIdx.x; j < kAnchors; j += blockDim.x) {
    const float* rj = s_rows + s_order[j] * kDet;
    bool keep = rj[16] >= kMinScore;
    if (keep) {
      const float ja = __fmul_rn(__fsub_rn(rj[2], rj[0]), __fsub_rn(rj[3], rj[1]));
      for (int i = 0; i < j && keep; ++i) {
        const float* ri = s_rows + s_order[i] * kDet;
        const float ia = __fmul_rn(__fsub_rn(ri[2], ri[0]), __fsub_rn(ri[3], ri[1]));
        const float w = fmaxf(0.f, __fsub_rn(fminf(ri[2], rj[2]), fmaxf(ri[0], rj[0])));
        const float h = fmaxf(0.f, __fsub_rn(fminf(ri[3], rj[3]), fmaxf(ri[1], rj[1])));
        const float inter = __fmul_rn(w, h);
        const float iou = __fdiv_rn(inter, __fsub_rn(__fadd_rn(ia, ja), inter));
        if (iou > kIouThr) keep = false;          // NaN (0/0) compares false
      }
    }
    const float k = keep ? 1.f : 0.f;
    for (int c = 0; c < kDet; ++c) {
      float v = __fmul_rn(__fmul_rn(rj[c], k), 256.f);
      if (c == 0 || c == 2) v = __fsub_rn(v, g.top);
      if (c == 1 || c == 3) v = __fsub_rn(v, g.left);
      o[j * kDet + c] = __fdiv_rn(v, g.scale);
    }
  }
}

// One CTA per image: the first row of dets [896][17] whose column 0 != 0 as numpy compares it (-0.0 is zero, NaN is not),
// copied bit for bit, or a zero row.  The host geometry of img_to_face reads only that row (models/objects.py:283-284).
__global__ void __launch_bounds__(128) blaze_first_kernel(const float* __restrict__ dets, float* __restrict__ first) {
  __shared__ int s_first;
  if (threadIdx.x == 0) s_first = kAnchors;
  __syncthreads();
  const float* d = dets + static_cast<long long>(blockIdx.x) * kAnchors * kDet;
  int mine = kAnchors;
  for (int i = threadIdx.x; i < kAnchors; i += blockDim.x)
    if (d[i * kDet] != 0.f) { mine = i; break; }                  // unordered !=: true for NaN
  if (mine < kAnchors) atomicMin(&s_first, mine);
  __syncthreads();
  const int r = s_first;
  if (threadIdx.x < kDet)
    first[static_cast<long long>(blockIdx.x) * kDet + threadIdx.x] = r < kAnchors ? d[r * kDet + threadIdx.x] : 0.f;
}

// the letterbox geometry of BlazeFace.__call__ (:155-165) for an h x w image
struct Fit { double scale; int new_w, new_h, top, left; };
static Fit fit(int h, int w) {
  Fit f;
  f.scale = std::min(256.0 / w, 256.0 / h);
  f.new_w = static_cast<int>(w * f.scale);
  f.new_h = static_cast<int>(h * f.scale);
  f.top = (kSide - f.new_h) / 2;
  f.left = (kSide - f.new_w) / 2;
  return f;
}

static int decode_launch(const float* anchors, const float* boxes, const float* scores, const int32_t* sizes, int B, float* dets,
                         cudaStream_t st) {
  const size_t smem = kDecodeSmem;
  for (int b0 = 0; b0 < B; b0 += CC_MAX_FRAMES) {
    const int nb = std::min(B - b0, CC_MAX_FRAMES);
    DecodeTable t{};
    for (int i = 0; i < nb; ++i) {
      const Fit f = fit(sizes[2 * (b0 + i)], sizes[2 * (b0 + i) + 1]);
      t.im[i] = DecodeImage{static_cast<float>(f.scale), static_cast<float>(f.top), static_cast<float>(f.left)};
    }
    const long long off = static_cast<long long>(b0) * kAnchors;
    blaze_decode_kernel<<<nb, 1024, smem, st>>>(boxes + off * kCoords, scores + off, anchors, dets + off * kDet, t);
    CC_CHECK_CUDA(cudaGetLastError());
  }
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ model
struct BlazeW { const float *dw, *dwb, *pw, *pwb; };

struct BlazeModel {
  HostTensors host;                               // the create call's tensors; emptied before it returns
  float* dev = nullptr;                           // every tensor, one allocation
  std::vector<float> pack;
  const float *stem_w = nullptr, *stem_b = nullptr, *anchors = nullptr;
  const float *c8w, *c8b, *c16w, *c16b, *r8w, *r8b, *r16w, *r16b;
  BlazeW blk[kBlocks], fin;
  void* ws = nullptr;
  size_t ws_bytes = 0;
  ~BlazeModel() { if (dev) cudaFree(dev); }

  // host offsets first (dev == nullptr), then rebased onto the device allocation
  std::vector<std::pair<const float**, size_t>> fix;
  // rows > 0: a [rows][n / rows] matrix stored transposed, [n / rows][rows]
  int take(const std::string& name, long long n, const float** out, int rows = 0) {
    const float* h;
    if (int rc = host.get(name, n, &h)) return rc;
    fix.push_back({out, pack.size()});
    if (rows > 0) {
      const long long cols = n / rows;
      for (long long c = 0; c < cols; ++c)
        for (int r = 0; r < rows; ++r) pack.push_back(h[r * cols + c]);
    } else {
      pack.insert(pack.end(), h, h + n);
    }
    while (pack.size() % 4) pack.push_back(0.f);  // 16-byte aligned tensors (the heads read float4)
    return CC_OK;
  }
};

struct Layout { uint8_t* lb; float *x0, *x1, *h8; };
static size_t layout(int B, uint8_t* base, Layout* L) {
  Bump b;
  b.dry = base == nullptr;
  b.base = base;
  L->lb = static_cast<uint8_t*>(b.take(static_cast<size_t>(B) * kSide * kSide * 3));
  L->x0 = static_cast<float*>(b.take(static_cast<size_t>(B) * 128 * 128 * 24 * 4));
  L->x1 = static_cast<float*>(b.take(static_cast<size_t>(B) * 128 * 128 * 24 * 4));
  L->h8 = static_cast<float*>(b.take(static_cast<size_t>(B) * 8 * 8 * 96 * 4));
  return b.off + 1024;
}

}  // namespace cc

using namespace cc;

struct cc_blazeface { BlazeModel m; };

extern "C" {

int cc_blazeface_create(int n_tensors, const char* const* names, const float* const* h_data, const int64_t* numels,
                        cc_blazeface** out) {
  CC_REQUIRE(out, "cc_blazeface_create: null argument");
  CC_REQUIRE(device_sm_count() > 0, "cc_blazeface_create: no sm_90 (H100) device");
  std::unique_ptr<cc_blazeface> h(new cc_blazeface());
  BlazeModel& M = h->m;
  int rc = 0;
  if ((rc = M.host.fill("cc_blazeface_create", n_tensors, names, h_data, numels))) return rc;
  if ((rc = M.take("conv_tiny.weight", 24 * 3 * 25, &M.stem_w)) || (rc = M.take("conv_tiny.bias", 24, &M.stem_b)) ||
      (rc = M.take("anchors", kAnchors * 4, &M.anchors)) ||
      (rc = M.take("classifier_8_tiny.weight", 2 * 96, &M.c8w)) || (rc = M.take("classifier_8_tiny.bias", 2, &M.c8b)) ||
      (rc = M.take("classifier_16_tiny.weight", 6 * 96, &M.c16w)) || (rc = M.take("classifier_16_tiny.bias", 6, &M.c16b)) ||
      (rc = M.take("regressor_8_tiny.weight", 32 * 96, &M.r8w)) || (rc = M.take("regressor_8_tiny.bias", 32, &M.r8b)) ||
      (rc = M.take("regressor_16_tiny.weight", 96 * 96, &M.r16w)) || (rc = M.take("regressor_16_tiny.bias", 96, &M.r16b)))
    return rc;
  for (int i = 0; i <= kBlocks; ++i) {
    const std::string p = i < kBlocks ? "backbone_tiny.list." + std::to_string(i) : std::string("final");
    const int cin = i < kBlocks ? block_cin(i) : 96, cout = i < kBlocks ? block_cout(i) : 96;
    BlazeW& b = i < kBlocks ? M.blk[i] : M.fin;
    if ((rc = M.take(p + ".conv0_tiny.weight", cin * 9, &b.dw)) || (rc = M.take(p + ".conv0_tiny.bias", cin, &b.dwb)) ||
        (rc = M.take(p + ".conv1_tiny.weight", static_cast<long long>(cout) * cin, &b.pw, cout)) ||
        (rc = M.take(p + ".conv1_tiny.bias", cout, &b.pwb)))
      return rc;
  }
  M.host.clear();
  CC_CHECK_CUDA(cudaMalloc(&M.dev, M.pack.size() * 4));
  CC_CHECK_CUDA(cudaMemcpy(M.dev, M.pack.data(), M.pack.size() * 4, cudaMemcpyHostToDevice));
  for (auto& f : M.fix) *f.first = M.dev + f.second;
  M.fix.clear();
  M.pack.clear();
  const size_t big = block_smem(96, 96, 2);
  CC_CHECK_CUDA(cudaFuncSetAttribute(blaze_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(big)));
  CC_CHECK_CUDA(cudaFuncSetAttribute(blaze_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kDecodeSmem)));
  *out = h.release();
  return CC_OK;
}

int cc_blazeface_destroy(cc_blazeface* h) {
  delete h;
  return CC_OK;
}

int cc_blazeface_workspace_bytes(cc_blazeface* h, int B, size_t* bytes) {
  CC_REQUIRE(h && bytes && B > 0, "cc_blazeface_workspace_bytes: bad argument");
  Layout L;
  *bytes = layout(B, nullptr, &L);
  return CC_OK;
}

int cc_blazeface_set_workspace(cc_blazeface* h, void* d_workspace, size_t bytes) {
  if (int rc = check_workspace("cc_blazeface_set_workspace", h, d_workspace)) return rc;
  h->m.ws = d_workspace;
  h->m.ws_bytes = d_workspace ? bytes : 0;
  return CC_OK;
}

int cc_blazeface_decode(cc_blazeface* h, const float* d_boxes, const float* d_scores, int B, const int32_t* h_sizes, float* d_dets,
                        void* stream) {
  CC_REQUIRE(h && d_boxes && d_scores && h_sizes && d_dets && B > 0, "cc_blazeface_decode: bad argument");
  for (int b = 0; b < B; ++b) {
    CC_REQUIRE(h_sizes[2 * b] > 0 && h_sizes[2 * b + 1] > 0, "cc_blazeface_decode: image %d has size %dx%d", b, h_sizes[2 * b + 1],
               h_sizes[2 * b]);
  }
  return decode_launch(h->m.anchors, d_boxes, d_scores, h_sizes, B, d_dets, static_cast<cudaStream_t>(stream));
}

int cc_blazeface_first(const float* d_dets, int B, float* d_first, void* stream) {
  CC_REQUIRE(d_dets && d_first && B > 0, "cc_blazeface_first: bad argument (dets %p, B = %d, first %p)", d_dets, B, d_first);
  blaze_first_kernel<<<B, 128, 0, static_cast<cudaStream_t>(stream)>>>(d_dets, d_first);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

int cc_blazeface_forward(cc_blazeface* h, const cc_frame* frames, int B, float* d_boxes, float* d_scores, float* d_dets,
                         void* stream) {
  CC_REQUIRE(h && frames && d_boxes && d_scores && d_dets && B > 0, "cc_blazeface_forward: bad argument");
  BlazeModel& M = h->m;
  Layout L;
  const size_t need = layout(B, nullptr, &L);
  CC_REQUIRE(M.ws && M.ws_bytes >= need, "cc_blazeface_forward: the workspace holds %zu bytes, B = %d needs %zu "
             "(cc_blazeface_workspace_bytes / cc_blazeface_set_workspace)", M.ws_bytes, B, need);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_boxes) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_scores) & 3) == 0 &&
             (reinterpret_cast<uintptr_t>(d_dets) & 3) == 0, "cc_blazeface_forward: misaligned output");
  std::vector<int32_t> sizes(2 * static_cast<size_t>(B));
  for (int b = 0; b < B; ++b) {
    const cc_frame& f = frames[b];
    CC_REQUIRE(f.data && f.fmt == CC_FRAME_BGR_U8 && f.h > 0 && f.w > 0,
               "cc_blazeface_forward: image %d must be a uint8 [h,w,3] device image (data %p, format %d, %dx%d)", b, f.data, f.fmt,
               f.w, f.h);
    const Fit g = fit(f.h, f.w);
    CC_REQUIRE(g.new_w >= 1 && g.new_h >= 1, "cc_blazeface_forward: image %d (%dx%d) resizes to an empty %dx%d", b, f.w, f.h,
               g.new_w, g.new_h);
    sizes[2 * b] = f.h;
    sizes[2 * b + 1] = f.w;
  }
  layout(B, static_cast<uint8_t*>(M.ws), &L);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  LetterboxTable t;
  t.Hout = kSide; t.Wout = kSide; t.out_f32 = 0;
  for (int b0 = 0; b0 < B; b0 += CC_MAX_FRAMES) {
    t.B = std::min(B - b0, CC_MAX_FRAMES);
    t.out = L.lb + static_cast<size_t>(b0) * kSide * kSide * 3;
    for (int i = 0; i < t.B; ++i) {
      const cc_frame& f = frames[b0 + i];
      const Fit g = fit(f.h, f.w);
      LetterboxFrame& lf = t.f[i];
      lf.in = f.data; lf.fmt = CC_FRAME_BGR_U8; lf.Hin = f.h; lf.Win = f.w; lf.Hr = g.new_h; lf.Wr = g.new_w;
      lf.pad_y = g.top; lf.pad_x = g.left;
      lf.sx = static_cast<float>(static_cast<double>(f.w) / g.new_w);
      lf.sy = static_cast<float>(static_cast<double>(f.h) / g.new_h);
    }
    if (int rc = letterbox_frames_launch(t, st)) return rc;
  }
  blaze_stem_kernel<<<dim3(128 * 128 / 128, B), 128, 0, st>>>(L.lb, M.stem_w, M.stem_b, L.x0);
  CC_CHECK_CUDA(cudaGetLastError());
  float *x = L.x0, *y = L.x1;
  int H = 128;
  for (int i = 0; i < kBlocks; ++i) {
    const BlazeW& w = M.blk[i];
    const BlockArgs a{x, y, w.dw, w.dwb, w.pw, w.pwb, H, H, block_cin(i), block_cout(i), block_stride(i), 1};
    if (int rc = block_launch(a, B, st)) return rc;
    H /= block_stride(i);
    std::swap(x, y);
  }
  const BlockArgs fa{x, L.h8, M.fin.dw, M.fin.dwb, M.fin.pw, M.fin.pwb, H, H, 96, 96, 2, 0};
  if (int rc = block_launch(fa, B, st)) return rc;
  const HeadArgs ha{x, L.h8, M.c8w, M.c8b, M.c16w, M.c16b, M.r8w, M.r8b, M.r16w, M.r16b, d_boxes, d_scores, B};
  const long long total = static_cast<long long>(B) * kAnchors * kDet;
  const long long blocks = std::min((total + 255) / 256, 132LL * 16);
  blaze_heads_kernel<<<static_cast<int>(blocks), 256, 0, st>>>(ha);
  CC_CHECK_CUDA(cudaGetLastError());
  return decode_launch(M.anchors, d_boxes, d_scores, sizes.data(), B, d_dets, st);
}

}  // extern "C"
