// Crop -> bicubic resize -> normalise, on the device (SURVEY.md §8 b1 + §8f N3).
//
// Replaces, for objects cut out of frames that are already in HBM for the detector: the crop of
// `VideoCapture.save_object` (clearcam.py:396), the BGR->RGB swap (models/objects.py:249) and `ObjectFinder.preprocess`
// (models/objects.py:237-242: cv2.resize(INTER_CUBIC) -> /255 -> (x-0.5)/0.5 -> CHW), skipping the reference's JPEG
// write/read in between.  I420 frames (ffmpeg yuv420p) are converted to RGB per tap, exactly as
// cv2.cvtColor(COLOR_YUV2RGB_I420) converts the whole frame, so a crop equals the crop of the converted frame.  Bit-exact with OpenCV's own 8-bit bicubic (see oracle/clip_preprocess.py for the arithmetic
// and its pinning against cv2): taps in float32 with one rounding per operation (hence the explicit _rn intrinsics —
// no fused multiply-add), 11-bit fixed-point taps, exact int32 horizontal pass, float32 vertical pass, round-half-even.
//
// HBM-bound and tiny next to the encoder (K x 224 x 224 outputs, 48 byte reads each, served from L1/L2): one thread per
// output pixel, three channels, coalesced plane writes.  Each rect carries its own source (frame pointer, extent, format),
// so one call takes crops of frames of any shapes and formats (cc_clip_preprocess_frames).
#include <cstdint>
#include <vector>

#include "cc_common.h"
#include "clearcam_b200.h"
#include "ops.cuh"

namespace cc {
namespace {

constexpr int kRectsPerLaunch = 64;
struct CropRect {
  CropSource src;                   // the rect's frame, its extent and format (RGB / BGR / I420)
  int x1, y1, x2, y2;               // validated on the host
};
struct CropParams {
  float* out;
  int S, k0;
  CropRect rect[kRectsPerLaunch];
};

// source index of the first tap (+1) and the four fixed-point taps for destination index d (resize.cpp, a = -0.75)
__device__ __forceinline__ void cubic_taps(int d, int src, int dst, int& s, int taps[4]) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(dst), static_cast<double>(src)));
  const float f = static_cast<float>(__dsub_rn(__dmul_rn(__dadd_rn(static_cast<double>(d), 0.5), scale), 0.5));
  const float fl = floorf(f);
  s = static_cast<int>(fl);
  const float x = __fsub_rn(f, fl);
  const float x1 = __fadd_rn(x, 1.f), xm = __fsub_rn(1.f, x);
  // 5A = -3.75, 8A = -6, 4A = -3, A+2 = 1.25, A+3 = 2.25
  const float c0 = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(-0.75f, x1), -3.75f), x1), -6.f), x1), -3.f);
  const float c1 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, x), 2.25f), x), x), 1.f);
  const float c2 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, xm), 2.25f), xm), xm), 1.f);
  const float c3 = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c0), c1), c2);
  taps[0] = __float2int_rn(__fmul_rn(c0, 2048.f));
  taps[1] = __float2int_rn(__fmul_rn(c1, 2048.f));
  taps[2] = __float2int_rn(__fmul_rn(c2, 2048.f));
  taps[3] = __float2int_rn(__fmul_rn(c3, 2048.f));
}

// One output pixel of rect k.  I420: the frame is [H*3/2, W] planar YUV 4:2:0, converted per tap (to BGR, then swapped
// like a BGR frame); otherwise packed RGB / BGR, swapped unless RGB.
template <bool I420>
__device__ __forceinline__ void crop_resize_pixel(const CropParams& p, const CropRect& rc, int k, int dx, int dy) {
  const CropSource& f = rc.src;
  const int x1 = rc.x1, y1 = rc.y1;
  const int cw = rc.x2 - x1, ch = rc.y2 - y1;
  const uint8_t* img = I420 ? f.frame : f.frame + static_cast<size_t>(y1) * f.W * 3 + static_cast<size_t>(x1) * 3;
  int sx, sy, ax[4], ay[4];
  cubic_taps(dx, cw, p.S, sx, ax);
  cubic_taps(dy, ch, p.S, sy, ay);
  int hor[4][3];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int yy = min(max(sy - 1 + r, 0), ch - 1);
    const uint8_t* row = img + static_cast<size_t>(yy) * f.W * 3;
    int acc[3] = {0, 0, 0};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int xx = min(max(sx - 1 + j, 0), cw - 1);
      if constexpr (I420) {
        int px[3];
        i420_bgr(img, f.H, f.W, y1 + yy, x1 + xx, px);       // absolute frame coordinates: the chroma of the full frame
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += px[c] * ax[j];
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += static_cast<int>(__ldg(row + xx * 3 + c)) * ax[j];
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) hor[r][c] = acc[c];
  }
  const float kInv = 1.0f / (2048.f * 2048.f);
  float b[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) b[r] = __fmul_rn(static_cast<float>(ay[r]), kInv);
  const int tail = (p.S * 3) / 8 * 8;            // interleaved elements past the last group of 8 take the integer form
  const int swap = f.fmt != 0;                   // source channel order is BGR (the crop is RGB)
  float* out = p.out + static_cast<size_t>(p.k0 + k) * 3 * p.S * p.S + static_cast<size_t>(dy) * p.S + dx;
#pragma unroll
  for (int c = 0; c < 3; ++c) {                  // c indexes the crop's channel order after the optional BGR->RGB swap
    const int sc = swap ? 2 - c : c;
    int v;
    if (dx * 3 + c < tail) {
      float t = __fmul_rn(static_cast<float>(hor[3][sc]), b[3]);
      t = __fadd_rn(__fmul_rn(static_cast<float>(hor[2][sc]), b[2]), t);
      t = __fadd_rn(__fmul_rn(static_cast<float>(hor[1][sc]), b[1]), t);
      t = __fadd_rn(__fmul_rn(static_cast<float>(hor[0][sc]), b[0]), t);
      v = __float2int_rn(t);
    } else {
      const long long s = static_cast<long long>(hor[0][sc]) * ay[0] + static_cast<long long>(hor[1][sc]) * ay[1] +
                          static_cast<long long>(hor[2][sc]) * ay[2] + static_cast<long long>(hor[3][sc]) * ay[3];
      v = static_cast<int>((s + (1 << 21)) >> 22);
    }
    v = min(max(v, 0), 255);
    const float n = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v), 255.f), 0.5f), 0.5f);     // models/objects.py:239-240
    out[static_cast<size_t>(c) * p.S * p.S] = n;
  }
}

// one CTA row of one rect (blockIdx.z): the source format is read per rect, so the branch is uniform per CTA
__global__ void __launch_bounds__(256) crop_resize_kernel(const __grid_constant__ CropParams p) {
  const int dx = blockIdx.x * 32 + threadIdx.x, dy = blockIdx.y * 8 + threadIdx.y, k = blockIdx.z;
  if (dx >= p.S || dy >= p.S) return;
  const CropRect& rc = p.rect[k];
  if (rc.src.fmt == 2) crop_resize_pixel<true>(p, rc, k, dx, dy);
  else crop_resize_pixel<false>(p, rc, k, dx, dy);
}

// the launches of one call over crops whose sources and rects are checked
int crop_resize_sources(const CropSource* src, const int32_t* rects, int K, int size, float* d_out, cudaStream_t st) {
  for (int k0 = 0; k0 < K; k0 += kRectsPerLaunch) {
    CropParams p;
    p.out = d_out;
    p.S = size;
    p.k0 = k0;
    const int n = K - k0 < kRectsPerLaunch ? K - k0 : kRectsPerLaunch;
    for (int i = 0; i < n; ++i) {
      const int32_t* r = rects + 5 * (k0 + i);
      p.rect[i] = CropRect{src[k0 + i], r[1], r[2], r[3], r[4]};
    }
    const dim3 grid((size + 31) / 32, (size + 7) / 8, n);
    crop_resize_kernel<<<grid, dim3(32, 8), 0, st>>>(p);
    CC_CHECK_CUDA(cudaGetLastError());
  }
  return CC_OK;
}

}  // namespace
}  // namespace cc

extern "C" int cc_clip_preprocess_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int size, float* d_out,
                                         void* stream) {
  using namespace cc;
  const char* who = "cc_clip_preprocess_frames";
  CC_REQUIRE(d_out, "%s: null pointer", who);
  CC_REQUIRE(size >= 1 && size <= 4096, "%s: bad size %d", who, size);
  std::vector<CropSource> src(K > 0 ? K : 0);
  if (int rc = table_crop_sources(who, frames, n_frames, rects, K, src.data())) return rc;
  return crop_resize_sources(src.data(), rects, K, size, d_out, static_cast<cudaStream_t>(stream));
}
