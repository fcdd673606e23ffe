// The image arithmetic of the reference's img_to_face (models/objects.py:263-354), byte for byte with cv2 4.13
// (oracle/face_align.py states it; the per-face geometry stays on the host in the reference's own numpy expressions).
//   face_canvas_kernel  cv2.resize(INTER_LINEAR) of each image to a long side of 640 and the zero border to 640x640
//                       (:265-272); an exact 2x reduction is cv2's INTER_AREA average, as cv2 picks it
//   face_align_kernel   both cv2.warpAffine calls (INTER_LINEAR, zero border) and the final channel swap (:325-346).  The
//                       rotated canvas is not stored: each tap of the second warp evaluates the first warp at that integer
//                       pixel, which is exactly the uint8 value cv2's intermediate image holds there.
// Both read their images through a row pitch, so one body serves contiguous [h,w,3] images and the h x w corners of a
// padded [K,Hmax,Wmax,3] batch; kSwapRB reads a BGR slot as the RGB image cv2.cvtColor(slot, BGR2RGB) the reference passes
// to img_to_face.
// Float64 coordinate arithmetic uses _rn intrinsics so that no multiply-add is contracted: the products and sums round as
// cv2's do on the host.
#include "clearcam_b200.h"
#include "cc_common.h"
#include <algorithm>
#include <cstdint>
#include <vector>

namespace cc {

static constexpr int kCanvas = 640, kFace = 112, kAlignJobs = 24, kCanvasJobs = 64;

struct CanvasJob { const uint8_t* src; int pitch, h, w, rw, rh, top, left, area2; double sx, sy; };   // pitch: bytes per row
struct CanvasTable { uint8_t* out; CanvasJob j[kCanvasJobs]; };

// cv2's resize coefficient of output index d along an axis: source index and 11-bit weights (clamp_w: the column axis,
// whose weight cv2 zeroes at the ends; rows keep their weights and clamp the index)
__device__ __forceinline__ void lin_coef(int d, double scale, int n, bool clamp_w, int& s0, int& s1, int& w0, int& w1) {
  float f = static_cast<float>(__dsub_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), 0.5));
  int s = static_cast<int>(floorf(f));
  f -= static_cast<float>(s);
  if (clamp_w && (s < 0 || s >= n - 1)) { f = 0.f; s = s < 0 ? 0 : n - 1; }
  w0 = __float2int_rn(__fmul_rn(1.f - f, 2048.f));
  w1 = __float2int_rn(__fmul_rn(f, 2048.f));
  s0 = min(max(s, 0), n - 1);
  s1 = min(max(s + 1, 0), n - 1);
}

// channel c of the image the kernels compute on is channel ch<kSwapRB>(c) of the source
template <bool kSwapRB>
__device__ __forceinline__ int ch(int c) { return kSwapRB ? 2 - c : c; }

template <bool kSwapRB>
__global__ void __launch_bounds__(256) face_canvas_kernel(const __grid_constant__ CanvasTable t) {
  const CanvasJob& j = t.j[blockIdx.y];
  uint8_t* out = t.out + static_cast<long long>(blockIdx.y) * kCanvas * kCanvas * 3;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < kCanvas * kCanvas; p += gridDim.x * blockDim.x) {
    const int y = p / kCanvas - j.top, x = p % kCanvas - j.left;
    uint8_t* o = out + 3 * p;
    if (y < 0 || y >= j.rh || x < 0 || x >= j.rw) { o[0] = o[1] = o[2] = 0; continue; }
    if (j.rw == j.w && j.rh == j.h) {
      const uint8_t* s = j.src + static_cast<long long>(y) * j.pitch + x * 3;
      o[0] = s[ch<kSwapRB>(0)]; o[1] = s[ch<kSwapRB>(1)]; o[2] = s[ch<kSwapRB>(2)];
      continue;
    }
    if (j.area2) {
      const uint8_t* a = j.src + static_cast<long long>(2 * y) * j.pitch + 6 * x;
      const uint8_t* b = a + j.pitch;
      for (int c = 0; c < 3; ++c) {
        const int s = ch<kSwapRB>(c);
        o[c] = static_cast<uint8_t>((a[s] + a[3 + s] + b[s] + b[3 + s] + 2) >> 2);
      }
      continue;
    }
    int x0, x1, a0, a1, y0, y1, b0, b1;
    lin_coef(x, j.sx, j.w, true, x0, x1, a0, a1);
    lin_coef(y, j.sy, j.h, false, y0, y1, b0, b1);
    const uint8_t* r0 = j.src + static_cast<long long>(y0) * j.pitch;
    const uint8_t* r1 = j.src + static_cast<long long>(y1) * j.pitch;
    for (int c = 0; c < 3; ++c) {
      const int s = ch<kSwapRB>(c);
      const int h0 = r0[3 * x0 + s] * a0 + r0[3 * x1 + s] * a1;
      const int h1 = r1[3 * x0 + s] * a0 + r1[3 * x1 + s] * a1;
      o[c] = static_cast<uint8_t>((((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2);
    }
  }
}

// one warp: the inverse matrix m (float64, as cv2 inverts it) -> fixed-point source position of output pixel (x, y)
__device__ __forceinline__ void warp_pos(const double* m, int x, int y, int& ix, int& fx, int& iy, int& fy) {
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], y), m[2]), 1024.0)) + 16;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], y), m[5]), 1024.0)) + 16;
  const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(m[0], x), 1024.0))) >> 5;
  const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(m[3], x), 1024.0))) >> 5;
  ix = X >> 5; fx = X & 31; iy = Y >> 5; fy = Y & 31;
}

struct AlignJob {
  const uint8_t* src; int pitch, h, w;  // the original image [h,w,3], rows pitch bytes apart
  int x1, y1, cw, ch;                 // the crop
  int rw, rh;                         // the rotated canvas
  double rot[6], fin[6];              // inverse matrices of the two warps
};
struct AlignTable { uint8_t* out; AlignJob j[kAlignJobs]; };

// pixel (x, y) of the rotated canvas (cv2.warpAffine of the crop): 3 channels
template <bool kSwapRB>
__device__ __forceinline__ void rotated_px(const AlignJob& j, int x, int y, int* v) {
  v[0] = v[1] = v[2] = 0;
  if (x < 0 || x >= j.rw || y < 0 || y >= j.rh) return;        // outside the intermediate image: the second warp's border
  int ix, fx, iy, fy;
  warp_pos(j.rot, x, y, ix, fx, iy, fy);
  const int wt[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int yy = iy + (t >> 1), xx = ix + (t & 1);
    if (yy < 0 || yy >= j.ch || xx < 0 || xx >= j.cw) continue;  // outside the crop: the first warp's border
    const uint8_t* s = j.src + static_cast<long long>(j.y1 + yy) * j.pitch + (j.x1 + xx) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += s[ch<kSwapRB>(c)] * wt[t];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = min((acc[c] + (1 << 14)) >> 15, 255);
}

template <bool kSwapRB>
__global__ void __launch_bounds__(128) face_align_kernel(const __grid_constant__ AlignTable t) {
  const AlignJob& j = t.j[blockIdx.y];
  uint8_t* out = t.out + static_cast<long long>(blockIdx.y) * kFace * kFace * 3;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < kFace * kFace; p += gridDim.x * blockDim.x) {
    int ix, fx, iy, fy;
    warp_pos(j.fin, p % kFace, p / kFace, ix, fx, iy, fy);
    const int wt[4] = {(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32};
    int acc[3] = {0, 0, 0};
#pragma unroll
    for (int t4 = 0; t4 < 4; ++t4) {
      int v[3];
      rotated_px<kSwapRB>(j, ix + (t4 & 1), iy + (t4 >> 1), v);
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] += v[c] * wt[t4];
    }
    uint8_t* o = out + 3 * p;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[2 - c] = static_cast<uint8_t>(min((acc[c] + (1 << 14)) >> 15, 255));   // RGB2BGR
  }
}

// cv2's inversion of a 2x3 matrix inside warpAffine
static void invert(const double* M, double* m) {
  for (int i = 0; i < 6; ++i) m[i] = M[i];
  double D = m[0] * m[4] - m[1] * m[3];
  D = D != 0 ? 1. / D : 0;
  const double a11 = m[4] * D, a22 = m[0] * D;
  m[0] = a11; m[1] *= -D; m[3] *= -D; m[4] = a22;
  const double b1 = -m[0] * m[2] - m[1] * m[5], b2 = -m[3] * m[2] - m[4] * m[5];
  m[2] = b1; m[5] = b2;
}

static int canvas_check(const char* fn, int b, int h, int w) {
  const double s = 640.0 / std::max(h, w);
  CC_REQUIRE(static_cast<int>(w * s) >= 1 && static_cast<int>(h * s) >= 1, "%s: image %d (%dx%d) resizes to nothing", fn, b, w, h);
  return CC_OK;
}

// the canvas job of the h x w image at src, rows pitch bytes apart
static CanvasJob canvas_job(const uint8_t* src, int pitch, int h, int w) {
  CanvasJob j{};
  const double s = 640.0 / std::max(h, w);
  j.src = src; j.pitch = pitch; j.h = h; j.w = w;
  j.rw = static_cast<int>(w * s); j.rh = static_cast<int>(h * s);
  j.top = (kCanvas - j.rh) / 2; j.left = (kCanvas - j.rw) / 2;
  j.area2 = (j.w == 2 * j.rw && j.h == 2 * j.rh) ? 1 : 0;
  j.sx = 1.0 / (static_cast<double>(j.rw) / j.w);   // cv2: scale_x = 1 / inv_scale_x
  j.sy = 1.0 / (static_cast<double>(j.rh) / j.h);
  return j;
}

template <bool kSwapRB>
static int canvas_launch(const std::vector<CanvasJob>& jobs, uint8_t* d_out, cudaStream_t st) {
  const int B = static_cast<int>(jobs.size());
  for (int b0 = 0; b0 < B; b0 += kCanvasJobs) {
    const int nb = std::min(B - b0, kCanvasJobs);
    CanvasTable t{};
    t.out = d_out + static_cast<long long>(b0) * kCanvas * kCanvas * 3;
    for (int i = 0; i < nb; ++i) t.j[i] = jobs[b0 + i];
    face_canvas_kernel<kSwapRB><<<dim3(132 * 4 / nb > 0 ? std::min(132 * 4 / nb + 1, 1600) : 1, nb), 256, 0, st>>>(t);
    CC_CHECK_CUDA(cudaGetLastError());
  }
  return CC_OK;
}

static int align_check(const char* fn, int k, const cc_face_warp& f) {
  CC_REQUIRE(f.h > 0 && f.w > 0 && f.x1 >= 0 && f.y1 >= 0 && f.x2 > f.x1 && f.y2 > f.y1 && f.x2 <= f.w && f.y2 <= f.h &&
             f.rot_w > 0 && f.rot_h > 0,
             "%s: face %d: crop (%d,%d)-(%d,%d) of a %dx%d image, rotated %dx%d", fn, k, f.x1, f.y1, f.x2, f.y2, f.w, f.h, f.rot_w,
             f.rot_h);
  return CC_OK;
}

// the align job of face f of the image at src, rows pitch bytes apart
static AlignJob align_job(const cc_face_warp& f, const uint8_t* src, int pitch) {
  AlignJob j{};
  j.src = src; j.pitch = pitch; j.h = f.h; j.w = f.w;
  j.x1 = f.x1; j.y1 = f.y1; j.cw = f.x2 - f.x1; j.ch = f.y2 - f.y1; j.rw = f.rot_w; j.rh = f.rot_h;
  invert(f.rot, j.rot);
  invert(f.transform, j.fin);
  return j;
}

template <bool kSwapRB>
static int align_launch(const std::vector<AlignJob>& jobs, uint8_t* d_out, cudaStream_t st) {
  const int K = static_cast<int>(jobs.size());
  for (int k0 = 0; k0 < K; k0 += kAlignJobs) {
    const int nk = std::min(K - k0, kAlignJobs);
    AlignTable t{};
    t.out = d_out + static_cast<long long>(k0) * kFace * kFace * 3;
    for (int i = 0; i < nk; ++i) t.j[i] = jobs[k0 + i];
    face_align_kernel<kSwapRB><<<dim3(kFace * kFace / 128 + 1, nk), 128, 0, st>>>(t);
    CC_CHECK_CUDA(cudaGetLastError());
  }
  return CC_OK;
}

static int slots_check(const char* fn, const uint8_t* d_slots, int n_slots, int Hmax, int Wmax, const int32_t* h_slot, int K,
                       const void* d_out) {
  CC_REQUIRE(d_slots && h_slot && d_out && n_slots > 0 && K > 0 && Hmax > 0 && Wmax > 0,
             "%s: bad argument (slots %p, %d slots of %dx%d, slot table %p, %d images, out %p)", fn, d_slots, n_slots, Wmax, Hmax,
             h_slot, K, d_out);
  CC_REQUIRE(static_cast<long long>(Wmax) * 3 <= INT32_MAX, "%s: slots %d pixels wide", fn, Wmax);
  for (int k = 0; k < K; ++k)
    CC_REQUIRE(h_slot[k] >= 0 && h_slot[k] < n_slots, "%s: image %d names slot %d of %d", fn, k, h_slot[k], n_slots);
  return CC_OK;
}

static const uint8_t* slot_ptr(const uint8_t* d_slots, int slot, int Hmax, int Wmax) {
  return d_slots + static_cast<long long>(slot) * Hmax * Wmax * 3;
}

}  // namespace cc

using namespace cc;

extern "C" {

int cc_face_canvas(const cc_frame* frames, int B, uint8_t* d_out, void* stream) {
  CC_REQUIRE(frames && d_out && B > 0, "cc_face_canvas: bad argument");
  std::vector<CanvasJob> jobs(B);
  for (int b = 0; b < B; ++b) {
    const cc_frame& f = frames[b];
    CC_REQUIRE(f.data && f.fmt == CC_FRAME_BGR_U8 && f.h > 0 && f.w > 0,
               "cc_face_canvas: image %d must be a uint8 [h,w,3] device image (data %p, format %d, %dx%d)", b, f.data, f.fmt, f.w, f.h);
    if (int rc = canvas_check("cc_face_canvas", b, f.h, f.w)) return rc;
    jobs[b] = canvas_job(static_cast<const uint8_t*>(f.data), f.w * 3, f.h, f.w);
  }
  return canvas_launch<false>(jobs, d_out, static_cast<cudaStream_t>(stream));
}

int cc_face_canvas_slots(const uint8_t* d_slots, int n_slots, int Hmax, int Wmax, const int32_t* h_slot, const int32_t* h_sizes,
                         int B, uint8_t* d_out, void* stream) {
  if (int rc = slots_check("cc_face_canvas_slots", d_slots, n_slots, Hmax, Wmax, h_slot, B, d_out)) return rc;
  CC_REQUIRE(h_sizes, "cc_face_canvas_slots: h_sizes is NULL");
  std::vector<CanvasJob> jobs(B);
  for (int b = 0; b < B; ++b) {
    const int h = h_sizes[2 * b], w = h_sizes[2 * b + 1];
    CC_REQUIRE(h > 0 && w > 0 && h <= Hmax && w <= Wmax, "cc_face_canvas_slots: image %d (%dx%d) does not fit a %dx%d slot", b, w, h,
               Wmax, Hmax);
    if (int rc = canvas_check("cc_face_canvas_slots", b, h, w)) return rc;
    jobs[b] = canvas_job(slot_ptr(d_slots, h_slot[b], Hmax, Wmax), Wmax * 3, h, w);
  }
  return canvas_launch<true>(jobs, d_out, static_cast<cudaStream_t>(stream));
}

int cc_face_align(const cc_face_warp* jobs, int K, uint8_t* d_out, void* stream) {
  CC_REQUIRE(jobs && d_out && K > 0, "cc_face_align: bad argument");
  std::vector<AlignJob> aj(K);
  for (int k = 0; k < K; ++k) {
    const cc_face_warp& f = jobs[k];
    CC_REQUIRE(f.src, "cc_face_align: face %d has no image", k);
    if (int rc = align_check("cc_face_align", k, f)) return rc;
    aj[k] = align_job(f, static_cast<const uint8_t*>(f.src), f.w * 3);
  }
  return align_launch<false>(aj, d_out, static_cast<cudaStream_t>(stream));
}

int cc_face_align_slots(const uint8_t* d_slots, int n_slots, int Hmax, int Wmax, const int32_t* h_slot, const cc_face_warp* faces,
                        int K, uint8_t* d_out, void* stream) {
  if (int rc = slots_check("cc_face_align_slots", d_slots, n_slots, Hmax, Wmax, h_slot, K, d_out)) return rc;
  CC_REQUIRE(faces, "cc_face_align_slots: faces is NULL");
  std::vector<AlignJob> aj(K);
  for (int k = 0; k < K; ++k) {
    const cc_face_warp& f = faces[k];
    if (int rc = align_check("cc_face_align_slots", k, f)) return rc;
    CC_REQUIRE(f.h <= Hmax && f.w <= Wmax, "cc_face_align_slots: face %d: a %dx%d image does not fit a %dx%d slot", k, f.w, f.h,
               Wmax, Hmax);
    aj[k] = align_job(f, slot_ptr(d_slots, h_slot[k], Hmax, Wmax), Wmax * 3);
  }
  return align_launch<true>(aj, d_out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
