// Detect-head tail and postprocess of the reference detector as warp/CTA-level kernels.
//   decode_kernel      : DDetect.__call__ tail  (detection/yolov9.py:209-219) = make_anchors (:247-261), DFL softmax
//                        expectation (:279-282), dist2bbox (:263-271), x stride, sigmoid; then the head of
//                        postprocess (:440-448): xywh->xyxy, argmax/max over 80 classes, conf threshold.
//   postprocess_kernel : top-300 by prob, sorted descending with ties in ascending anchor index (:449-451),
//                        300x300 IoU (:423-437), strict upper triangle & same class & IoU>thr -> zero row (:453-458),
//                        then scale_boxes/clip_boxes (:406-421).  One CTA per image.
// fp32 throughout with explicit _rn intrinsics where an FMA contraction would change the reference's rounding.
#include "ops.cuh"
#include "cc_common.h"
#include <math_constants.h>

namespace cc {

// ------------------------------------------------------------------------------------------------ decode
// one thread per anchor; 144 fp32 logits in (float4 loads), 6 floats out.
__global__ void decode_kernel(DecodeParams p) {
  const long long total = static_cast<long long>(p.B) * p.A;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(idx / p.A);
    int a = static_cast<int>(idx % p.A);
    const int a_global = a;
    int lvl = 0;
    while (lvl < 2 && a >= p.h[lvl] * p.w[lvl]) { a -= p.h[lvl] * p.w[lvl]; ++lvl; }
    const int hw = p.h[lvl] * p.w[lvl];
    const int y = a / p.w[lvl], x = a % p.w[lvl];
    const float ax = static_cast<float>(x) + 0.5f, ay = static_cast<float>(y) + 0.5f;
    const float4* bl = reinterpret_cast<const float4*>(p.box[lvl] + (static_cast<long long>(b) * hw + a) * 64);
    float dist[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      float v[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 t = __ldg(bl + s * 4 + q);
        v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
      }
      float m = v[0];
#pragma unroll
      for (int i = 1; i < 16; ++i) m = fmaxf(m, v[i]);
      float den = 0.f, num = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float e = expf(v[i] - m);
        den += e;
        v[i] = e;
      }
      // softmax first (e/den), then the arange(16)-weighted sum, like softmax(...) followed by the 1x1 conv
#pragma unroll
      for (int i = 0; i < 16; ++i) num = __fadd_rn(num, __fmul_rn(__fdiv_rn(v[i], den), static_cast<float>(i)));
      dist[s] = num;
    }
    const float st = p.stride[lvl];
    const float x1 = __fsub_rn(ax, dist[0]), y1 = __fsub_rn(ay, dist[1]);
    const float x2 = __fadd_rn(ax, dist[2]), y2 = __fadd_rn(ay, dist[3]);
    const float xc = __fmul_rn(__fdiv_rn(__fadd_rn(x1, x2), 2.0f), st), yc = __fmul_rn(__fdiv_rn(__fadd_rn(y1, y2), 2.0f), st);
    const float w = __fmul_rn(__fsub_rn(x2, x1), st), h = __fmul_rn(__fsub_rn(y2, y1), st);

    const float4* cl = reinterpret_cast<const float4*>(p.cls[lvl] + (static_cast<long long>(b) * hw + a) * 80);
    float best = -1.f;
    int besti = 0;
    float* raw = p.raw ? p.raw + static_cast<long long>(b) * 84 * p.A + a_global : nullptr;
#pragma unroll 4
    for (int q = 0; q < 20; ++q) {
      const float4 t = __ldg(cl + q);
      const float l[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float pr = __fdiv_rn(1.0f, 1.0f + expf(-l[j]));  // sigmoid
        if (pr > best) { best = pr; besti = 4 * q + j; }       // first maximum wins ties (argmax)
        if (raw) raw[static_cast<long long>(4 + 4 * q + j) * p.A] = pr;
      }
    }
    if (raw) { raw[0] = xc; raw[p.A] = yc; raw[2LL * p.A] = w; raw[3LL * p.A] = h; }
    float* o = p.pred + idx * 6;
    o[0] = __fsub_rn(xc, __fdiv_rn(w, 2.0f));
    o[1] = __fsub_rn(yc, __fdiv_rn(h, 2.0f));
    o[2] = __fadd_rn(xc, __fdiv_rn(w, 2.0f));
    o[3] = __fadd_rn(yc, __fdiv_rn(h, 2.0f));
    o[4] = best >= p.conf_thr ? best : 0.f;
    o[5] = static_cast<float>(besti);
  }
}

int decode_launch(const DecodeParams& p, cudaStream_t s) {
  const long long total = static_cast<long long>(p.B) * p.A;
  if (total == 0) return CC_OK;
  long long blocks = (total + 127) / 128;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  decode_kernel<<<static_cast<int>(blocks), 128, 0, s>>>(p);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ head of postprocess
// detection/yolov9.py:440-448 on a (B, 4 + nc, A) head output [xc, yc, w, h, class probabilities]: xywh -> xyxy, max /
// first argmax over the classes, confidence threshold -> [B, A, 6].  thread == anchor: every one of the 4 + nc reads is
// coalesced across the warp (the anchor is the fastest axis).  The model path never runs this (decode_kernel produces the
// same six values straight from the logits); it serves the standalone `postprocess(output)` of the reference's API.
__global__ void pred_from_raw_kernel(const float* __restrict__ raw, int B, int A, int nc, float conf_thr, float* __restrict__ pred) {
  const long long total = static_cast<long long>(B) * A;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(idx / A), a = static_cast<int>(idx - static_cast<long long>(b) * A);
    const float* r = raw + static_cast<long long>(b) * (4 + nc) * A + a;
    const float xc = __ldg(r), yc = __ldg(r + A), w = __ldg(r + 2LL * A), h = __ldg(r + 3LL * A);
    float best = __ldg(r + 4LL * A);
    int besti = 0;
    for (int c = 1; c < nc; ++c) {
      const float v = __ldg(r + static_cast<long long>(4 + c) * A);
      if (v > best) { best = v; besti = c; }     // first maximum wins ties (argmax)
    }
    float* o = pred + idx * 6;
    o[0] = __fsub_rn(xc, __fdiv_rn(w, 2.0f));
    o[1] = __fsub_rn(yc, __fdiv_rn(h, 2.0f));
    o[2] = __fadd_rn(xc, __fdiv_rn(w, 2.0f));
    o[3] = __fadd_rn(yc, __fdiv_rn(h, 2.0f));
    o[4] = best >= conf_thr ? best : 0.f;
    o[5] = static_cast<float>(besti);
  }
}

int pred_from_raw_launch(const float* raw, int B, int A, int nc, float conf_thr, float* pred, cudaStream_t s) {
  CC_REQUIRE(B >= 0 && A >= 0 && nc >= 1, "pred_from_raw: bad shape B=%d A=%d nc=%d", B, A, nc);
  const long long total = static_cast<long long>(B) * A;
  if (total == 0) return CC_OK;
  long long blocks = (total + 127) / 128;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  pred_from_raw_kernel<<<static_cast<int>(blocks), 128, 0, s>>>(raw, B, A, nc, conf_thr, pred);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ postprocess
static constexpr int kPostThreads = 1024;
static constexpr int kMaxDet = 512;  // smem sized for max_det <= 512

__device__ __forceinline__ unsigned long long make_key(float prob, int idx) {
  // prob >= 0 -> its bit pattern orders like the value; ties broken towards the smaller anchor index
  return (static_cast<unsigned long long>(__float_as_uint(prob)) << 32) |
         static_cast<unsigned long long>(0xFFFFFFFFu - static_cast<unsigned>(idx));
}

__global__ void __launch_bounds__(kPostThreads) postprocess_kernel(PostParams p) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long sel[kMaxDet];
  __shared__ float rows[kMaxDet][6];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_remaining, s_count;

  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  const float* pred = p.pred + static_cast<long long>(b) * p.A * 6;
  const int K = p.max_det < p.A ? p.max_det : p.A;

  // ---- radix select of the K-th largest key, 8 bits per pass, MSB first
  if (tid == 0) { s_prefix = 0ull; s_remaining = K; s_count = 0; }
  __syncthreads();
  for (int pass = 7; pass >= 0; --pass) {
    for (int i = tid; i < 256; i += kPostThreads) hist[i] = 0;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    const unsigned long long hi_mask = pass == 7 ? 0ull : (~0ull << (8 * (pass + 1)));
    for (int i = tid; i < p.A; i += kPostThreads) {
      const unsigned long long k = make_key(__ldg(pred + i * 6 + 4), i);
      if ((k & hi_mask) == prefix) atomicAdd(&hist[(k >> (8 * pass)) & 255], 1u);
    }
    __syncthreads();
    if (tid == 0) {
      int rem = s_remaining;
      int bin = 255;
      for (; bin > 0; --bin) {
        const int c = static_cast<int>(hist[bin]);
        if (c >= rem) break;
        rem -= c;
      }
      s_remaining = rem;
      s_prefix = prefix | (static_cast<unsigned long long>(bin) << (8 * pass));
    }
    __syncthreads();
  }
  const unsigned long long kth = s_prefix;  // keys are unique -> exactly K keys are >= kth

  // ---- compact the selected keys, then bitonic-sort them descending (padding = 0 < any real key)
  for (int i = tid; i < kMaxDet; i += kPostThreads) sel[i] = 0ull;
  __syncthreads();
  for (int i = tid; i < p.A; i += kPostThreads) {
    const unsigned long long k = make_key(__ldg(pred + i * 6 + 4), i);
    if (k >= kth) {
      const int pos = atomicAdd(&s_count, 1);
      if (pos < kMaxDet) sel[pos] = k;
    }
  }
  __syncthreads();
  for (int size = 2; size <= kMaxDet; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = tid; t < kMaxDet / 2; t += kPostThreads) {
        const int lo = (t / stride) * 2 * stride + (t % stride);
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);  // first half of each `size` block descending
        const unsigned long long a = sel[lo], c = sel[hi];
        if ((a < c) == desc) { sel[lo] = c; sel[hi] = a; }
      }
      __syncthreads();
    }
  }

  // ---- gather rows
  for (int r = tid; r < K; r += kPostThreads) {
    const int idx = static_cast<int>(0xFFFFFFFFu - static_cast<unsigned>(sel[r] & 0xFFFFFFFFull));
    const float* src = pred + static_cast<long long>(idx) * 6;
#pragma unroll
    for (int j = 0; j < 6; ++j) rows[r][j] = __ldg(src + j);
  }
  __syncthreads();

  // ---- one-shot suppression: row j is zeroed iff ANY i<j has the same class and IoU(i,j) > thr
  for (int j = tid; j < p.max_det; j += kPostThreads) {
    float* o = p.out + (static_cast<long long>(b) * p.max_det + j) * 6;
    if (j >= K) {
#pragma unroll
      for (int q = 0; q < 6; ++q) o[q] = 0.f;
      continue;
    }
    const float jx1 = rows[j][0], jy1 = rows[j][1], jx2 = rows[j][2], jy2 = rows[j][3], jc = rows[j][5];
    const float ja = __fmul_rn(__fsub_rn(jx2, jx1), __fsub_rn(jy2, jy1));
    bool keep = true;
    for (int i = 0; i < j; ++i) {
      if (rows[i][5] != jc) continue;
      const float ix1 = rows[i][0], iy1 = rows[i][1], ix2 = rows[i][2], iy2 = rows[i][3];
      const float ia = __fmul_rn(__fsub_rn(ix2, ix1), __fsub_rn(iy2, iy1));
      const float w = fmaxf(0.f, __fsub_rn(fminf(ix2, jx2), fmaxf(ix1, jx1)));
      const float h = fmaxf(0.f, __fsub_rn(fminf(iy2, jy2), fmaxf(iy1, jy1)));
      const float inter = __fmul_rn(w, h);
      const float uni = __fsub_rn(__fadd_rn(ia, ja), inter);
      const float iou = __fdiv_rn(inter, uni);
      if (iou > p.iou_thr) { keep = false; break; }
    }
    const float k = keep ? 1.f : 0.f;
    float x1 = __fmul_rn(jx1, k), y1 = __fmul_rn(jy1, k), x2 = __fmul_rn(jx2, k), y2 = __fmul_rn(jy2, k);
    if (p.do_scale) {
      x1 = fminf(fmaxf(__fdiv_rn(__fsub_rn(x1, p.pad_x), p.gain), 0.f), p.clip_w);
      x2 = fminf(fmaxf(__fdiv_rn(__fsub_rn(x2, p.pad_x), p.gain), 0.f), p.clip_w);
      y1 = fminf(fmaxf(__fdiv_rn(__fsub_rn(y1, p.pad_y), p.gain), 0.f), p.clip_h);
      y2 = fminf(fmaxf(__fdiv_rn(__fsub_rn(y2, p.pad_y), p.gain), 0.f), p.clip_h);
    }
    o[0] = x1; o[1] = y1; o[2] = x2; o[3] = y2;
    o[4] = __fmul_rn(rows[j][4], k);
    o[5] = __fmul_rn(jc, k);
  }
}

int postprocess_launch(const PostParams& p, cudaStream_t s) {
  CC_REQUIRE(p.max_det >= 1 && p.max_det <= kMaxDet, "postprocess: max_det must be in [1,%d]", kMaxDet);
  if (p.B == 0) return CC_OK;
  postprocess_kernel<<<p.B, kPostThreads, 0, s>>>(p);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // namespace cc
