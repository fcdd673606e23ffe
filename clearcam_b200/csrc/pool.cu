// Memory-bound NHWC kernels of the detector: pools, upsample, CBFuse, letterbox, stem.
// All are HBM/L2-bound byte movers: one thread = one output pixel x 8 channels (one 16-byte vector), consecutive
// threads = consecutive channel vectors then consecutive pixels -> fully coalesced 16-B accesses; grids are
// sized to cover the tensor once (grid-stride, capped at a multiple of the 148 SMs).
#include "ops.cuh"
#include "cc_common.h"
#include "clearcam_b200.h"
#include <stdlib.h>

namespace cc {

struct bf8 { float v[8]; };

// Element type of a slice: bf16 (default path) or float (fp32-accurate mode, TSlice::f32).  All kernels below compute in
// fp32 either way; only the loads / stores of 8 consecutive channels differ.
template <typename E> struct Vec8;
template <> struct Vec8<__nv_bfloat16> {
  typedef uint4 raw_t;                                       // 8 packed elements as loaded (kept packed while in flight)
  static __device__ __forceinline__ raw_t ld_raw(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
  static __device__ __forceinline__ bf8 ld(const __nv_bfloat16* p) { return unpack(ld_raw(p)); }
  static __device__ __forceinline__ bf8 unpack(const raw_t& u) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    bf8 r;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      r.v[2 * i] = __uint_as_float(w[i] << 16);            // bf16 -> fp32 is a shift
      r.v[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    }
    return r;
  }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, const bf8& r) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(r.v[2 * i], r.v[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  }
  static __device__ __forceinline__ float round_store(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
};
template <> struct Vec8<float> {
  typedef bf8 raw_t;
  static __device__ __forceinline__ raw_t ld_raw(const float* p) { return ld(p); }
  static __device__ __forceinline__ bf8 unpack(const raw_t& u) { return u; }
  static __device__ __forceinline__ bf8 ld(const float* p) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    bf8 r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
  }
  static __device__ __forceinline__ void st(float* p, const bf8& r) {
    reinterpret_cast<float4*>(p)[0] = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
    reinterpret_cast<float4*>(p)[1] = make_float4(r.v[4], r.v[5], r.v[6], r.v[7]);
  }
  static __device__ __forceinline__ float round_store(float x) { return x; }
};
template <typename E>
__device__ __forceinline__ const E* at(const TSlice& t, int n, int h, int w, int c) {
  return reinterpret_cast<const E*>(t.p) + ((static_cast<long long>(n) * t.H + h) * t.W + w) * t.cs + t.co + c;
}
template <typename E>
__device__ __forceinline__ E* at_w(const TSlice& t, int n, int h, int w, int c) {
  return reinterpret_cast<E*>(t.p) + ((static_cast<long long>(n) * t.H + h) * t.W + w) * t.cs + t.co + c;
}
// launch KERNEL<bf16> or KERNEL<float> by the slice's element type
#define CC_LAUNCH_E(KERNEL, F32, GRID, BLOCK, STREAM, ...)                                   \
  do {                                                                                        \
    if (F32) KERNEL<float><<<GRID, BLOCK, 0, STREAM>>>(__VA_ARGS__);                          \
    else KERNEL<__nv_bfloat16><<<GRID, BLOCK, 0, STREAM>>>(__VA_ARGS__);                      \
  } while (0)

static int grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = 132LL * 32;
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

#define CC_GRID_STRIDE(idx, total) \
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < (total); \
       idx += static_cast<long long>(gridDim.x) * blockDim.x)

// Row-structured launches for the pools: blockIdx.z = image, blockIdx.y = output row, x covers (pixel, 8-channel vector)
// of that row with 32-bit index math.  The first version decoded a flat 64-bit index per element — four 64-bit divisions,
// several hundred instructions, more than the actual work of a pool; the kernels were instruction-bound at 1.4-3 TB/s.
struct RowIdx { int n, h, w, c; bool ok; };
__device__ __forceinline__ RowIdx row_index(int W, int c8) {
  RowIdx r;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  r.n = blockIdx.z;
  r.h = blockIdx.y;
  r.w = i / c8;
  r.c = (i - r.w * c8) * 8;
  r.ok = r.w < W;
  return r;
}
static dim3 row_grid(const TSlice& out, int threads) {
  const int per_row = out.W * (out.C / 8);
  return dim3((per_row + threads - 1) / threads, out.H, out.N);
}
static int row_threads(const TSlice& out) {
  const int per_row = out.W * (out.C / 8);
  return per_row >= 256 ? 256 : (per_row >= 128 ? 128 : 64);
}

// ---------------------------------------------------------------- avg 2x2 s1 -> same-size zero-edged map
template <typename E>
__global__ void avgpool2_pad_kernel(TSlice in, TSlice out) {
  const RowIdx q = row_index(out.W, in.C / 8);
  if (!q.ok) return;
  bf8 r;
  if (q.h < in.H - 1 && q.w < in.W - 1) {
    const E* p0 = at<E>(in, q.n, q.h, q.w, q.c);
    const E* p1 = p0 + static_cast<long long>(in.W) * in.cs;
    const bf8 a = Vec8<E>::ld(p0), b = Vec8<E>::ld(p0 + in.cs), d = Vec8<E>::ld(p1), e = Vec8<E>::ld(p1 + in.cs);
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = ((a.v[i] + b.v[i]) + (d.v[i] + e.v[i])) * 0.25f;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = 0.f;
  }
  Vec8<E>::st(at_w<E>(out, q.n, q.h, q.w, q.c), r);
}
int avgpool2_pad_launch(const TSlice& in, const TSlice& out, cudaStream_t s) {
  CC_REQUIRE(in.C % 8 == 0 && in.co % 8 == 0 && in.cs % 8 == 0 && out.co % 8 == 0 && out.cs % 8 == 0 && in.C == out.C &&
                 in.H == out.H && in.W == out.W, "avgpool2_pad: bad slices");
  CC_REQUIRE(out.H <= 65535 && out.N <= 65535, "avgpool2_pad: tensor too large for the row grid");
  CC_REQUIRE(in.f32 == out.f32, "avgpool2_pad: mixed element types");
  const int t = row_threads(out);
  CC_LAUNCH_E(avgpool2_pad_kernel, in.f32, row_grid(out, t), t, s, in, out);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- max3x3 s2 p1 of avg2x2 s1 (ADown branch 2)
// Output (oy, ox) = max over the avg map at rows 2oy-1..2oy+1, cols 2ox-1..2ox+1 (inside the (H-1)x(W-1) avg map), each
// avg = ((a+b)+(d+e))*0.25 rounded to bf16 first (the reference max-pools the stored avg map).  Separable: the row-pair
// sums (a+b) are shared by vertically adjacent averages, so the 4x4 input window is read once (16 vector loads instead of
// 36) and the additions keep the reference's order.
template <typename E>
__global__ void __launch_bounds__(256, 2) avgmax_pool_kernel(TSlice in, TSlice out) {
  const RowIdx q = row_index(out.W, in.C / 8);
  if (!q.ok) return;
  const int Ha = in.H - 1, Wa = in.W - 1;
  const int y0 = 2 * q.h - 1, x0 = 2 * q.w - 1;
  // all 16 vector loads of the 4x4 window go out first (clamped coordinates: always in bounds, never used when the
  // position is outside the map) — the kernel is latency-bound, so bytes in flight per SM are what buys bandwidth
  typename Vec8<E>::raw_t raw[4][4];
  const E* base = at<E>(in, q.n, 0, 0, q.c);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int y = min(max(y0 + r, 0), in.H - 1);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int x = min(max(x0 + c, 0), in.W - 1);
      raw[r][c] = Vec8<E>::ld_raw(base + (static_cast<long long>(y) * in.W + x) * in.cs);
    }
  }
  bool cv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) cv[c] = (x0 + c >= 0) && (x0 + c < Wa);
  float m[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) m[i] = -INFINITY;
  float hp[3][8];                    // row-pair sums (a+b) of the previous input row
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    float h[3][8];
    {
      const bf8 v0 = Vec8<E>::unpack(raw[r][0]), v1 = Vec8<E>::unpack(raw[r][1]), v2 = Vec8<E>::unpack(raw[r][2]),
                v3 = Vec8<E>::unpack(raw[r][3]);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        h[0][i] = v0.v[i] + v1.v[i];
        h[1][i] = v1.v[i] + v2.v[i];
        h[2][i] = v2.v[i] + v3.v[i];
      }
    }
    if (r >= 1) {
      const int ya = y0 + r - 1;     // avg row = input rows (ya, ya+1)
      if (ya >= 0 && ya < Ha) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (cv[c]) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              // the reference max-pools the STORED (rounded) avg map; rounding to the storage type is monotonic, so
              // max(round(a_i)) == round(max(a_i)) and the one rounding happens in the final store (nine bf16 conversions
              // per element kept this kernel bound by the conversion unit: ncu sm__inst_executed_pipe_xu 37 %)
              m[i] = fmaxf(m[i], hp[c][i] + h[c][i]);          // (x 0.25 after the max: an exact scaling commutes with it)
            }
          }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int i = 0; i < 8; ++i) hp[c][i] = h[c][i];
  }
  bf8 o;
#pragma unroll
  for (int i = 0; i < 8; ++i) o.v[i] = m[i] * 0.25f;
  Vec8<E>::st(at_w<E>(out, q.n, q.h, q.w, q.c), o);
}
int avgmax_pool_launch(const TSlice& in, const TSlice& out, cudaStream_t s) {
  CC_REQUIRE(in.C % 8 == 0 && in.co % 8 == 0 && in.cs % 8 == 0 && out.co % 8 == 0 && out.cs % 8 == 0 && in.C == out.C,
             "avgmax_pool: bad slices");
  CC_REQUIRE(out.H == (in.H - 1 + 2 - 3) / 2 + 1 && out.W == (in.W - 1 + 2 - 3) / 2 + 1, "avgmax_pool: bad output extent");
  CC_REQUIRE(out.H <= 65535 && out.N <= 65535, "avgmax_pool: tensor too large for the row grid");
  CC_REQUIRE(in.f32 == out.f32, "avgmax_pool: mixed element types");
  const int t = row_threads(out);
  CC_LAUNCH_E(avgmax_pool_kernel, in.f32, row_grid(out, t), t, s, in, out);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- max 5x5 s1 p2
template <typename E>
__global__ void maxpool5_kernel(TSlice in, TSlice out) {
  const RowIdx q = row_index(out.W, in.C / 8);
  if (!q.ok) return;
  bf8 m;
#pragma unroll
  for (int i = 0; i < 8; ++i) m.v[i] = -INFINITY;
  for (int dy = -2; dy <= 2; ++dy) {
    const int y = q.h + dy;
    if (y < 0 || y >= in.H) continue;
    for (int dx = -2; dx <= 2; ++dx) {
      const int x = q.w + dx;
      if (x < 0 || x >= in.W) continue;
      const bf8 a = Vec8<E>::ld(at<E>(in, q.n, y, x, q.c));
#pragma unroll
      for (int i = 0; i < 8; ++i) m.v[i] = fmaxf(m.v[i], a.v[i]);
    }
  }
  Vec8<E>::st(at_w<E>(out, q.n, q.h, q.w, q.c), m);
}
int maxpool5_launch(const TSlice& in, const TSlice& out, cudaStream_t s) {
  CC_REQUIRE(in.C % 8 == 0 && in.co % 8 == 0 && in.cs % 8 == 0 && out.co % 8 == 0 && out.cs % 8 == 0 && in.C == out.C &&
                 in.H == out.H && in.W == out.W, "maxpool5: bad slices");
  CC_REQUIRE(out.H <= 65535 && out.N <= 65535, "maxpool5: tensor too large for the row grid");
  const int t = row_threads(out);
  CC_REQUIRE(in.f32 == out.f32, "maxpool5: mixed element types");
  CC_LAUNCH_E(maxpool5_kernel, in.f32, row_grid(out, t), t, s, in, out);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- SPP: three cascaded 5x5 max pools in one launch
// SPPELAN (detection/yolov9.py:134-149) max-pools its cv1 output three times in a row (5x5, s1, p2) and concatenates all four
// maps.  At 20x20 the three launches were latency, not work (3 x ~18 us for 13 MB).  One block per (image, 64-channel block)
// keeps the map in shared memory, runs each pool separably (row max, column max: exact, max does not round) and writes the
// three results into their channel slices of the concat buffer.  Requires H*W*128 B * 2 buffers of shared memory.
__device__ __forceinline__ uint4 max_bf16x8(uint4 a, uint4 b) {
  uint4 r;
  __nv_bfloat162* pa = reinterpret_cast<__nv_bfloat162*>(&a);
  __nv_bfloat162* pb = reinterpret_cast<__nv_bfloat162*>(&b);
  __nv_bfloat162* pr = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) pr[i] = __hmax2(pa[i], pb[i]);
  return r;
}
__global__ void __launch_bounds__(256) spp3_kernel(TSlice cat, int c1) {
  extern __shared__ uint4 spp_smem[];
  const int HW = cat.H * cat.W, W = cat.W, H = cat.H;
  uint4* sA = spp_smem;             // [HW][8] current map
  uint4* sB = spp_smem + HW * 8;    // [HW][8] row maxima
  const int n = blockIdx.y, c0 = blockIdx.x * 64;
  const __nv_bfloat16* src = cat.p + static_cast<long long>(n) * HW * cat.cs + cat.co + c0;
  for (int i = threadIdx.x; i < HW * 8; i += 256) {
    const int px = i >> 3, v = i & 7;
    sA[i] = __ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(px) * cat.cs + v * 8));
  }
  __syncthreads();
  for (int pass = 1; pass <= 3; ++pass) {
    for (int i = threadIdx.x; i < HW * 8; i += 256) {
      const int px = i >> 3, v = i & 7, y = px / W, x = px - y * W;
      uint4 m = sA[i];
#pragma unroll
      for (int dx = -2; dx <= 2; ++dx)
        if (dx != 0 && x + dx >= 0 && x + dx < W) m = max_bf16x8(m, sA[(px + dx) * 8 + v]);
      sB[i] = m;
    }
    __syncthreads();
    __nv_bfloat16* dst = cat.p + static_cast<long long>(n) * HW * cat.cs + cat.co + pass * c1 + c0;
    for (int i = threadIdx.x; i < HW * 8; i += 256) {
      const int px = i >> 3, v = i & 7, y = px / W;
      uint4 m = sB[i];
#pragma unroll
      for (int dy = -2; dy <= 2; ++dy)
        if (dy != 0 && y + dy >= 0 && y + dy < H) m = max_bf16x8(m, sB[(px + dy * W) * 8 + v]);
      sA[i] = m;                    // (every thread rewrites only its own element: readers of sA are behind the barrier above)
      *reinterpret_cast<uint4*>(dst + static_cast<long long>(px) * cat.cs + v * 8) = m;
    }
    __syncthreads();
  }
}
bool spp3_supported(const TSlice& cat, int c1) {
  return !cat.f32 && c1 % 64 == 0 && cat.co % 8 == 0 && cat.cs % 8 == 0 && static_cast<size_t>(cat.H) * cat.W * 128 * 2 <= 200 * 1024;
}
int spp3_launch(const TSlice& cat, int c1, cudaStream_t s) {
  CC_REQUIRE(spp3_supported(cat, c1) && cat.C >= 4 * c1, "spp3: unsupported slice");
  const int smem = cat.H * cat.W * 128 * 2;
  static int attr_max = 0;
  if (smem > attr_max) {
    CC_CHECK_CUDA(cudaFuncSetAttribute(spp3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_max = smem;
  }
  spp3_kernel<<<dim3(c1 / 64, cat.N), 256, smem, s>>>(cat, c1);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- nearest x2
template <typename E>
__global__ void upsample2_kernel(TSlice in, TSlice out) {
  const RowIdx q = row_index(out.W, in.C / 8);
  if (!q.ok) return;
  const uint4* src = reinterpret_cast<const uint4*>(at<E>(in, q.n, q.h >> 1, q.w >> 1, q.c));
  uint4* dst = reinterpret_cast<uint4*>(at_w<E>(out, q.n, q.h, q.w, q.c));
#pragma unroll
  for (int i = 0; i < static_cast<int>(sizeof(E)) / 2; ++i) dst[i] = __ldg(src + i);   // 8 channels = 16 B (bf16) or 32 B (float)
}
int upsample2_launch(const TSlice& in, const TSlice& out, cudaStream_t s) {
  CC_REQUIRE(in.C % 8 == 0 && in.co % 8 == 0 && in.cs % 8 == 0 && out.co % 8 == 0 && out.cs % 8 == 0 && in.C == out.C &&
                 out.H == 2 * in.H && out.W == 2 * in.W, "upsample2: bad slices");
  CC_REQUIRE(out.H <= 65535 && out.N <= 65535, "upsample2: tensor too large for the row grid");
  const int t = row_threads(out);
  CC_REQUIRE(in.f32 == out.f32, "upsample2: mixed element types");
  CC_LAUNCH_E(upsample2_kernel, in.f32, row_grid(out, t), t, s, in, out);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- CBFuse
template <typename E>
__global__ void cbfuse_kernel(CBFuseParams p) {
  const RowIdx q = row_index(p.out.W, p.out.C / 8);
  if (!q.ok) return;
  bf8 acc;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc.v[i] = 0.f;
  for (int k = 0; k < p.nsrc; ++k) {
    // nearest: src = floor(dst * in / out); the maps of the reference graphs are power-of-two multiples of each other, so
    // the host passes the ratio as a shift (two integer divisions per source per thread made this kernel instruction-bound:
    // 1.5 TB/s at 320x320)
    const int sh = p.shift[k] >= 0 ? (q.h >> p.shift[k]) : (q.h * p.src[k].H) / p.out.H;
    const int sw = p.shift[k] >= 0 ? (q.w >> p.shift[k]) : (q.w * p.src[k].W) / p.out.W;
    const bf8 a = Vec8<E>::ld(at<E>(p.src[k], q.n, sh, sw, q.c));
#pragma unroll
    for (int i = 0; i < 8; ++i) acc.v[i] = (k == 0) ? a.v[i] : acc.v[i] + a.v[i];
  }
  const bf8 l = Vec8<E>::ld(at<E>(p.last, q.n, q.h, q.w, q.c));
#pragma unroll
  for (int i = 0; i < 8; ++i) acc.v[i] += l.v[i];
  Vec8<E>::st(at_w<E>(p.out, q.n, q.h, q.w, q.c), acc);
}
int cbfuse_launch(const CBFuseParams& p0, cudaStream_t s) {
  CBFuseParams p = p0;
  CC_REQUIRE(p.nsrc >= 1 && p.nsrc <= 5 && p.out.C % 8 == 0, "cbfuse: bad params");
  for (int k = 0; k < p.nsrc; ++k) {
    p.shift[k] = -1;
    for (int sft = 0; sft < 8; ++sft)
      if ((p.src[k].H << sft) == p.out.H && (p.src[k].W << sft) == p.out.W) p.shift[k] = sft;
  }
  CC_REQUIRE(p.out.H <= 65535 && p.out.N <= 65535, "cbfuse: tensor too large for the row grid");
  const int t = row_threads(p.out);
  CC_LAUNCH_E(cbfuse_kernel, p.out.f32, row_grid(p.out, t), t, s, p);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- fp32 -> six bf16 planes (fp32-accurate mode)
// one thread = one pixel x 4 channels: float4 in, six 8-byte stores out (plane p of pixel i at out[i*6C + p*C + c])
__global__ void split_planes_kernel(const float* __restrict__ in, long long npix, int cs, int co, int C, __nv_bfloat16* __restrict__ out) {
  const int c4n = C >> 2;
  const long long total = npix * c4n;
  CC_GRID_STRIDE(idx, total) {
    const long long pix = idx / c4n;
    const int c = static_cast<int>(idx - pix * c4n) << 2;
    const float4 x = __ldg(reinterpret_cast<const float4*>(in + pix * cs + co + c));
    const float xs[4] = {x.x, x.y, x.z, x.w};
    uint32_t hi[2], mid[2], lo[2];
    __nv_bfloat16 h[4], m[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      h[j] = __float2bfloat16_rn(xs[j]);
      const float r1 = xs[j] - __bfloat162float(h[j]);          // exact (Sterbenz-like: the bf16 is within half an ulp)
      m[j] = __float2bfloat16_rn(r1);
      const float r2 = r1 - __bfloat162float(m[j]);             // exact
      l[j] = __float2bfloat16_rn(r2);                           // 8 + 8 + 8 mantissa bits: x == hi + mid + lo
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      __nv_bfloat162 t;
      t.x = h[2 * j]; t.y = h[2 * j + 1]; hi[j] = *reinterpret_cast<uint32_t*>(&t);
      t.x = m[2 * j]; t.y = m[2 * j + 1]; mid[j] = *reinterpret_cast<uint32_t*>(&t);
      t.x = l[2 * j]; t.y = l[2 * j + 1]; lo[j] = *reinterpret_cast<uint32_t*>(&t);
    }
    __nv_bfloat16* o = out + pix * (6LL * C) + c;
    *reinterpret_cast<uint2*>(o) = make_uint2(lo[0], lo[1]);
    *reinterpret_cast<uint2*>(o + C) = make_uint2(mid[0], mid[1]);
    *reinterpret_cast<uint2*>(o + 2 * C) = make_uint2(hi[0], hi[1]);
    *reinterpret_cast<uint2*>(o + 3 * C) = make_uint2(mid[0], mid[1]);
    *reinterpret_cast<uint2*>(o + 4 * C) = make_uint2(hi[0], hi[1]);
    *reinterpret_cast<uint2*>(o + 5 * C) = make_uint2(hi[0], hi[1]);
  }
}
int split_planes_launch(const TSlice& in, __nv_bfloat16* out, cudaStream_t s) {
  CC_REQUIRE(in.f32 && in.C % 4 == 0 && in.co % 4 == 0 && in.cs % 4 == 0, "split_planes: needs an fp32 slice with 16-byte aligned channels");
  const long long npix = static_cast<long long>(in.N) * in.H * in.W;
  split_planes_kernel<<<grid_for(npix * (in.C / 4), 256), 256, 0, s>>>(reinterpret_cast<const float*>(in.p), npix, in.cs, in.co, in.C, out);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- fp32-accurate mode: bias + activation + residual pass
__global__ void finish_f32_kernel(FinishParams p) {
  const int c4n = p.C >> 2;
  const long long total = p.npix * c4n;
  CC_GRID_STRIDE(idx, total) {
    const long long pix = idx / c4n;
    const int c = static_cast<int>(idx - pix * c4n) << 2;
    const float4 a = __ldg(reinterpret_cast<const float4*>(p.acc + pix * p.C + c));
    const float4 b = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float v[4] = {a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w};
    if (p.act == 1) {                                     // SiLU as the fp32 reference computes it: x * sigmoid(x), sigmoid = 1 / (1 + exp(-x))
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = __fmul_rn(v[j], __fdiv_rn(1.0f, 1.0f + expf(-v[j])));
    }
    if (p.res) {
      const float4 r = __ldg(reinterpret_cast<const float4*>(p.res + pix * p.res_cs + p.res_co + c));
      v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
    }
    *reinterpret_cast<float4*>(p.out + pix * p.out_cs + p.out_co + c) = make_float4(v[0], v[1], v[2], v[3]);
  }
}
int finish_f32_launch(const FinishParams& p, cudaStream_t s) {
  CC_REQUIRE(p.C % 4 == 0 && p.out_cs % 4 == 0 && p.out_co % 4 == 0 && (!p.res || (p.res_cs % 4 == 0 && p.res_co % 4 == 0)) && (p.act == 0 || p.act == 1),
             "finish_f32: bad slices / activation");
  finish_f32_kernel<<<grid_for(p.npix * (p.C / 4), 256), 256, 0, s>>>(p);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ---------------------------------------------------------------- letterbox (bilinear, reference semantics)
__device__ __forceinline__ void lerp_idx(int i, int n_in, float scale, int& lo, int& hi, float& w) {
  // idx = clip((i+0.5)*in/out - 0.5, 0, in-1); `scale` = float(in/out) computed on the host in double
  float idx = __fsub_rn(__fmul_rn(static_cast<float>(i) + 0.5f, scale), 0.5f);
  idx = fminf(fmaxf(idx, 0.f), static_cast<float>(n_in - 1));
  lo = static_cast<int>(floorf(idx));
  hi = static_cast<int>(ceilf(idx));
  w = idx - static_cast<float>(lo);
}
__device__ __forceinline__ int lerp_u8(int a, int b, int wi) {
  int diff = ((b - a + 128) & 255) - 128;     // int8 wrap-around of the reference's uint8 subtraction
  return (a + ((diff * wi + 64) >> 7)) & 255;
}
// One image of the batch.  FMT: CC_FRAME_* code of its frame, a template argument so the per-pixel path has no format
// branch (the kernel picks the instance once per CTA: a CTA covers one image).  out: the image's [Hout,Wout,3] slot.
template <int FMT>
__device__ __forceinline__ void letterbox_image(const LetterboxFrame& p, int Hout, int Wout, void* out) {
  const long long total = static_cast<long long>(Hout) * Wout;
  CC_GRID_STRIDE(idx, total) {
    const int x = static_cast<int>(idx % Wout);
    const int y = static_cast<int>(idx / Wout);
    const int ry = y - p.pad_y, rx = x - p.pad_x;
    const bool inside = ry >= 0 && ry < p.Hr && rx >= 0 && rx < p.Wr;
    int xl = 0, xh = 0, yl = 0, yh = 0;
    float wx = 0.f, wy = 0.f;
    if (inside) {
      if (p.Wr != p.Win) lerp_idx(rx, p.Win, p.sx, xl, xh, wx); else { xl = xh = rx; }
      if (p.Hr != p.Hin) lerp_idx(ry, p.Hin, p.sy, yl, yh, wy); else { yl = yh = ry; }
    }
    if constexpr (FMT == CC_FRAME_BGR_F32) {
      const float* src = static_cast<const float*>(p.in);
      float* dst = static_cast<float*>(out) + idx * 3;
      for (int c = 0; c < 3; ++c) {
        float r = 0.f;
        if (inside) {
          const float a = src[(static_cast<long long>(yl) * p.Win + xl) * 3 + c], b = src[(static_cast<long long>(yl) * p.Win + xh) * 3 + c];
          const float d = src[(static_cast<long long>(yh) * p.Win + xl) * 3 + c], e = src[(static_cast<long long>(yh) * p.Win + xh) * 3 + c];
          const float top = __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), wx));
          const float bot = __fadd_rn(d, __fmul_rn(__fsub_rn(e, d), wx));
          r = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), wy));
        }
        dst[c] = r;
      }
    } else {
      uint8_t* dst = static_cast<uint8_t*>(out) + idx * 3;
      const int wxi = static_cast<int>(static_cast<short>(wx * 128.f + 0.5f));
      const int wyi = static_cast<int>(static_cast<short>(wy * 128.f + 0.5f));
      // the four taps as BGR: a = (yl,xl), b = (yl,xh), d = (yh,xl), e = (yh,xh)
      int a[3] = {0, 0, 0}, b[3] = {0, 0, 0}, d[3] = {0, 0, 0}, e[3] = {0, 0, 0};
      if (inside) {
        if constexpr (FMT == CC_FRAME_I420_U8) {
          const uint8_t* src = static_cast<const uint8_t*>(p.in);
          i420_bgr(src, p.Hin, p.Win, yl, xl, a);
          i420_bgr(src, p.Hin, p.Win, yl, xh, b);
          i420_bgr(src, p.Hin, p.Win, yh, xl, d);
          i420_bgr(src, p.Hin, p.Win, yh, xh, e);
        } else {
          const uint8_t* src = static_cast<const uint8_t*>(p.in);
          for (int c = 0; c < 3; ++c) {
            a[c] = src[(static_cast<long long>(yl) * p.Win + xl) * 3 + c]; b[c] = src[(static_cast<long long>(yl) * p.Win + xh) * 3 + c];
            d[c] = src[(static_cast<long long>(yh) * p.Win + xl) * 3 + c]; e[c] = src[(static_cast<long long>(yh) * p.Win + xh) * 3 + c];
          }
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        int r = 0;
        if (inside) {
          const int top = (p.Wr != p.Win) ? lerp_u8(a[c], b[c], wxi) : a[c];
          const int bot = (p.Wr != p.Win) ? lerp_u8(d[c], e[c], wxi) : d[c];
          r = (p.Hr != p.Hin) ? lerp_u8(top, bot, wyi) : top;
        }
        dst[c] = static_cast<uint8_t>(r);
      }
    }
  }
}
// blockIdx.y = image of the table; x covers its pixels
__global__ void __launch_bounds__(256) letterbox_kernel(const __grid_constant__ LetterboxTable t) {
  const LetterboxFrame& f = t.f[blockIdx.y];
  const long long img = static_cast<long long>(t.Hout) * t.Wout * 3;
  void* out = t.out_f32 ? static_cast<void*>(static_cast<float*>(t.out) + blockIdx.y * img)
                        : static_cast<void*>(static_cast<uint8_t*>(t.out) + blockIdx.y * img);
  if (!f.in) {                                   // padding image
    if (t.out_f32) { float* o = static_cast<float*>(out); CC_GRID_STRIDE(i, img) o[i] = 0.f; }
    else { uint8_t* o = static_cast<uint8_t*>(out); CC_GRID_STRIDE(i, img) o[i] = 0; }
    return;
  }
  switch (f.fmt) {
    case CC_FRAME_BGR_F32: letterbox_image<CC_FRAME_BGR_F32>(f, t.Hout, t.Wout, out); break;
    case CC_FRAME_I420_U8: letterbox_image<CC_FRAME_I420_U8>(f, t.Hout, t.Wout, out); break;
    default: letterbox_image<CC_FRAME_BGR_U8>(f, t.Hout, t.Wout, out); break;
  }
}
int letterbox_frames_launch(const LetterboxTable& t, cudaStream_t s) {
  CC_REQUIRE(t.B >= 1 && t.B <= CC_MAX_FRAMES && t.Hout > 0 && t.Wout > 0 && t.out, "letterbox: bad table (B=%d, %dx%d)", t.B, t.Hout, t.Wout);
  for (int i = 0; i < t.B; ++i) {
    const LetterboxFrame& f = t.f[i];
    if (!f.in) continue;
    CC_REQUIRE((f.fmt == CC_FRAME_BGR_F32) == (t.out_f32 != 0) && (f.fmt == CC_FRAME_BGR_U8 || f.fmt == CC_FRAME_BGR_F32 || f.fmt == CC_FRAME_I420_U8),
               "letterbox: image %d has frame format %d (out_f32 %d)", i, f.fmt, t.out_f32);
    CC_REQUIRE(f.fmt != CC_FRAME_I420_U8 || (f.Hin % 2 == 0 && f.Win % 2 == 0), "letterbox: I420 frame %dx%d has an odd side", f.Hin, f.Win);
    CC_REQUIRE(f.pad_y >= 0 && f.pad_x >= 0 && f.Hr >= 0 && f.Wr >= 0 &&f.pad_y + f.Hr <= t.Hout && f.pad_x + f.Wr <= t.Wout,
               "letterbox: image %d (%dx%d at %d,%d) does not fit %dx%d", i, f.Hr, f.Wr, f.pad_y, f.pad_x, t.Hout, t.Wout);
  }
  // as many CTAs in all as the batch-wide grid-stride launch it replaces (grid_for's cap), at least one per image
  const long long per_img = (static_cast<long long>(t.Hout) * t.Wout + 255) / 256;
  long long gx = 132LL * 32 / t.B;
  gx = gx < 1 ? 1 : (gx > per_img ? per_img : gx);
  letterbox_kernel<<<dim3(static_cast<unsigned>(gx), t.B), 256, 0, s>>>(t);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}
int letterbox_launch(const LetterboxParams& p, cudaStream_t s) {
  CC_REQUIRE(p.fmt == CC_FRAME_BGR_U8 || p.fmt == CC_FRAME_BGR_F32 || p.fmt == CC_FRAME_I420_U8, "letterbox: unknown frame format %d", p.fmt);
  CC_REQUIRE(p.fmt != CC_FRAME_I420_U8 || (p.Hin % 2 == 0 && p.Win % 2 == 0), "letterbox: I420 frame %dx%d has an odd side", p.Hin, p.Win);
  const bool f32 = p.fmt == CC_FRAME_BGR_F32;
  const long long hw = static_cast<long long>(p.Hin) * p.Win;
  const long long in_bytes = f32 ? hw * 12 : p.fmt == CC_FRAME_I420_U8 ? hw * 3 / 2 : hw * 3;
  const long long out_bytes = static_cast<long long>(p.Hout) * p.Wout * 3 * (f32 ? 4 : 1);
  LetterboxTable t;
  t.Hout = p.Hout; t.Wout = p.Wout; t.out_f32 = f32 ? 1 : 0;
  for (int b0 = 0; b0 < p.B; b0 += CC_MAX_FRAMES) {          // the table holds CC_MAX_FRAMES images per launch
    t.B = p.B - b0 < CC_MAX_FRAMES ? p.B - b0 : CC_MAX_FRAMES;
    t.out = static_cast<uint8_t*>(p.out) + b0 * out_bytes;
    for (int i = 0; i < t.B; ++i) {
      LetterboxFrame& f = t.f[i];
      f.in = static_cast<const uint8_t*>(p.in) + (b0 + i) * in_bytes;
      f.fmt = p.fmt; f.Hin = p.Hin; f.Win = p.Win; f.Hr = p.Hr; f.Wr = p.Wr; f.pad_y = p.pad_y; f.pad_x = p.pad_x;
      f.sx = p.sx; f.sy = p.sy;
    }
    if (int rc = letterbox_frames_launch(t, s)) return rc;
  }
  return CC_OK;
}

// ---------------------------------------------------------------- stem conv (Cin = 3)
// block = 128 threads = 128 consecutive output pixels of one row-major run; weights (27 x Cout fp32) in smem.
// Each thread gathers its 27 inputs once (RGB order, /255) and produces all Cout channels, 16 at a time.
// F32: float frames (else uint8);  E: output element type (float = fp32-accurate mode: exact division in the SiLU)
template <bool F32, typename E>
__global__ void __launch_bounds__(128) stem_kernel(StemParams p) {
  extern __shared__ float sw[];  // [27][Cout] then bias[Cout]
  const int Cout = p.Cout;
  for (int i = threadIdx.x; i < 27 * Cout; i += blockDim.x) {
    const int co = i % Cout, k = i / Cout;  // k = (r*3+s)*3 + c
    sw[i] = p.w[co * 27 + k];
  }
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) sw[27 * Cout + i] = p.bias[i];
  __syncthreads();
  const int Ho = p.H / 2, Wo = p.W / 2;
  const long long total = static_cast<long long>(p.B) * Ho * Wo;
  CC_GRID_STRIDE(idx, total) {
    const int ox = static_cast<int>(idx % Wo);
    const int oy = static_cast<int>((idx / Wo) % Ho);
    const int n = static_cast<int>(idx / (static_cast<long long>(Wo) * Ho));
    float in[27];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = 2 * oy + r - 1;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ix = 2 * ox + s - 1;
        const bool ok = iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
        const long long off = ((static_cast<long long>(n) * p.H + iy) * p.W + ix) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          float v = 0.f;
          if (ok) {
            // channel flip: network channel c (RGB) = frame channel 2-c (BGR);  x/255 as an IEEE division
            if (F32) v = static_cast<const float*>(p.in)[off + 2 - c];
            else v = static_cast<float>(static_cast<const uint8_t*>(p.in)[off + 2 - c]);
            v = __fdiv_rn(v, 255.0f);
          }
          in[(r * 3 + s) * 3 + c] = v;
        }
      }
    }
    E* dst = reinterpret_cast<E*>(p.out.p) + ((static_cast<long long>(n) * Ho + oy) * Wo + ox) * p.out.cs + p.out.co;
    for (int c0 = 0; c0 < Cout; c0 += 8) {
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = sw[27 * Cout + c0 + j];
#pragma unroll
      for (int k = 0; k < 27; ++k) {
        const float4 w0 = *reinterpret_cast<const float4*>(&sw[k * Cout + c0]);
        const float4 w1 = *reinterpret_cast<const float4*>(&sw[k * Cout + c0 + 4]);
        acc[0] = fmaf(in[k], w0.x, acc[0]); acc[1] = fmaf(in[k], w0.y, acc[1]);
        acc[2] = fmaf(in[k], w0.z, acc[2]); acc[3] = fmaf(in[k], w0.w, acc[3]);
        acc[4] = fmaf(in[k], w1.x, acc[4]); acc[5] = fmaf(in[k], w1.y, acc[5]);
        acc[6] = fmaf(in[k], w1.z, acc[6]); acc[7] = fmaf(in[k], w1.w, acc[7]);
      }
      bf8 o;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        o.v[j] = sizeof(E) == 4 ? acc[j] / (1.0f + expf(-acc[j])) : __fdividef(acc[j], 1.0f + __expf(-acc[j]));
      Vec8<E>::st(dst + c0, o);
    }
  }
}

int stem_launch(const StemParams& p, cudaStream_t s) {
  CC_REQUIRE(p.Cout % 8 == 0 && p.H % 2 == 0 && p.W % 2 == 0 && p.out.cs % 8 == 0 && p.out.co % 8 == 0, "stem: bad shape");
  const long long total = static_cast<long long>(p.B) * (p.H / 2) * (p.W / 2);
  const int smem = (27 + 1) * p.Cout * sizeof(float);
  long long blocks = (total + 127) / 128;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  if (p.out.f32) {
    if (p.is_f32) stem_kernel<true, float><<<static_cast<int>(blocks), 128, smem, s>>>(p);
    else stem_kernel<false, float><<<static_cast<int>(blocks), 128, smem, s>>>(p);
  } else {
    if (p.is_f32) stem_kernel<true, __nv_bfloat16><<<static_cast<int>(blocks), 128, smem, s>>>(p);
    else stem_kernel<false, __nv_bfloat16><<<static_cast<int>(blocks), 128, smem, s>>>(p);
  }
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // namespace cc
