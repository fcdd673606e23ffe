// Stem conv on Hopper warpgroup MMA straight from the uint8 frame (no im2col round trip through HBM).
//
// What it replaces in the reference: `frame[..., ::-1] / 255` (detection/yolov9.py:378-379) folded into model[0] =
// Conv(3, c, 3, 2) = conv 3x3 / s2 / p1 + bias + SiLU (:33-38, :303; also model[1] and model[15] of size e).
//
// Raw pixel values 0..255 are exact in bf16, the weights are bf16(w / 255) with the 27 taps in (r, s, RGB) order (RGB
// channel c = frame channel 2 - c), K padded to 32.  GEMM view: M = output pixels (flattened n, oy, ox), N = Cout, K = 32.
// One CTA = 128 threads = one warpgroup = one 128-pixel tile at a time:
//   thread == output pixel: 27 byte gathers (L1-resident: neighbouring pixels share two thirds of their window)
//     -> its 64-B row of the A tile, written in the SWIZZLE_64B K-major layout the MMA reads
//   the warpgroup: four wgmma (two 64-row halves x two K = 16 steps, N = Cout), accumulators in registers
//   from the accumulator fragments: +bias -> SiLU -> bf16 -> swizzled staging -> ONE TMA store of the tile
// The chain inside a CTA is serial; 5 CTAs are co-resident per SM (28 KB shared memory each) and hide each other's
// latencies; 5 x 128 threads leave each thread up to 102 registers, and the Cout = 64 variant needs 94 to keep its
// accumulators without serialising the wgmma.
// Bound: HBM (frame bytes in, 2*Cout bytes per output pixel out).
#include "ops.cuh"
#include "cc_common.h"
#include "cc_ptx.cuh"

namespace cc {


__device__ __forceinline__ float stem_silu(float x) {
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}
__device__ __forceinline__ uint32_t stem_pack(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int COUT>
__global__ void __launch_bounds__(128, 5) stem_tc_kernel(const __grid_constant__ StemTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                 // 128 rows x 64 B
  uint8_t* sW = sA + 8192;            // Cout rows x 64 B (<= 4 KB)
  uint8_t* sC = sW + 4096;            // 128 rows x 2*Cout B staging (<= 16 KB)
  float* sBias = reinterpret_cast<float*>(sC + 16384);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) tma_prefetch_desc(&p.tmC);
  for (int i = tid; i < COUT * 4; i += 128) {      // weights -> SWIZZLE_64B K-major rows
    const int r = i >> 2, j = i & 3;
    *reinterpret_cast<uint4*>(sW + r * 64 + ((j ^ ((r >> 1) & 3)) << 4)) = __ldg(reinterpret_cast<const uint4*>(p.w + r * 32) + j);
  }
  if (tid < COUT) sBias[tid] = __ldg(p.bias + tid);
  __syncthreads();

  const int Ho = p.H >> 1, Wo = p.W >> 1;
  const uint64_t dconst = gmma_desc_const(64, 512);   // SWIZZLE_64B, SBO = 8 rows x 64 B
  const uint64_t adesc = dconst | ((smem_u32(sA) & 0x3FFFF) >> 4), bdesc = dconst | ((smem_u32(sW) & 0x3FFFF) >> 4);
  constexpr uint32_t rb = COUT * 2, swz_mask = (rb >> 4) - 1;   // staging row bytes (32 / 64 / 128) and its TMA swizzle span

  for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
    // ---- gather: this thread's output pixel
    const long long idx = static_cast<long long>(tile) * 128 + tid;
    float v[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = 0.f;
    if (idx < p.Mrows) {
      const int n = static_cast<int>(idx / (static_cast<long long>(Ho) * Wo));
      const int rem = static_cast<int>(idx - static_cast<long long>(n) * Ho * Wo);
      const int oy = rem / Wo, ox = rem - oy * Wo;
      const uint8_t* img = p.in + static_cast<long long>(n) * p.H * p.W * 3;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int iy = 2 * oy + r - 1;
        if (iy < 0 || iy >= p.H) continue;
        const uint8_t* rowp = img + static_cast<long long>(iy) * p.W * 3;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int ix = 2 * ox + s - 1;
          if (ix < 0 || ix >= p.W) continue;
          const uint8_t* px = rowp + ix * 3;
#pragma unroll
          // byte -> float without the conversion unit (I2F shares its pipe with the MUFU.TANH of the epilogue):
          // 0x4B000000 | b is the float 2^23 + b exactly, one subtraction leaves b
          for (int c = 0; c < 3; ++c) v[(r * 3 + s) * 3 + c] = __uint_as_float(0x4B000000u | __ldg(px + 2 - c)) - 8388608.0f;
        }
      }
    }
    if (tid == 0) tma_store_wait_read<0>();     // the previous tile's store has read the staging buffer
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint4*>(sA + tid * 64 + ((j ^ ((tid >> 1) & 3)) << 4)) =
          make_uint4(stem_pack(v[8 * j], v[8 * j + 1]), stem_pack(v[8 * j + 2], v[8 * j + 3]), stem_pack(v[8 * j + 4], v[8 * j + 5]),
                     stem_pack(v[8 * j + 6], v[8 * j + 7]));
    fence_proxy_async_smem();                   // generic-proxy A tile -> visible to wgmma
    __syncthreads();
    // ---- the warpgroup: rows 0..63 and 64..127 of the tile, K = 32 in two steps
    float acc0[COUT / 2], acc1[COUT / 2];
    wgmma_fence();
    Wgmma<COUT>::mma(acc0, adesc, bdesc, 0u);
    Wgmma<COUT>::mma(acc0, adesc + 2, bdesc + 2, 1u);
    Wgmma<COUT>::mma(acc1, adesc + (4096 >> 4), bdesc, 0u);
    Wgmma<COUT>::mma(acc1, adesc + (4096 >> 4) + 2, bdesc + 2, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(acc0);
    wgmma_fence_acc(acc1);
    // ---- epilogue from the fragments: +bias -> SiLU -> bf16 pairs -> swizzled staging
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float* acc = h ? acc1 : acc0;
#pragma unroll
      for (int i = 0; i < COUT / 8; ++i) {
        const int col = 8 * i + 2 * (lane & 3);
        const float b0 = sBias[col], b1 = sBias[col + 1];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int r = 64 * h + 16 * warp + (lane >> 2) + 8 * q;
          const uint32_t off = r * rb + col * 2;
          *reinterpret_cast<uint32_t*>(sC + (off ^ (((off >> 7) & swz_mask) << 4))) =
              stem_pack(stem_silu(acc[4 * i + 2 * q] + b0), stem_silu(acc[4 * i + 2 * q + 1] + b1));
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (tid == 0) {
      tma_store_2d(&p.tmC, sC, 0, tile * 128);   // rows past Mrows are clipped
      tma_store_commit();
    }
  }
  if (tid == 0) tma_store_wait_all();
}

int stem_tc_build(int B, int H, int W, const __nv_bfloat16* w32, const float* bias, int Cout, const TSlice& out, StemTcParams* q) {
  CC_REQUIRE(H % 2 == 0 && W % 2 == 0, "stem_tc: odd frame %dx%d", H, W);
  CC_REQUIRE(Cout == 16 || Cout == 32 || Cout == 64, "stem_tc: Cout=%d (16, 32 or 64)", Cout);
  CC_REQUIRE(!out.f32 && out.C == Cout && (out.cs * 2) % 16 == 0 && (out.co * 2) % 16 == 0, "stem_tc: bad output slice");
  PFN_encodeTiled enc = get_encode_tiled();
  CC_REQUIRE(enc != nullptr, "stem_tc: cuTensorMapEncodeTiled unavailable");
  StemTcParams& p = *q;
  p = StemTcParams{};
  p.in = nullptr; p.w = w32; p.bias = bias; p.B = B; p.H = H; p.W = W; p.Cout = Cout;
  p.Mrows = static_cast<long long>(B) * (H / 2) * (W / 2);
  CC_REQUIRE(p.Mrows < (1ll << 31) - 128, "stem_tc: too many output pixels");
  p.tiles = static_cast<int>((p.Mrows + 127) / 128);
  cuuint64_t dims[2] = {cuuint64_t(Cout), cuuint64_t(p.Mrows)};
  cuuint64_t strides[1] = {cuuint64_t(out.cs) * 2};
  cuuint32_t box[2] = {cuuint32_t(Cout), 128}, estr[2] = {1, 1};
  const CUtensorMapSwizzle swz = Cout == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (Cout == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult r = enc(&p.tmC, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, out.p + out.co, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  CC_REQUIRE(r == CUDA_SUCCESS, "stem_tc: tensor map failed: %d", int(r));
  return CC_OK;
}

template <int COUT>
static cudaError_t stem_launch_cout(const StemTcParams& p, int grid, int smem, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(stem_tc_kernel<COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  stem_tc_kernel<COUT><<<grid, 128, smem, st>>>(p);
  return cudaSuccess;
}

int stem_tc_launch(const StemTcParams& q, const uint8_t* frames, cudaStream_t st) {
  StemTcParams p = q;
  p.in = frames;
  const int smem = 1024 + 8192 + 4096 + 16384 + 256;
  const int sms = device_sm_count();
  int grid = 5 * (sms > 0 ? sms : 132);
  if (grid > p.tiles) grid = p.tiles;
  switch (p.Cout) {
    case 16: CC_CHECK_CUDA(stem_launch_cout<16>(p, grid, smem, st)); break;
    case 32: CC_CHECK_CUDA(stem_launch_cout<32>(p, grid, smem, st)); break;
    default: CC_CHECK_CUDA(stem_launch_cout<64>(p, grid, smem, st)); break;
  }
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // namespace cc
