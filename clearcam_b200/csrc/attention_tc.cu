// Multi-head attention on Hopper warpgroup MMA (sm_90a), d_head = 64:  ctx = softmax(Q K^T / 8 [+ causal mask]) V per
// (image, head).  Reference: models/objects.py:108-118 (image tower), :157-168 (text tower, causal).
//
// One CTA = one warpgroup = 64 query rows of one (image, head).  Q, the K rows and a V^T copy of the keys it needs are
// TMA-loaded once (128B-swizzled, K-major), then the warpgroup walks 64-key blocks with an online softmax (flash):
//   S[64 x 64]  = Q[64 x 64] . K_j[64 x 64]^T     wgmma, both operands from shared memory, fp32 accumulators in registers
//   softmax     : row max / rescale / exp2 on the accumulator fragments (a row lives in the four lanes of a quad)
//   O[64 x 64] += P_j[64 x 64] . Vt_j[64 x 64]^T  wgmma with P straight from registers (the S fragment, rounded to bf16)
//   ctx         = O / rowsum -> bf16
// V is consumed as a K-major B operand, so a small pre-pass writes V^T per head ([B*H*64, Lk], keys contiguous, zero
// padded to Lk = ceil(L/64)*64); Q and K are read in place from the fused QKV buffer through one 2-D tensor map.
#include "ops.cuh"
#include "cc_common.h"
#include "cc_ptx.cuh"
#include <math.h>

namespace cc {

static constexpr int kMaxLk = 384;   // shared memory holds K and V^T of up to 384 keys (2 x 48 KB)

struct AttnParams {
  CUtensorMap tmQK;   // qkv viewed as [B*L rows][3W cols], box 64 rows x 64 cols
  CUtensorMap tmVt;   // Vt [B*H*64 rows][Lk cols], box 64 rows x 64 cols
  __nv_bfloat16* ctx;
  int L, Lk, H, W, causal;
};

// ---------------------------------------------------------------- V^T pre-pass
__global__ void __launch_bounds__(256) vt_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ vt, int L,
                                                 int Lk, int H, int W) {
  __shared__ __nv_bfloat16 tile[64][66];
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  const int t0 = blockIdx.y * 64;
  const __nv_bfloat16* src = qkv + static_cast<long long>(b) * L * 3 * W + 2 * W + h * 64;
  for (int i = threadIdx.x; i < 64 * 8; i += 256) {   // 64 tokens x 8 chunks of 8 d
    const int t = i >> 3, c = (i & 7) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (t0 + t < L) v = __ldg(reinterpret_cast<const uint4*>(src + static_cast<long long>(t0 + t) * 3 * W + c));
    const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) tile[t][c + j] = e[j];
  }
  __syncthreads();
  __nv_bfloat16* dst = vt + static_cast<long long>(bh) * 64 * Lk + t0;
  for (int i = threadIdx.x; i < 64 * 64; i += 256) {
    const int d = i >> 6, t = i & 63;
    dst[static_cast<long long>(d) * Lk + t] = tile[t][d];
  }
}

__device__ __forceinline__ uint32_t attn_pack(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float attn_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ---------------------------------------------------------------- main kernel
__global__ void __launch_bounds__(128) attention_tc_kernel(const __grid_constant__ AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int qb = blockIdx.x, bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int L = p.L;
  const int nkb_all = p.Lk >> 6;
  // causal: the keys of this query block's rows end at its last row
  const int nkb = p.causal ? (qb + 1 < nkb_all ? qb + 1 : nkb_all) : nkb_all;
  uint8_t* sQ = smem;                       // [64 rows][128 B]
  uint8_t* sK = sQ + 8192;                  // nkb x [64 keys][128 B]
  uint8_t* sV = sK + nkb_all * 8192;        // nkb x [64 d][128 B] (keys of block j)
  uint64_t* bar = reinterpret_cast<uint64_t*>(sV + nkb_all * 8192);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int row0 = b * L;                   // first token of this image in the QKV / ctx buffers

  if (tid == 0) {
    tma_prefetch_desc(&p.tmQK);
    tma_prefetch_desc(&p.tmVt);
    mbar_init(bar, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(bar, 8192 + 2 * nkb * 8192);
    tma_load_2d(sQ, &p.tmQK, bar, h * 64, row0 + 64 * qb);
    for (int j = 0; j < nkb; ++j) {
      tma_load_2d(sK + j * 8192, &p.tmQK, bar, p.W + h * 64, row0 + 64 * j);
      tma_load_2d(sV + j * 8192, &p.tmVt, bar, 64 * j, bh * 64);
    }
  }
  __syncthreads();
  mbar_wait(bar, 0);

  const uint64_t qdesc = gmma_desc(smem_u32(sQ), 128);
  const uint64_t kdesc = gmma_desc(smem_u32(sK), 128);
  const uint64_t vdesc = gmma_desc(smem_u32(sV), 128);
  const float kScale = 0.125f * 1.4426950408889634f;   // 1/sqrt(64) * log2(e)
  const int q0 = 64 * qb + 16 * warp + (lane >> 2), q1 = q0 + 8;   // this thread's two query rows
  const int cq = 2 * (lane & 3);                                   // its first column inside each 8-column group

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int j = 0; j < nkb; ++j) {
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<64>::mma(s, qdesc + 2 * k, kdesc + j * (8192 >> 4) + 2 * k, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    // mask (keys past the image, or after the query when causal), scale to the log2 domain, row maxima
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = 64 * j + 8 * i + cq + e;
        const bool ok0 = key < L && (!p.causal || key <= q0), ok1 = key < L && (!p.causal || key <= q1);
        s[4 * i + e] = ok0 ? s[4 * i + e] * kScale : -INFINITY;
        s[4 * i + 2 + e] = ok1 ? s[4 * i + 2 + e] * kScale : -INFINITY;
        mx0 = fmaxf(mx0, s[4 * i + e]);
        mx1 = fmaxf(mx1, s[4 * i + 2 + e]);
      }
#pragma unroll
    for (int d = 1; d <= 2; d <<= 1) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, d));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, d));
    }
    // key 0 is visible to every row, so after the first block the maxima are finite
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float a0 = attn_exp2(m0 - mn0), a1 = attn_exp2(m1 - mn1);
    m0 = mn0; m1 = mn1;
    float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        s[4 * i + e] = attn_exp2(s[4 * i + e] - mn0);
        s[4 * i + 2 + e] = attn_exp2(s[4 * i + 2 + e] - mn1);
        sum0 += s[4 * i + e];
        sum1 += s[4 * i + 2 + e];
        o[4 * i + e] *= a0;
        o[4 * i + 2 + e] *= a1;
      }
    l0 = l0 * a0 + sum0;
    l1 = l1 * a1 + sum1;
    // P (bf16, unnormalised, <= 1) as the register A operand: K step kk covers keys 16 kk .. 16 kk + 15 of the block
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      a[kk][0] = attn_pack(s[8 * kk + 0], s[8 * kk + 1]);
      a[kk][1] = attn_pack(s[8 * kk + 2], s[8 * kk + 3]);
      a[kk][2] = attn_pack(s[8 * kk + 4], s[8 * kk + 5]);
      a[kk][3] = attn_pack(s[8 * kk + 6], s[8 * kk + 7]);
    }
    wgmma_fence_acc(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs_m64n64(o, a[kk], vdesc + j * (8192 >> 4) + 2 * kk, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
  }
#pragma unroll
  for (int d = 1; d <= 2; d <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, d);
    l1 += __shfl_xor_sync(0xffffffffu, l1, d);
  }
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  __nv_bfloat16* out0 = p.ctx + (static_cast<long long>(row0) + q0) * p.W + h * 64 + cq;
  __nv_bfloat16* out1 = out0 + 8ll * p.W;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (q0 < L) *reinterpret_cast<uint32_t*>(out0 + 8 * i) = attn_pack(o[4 * i] * inv0, o[4 * i + 1] * inv0);
    if (q1 < L) *reinterpret_cast<uint32_t*>(out1 + 8 * i) = attn_pack(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
  }
}

// ---------------------------------------------------------------- host
bool attention_tc_supported(int L) {
  // sequences longer than 128 tokens (ViT-L/14's 257) that fit; shorter ones run the mma.sync kernel of vit.cu
  return L > 128 && (L + 63) / 64 * 64 <= kMaxLk;
}
int attention_tc_max_len() { return kMaxLk; }
size_t attention_tc_workspace_bytes(int B, int L, int H) {
  return static_cast<size_t>(B) * H * 64 * ((L + 63) / 64 * 64) * 2;
}

int attention_tc_launch(const __nv_bfloat16* qkv, __nv_bfloat16* ctx, __nv_bfloat16* vt_ws, int B, int L, int H, int causal,
                        cudaStream_t st) {
  if (B == 0) return CC_OK;
  const int W = H * 64, Lk = (L + 63) / 64 * 64, nkb = Lk / 64;
  CC_REQUIRE(Lk <= kMaxLk, "attention_tc: sequence length %d too long", L);
  PFN_encodeTiled enc = get_encode_tiled();
  CC_REQUIRE(enc != nullptr, "attention_tc: cuTensorMapEncodeTiled unavailable");
  AttnParams p{};
  p.ctx = ctx; p.L = L; p.Lk = Lk; p.H = H; p.W = W; p.causal = causal;
  {
    cuuint64_t dims[2] = {cuuint64_t(3) * W, cuuint64_t(B) * L};
    cuuint64_t strides[1] = {cuuint64_t(3) * W * 2};
    cuuint32_t box[2] = {64, 64}, estr[2] = {1, 1};
    CUresult r = enc(&p.tmQK, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<__nv_bfloat16*>(qkv), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CC_REQUIRE(r == CUDA_SUCCESS, "attention_tc: tensor map (QK) failed: %d", int(r));
  }
  {
    cuuint64_t dims[2] = {cuuint64_t(Lk), cuuint64_t(B) * H * 64};
    cuuint64_t strides[1] = {cuuint64_t(Lk) * 2};
    cuuint32_t box[2] = {64, 64}, estr[2] = {1, 1};
    CUresult r = enc(&p.tmVt, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, vt_ws, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CC_REQUIRE(r == CUDA_SUCCESS, "attention_tc: tensor map (Vt) failed: %d", int(r));
  }
  vt_kernel<<<dim3(B * H, nkb), 256, 0, st>>>(qkv, vt_ws, L, Lk, H, W);
  CC_CHECK_CUDA(cudaGetLastError());
  const int smem = 1024 + 8192 + 2 * nkb * 8192 + 64;
  static bool attr_set = false;
  if (!attr_set) {
    CC_CHECK_CUDA(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 1024 + 8192 + 2 * (kMaxLk / 64) * 8192 + 64));
    attr_set = true;
  }
  attention_tc_kernel<<<dim3((L + 63) / 64, B * H), 128, smem, st>>>(p);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // namespace cc
