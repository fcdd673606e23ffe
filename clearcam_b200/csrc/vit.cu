// CLIP ViT encoder kernels other than the GEMMs (those run on conv_gemm.cu's wgmma kernel as 1x1 "convs").
// Reference: models/objects.py:94-133 (image tower), :145-186 (text tower).
//   patchify        : NCHW fp32 image -> bf16 patch matrix [B*P, Kpad]  (the 14x14/s14 conv :95 as a GEMM operand)
//   embed_ln_pre    : class token + positional embedding + ln_pre        (:96-102)  -> fp32 residual stream
//   text_embed      : token_embedding[ids] + positional_embedding_text   (:148-149) and the EOT row index (:183)
//   layernorm       : fp32 rows -> bf16 rows (optionally a gathered subset of rows: token 0 / EOT row) (:105,:121,:131)
//   attention       : softmax(QK^T/8 [+causal]) V per (image, head), d_head = 64 (:108-118, :157-168)
//   l2norm          : e / (||e|| + eps)                                  (:134, :186)
// Memory-bound kernels: warp per row, 16-byte vector accesses, fp32 statistics.
#include "ops.cuh"
#include "cc_common.h"
#include <cuda_bf16.h>
#include <type_traits>

namespace cc {

// ------------------------------------------------------------------------------------------------ patchify
// one thread = 8 consecutive K elements of one patch row (16-B store)
__global__ void patchify_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out, int B, int S, int p,
                                int Kpad) {
  const int G = S / p, P = G * G, K = 3 * p * p;
  const int k8 = Kpad / 8;
  const long long total = static_cast<long long>(B) * P * k8;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int kk = static_cast<int>(idx % k8) * 8;
    const long long row = idx / k8;
    const int t = static_cast<int>(row % P);
    const int b = static_cast<int>(row / P);
    const int gy = t / G, gx = t % G;
    uint32_t w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = kk + 2 * q + e;
        float val = 0.f;
        if (k < K) {
          const int c = k / (p * p), r = (k / p) % p, s = k % p;
          val = __ldg(x + ((static_cast<long long>(b) * 3 + c) * S + gy * p + r) * S + gx * p + s);
        }
        v[e] = val;
      }
      __nv_bfloat162 h = __floats2bfloat162_rn(v[0], v[1]);
      w[q] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(out + row * Kpad + kk) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}
int patchify_launch(const float* x, __nv_bfloat16* out, int B, int S, int p, int Kpad, cudaStream_t st) {
  CC_REQUIRE(S % p == 0 && Kpad % 8 == 0 && Kpad >= 3 * p * p, "patchify: bad shape");
  const long long total = static_cast<long long>(B) * (S / p) * (S / p) * (Kpad / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 32) blocks = 132LL * 32;
  patchify_kernel<<<static_cast<int>(blocks < 1 ? 1 : blocks), 256, 0, st>>>(x, out, B, S, p, Kpad);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ warp LN helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// LayerNorm of one row held as `n4` float4 per lane (W = 128*n4), eps 1e-5, two-pass statistics in fp32.
template <int N4>
__device__ __forceinline__ void ln_row(float4 (&v)[N4], const float* __restrict__ gamma, const float* __restrict__ beta,
                                       int lane, int W) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N4; ++i) s += v[i].x + v[i].y + v[i].z + v[i].w;
  const float mean = warp_sum(s) / static_cast<float>(W);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < N4; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += a * a + b * b + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) / static_cast<float>(W) + 1e-5f);
#pragma unroll
  for (int i = 0; i < N4; ++i) {
    const int c = (i * 32 + lane) * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float4 bt = __ldg(reinterpret_cast<const float4*>(beta + c));
    v[i].x = (v[i].x - mean) * rstd * g.x + bt.x;
    v[i].y = (v[i].y - mean) * rstd * g.y + bt.y;
    v[i].z = (v[i].z - mean) * rstd * g.z + bt.z;
    v[i].w = (v[i].w - mean) * rstd * g.w + bt.w;
  }
}

// ------------------------------------------------------------------------------------------------ embed + ln_pre
template <int N4>
__global__ void embed_ln_pre_kernel(float* __restrict__ x, const float* __restrict__ cls, const float* __restrict__ pos,
                                    const float* __restrict__ gamma, const float* __restrict__ beta, int rows, int L, int W) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += gridDim.x * wpb) {
    const int t = row % L;
    float* xr = x + static_cast<long long>(row) * W;
    float4 v[N4];
#pragma unroll
    for (int i = 0; i < N4; ++i) {
      const int c = (i * 32 + lane) * 4;
      const float4 a = (t == 0) ? __ldg(reinterpret_cast<const float4*>(cls + c)) : *reinterpret_cast<const float4*>(xr + c);
      const float4 pe = __ldg(reinterpret_cast<const float4*>(pos + static_cast<long long>(t) * W + c));
      v[i] = make_float4(a.x + pe.x, a.y + pe.y, a.z + pe.z, a.w + pe.w);
    }
    ln_row<N4>(v, gamma, beta, lane, W);
#pragma unroll
    for (int i = 0; i < N4; ++i) *reinterpret_cast<float4*>(xr + (i * 32 + lane) * 4) = v[i];
  }
}

// ------------------------------------------------------------------------------------------------ layernorm -> bf16
template <int N4>
__global__ void layernorm_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                      const float* __restrict__ gamma, const float* __restrict__ beta, int rows, int W,
                                      long long row_stride, const int* __restrict__ row_idx) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < rows; r += gridDim.x * wpb) {
    const long long src_row = row_idx ? static_cast<long long>(__ldg(row_idx + r)) : static_cast<long long>(r) * row_stride;
    const float* xr = x + src_row * W;
    float4 v[N4];
#pragma unroll
    for (int i = 0; i < N4; ++i) v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
    ln_row<N4>(v, gamma, beta, lane, W);
    __nv_bfloat16* o = out + static_cast<long long>(r) * W;
#pragma unroll
    for (int i = 0; i < N4; ++i) {
      __nv_bfloat162 h0 = __floats2bfloat162_rn(v[i].x, v[i].y), h1 = __floats2bfloat162_rn(v[i].z, v[i].w);
      *reinterpret_cast<uint2*>(o + (i * 32 + lane) * 4) =
          make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
    }
  }
}

template <typename F>
static int dispatch_n4(int W, F&& f) {
  switch (W / 128) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 5: return f(std::integral_constant<int, 5>{});
    case 6: return f(std::integral_constant<int, 6>{});
    case 8: return f(std::integral_constant<int, 8>{});
    case 10: return f(std::integral_constant<int, 10>{});
    case 12: return f(std::integral_constant<int, 12>{});
    default: break;
  }
  set_error("layernorm: width %d not supported (need a multiple of 128 up to 1536)", W);
  return CC_ERR_INVALID;
}

int embed_ln_pre_launch(float* x, const float* cls, const float* pos, const float* gamma, const float* beta, int rows, int L,
                        int W, cudaStream_t st) {
  CC_REQUIRE(W % 128 == 0, "embed_ln_pre: width %d not a multiple of 128", W);
  const int blocks = rows < 132 * 8 ? (rows + 7) / 8 : 132 * 4;
  return dispatch_n4(W, [&](auto n4) -> int {
    embed_ln_pre_kernel<decltype(n4)::value><<<blocks < 1 ? 1 : blocks, 256, 0, st>>>(x, cls, pos, gamma, beta, rows, L, W);
    CC_CHECK_CUDA(cudaGetLastError());
    return static_cast<int>(CC_OK);
  });
}

int layernorm_bf16_launch(const float* x, __nv_bfloat16* out, const float* gamma, const float* beta, int rows, int W,
                          long long row_stride, const int* row_idx, cudaStream_t st) {
  CC_REQUIRE(W % 128 == 0, "layernorm: width %d not a multiple of 128", W);
  if (rows == 0) return CC_OK;
  const int blocks = rows < 132 * 8 ? (rows + 7) / 8 : 132 * 4;
  return dispatch_n4(W, [&](auto n4) -> int {
    layernorm_bf16_kernel<decltype(n4)::value><<<blocks < 1 ? 1 : blocks, 256, 0, st>>>(x, out, gamma, beta, rows, W, row_stride, row_idx);
    CC_CHECK_CUDA(cudaGetLastError());
    return static_cast<int>(CC_OK);
  });
}

// ------------------------------------------------------------------------------------------------ text embedding
// x[b,t,:] = tok[ids[b,t],:] + pos[t,:]; eot_row[b] = b*L + argmax_t ids[b,t] (first maximum)
__global__ void text_embed_kernel(const int* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                                  float* __restrict__ x, int* __restrict__ eot_row, int B, int L, int W, int vocab) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int rows = B * L;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += gridDim.x * wpb) {
    const int t = row % L;
    int id = __ldg(ids + row);
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const float* tr = tok + static_cast<long long>(id) * W;
    const float* pr = pos + static_cast<long long>(t) * W;
    float* xr = x + static_cast<long long>(row) * W;
    for (int c = lane * 4; c < W; c += 128) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(tr + c));
      const float4 p = __ldg(reinterpret_cast<const float4*>(pr + c));
      *reinterpret_cast<float4*>(xr + c) = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
    }
    if (t == 0 && lane == 0) {
      int best = __ldg(ids + row), bi = 0;
      for (int j = 1; j < L; ++j) {
        const int v = __ldg(ids + row + j);
        if (v > best) { best = v; bi = j; }
      }
      eot_row[row / L] = row + bi;
    }
  }
}
int text_embed_launch(const int* ids, const float* tok, const float* pos, float* x, int* eot_row, int B, int L, int W,
                      int vocab, cudaStream_t st) {
  CC_REQUIRE(W % 4 == 0, "text_embed: bad width");
  const int rows = B * L;
  const int blocks = rows < 132 * 8 ? (rows + 7) / 8 : 132 * 4;
  text_embed_kernel<<<blocks < 1 ? 1 : blocks, 256, 0, st>>>(ids, tok, pos, x, eot_row, B, L, W, vocab);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ l2 normalise
__global__ void l2norm_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int D, long long out_stride,
                              float eps) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < rows; r += gridDim.x * wpb) {
    const float* x = in + static_cast<long long>(r) * D;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) s += x[c] * x[c];
    const float inv = 1.0f / (sqrtf(warp_sum(s)) + eps);
    float* o = out + static_cast<long long>(r) * out_stride;
    for (int c = lane; c < D; c += 32) o[c] = x[c] * inv;
  }
}
int l2norm_launch(const float* in, float* out, int rows, int D, long long out_stride, float eps, cudaStream_t st) {
  if (rows == 0) return CC_OK;
  const int blocks = (rows + 7) / 8;
  l2norm_kernel<<<blocks > 132 * 4 ? 132 * 4 : blocks, 256, 0, st>>>(in, out, rows, D, out_stride, eps);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ attention
// One CTA per (batch, head); K and V of the head live in shared memory ([Lp][72] bf16, 144-B pitch = conflict-free
// for both the 32-bit B-fragment reads of K and ldmatrix.trans on V); each warp owns 16-query blocks and runs an
// online-softmax (flash) loop over 16-key blocks with mma.sync m16n8k16 bf16 (fp32 accumulate).
// Serves the short sequences (several CTAs per SM hide the per-CTA chain); the long ones run on attention_tc.cu (wgmma).
static constexpr int kAttnPitch = 72;  // bf16 elements per smem row

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

static constexpr int kAttnWarps = 5;    // warps per CTA
static constexpr int kAttnSplitMax = 2; // CTAs per (image, head) for long sequences: each takes half of the 16-query blocks

template <bool CAUSAL>
__global__ void __launch_bounds__(32 * kAttnWarps) attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ ctx,
                                                        int L, int H) {
  extern __shared__ __align__(16) __nv_bfloat16 smem_attn[];
  const int W = H * 64;
  const int Lp = (L + 15) & ~15;
  __nv_bfloat16* Ks = smem_attn;
  __nv_bfloat16* Vs = smem_attn + static_cast<size_t>(Lp) * kAttnPitch;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * L * 3 * W + h * 64;

  // ---- stage K and V of this head (zero rows beyond L)
  for (int i = threadIdx.x; i < Lp * 8; i += blockDim.x) {
    const int t = i >> 3, ch = (i & 7) * 8;
    uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
    if (t < L) {
      kv = __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(t) * 3 * W + W + ch));
      vv = __ldg(reinterpret_cast<const uint4*>(base + static_cast<long long>(t) * 3 * W + 2 * W + ch));
    }
    *reinterpret_cast<uint4*>(Ks + t * kAttnPitch + ch) = kv;
    *reinterpret_cast<uint4*>(Vs + t * kAttnPitch + ch) = vv;
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const float kLog2e = 1.4426950408889634f;

  const int nqb = (L + 15) / 16, per = (nqb + gridDim.y - 1) / gridDim.y;
  const int qb_lo = blockIdx.y * per, qb_hi = (qb_lo + per < nqb) ? qb_lo + per : nqb;
  for (int qb = qb_lo + warp; qb < qb_hi; qb += kAttnWarps) {
    const int r0 = qb * 16 + g, r1 = r0 + 8;
    // Q fragments, pre-scaled by 1/sqrt(64) = 2^-3 (exact in bf16)
    uint32_t qa[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = (e & 1) ? r1 : r0;
        const int col = ks * 16 + ((e & 2) ? 8 : 0) + 2 * t4;
        uint32_t w = 0;
        if (row < L) w = __ldg(reinterpret_cast<const uint32_t*>(base + static_cast<long long>(row) * 3 * W + col));
        __nv_bfloat162 hh = *reinterpret_cast<__nv_bfloat162*>(&w);
        hh = __hmul2(hh, __floats2bfloat162_rn(0.125f, 0.125f));
        qa[ks][e] = *reinterpret_cast<uint32_t*>(&hh);
      }
    }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    float o[8][4];
#pragma unroll
    for (int d = 0; d < 8; ++d) o[d][0] = o[d][1] = o[d][2] = o[d][3] = 0.f;

    const int kb_end = CAUSAL ? ((qb * 16 + 15 < L - 1 ? qb * 16 + 15 : L - 1) / 16 + 1) : Lp / 16;
    for (int kb = 0; kb < kb_end; ++kb) {
      float s[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
        const __nv_bfloat16* kr = Ks + (kb * 16 + nt * 8 + g) * kAttnPitch + 2 * t4;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr + ks * 16);
          const uint32_t b1 = *reinterpret_cast<const uint32_t*>(kr + ks * 16 + 8);
          mma_bf16_16816(s[nt], qa[ks], b0, b1);
        }
      }
      // mask: padded keys, and (text tower) keys after the query
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = kb * 16 + nt * 8 + 2 * t4 + (e & 1);
          const int row = (e & 2) ? r1 : r0;
          if (key >= L || (CAUSAL && key > row)) s[nt][e] = -INFINITY;
        }
      float mx0 = fmaxf(fmaxf(s[0][0], s[0][1]), fmaxf(s[1][0], s[1][1]));
      float mx1 = fmaxf(fmaxf(s[0][2], s[0][3]), fmaxf(s[1][2], s[1][3]));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
      // rows that are pure padding (r >= L) see only finite zeros; every real row has key 0 unmasked -> mn finite
      const bool grew = (mn0 != m0) | (mn1 != m1);
      const float c0 = mn0 * kLog2e, c1 = mn1 * kLog2e;
      float p[2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        p[nt][0] = fast_exp2(fmaf(s[nt][0], kLog2e, -c0)); p[nt][1] = fast_exp2(fmaf(s[nt][1], kLog2e, -c0));
        p[nt][2] = fast_exp2(fmaf(s[nt][2], kLog2e, -c1)); p[nt][3] = fast_exp2(fmaf(s[nt][3], kLog2e, -c1));
      }
      if (__any_sync(0xffffffffu, grew)) {   // the running maximum moved for some row of this warp: rescale
        const float a0 = fast_exp2((m0 - mn0) * kLog2e), a1 = fast_exp2((m1 - mn1) * kLog2e);
        l0 *= a0; l1 *= a1;
#pragma unroll
        for (int d = 0; d < 8; ++d) { o[d][0] *= a0; o[d][1] *= a0; o[d][2] *= a1; o[d][3] *= a1; }
      }
      m0 = mn0; m1 = mn1;
      l0 += p[0][0] + p[0][1] + p[1][0] + p[1][1];
      l1 += p[0][2] + p[0][3] + p[1][2] + p[1][3];
      const uint32_t pa[4] = {pack2(p[0][0], p[0][1]), pack2(p[0][2], p[0][3]), pack2(p[1][0], p[1][1]), pack2(p[1][2], p[1][3])};
      // P.V: B fragments of V via ldmatrix.trans (two 8-wide d tiles per instruction)
#pragma unroll
      for (int dp = 0; dp < 4; ++dp) {
        const int lrow = lane & 15, dsel = lane >> 4;
        const uint32_t addr = static_cast<uint32_t>(__cvta_generic_to_shared(Vs + (kb * 16 + lrow) * kAttnPitch + (2 * dp + dsel) * 8));
        uint32_t v0, v1, v2, v3;
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                     : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "r"(addr));
        mma_bf16_16816(o[2 * dp], pa, v0, v1);
        mma_bf16_16816(o[2 * dp + 1], pa, v2, v3);
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    __nv_bfloat16* out0 = ctx + (static_cast<long long>(b) * L + r0) * W + h * 64 + 2 * t4;
    __nv_bfloat16* out1 = ctx + (static_cast<long long>(b) * L + r1) * W + h * 64 + 2 * t4;
#pragma unroll
    for (int d = 0; d < 8; ++d) {
      if (r0 < L) *reinterpret_cast<uint32_t*>(out0 + d * 8) = pack2(o[d][0] * i0, o[d][1] * i0);
      if (r1 < L) *reinterpret_cast<uint32_t*>(out1 + d * 8) = pack2(o[d][2] * i1, o[d][3] * i1);
    }
  }
}

int attention_launch(const __nv_bfloat16* qkv, __nv_bfloat16* ctx, int B, int L, int H, int causal, cudaStream_t st) {
  if (B == 0) return CC_OK;
  const int Lp = (L + 15) & ~15;
  const int smem = 2 * Lp * kAttnPitch * 2;
  CC_REQUIRE(smem <= 200 * 1024, "attention: sequence length %d too long for the single-CTA kernel", L);
  static bool attr_set = false;
  if (!attr_set) {
    CC_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CC_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const dim3 grid(B * H, ((L + 15) / 16 > 2 * kAttnWarps) ? kAttnSplitMax : 1);   // short sequences: one CTA stages K/V once
  if (causal) attention_kernel<true><<<grid, 32 * kAttnWarps, smem, st>>>(qkv, ctx, L, H);
  else attention_kernel<false><<<grid, 32 * kAttnWarps, smem, st>>>(qkv, ctx, L, H);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

// ------------------------------------------------------------------------------------------------ search
// scores[q, n] = <index[n,:], query[q,:]>  (ObjectFinder.search, models/objects.py:373). HBM-bound: each index row
// is read once (float4) by one warp and dotted with up to 8 queries held in registers/smem.
__global__ void search_scores_kernel(const float* __restrict__ index, const float* __restrict__ q, float* __restrict__ scores,
                                     int N, int D, int Q) {
  extern __shared__ float sq[];  // [Q][D]
  for (int i = threadIdx.x; i < Q * D; i += blockDim.x) sq[i] = q[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int n = blockIdx.x * wpb + (threadIdx.x >> 5); n < N; n += gridDim.x * wpb) {
    const float* row = index + static_cast<long long>(n) * D;
    for (int q0 = 0; q0 < Q; q0 += 4) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int c = lane; c < D; c += 32) {
        const float v = __ldg(row + c);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (q0 + j < Q) acc[j] = fmaf(v, sq[(q0 + j) * D + c], acc[j]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float s = warp_sum(acc[j]);
        if (lane == 0 && q0 + j < Q) scores[static_cast<long long>(q0 + j) * N + n] = s;
      }
    }
  }
}
int search_scores_launch(const float* index, const float* q, float* scores, int N, int D, int Q, cudaStream_t st) {
  if (N == 0 || Q == 0) return CC_OK;
  const int smem = Q * D * 4;
  CC_REQUIRE(smem <= 48 * 1024, "search: %d queries x %d dims exceed the 48 KB query buffer", Q, D);
  int blocks = (N + 7) / 8;
  if (blocks > 132 * 8) blocks = 132 * 8;
  search_scores_kernel<<<blocks, 256, smem, st>>>(index, q, scores, N, D, Q);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}


// ------------------------------------------------------------------------------------------------ search, top-k on the device
// ObjectFinder.search (models/objects.py:356-390) keeps, per object id, the best-scoring image and returns the k best of
// those.  Here: (1) one warp per index row computes the dot product and folds it into its group's best with one 64-bit
// atomicMax on (orderable score << 32 | ~row) — a row of an earlier index wins an exact tie; (2) one CTA extracts the k best
// groups.  Only k (row, score) pairs cross PCIe instead of N scores.
__device__ __forceinline__ uint32_t f32_orderable(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float f32_from_orderable(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}
__global__ void search_group_best_kernel(const float* __restrict__ index, const float* __restrict__ q, const int* __restrict__ group,
                                         const uint8_t* __restrict__ mask, unsigned long long* __restrict__ best, int N, int D) {
  extern __shared__ float sq[];  // [D]
  for (int i = threadIdx.x; i < D; i += blockDim.x) sq[i] = q[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int n = blockIdx.x * wpb + (threadIdx.x >> 5); n < N; n += gridDim.x * wpb) {
    if (mask && !mask[n]) continue;
    const float* row = index + static_cast<long long>(n) * D;
    float acc = 0.f;
    for (int c = lane; c < D; c += 32) acc = fmaf(__ldg(row + c), sq[c], acc);     // same summation order as search_scores_kernel
    const float s = warp_sum(acc);
    if (lane == 0)
      atomicMax(best + group[n], (static_cast<unsigned long long>(f32_orderable(s)) << 32) | (0xFFFFFFFFu - static_cast<uint32_t>(n)));
  }
}
__global__ void __launch_bounds__(1024) search_topk_kernel(unsigned long long* __restrict__ best, int G, int k, int* __restrict__ out_rows,
                                                           float* __restrict__ out_scores) {
  __shared__ unsigned long long s_key[32];
  __shared__ int s_idx[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = 0; r < k; ++r) {
    unsigned long long bk = 0;
    int bi = -1;
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
      const unsigned long long v = best[g];
      if (v > bk) { bk = v; bi = g; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ok = __shfl_xor_sync(0xFFFFFFFFu, bk, o);
      const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
      if (ok > bk) { bk = ok; bi = oi; }
    }
    if (lane == 0) { s_key[warp] = bk; s_idx[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      bk = lane < (blockDim.x >> 5) ? s_key[lane] : 0ull;
      bi = lane < (blockDim.x >> 5) ? s_idx[lane] : -1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long ok = __shfl_xor_sync(0xFFFFFFFFu, bk, o);
        const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
        if (ok > bk) { bk = ok; bi = oi; }
      }
      if (lane == 0) {
        if (bi >= 0) {
          out_rows[r] = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(bk & 0xFFFFFFFFull));
          out_scores[r] = f32_from_orderable(static_cast<uint32_t>(bk >> 32));
          best[bi] = 0ull;                       // taken
        } else {
          out_rows[r] = -1;                      // fewer than k groups matched
          out_scores[r] = 0.f;
        }
      }
    }
    __syncthreads();
  }
}
int search_topk_launch(const float* index, const float* q, const int* group, const uint8_t* mask, unsigned long long* best, int N, int D,
                       int G, int k, int* out_rows, float* out_scores, cudaStream_t st) {
  CC_REQUIRE(D * 4 <= 48 * 1024, "search: %d dims exceed the 48 KB query buffer", D);
  CC_CHECK_CUDA(cudaMemsetAsync(best, 0, static_cast<size_t>(G > 0 ? G : 1) * sizeof(unsigned long long), st));
  if (N > 0) {
    int blocks = (N + 7) / 8;
    if (blocks > 132 * 8) blocks = 132 * 8;
    search_group_best_kernel<<<blocks, 256, D * 4, st>>>(index, q, group, mask, best, N, D);
    CC_CHECK_CUDA(cudaGetLastError());
  }
  search_topk_kernel<<<1, 1024, 0, st>>>(best, G, k, out_rows, out_scores);
  CC_CHECK_CUDA(cudaGetLastError());
  return CC_OK;
}

}  // namespace cc
