// Implicit-GEMM conv / linear on Hopper warpgroup MMA (sm_90a). See conv_gemm.cuh for what it replaces in the reference.
//
// GEMM view: M = output pixels (N*H*W), N = Cout, K = kh*kw*Cin.
//   * CTA tile: 128 pixels x BN channels (BN in {16, 32, 64, 128}); the 128 pixels are a TW x TH x TN box of the NHWC
//     output (TW*TH*TN = 128, chosen per layer so 20x20/40x40 maps tile without waste).
//   * K loop: for each filter tap (r,s) and each BK-channel chunk, ONE TMA box load of the input shifted by
//     the tap offset (TMA zero-fills out-of-bounds = conv padding) + one TMA box of the weights (or, when the weights of
//     the layer fit, all of them once per CTA: "resident" weights).
//     stride 2 uses a 5-D "pixel pair" view (dims: 2*C, W/2, 2, H/2, N) so every tap is again a dense box.
//   * smem tiles are K-major, 128/64/32-byte swizzled (BK = 64/32/16 channels) exactly as TMA writes them;
//     wgmma.mma_async (M=64, N=BN, K=16) reads them through shared-memory descriptors, accumulators in registers.
//   * warpgroup roles: wg0 = TMA producer (one thread), wg1 / wg2 = consumers, each owning 64 rows of the tile:
//     wgmma mainloop -> fp32 accumulators to smem -> thread pair == output row: bias -> SiLU/GELU -> (+residual) ->
//     bf16/fp32 in place -> coalesced 16-B stores.
//   * persistent: grid = min(tiles, SMs), static round-robin tile schedule.
#include "conv_gemm.cuh"
#include "cc_common.h"
#include "cc_ptx.cuh"
#include <math.h>
#include <stdlib.h>
#include <string.h>

namespace cc {

static constexpr int kConsumers = 2;                       // consumer warpgroups (64 rows each)
static constexpr int kThreads = 128 * (1 + kConsumers);     // wg0 producer + consumers
static constexpr int kEpiThreads = 128 * kConsumers;
static constexpr int kTileM = 128;
static constexpr int kMaxBN = 128;
static constexpr int kMaxSmem = 232448;  // 227 KB

__device__ __forceinline__ float tanh_approx(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(x));
  return t;
}

// Epilogue activations.  tanh.approx / ex2.approx / rcp.approx all run on the multi-function unit, so an activation that
// needs two of them (ex2 + rcp) costs twice the MUFU time of the tanh form:
//   ACT_SILU       : x*sigmoid(x) = h + h*tanh(h), h = x/2 : ONE MUFU (tanh.approx.f32, |abs err| <= 2^-11 on tanh, i.e.
//                    <= |x| * 2.4e-4 on the result, below the bf16 rounding of the stored value for x > -2)
//   ACT_SILU_EXACT : x / (1 + 2^(-x log2 e)) with ex2.approx + rcp.approx (two MUFU, ~1e-7 relative)
//   ACT_GELU_TANH  : 0.5x(1+tanh(sqrt(2/pi)(x+0.044715x^3)))  (models/objects.py:125 gelu()), one MUFU
template <int ACT>
__device__ __forceinline__ float act_apply(float x) {
  if (ACT == ACT_SILU) {
    const float h = 0.5f * x;
    return fmaf(h, tanh_approx(h), h);
  } else if (ACT == ACT_SILU_EXACT) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fminf(x * -1.4426950408889634f, 126.0f)));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return x * r;
  } else if (ACT == ACT_GELU_TANH) {
    const float u = 0.7978845608028654f * fmaf(0.044715f * x * x, x, x);
    const float h = 0.5f * x;
    return fmaf(h, tanh_approx(u), h);
  }
  return x;
}

// x / d for x < 2^31 with the host-computed (mul, shift) of fast_div(): (umulhi(mul, x) + x) >> shift
__device__ __forceinline__ int fdiv(int x, const uint32_t fd[2]) {
  return static_cast<int>((__umulhi(fd[0], static_cast<uint32_t>(x)) + static_cast<uint32_t>(x)) >> fd[1]);
}
// tile -> n block, tile origin
struct TileXY { int nb, w0, h0, n0; };
__device__ __forceinline__ TileXY tile_origin(const GemmParams& p, int tile) {
  TileXY t;
  const int m = fdiv(tile, p.fd_nb);
  t.nb = tile - m * p.n_blocks;
  const int mh = fdiv(m, p.fd_tw);                 // m / tiles_w
  t.w0 = (m - mh * p.tiles_w) << p.lTW;
  const int n = fdiv(m, p.fd_twh);                 // m / (tiles_w * tiles_h)
  t.h0 = (mh - n * p.tiles_h) << p.lTH;
  t.n0 = n << p.lTN;
  return t;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// One k-block (BK channels = KPB steps of K = 16) of this warpgroup's 64 x BN accumulator.
template <int BN>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint64_t adesc, uint64_t bdesc, int kpb, bool first) {
  Wgmma<BN>::mma(acc, adesc, bdesc, first ? 0u : 1u);
  for (int k = 1; k < kpb; ++k) Wgmma<BN>::mma(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
}

template <int ACT, bool F32, int BN>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_kernel(const __grid_constant__ GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment for the 128B-swizzled tiles
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  const int wg = threadIdx.x >> 7;
  const uint32_t row_bytes = p.BK * 2;
  const uint32_t a_bytes = kTileM * row_bytes;
  const uint32_t b_bytes = BN * row_bytes;
  const int S = p.stages;
  constexpr int es = F32 ? 4 : 2;
  constexpr uint32_t pitch = BN * 4 + 16;                 // fp32 accumulator row in the staging buffer (+16 B: bank spread)
  const int num_kb = p.num_taps * p.chunks_per_tap;

  uint8_t* sA = smem;
  uint8_t* sB = sA + S * a_bytes;
  // resident-B mode: sB holds ALL k-blocks of the weights (loaded once); the ring then carries A only
  uint8_t* sStage = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sB + (p.b_res ? num_kb : S) * b_bytes) + 15) & ~uintptr_t(15));
  float* sBias = reinterpret_cast<float*>(sStage + kTileM * pitch);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sBias + p.cout);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + S;
  uint64_t* bres_bar = bars + 2 * S;

  if (p.trace && blockIdx.x == 0 && threadIdx.x == 0) p.trace[0] = globaltimer_ns();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumers);   // one arrival per consumer warpgroup
    }
    mbar_init(bres_bar, 1);
    fence_mbar_init();
  }
  if (wg > 0) {  // bias -> smem once per CTA (epilogue reads it as broadcast LDS.128)
    for (int i = threadIdx.x - 128; i < p.cout; i += kEpiThreads) sBias[i] = p.bias ? __ldg(p.bias + i) : 0.f;
  }
  __syncthreads();
  // PDL: let the next kernel start its prologue as our CTAs retire; everything that only touches WEIGHTS (bias above,
  // resident weight tiles below) runs before griddepcontrol.wait, i.e. overlaps the previous kernel's tail.
  // Activations of the previous layer are read only by the TMA producer (A operand) and the epilogue (residual):
  // both execute pdl_wait() first.
  pdl_trigger();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // ===================== TMA producer =====================
      int stage = 0;
      uint32_t phase = 0;
      if (p.b_res) {   // weights are not produced by the previous kernel: issued BEFORE the grid dependency wait
        mbar_arrive_expect_tx(bres_bar, num_kb * b_bytes);
        for (int kb = 0; kb < num_kb; ++kb) tma_load_2d(sB + kb * b_bytes, &p.tmB, bres_bar, kb * p.BK, 0);
      }
      pdl_wait();
      if (p.trace && blockIdx.x == 0) p.trace[1] = globaltimer_ns();
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const TileXY tx = tile_origin(p, tile);
        int kb = 0;
        for (int t = 0; t < p.num_taps; ++t) {
          const int c_base = p.tap[t][0];
          const int c1 = tx.w0 + p.tap[t][1];
          const int c2 = p.s2 ? p.tap[t][2] : tx.h0 + p.tap[t][2];
          const int c3 = p.s2 ? tx.h0 + p.tap[t][3] : tx.n0;
          const int c4 = p.s2 ? tx.n0 : 0;
          for (int ch = 0; ch < p.chunks_per_tap; ++ch, ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], p.b_res ? a_bytes : a_bytes + b_bytes);
            tma_load_5d(sA + stage * a_bytes, &p.tmA, &full_bar[stage], c_base + ch * p.BK, c1, c2, c3, c4);
            if (!p.b_res) tma_load_2d(sB + stage * b_bytes, &p.tmB, &full_bar[stage], kb * p.BK, tx.nb * BN);
            if (++stage == S) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ===================== consumers: warpgroup c owns rows [64 c, 64 c + 64) of every tile =====================
    const int c = wg - 1;
    const int et = static_cast<int>(threadIdx.x) - 128;      // 0 .. 255 over both consumers
    const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
    const int kpb = p.BK >> 4;
    const uint64_t dconst = gmma_desc_const(row_bytes, 8u * row_bytes);
    const uint32_t sA16 = ((smem_u32(sA) & 0x3FFFF) >> 4) + ((c * 64 * row_bytes) >> 4), sB16 = (smem_u32(sB) & 0x3FFFF) >> 4;
    const uint32_t a16 = a_bytes >> 4, b16 = b_bytes >> 4;
    const uint32_t stg32 = smem_u32(sStage), sbias32 = smem_u32(sBias);
    const int TWm = (1 << p.lTW) - 1, THm = (1 << p.lTH) - 1;
    // register phase: thread pair == output row, the pair's halves take columns [0, BN/2) and [BN/2, BN).  A bf16 result is
    // written back over the fp32 accumulators it was computed from; the second half's results go after the first half's
    // fp32 values (byte BN*2 on), so neither thread overwrites values the other has yet to read.
    // (BN = 16 is one 16-column chunk: the first thread of the pair converts it alone)
    constexpr bool kSplit = BN >= 32;
    constexpr int kHalfCols = kSplit ? BN / 2 : BN;
    const int row = et >> 1, half = et & 1;
    const uint32_t out_off = F32 ? 0u : static_cast<uint32_t>(half) * BN * 2;    // bf16: where this half's fp32 columns start
    int stage = 0;
    uint32_t phase = 0;
    bool first_tile = true;
    if (p.b_res) mbar_wait(bres_bar, 0);
    pdl_wait();   // residual reads below depend on the previous kernel's output
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const TileXY tx = tile_origin(p, tile);
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (first_tile && kb == 0 && p.trace && blockIdx.x == 0 && et == 0) p.trace[3] = globaltimer_ns();
        wgmma_fence_acc(acc);
        wgmma_fence();
        mma_kblock<BN>(acc, dconst | (sA16 + stage * a16), dconst | (sB16 + (p.b_res ? kb : stage) * b16), kpb, kb == 0);
        wgmma_commit();
        wgmma_fence_acc(acc);
        wgmma_wait<1>();       // the previous k-block's MMAs are done: release its stage
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      if (first_tile && p.trace && blockIdx.x == 0 && et == 0) p.trace[5] = globaltimer_ns();
      first_tile = false;

      // ---- accumulators -> staging (fp32 rows of `pitch` bytes)
      named_bar_sync(1, kEpiThreads);     // the previous tile's copy-out has read the staging buffer
      {
        const int r0 = c * 64 + wq * 16 + (lane >> 2);
        const uint32_t base = stg32 + r0 * pitch + (lane & 3) * 8;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(base + i * 32), "f"(acc[4 * i]), "f"(acc[4 * i + 1]) : "memory");
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(base + 8 * pitch + i * 32), "f"(acc[4 * i + 2]), "f"(acc[4 * i + 3]) : "memory");
        }
      }
      named_bar_sync(1, kEpiThreads);

      // ---- register phase: this thread's pixel, columns [half BN/2, (half+1) BN/2)
      const int nb = tx.nb, w0 = tx.w0, h0 = tx.h0, n0 = tx.n0;
      const int pw = w0 + (row & TWm), ph = h0 + ((row >> p.lTW) & THm), pn = n0 + (row >> (p.lTW + p.lTH));
      const bool pvalid = (pw < p.W) && (ph < p.H) && (pn < p.N);
      const long long ppix = static_cast<long long>(pn) * p.out_ns + ph * p.W + pw;
      // pre-activation addend from a half-resolution fp32 map (nearest x2 upsample by addressing): this pixel's source row
      const float* const pre_row = (p.pre != nullptr && pvalid)
          ? p.pre + ((static_cast<long long>(pn) * p.pre_h + (ph >> 1)) * p.pre_w + (pw >> 1)) * p.cout : nullptr;
      const uint32_t srow = stg32 + row * pitch;
#pragma unroll 1
      for (int cc = half * kHalfCols; cc < (kSplit || half == 0 ? (half + 1) * kHalfCols : 0); cc += 16) {
        const int gcol = nb * BN + cc;   // global output channel of column cc
        float f[16];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 vu = lds_u4(srow + (cc + 4 * j) * 4);
          const float4 v = make_float4(__uint_as_float(vu.x), __uint_as_float(vu.y), __uint_as_float(vu.z), __uint_as_float(vu.w));
          float4 b4 = lds_f4(sbias32 + (gcol + 4 * j) * 4);
          if (pre_row != nullptr) {
            const float4 q4 = __ldg(reinterpret_cast<const float4*>(pre_row + gcol) + j);
            b4.x += q4.x; b4.y += q4.y; b4.z += q4.z; b4.w += q4.w;
          }
          f[4 * j] = act_apply<ACT>(v.x + b4.x);
          f[4 * j + 1] = act_apply<ACT>(v.y + b4.y);
          f[4 * j + 2] = act_apply<ACT>(v.z + b4.z);
          f[4 * j + 3] = act_apply<ACT>(v.w + b4.w);
        }
        if (p.res != nullptr && pvalid) {
          if (F32) {
            const float4* r4 = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.res) + ppix * p.res_cs + p.res_co + gcol);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 r = __ldg(r4 + j);
              f[4 * j + 0] += r.x; f[4 * j + 1] += r.y; f[4 * j + 2] += r.z; f[4 * j + 3] += r.w;
            }
          } else {
            const uint4* r4 = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + ppix * p.res_cs + p.res_co + gcol);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              const uint4 r = __ldg(r4 + j);
              const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                // bf16 -> fp32 is a 16-bit shift
                f[8 * j + 2 * q + 0] += __uint_as_float(rr[q] << 16);
                f[8 * j + 2 * q + 1] += __uint_as_float(rr[q] & 0xFFFF0000u);
              }
            }
          }
        }
        // in place: fp32 results over their own accumulators; bf16 results of column cc at out_off + 2 (cc - half BN/2), which
        // only covers fp32 columns of this thread that it has already read
        const uint32_t dst = F32 ? srow + cc * 4 : srow + out_off + (cc - half * kHalfCols) * 2;
        if (F32) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            sts_u4(dst + 16 * j, __float_as_uint(f[4 * j]), __float_as_uint(f[4 * j + 1]), __float_as_uint(f[4 * j + 2]), __float_as_uint(f[4 * j + 3]));
        } else {
#pragma unroll
          for (int j = 0; j < 2; ++j)
            sts_u4(dst + 16 * j, pack_bf16x2(f[8 * j], f[8 * j + 1]), pack_bf16x2(f[8 * j + 2], f[8 * j + 3]),
                   pack_bf16x2(f[8 * j + 4], f[8 * j + 5]), pack_bf16x2(f[8 * j + 6], f[8 * j + 7]));
        }
      }
      named_bar_sync(1, kEpiThreads);    // results staged

      // ---- coalesced copy-out, division free: a set of `1 << lg` (power of two >= chunks per row) threads owns one row
      constexpr int cpr = (BN * es) >> 4;  // 16-B chunks per row (2..32)
      constexpr int hcpr = cpr / 2;        // chunks of one half
      constexpr int lg = cpr > 16 ? 5 : (cpr > 8 ? 4 : (cpr > 4 ? 3 : (cpr > 2 ? 2 : 1)));
      const int chk = et & ((1 << lg) - 1);
      constexpr int rstep = kEpiThreads >> lg;
      if (chk < cpr) {
        // bf16: the second half's results start at byte 2 BN of the staging row (see out_off)
        const uint32_t soff = (F32 || !kSplit) ? chk * 16 : (chk < hcpr ? chk * 16 : BN * 2 + (chk - hcpr) * 16);
        uint8_t* gbase = reinterpret_cast<uint8_t*>(p.out) + static_cast<size_t>(p.out_co + nb * BN) * es + chk * 16;
        for (int r = et >> lg; r < kTileM; r += rstep) {
          const int qw = w0 + (r & TWm), qh = h0 + ((r >> p.lTW) & THm), qn = n0 + (r >> (p.lTW + p.lTH));
          if (qw < p.W && qh < p.H && qn < p.N) {
            const long long pix = static_cast<long long>(qn) * p.out_ns + qh * p.W + qw;
            const uint4 val = lds_u4(stg32 + r * pitch + soff);
            *reinterpret_cast<uint4*>(gbase + pix * p.out_cs * es) = val;
          }
        }
      }
    }
    if (p.trace != nullptr && blockIdx.x == 0 && et == 0) p.trace[6] = globaltimer_ns();   // last epilogue of CTA 0 done
  }
  if (p.trace && threadIdx.x == 0) {
    atomicMax(p.trace + 2, globaltimer_ns());
    if (blockIdx.x == 0) p.trace[7] = globaltimer_ns();
  }
}

// ------------------------------------------------------------------------------------------------ host

bool conv_gemm_supported(const ConvDesc& d) {
  if (d.Cin % 16 != 0 || d.Cout % 16 != 0) return false;
  if (!(d.k == 1 || d.k == 3)) return false;
  if (!(d.stride == 1 || d.stride == 2)) return false;
  if (d.stride == 2 && (d.k != 3 || (d.Hin & 1) || (d.Win & 1))) return false;
  if (d.in_co % 8 != 0 || d.in_cs % 8 != 0) return false;
  return true;
}

int conv_gemm_build(const ConvDesc& d, int num_sms, GemmLaunch* L) {
  CC_REQUIRE(conv_gemm_supported(d), "conv_gemm: unsupported shape Cin=%d Cout=%d k=%d s=%d Hin=%d Win=%d", d.Cin, d.Cout,
             d.k, d.stride, d.Hin, d.Win);
  PFN_encodeTiled enc = get_encode_tiled();
  CC_REQUIRE(enc != nullptr, "conv_gemm: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  const int es = d.out_f32 ? 4 : 2;
  CC_REQUIRE((d.out_cs * es) % 16 == 0 && (d.out_co * es) % 16 == 0, "conv_gemm: output slice not 16-B aligned");
  if (d.res) CC_REQUIRE((d.res_cs * es) % 16 == 0 && (d.res_co * es) % 16 == 0, "conv_gemm: residual slice not 16-B aligned");

  GemmParams& p = L->p;
  memset(&p, 0, sizeof(p));
  const int Hout = d.stride == 2 ? d.Hin / 2 : d.Hin;
  const int Wout = d.stride == 2 ? d.Win / 2 : d.Win;
  p.W = Wout; p.H = Hout; p.N = d.N;

  // ---- K blocking
  p.BK = (d.Cin % 64 == 0) ? 64 : (d.Cin % 32 == 0 ? 32 : 16);
  p.num_taps = d.k * d.k;
  p.chunks_per_tap = d.Cin / p.BK;
  // ---- N blocking: a power of two in [16, 128] that divides Cout (the kernel is compiled for those four widths); an
  // override is taken as an upper bound
  const long long mt = (static_cast<long long>(d.N) * Hout * Wout + 127) / 128;
  const int maxbn = d.bn_override > 0 && d.bn_override < kMaxBN ? d.bn_override : kMaxBN;
  int BN = 16;
  while (BN * 2 <= maxbn && d.Cout % (BN * 2) == 0) BN *= 2;
  // if the machine would be under-filled, halve the N tile (more, smaller tiles)
  if (d.bn_override == 0)
    while (BN > 64 && mt * (d.Cout / BN) < num_sms) BN /= 2;
  CC_REQUIRE(BN >= 16 && BN <= kMaxBN && d.Cout % BN == 0, "conv_gemm: bad BN=%d for Cout=%d", BN, d.Cout);
  p.BN = BN;
  p.n_blocks = d.Cout / BN;
  p.cout = d.Cout;

  // ---- M tile box: maximise useful pixels per 128-row tile
  int best[3] = {7, 0, 0};
  double best_eff = -1;
  for (int lw = 0; lw <= 7; ++lw)
    for (int lh = 0; lw + lh <= 7; ++lh) {
      const int ln = 7 - lw - lh;
      const int tw = 1 << lw, th = 1 << lh, tn = 1 << ln;
      const double cover = double((Wout + tw - 1) / tw * tw) * ((Hout + th - 1) / th * th) * ((d.N + tn - 1) / tn * tn);
      double eff = double(Wout) * Hout * d.N / cover + 1e-6 * lw - 1e-7 * ln;  // ties: wider rows, fewer images
      if (eff > best_eff) { best_eff = eff; best[0] = lw; best[1] = lh; best[2] = ln; }
    }
  p.lTW = best[0]; p.lTH = best[1]; p.lTN = best[2];
  const int TW = 1 << p.lTW, TH = 1 << p.lTH, TN = 1 << p.lTN;
  p.tiles_w = (Wout + TW - 1) / TW;
  p.tiles_h = (Hout + TH - 1) / TH;
  p.tiles_n = (d.N + TN - 1) / TN;
  p.num_tiles = p.tiles_w * p.tiles_h * p.tiles_n * p.n_blocks;
  p.s2 = d.stride == 2;

  // ---- taps
  const int pad = d.k / 2;
  for (int r = 0; r < d.k; ++r)
    for (int s = 0; s < d.k; ++s) {
      int* t = p.tap[r * d.k + s];
      if (!p.s2) {
        t[0] = 0; t[1] = s - pad; t[2] = r - pad; t[3] = 0;
      } else {
        // input col 2x+s-1: s=0 -> (pair x-1, odd), s=1 -> (pair x, even), s=2 -> (pair x, odd); same for rows
        const int wp = (s == 1) ? 0 : 1, dw = (s == 0) ? -1 : 0;
        const int hp = (r == 1) ? 0 : 1, dh = (r == 0) ? -1 : 0;
        t[0] = wp * d.in_cs; t[1] = dw; t[2] = hp; t[3] = dh;
      }
    }

  // ---- tensor maps
  const CUtensorMapSwizzle swz = p.BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                               : p.BK == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  {
    void* base = const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(d.in)) + size_t(d.in_co) * 2;
    CC_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "conv_gemm: input slice not 16-B aligned");
    cuuint64_t dims[5], strides[4];
    cuuint32_t box[5], estr[5] = {1, 1, 1, 1, 1};
    const cuuint64_t px = cuuint64_t(d.in_cs) * 2;  // bytes per pixel
    if (!p.s2) {
      dims[0] = d.Cin; dims[1] = d.Win; dims[2] = d.Hin; dims[3] = d.N; dims[4] = 1;
      strides[0] = px; strides[1] = px * d.Win; strides[2] = px * d.Win * d.Hin; strides[3] = px * d.Win * d.Hin * d.N;
      box[0] = p.BK; box[1] = TW; box[2] = TH; box[3] = TN; box[4] = 1;
    } else {
      dims[0] = d.in_cs + d.Cin; dims[1] = d.Win / 2; dims[2] = 2; dims[3] = d.Hin / 2; dims[4] = d.N;
      strides[0] = 2 * px; strides[1] = px * d.Win; strides[2] = 2 * px * d.Win; strides[3] = px * d.Win * d.Hin;
      box[0] = p.BK; box[1] = TW; box[2] = 1; box[3] = TH; box[4] = TN;
    }
    CUresult r = enc(&p.tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CC_REQUIRE(r == CUDA_SUCCESS, "conv_gemm: cuTensorMapEncodeTiled(A) failed: %d (dims %llu,%llu,%llu,%llu,%llu)", int(r),
               dims[0], dims[1], dims[2], dims[3], dims[4]);
  }
  {     // weights [Cout][Ktot] bf16, box = BK x BN
    const cuuint64_t Ktot = cuuint64_t(d.k) * d.k * d.Cin;
    cuuint64_t dims[2] = {Ktot, cuuint64_t(d.Cout)};
    cuuint64_t strides[1] = {Ktot * 2};
    cuuint32_t box[2] = {cuuint32_t(p.BK), cuuint32_t(BN)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d.w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CC_REQUIRE(r == CUDA_SUCCESS, "conv_gemm: cuTensorMapEncodeTiled(B) failed: %d", int(r));
  }

  // ---- epilogue
  p.out = d.out; p.out_cs = d.out_cs; p.out_co = d.out_co; p.out_f32 = d.out_f32;
  p.bias = d.bias; p.act = d.act;
  p.res = d.res; p.res_cs = d.res_cs; p.res_co = d.res_co;
  p.out_ns = d.out_ns > 0 ? d.out_ns : Hout * Wout;
  p.pre = d.pre; p.pre_h = d.pre_h; p.pre_w = d.pre_w;
  if (d.pre) CC_REQUIRE(d.pre_h * 2 == Hout && d.pre_w * 2 == Wout && d.Cout % 4 == 0, "conv_gemm: the pre-activation addend must be a half-resolution map of the output");
  {
    auto fast_div = [](uint32_t d, uint32_t fd[2]) {      // q = (umulhi(mul, x) + x) >> shift for x < 2^31
      uint32_t l = 0;
      while ((1ull << l) < d) ++l;
      fd[0] = static_cast<uint32_t>(((1ull << 32) * ((1ull << l) - d)) / d + 1);
      fd[1] = l;
    };
    fast_div(p.n_blocks, p.fd_nb);
    fast_div(p.tiles_w, p.fd_tw);
    fast_div(p.tiles_w * p.tiles_h, p.fd_twh);
  }

  // ---- smem budget -> pipeline depth.  Fixed part: alignment slack, the fp32 staging tile, bias, barriers.
  const int a_bytes = kTileM * p.BK * 2, b_bytes = BN * p.BK * 2;
  const int fixed = 1024 + kTileM * (BN * 4 + 16) + 16 + d.Cout * 4 + 8 * 20;
  const int num_kb = p.num_taps * p.chunks_per_tap;
  const int bres_bytes = b_bytes * num_kb;
  // resident weights (single N block) when they leave room for at least four activation stages: the ring then carries
  // A only and the weights cross the L2 once per CTA instead of once per tile
  p.b_res = (p.n_blocks == 1 && (kMaxSmem - fixed - bres_bytes) / a_bytes >= 4) ? 1 : 0;
  int S = p.b_res ? (kMaxSmem - fixed - bres_bytes) / a_bytes : (kMaxSmem - fixed) / (a_bytes + b_bytes);
  if (S > 8) S = 8;
  CC_REQUIRE(S >= 2, "conv_gemm: tile does not fit shared memory (BN=%d BK=%d)", BN, p.BK);
  CC_REQUIRE(S <= 8, "conv_gemm: too many stages");
  p.stages = S;
  L->smem_bytes = fixed + (p.b_res ? bres_bytes + S * a_bytes : S * (a_bytes + b_bytes));
  L->grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  L->flops = 2.0 * double(d.N) * Hout * Wout * d.Cout * d.k * d.k * d.Cin;
  L->bytes = double(d.N) * d.Hin * d.Win * d.Cin * 2 + double(d.N) * Hout * Wout * d.Cout * es * (d.res ? 2 : 1) +
             double(d.Cout) * d.k * d.k * d.Cin * 2;
  return CC_OK;
}

template <int ACT, bool F32, int BN>
static int launch_bn(const GemmLaunch& L, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    CC_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<ACT, F32, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(L.grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = L.smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CC_CHECK_CUDA(cudaLaunchKernelEx(&cfg, conv_gemm_kernel<ACT, F32, BN>, L.p));
  return CC_OK;
}

template <int ACT, bool F32>
static int launch_variant(const GemmLaunch& L, cudaStream_t stream) {
  switch (L.p.BN) {
    case 16: return launch_bn<ACT, F32, 16>(L, stream);
    case 32: return launch_bn<ACT, F32, 32>(L, stream);
    case 64: return launch_bn<ACT, F32, 64>(L, stream);
    case 128: return launch_bn<ACT, F32, 128>(L, stream);
  }
  set_error("conv_gemm: no kernel for BN=%d", L.p.BN);
  return CC_ERR_INVALID;
}

int conv_gemm_launch(const GemmLaunch& L, cudaStream_t stream) {
  const bool f32 = L.p.out_f32 != 0;
  static const int exact_env = getenv("CC_SILU_EXACT") ? atoi(getenv("CC_SILU_EXACT")) : 0;
  int act = L.p.act;
  if (act == ACT_SILU && exact_env) act = ACT_SILU_EXACT;
  switch (act) {
    case ACT_NONE: return f32 ? launch_variant<ACT_NONE, true>(L, stream) : launch_variant<ACT_NONE, false>(L, stream);
    case ACT_SILU: return f32 ? launch_variant<ACT_SILU, true>(L, stream) : launch_variant<ACT_SILU, false>(L, stream);
    case ACT_GELU_TANH:
      return f32 ? launch_variant<ACT_GELU_TANH, true>(L, stream) : launch_variant<ACT_GELU_TANH, false>(L, stream);
    case ACT_SILU_EXACT:
      return f32 ? launch_variant<ACT_SILU_EXACT, true>(L, stream) : launch_variant<ACT_SILU_EXACT, false>(L, stream);
  }
  set_error("conv_gemm: unknown activation %d", L.p.act);
  return CC_ERR_INVALID;
}

}  // namespace cc
