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
//   * warpgroup roles ("ping-pong"): wg0 = TMA producer (one thread), wg1 / wg2 = consumers that take the CTA's tiles
//     in turn, each owning a whole 128 x BN tile (two m64 wgmmas per k16).
//     An ordering barrier makes their mainloops alternate, so one warpgroup's epilogue (bias -> SiLU/GELU -> +residual
//     on the accumulator registers -> bf16/fp32 into its own swizzled staging tile -> TMA tensor store) runs while the
//     other one's MMAs keep the tensor cores busy.
//   * persistent: grid = min(tiles, SMs), static round-robin tile schedule.
#include "conv_gemm.cuh"
#include "cc_common.h"
#include "cc_ptx.cuh"
#include <math.h>
#include <string.h>
#include <type_traits>

namespace cc {

static constexpr int kConsumers = 2;                       // consumer warpgroups (whole tiles, alternating)
static constexpr int kThreads = 128 * (1 + kConsumers);     // wg0 producer + consumers
static constexpr int kEpiThreads = 128 * kConsumers;
static constexpr int kTileM = 128;
static constexpr int kMaxBN = 128;
static constexpr int kMaxSmem = 232448;  // 227 KB
static constexpr int kBarriers = 24;      // full[S <= 8], empty[S], resident weights, turn[2], residual[2]

// Output staging of one consumer warpgroup.  The 128 x BN tile is cut into column boxes of one swizzle span (<= 128 B)
// x 128 rows, each written with the span's XOR swizzle (conflict-free fragment stores) and stored by one TMA box.  fp32
// tiles of BN = 128 (the CLIP residual stream, the fp32-accurate mode) go out in two column passes of 32 KB so the operand
// ring keeps its depth.
__host__ __device__ constexpr int epi_box_bytes(int bn, int es) { return bn * es < 128 ? bn * es : 128; }
__host__ __device__ constexpr int epi_passes(int bn, int es) { return es == 4 && bn == 128 ? 2 : 1; }
__host__ __device__ constexpr int epi_stage_bytes(int bn, int es) { return kTileM * bn * es / epi_passes(bn, es); }

__device__ __forceinline__ float tanh_approx(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(x));
  return t;
}

// Epilogue activations, each ONE multi-function-unit op (tanh.approx.f32); x / (1 + exp(-x)) would take two (ex2 + rcp):
//   ACT_SILU       : x*sigmoid(x) = h + h*tanh(h), h = x/2 (|abs err| <= 2^-11 on tanh, i.e. <= |x| * 2.4e-4 on the
//                    result, below the bf16 rounding of the stored value for x > -2)
//   ACT_GELU_TANH  : 0.5x(1+tanh(sqrt(2/pi)(x+0.044715x^3)))  (models/objects.py:125 gelu())
// ACT_PRELU (the face embedder's conv -> BN -> PReLU, models/adaface.py:54,86) is applied in the epilogue itself: its bias
// is a [9][Cout] table indexed by the output pixel's border class, 3 * (top 0 / interior 1 / bottom 2) + (left 0 / interior 1
// / right 2), so that an affine map folded in front of a zero-padded 3x3 conv stays exact at the borders; then
// x > 0 ? x : slope[c] * x.
template <int ACT>
__device__ __forceinline__ float act_apply(float x) {
  if (ACT == ACT_SILU) {
    const float h = 0.5f * x;
    return fmaf(h, tanh_approx(h), h);
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

// One k-block (BK channels = KPB steps of K = 16) of a 128 x BN tile: rows [0, 64) into acc0, rows [64, 128) into acc1
// (`ahalf` = descriptor offset of row 64).  Each accumulator sees the same k order as a single m64 warpgroup would.
// KPB is a compile-time constant so the 2 KPB wgmmas go out as one batch: with a runtime trip count ptxas waits for each
// pair before issuing the next, and only one consumer is in its mainloop at a time to cover such gaps.
template <int BN, int KPB>
__device__ __forceinline__ void mma_kblock(float (&acc0)[BN / 2], float (&acc1)[BN / 2], uint64_t adesc, uint64_t bdesc,
                                           uint32_t ahalf, bool first) {
#pragma unroll
  for (int k = 0; k < KPB; ++k) {
    Wgmma<BN>::mma(acc0, adesc + 2 * k, bdesc + 2 * k, first && k == 0 ? 0u : 1u);
    Wgmma<BN>::mma(acc1, adesc + ahalf + 2 * k, bdesc + 2 * k, first && k == 0 ? 0u : 1u);
  }
}

// N2 > 0: the chained mode (conv_gemm_chain_build).  After a tile of n block p.ch_nb is in the staging (and stored, if
// p.ch_store1), its consumer runs the N2 x N2 1x1 conv over [staging run | partner box] with wgmma A read straight from the
// staging, then a second bias -> ACT2 -> bf16 / fp32 (F2) epilogue into the same region and a TMA store to tmO2.
template <int ACT, bool F32, int BN, int N2 = 0, int ACT2 = ACT_NONE, bool F2 = false>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_kernel(const __grid_constant__ GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment for the 128B-swizzled tiles
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  constexpr int es = F32 ? 4 : 2;
  constexpr int kBoxBytes = epi_box_bytes(BN, es);
  constexpr int kBoxCols = kBoxBytes / es;
  constexpr int kBoxTile = kTileM * kBoxBytes;                  // one column box in smem (a multiple of 4 KB)
  constexpr int kPasses = epi_passes(BN, es);
  constexpr int kPassCols = BN / kPasses;
  constexpr int kPassBoxes = kPassCols / kBoxCols;
  constexpr int kStageBytes = epi_stage_bytes(BN, es);
  constexpr uint32_t kSwz = kBoxBytes == 128 ? 0x70 : (kBoxBytes == 64 ? 0x30 : 0x10);   // 16-B chunk bits XORed by row
  constexpr bool CHAIN = N2 > 0;
  static_assert(!CHAIN || !F32, "a chained 1x1 reads a bf16 staging tile");
  constexpr int kW2Bytes = (N2 * N2 * 2 + 1023) & ~1023;     // the 1x1's weights, resident for the whole kernel
  // a chained launch takes no pre-activation addend, and one with a 128-channel tile no residual: next to 128 accumulator
  // registers their epilogue code would spill (conv_gemm_chain_build refuses them)
  constexpr bool kPre = !CHAIN, kRes = !(CHAIN && BN == 128);
  constexpr bool kPrelu = ACT == ACT_PRELU;
  static_assert(!kPrelu || (!F32 && !CHAIN), "ACT_PRELU writes bf16 and chains nothing");
  constexpr int kBiasRows = kPrelu ? 10 : 1;                  // ACT_PRELU: 9 border-class bias rows, then the slopes

  const int wg = threadIdx.x >> 7;
  const uint32_t row_bytes = p.BK * 2;
  const uint32_t a_bytes = kTileM * row_bytes;
  const uint32_t b_bytes = BN * row_bytes;
  const int S = p.stages;
  const int num_kb = p.num_taps * p.chunks_per_tap;

  const int region = CHAIN ? p.ch_stage : kStageBytes;      // one consumer's staging region
  uint8_t* sStage = smem;                                     // kConsumers x region, 1024-B aligned
  uint8_t* sW2 = sStage + kConsumers * region;
  uint8_t* sA = sW2 + kW2Bytes;
  uint8_t* sB = sA + S * a_bytes;
  // resident-B mode: sB holds ALL k-blocks of the weights (loaded once); the ring then carries A only
  float* sBias = reinterpret_cast<float*>(sB + (p.b_res ? num_kb : S) * b_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sBias + kBiasRows * p.cout + N2);   // chained: the 1x1's bias follows
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + S;
  uint64_t* bres_bar = bars + 2 * S;
  uint64_t* turn_bar = bars + 2 * S + 1;    // [c]: consumer c may start its next mainloop
  uint64_t* res_bar = bars + 2 * S + 3;     // [c]: residual tile of consumer c landed in its staging
  uint64_t* w2_bar = bars + 2 * S + 5;      // chained: the 1x1's weights landed
  uint64_t* par_bar = bars + 2 * S + 6;     // chained, [c]: partner box of consumer c landed

  if (p.trace && blockIdx.x == 0 && threadIdx.x == 0) p.trace[0] = globaltimer_ns();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    tma_prefetch_desc(&p.tmO);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 1);   // released by the one consumer warpgroup that read the stage
    }
    mbar_init(bres_bar, 1);
    for (int c = 0; c < kConsumers; ++c) {
      mbar_init(&turn_bar[c], 1);
      mbar_init(&res_bar[c], 1);
    }
    if constexpr (CHAIN) {
      mbar_init(w2_bar, 1);
      for (int c = 0; c < kConsumers; ++c) mbar_init(&par_bar[c], 1);
    }
    fence_mbar_init();
  }
  if (wg > 0) {  // bias -> smem once per CTA
    if constexpr (kPrelu) {
      for (int i = threadIdx.x - 128; i < 9 * p.cout; i += kEpiThreads) sBias[i] = __ldg(p.bias + i);
      for (int i = threadIdx.x - 128; i < p.cout; i += kEpiThreads) sBias[9 * p.cout + i] = __ldg(p.slope + i);
    } else {
      for (int i = threadIdx.x - 128; i < p.cout; i += kEpiThreads) sBias[i] = p.bias ? __ldg(p.bias + i) : 0.f;
    }
    if constexpr (CHAIN)
      for (int i = threadIdx.x - 128; i < N2; i += kEpiThreads) sBias[p.cout + i] = p.bias2 ? __ldg(p.bias2 + i) : 0.f;
  }
  __syncthreads();
  // PDL: let the next kernel start its prologue as our CTAs retire; everything that only touches WEIGHTS (bias above,
  // resident weight tiles below) runs before griddepcontrol.wait, i.e. overlaps the previous kernel's tail.
  // Activations of the previous layer are read only by the TMA producer (A operand) and the consumers (residual, pre
  // addend): both execute pdl_wait() first.
  pdl_trigger();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // ===================== TMA producer: every tile of the CTA, in order, into one ring =====================
      int stage = 0;
      uint32_t phase = 0;
      if (p.b_res) {   // weights are not produced by the previous kernel: issued BEFORE the grid dependency wait
        mbar_arrive_expect_tx(bres_bar, num_kb * b_bytes);
        for (int kb = 0; kb < num_kb; ++kb) tma_load_2d(sB + kb * b_bytes, &p.tmB, bres_bar, kb * p.BK, 0);
      }
      if constexpr (CHAIN) {   // the 1x1's weights: K blocks of ch_bk2 channels x N2 rows, as the standalone launch loads them
        mbar_arrive_expect_tx(w2_bar, N2 * N2 * 2);
        for (int kb = 0; kb < N2 / p.ch_bk2; ++kb) tma_load_2d(sW2 + kb * N2 * p.ch_bk2 * 2, &p.tmW2, w2_bar, kb * p.ch_bk2, 0);
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
    // ===================== consumers: warpgroup c owns the CTA's local tiles c, c + 2, c + 4, ... =====================
    const int c = wg - 1;
    const int t = threadIdx.x & 127;
    const bool lead = t == 0;
    const int lane = t & 31, wq = t >> 5;
    const uint64_t dconst = gmma_desc_const(row_bytes, 8u * row_bytes);
    const uint32_t sA16 = (smem_u32(sA) & 0x3FFFF) >> 4, sB16 = (smem_u32(sB) & 0x3FFFF) >> 4;
    const uint32_t a16 = a_bytes >> 4, b16 = b_bytes >> 4, ahalf = (64 * row_bytes) >> 4;
    const uint32_t stg = smem_u32(sStage + c * region), sbias32 = smem_u32(sBias);
    const int TWm = (1 << p.lTW) - 1, THm = (1 << p.lTH) - 1;
    // the residual of column pass `pass` of the tile at (nb, w0, h0, n0) -> this warpgroup's staging, on res_bar[c]
    auto load_res = [&](const TileXY& tx, int pass) {
      mbar_arrive_expect_tx(&res_bar[c], kStageBytes);
#pragma unroll
      for (int b = 0; b < kPassBoxes; ++b)
        tma_load_4d(stg + b * kBoxTile, &p.tmR, &res_bar[c], tx.nb * BN + pass * kPassCols + b * kBoxCols, tx.w0, tx.h0, tx.n0);
    };
    if (p.b_res) mbar_wait(bres_bar, 0);
    if constexpr (CHAIN) mbar_wait(w2_bar, 0);
    pdl_wait();   // residual / pre reads depend on the previous kernel's output
    // barrier phases follow from the local tile index j: this consumer's (j / 2)-th tile; consumer 0 runs the CTA's first
    // mainloop (j = 0) without waiting
    for (int j = c; blockIdx.x + j * gridDim.x < p.num_tiles; j += kConsumers) {
      const TileXY tx = tile_origin(p, blockIdx.x + j * gridDim.x);
      // prefetch the residual while the mainloop runs, once the previous tile's stores have read the staging
      if (kRes && p.res != nullptr && lead) {
        tma_store_wait_read<0>();
        load_res(tx, 0);
      }
      if (CHAIN && p.ch_part && lead) {   // (one n block) the partner box goes right after the staging tile
        tma_store_wait_read<0>();
        mbar_arrive_expect_tx(&par_bar[c], kBoxTile);
        tma_load_4d(stg + kStageBytes, &p.tmP, &par_bar[c], 0, tx.w0, tx.h0, tx.n0);
      }
      if (j > 0) mbar_wait(&turn_bar[c], ((j >> 1) + (c == 0)) & 1);

      float acc0[BN / 2], acc1[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
      // this tile's k-blocks follow those of the CTA's earlier tiles in the ring
      const int g0 = j * num_kb;
      int stage = g0 % S;
      uint32_t phase = (g0 / S) & 1;
      int prev = -1;
      auto mainloop = [&](auto kpb_c) {    // BK = 16 KPB
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          if (j == 0 && kb == 0 && p.trace && blockIdx.x == 0 && lead) p.trace[3] = globaltimer_ns();
          wgmma_fence_acc(acc0);
          wgmma_fence_acc(acc1);
          wgmma_fence();
          mma_kblock<BN, decltype(kpb_c)::value>(acc0, acc1, dconst | (sA16 + stage * a16),
                                                 dconst | (sB16 + (p.b_res ? kb : stage) * b16), ahalf, kb == 0);
          wgmma_commit();
          wgmma_fence_acc(acc0);
          wgmma_fence_acc(acc1);
          wgmma_wait<1>();       // the previous k-block's MMAs are done: release its stage
          if (prev >= 0 && lead) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      };
      if (p.BK == 64) mainloop(std::integral_constant<int, 4>{});
      else if (p.BK == 32) mainloop(std::integral_constant<int, 2>{});
      else mainloop(std::integral_constant<int, 1>{});
      if (lead) mbar_arrive(&turn_bar[c ^ 1]);   // every MMA of this tile is issued: the other consumer's mainloop may start
      wgmma_wait<0>();
      wgmma_fence_acc(acc0);
      wgmma_fence_acc(acc1);
      if (lead) mbar_arrive(&empty_bar[prev]);
      if (j == 0 && p.trace && blockIdx.x == 0 && lead) p.trace[5] = globaltimer_ns();

      // ---- epilogue on the accumulator fragments.  Thread t holds rows 64 m + 16 (t / 32) + (t % 32) / 4 + 8 r (m, r in
      // {0, 1}: fragment quarter q = 2 m + r) and columns 8 i + 2 (t % 4) + {0, 1}.
      const int nb = tx.nb;
      const uint32_t bias_t = sbias32 + (nb * BN + 2 * (lane & 3)) * 4;   // this thread's first bias pair
      // one column pass (a compile-time constant, so every accumulator index below is static and stays in registers)
      auto epilogue_pass = [&](auto pass_c) {
        constexpr int pass = decltype(pass_c)::value;
        if (kRes && p.res != nullptr) {  // the residual landed in the staging (loaded after the previous stores had read it)
          mbar_wait(&res_bar[c], ((j >> 1) * kPasses + pass) & 1);
        } else {
          if (lead) tma_store_wait_read<0>();   // the previous tile's stores have read the staging
          named_bar_sync(1 + c, 128);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int row = 64 * (q >> 1) + 16 * wq + (lane >> 2) + 8 * (q & 1);
          // pre-activation addend from a half-resolution fp32 map (nearest x2 upsample by addressing): this row's source
          const float* pre_row = nullptr;
          if (kPre && p.pre != nullptr) {
            const int pw = tx.w0 + (row & TWm), ph = tx.h0 + ((row >> p.lTW) & THm), pn = tx.n0 + (row >> (p.lTW + p.lTH));
            if ((pw < p.W) && (ph < p.H) && (pn < p.N))
              pre_row = p.pre + ((static_cast<long long>(pn) * p.pre_h + (ph >> 1)) * p.pre_w + (pw >> 1)) * p.cout + nb * BN;
          }
          // ACT_PRELU: this row's bias row (its border class) and the slopes
          uint32_t bias_q = bias_t;
          [[maybe_unused]] uint32_t slope_q = 0;
          if constexpr (kPrelu) {
            const int pw = tx.w0 + (row & TWm), ph = tx.h0 + ((row >> p.lTW) & THm);
            const int cls = 3 * (ph == 0 ? 0 : (ph == p.H - 1 ? 2 : 1)) + (pw == 0 ? 0 : (pw == p.W - 1 ? 2 : 1));
            bias_q = bias_t + cls * p.cout * 4;
            slope_q = bias_t + 9 * p.cout * 4;
          }
          // staging address of (row, column): the TMA box swizzle XORs the 16-B chunk index with bits of the row offset
          const uint32_t roff = static_cast<uint32_t>(row * kBoxBytes), rxor = (roff >> 3) & kSwz;
          const uint32_t rbase = stg + roff;
#pragma unroll
          for (int i = pass * kPassCols / 8; i < (pass + 1) * kPassCols / 8; ++i) {
            const int col = 8 * i + 2 * (lane & 3);
            const float2 bb = lds_f2(bias_q + 32 * i);
            const int pc = col - pass * kPassCols;
            float b0 = bb.x, b1 = bb.y;
            if (pre_row != nullptr) {
              const float2 pq = __ldg(reinterpret_cast<const float2*>(pre_row + col));
              b0 += pq.x; b1 += pq.y;
            }
            const int k = 4 * i + 2 * (q & 1);
            float f0 = act_apply<ACT>(((q >> 1) ? acc1[k] : acc0[k]) + b0);
            float f1 = act_apply<ACT>(((q >> 1) ? acc1[k + 1] : acc0[k + 1]) + b1);
            if constexpr (kPrelu) {
              const float2 sl = lds_f2(slope_q + 32 * i);
              f0 = f0 > 0.f ? f0 : sl.x * f0;
              f1 = f1 > 0.f ? f1 : sl.y * f1;
            }
            const uint32_t addr = rbase + (pc / kBoxCols) * kBoxTile + (((pc % kBoxCols) * es) ^ rxor);
            if (F32) {
              if (kRes && p.res != nullptr) {
                const float2 r = lds_f2(addr);
                f0 += r.x; f1 += r.y;
              }
              sts_f2(addr, f0, f1);
            } else {
              if (kRes && p.res != nullptr) {
                const uint32_t r = lds_u32(addr);   // bf16 -> fp32 is a 16-bit shift
                f0 += __uint_as_float(r << 16);
                f1 += __uint_as_float(r & 0xFFFF0000u);
              }
              sts_u32(addr, pack_bf16x2(f0, f1));
            }
          }
        }
        fence_proxy_async_smem();      // generic-proxy writes -> visible to the TMA store
        named_bar_sync(1 + c, 128);
        if (lead && (!CHAIN || p.ch_store1)) {
          // the box is clipped at the edges of the output slice [out_co, out_co + Cout) x W x H x N
#pragma unroll
          for (int b = 0; b < kPassBoxes; ++b)
            tma_store_4d(&p.tmO, stg + b * kBoxTile, nb * BN + pass * kPassCols + b * kBoxCols, tx.w0, tx.h0, tx.n0);
          tma_store_commit();
        }
        if (lead) {
          if (kRes && p.res != nullptr && pass + 1 < kPasses) {
            tma_store_wait_read<0>();
            load_res(tx, pass + 1);
          }
        }
      };
      epilogue_pass(std::integral_constant<int, 0>{});
      if constexpr (kPasses > 1) epilogue_pass(std::integral_constant<int, 1>{});
      if constexpr (CHAIN) {
        if (tx.nb == p.ch_nb) {
          // ---- the chained 1x1.  A operand: the staging boxes (K-major, swizzled as a ring stage of BK = kBoxCols), then the
          // partner box; k16 step k reads input channel 16 k of the 1x1 as the standalone launch does, with its instruction
          // N (= N2) and its weight blocks, so each accumulator sees the same sequence of MMAs
          constexpr int es2 = F2 ? 4 : 2;
          constexpr int kBox2 = epi_box_bytes(N2, es2), kBoxCols2 = kBox2 / es2, kBoxTile2 = kTileM * kBox2;
          constexpr uint32_t kSwz2 = kBox2 == 128 ? 0x70 : (kBox2 == 64 ? 0x30 : 0x10);
          if (p.ch_part) mbar_wait(&par_bar[c], (j >> 1) & 1);
          // every value below is pinned after the mainloop (the empty asm), so that none is hoisted out of the tile loop and
          // kept live next to the mainloop's accumulators
          uint32_t stg_c = stg, bk2 = p.ch_bk2, k0 = p.ch_k0, part = p.ch_part;
          asm volatile("" : "+r"(stg_c), "+r"(bk2), "+r"(k0), "+r"(part));
          const uint64_t adc = gmma_desc_const(kBoxBytes, 8u * kBoxBytes);
          const uint64_t bdc = gmma_desc_const(bk2 * 2, 16u * bk2);
          const uint32_t stg16 = (stg_c & 0x3FFFF) >> 4, w16 = ((stg_c + (kConsumers - c) * region) & 0x3FFFF) >> 4;
          const uint32_t ahalf2 = (64 * kBoxBytes) >> 4, wblk16 = (N2 * bk2 * 2) >> 4;
          const int run16 = N2 / 16 - (part ? kBoxCols / 16 : 0);
          // rows [0, 64) and then [64, 128), one m64 accumulator at a time (each sees the same MMAs as in the standalone
          // launch).  When the 1x1's output boxes have the staging boxes' 128-B span, output rows [0, 64) overwrite only A rows
          // [0, 64) of every box, so each half is written as soon as its MMAs are done (kDirect); otherwise the first half's
          // outputs wait in registers, packed, until the second half's MMAs have read the whole staging.
          constexpr bool kDirect = kBox2 == kBoxBytes;
          constexpr int kHeld = kDirect ? 1 : (F2 ? N2 / 2 : N2 / 4);
          uint32_t held[kHeld];
          float d[N2 / 2];
          const uint32_t bias2_t = sbias32 + (p.cout + 2 * (lane & 3)) * 4;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int i = 0; i < N2 / 2; ++i) d[i] = 0.f;
            wgmma_fence_acc(d);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < N2 / 16; ++k) {
              const int ach = k < run16 ? k0 + 16 * k : BN + 16 * (k - run16);   // staging channel (the partner box follows)
              const uint64_t ad = adc | (stg16 + (ach / kBoxCols) * (kBoxTile >> 4) + 2 * ((ach % kBoxCols) / 16) + h * ahalf2);
              const uint64_t bd = bdc | (w16 + (16 * k / bk2) * wblk16 + 2 * ((16 * k % bk2) / 16));
              Wgmma<N2>::mma(d, ad, bd, k == 0 ? 0u : 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(d);
            if (kDirect || h == 1) {
              if (lead && p.ch_store1 && h == (kDirect ? 0 : 1)) tma_store_wait_read<0>();   // the first output's store has read it
              named_bar_sync(1 + c, 128);                  // every warp's MMAs of this half have read the staging
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const int row = 64 * h + 16 * wq + (lane >> 2) + 8 * r;
              const uint32_t roff = static_cast<uint32_t>(row * kBox2), rxor = (roff >> 3) & kSwz2;
              const uint32_t rbase = stg_c + roff;
              const uint32_t row0 = static_cast<uint32_t>((row - 64) * kBox2), rxor0 = (row0 >> 3) & kSwz2;   // its first-half row
#pragma unroll
              for (int i = 0; i < N2 / 8; ++i) {
                const int col = 8 * i + 2 * (lane & 3);
                const float2 bb = lds_f2(bias2_t + 32 * i);
                const int k = 4 * i + 2 * r;
                const float f0 = act_apply<ACT2>(d[k] + bb.x);
                const float f1 = act_apply<ACT2>(d[k + 1] + bb.y);
                const int hi = kDirect ? 0 : r * (N2 / 8) + i;
                const uint32_t cb = (col / kBoxCols2) * kBoxTile2, cc = (col % kBoxCols2) * es2;
                if (kDirect || h == 1) {
                  if (F2) sts_f2(rbase + cb + (cc ^ rxor), f0, f1);
                  else sts_u32(rbase + cb + (cc ^ rxor), pack_bf16x2(f0, f1));
                }
                if (!kDirect && h == 0) {
                  if (F2) { held[2 * hi] = __float_as_uint(f0); held[2 * hi + 1] = __float_as_uint(f1); }
                  else held[hi] = pack_bf16x2(f0, f1);
                }
                if (!kDirect && h == 1) {
                  if (F2) sts_f2(stg_c + row0 + cb + (cc ^ rxor0), __uint_as_float(held[2 * hi]), __uint_as_float(held[2 * hi + 1]));
                  else sts_u32(stg_c + row0 + cb + (cc ^ rxor0), held[hi]);
                }
              }
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(1 + c, 128);
          if (lead) {
#pragma unroll
            for (int b = 0; b < N2 / kBoxCols2; ++b) tma_store_4d(&p.tmO2, stg + b * kBoxTile2, b * kBoxCols2, tx.w0, tx.h0, tx.n0);
            tma_store_commit();
          }
        }
      }
    }
    if (lead) {
      tma_store_wait_all();    // the output is complete in global memory before the CTA retires (PDL successors read it)
      if (p.trace != nullptr && blockIdx.x == 0) atomicMax(p.trace + 6, globaltimer_ns());   // last epilogue of CTA 0 done
    }
  }
  if (p.trace && threadIdx.x == 0) {
    atomicMax(p.trace + 2, globaltimer_ns());
    if (blockIdx.x == 0) p.trace[7] = globaltimer_ns();
  }
}

// ------------------------------------------------------------------------------------------------ host

bool conv_gemm_supported(const ConvDesc& d) {
  if (d.in.C % 16 != 0 || d.out.C % 16 != 0) return false;
  if (!(d.k == 1 || d.k == 3)) return false;
  if (!(d.stride == 1 || d.stride == 2)) return false;
  if (d.stride == 2 && (d.k != 3 || (d.in.H & 1) || (d.in.W & 1))) return false;
  if (d.in.co % 8 != 0 || d.in.cs % 8 != 0) return false;
  return true;
}

// N tile: a power of two in [16, 128] that divides Cout (the kernel is compiled for those four widths); an override is taken
// as an upper bound.  If the machine would be under-filled, the tile is halved (more, smaller tiles).
static int pick_bn(int cout, long long m_tiles, int bn_override, int num_sms) {
  const int maxbn = bn_override > 0 && bn_override < kMaxBN ? bn_override : kMaxBN;
  int BN = 16;
  while (BN * 2 <= maxbn && cout % (BN * 2) == 0) BN *= 2;
  if (bn_override == 0)
    while (BN > 64 && m_tiles * (cout / BN) < num_sms) BN /= 2;
  return BN;
}
static int pick_bk(int cin) { return (cin % 64 == 0) ? 64 : (cin % 32 == 0 ? 32 : 16); }

// the swizzle whose span is one box row: the kernel reads / writes the shared-memory tile with the same XOR
static CUtensorMapSwizzle swizzle_of(int span_bytes) {
  return span_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : span_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
}

// The slice s (elements of es bytes) as [N][H][W][C] at the launch's output pixels with the buffer's strides, ns pixels from
// one image to the next; box = `cols` channels x the 128-pixel tile box.  For the epilogue's TMA stores and loads.
static int encode_slice(const GemmParams& p, CUtensorMap* tm, const TSlice& s, int es, int cols, int ns, const char* who, const char* what) {
  CC_REQUIRE((size_t(s.cs) * es) % 16 == 0 && (size_t(s.co) * es) % 16 == 0, "%s: %s slice not 16-B aligned", who, what);
  void* base = reinterpret_cast<uint8_t*>(s.p) + size_t(s.co) * es;
  cuuint64_t dims[4] = {cuuint64_t(s.C), cuuint64_t(p.W), cuuint64_t(p.H), cuuint64_t(p.N)};
  const cuuint64_t px = cuuint64_t(s.cs) * es;     // bytes per pixel
  cuuint64_t strides[3] = {px, px * p.W, px * ns};
  cuuint32_t box[4] = {cuuint32_t(cols), cuuint32_t(1 << p.lTW), cuuint32_t(1 << p.lTH), cuuint32_t(1 << p.lTN)};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = get_encode_tiled()(tm, es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, dims, strides,
                                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_of(cols * es), CU_TENSOR_MAP_L2_PROMOTION_NONE,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  CC_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled(%s) failed: %d", who, what, int(r));
  return CC_OK;
}

// Shared-memory budget -> pipeline depth of a launch whose tiling is set: the arithmetic the kernel's carve-up follows.
// `fixed`: everything but the operands (alignment slack, the consumers' staging, bias, barriers, a chained 1x1's weights).
// The weights of a single N block stay resident when they leave room for at least four activation stages: the ring then
// carries A only and the weights cross the L2 once per CTA instead of once per tile.  Returns the stage count (at most 8).
static int set_smem_budget(GemmLaunch* L, int fixed) {
  GemmParams& p = L->p;
  const int a_bytes = kTileM * p.BK * 2, b_bytes = p.BN * p.BK * 2;
  const int bres_bytes = b_bytes * p.num_taps * p.chunks_per_tap;
  p.b_res = (p.n_blocks == 1 && (kMaxSmem - fixed - bres_bytes) / a_bytes >= 4) ? 1 : 0;
  int S = p.b_res ? (kMaxSmem - fixed - bres_bytes) / a_bytes : (kMaxSmem - fixed) / (a_bytes + b_bytes);
  if (S > 8) S = 8;
  p.stages = S;
  L->smem_bytes = fixed + (p.b_res ? bres_bytes + S * a_bytes : S * (a_bytes + b_bytes));
  return S;
}

// with_out = false: no first output (a chained launch that drops it; tmO stays unset)
static int gemm_build(const ConvDesc& d, int num_sms, GemmLaunch* L, bool with_out) {
  const int Cin = d.in.C, Cout = d.out.C, N = d.in.N;
  CC_REQUIRE(conv_gemm_supported(d), "conv_gemm: unsupported shape Cin=%d Cout=%d k=%d s=%d Hin=%d Win=%d", Cin, Cout,
             d.k, d.stride, d.in.H, d.in.W);
  PFN_encodeTiled enc = get_encode_tiled();
  CC_REQUIRE(enc != nullptr, "conv_gemm: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  const int es = d.out.f32 ? 4 : 2;

  GemmParams& p = L->p;
  memset(&p, 0, sizeof(p));
  const int Hout = conv_out(d.in.H, d.stride), Wout = conv_out(d.in.W, d.stride);
  p.W = Wout; p.H = Hout; p.N = N;

  // ---- K blocking
  p.BK = pick_bk(Cin);
  p.num_taps = d.k * d.k;
  p.chunks_per_tap = Cin / p.BK;
  // ---- N blocking
  const long long mt = (static_cast<long long>(N) * Hout * Wout + 127) / 128;
  const int BN = pick_bn(Cout, mt, d.bn_override, num_sms);
  CC_REQUIRE(BN >= 16 && BN <= kMaxBN && Cout % BN == 0, "conv_gemm: bad BN=%d for Cout=%d", BN, Cout);
  p.BN = BN;
  p.n_blocks = Cout / BN;
  p.cout = Cout;

  // ---- M tile box: maximise useful pixels per 128-row tile
  int best[3] = {7, 0, 0};
  double best_eff = -1;
  for (int lw = 0; lw <= 7; ++lw)
    for (int lh = 0; lw + lh <= 7; ++lh) {
      const int ln = 7 - lw - lh;
      const int tw = 1 << lw, th = 1 << lh, tn = 1 << ln;
      const double cover = double((Wout + tw - 1) / tw * tw) * ((Hout + th - 1) / th * th) * ((N + tn - 1) / tn * tn);
      double eff = double(Wout) * Hout * N / cover + 1e-6 * lw - 1e-7 * ln;  // ties: wider rows, fewer images
      if (eff > best_eff) { best_eff = eff; best[0] = lw; best[1] = lh; best[2] = ln; }
    }
  p.lTW = best[0]; p.lTH = best[1]; p.lTN = best[2];
  const int TW = 1 << p.lTW, TH = 1 << p.lTH, TN = 1 << p.lTN;
  p.tiles_w = (Wout + TW - 1) / TW;
  p.tiles_h = (Hout + TH - 1) / TH;
  p.tiles_n = (N + TN - 1) / TN;
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
        t[0] = wp * d.in.cs; t[1] = dw; t[2] = hp; t[3] = dh;
      }
    }

  // ---- tensor maps
  const CUtensorMapSwizzle swz = swizzle_of(p.BK * 2);
  {
    const int Hin = d.in.H, Win = d.in.W;
    void* base = reinterpret_cast<uint8_t*>(d.in.p) + size_t(d.in.co) * 2;
    CC_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "conv_gemm: input slice not 16-B aligned");
    cuuint64_t dims[5], strides[4];
    cuuint32_t box[5], estr[5] = {1, 1, 1, 1, 1};
    const cuuint64_t px = cuuint64_t(d.in.cs) * 2;  // bytes per pixel
    if (!p.s2) {
      dims[0] = Cin; dims[1] = Win; dims[2] = Hin; dims[3] = N; dims[4] = 1;
      strides[0] = px; strides[1] = px * Win; strides[2] = px * Win * Hin; strides[3] = px * Win * Hin * N;
      box[0] = p.BK; box[1] = TW; box[2] = TH; box[3] = TN; box[4] = 1;
    } else {
      dims[0] = d.in.cs + Cin; dims[1] = Win / 2; dims[2] = 2; dims[3] = Hin / 2; dims[4] = N;
      strides[0] = 2 * px; strides[1] = px * Win; strides[2] = 2 * px * Win; strides[3] = px * Win * Hin;
      box[0] = p.BK; box[1] = TW; box[2] = 1; box[3] = TH; box[4] = TN;
    }
    CUresult r = enc(&p.tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, base, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CC_REQUIRE(r == CUDA_SUCCESS, "conv_gemm: cuTensorMapEncodeTiled(A) failed: %d (dims %llu,%llu,%llu,%llu,%llu)", int(r),
               dims[0], dims[1], dims[2], dims[3], dims[4]);
  }
  {     // weights [Cout][Ktot] bf16, box = BK x BN
    const cuuint64_t Ktot = cuuint64_t(d.k) * d.k * Cin;
    cuuint64_t dims[2] = {Ktot, cuuint64_t(Cout)};
    cuuint64_t strides[1] = {Ktot * 2};
    cuuint32_t box[2] = {cuuint32_t(p.BK), cuuint32_t(BN)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d.w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CC_REQUIRE(r == CUDA_SUCCESS, "conv_gemm: cuTensorMapEncodeTiled(B) failed: %d", int(r));
  }

  // ---- epilogue
  p.out = d.out.p; p.out_cs = d.out.cs; p.out_co = d.out.co; p.out_f32 = d.out.f32;
  p.bias = d.bias; p.act = d.act; p.slope = d.slope;
  const bool prelu = d.act == ACT_PRELU;
  if (prelu)
    CC_REQUIRE(d.bias && d.slope && !d.out.f32 && !d.pre, "conv_gemm: ACT_PRELU needs its [9][Cout] bias table and slopes, and writes bf16");
  p.res = d.res.p; p.res_cs = d.res.cs; p.res_co = d.res.co;
  p.out_ns = d.out_ns > 0 ? d.out_ns : Hout * Wout;
  p.pre = d.pre; p.pre_h = d.pre_h; p.pre_w = d.pre_w;
  if (d.pre) CC_REQUIRE(d.pre_h * 2 == Hout && d.pre_w * 2 == Wout && Cout % 4 == 0, "conv_gemm: the pre-activation addend must be a half-resolution map of the output");
  // output slice (and residual): box = one staging column box (one swizzle span) x the pixel box
  const int box_cols = epi_box_bytes(BN, es) / es;
  if (with_out)
    if (int rc = encode_slice(p, &p.tmO, d.out, es, box_cols, p.out_ns, "conv_gemm", "output")) return rc;
  if (d.res.p)
    if (int rc = encode_slice(p, &p.tmR, d.res, es, box_cols, p.out_ns, "conv_gemm", "residual")) return rc;
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

  // ---- smem budget -> pipeline depth.  Fixed part: alignment slack, one output staging tile per consumer, bias, barriers.
  const int S = set_smem_budget(L, 1024 + kConsumers * epi_stage_bytes(BN, es) + Cout * 4 * (prelu ? 10 : 1) + 8 * kBarriers);
  CC_REQUIRE(S >= 2, "conv_gemm: tile does not fit shared memory (BN=%d BK=%d)", BN, p.BK);
  L->grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  L->flops = 2.0 * double(N) * Hout * Wout * Cout * d.k * d.k * Cin;
  L->bytes = double(N) * d.in.H * d.in.W * Cin * 2 + double(N) * Hout * Wout * Cout * es * ((with_out ? 1 : 0) + (d.res.p ? 1 : 0)) +
             double(Cout) * d.k * d.k * Cin * 2;
  return CC_OK;
}

int conv_gemm_build(const ConvDesc& d, int num_sms, GemmLaunch* L) {
  CC_REQUIRE(d.out.p != nullptr, "conv_gemm: no output");
  return gemm_build(d, num_sms, L, true);
}

static int chain_launch(const GemmLaunch& L, cudaStream_t stream, bool dry);

// The 1x1 c chains onto the conv d when
//   * d is a SiLU conv with a bf16 output and c is square, Cout2 <= 128 channels (so <= 32 KB of weights), SiLU into bf16 or
//     no activation into fp32 (at most 64 channels: one 128 x 256-B tile), and the standalone launch of c would tile it as
//     one n block (its instruction N is then Cout2);
//   * c's input is a run of d's output channels [k0, k0 + run) inside one n block, starting on a k16 step, optionally
//     followed by a partner slice exactly one staging box wide;
//   * d's first output may be dropped only when d has one n block, and the operand ring keeps at least 4 stages.
int conv_gemm_chain_build(const ConvDesc& d, const ChainDesc& c, int num_sms, GemmLaunch* L) {
  const int N2 = c.out.C, part_C = c.part.p ? c.part.C : 0;
  CC_REQUIRE(c.w && c.out.p && (d.out.p || !c.store1), "conv_gemm chain: NULL weights or output");
  CC_REQUIRE(d.act == ACT_SILU && !d.out.f32, "conv_gemm chain: the first conv must be SiLU into bf16");
  CC_REQUIRE(!d.pre, "conv_gemm chain: the first conv takes no pre-activation addend");
  CC_REQUIRE(N2 >= 16 && N2 <= kMaxBN && N2 % 16 == 0, "conv_gemm chain: the 1x1 has %d channels (16..128)", N2);
  CC_REQUIRE((c.act == ACT_SILU && !c.out.f32) || (c.act == ACT_NONE && c.out.f32 && N2 <= 64),
             "conv_gemm chain: the 1x1 is SiLU into bf16 or no activation into fp32 (<= 64 channels)");
  const int Hout = conv_out(d.in.H, d.stride), Wout = conv_out(d.in.W, d.stride);
  const long long mt = (static_cast<long long>(d.in.N) * Hout * Wout + 127) / 128;
  CC_REQUIRE(pick_bn(N2, mt, 0, num_sms) == N2, "conv_gemm chain: the standalone 1x1 would tile its %d channels in blocks", N2);
  if (int rc = gemm_build(d, num_sms, L, c.store1)) return rc;
  GemmParams& p = L->p;
  const int BN = p.BN;
  const int box_bytes = epi_box_bytes(BN, 2), box_cols = box_bytes / 2, box_tile = kTileM * box_bytes;
  const int run = N2 - part_C;
  CC_REQUIRE(!c.part.p || part_C == box_cols, "conv_gemm chain: the partner slice must be one staging box (%d channels)", box_cols);
  CC_REQUIRE(run > 0 && c.k0 >= 0 && c.k0 % 16 == 0 && c.k0 / BN == (c.k0 + run - 1) / BN && c.k0 + run <= d.out.C,
             "conv_gemm chain: input run [%d, %d) is not inside one %d-channel n block", c.k0, c.k0 + run, BN);
  CC_REQUIRE(!(d.res.p && BN == 128), "conv_gemm chain: a 128-channel tile takes no residual");
  CC_REQUIRE((c.store1 && !c.part.p) || p.n_blocks == 1, "conv_gemm chain: a dropped first output or a partner needs one n block");
  p.ch_n2 = N2;
  p.ch_nb = c.k0 / BN;
  p.ch_k0 = c.k0 - p.ch_nb * BN;
  p.ch_part = c.part.p ? 1 : 0;
  p.ch_store1 = c.store1 ? 1 : 0;
  p.ch_bk2 = pick_bk(N2);
  p.act2 = c.act;
  p.out2_f32 = c.out.f32;
  p.bias2 = c.bias;
  const int es2 = c.out.f32 ? 4 : 2;
  {     // 1x1 weights [Cout2][Cin2 = Cout2], box = BK2 x Cout2
    cuuint64_t dims[2] = {cuuint64_t(N2), cuuint64_t(N2)};
    cuuint64_t strides[1] = {cuuint64_t(N2) * 2};
    cuuint32_t box[2] = {cuuint32_t(p.ch_bk2), cuuint32_t(N2)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = get_encode_tiled()(&p.tmW2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(c.w), dims, strides, box, estr,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_of(p.ch_bk2 * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CC_REQUIRE(r == CUDA_SUCCESS, "conv_gemm chain: cuTensorMapEncodeTiled(W2) failed: %d", int(r));
  }
  if (c.part.p)
    if (int rc = encode_slice(p, &p.tmP, c.part, 2, box_cols, Hout * Wout, "conv_gemm chain", "partner")) return rc;
  if (int rc = encode_slice(p, &p.tmO2, c.out, es2, epi_box_bytes(N2, es2) / es2, Hout * Wout, "conv_gemm chain", "out2")) return rc;

  // ---- smem: each consumer's region holds its staging tile and the partner box, then the 1x1's output tile
  const int stage1 = epi_stage_bytes(BN, 2) + (c.part.p ? box_tile : 0), stage2 = kTileM * N2 * es2;
  p.ch_stage = ((stage1 > stage2 ? stage1 : stage2) + 1023) & ~1023;
  const int w2_bytes = (N2 * N2 * 2 + 1023) & ~1023;
  const int S = set_smem_budget(L, 1024 + kConsumers * p.ch_stage + w2_bytes + (d.out.C + N2) * 4 + 8 * kBarriers);
  CC_REQUIRE(S >= 4, "conv_gemm chain: the operand ring would keep %d stages (at least 4)", S);
  const double px = double(d.in.N) * Hout * Wout;
  L->flops += 2.0 * px * N2 * N2;
  L->bytes += px * (part_C * 2 + N2 * es2) + double(N2) * N2 * 2;
  CC_REQUIRE(chain_launch(*L, nullptr, true) == CC_OK, "conv_gemm chain: no chained kernel for BN=%d and a %d-channel 1x1 (act %d, fp32 %d)",
             BN, N2, c.act, c.out.f32);
  return CC_OK;
}

template <int ACT, bool F32, int BN, int N2 = 0, int ACT2 = ACT_NONE, bool F2 = false>
static int launch_bn(const GemmLaunch& L, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    CC_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<ACT, F32, BN, N2, ACT2, F2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
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
  CC_CHECK_CUDA(cudaLaunchKernelEx(&cfg, conv_gemm_kernel<ACT, F32, BN, N2, ACT2, F2>, L.p));
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

// The chained instances: (producer BN, 1x1 channels) of the detector's chains (yolo.cu), SiLU into bf16, and the head's
// 64 -> 64 logits (no activation, fp32).  dry: only report whether the instance exists.
static int chain_launch(const GemmLaunch& L, cudaStream_t stream, bool dry) {
  const GemmParams& p = L.p;
  const int key = p.BN * 1000 + p.ch_n2;
  if (p.act2 == ACT_NONE && p.out2_f32) {
    if (key == 64064) return dry ? CC_OK : launch_bn<ACT_SILU, false, 64, 64, ACT_NONE, true>(L, stream);
  } else if (p.act2 == ACT_SILU && !p.out2_f32) {
    switch (key) {
      case 16032: return dry ? CC_OK : launch_bn<ACT_SILU, false, 16, 32, ACT_SILU, false>(L, stream);
      case 32032: return dry ? CC_OK : launch_bn<ACT_SILU, false, 32, 32, ACT_SILU, false>(L, stream);
      case 32064: return dry ? CC_OK : launch_bn<ACT_SILU, false, 32, 64, ACT_SILU, false>(L, stream);
      case 64032: return dry ? CC_OK : launch_bn<ACT_SILU, false, 64, 32, ACT_SILU, false>(L, stream);
      case 64064: return dry ? CC_OK : launch_bn<ACT_SILU, false, 64, 64, ACT_SILU, false>(L, stream);
      case 64128: return dry ? CC_OK : launch_bn<ACT_SILU, false, 64, 128, ACT_SILU, false>(L, stream);
      case 128064: return dry ? CC_OK : launch_bn<ACT_SILU, false, 128, 64, ACT_SILU, false>(L, stream);
      case 128128: return dry ? CC_OK : launch_bn<ACT_SILU, false, 128, 128, ACT_SILU, false>(L, stream);
    }
  }
  set_error("conv_gemm: no chained kernel for BN=%d, 1x1 of %d channels, act %d, fp32 %d", p.BN, p.ch_n2, p.act2, p.out2_f32);
  return CC_ERR_INVALID;
}

int conv_gemm_launch(const GemmLaunch& L, cudaStream_t stream) {
  if (L.p.ch_n2 > 0) return chain_launch(L, stream, false);
  const bool f32 = L.p.out_f32 != 0;
  switch (L.p.act) {
    case ACT_NONE: return f32 ? launch_variant<ACT_NONE, true>(L, stream) : launch_variant<ACT_NONE, false>(L, stream);
    case ACT_SILU: return f32 ? launch_variant<ACT_SILU, true>(L, stream) : launch_variant<ACT_SILU, false>(L, stream);
    case ACT_GELU_TANH:
      return f32 ? launch_variant<ACT_GELU_TANH, true>(L, stream) : launch_variant<ACT_GELU_TANH, false>(L, stream);
    case ACT_PRELU:
      if (!f32) return launch_variant<ACT_PRELU, false>(L, stream);
      break;
  }
  set_error("conv_gemm: unknown activation %d", L.p.act);
  return CC_ERR_INVALID;
}

}  // namespace cc
