// Baseline JPEG of object crops on the device, byte-identical to cv2.imwrite / cv2.imencode (OpenCV 4.13 with
// libjpeg-turbo: 4:2:0, integer DCT, Annex K tables scaled by the quality, no optimisation, no restart markers).
// oracle/jpeg.py states the arithmetic and is pinned to cv2; everything here is integer code restating it.
//
// Replaces the per-object thumbnail of `VideoCapture.save_object` (clearcam.py:373-399, cv2.imwrite of the crop of the
// frame) for frames that are already in HBM for the detector: only the compressed bytes cross PCIe.
//
// One call, per group of up to kCropsPerLaunch crops (the crop table travels as a kernel parameter, so there is no copy,
// no allocation and no host sync), runs eight stream-ordered launches over all of its crops.  In the transform's table
// every crop carries its own source (frame pointer, extent, RGB / BGR / I420), so the crops of one call may come from
// frames of any shapes and formats (cc_jpeg_encode_crops_frames).
//   1. transform  one CTA per MCU (16x16 pixels): gather with libjpeg's edge replication, YCbCr, h2v2 downsampling,
//                 8x8 integer DCT, quantisation -> int16 zigzag coefficients of the 6 blocks, dummy blocks included
//   2. lengths    one CTA per tile of kTileMcus MCUs, a warp per block: the bit length of every block's Huffman codes
//   3. scan       one CTA: per crop, exclusive scan of the tile bit lengths (tile bit offsets, crop bit totals)
//   4. zero       clears the used part of each crop's bit scratch
//   5. pack       per tile: each warp assembles a block's bits in shared memory, stores its inner words and ORs its two
//                 edge words into the crop's big-endian bit scratch; the crop's last tile pads the final byte with 1s
//   6. count      per tile: 0xFF bytes among the bytes whose first bit lies in the tile
//   7. scan       per crop, exclusive scan of those counts; the encoded length of each crop
//   8. scatter    per tile: bytes with 0xFF -> 0xFF 0x00 stuffing behind the header; tile 0 writes the header, the last
//                 tile the EOI marker
#include <cstdint>
#include <cstring>
#include <vector>
#include <algorithm>

#include "cc_common.h"
#include "clearcam_b200.h"
#include "ops.cuh"

namespace cc {
namespace {

constexpr int kCropsPerLaunch = 256;
constexpr int kTileMcus = 64;                       // MCUs (6 blocks each) per entropy tile
constexpr int kMaxBlockBits = 22 + 63 * 26;         // DC: 11-bit code + 11 bits; AC: 16-bit code + 10 bits
constexpr int kHeaderBytes = 623;
constexpr int kSofHeight = 163;                     // byte offsets of the SOF0 height / width in the header
constexpr int kZeroWords = 4096;                    // scratch words cleared per CTA of the zero kernel
constexpr int kMaxSide = 65535;                     // a JPEG frame header holds 16-bit sizes

struct JpegCrop {
  int x1, y1, w, h;
  int mw, nmcu;           // MCUs per row, MCUs
  int mcu0, tile0, ntile; // first MCU / tile of the crop in the launch group
  int zero0;              // first CTA of the crop in the zero kernel
  long long word0;        // first word of the crop's bit scratch
  long long out;          // byte offset of the crop in d_out
};

struct HuffTables {
  uint32_t dc[2][12];     // (code << 5) | length, luma / chroma
  uint32_t ac[2][256];
};

struct JpegParams {
  int K, n_mcu, n_tile;
  int16_t* coef;                   // [n_mcu * 6][64], zigzag order
  uint32_t* blen;                  // [n_mcu * 6] bits per block
  unsigned long long* tbits;       // [n_tile] bits per tile, then the tile's bit offset in its crop
  unsigned long long* tff;         // [n_tile] 0xFF bytes per tile, then those before the tile in its crop
  unsigned long long* cbits;       // [K] bits of each crop's scan data
  uint32_t* words;                 // bit scratch, MSB first
  uint8_t* out;
  long long* lengths;              // [K] encoded bytes of each crop
  uint16_t qdiv[2][64];            // 8 x quantisation table, natural order
  HuffTables huff;
  uint8_t header[kHeaderBytes];
  JpegCrop crop[kCropsPerLaunch];
};
// the largest launch (the scan kernel) passes two ints beside the table; 32,764 bytes is the kernel parameter limit
static_assert(sizeof(JpegParams) + 2 * sizeof(int) <= 32764, "the crop table no longer fits the kernel parameters");

// The transform's own, smaller table: only it reads the pixels, so only it carries each crop's source (the seven entropy
// launches keep the table above and pay nothing for the sources).
struct TransformCrop {
  CropSource src;         // the crop's frame, its extent and format
  int x1, y1, w, h;
  int mw, mcu0;           // MCUs per row, first MCU of the crop in the launch group
};
struct TransformParams {
  int K;
  int16_t* coef;                   // [n_mcu * 6][64], zigzag order
  uint16_t qdiv[2][64];            // 8 x quantisation table, natural order
  TransformCrop crop[kCropsPerLaunch];
};
static_assert(sizeof(TransformParams) <= 32764, "the transform's crop table no longer fits the kernel parameters");

__constant__ uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

__device__ __forceinline__ int find_crop_by_mcu(const TransformParams& p, int m) {
  int lo = 0, hi = p.K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.crop[mid].mcu0 <= m) lo = mid; else hi = mid - 1;
  }
  return lo;
}
__device__ __forceinline__ int find_crop_by_tile(const JpegParams& p, int t) {
  int lo = 0, hi = p.K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.crop[mid].tile0 <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

constexpr int fix16(double x) { return static_cast<int>(x * 65536.0 + 0.5); }

// ------------------------------------------------------------------------------------------------ 1. transform
constexpr int kC0_298 = 2446, kC0_390 = 3196, kC0_541 = 4433, kC0_765 = 6270, kC0_899 = 7373, kC1_175 = 9633;
constexpr int kC1_501 = 12299, kC1_847 = 15137, kC1_961 = 16069, kC2_053 = 16819, kC2_562 = 20995, kC3_072 = 25172;

// one 8-point pass of the integer DCT on d[0], d[s], ..., d[7s]; col: the second (column) pass
template <bool COL>
__device__ __forceinline__ void fdct8(int* d, int s) {
  constexpr int kSh = COL ? 15 : 11;                // CONST_BITS +/- PASS1_BITS
  const int tmp0 = d[0] + d[7 * s], tmp7 = d[0] - d[7 * s];
  const int tmp1 = d[s] + d[6 * s], tmp6 = d[s] - d[6 * s];
  const int tmp2 = d[2 * s] + d[5 * s], tmp5 = d[2 * s] - d[5 * s];
  const int tmp3 = d[3 * s] + d[4 * s], tmp4 = d[3 * s] - d[4 * s];
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  if (COL) {
    d[0] = (tmp10 + tmp11 + 2) >> 2;
    d[4 * s] = (tmp10 - tmp11 + 2) >> 2;
  } else {
    d[0] = (tmp10 + tmp11) * 4;
    d[4 * s] = (tmp10 - tmp11) * 4;
  }
  constexpr int kHalf = 1 << (kSh - 1);
  int z1 = (tmp12 + tmp13) * kC0_541;
  d[2 * s] = (z1 + tmp13 * kC0_765 + kHalf) >> kSh;
  d[6 * s] = (z1 - tmp12 * kC1_847 + kHalf) >> kSh;
  z1 = tmp4 + tmp7;
  int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
  const int z5 = (z3 + z4) * kC1_175;
  z1 = -z1 * kC0_899;
  z2 = -z2 * kC2_562;
  z3 = -z3 * kC1_961 + z5;
  z4 = -z4 * kC0_390 + z5;
  d[7 * s] = (tmp4 * kC0_298 + z1 + z3 + kHalf) >> kSh;
  d[5 * s] = (tmp5 * kC2_053 + z2 + z4 + kHalf) >> kSh;
  d[3 * s] = (tmp6 * kC3_072 + z2 + z3 + kHalf) >> kSh;
  d[s] = (tmp7 * kC1_501 + z1 + z4 + kHalf) >> kSh;
}

// the crop's source format (CropSource::fmt) is read per CTA: one MCU belongs to one crop, so the branch is uniform
__global__ void __launch_bounds__(256) jpeg_transform_kernel(const __grid_constant__ TransformParams p) {
  __shared__ int cb[16][16], cr[16][16];
  __shared__ int blk[6][64];
  __shared__ int dc[4];
  const int m = blockIdx.x, t = threadIdx.x;
  const TransformCrop& c = p.crop[find_crop_by_mcu(p, m)];
  const int mi = m - c.mcu0, my = mi / c.mw, mx = mi - my * c.mw;
  const int py = t >> 4, px = t & 15;
  // columns replicated before downsampling, rows to the 2-row group (and, for luma, on to the MCU: same pixel)
  const int yy = c.y1 + min(my * 16 + py, c.h - 1), xx = c.x1 + min(mx * 16 + px, c.w - 1);
  int r, g, b;
  if (c.src.fmt == 2) {
    int bgr[3];
    i420_bgr(c.src.frame, c.src.H, c.src.W, yy, xx, bgr);
    b = bgr[0]; g = bgr[1]; r = bgr[2];
  } else {
    const uint8_t* px3 = c.src.frame + (static_cast<size_t>(yy) * c.src.W + xx) * 3;
    const int c0 = __ldg(px3), c1 = __ldg(px3 + 1), c2 = __ldg(px3 + 2);
    const bool rgb = c.src.fmt == 0;
    r = rgb ? c0 : c2; g = c1; b = rgb ? c2 : c0;
  }
  constexpr int kHalf = 1 << 15, kCbCrOff = (128 << 16) + kHalf - 1;
  const int Y = (fix16(0.299) * r + fix16(0.587) * g + fix16(0.114) * b + kHalf) >> 16;
  cb[py][px] = (-fix16(0.16874) * r - fix16(0.33126) * g + fix16(0.5) * b + kCbCrOff) >> 16;
  cr[py][px] = (fix16(0.5) * r - fix16(0.41869) * g - fix16(0.08131) * b + kCbCrOff) >> 16;
  blk[(py >> 3) * 2 + (px >> 3)][(py & 7) * 8 + (px & 7)] = Y - 128;
  __syncthreads();
  if (t < 128) {
    // h2v2: chroma row r of the MCU averages input rows 2r, 2r+1; past the last chroma row of the image
    // (ceil(h/2) rows) the downsampled rows are replicated, not the input rows
    const int comp = t >> 6, rr = (t >> 3) & 7, cc = t & 7;
    const int last = (c.h + 1) / 2 - 1 - my * 8;
    const int sr = min(rr, last);
    const int (*src)[16] = comp ? cr : cb;
    const int s = src[2 * sr][2 * cc] + src[2 * sr][2 * cc + 1] + src[2 * sr + 1][2 * cc] + src[2 * sr + 1][2 * cc + 1];
    blk[4 + comp][rr * 8 + cc] = ((s + 1 + (cc & 1)) >> 2) - 128;
  }
  __syncthreads();
  if (t < 48) fdct8<false>(&blk[t >> 3][(t & 7) * 8], 1);
  __syncthreads();
  if (t < 48) fdct8<true>(&blk[t >> 3][t & 7], 8);
  __syncthreads();
  const int bw = (c.w + 7) >> 3, bh = (c.h + 7) >> 3;
  auto quant = [&](int j, int nat) {
    const int x = blk[j][nat], d = p.qdiv[j < 4 ? 0 : 1][nat];
    const int q = static_cast<int>((static_cast<unsigned>(abs(x)) + (d >> 1)) / static_cast<unsigned>(d));
    return x < 0 ? -q : q;
  };
  if (t == 0) {
    // dummy blocks: right of the last block column, the DC of the block to the left; in a row below the last block row,
    // the DC of the last block of the row above in this MCU (Y1, itself possibly a copy of Y0)
    const bool right = mx * 2 + 1 >= bw, bottom = my * 2 + 1 >= bh;
    const int d0 = quant(0, 0);
    const int d1 = right ? d0 : quant(1, 0);
    const int d2 = bottom ? d1 : quant(2, 0);
    const int d3 = bottom ? d1 : right ? d2 : quant(3, 0);
    dc[0] = d0; dc[1] = d1; dc[2] = d2; dc[3] = d3;
  }
  __syncthreads();
  int16_t* dst = p.coef + static_cast<size_t>(m) * 6 * 64;
  for (int i = t; i < 6 * 64; i += 256) {
    const int j = i >> 6, zz = i & 63;
    int v;
    if (j < 4 && ((mx * 2 + (j & 1)) >= bw || (my * 2 + (j >> 1)) >= bh)) v = zz == 0 ? dc[j] : 0;
    else v = zz == 0 && j < 4 ? dc[j] : quant(j, kZigzag[zz]);
    dst[i] = static_cast<int16_t>(v);
  }
}

// ------------------------------------------------------------------------------------------------ 2 + 5. Huffman codes
// The codes of one block, two zigzag positions per lane (2*lane, 2*lane+1): position 0 carries the DC difference,
// a nonzero AC coefficient its run of zeros (ZRL codes for each 16, then the run/size code) and its amplitude bits, and
// position 63, when zero, the end-of-block code.  Each field group is at most 3 * 11 + 16 + 10 = 59 bits.
struct Tok {
  unsigned long long v0, v1;
  int l0, l1;
};

__device__ __forceinline__ int nbits(int v) { return 32 - __clz(abs(v)); }

__device__ __forceinline__ void ac_token(const uint32_t* ac, int run, int v, unsigned long long& bits, int& len) {
  bits = 0; len = 0;
  const uint32_t zrl = ac[0xF0];
  for (; run > 15; run -= 16) { bits = (bits << (zrl & 31)) | (zrl >> 5); len += zrl & 31; }
  const int n = nbits(v);
  const uint32_t e = ac[(run << 4) | n];
  bits = (bits << (e & 31)) | (e >> 5);
  bits = (bits << n) | (static_cast<unsigned>(v < 0 ? v - 1 : v) & ((1u << n) - 1));
  len += (e & 31) + n;
}

__device__ __forceinline__ Tok block_tokens(const int16_t* coef, int pred, const uint32_t* dc, const uint32_t* ac, int lane) {
  const uint32_t pair = reinterpret_cast<const uint32_t*>(coef)[lane];
  const int a = static_cast<int16_t>(pair & 0xFFFF), b = static_cast<int16_t>(pair >> 16);
  // highest "nonzero" position of each lane's pair (position 0 always counts: the run of position 1 starts there)
  const int hp = b ? 2 * lane + 1 : (a || lane == 0) ? 2 * lane : -1;
  const unsigned any = __ballot_sync(0xffffffffu, hp >= 0);
  const int below = any & ((1u << lane) - 1u) ? 31 - __clz(any & ((1u << lane) - 1u)) : 0;
  const int prev_lane = __shfl_sync(0xffffffffu, hp, below);
  Tok k{0, 0, 0, 0};
  const int prev_a = lane == 0 ? 0 : prev_lane;
  if (lane == 0) {
    const int diff = a - pred, n = nbits(diff);
    const uint32_t e = dc[n];
    k.v0 = (static_cast<unsigned long long>(e >> 5) << n) | (static_cast<unsigned>(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1));
    k.l0 = (e & 31) + n;
  } else if (a) {
    ac_token(ac, 2 * lane - prev_a - 1, a, k.v0, k.l0);
  }
  if (b) {
    ac_token(ac, 2 * lane + 1 - (a || lane == 0 ? 2 * lane : prev_a) - 1, b, k.v1, k.l1);
  } else if (lane == 31) {
    const uint32_t e = ac[0x00];
    k.v1 = e >> 5; k.l1 = e & 31;
  }
  return k;
}

__device__ __forceinline__ int dc_pred(const int16_t* coef_m, int j, bool first_mcu) {
  // DC predictor: Y0 <- Y3 of the previous MCU, Y1..Y3 <- the previous Y block, Cb / Cr <- the previous MCU's
  if (j >= 1 && j <= 3) return coef_m[(j - 1) * 64];
  if (first_mcu) return 0;
  return coef_m[(j == 0 ? 3 - 6 : j - 6) * 64];
}

__device__ __forceinline__ void load_tables(const JpegParams& p, uint32_t* sdc, uint32_t* sac) {
  for (int i = threadIdx.x; i < 24; i += blockDim.x) sdc[i] = p.huff.dc[i / 12][i % 12];
  for (int i = threadIdx.x; i < 512; i += blockDim.x) sac[i] = p.huff.ac[i >> 8][i & 255];
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256) jpeg_lengths_kernel(const __grid_constant__ JpegParams p) {
  __shared__ uint32_t sdc[24], sac[512];
  __shared__ unsigned long long wsum[8];
  load_tables(p, sdc, sac);
  __syncthreads();
  const int tile = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const JpegCrop& c = p.crop[find_crop_by_tile(p, tile)];
  const int m_first = (tile - c.tile0) * kTileMcus, m_end = min(m_first + kTileMcus, c.nmcu);
  unsigned long long acc = 0;
  for (int bi = m_first * 6 + warp; bi < m_end * 6; bi += 8) {
    const int mi = bi / 6, j = bi - mi * 6, comp = j < 4 ? 0 : 1;
    const int16_t* cm = p.coef + static_cast<size_t>(c.mcu0 + mi) * 6 * 64;
    const int pred = lane == 0 ? dc_pred(cm, j, mi == 0) : 0;
    const Tok k = block_tokens(cm + j * 64, pred, sdc + 12 * comp, sac + 256 * comp, lane);
    const int len = warp_sum(k.l0 + k.l1);
    if (lane == 0) p.blen[static_cast<size_t>(c.mcu0) * 6 + bi] = len;
    acc += len;
  }
  if (lane == 0) wsum[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int w = 0; w < 8; ++w) s += wsum[w];
    p.tbits[tile] = s;
  }
}

// ------------------------------------------------------------------------------------------------ 3 + 7. per-crop scans
// mode 0: tbits -> exclusive offsets within the crop, cbits = crop totals.  mode 1: tff -> exclusive counts, lengths.
__global__ void __launch_bounds__(1024) jpeg_scan_kernel(const __grid_constant__ JpegParams p, int mode, int k_base) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < p.K; k += 32) {
    const JpegCrop& c = p.crop[k];
    unsigned long long* a = (mode == 0 ? p.tbits : p.tff) + c.tile0;
    unsigned long long carry = 0;
    for (int i0 = 0; i0 < c.ntile; i0 += 32) {
      const int i = i0 + lane;
      const unsigned long long v = i < c.ntile ? a[i] : 0;
      unsigned long long s = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long u = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += u;
      }
      if (i < c.ntile) a[i] = carry + s - v;
      carry += __shfl_sync(0xffffffffu, s, 31);
    }
    if (lane == 0) {
      if (mode == 0) p.cbits[k] = carry;
      else p.lengths[k_base + k] = kHeaderBytes + static_cast<long long>((p.cbits[k] + 7) >> 3) + static_cast<long long>(carry) + 2;
    }
  }
}

// ------------------------------------------------------------------------------------------------ 4. zero
__global__ void __launch_bounds__(256) jpeg_zero_kernel(const __grid_constant__ JpegParams p) {
  int lo = 0, hi = p.K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.crop[mid].zero0 <= static_cast<int>(blockIdx.x)) lo = mid; else hi = mid - 1;
  }
  const JpegCrop& c = p.crop[lo];
  const long long used = static_cast<long long>((p.cbits[lo] + 31) >> 5) + 1;
  const long long w0 = static_cast<long long>(blockIdx.x - c.zero0) * kZeroWords;
  for (long long w = w0 + threadIdx.x; w < min(used, w0 + kZeroWords); w += 256) p.words[c.word0 + w] = 0;
}

// ------------------------------------------------------------------------------------------------ 5. pack
constexpr int kWarpWords = 64;      // (kMaxBlockBits + 31) / 32 + 1 <= 64

__device__ __forceinline__ void or_bits(uint32_t* buf, int pos, unsigned long long v, int len) {
  if (!len) return;
  const int w = pos >> 5, sh = pos & 31;
  const unsigned __int128 x = static_cast<unsigned __int128>(v) << (96 - sh - len);
  const uint32_t a = static_cast<uint32_t>(x >> 64), b = static_cast<uint32_t>(x >> 32), c = static_cast<uint32_t>(x);
  if (a) atomicOr(buf + w, a);
  if (b) atomicOr(buf + w + 1, b);
  if (c) atomicOr(buf + w + 2, c);
}

__global__ void __launch_bounds__(256) jpeg_pack_kernel(const __grid_constant__ JpegParams p) {
  __shared__ uint32_t sdc[24], sac[512];
  __shared__ unsigned long long boff[kTileMcus * 6];
  __shared__ uint32_t wbuf[8][kWarpWords + 4];
  load_tables(p, sdc, sac);
  const int tile = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k = find_crop_by_tile(p, tile);
  const JpegCrop& c = p.crop[k];
  const int m_first = (tile - c.tile0) * kTileMcus, m_end = min(m_first + kTileMcus, c.nmcu);
  const int nb = (m_end - m_first) * 6;
  const uint32_t* bl = p.blen + (static_cast<size_t>(c.mcu0) + m_first) * 6;
  // exclusive scan of the tile's block lengths by warp 0: 12 consecutive blocks per lane
  if (warp == 0) {
    constexpr int kPer = kTileMcus * 6 / 32;
    unsigned long long loc = 0;
    for (int i = 0; i < kPer; ++i) loc += lane * kPer + i < nb ? bl[lane * kPer + i] : 0;
    unsigned long long s = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += u;
    }
    unsigned long long run = p.tbits[tile] + s - loc;
    for (int i = 0; i < kPer; ++i) {
      const int bi = lane * kPer + i;
      if (bi < nb) { boff[bi] = run; run += bl[bi]; }
    }
  }
  __syncthreads();
  uint32_t* buf = wbuf[warp];
  uint32_t* words = p.words + c.word0;
  for (int bi = warp; bi < nb; bi += 8) {
    const int mi = m_first + bi / 6, j = bi % 6, comp = j < 4 ? 0 : 1;
    const int16_t* cm = p.coef + static_cast<size_t>(c.mcu0 + mi) * 6 * 64;
    const int pred = lane == 0 ? dc_pred(cm, j, mi == 0) : 0;
    const Tok t = block_tokens(cm + j * 64, pred, sdc + 12 * comp, sac + 256 * comp, lane);
    int s = t.l0 + t.l1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += u;
    }
    const int total = __shfl_sync(0xffffffffu, s, 31);
    const unsigned long long off = boff[bi];
    const int sh = static_cast<int>(off & 31);
    buf[lane] = 0; buf[lane + 32] = 0;
    if (lane < 4) buf[64 + lane] = 0;
    __syncwarp();
    const int pos = sh + s - t.l0 - t.l1;
    or_bits(buf, pos, t.v0, t.l0);
    or_bits(buf, pos + t.l0, t.v1, t.l1);
    __syncwarp();
    const int nw = (sh + total + 31) >> 5;
    const long long w0 = static_cast<long long>(off >> 5);
    for (int i = lane; i < nw; i += 32) {
      if (i == 0 || i == nw - 1) atomicOr(words + w0 + i, buf[i]);     // shared with the neighbouring blocks
      else words[w0 + i] = buf[i];
    }
    __syncwarp();
  }
  if (tile == c.tile0 + c.ntile - 1 && threadIdx.x == 0) {
    const unsigned long long T = p.cbits[k];
    const int used = static_cast<int>(T & 7);
    if (used) {                                   // pad the last byte with 1-bits
      const int b0 = static_cast<int>(T & 31) & ~7;
      atomicOr(words + (T >> 5), ((1u << (8 - used)) - 1u) << (24 - b0));
    }
  }
}

// ------------------------------------------------------------------------------------------------ 6 + 8. stuffing
__device__ __forceinline__ uint32_t byte_at(const uint32_t* words, long long i) {
  return (words[i >> 2] >> (24 - 8 * (i & 3))) & 0xFF;
}

// bytes [b_begin, b_end) of the crop's scan data are those whose first bit lies in the tile
__device__ __forceinline__ void tile_bytes(const JpegParams& p, int k, int tile, long long& b0, long long& b1) {
  const JpegCrop& c = p.crop[k];
  const unsigned long long o0 = p.tbits[tile];
  const unsigned long long o1 = tile + 1 < c.tile0 + c.ntile ? p.tbits[tile + 1] : p.cbits[k];
  b0 = static_cast<long long>((o0 + 7) >> 3);
  b1 = static_cast<long long>((o1 + 7) >> 3);
}

__global__ void __launch_bounds__(256) jpeg_count_kernel(const __grid_constant__ JpegParams p) {
  __shared__ int wsum[8];
  const int tile = blockIdx.x, k = find_crop_by_tile(p, tile);
  long long b0, b1;
  tile_bytes(p, k, tile, b0, b1);
  const uint32_t* words = p.words + p.crop[k].word0;
  int n = 0;
  for (long long i = b0 + threadIdx.x; i < b1; i += 256) n += byte_at(words, i) == 0xFF;
  n = warp_sum(n);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < 8; ++w) s += wsum[w];
    p.tff[tile] = s;
  }
}

__global__ void __launch_bounds__(256) jpeg_scatter_kernel(const __grid_constant__ JpegParams p, int k_base) {
  __shared__ int wsum[8];
  __shared__ long long carry_s;
  const int tile = blockIdx.x, k = find_crop_by_tile(p, tile), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const JpegCrop& c = p.crop[k];
  uint8_t* out = p.out + c.out;
  if (tile == c.tile0) {
    for (int i = threadIdx.x; i < kHeaderBytes; i += 256) {
      uint8_t v = p.header[i];
      if (i == kSofHeight) v = static_cast<uint8_t>(c.h >> 8);
      if (i == kSofHeight + 1) v = static_cast<uint8_t>(c.h);
      if (i == kSofHeight + 2) v = static_cast<uint8_t>(c.w >> 8);
      if (i == kSofHeight + 3) v = static_cast<uint8_t>(c.w);
      out[i] = v;
    }
  }
  if (tile == c.tile0 + c.ntile - 1 && threadIdx.x == 0) {
    const long long len = p.lengths[k_base + k];
    out[len - 2] = 0xFF;
    out[len - 1] = 0xD9;
  }
  long long b0, b1;
  tile_bytes(p, k, tile, b0, b1);
  const uint32_t* words = p.words + c.word0;
  if (threadIdx.x == 0) carry_s = kHeaderBytes + b0 + static_cast<long long>(p.tff[tile]);
  __syncthreads();
  for (long long i0 = b0; i0 < b1; i0 += 4 * 256) {
    uint32_t v[4];
    int n = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long i = i0 + 4 * threadIdx.x + j;
      v[j] = i < b1 ? byte_at(words, i) : 0;
      n += v[j] == 0xFF;
    }
    int s = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += u;
    }
    if (lane == 31) wsum[warp] = s;
    __syncthreads();
    int before = s - n;
    for (int w = 0; w < warp; ++w) before += wsum[w];
    long long d = carry_s + (i0 - b0) + 4 * threadIdx.x + before;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (i0 + 4 * threadIdx.x + j < b1) {
        out[d++] = static_cast<uint8_t>(v[j]);
        if (v[j] == 0xFF) out[d++] = 0;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < 8; ++w) tot += wsum[w];
      carry_s += tot;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ host side
// ITU-T T.81 Annex K tables
const uint8_t kLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                            14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                            18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                            49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const uint8_t kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                              99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                              99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const uint8_t kZigzagHost[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
const uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
const uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D};
const uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16,
    0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6,
    0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8,
    0xD9, 0xDA, 0xE1, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA};
const uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
const uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34,
    0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8A, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4,
    0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6,
    0xD7, 0xD8, 0xD9, 0xDA, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA};

// canonical code assignment (T.81 Annex C): (code << 5) | length per symbol
void huff_codes(const uint8_t* bits, const uint8_t* vals, uint32_t* table) {
  uint32_t code = 0;
  int k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < bits[len - 1]; ++i, ++k, ++code) table[vals[k]] = (code << 5) | len;
    code <<= 1;
  }
}

void put_marker(std::vector<uint8_t>& h, uint8_t code, const std::vector<uint8_t>& payload) {
  const size_t n = payload.size() + 2;
  h.insert(h.end(), {0xFF, code, static_cast<uint8_t>(n >> 8), static_cast<uint8_t>(n)});
  h.insert(h.end(), payload.begin(), payload.end());
}

// quality (0..100, 0 as 1) -> 8 x table entries (natural order), the header with a 0 x 0 SOF0 size, the code tables
void fill_tables(int quality, JpegParams& p) {
  const int q = std::min(std::max(quality, 1), 100);
  const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
  uint8_t qt[2][64];
  for (int i = 0; i < 64; ++i) {
    qt[0][i] = static_cast<uint8_t>(std::min(std::max((kLumaQ[i] * scale + 50) / 100, 1), 255));
    qt[1][i] = static_cast<uint8_t>(std::min(std::max((kChromaQ[i] * scale + 50) / 100, 1), 255));
    p.qdiv[0][i] = static_cast<uint16_t>(qt[0][i] * 8);
    p.qdiv[1][i] = static_cast<uint16_t>(qt[1][i] * 8);
  }
  std::memset(&p.huff, 0, sizeof(p.huff));
  huff_codes(kDcLumaBits, kDcVals, p.huff.dc[0]);
  huff_codes(kDcChromaBits, kDcVals, p.huff.dc[1]);
  huff_codes(kAcLumaBits, kAcLumaVals, p.huff.ac[0]);
  huff_codes(kAcChromaBits, kAcChromaVals, p.huff.ac[1]);
  std::vector<uint8_t> h = {0xFF, 0xD8};
  put_marker(h, 0xE0, {'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});
  for (int t = 0; t < 2; ++t) {
    std::vector<uint8_t> d = {static_cast<uint8_t>(t)};
    for (int i = 0; i < 64; ++i) d.push_back(qt[t][kZigzagHost[i]]);
    put_marker(h, 0xDB, d);
  }
  put_marker(h, 0xC0, {8, 0, 0, 0, 0, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
  const uint8_t* bits[4] = {kDcLumaBits, kAcLumaBits, kDcChromaBits, kAcChromaBits};
  const uint8_t* vals[4] = {kDcVals, kAcLumaVals, kDcVals, kAcChromaVals};
  const uint8_t cls[4] = {0x00, 0x10, 0x01, 0x11};
  for (int i = 0; i < 4; ++i) {
    std::vector<uint8_t> d = {cls[i]};
    int n = 0;
    for (int l = 0; l < 16; ++l) { d.push_back(bits[i][l]); n += bits[i][l]; }
    d.insert(d.end(), vals[i], vals[i] + n);
    put_marker(h, 0xC4, d);
  }
  put_marker(h, 0xDA, {3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
  std::memcpy(p.header, h.data(), kHeaderBytes);
}

struct Geo {
  int mw, mh;
  long long nmcu() const { return static_cast<long long>(mw) * mh; }
  long long words() const { return (nmcu() * 6 * kMaxBlockBits + 31) / 32 + 1; }
  long long bound() const { return kHeaderBytes + 2 * ((nmcu() * 6 * kMaxBlockBits + 7) / 8 + 1) + 2; }
};
Geo geo(int w, int h) { return Geo{(w + 15) / 16, (h + 15) / 16}; }

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// Workspace layout of one launch group of crops
struct Layout {
  long long n_mcu = 0, n_tile = 0, words = 0;
  size_t coef, blen, tbits, tff, cbits, wordsb, total;
};
Layout layout(const int32_t* rects, int k0, int n, bool with_coef) {
  Layout L;
  for (int i = 0; i < n; ++i) {
    const int32_t* r = rects + 5 * (k0 + i);
    const Geo g = geo(r[3] - r[1], r[4] - r[2]);
    L.n_mcu += g.nmcu();
    L.n_tile += (g.nmcu() + kTileMcus - 1) / kTileMcus;
    L.words += g.words();
  }
  size_t off = 0;
  L.coef = off; off += with_coef ? align256(static_cast<size_t>(L.n_mcu) * 6 * 64 * 2) : 0;
  L.blen = off; off += align256(static_cast<size_t>(L.n_mcu) * 6 * 4);
  L.tbits = off; off += align256(static_cast<size_t>(L.n_tile) * 8);
  L.tff = off; off += align256(static_cast<size_t>(L.n_tile) * 8);
  L.cbits = off; off += align256(static_cast<size_t>(n) * 8);
  L.wordsb = off; off += align256(static_cast<size_t>(L.words) * 4);
  L.total = off;
  return L;
}

// the crop table of crops [k0, k0 + n); with_coef: coefficients at d_coef (the tap) instead of the workspace
void fill_params(JpegParams& p, TransformParams& t, const CropSource* src, const int32_t* rects, int k0, int n, uint8_t* ws,
                 const Layout& L, int16_t* d_coef, uint8_t* d_out, const int64_t* out_offsets, int64_t* d_lengths) {
  p.K = n;
  p.n_mcu = static_cast<int>(L.n_mcu); p.n_tile = static_cast<int>(L.n_tile);
  p.coef = d_coef ? d_coef : reinterpret_cast<int16_t*>(ws + L.coef);
  p.blen = reinterpret_cast<uint32_t*>(ws + L.blen);
  p.tbits = reinterpret_cast<unsigned long long*>(ws + L.tbits);
  p.tff = reinterpret_cast<unsigned long long*>(ws + L.tff);
  p.cbits = reinterpret_cast<unsigned long long*>(ws + L.cbits);
  p.words = reinterpret_cast<uint32_t*>(ws + L.wordsb);
  p.out = d_out;
  p.lengths = reinterpret_cast<long long*>(d_lengths);
  t.K = n; t.coef = p.coef;
  std::memcpy(t.qdiv, p.qdiv, sizeof(t.qdiv));
  int mcu = 0, tile = 0, zero = 0;
  long long word = 0;
  for (int i = 0; i < n; ++i) {
    const int32_t* r = rects + 5 * (k0 + i);
    JpegCrop& c = p.crop[i];
    c.x1 = r[1]; c.y1 = r[2]; c.w = r[3] - r[1]; c.h = r[4] - r[2];
    const Geo g = geo(c.w, c.h);
    c.mw = g.mw; c.nmcu = static_cast<int>(g.nmcu());
    c.mcu0 = mcu; c.tile0 = tile; c.ntile = (c.nmcu + kTileMcus - 1) / kTileMcus; c.zero0 = zero;
    c.word0 = word;
    c.out = out_offsets ? out_offsets[k0 + i] : 0;
    t.crop[i] = TransformCrop{src[k0 + i], c.x1, c.y1, c.w, c.h, c.mw, c.mcu0};
    mcu += c.nmcu; tile += c.ntile; word += g.words();
    zero += static_cast<int>((g.words() + kZeroWords - 1) / kZeroWords);
  }
}

int total_zero_ctas(const JpegParams& p) {
  const JpegCrop& c = p.crop[p.K - 1];
  const long long w = geo(c.w, c.h).words();
  return c.zero0 + static_cast<int>((w + kZeroWords - 1) / kZeroWords);
}

// cc_jpeg_encode_crops_frames from the point where the crops' sources and rects are checked
int encode_sources(const char* who, const CropSource* src, const int32_t* rects, int K, int quality, uint8_t* d_out,
                   int64_t out_bytes, const int64_t* out_offsets, int64_t* d_lengths, void* d_workspace, size_t ws_bytes,
                   size_t* ws_needed, void* stream) {
  size_t need = 0;
  for (int k0 = 0; k0 < K; k0 += kCropsPerLaunch)
    need = std::max(need, layout(rects, k0, std::min(K - k0, kCropsPerLaunch), true).total);
  if (ws_needed) *ws_needed = need;
  if (!d_out) return CC_OK;                      // workspace size query
  CC_REQUIRE(out_offsets && d_lengths, "%s: out_offsets and d_lengths must not be NULL", who);
  CC_REQUIRE(need == 0 || (d_workspace && ws_bytes >= need), "%s: workspace of %zu bytes too small (%zu needed)", who,
             d_workspace ? ws_bytes : size_t(0), need);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0 && (reinterpret_cast<uintptr_t>(d_lengths) & 7) == 0,
             "%s: d_workspace must be 256-byte aligned and d_lengths 8-byte aligned", who);
  // each crop's region [offset, offset + bound) inside d_out, no two overlapping
  std::vector<std::pair<int64_t, int64_t>> regions(K);
  for (int k = 0; k < K; ++k) {
    const int32_t* r = rects + 5 * k;
    const int64_t b = geo(r[3] - r[1], r[4] - r[2]).bound();
    CC_REQUIRE(out_offsets[k] >= 0 && out_offsets[k] <= out_bytes - b,
               "%s: crop %d at offset %lld with bound %lld exceeds the output capacity of %lld bytes", who, k,
               static_cast<long long>(out_offsets[k]), static_cast<long long>(b), static_cast<long long>(out_bytes));
    regions[k] = {out_offsets[k], b};
  }
  std::vector<int> order(K);
  for (int k = 0; k < K; ++k) order[k] = k;
  std::sort(order.begin(), order.end(), [&](int a, int b) { return regions[a].first < regions[b].first; });
  for (int i = 1; i < K; ++i)
    CC_REQUIRE(regions[order[i - 1]].first + regions[order[i - 1]].second <= regions[order[i]].first,
               "%s: the output regions of crops %d and %d overlap (offset + cc_jpeg_bound)", who, order[i - 1], order[i]);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  static thread_local JpegParams p;              // ~17 KB of kernel parameters, kept off the stack
  static thread_local TransformParams t;         // ~12 KB
  fill_tables(quality, p);
  for (int k0 = 0; k0 < K; k0 += kCropsPerLaunch) {
    const int n = std::min(K - k0, kCropsPerLaunch);
    const Layout L = layout(rects, k0, n, true);
    fill_params(p, t, src, rects, k0, n, static_cast<uint8_t*>(d_workspace), L, nullptr, d_out, out_offsets, d_lengths);
    jpeg_transform_kernel<<<p.n_mcu, 256, 0, st>>>(t);
    jpeg_lengths_kernel<<<p.n_tile, 256, 0, st>>>(p);
    jpeg_scan_kernel<<<1, 1024, 0, st>>>(p, 0, k0);
    jpeg_zero_kernel<<<total_zero_ctas(p), 256, 0, st>>>(p);
    jpeg_pack_kernel<<<p.n_tile, 256, 0, st>>>(p);
    jpeg_count_kernel<<<p.n_tile, 256, 0, st>>>(p);
    jpeg_scan_kernel<<<1, 1024, 0, st>>>(p, 1, k0);
    jpeg_scatter_kernel<<<p.n_tile, 256, 0, st>>>(p, k0);
    CC_CHECK_CUDA(cudaGetLastError());
  }
  return CC_OK;
}

}  // namespace

int table_crop_sources(const char* who, const cc_frame* frames, int n_frames, const int32_t* rects, int K, CropSource* src) {
  CC_REQUIRE(frames && (rects || K == 0), "%s: null pointer", who);
  CC_REQUIRE(n_frames > 0 && K >= 0, "%s: bad sizes n_frames=%d K=%d", who, n_frames, K);
  for (int i = 0; i < n_frames; ++i) {
    const cc_frame& f = frames[i];
    CC_REQUIRE(f.data, "%s: frame %d is NULL", who, i);
    CC_REQUIRE(f.fmt == CC_FRAME_BGR_U8 || f.fmt == CC_FRAME_I420_U8 || f.fmt == CC_FRAME_RGB_U8,
               "%s: frame %d has format %d: unknown source format %d for a crop (CC_FRAME_BGR_U8 0, CC_FRAME_I420_U8 2 or "
               "CC_FRAME_RGB_U8 3)", who, i, f.fmt, f.fmt);
    CC_REQUIRE(f.h > 0 && f.w > 0, "%s: frame %d has a bad size %dx%d", who, i, f.w, f.h);
    CC_REQUIRE(f.fmt != CC_FRAME_I420_U8 || (f.h % 2 == 0 && f.w % 2 == 0),
               "%s: frame %d: an I420 frame needs an even height and width, got %dx%d", who, i, f.w, f.h);
  }
  for (int k = 0; k < K; ++k) {
    const int32_t* r = rects + 5 * k;
    CC_REQUIRE(r[0] >= 0 && r[0] < n_frames, "%s: rect %d names frame %d of a %d-frame table", who, k, r[0], n_frames);
    const cc_frame& f = frames[r[0]];
    CC_REQUIRE(r[1] >= 0 && r[2] >= 0 && r[3] > r[1] && r[4] > r[2] && r[3] <= f.w && r[4] <= f.h,
               "%s: rect %d (frame %d, %d,%d-%d,%d) is empty or outside its %dx%d frame", who, k, r[0], r[1], r[2], r[3], r[4],
               f.w, f.h);
    const int fmt = f.fmt == CC_FRAME_RGB_U8 ? 0 : f.fmt == CC_FRAME_BGR_U8 ? 1 : 2;
    src[k] = CropSource{static_cast<const uint8_t*>(f.data), f.h, f.w, fmt};
  }
  return CC_OK;
}

int check_table_jpeg(const char* who, const int32_t* rects, int K, int quality) {
  CC_REQUIRE(quality >= 0 && quality <= 100, "%s: quality %d outside 0..100", who, quality);
  for (int k = 0; k < K; ++k)
    CC_REQUIRE(rects[5 * k + 3] - rects[5 * k + 1] <= kMaxSide && rects[5 * k + 4] - rects[5 * k + 2] <= kMaxSide,
               "%s: rect %d is larger than %d pixels", who, k, kMaxSide);
  return CC_OK;
}

int jpeg_coeffs_sources(const CropSource* src, const int32_t* rects, int K, int quality, int16_t* d_coef, int64_t* n_blocks,
                        cudaStream_t st) {
  long long blocks = 0;
  for (int k = 0; k < K; ++k) blocks += geo(rects[5 * k + 3] - rects[5 * k + 1], rects[5 * k + 4] - rects[5 * k + 2]).nmcu() * 6;
  if (n_blocks) *n_blocks = blocks;
  if (!d_coef) return CC_OK;                     // size query
  static thread_local JpegParams p;
  static thread_local TransformParams t;
  fill_tables(quality, p);
  long long done = 0;
  for (int k0 = 0; k0 < K; k0 += kCropsPerLaunch) {
    const int n = std::min(K - k0, kCropsPerLaunch);
    const Layout L = layout(rects, k0, n, false);
    fill_params(p, t, src, rects, k0, n, nullptr, L, d_coef + done * 64, nullptr, nullptr, nullptr);
    jpeg_transform_kernel<<<p.n_mcu, 256, 0, st>>>(t);
    CC_CHECK_CUDA(cudaGetLastError());
    done += L.n_mcu * 6;
  }
  return CC_OK;
}

// the quantisation tables the encoder writes for `quality` (natural order): what a decoder of its files dequantises with
void jpeg_quant_tables(int quality, uint16_t qt[2][64]) {
  static thread_local JpegParams p;
  fill_tables(quality, p);
  for (int t = 0; t < 2; ++t)
    for (int i = 0; i < 64; ++i) qt[t][i] = static_cast<uint16_t>(p.qdiv[t][i] / 8);
}

}  // namespace cc

using namespace cc;

extern "C" int cc_jpeg_bound(int w, int h, int64_t* bytes) {
  CC_REQUIRE(bytes != nullptr, "cc_jpeg_bound: bytes is NULL");
  CC_REQUIRE(w >= 1 && h >= 1 && w <= kMaxSide && h <= kMaxSide, "cc_jpeg_bound: bad size %dx%d (1..%d)", w, h, kMaxSide);
  *bytes = geo(w, h).bound();
  return CC_OK;
}

extern "C" int cc_jpeg_encode_crops_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int quality,
                                           uint8_t* d_out, int64_t out_bytes, const int64_t* out_offsets, int64_t* d_lengths,
                                           void* d_workspace, size_t ws_bytes, size_t* ws_needed, void* stream) {
  const char* who = "cc_jpeg_encode_crops_frames";
  std::vector<CropSource> src(std::max(K, 0));
  if (int rc = table_crop_sources(who, frames, n_frames, rects, K, src.data())) return rc;
  if (int rc = check_table_jpeg(who, rects, K, quality)) return rc;
  return encode_sources(who, src.data(), rects, K, quality, d_out, out_bytes, out_offsets, d_lengths, d_workspace, ws_bytes,
                        ws_needed, stream);
}

extern "C" int cc_jpeg_coeffs_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int quality,
                                     int16_t* d_coef, int64_t* n_blocks, void* stream) {
  const char* who = "cc_jpeg_coeffs_frames";
  std::vector<CropSource> src(std::max(K, 0));
  if (int rc = table_crop_sources(who, frames, n_frames, rects, K, src.data())) return rc;
  if (int rc = check_table_jpeg(who, rects, K, quality)) return rc;
  jpeg_coeffs_sources(src.data(), rects, K, quality, nullptr, n_blocks, nullptr);
  if (!d_coef) return CC_OK;                     // size query
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_coef) & 3) == 0, "%s: d_coef must be 4-byte aligned", who);
  return jpeg_coeffs_sources(src.data(), rects, K, quality, d_coef, nullptr, static_cast<cudaStream_t>(stream));
}
