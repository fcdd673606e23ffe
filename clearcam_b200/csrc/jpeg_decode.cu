// Baseline / extended-sequential Huffman JPEG -> BGR uint8 on the device, pixel for pixel what cv2.imdecode(buf,
// IMREAD_COLOR) returns (OpenCV 4.13 with libjpeg-turbo 3.1: islow inverse DCT, fancy upsampling, table-driven YCbCr ->
// BGR).  oracle/jpeg_decode.py states the arithmetic and is pinned to cv2; everything here is integer code restating it.
//
// Replaces the host decodes of the reference's thumbnail reads (clearcam.py:272-279 cv2.imread before clip_latest_img,
// run_clip's preprocess_clip for search by image, models/objects.py:244-251).
//
// cc_jpeg_parse (host) reads the markers of K files into a per-image table: sizes, sampling, quantisation tables, Huffman
// lookup tables, restart interval, the scan's place in the data, and where each image's intermediates go in the workspace.
// Files the device does not decode get a status (unsupported or corrupt) there and are left to the caller.
// cc_jpeg_decode then runs, on the caller's stream, with no allocation and no host sync:
//   1. status     the table's status per image into d_status
//   2. count      per 1 KB chunk of scan data: bytes kept after removing FF 00 stuffing, fill bytes and RSTn markers
//   3. scan       per image (a warp): chunk offsets; interval bounds; wrong RSTn count -> corrupt
//   4. scatter    destuffed bytes to the image's buffer; each RSTn's position is the next interval's start
//   5. layout     per image: every restart interval cut into subsequences of kSubBits bits
//   6. sync       self-synchronising decode (Weissenberger & Schmidt, ICPP 2018 / HiPC 2021), one cooperative launch: a
//                 thread per subsequence decodes from a guessed state (bit position, block of the MCU, zigzag index) to its
//                 end; the threads of a CTA then take their predecessor's end state as their start and decode again until
//                 nothing changes; passes over all tiles, each reading the tile edges of the pass before, repeat the same
//                 across CTA boundaries until a pass changes nothing
//   8. counts     per interval (a warp): every start equals its predecessor's end (guaranteed by 6; checked, and an image
//                 that failed it would be left to the host as unsupported),
//                 exclusive scan of the blocks completed per subsequence -> each subsequence's first block; too few blocks
//                 -> corrupt
//   9. write      from the synchronised states, every coefficient to its block (int16, zigzag; DC as a difference)
//  10. dc         DC differences -> values per component: per chunk of 256 MCUs (a warp) the sums, then each chunk adds
//                 the sums before it in its interval and scans its MCUs
//  11. idct       per block: dequantise, islow IDCT, range limit -> the component's sample plane
//  12. pixels     per output pixel: fancy upsampling of the chroma planes, YCbCr -> BGR into the padded batch
// Kernels 11 and 12 also turn the encoder's quantised coefficients of object crops into the pixels of their JPEG files
// (cc_jpeg_crops_decoded), with no entropy coding in between.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>
#include <algorithm>
#include <climits>

#include "cc_common.h"
#include "clearcam_b200.h"
#include "ops.cuh"

#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace cc {
void jpeg_quant_tables(int quality, uint16_t qt[2][64]);   // jpeg.cu

namespace {

constexpr int kChunk = 1024;            // scan bytes per CTA of the destuffing kernels (256 threads x 4)
constexpr int kSubBits = 256;           // bits per self-synchronising subsequence
constexpr int kSyncCta = 128;           // subsequences per CTA of the sync kernels
constexpr int kReconPerLaunch = 128;    // images per launch of the reconstruction kernels
constexpr int kDcChunk = 256;           // MCUs per warp of the DC passes

struct HuffDev {
  uint16_t look[512];                   // next 9 bits -> (length << 8) | symbol; length 0: the code is longer
  int32_t maxcode[18];                  // largest code of each length, -1 if none
  int32_t valoff[18];                   // index of a code's symbol = code + valoff[length]
  uint8_t vals[256];
};

struct JpegImage {
  int32_t status, w, h, ncomp, hs, vs, mcux, mcuy, bpm, ri, nint, nchunk;
  int8_t blk_dc[8], blk_ac[8], blk_comp[8];
  long long scan_off, scan_len;
  long long chunk0, dst0, iv0, sub0, nsub_max, blk0, plane0;
  uint16_t qt[3][64];                   // per component, natural order
  HuffDev dc[4], ac[4];
};

__constant__ uint8_t kDeZigzag[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
                                      41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
                                      46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};

struct JdecParams {
  const uint8_t* data;
  const JpegImage* tab;
  int K;
  int32_t* status;
  int32_t* chunk_kept;                  // [chunks], then exclusive offsets within the image
  int32_t* chunk_rst;
  int32_t* dlen;                        // [K] destuffed bytes
  uint8_t* dbuf;                        // destuffed scan data
  int32_t* ivstart;                     // [intervals + K]: byte offset of each interval, then the end
  int32_t* subbase;                     // [intervals + K]: first subsequence of each interval, then the total
  unsigned long long* st;               // [slots] start state of each subsequence
  unsigned long long* en;               // [slots] end state
  int32_t* cnt;                         // [slots] blocks completed
  int32_t* err;                         // [slots] blocks completed before the first invalid code, INT_MAX if none
  unsigned long long* edge;             // [2][tiles] end state of each sync tile's last subsequence, by pass parity
  int32_t* flag;                        // [3] "a tile changed" per pass, by pass mod 3
  int32_t* bbase;                       // [slots] first block (relative to the image)
  int32_t* dcsum;                       // [intervals][dc_chunks][3] DC difference sums per chunk of kDcChunk MCUs
  int16_t* coef;
  long long n_chunk, n_iv, n_slot;
  int dc_chunks;                        // chunks of the longest interval
};

template <typename F>
__device__ __forceinline__ int find_image(const JdecParams& p, long long i, F key) {
  int lo = 0, hi = p.K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (key(p.tab[mid]) <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------------ 1-5. destuffing
__global__ void jdec_status_kernel(const __grid_constant__ JdecParams p) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < p.K) p.status[k] = p.tab[k].status;
}

// byte i of a scan of n bytes: kept (data), and whether it is an RSTn code byte
__device__ __forceinline__ void classify(const uint8_t* s, long long n, long long i, bool& kept, bool& rst) {
  const int c = s[i];
  const int prev = i > 0 ? s[i - 1] : -1, next = i + 1 < n ? s[i + 1] : -1;
  kept = true; rst = false;
  if (c == 0xFF && next != 0x00) kept = false;                         // fill byte or a marker's prefix
  else if (prev == 0xFF && c != 0xFF) { kept = false; rst = c != 0x00; }  // stuffed zero, or RSTn
}

__global__ void __launch_bounds__(256) jdec_count_kernel(const __grid_constant__ JdecParams p) {
  __shared__ int sk[8], sr[8];
  const long long c = blockIdx.x;
  const int k = find_image(p, c, [](const JpegImage& t) { return t.chunk0; });
  const JpegImage& im = p.tab[k];
  int kept = 0, rst = 0;
  if (c < im.chunk0 + im.nchunk) {
    const uint8_t* s = p.data + im.scan_off;
    const long long b0 = (c - im.chunk0) * kChunk;
    for (int j = 0; j < 4; ++j) {
      const long long i = b0 + threadIdx.x * 4 + j;
      if (i >= im.scan_len) break;
      bool kk, rr;
      classify(s, im.scan_len, i, kk, rr);
      kept += kk; rst += rr;
    }
  }
  for (int o = 16; o; o >>= 1) { kept += __shfl_xor_sync(~0u, kept, o); rst += __shfl_xor_sync(~0u, rst, o); }
  if ((threadIdx.x & 31) == 0) { sk[threadIdx.x >> 5] = kept; sr[threadIdx.x >> 5] = rst; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0, b = 0;
    for (int w = 0; w < 8; ++w) { a += sk[w]; b += sr[w]; }
    p.chunk_kept[c] = a; p.chunk_rst[c] = b;
  }
}

__device__ __forceinline__ int warp_excl(int v, int lane, int& total) {
  int s = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(~0u, s, o);
    if (lane >= o) s += u;
  }
  total = __shfl_sync(~0u, s, 31);
  return s - v;
}

__global__ void jdec_scan_kernel(const __grid_constant__ JdecParams p) {
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= p.K) return;
  const JpegImage& im = p.tab[k];
  if (im.status != CC_JPEG_OK) return;
  int ck = 0, cr = 0;
  for (int i0 = 0; i0 < im.nchunk; i0 += 32) {
    const int i = i0 + lane;
    const int a = i < im.nchunk ? p.chunk_kept[im.chunk0 + i] : 0, b = i < im.nchunk ? p.chunk_rst[im.chunk0 + i] : 0;
    int ta, tb;
    const int ea = warp_excl(a, lane, ta), eb = warp_excl(b, lane, tb);
    if (i < im.nchunk) { p.chunk_kept[im.chunk0 + i] = ck + ea; p.chunk_rst[im.chunk0 + i] = cr + eb; }
    ck += ta; cr += tb;
  }
  if (lane == 0) {
    p.dlen[k] = ck;
    p.ivstart[im.iv0 + k] = 0;
    p.ivstart[im.iv0 + k + im.nint] = ck;
    if (cr != im.nint - 1) p.status[k] = CC_JPEG_CORRUPT;
  }
}

__global__ void __launch_bounds__(256) jdec_scatter_kernel(const __grid_constant__ JdecParams p) {
  __shared__ int sk[8], sr[8];
  const long long c = blockIdx.x;
  const int k = find_image(p, c, [](const JpegImage& t) { return t.chunk0; });
  const JpegImage& im = p.tab[k];
  if (c >= im.chunk0 + im.nchunk || im.status != CC_JPEG_OK) return;
  const uint8_t* s = p.data + im.scan_off;
  const long long b0 = (c - im.chunk0) * kChunk;
  bool kk[4], rr[4];
  int kept = 0, rst = 0;
  for (int j = 0; j < 4; ++j) {
    const long long i = b0 + threadIdx.x * 4 + j;
    kk[j] = rr[j] = false;
    if (i < im.scan_len) classify(s, im.scan_len, i, kk[j], rr[j]);
    kept += kk[j]; rst += rr[j];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int tk, tr;
  int ek = warp_excl(kept, lane, tk), er = warp_excl(rst, lane, tr);
  if (lane == 0) { sk[warp] = tk; sr[warp] = tr; }
  __syncthreads();
  for (int w = 0; w < warp; ++w) { ek += sk[w]; er += sr[w]; }
  long long o = p.chunk_kept[c] + ek;
  int r = p.chunk_rst[c] + er;
  for (int j = 0; j < 4; ++j) {
    const long long i = b0 + threadIdx.x * 4 + j;
    if (kk[j]) p.dbuf[im.dst0 + o++] = s[i];
    if (rr[j]) {
      if (s[i] != 0xD0 + (r & 7) || r >= im.nint - 1) p.status[k] = CC_JPEG_CORRUPT;
      else p.ivstart[im.iv0 + k + r + 1] = static_cast<int32_t>(o);
      ++r;
    }
  }
}

__global__ void jdec_layout_kernel(const __grid_constant__ JdecParams p) {
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= p.K) return;
  const JpegImage& im = p.tab[k];
  if (im.status != CC_JPEG_OK) return;
  const int32_t* iv = p.ivstart + im.iv0 + k;
  int32_t* sb = p.subbase + im.iv0 + k;
  int carry = 0;
  for (int j0 = 0; j0 < im.nint; j0 += 32) {
    const int j = j0 + lane;
    int n = 0;
    if (j < im.nint) {
      const long long bits = 8ll * (iv[j + 1] - iv[j]);
      n = static_cast<int>(std::max(1ll, (bits + kSubBits - 1) / kSubBits));
    }
    int tot;
    const int e = warp_excl(n, lane, tot);
    if (j < im.nint) sb[j] = carry + e;
    carry += tot;
  }
  if (lane == 0) sb[im.nint] = carry;
}

// ------------------------------------------------------------------------------------------------ 6-9. entropy decode
struct Slot {
  int k, j, q;                          // image, interval, subsequence within the interval (-1: no work)
  long long lo, hi, end;                // the image's destuffed data; subsequence end bit; interval end bit
};

__device__ __forceinline__ Slot slot_of(const JdecParams& p, long long g) {
  Slot s{-1, 0, 0, 0, 0, 0};
  if (g >= p.n_slot) return s;
  const int k = find_image(p, g, [](const JpegImage& t) { return t.sub0; });
  const JpegImage& im = p.tab[k];
  if (p.status[k] != CC_JPEG_OK) return s;
  const int32_t* sb = p.subbase + im.iv0 + k;
  const long long loc = g - im.sub0;
  if (loc >= sb[im.nint]) return s;
  int lo = 0, hi = im.nint - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sb[mid] <= loc) lo = mid; else hi = mid - 1;
  }
  const int32_t* iv = p.ivstart + im.iv0 + k;
  s.k = k; s.j = lo; s.q = static_cast<int>(loc - sb[lo]);
  const long long b0 = 8ll * iv[lo];
  s.end = 8ll * iv[lo + 1];
  s.hi = std::min(b0 + static_cast<long long>(s.q + 1) * kSubBits, s.end);
  s.lo = b0 + static_cast<long long>(s.q) * kSubBits;
  return s;
}

__device__ __forceinline__ unsigned long long pack_state(long long pos, int blk, int zz) {
  return (static_cast<unsigned long long>(pos) << 16) | (static_cast<unsigned>(blk) << 8) | static_cast<unsigned>(zz);
}

// 32 bits of the destuffed buffer from bit `pos`, zeros past `nbytes`
__device__ __forceinline__ uint32_t peek32(const uint8_t* b, long long nbytes, long long pos) {
  const long long i = pos >> 3;
  uint64_t v = 0;
#pragma unroll
  for (int j = 0; j < 5; ++j) v = (v << 8) | (i + j < nbytes ? b[i + j] : 0u);
  return static_cast<uint32_t>(v >> (8 - (pos & 7)));
}

__device__ __forceinline__ int huff_decode(const HuffDev& t, uint32_t w16, int& len) {
  const int e = t.look[w16 >> 7];
  if (e >> 8) { len = e >> 8; return e & 255; }
  for (int l = 10; l <= 16; ++l) {
    const int code = static_cast<int>(w16 >> (16 - l));
    if (code <= t.maxcode[l]) { len = l; return t.vals[(code + t.valoff[l]) & 255]; }
  }
  len = 0;
  return 0;
}

// Decode symbols from `state` while the position is below `stop`; a symbol must end by `end` (the interval's last bit:
// one that would not stops the decode there).  Counts the blocks completed; `err` = the blocks completed before the first
// invalid code (INT_MAX if none), after which decoding goes on one bit later from block 0, zigzag 0 (a guessed state meets
// invalid codes; on the synchronised chain one is corruption).  With WRITE, stores the coefficients of blocks [0, limit) at
// coef (block 0 = the first block completed or continued here).  Returns the end state.
template <bool WRITE>
__device__ unsigned long long run(const JpegImage& im, const uint8_t* b, long long nbytes, unsigned long long state, long long stop,
                                  long long end, int& done, int& err, int16_t* coef = nullptr, int limit = 0) {
  done = 0;
  err = INT_MAX;
  long long pos = static_cast<long long>(state >> 16);
  int blk = (state >> 8) & 255, zz = state & 255;
  while (pos < stop) {
    if (WRITE && done >= limit) break;
    const uint32_t w = peek32(b, nbytes, pos);
    const HuffDev& t = zz == 0 ? im.dc[im.blk_dc[blk]] : im.ac[im.blk_ac[blk]];
    int L;
    const int sym = huff_decode(t, w >> 16, L);
    if (!L) {
      err = min(err, done);
      pos += 1; blk = 0; zz = 0;
      continue;
    }
    const int s = zz == 0 ? sym : sym & 15, r = zz == 0 ? 0 : sym >> 4;
    if (pos + L + s > end) return pack_state(end, blk, zz);
    int v = 0;
    if (s) {
      const int x = static_cast<int>((w << L) >> (32 - s));
      v = x < (1 << (s - 1)) ? x - (1 << s) + 1 : x;
    }
    pos += L + s;
    if (zz == 0) {
      if (WRITE) coef[static_cast<long long>(done) * 64] = static_cast<int16_t>(v);
      zz = 1;
    } else if (s) {
      zz += r;
      if (WRITE) coef[static_cast<long long>(done) * 64 + min(zz, 63)] = static_cast<int16_t>(v);
      zz += 1;
    } else if (r == 15) {
      zz += 16;
    } else {
      zz = 64;
    }
    if (zz >= 64) {
      zz = 0;
      blk = blk + 1 < im.bpm ? blk + 1 : 0;
      ++done;
    }
  }
  return pack_state(pos, blk, zz);
}

__device__ __forceinline__ const uint8_t* dbuf_of(const JdecParams& p, int k, long long& nbytes) {
  nbytes = p.dlen[k];
  return p.dbuf + p.tab[k].dst0;
}

// One tile of kSyncCta subsequences.  first: every subsequence decodes from its guess; otherwise the tile's first
// subsequence takes its predecessor's end state from the previous pass (edge_in) and the tile only works if that changed.
// Then CTA-wide rounds give each subsequence its predecessor's end state as its start and decode again until nothing
// changes.  Returns whether anything changed; edge_out gets the end state of the tile's last subsequence.
__device__ bool sync_tile(const JdecParams& p, long long tile, bool first, const unsigned long long* edge_in,
                          unsigned long long* edge_out, unsigned long long* sen, int* again) {
  const long long g = tile * kSyncCta + threadIdx.x;
  const Slot s = slot_of(p, g);
  const int t = threadIdx.x;
  long long nbytes = 0;
  const uint8_t* b = s.k >= 0 ? dbuf_of(p, s.k, nbytes) : nullptr;
  const JpegImage* im = s.k >= 0 ? &p.tab[s.k] : nullptr;
  int done = 0, err = INT_MAX;
  unsigned long long st = 0, en = 0;
  bool any = first;
  if (first) {
    if (s.k >= 0) {
      st = pack_state(s.lo, 0, 0);
      en = run<false>(*im, b, nbytes, st, s.hi, s.end, done, err);
    }
  } else {
    if (s.k >= 0) { st = p.st[g]; en = p.en[g]; done = p.cnt[g]; err = p.err[g]; }
    if (t == 0) *again = s.k >= 0 && s.q > 0 && edge_in[tile - 1] != st;
    __syncthreads();
    any = *again;
    if (any && t == 0) {
      st = edge_in[tile - 1];
      en = run<false>(*im, b, nbytes, st, s.hi, s.end, done, err);
    }
  }
  if (any) {
    sen[t] = en;
    __syncthreads();
    for (int round = 0; round < kSyncCta; ++round) {
      bool changed = false;
      if (s.k >= 0 && s.q > 0 && t > 0 && sen[t - 1] != st) {
        st = sen[t - 1];
        changed = true;
      }
      __syncthreads();
      if (changed) {
        en = run<false>(*im, b, nbytes, st, s.hi, s.end, done, err);
        sen[t] = en;
      }
      if (!__syncthreads_or(changed)) break;
    }
    if (s.k >= 0) { p.st[g] = st; p.en[g] = en; p.cnt[g] = done; p.err[g] = err; }
  }
  if (t == kSyncCta - 1) edge_out[tile] = en;
  __syncthreads();                                    // sen / again are reused by the CTA's next tile
  return any;
}

// Cooperative (persistent) launch: pass 0 synchronises every tile from its guesses; each further pass starts every tile
// from its predecessor's end state of the pass before (double-buffered, so a pass reads nothing written in the same pass
// and the result does not depend on scheduling), until a pass changes nothing.  After pass r every chain of r tiles is
// exact, so the loop ends; a wrong guess usually falls into step within a few subsequences, so one or two passes do.
__global__ void __launch_bounds__(kSyncCta) jdec_sync_kernel(const __grid_constant__ JdecParams p) {
  __shared__ unsigned long long sen[kSyncCta];
  __shared__ int again;
  cg::grid_group grid = cg::this_grid();
  const long long ntile = (p.n_slot + kSyncCta - 1) / kSyncCta;
  for (int pass = 0;; ++pass) {
    if (blockIdx.x == 0 && threadIdx.x == 0) p.flag[(pass + 1) % 3] = 0;     // last read two passes ago
    bool changed = false;
    for (long long tile = blockIdx.x; tile < ntile; tile += gridDim.x)
      changed |= sync_tile(p, tile, pass == 0, p.edge + ((pass + 1) & 1) * ntile, p.edge + (pass & 1) * ntile, sen, &again);
    if (pass > 0 && changed && threadIdx.x == 0) atomicExch(p.flag + pass % 3, 1);
    grid.sync();
    if (pass > 0 && atomicAdd(p.flag + pass % 3, 0) == 0) break;
  }
}

__device__ __forceinline__ int interval_blocks(const JpegImage& im, int j) {
  const int nmcu = im.mcux * im.mcuy;
  const int ri = im.ri ? im.ri : nmcu;
  return std::min(ri, nmcu - j * ri) * im.bpm;
}

// warp per interval: synchronisation check and the first block of every subsequence
__global__ void jdec_counts_kernel(const __grid_constant__ JdecParams p) {
  const long long gi = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gi >= p.n_iv) return;
  const int k = find_image(p, gi, [](const JpegImage& t) { return t.iv0; });
  const JpegImage& im = p.tab[k];
  const int j = static_cast<int>(gi - im.iv0);
  if (j >= im.nint || p.status[k] != CC_JPEG_OK) return;
  const int32_t* sb = p.subbase + im.iv0 + k;
  const long long g0 = im.sub0 + sb[j], n = sb[j + 1] - sb[j];
  const int base = j * (im.ri ? im.ri : im.mcux * im.mcuy) * im.bpm;
  const int want = interval_blocks(im, j);
  int carry = 0;
  bool synced = true, invalid = false;
  for (long long i0 = 0; i0 < n; i0 += 32) {
    const long long i = i0 + lane;
    const int c = i < n ? p.cnt[g0 + i] : 0;
    if (i < n && i > 0 && p.st[g0 + i] != p.en[g0 + i - 1]) synced = false;
    int tot;
    const int e = warp_excl(c, lane, tot);
    if (i < n) {
      p.bbase[g0 + i] = base + carry + e;
      const int er = p.err[g0 + i];
      invalid |= er != INT_MAX && carry + e + er < want;
    }
    carry += tot;
  }
  synced = __all_sync(~0u, synced);
  invalid = __any_sync(~0u, invalid);
  if (lane == 0) {
    if (!synced) atomicCAS(p.status + k, CC_JPEG_OK, CC_JPEG_UNSUPPORTED);
    else if (invalid || carry < want) atomicCAS(p.status + k, CC_JPEG_OK, CC_JPEG_CORRUPT);
  }
}

__global__ void __launch_bounds__(kSyncCta) jdec_write_kernel(const __grid_constant__ JdecParams p) {
  const long long g = static_cast<long long>(blockIdx.x) * kSyncCta + threadIdx.x;
  const Slot s = slot_of(p, g);
  if (s.k < 0) return;
  const JpegImage& im = p.tab[s.k];
  const int base = s.j * (im.ri ? im.ri : im.mcux * im.mcuy) * im.bpm;
  const int first = p.bbase[g], limit = base + interval_blocks(im, s.j) - first;
  if (limit <= 0) return;
  long long nbytes;
  const uint8_t* b = dbuf_of(p, s.k, nbytes);
  int done, err;
  run<true>(im, b, nbytes, p.st[g], s.hi, s.end, done, err, p.coef + (im.blk0 + first) * 64, limit);
}

// DC differences -> values, per component, in two passes over chunks of kDcChunk MCUs of each interval (a warp per chunk,
// grid x = interval, y * 8 + warp = chunk): the sums of each chunk's differences, then every chunk adds the sums of the
// chunks before it in its interval and scans its own MCUs.  Integer sums: the values are those of one sequential walk.
__device__ __forceinline__ bool dc_chunk(const JdecParams& p, int& k, int& j, int& m0, int& m1) {
  const long long gi = blockIdx.x;
  const int c = blockIdx.y * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (gi >= p.n_iv) return false;
  k = find_image(p, gi, [](const JpegImage& t) { return t.iv0; });
  const JpegImage& im = p.tab[k];
  j = static_cast<int>(gi - im.iv0);
  if (j >= im.nint || p.status[k] != CC_JPEG_OK) return false;
  const int nm = interval_blocks(im, j) / im.bpm;
  m0 = c * kDcChunk;
  m1 = min(nm, m0 + kDcChunk);
  return m0 < nm;
}

__device__ __forceinline__ int16_t* dc_base(const JdecParams& p, const JpegImage& im, int j) {
  const int ri = im.ri ? im.ri : im.mcux * im.mcuy;
  return p.coef + (im.blk0 + static_cast<long long>(j) * ri * im.bpm) * 64;
}

__global__ void jdec_dc_sum_kernel(const __grid_constant__ JdecParams p) {
  int k, j, m0, m1;
  if (!dc_chunk(p, k, j, m0, m1)) return;
  const JpegImage& im = p.tab[k];
  const int16_t* c0 = dc_base(p, im, j);
  const int lane = threadIdx.x & 31;
  int sum[3] = {0, 0, 0};
  for (int m = m0 + lane; m < m1; m += 32)
    for (int bl = 0; bl < im.bpm; ++bl) sum[im.blk_comp[bl]] += c0[(static_cast<long long>(m) * im.bpm + bl) * 64];
  for (int c = 0; c < 3; ++c)
    for (int o = 16; o; o >>= 1) sum[c] += __shfl_xor_sync(~0u, sum[c], o);
  if (lane == 0) {
    int32_t* d = p.dcsum + (static_cast<long long>(blockIdx.x) * p.dc_chunks + m0 / kDcChunk) * 3;
    d[0] = sum[0]; d[1] = sum[1]; d[2] = sum[2];
  }
}

__global__ void jdec_dc_apply_kernel(const __grid_constant__ JdecParams p) {
  int k, j, m0, m1;
  if (!dc_chunk(p, k, j, m0, m1)) return;
  const JpegImage& im = p.tab[k];
  int16_t* c0 = dc_base(p, im, j);
  const int lane = threadIdx.x & 31;
  int carry[3] = {0, 0, 0};
  const int32_t* s = p.dcsum + static_cast<long long>(blockIdx.x) * p.dc_chunks * 3;
  for (int q = lane; q < m0 / kDcChunk; q += 32)
    for (int c = 0; c < 3; ++c) carry[c] += s[q * 3 + c];
  for (int c = 0; c < 3; ++c)
    for (int o = 16; o; o >>= 1) carry[c] += __shfl_xor_sync(~0u, carry[c], o);
  for (int mb = m0; mb < m1; mb += 32) {
    const int m = mb + lane;
    int sum[3] = {0, 0, 0};
    if (m < m1)
      for (int bl = 0; bl < im.bpm; ++bl) sum[im.blk_comp[bl]] += c0[(static_cast<long long>(m) * im.bpm + bl) * 64];
    int ex[3];
    for (int c = 0; c < 3; ++c) {
      int tot;
      ex[c] = warp_excl(sum[c], lane, tot) + carry[c];
      carry[c] += tot;
    }
    if (m < m1) {
      for (int bl = 0; bl < im.bpm && bl < 6; ++bl) {
        int16_t* d = c0 + (static_cast<long long>(m) * im.bpm + bl) * 64;
        ex[im.blk_comp[bl]] += *d;
        *d = static_cast<int16_t>(ex[im.blk_comp[bl]]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ 11-12. reconstruction
struct ReconImg {
  int k, w, h, ncomp, hs, vs, mcux, mcuy;
  long long blk0, plane0, bfirst;       // first block in the coefficients; plane bytes; first block of the launch group
  int qt[3];                            // element offset of each component's table in qbase
  uint8_t* dst;                         // BGR pixel (0, 0) of the image's destination
  long long pitch;                      // bytes between its rows
};

struct ReconParams {
  const int16_t* coef;
  uint8_t* planes;
  int32_t* status;                      // per output slot; images not OK are skipped, the IDCT marks out-of-range ones
  const uint16_t* qbase;
  int n;
  long long nblk;
  ReconImg img[kReconPerLaunch];
};

__device__ __forceinline__ void plane_dims(const ReconImg& r, int c, int& pw, int& ph, long long& off) {
  const int H0 = r.hs * 8, V0 = r.vs * 8;
  const long long s0 = static_cast<long long>(r.mcux) * H0 * r.mcuy * V0, s1 = static_cast<long long>(r.mcux) * 8 * r.mcuy * 8;
  pw = c == 0 ? r.mcux * H0 : r.mcux * 8;
  ph = c == 0 ? r.mcuy * V0 : r.mcuy * 8;
  off = r.plane0 + (c == 0 ? 0 : c == 1 ? s0 : s0 + s1);
}

constexpr int kIdctIn = 16383;          // oracle.jpeg_decode.IDCT_IN_LIMIT

template <int SHIFT>
__device__ __forceinline__ void idct8(const int* d, int* o) {
  constexpr int kC0_298 = 2446, kC0_390 = 3196, kC0_541 = 4433, kC0_765 = 6270, kC0_899 = 7373, kC1_175 = 9633;
  constexpr int kC1_501 = 12299, kC1_847 = 15137, kC1_961 = 16069, kC2_053 = 16819, kC2_562 = 20995, kC3_072 = 25172;
  long long z2 = d[2], z3 = d[6];
  long long z1 = (z2 + z3) * kC0_541;
  const long long tmp2 = z1 - z3 * kC1_847, tmp3 = z1 + z2 * kC0_765;
  const long long tmp0 = static_cast<long long>(d[0] + d[4]) << 13, tmp1 = static_cast<long long>(d[0] - d[4]) << 13;
  const long long t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  long long a0 = d[7], a1 = d[5], a2 = d[3], a3 = d[1];
  z1 = a0 + a3; z2 = a1 + a2; z3 = a0 + a2;
  long long z4 = a1 + a3;
  const long long z5 = (z3 + z4) * kC1_175;
  a0 *= kC0_298; a1 *= kC2_053; a2 *= kC3_072; a3 *= kC1_501;
  z1 *= -kC0_899; z2 *= -kC2_562; z3 = z3 * -kC1_961 + z5; z4 = z4 * -kC0_390 + z5;
  a0 += z1 + z3; a1 += z2 + z4; a2 += z2 + z3; a3 += z1 + z4;
  constexpr long long R = 1ll << (SHIFT - 1);
  o[0] = static_cast<int>((t10 + a3 + R) >> SHIFT); o[7] = static_cast<int>((t10 - a3 + R) >> SHIFT);
  o[1] = static_cast<int>((t11 + a2 + R) >> SHIFT); o[6] = static_cast<int>((t11 - a2 + R) >> SHIFT);
  o[2] = static_cast<int>((t12 + a1 + R) >> SHIFT); o[5] = static_cast<int>((t12 - a1 + R) >> SHIFT);
  o[3] = static_cast<int>((t13 + a0 + R) >> SHIFT); o[4] = static_cast<int>((t13 - a0 + R) >> SHIFT);
}

__device__ __forceinline__ uint8_t range_limit(int x) {
  const int j = x & 1023;
  return static_cast<uint8_t>(j < 128 ? j + 128 : j < 512 ? 255 : j < 896 ? 0 : j - 896);
}

// 8 threads per block: column t, then row t; 32 blocks per CTA
__global__ void __launch_bounds__(256) jdec_idct_kernel(const __grid_constant__ ReconParams p) {
  __shared__ int ws[32][8][9];
  const long long gb = static_cast<long long>(blockIdx.x) * 32 + (threadIdx.x >> 3);
  const int lb = threadIdx.x >> 3, t = threadIdx.x & 7;
  const bool live = gb < p.nblk;
  int i = 0;
  if (live) {
    int lo = 0, hi = p.n - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (p.img[mid].bfirst <= gb) lo = mid; else hi = mid - 1;
    }
    i = lo;
  }
  const ReconImg& r = p.img[i];
  const bool ok = live && (!p.status || p.status[r.k] == CC_JPEG_OK);
  const long long b = gb - r.bfirst;
  const int bpm = r.ncomp == 1 ? 1 : r.hs * r.vs + 2;
  const long long m = b / bpm;
  const int bl = static_cast<int>(b - m * bpm);
  const int c = bl < r.hs * r.vs ? 0 : bl - r.hs * r.vs + 1;
  const int16_t* cf = p.coef + (r.blk0 + b) * 64;
  const uint16_t* q = p.qbase + r.qt[c];
  bool bad = false;
  int col[8], o[8];
  if (ok) {
#pragma unroll
    for (int y = 0; y < 8; ++y) {
      col[y] = static_cast<int>(cf[kDeZigzag[y * 8 + t]]) * static_cast<int>(q[y * 8 + t]);
      bad |= abs(col[y]) > kIdctIn;
    }
    idct8<11>(col, o);
#pragma unroll
    for (int y = 0; y < 8; ++y) { ws[lb][y][t] = o[y]; bad |= abs(o[y]) > kIdctIn; }
  }
  __syncwarp();
  if (!ok) return;
  int row[8];
#pragma unroll
  for (int x = 0; x < 8; ++x) row[x] = ws[lb][t][x];
  idct8<18>(row, o);
  int pw, ph;
  long long off;
  plane_dims(r, c, pw, ph, off);
  const int mx = static_cast<int>(m % r.mcux), my = static_cast<int>(m / r.mcux);
  const int inner = c == 0 ? bl : 0;
  const int bx = r.ncomp == 1 ? mx : mx * (c == 0 ? r.hs : 1) + inner % r.hs;
  const int by = r.ncomp == 1 ? my : my * (c == 0 ? r.vs : 1) + inner / r.hs;
  uint8_t* dst = p.planes + off + static_cast<long long>(by * 8 + t) * pw + bx * 8;
#pragma unroll
  for (int x = 0; x < 8; ++x) { bad |= o[x] < -512 || o[x] > 511; dst[x] = range_limit(o[x]); }
  if (bad && p.status) atomicCAS(p.status + r.k, CC_JPEG_OK, CC_JPEG_UNSUPPORTED);
}

__device__ __forceinline__ int fix16(double x) { return static_cast<int>(x * 65536.0 + 0.5); }

__global__ void __launch_bounds__(256) jdec_pixels_kernel(const __grid_constant__ ReconParams p) {
  const ReconImg& r = p.img[blockIdx.z];
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= r.w || y >= r.h) return;
  if (p.status && p.status[r.k] != CC_JPEG_OK) return;
  int pw, ph;
  long long off;
  plane_dims(r, 0, pw, ph, off);
  const int Y = p.planes[off + static_cast<long long>(y) * pw + x];
  uint8_t* o = r.dst + static_cast<long long>(y) * r.pitch + x * 3;
  if (r.ncomp == 1) { o[0] = o[1] = o[2] = static_cast<uint8_t>(Y); return; }
  int ch[2];
  const int dw = (r.w + r.hs - 1) / r.hs, dh = (r.h + r.vs - 1) / r.vs;
  for (int c = 0; c < 2; ++c) {
    plane_dims(r, c + 1, pw, ph, off);
    const uint8_t* P = p.planes + off;
    auto at = [&](int yy, int xx) { return static_cast<int>(P[static_cast<long long>(yy) * pw + xx]); };
    if (r.hs == 1 && r.vs == 1) { ch[c] = at(y, x); continue; }
    if (r.hs == 2 && dw <= 2) { ch[c] = at(r.vs == 2 ? y >> 1 : y, x >> 1); continue; }    // box replication
    if (r.vs == 2) {
      const int ny = y >> 1, fy = min(max((y & 1) ? ny + 1 : ny - 1, 0), dh - 1);
      if (r.hs == 1) { ch[c] = (3 * at(ny, x) + at(fy, x) + ((y & 1) ? 2 : 1)) >> 2; continue; }
      const int cx = x >> 1, ox = min(max((x & 1) ? cx + 1 : cx - 1, 0), dw - 1);
      const int s0 = 3 * at(ny, cx) + at(fy, cx), s1 = 3 * at(ny, ox) + at(fy, ox);
      ch[c] = (3 * s0 + s1 + ((x & 1) ? 7 : 8)) >> 4;
      continue;
    }
    const int cx = x >> 1, ox = min(max((x & 1) ? cx + 1 : cx - 1, 0), dw - 1);                    // h2v1
    ch[c] = (3 * at(y, cx) + at(y, ox) + ((x & 1) ? 2 : 1)) >> 2;
  }
  const int cb = ch[0] - 128, cr = ch[1] - 128;
  constexpr int kHalf = 1 << 15;
  const int R = Y + ((fix16(1.40200) * cr + kHalf) >> 16);
  const int G = Y + ((-fix16(0.71414) * cr + (-fix16(0.34414) * cb + kHalf)) >> 16);
  const int B = Y + ((fix16(1.77200) * cb + kHalf) >> 16);
  o[0] = static_cast<uint8_t>(min(max(B, 0), 255));
  o[1] = static_cast<uint8_t>(min(max(G, 0), 255));
  o[2] = static_cast<uint8_t>(min(max(R, 0), 255));
}

int launch_recon(ReconParams& p, const std::vector<ReconImg>& imgs, cudaStream_t st) {
  for (size_t i0 = 0; i0 < imgs.size(); i0 += kReconPerLaunch) {
    const int n = static_cast<int>(std::min(imgs.size() - i0, static_cast<size_t>(kReconPerLaunch)));
    long long nb = 0;
    int hmax = 1, wmax = 1;
    for (int i = 0; i < n; ++i) {
      p.img[i] = imgs[i0 + i];
      p.img[i].bfirst = nb;
      const ReconImg& r = p.img[i];
      nb += static_cast<long long>(r.mcux) * r.mcuy * (r.ncomp == 1 ? 1 : r.hs * r.vs + 2);
      hmax = std::max(hmax, r.h); wmax = std::max(wmax, r.w);
    }
    p.n = n; p.nblk = nb;
    if (nb) jdec_idct_kernel<<<static_cast<unsigned>((nb + 31) / 32), 256, 0, st>>>(p);
    jdec_pixels_kernel<<<dim3((wmax + 31) / 32, (hmax + 7) / 8, n), dim3(32, 8), 0, st>>>(p);
    CC_CHECK_CUDA(cudaGetLastError());
  }
  return CC_OK;
}

struct QtArg { uint16_t q[128]; };
__global__ void jdec_ok_kernel(int32_t* status, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < K) status[k] = CC_JPEG_OK;
}
__global__ void jdec_put_qt_kernel(const __grid_constant__ QtArg a, uint16_t* dst) { dst[threadIdx.x] = a.q[threadIdx.x]; }

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// the sync kernel on as many CTAs as can be resident at once (a cooperative launch), at most one per tile
int launch_sync(const JdecParams& p, unsigned tiles, cudaStream_t st) {
  int dev = 0, sms = 0, per_sm = 0;
  CC_CHECK_CUDA(cudaGetDevice(&dev));
  CC_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CC_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, jdec_sync_kernel, kSyncCta, 0));
  const unsigned grid = std::max(1u, std::min(tiles, static_cast<unsigned>(sms * per_sm)));
  void* args[] = {const_cast<JdecParams*>(&p)};
  CC_CHECK_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(jdec_sync_kernel), grid, kSyncCta, args, 0, st));
  return CC_OK;
}

long long plane_bytes(int ncomp, int hs, int vs, int mcux, int mcuy) {
  const long long luma = static_cast<long long>(mcux) * hs * 8 * mcuy * vs * 8;
  return ncomp == 1 ? luma : luma + 2ll * mcux * 8 * mcuy * 8;
}

// ------------------------------------------------------------------------------------------------ host: markers
struct Bad { int status; };

int be16(const uint8_t* b) { return (b[0] << 8) | b[1]; }

void make_huff(const uint8_t* counts, const uint8_t* vals, int nvals, bool dc, HuffDev& t) {
  std::memset(&t, 0, sizeof(t));
  std::memcpy(t.vals, vals, nvals);
  for (int l = 0; l < 18; ++l) t.maxcode[l] = -1;
  int code = 0, k = 0;
  for (int L = 1; L <= 16; ++L) {
    const int n = counts[L - 1];
    if (n) {
      t.valoff[L] = k - code;
      for (int i = 0; i < n; ++i, ++k, ++code) {
        // codes must fit in L bits and never be all ones (jpeg_make_d_derived_tbl); checked before the lookup is written
        if (code + 1 >= (1 << L)) throw Bad{CC_JPEG_CORRUPT};
        if (L <= 9) {
          const int lo = code << (9 - L);
          for (int e = 0; e < (1 << (9 - L)); ++e) t.look[lo + e] = static_cast<uint16_t>((L << 8) | vals[k]);
        }
      }
      t.maxcode[L] = code - 1;
    }
    code <<= 1;
  }
  if (dc)
    for (int i = 0; i < nvals; ++i)
      if (vals[i] > 15) throw Bad{CC_JPEG_CORRUPT};
}

int exif_orientation(const uint8_t* t, int n) {      // TIFF header + IFD0 of an Exif payload; 0 = no tag
  if (n < 8 || !((t[0] == 'I' && t[1] == 'I') || (t[0] == 'M' && t[1] == 'M'))) throw Bad{CC_JPEG_UNSUPPORTED};
  const bool big = t[0] == 'M';
  auto rd = [&](long long o, int w) {
    unsigned v = 0;
    for (int i = 0; i < w; ++i) v |= static_cast<unsigned>(t[o + i]) << (8 * (big ? w - 1 - i : i));
    return v;
  };
  const long long ifd = rd(4, 4);
  if (ifd + 2 > n) throw Bad{CC_JPEG_UNSUPPORTED};
  const int cnt = static_cast<int>(rd(ifd, 2));
  for (int i = 0; i < cnt; ++i) {
    const long long e = ifd + 2 + 12ll * i;
    if (e + 12 > n) throw Bad{CC_JPEG_UNSUPPORTED};
    if (rd(e, 2) == 0x0112) return static_cast<int>(rd(e + 8, 2));
  }
  return 0;
}

// oracle.jpeg_decode._parse, filling the device table
void parse_one(const uint8_t* b, long long n, JpegImage& im) {
  if (n < 4 || b[0] != 0xFF || b[1] != 0xD8) throw Bad{CC_JPEG_CORRUPT};
  long long pos = 2;
  bool have_q[4] = {false, false, false, false}, have_dc[4] = {}, have_ac[4] = {};
  static thread_local uint16_t qt[4][64];
  struct Spec { uint8_t counts[16]; uint8_t vals[256]; int n; };
  static thread_local Spec dcs[4], acs[4];
  bool sof = false, jfif = false;
  int adobe = -1, ri = 0;
  int comp_id[3] = {0, 0, 0}, comp_tq[3] = {0, 0, 0}, H0 = 1, V0 = 1;
  int td[3] = {0, 0, 0}, ta[3] = {0, 0, 0};
  static const uint8_t zz[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  while (true) {
    if (pos + 2 > n || b[pos] != 0xFF) throw Bad{CC_JPEG_CORRUPT};
    while (pos < n && b[pos] == 0xFF) ++pos;
    if (pos + 3 > n) throw Bad{CC_JPEG_CORRUPT};
    const int code = b[pos++];
    if (code == 0xD8 || code == 0xD9 || code == 0x01 || (code >= 0xD0 && code <= 0xD7)) throw Bad{CC_JPEG_CORRUPT};
    // markers libjpeg's read_markers does not know (JPG, JPGn, DHP, EXP, reserved): cv2 fails on them
    if (code < 0xC0 || code == 0xC8 || code == 0xDE || code == 0xDF || (code >= 0xF0 && code <= 0xFD)) throw Bad{CC_JPEG_CORRUPT};
    const int ln = be16(b + pos);
    if (ln < 2 || pos + ln > n) throw Bad{CC_JPEG_CORRUPT};
    const uint8_t* s = b + pos + 2;
    const int sl = ln - 2;
    pos += ln;
    if (code == 0xC0 || code == 0xC1) {
      if (sof || sl < 6) throw Bad{CC_JPEG_CORRUPT};
      const int P = s[0], h = be16(s + 1), w = be16(s + 3), nf = s[5];
      if (sl != 6 + 3 * nf || nf == 0 || h == 0 || w == 0) throw Bad{CC_JPEG_CORRUPT};
      if (P != 8) throw Bad{CC_JPEG_UNSUPPORTED};
      for (int i = 0; i < nf; ++i) {
        const int H = s[7 + 3 * i] >> 4, V = s[7 + 3 * i] & 15;
        if (H < 1 || H > 4 || V < 1 || V > 4 || s[8 + 3 * i] > 3) throw Bad{CC_JPEG_CORRUPT};
      }
      if (nf != 1 && nf != 3) throw Bad{CC_JPEG_UNSUPPORTED};
      for (int i = 0; i < nf; ++i) {
        comp_id[i] = s[6 + 3 * i]; comp_tq[i] = s[8 + 3 * i];
        for (int j = 0; j < i; ++j)
          if (comp_id[j] == comp_id[i]) throw Bad{CC_JPEG_UNSUPPORTED};
      }
      if (nf == 3) {
        H0 = s[7] >> 4; V0 = s[7] & 15;
        if (H0 > 2 || V0 > 2 || s[10] != 0x11 || s[13] != 0x11) throw Bad{CC_JPEG_UNSUPPORTED};
      }
      im.w = w; im.h = h; im.ncomp = nf;
      sof = true;
    } else if ((code >= 0xC2 && code <= 0xCF && code != 0xC4 && code != 0xC8) ) {
      throw Bad{CC_JPEG_UNSUPPORTED};                   // progressive, lossless, hierarchical, arithmetic (DAC)
    } else if (code == 0xDB) {
      int i = 0;
      while (i < sl) {
        const int pq = s[i] >> 4, tq = s[i] & 15, nb = pq ? 128 : 64;
        if (pq > 1 || tq > 3 || i + 1 + nb > sl) throw Bad{CC_JPEG_CORRUPT};
        for (int e = 0; e < 64; ++e) {
          const int v = pq ? be16(s + i + 1 + 2 * e) : s[i + 1 + e];
          if (v > 32767) throw Bad{CC_JPEG_UNSUPPORTED};
          qt[tq][zz[e]] = static_cast<uint16_t>(v);
        }
        have_q[tq] = true;
        i += 1 + nb;
      }
    } else if (code == 0xC4) {
      int i = 0;
      while (i < sl) {
        if (i + 17 > sl) throw Bad{CC_JPEG_CORRUPT};
        const int tc = s[i] >> 4, th = s[i] & 15;
        int tot = 0;
        for (int l = 0; l < 16; ++l) tot += s[i + 1 + l];
        if (tc > 1 || th > 3 || tot > 256 || i + 17 + tot > sl) throw Bad{CC_JPEG_CORRUPT};
        Spec& sp = tc ? acs[th] : dcs[th];
        std::memcpy(sp.counts, s + i + 1, 16);
        std::memcpy(sp.vals, s + i + 17, tot);
        sp.n = tot;
        (tc ? have_ac : have_dc)[th] = true;
        i += 17 + tot;
      }
    } else if (code == 0xDD) {
      if (sl != 2) throw Bad{CC_JPEG_CORRUPT};
      ri = be16(s);
    } else if (code == 0xE0) {
      jfif = jfif || (sl >= 14 && std::memcmp(s, "JFIF\0", 5) == 0);
    } else if (code == 0xE1) {
      if (sl >= 6 && std::memcmp(s, "Exif\0\0", 6) == 0) {
        const int o = exif_orientation(s + 6, sl - 6);
        if (o != 0 && o != 1) throw Bad{CC_JPEG_UNSUPPORTED};
      }
    } else if (code == 0xEE) {
      if (sl >= 12 && std::memcmp(s, "Adobe", 5) == 0) adobe = s[11];
    } else if (code == 0xDA) {
      if (!sof || sl < 1) throw Bad{CC_JPEG_CORRUPT};
      const int ns = s[0];
      if (sl != 4 + 2 * ns || ns == 0) throw Bad{CC_JPEG_CORRUPT};
      for (int i = 0; i < ns; ++i) {
        bool found = false;
        for (int c = 0; c < im.ncomp; ++c) found |= comp_id[c] == s[1 + 2 * i];
        if (!found || (s[2 + 2 * i] >> 4) > 3 || (s[2 + 2 * i] & 15) > 3) throw Bad{CC_JPEG_CORRUPT};
      }
      bool same = ns == im.ncomp;
      for (int i = 0; same && i < ns; ++i) same = s[1 + 2 * i] == comp_id[i];
      if (!same || s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0) throw Bad{CC_JPEG_UNSUPPORTED};
      for (int i = 0; i < ns; ++i) { td[i] = s[2 + 2 * i] >> 4; ta[i] = s[2 + 2 * i] & 15; }
      break;
    }
  }
  if (im.ncomp == 3 && !jfif && (adobe == 0 || (adobe < 0 && comp_id[0] == 82 && comp_id[1] == 71 && comp_id[2] == 66)))
    throw Bad{CC_JPEG_UNSUPPORTED};
  // the scan ends at the first marker that is not RSTn
  long long end = n;
  for (long long i = pos; i + 1 < n; ++i) {
    const uint8_t* f = static_cast<const uint8_t*>(std::memchr(b + i, 0xFF, static_cast<size_t>(n - 1 - i)));
    if (!f) break;
    i = f - b;
    const int m = b[i + 1];
    if (m == 0x00 || (m >= 0xD0 && m <= 0xD7)) { ++i; continue; }
    if (m == 0xFF) continue;
    end = i;
    if (m != 0xD9) throw Bad{CC_JPEG_UNSUPPORTED};
    break;
  }
  for (int c = 0; c < im.ncomp; ++c)
    if (!have_dc[td[c]] || !have_ac[ta[c]]) throw Bad{CC_JPEG_UNSUPPORTED};
  for (int c = 0; c < im.ncomp; ++c) {
    make_huff(dcs[td[c]].counts, dcs[td[c]].vals, dcs[td[c]].n, true, im.dc[td[c]]);
    make_huff(acs[ta[c]].counts, acs[ta[c]].vals, acs[ta[c]].n, false, im.ac[ta[c]]);
  }
  for (int c = 0; c < im.ncomp; ++c) {
    if (!have_q[comp_tq[c]]) throw Bad{CC_JPEG_CORRUPT};
    std::memcpy(im.qt[c], qt[comp_tq[c]], sizeof(im.qt[c]));
  }
  im.hs = im.ncomp == 1 ? 1 : H0;
  im.vs = im.ncomp == 1 ? 1 : V0;
  im.mcux = (im.w + 8 * im.hs - 1) / (8 * im.hs);
  im.mcuy = (im.h + 8 * im.vs - 1) / (8 * im.vs);
  im.bpm = im.ncomp == 1 ? 1 : im.hs * im.vs + 2;
  for (int bl = 0; bl < im.bpm && bl < 6; ++bl) {
    const int c = std::min(bl < im.hs * im.vs ? 0 : bl - im.hs * im.vs + 1, 2);
    im.blk_comp[bl] = static_cast<int8_t>(c);
    im.blk_dc[bl] = static_cast<int8_t>(td[c]);
    im.blk_ac[bl] = static_cast<int8_t>(ta[c]);
  }
  const long long nmcu = static_cast<long long>(im.mcux) * im.mcuy;
  im.ri = ri;
  im.nint = static_cast<int>(ri ? (nmcu + ri - 1) / ri : 1);
  im.scan_len = end - pos;
  im.scan_off = pos;                                   // relative to the file; made absolute by the caller
}

// where each image's intermediates live in the workspace
struct Layout {
  long long n_chunk = 0, n_iv = 0, n_slot = 0, n_blk = 0, dst = 0, planes = 0;
  int dc_chunks = 1;
  size_t chunk_kept, chunk_rst, dlen, dbuf, ivstart, subbase, st, en, cnt, err, edge, flag, bbase, dcsum, coef, planesb, total;
};

Layout layout(const JpegImage* tab, int K, bool with_coef) {
  Layout L;
  for (int k = 0; k < K; ++k) {
    const JpegImage& im = tab[k];
    if (im.status != CC_JPEG_OK) continue;
    L.n_chunk = std::max(L.n_chunk, im.chunk0 + im.nchunk);
    L.n_iv = std::max(L.n_iv, im.iv0 + im.nint);
    L.n_slot = std::max(L.n_slot, im.sub0 + im.nsub_max);
    L.n_blk = std::max(L.n_blk, im.blk0 + static_cast<long long>(im.mcux) * im.mcuy * im.bpm);
    L.dst = std::max(L.dst, im.dst0 + im.scan_len);
    L.planes = std::max(L.planes, im.plane0 + plane_bytes(im.ncomp, im.hs, im.vs, im.mcux, im.mcuy));
    const long long nmcu = static_cast<long long>(im.mcux) * im.mcuy, per_iv = im.ri ? std::min<long long>(im.ri, nmcu) : nmcu;
    L.dc_chunks = std::max(L.dc_chunks, static_cast<int>((per_iv + kDcChunk - 1) / kDcChunk));
  }
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
  L.chunk_kept = take(L.n_chunk * 4); L.chunk_rst = take(L.n_chunk * 4);
  L.dlen = take(static_cast<size_t>(K) * 4);
  L.dbuf = take(L.dst + 8);
  L.ivstart = take((L.n_iv + K) * 4); L.subbase = take((L.n_iv + K) * 4);
  L.st = take(L.n_slot * 8); L.en = take(L.n_slot * 8);
  L.cnt = take(L.n_slot * 4); L.err = take(L.n_slot * 4); L.bbase = take(L.n_slot * 4);
  L.edge = take(2 * ((L.n_slot + kSyncCta - 1) / kSyncCta) * 8); L.flag = take(3 * 4);
  L.dcsum = take(static_cast<size_t>(L.n_iv) * L.dc_chunks * 12);
  L.coef = with_coef ? take(L.n_blk * 128) : 0;
  L.planesb = take(L.planes);
  L.total = off;
  return L;
}

}  // namespace
}  // namespace cc

using namespace cc;

extern "C" size_t cc_jpeg_table_bytes(void) { return sizeof(JpegImage); }

extern "C" int cc_jpeg_parse(const uint8_t* h_data, int64_t data_bytes, const int64_t* offsets, const int64_t* lengths, int K,
                             void* h_table, int32_t* h_sizes, int32_t* h_status, int64_t* h_blocks) {
  const char* who = "cc_jpeg_parse";
  CC_REQUIRE(K >= 0 && (K == 0 || (h_data && offsets && lengths && h_table && h_sizes && h_status && h_blocks)),
             "%s: null pointer or K=%d < 0", who, K);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(h_table) & 15) == 0, "%s: h_table must be 16-byte aligned", who);
  for (int k = 0; k < K; ++k)
    CC_REQUIRE(offsets[k] >= 0 && lengths[k] >= 0 && offsets[k] + lengths[k] <= data_bytes,
               "%s: file %d [%lld, +%lld) is outside the %lld data bytes", who, k, static_cast<long long>(offsets[k]),
               static_cast<long long>(lengths[k]), static_cast<long long>(data_bytes));
  JpegImage* tab = static_cast<JpegImage*>(h_table);
  long long chunk = 0, dst = 0, iv = 0, sub = 0, blk = 0, plane = 0;
  for (int k = 0; k < K; ++k) {
    JpegImage& im = tab[k];
    std::memset(&im, 0, sizeof(im));
    try {
      parse_one(h_data + offsets[k], lengths[k], im);
      im.status = CC_JPEG_OK;
    } catch (const Bad& e) {
      const int w = im.w, h = im.h;
      std::memset(&im, 0, sizeof(im));
      im.status = e.status;
      im.w = w; im.h = h;
    }
    h_status[k] = im.status;
    h_sizes[2 * k] = im.w;
    h_sizes[2 * k + 1] = im.h;
    im.chunk0 = chunk; im.dst0 = dst; im.iv0 = iv; im.sub0 = sub; im.blk0 = blk; im.plane0 = plane;
    if (im.status != CC_JPEG_OK) { h_blocks[k] = 0; continue; }
    im.scan_off += offsets[k];
    im.nchunk = static_cast<int>((im.scan_len + kChunk - 1) / kChunk);
    im.nsub_max = (im.scan_len * 8 + kSubBits - 1) / kSubBits + im.nint;
    h_blocks[k] = static_cast<long long>(im.mcux) * im.mcuy * im.bpm;
    chunk += im.nchunk; dst += im.scan_len; iv += im.nint; sub += im.nsub_max; blk += h_blocks[k];
    plane += static_cast<long long>(align256(plane_bytes(im.ncomp, im.hs, im.vs, im.mcux, im.mcuy)));
  }
  return CC_OK;
}

// cc_jpeg_decode and cc_jpeg_decode_frames once their arguments are checked: image k (status OK) goes to dst[k], rows
// pitch[k] bytes apart
static int decode_checked(const uint8_t* d_data, const JpegImage* tab, const void* d_table, int K, const Layout& L,
                          uint8_t* const* dst, const long long* pitch, int32_t* d_status, int16_t* d_coef, void* d_workspace,
                          void* stream) {
  if (K == 0) return CC_OK;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  JdecParams p;
  p.data = d_data; p.tab = static_cast<const JpegImage*>(d_table); p.K = K; p.status = d_status;
  p.chunk_kept = reinterpret_cast<int32_t*>(ws + L.chunk_kept);
  p.chunk_rst = reinterpret_cast<int32_t*>(ws + L.chunk_rst);
  p.dlen = reinterpret_cast<int32_t*>(ws + L.dlen);
  p.dbuf = ws + L.dbuf;
  p.ivstart = reinterpret_cast<int32_t*>(ws + L.ivstart);
  p.subbase = reinterpret_cast<int32_t*>(ws + L.subbase);
  p.st = reinterpret_cast<unsigned long long*>(ws + L.st);
  p.en = reinterpret_cast<unsigned long long*>(ws + L.en);
  p.cnt = reinterpret_cast<int32_t*>(ws + L.cnt);
  p.err = reinterpret_cast<int32_t*>(ws + L.err);
  p.edge = reinterpret_cast<unsigned long long*>(ws + L.edge);
  p.flag = reinterpret_cast<int32_t*>(ws + L.flag);
  p.bbase = reinterpret_cast<int32_t*>(ws + L.bbase);
  p.dcsum = reinterpret_cast<int32_t*>(ws + L.dcsum);
  p.dc_chunks = L.dc_chunks;
  p.coef = d_coef ? d_coef : reinterpret_cast<int16_t*>(ws + L.coef);
  p.n_chunk = L.n_chunk; p.n_iv = L.n_iv; p.n_slot = L.n_slot;
  jdec_status_kernel<<<(K + 255) / 256, 256, 0, st>>>(p);
  if (L.n_blk) CC_CHECK_CUDA(cudaMemsetAsync(p.coef, 0, static_cast<size_t>(L.n_blk) * 128, st));
  const unsigned warps8 = static_cast<unsigned>((K + 7) / 8);
  if (L.n_chunk) jdec_count_kernel<<<static_cast<unsigned>(L.n_chunk), 256, 0, st>>>(p);
  jdec_scan_kernel<<<warps8, 256, 0, st>>>(p);
  if (L.n_chunk) jdec_scatter_kernel<<<static_cast<unsigned>(L.n_chunk), 256, 0, st>>>(p);
  jdec_layout_kernel<<<warps8, 256, 0, st>>>(p);
  if (L.n_slot) {
    const unsigned g = static_cast<unsigned>((L.n_slot + kSyncCta - 1) / kSyncCta);
    if (int rc = launch_sync(p, g, st)) return rc;
    const unsigned giv = static_cast<unsigned>((L.n_iv + 7) / 8);
    jdec_counts_kernel<<<giv, 256, 0, st>>>(p);
    jdec_write_kernel<<<g, kSyncCta, 0, st>>>(p);
    const dim3 gdc(static_cast<unsigned>(L.n_iv), static_cast<unsigned>((L.dc_chunks + 7) / 8));
    jdec_dc_sum_kernel<<<gdc, 256, 0, st>>>(p);
    jdec_dc_apply_kernel<<<gdc, 256, 0, st>>>(p);
  }
  CC_CHECK_CUDA(cudaGetLastError());
  static thread_local ReconParams rp;
  rp.coef = p.coef; rp.planes = ws + L.planesb; rp.status = d_status;
  rp.qbase = reinterpret_cast<const uint16_t*>(d_table);
  std::vector<ReconImg> imgs;
  for (int k = 0; k < K; ++k) {
    const JpegImage& im = tab[k];
    if (im.status != CC_JPEG_OK) continue;
    ReconImg r{k, im.w, im.h, im.ncomp, im.hs, im.vs, im.mcux, im.mcuy, im.blk0, im.plane0, 0, {0, 0, 0}, dst[k], pitch[k]};
    for (int c = 0; c < 3; ++c)
      r.qt[c] = static_cast<int>((k * sizeof(JpegImage) + offsetof(JpegImage, qt) + c * 128) / 2);
    imgs.push_back(r);
  }
  return launch_recon(rp, imgs, st);
}

static int check_tables(const char* who, const JpegImage* tab, int K, const void* d_data, const void* d_table, const int32_t* d_status,
                        const Layout& L, const void* d_workspace, size_t ws_bytes) {
  CC_REQUIRE(d_data && d_table && d_status, "%s: d_data, d_table and d_status must not be NULL", who);
  CC_REQUIRE(d_workspace && ws_bytes >= L.total, "%s: workspace of %zu bytes too small (%zu needed)", who,
             d_workspace ? ws_bytes : size_t(0), L.total);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0 && (reinterpret_cast<uintptr_t>(d_table) & 15) == 0,
             "%s: d_workspace must be 256-byte aligned, d_table 16-byte aligned", who);
  for (int k = 0; k < K; ++k)
    CC_REQUIRE(tab[k].status >= CC_JPEG_OK && tab[k].status <= CC_JPEG_CORRUPT, "%s: table entry %d is not from cc_jpeg_parse", who,
               k);
  return CC_OK;
}

extern "C" int cc_jpeg_decode(const uint8_t* d_data, const void* h_table, const void* d_table, int K, uint8_t* d_out, int Hmax,
                              int Wmax, int32_t* d_status, int16_t* d_coef, void* d_workspace, size_t ws_bytes, size_t* ws_needed,
                              void* stream) {
  const char* who = "cc_jpeg_decode";
  CC_REQUIRE(K >= 0 && (K == 0 || h_table), "%s: null table or K=%d < 0", who, K);
  const JpegImage* tab = static_cast<const JpegImage*>(h_table);
  const Layout L = layout(tab, K, d_coef == nullptr);
  if (ws_needed) *ws_needed = L.total;
  if (!d_out) return CC_OK;                           // workspace size query
  CC_REQUIRE(Hmax > 0 && Wmax > 0, "%s: bad batch size %dx%d", who, Hmax, Wmax);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_coef) & 15) == 0, "%s: d_coef must be 16-byte aligned", who);
  if (int rc = check_tables(who, tab, K, d_data, d_table, d_status, L, d_workspace, ws_bytes)) return rc;
  std::vector<uint8_t*> dst(K);
  std::vector<long long> pitch(K, 3ll * Wmax);
  for (int k = 0; k < K; ++k) {
    CC_REQUIRE(tab[k].status != CC_JPEG_OK || (tab[k].w <= Wmax && tab[k].h <= Hmax),
               "%s: image %d (%dx%d) does not fit the %dx%d batch", who, k, tab[k].w, tab[k].h, Wmax, Hmax);
    dst[k] = d_out + static_cast<long long>(k) * Hmax * Wmax * 3;
  }
  return decode_checked(d_data, tab, d_table, K, L, dst.data(), pitch.data(), d_status, d_coef, d_workspace, stream);
}

extern "C" int cc_jpeg_decode_frames(const uint8_t* d_data, const void* h_table, const void* d_table, int K, const cc_jpeg_dest* outs,
                                     int32_t* d_status, void* d_workspace, size_t ws_bytes, size_t* ws_needed, void* stream) {
  const char* who = "cc_jpeg_decode_frames";
  CC_REQUIRE(K >= 0 && (K == 0 || h_table), "%s: null table or K=%d < 0", who, K);
  const JpegImage* tab = static_cast<const JpegImage*>(h_table);
  const Layout L = layout(tab, K, true);
  if (ws_needed) *ws_needed = L.total;
  if (!outs) return CC_OK;                            // workspace size query
  if (int rc = check_tables(who, tab, K, d_data, d_table, d_status, L, d_workspace, ws_bytes)) return rc;
  std::vector<uint8_t*> dst(K);
  std::vector<long long> pitch(K);
  std::vector<std::pair<uintptr_t, uintptr_t>> spans;  // [first byte, end) of every destination the decode may write
  for (int k = 0; k < K; ++k) {
    const cc_jpeg_dest& o = outs[k];
    dst[k] = static_cast<uint8_t*>(o.data); pitch[k] = o.pitch;
    if (tab[k].status != CC_JPEG_OK) continue;
    CC_REQUIRE(o.data && o.h == tab[k].h && o.w == tab[k].w, "%s: destination %d is %dx%d%s, the image %dx%d", who, k, o.w, o.h,
               o.data ? "" : " at NULL", tab[k].w, tab[k].h);
    CC_REQUIRE(o.pitch >= 3ll * o.w, "%s: destination %d has a pitch of %lld bytes, below 3 x %d", who, k,
               static_cast<long long>(o.pitch), o.w);
    const uintptr_t a = reinterpret_cast<uintptr_t>(o.data);
    spans.emplace_back(a, a + static_cast<uintptr_t>((o.h - 1) * o.pitch + 3ll * o.w));
  }
  std::sort(spans.begin(), spans.end());
  for (size_t i = 1; i < spans.size(); ++i)
    CC_REQUIRE(spans[i].first >= spans[i - 1].second, "%s: two destinations overlap", who);
  return decode_checked(d_data, tab, d_table, K, L, dst.data(), pitch.data(), d_status, nullptr, d_workspace, stream);
}

// cc_jpeg_crops_decoded from the point where the crops' sources, rects and quality are checked
static int crops_decoded_sources(const char* who, const CropSource* src, const int32_t* rects, int K, int quality, uint8_t* d_out,
                                 int Hmax, int Wmax, int32_t* d_status, void* d_workspace, size_t ws_bytes, size_t* ws_needed,
                                 void* stream) {
  int64_t nb = 0;
  jpeg_coeffs_sources(src, rects, K, quality, nullptr, &nb, nullptr);     // counts the blocks
  std::vector<ReconImg> imgs(K);
  long long plane = 0, blk = 0;
  for (int k = 0; k < K; ++k) {
    const int* r = rects + 5 * k;
    const int w = r[3] - r[1], h = r[4] - r[2];
    ReconImg& x = imgs[k];
    x = ReconImg{k, w, h, 3, 2, 2, (w + 15) / 16, (h + 15) / 16, blk, plane, 0, {0, 64, 64}, nullptr, 3ll * Wmax};
    blk += 6ll * x.mcux * x.mcuy;
    plane += static_cast<long long>(align256(plane_bytes(3, 2, 2, x.mcux, x.mcuy)));
  }
  const size_t coef_bytes = align256(static_cast<size_t>(nb) * 128);
  const size_t need = 256 + coef_bytes + static_cast<size_t>(plane);
  if (ws_needed) *ws_needed = need;
  if (!d_out) return CC_OK;
  CC_REQUIRE(Hmax > 0 && Wmax > 0, "%s: bad batch size %dx%d", who, Hmax, Wmax);
  CC_REQUIRE(d_status || K == 0, "%s: d_status must not be NULL", who);
  for (int k = 0; k < K; ++k)
    CC_REQUIRE(imgs[k].w <= Wmax && imgs[k].h <= Hmax, "%s: crop %d (%dx%d) does not fit the %dx%d batch", who, k, imgs[k].w,
               imgs[k].h, Wmax, Hmax);
  CC_REQUIRE(d_workspace && ws_bytes >= need, "%s: workspace of %zu bytes too small (%zu needed)", who,
             d_workspace ? ws_bytes : size_t(0), need);
  CC_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, "%s: d_workspace must be 256-byte aligned", who);
  if (K == 0) return CC_OK;
  for (int k = 0; k < K; ++k) imgs[k].dst = d_out + static_cast<long long>(k) * Hmax * Wmax * 3;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  // the quantisation tables travel at the head of the workspace: a kernel argument writes them, no host copy
  static thread_local ReconParams rp;
  uint16_t qt[2][64];
  jpeg_quant_tables(quality, qt);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + 256);
  if (int rc = jpeg_coeffs_sources(src, rects, K, quality, coef, nullptr, st)) return rc;
  jdec_ok_kernel<<<(K + 255) / 256, 256, 0, st>>>(d_status, K);
  rp.coef = coef; rp.planes = ws + 256 + coef_bytes; rp.status = d_status;
  rp.qbase = reinterpret_cast<const uint16_t*>(ws);
  QtArg qa;
  std::memcpy(qa.q, qt, sizeof(qt));
  jdec_put_qt_kernel<<<1, 128, 0, st>>>(qa, reinterpret_cast<uint16_t*>(ws));
  return launch_recon(rp, imgs, st);
}

extern "C" int cc_jpeg_crops_decoded(const uint8_t* d_frames, int n_frames, int H, int W, int src_fmt, const int32_t* rects, int K,
                                     int quality, uint8_t* d_out, int Hmax, int Wmax, int32_t* d_status, void* d_workspace,
                                     size_t ws_bytes, size_t* ws_needed, void* stream) {
  // validates the frames, rects and quality exactly as the encoder does
  if (int rc = cc_jpeg_coeffs(d_frames, n_frames, H, W, src_fmt, rects, K, quality, nullptr, nullptr, nullptr)) return rc;
  std::vector<CropSource> src(K);
  uniform_crop_sources(d_frames, H, W, src_fmt, rects, K, src.data());
  return crops_decoded_sources("cc_jpeg_crops_decoded", src.data(), rects, K, quality, d_out, Hmax, Wmax, d_status, d_workspace,
                               ws_bytes, ws_needed, stream);
}

extern "C" int cc_jpeg_crops_decoded_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int quality,
                                            uint8_t* d_out, int Hmax, int Wmax, int32_t* d_status, void* d_workspace,
                                            size_t ws_bytes, size_t* ws_needed, void* stream) {
  const char* who = "cc_jpeg_crops_decoded_frames";
  std::vector<CropSource> src(K > 0 ? K : 0);
  if (int rc = table_crop_sources(who, frames, n_frames, rects, K, src.data())) return rc;
  if (int rc = check_table_jpeg(who, rects, K, quality)) return rc;
  return crops_decoded_sources(who, src.data(), rects, K, quality, d_out, Hmax, Wmax, d_status, d_workspace, ws_bytes, ws_needed,
                               stream);
}
