// clearcam_b200 — parameter blocks + launchers of the non-GEMM kernels on the hot path.
// All activations are NHWC; a tensor is addressed as (base pointer, channel stride `cs` = channels per
// pixel of the underlying buffer, channel offset `co`, channel count) so concat/chunk are free.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "clearcam_b200.h"

namespace cc {

struct DirectConvParams {
  const __nv_bfloat16* in; int in_cs, in_co, Cin;
  int N, Hin, Win;        // logical input extent used for bounds (may be smaller than the stored buffer)
  int Hbuf, Wbuf;         // stored buffer extent (row/col pitch)
  int k, stride, pad, groups;
  const __nv_bfloat16* w; // [Cout][k][k][Cin/groups]
  const float* bias;
  void* out; int out_cs, out_co, Cout, out_f32;
  int Hout, Wout;
  int act;
  const void* res; int res_cs, res_co;
};
int conv_direct_launch(const DirectConvParams& p, cudaStream_t stream);

// An NHWC tensor slice: bf16 elements, or float when f32 != 0 (fp32-accurate mode; cs / co / C count elements either way
// and p is then really a float*).
struct TSlice {
  __nv_bfloat16* p; int cs, co, C;   // buffer base, channels per pixel, first channel, channel count
  int N, H, W;
  int f32;
};
// Channels [co, co + C) of a buffer of cs channels per pixel.  The pixel extent may stay 0 where the reader fixes it: a conv's
// output and residual slices take the extent that follows from its input and stride (ConvDesc).
inline TSlice nhwc_slice(const void* p, int cs, int co, int C, int f32 = 0, int N = 0, int H = 0, int W = 0) {
  return TSlice{static_cast<__nv_bfloat16*>(const_cast<void*>(p)), cs, co, C, N, H, W, f32};
}
// A dense fp32 map of C channels per pixel (the head logits, the fused-upsample addend, the fp32-accurate partial sums)
inline TSlice dense_f32(const float* p, int C) { return nhwc_slice(p, C, 0, C, 1); }

// fp32-accurate mode: fp32 activation slice -> six bf16 planes per pixel [lo | mid | hi | mid | hi | hi] (x = hi + mid + lo
// exactly, each a bf16), the A operand of a tensor-core conv whose weights are laid out [hi | mid | lo | hi | mid | hi]:
// the six products with combined weight >= 2^-16 of an fp32 x fp32 product, smallest first.  out: dense [N*H*W][6*C] bf16.
int split_planes_launch(const TSlice& in, __nv_bfloat16* out, cudaStream_t s);

// fp32-accurate mode, last pass of a conv: out = [res +] act(acc + bias) over npix x C; acc dense [npix][C]; out / res fp32 slices
struct FinishParams {
  const float* acc; const float* bias; int act;
  long long npix; int C;
  float* out; int out_cs, out_co;
  const float* res; int res_cs, res_co;
};
int finish_f32_launch(const FinishParams& p, cudaStream_t s);

// avg_pool2d(k=2,s=1,p=0) written into a same-size map whose last row/col are zero (so the stride-2 conv that
// follows can use the even "pixel pair" TMA view).  detection/yolov9.py:47 (ADown), :62 (AConv).
int avgpool2_pad_launch(const TSlice& in, const TSlice& out, cudaStream_t s);
// max_pool2d(k=3,s=2,p=1) of avg_pool2d(k=2,s=1) in one pass (ADown second branch, detection/yolov9.py:47-50).
int avgmax_pool_launch(const TSlice& in, const TSlice& out, cudaStream_t s);
// max_pool2d(k=5,s=1,p=2)  (SP, detection/yolov9.py:127-132)
int maxpool5_launch(const TSlice& in, const TSlice& out, cudaStream_t s);
// the three cascaded SP pools of SPPELAN (detection/yolov9.py:134-149) in one launch: reads channels [0, c1) of the concat
// buffer `cat`, writes [c1, 2c1), [2c1, 3c1), [3c1, 4c1)
bool spp3_supported(const TSlice& cat, int c1);
int spp3_launch(const TSlice& cat, int c1, cudaStream_t s);
// nearest x2 upsample (Upsample, detection/yolov9.py:285-292)
int upsample2_launch(const TSlice& in, const TSlice& out, cudaStream_t s);
// CBFuse (detection/yolov9.py:230-245): out = sum_i nearest_resize(src_i) + last
struct CBFuseParams { TSlice src[5]; int nsrc; TSlice last; TSlice out; int shift[5]; };   // shift: filled by the launcher (log2 of out/src, -1 = general)
int cbfuse_launch(const CBFuseParams& p, cudaStream_t s);

// One I420 pixel as BGR, bit-exact with cv2.cvtColor(COLOR_YUV2BGR_I420): BT.601 limited range in 20-bit fixed point,
// the chroma sample of the 2x2 block holding frame pixel (y, x).  Used per tap by the letterbox and the crop kernels.
// The products stay within int32; >> is arithmetic on the negative sums.
__device__ __forceinline__ void i420_bgr(const uint8_t* __restrict__ fr, int H, int W, int y, int x, int bgr[3]) {
  const int hw = H * W, cw = W >> 1, ci = (y >> 1) * cw + (x >> 1);
  const int Y = __ldg(fr + y * W + x), u = __ldg(fr + hw + ci) - 128, v = __ldg(fr + hw + (hw >> 2) + ci) - 128;
  const int yy = max(Y - 16, 0) * 1220542 + (1 << 19);
  bgr[0] = min(max((yy + 2116026 * u) >> 20, 0), 255);
  bgr[1] = min(max((yy - 852492 * v - 409993 * u) >> 20, 0), 255);
  bgr[2] = min(max((yy + 1673527 * v) >> 20, 0), 255);
}

// Where the crop kernels (JPEG transform, CLIP crop-resize) read one crop: its frame and that frame's extent and format.
// Every crop carries its own source, so one launch cuts crops out of frames of different shapes and formats; the format
// branch is uniform per CTA.  fmt: 0 RGB or 1 BGR (packed [H,W,3]), 2 I420 ([H*3/2,W], H and W even).
struct CropSource { const uint8_t* frame; int H, W, fmt; };
// The sources of a frame-table call (CC_FRAME_RGB_U8 -> RGB, CC_FRAME_BGR_U8 -> BGR, CC_FRAME_I420_U8 -> I420), after
// checking the table and that every rect (frame, x1, y1, x2, y2) is non-empty and inside its own frame; CC_ERR_INVALID
// names the first bad entry.
int table_crop_sources(const char* who, const cc_frame* frames, int n_frames, const int32_t* rects, int K, CropSource* src);
// What a frame-table JPEG call checks beyond table_crop_sources (jpeg.cu): the quality and the 16-bit header sizes.
int check_table_jpeg(const char* who, const int32_t* rects, int K, int quality);
// The JPEG transform of crops whose sources and rects are checked (jpeg.cu): the cc_jpeg_coeffs_frames tap.
int jpeg_coeffs_sources(const CropSource* src, const int32_t* rects, int K, int quality, int16_t* d_coef, int64_t* n_blocks,
                        cudaStream_t st);

// Letterbox: bilinear resize (utils/helpers.py:127-131 semantics, W axis first then H, result cast to the
// input dtype after each axis) + zero pad (detection/yolov9.py:390-404).  fmt: a CC_FRAME_* code; out is HWC BGR, float32
// for CC_FRAME_BGR_F32, else uint8 (I420 taps are converted to BGR before the interpolation).
struct LetterboxParams {
  const void* in; void* out; int fmt;
  int B, Hin, Win, Hr, Wr, pad_y, pad_x, Hout, Wout;   // resized extent, pads, final extent
  float sx, sy;                                        // float(Win/Wr), float(Hin/Hr) computed in double on the host
};
// B frames of one shape and format (in = the first, the others follow contiguously) -> [B,Hout,Wout,3]
int letterbox_launch(const LetterboxParams& p, cudaStream_t s);
// The same kernel driven by a per-image table (frames of different shapes and formats into one [B,Hout,Wout,3] batch).  The
// table travels as the kernel parameter: no copy, no allocation, no sync.
struct LetterboxFrame {
  const void* in;                                      // the frame, or nullptr: a padding image, written as zeros
  int fmt, Hin, Win, Hr, Wr, pad_y, pad_x;
  float sx, sy;
};
struct LetterboxTable {
  void* out; int B, Hout, Wout, out_f32;               // out: float32 when out_f32 (CC_FRAME_BGR_F32 frames), else uint8
  LetterboxFrame f[CC_MAX_FRAMES];
};
int letterbox_frames_launch(const LetterboxTable& t, cudaStream_t s);

// Stem: frame[..., ::-1]/255 -> Conv 3x3 s2 p1 (Cin=3) -> bias -> SiLU -> NHWC bf16
// (detection/yolov9.py:378-379 fused into model[0] / model[1],model[15] of size e).  fp32 weights [Cout][3][3][3] (RGB order).
struct StemParams {
  const void* in; int is_f32; int B, H, W;    // HWC BGR frame(s)
  const float* w; const float* bias; int Cout;
  TSlice out;                                  // [B,H/2,W/2,Cout]
};
int stem_launch(const StemParams& p, cudaStream_t s);
// uint8 stem on tensor cores (stem_tc.cu): the A tile is gathered from the frame into shared memory by the CTA itself.
// Built once per plan (output tensor map), launched with the frame pointer of the call.
struct StemTcParams {
  CUtensorMap tmC;           // 2-D [Mrows][Cout] bf16 view of the output slice (row pitch = cs), box [128][Cout]
  const uint8_t* in;         // [B][H][W][3] BGR
  const __nv_bfloat16* w;    // [Cout][32]
  const float* bias;         // [Cout]
  int B, H, W, Cout;
  long long Mrows;
  int tiles;
};
int stem_tc_build(int B, int H, int W, const __nv_bfloat16* w32, const float* bias, int Cout, const TSlice& out, StemTcParams* p);
int stem_tc_launch(const StemTcParams& p, const uint8_t* frames, cudaStream_t s);

// Detect head tail: DFL softmax-expectation, dist2bbox, x stride, sigmoid, max/argmax, conf threshold
// (detection/yolov9.py:209-219, 273-282, 263-271, 440-448).  Inputs are the fp32 logits of the three scales.
struct DecodeParams {
  const float* box[3]; const float* cls[3];   // [B,h,w,64], [B,h,w,80] fp32
  int h[3], w[3]; float stride[3];
  int B, A;                                   // A = sum h*w
  float conf_thr;
  float* pred;                                // [B,A,6] x1,y1,x2,y2,prob(>=thr else 0),class
  float* raw;                                 // optional [B,84,A] (xc,yc,w,h,80 probs) for parity taps, or nullptr
};
int decode_launch(const DecodeParams& p, cudaStream_t s);

// head of postprocess (detection/yolov9.py:440-448) on a [B, 4+nc, A] head output -> pred [B, A, 6]
int pred_from_raw_launch(const float* raw, int B, int A, int nc, float conf_thr, float* pred, cudaStream_t s);

// postprocess tail (detection/yolov9.py:449-458) + scale_boxes/clip_boxes (:406-421), one CTA per image.
struct PostScale { float pad_x, pad_y, gain, clip_w, clip_h; };   // scale_boxes of one image
struct PostParams {
  const float* pred; int B, A; int max_det; float iou_thr;
  PostScale scale; int do_scale;              // one scale_boxes for the whole batch
  float* out;                                 // [B,max_det,6]
};
// per_image: NULL (every image takes p.scale), or B <= CC_MAX_FRAMES entries, image b taking per_image[b]; either way the
// scales reach the kernel as a parameter table
int postprocess_launch(const PostParams& p, cudaStream_t s, const PostScale* per_image = nullptr);

// ---- CLIP ViT kernels (vit.cu) ----
int patchify_launch(const float* x, __nv_bfloat16* out, int B, int S, int p, int Kpad, cudaStream_t st);
int embed_ln_pre_launch(float* x, const float* cls, const float* pos, const float* gamma, const float* beta, int rows, int L,
                        int W, cudaStream_t st);
int layernorm_bf16_launch(const float* x, __nv_bfloat16* out, const float* gamma, const float* beta, int rows, int W,
                          long long row_stride, const int* row_idx, cudaStream_t st);
int text_embed_launch(const int* ids, const float* tok, const float* pos, float* x, int* eot_row, int B, int L, int W,
                      int vocab, cudaStream_t st);
int l2norm_launch(const float* in, float* out, int rows, int D, long long out_stride, float eps, cudaStream_t st);
bool layernorm_width_supported(int W);   // the widths the LayerNorm kernels are instantiated for: 128 x {1..6, 8, 10, 12}
int attention_launch(const __nv_bfloat16* qkv, __nv_bfloat16* ctx, int B, int L, int H, int causal, cudaStream_t st);
int attention_max_len();      // longest sequence whose K and V fit the mma.sync kernel's shared memory
// wgmma attention (attention_tc.cu); vt_ws: workspace of attention_tc_workspace_bytes() for the per-head V^T copy
bool attention_tc_supported(int L);
int attention_tc_max_len();
size_t attention_tc_workspace_bytes(int B, int L, int H);
int attention_tc_launch(const __nv_bfloat16* qkv, __nv_bfloat16* ctx, __nv_bfloat16* vt_ws, int B, int L, int H, int causal,
                        cudaStream_t st);
int search_scores_launch(const float* index, const float* q, float* scores, int N, int D, int Q, cudaStream_t st);
int search_topk_launch(const float* index, const float* q, const int* group, const uint8_t* mask, unsigned long long* best, int N, int D,
                       int G, int k, int* out_rows, float* out_scores, cudaStream_t st);

}  // namespace cc
