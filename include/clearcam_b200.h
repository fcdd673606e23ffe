/* clearcam_b200 — C-ABI of the H100-native per-frame vision hot path of roryclear/clearcam.
 *
 * The reference has no FFI: its boundary is Python call signatures (SURVEY.md §8b).  This header is the
 * C-ABI that sits UNDER those signatures; clearcam_b200/detection/yolov9.py and clearcam_b200/models/objects.py
 * bind it with ctypes and keep the reference's names/arguments.  Conventions:
 *   - every function returns int: 0 = ok, <0 = error (cc_last_error() gives the message); nothing aborts/throws
 *     (the reference's caller supervises failures itself: clearcam.py:543-546);
 *   - all pointers named d_* are DEVICE pointers owned by the caller (torch tensors on the Python side);
 *     h_* are host pointers; `stream` is a cudaStream_t passed as void* (NULL = default stream);
 *   - calls are stream-ordered and never synchronise; one handle per GPU, not thread-safe per handle
 *     (the reference funnels all model calls to one thread: clearcam.py:1214-1226);
 *   - activations are NHWC, bf16 unless stated; a tensor slice is (ptr, cs = channels per pixel of the
 *     underlying buffer, co = first channel, C = channel count).
 */
#ifndef CLEARCAM_B200_H
#define CLEARCAM_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CC_ABI_VERSION 5

int cc_version(void);
const char* cc_last_error(void);
/* number of SMs of the current device if it is sm_90 (H100), else <0 */
int cc_device_check(void);

/* activation codes */
#define CC_ACT_NONE 0
#define CC_ACT_SILU 1      /* x*sigmoid(x): detection/yolov9.py:38 */
#define CC_ACT_GELU_TANH 2 /* tinygrad Tensor.gelu(): models/objects.py:125,179 */
#define CC_ACT_PRELU 3     /* where(x > 0, x, slope * x): models/adaface.py:54,86 (the face embedder; see cc_conv_op) */

/* ---- kernel-level ops (used by the graphs below and exposed for the parity tests) ---- */

/* One conv launch, as cc_conv takes it and as cc_yolo_op_conv / cc_clip_op_conv / cc_face_op_conv report a plan's launch: Conv2d(bias) [+act] [+residual], k in
 * {1,3}, stride in {1,2}, pad = k/2, NHWC bf16 in, bf16|fp32 out.  Replaces nn.Conv2d + .silu() of detection/yolov9.py:33-38
 * (and the bare nn.Conv2d of :173,:186,:224).
 *   kind     CC_CONV_OP_GEMM: the wgmma implicit-GEMM kernel; CC_CONV_OP_CHAIN: the same with a 1x1 conv in its epilogue;
 *            CC_CONV_OP_DIRECT: the CUDA-core direct kernel, the only one that takes groups != 1.  The plan taps report
 *            CC_CONV_OP_NONE for an op that is not a conv (the rest is then zero), and name: the op's name.
 *   in, out, res  NHWC slices (cc_slice: buffer p, channels per pixel cs, first channel co, channels C, extent N x H x W,
 *            f32: float elements, else bf16).  in is bf16, Cin = in.C; Cout = out.C; res (res.p == NULL: none) has out's
 *            dtype, is added after the activation and may be the output slice itself.  out and res have the output extent
 *            N x Ho x Wo of in's N x H x W: Ho = (H - 1) / stride + 1, Wo likewise.
 *   w, bias  bf16 [Cout][k][k][Cin/groups]; fp32 [Cout] or NULL.
 *   act      CC_ACT_*.  CC_ACT_PRELU is the face embedder's epilogue (wgmma, bf16 out only):
 *              out = where(y > 0, y, slope[c] * y) (+ res),  y = conv(x) + bias[cls][c]
 *            where cls = 3 * (h == 0 ? 0 : h == Ho-1 ? 2 : 1) + (w == 0 ? 0 : w == Wo-1 ? 2 : 1) is the output pixel's border
 *            class; bias is then the fp32 [9][Cout] table and slope fp32 [Cout] (NULL for the other activations).  A
 *            per-channel affine map applied before a zero-padded 3x3 conv folds into the weights and this table exactly (the
 *            shift summed over the taps inside the map).
 *   pre      NULL, or the fused Upsample -> Concat addend (wgmma only): out = act(conv(x) + bias + pre[n, h/2, w/2, :]) [the
 *            first conv of a RepNCSPELAN4 after an upsample].  pre: dense fp32 [N][pre_h][pre_w][Cout], 16-byte aligned; Ho
 *            and Wo even, pre_h = Ho/2, pre_w = Wo/2.
 *   CHAIN    a SiLU conv into bf16 and the square 1x1 conv w2 (bf16 [Cout2][Cout2], Cout2 = out2.C), bias2, act2 whose input
 *            is the first conv's output channels [k0, k0 + Cout2 - part.C) followed by the partner slice `part` (bf16, same
 *            pixels; part.p == NULL: none), into out2: CC_ACT_SILU into bf16 or CC_ACT_NONE into fp32.  store1 = 0 drops
 *            the first output (out.p may then be NULL; out.C still gives Cout).  The results equal the two convs launched
 *            one after the other bit for bit.
 *   BN       an upper bound on the wgmma N tile that also keeps every tile that wide; 0 = the planner chooses.  Reported:
 *            the N tile as built.
 *   BK .. narrow_tiles  reported only (cc_conv ignores them), the tiling of a tensor-core launch as built: K block BK, the
 *            128-pixel tile box 2^lTW x 2^lTH x 2^lTN (w, h, images), the stride-2 pair view s2, the pipeline stages,
 *            resident weights b_res, the persistent grid and the tile count; BNn, the narrow tile width (0: every tile is BN
 *            wide), and how many of the tiles are that narrow (the last wave's tiles split along N, and the remainder channel
 *            block when BN does not divide Cout).
 *   out_ns   pixels per image in the out and res buffers, 0 = dense (Ho * Wo).  A larger pitch leaves the pixels past Ho * Wo
 *            of each image untouched (the CLIP patch embedding writes tokens 1..L-1 of each image's L-row stream this way:
 *            out.p one row past the buffer's start, Ho * Wo = L - 1, out_ns = L).  GEMM kind only; out_ns < Ho * Wo fails. */
#define CC_CONV_OP_NONE 0
#define CC_CONV_OP_GEMM 1
#define CC_CONV_OP_CHAIN 2
#define CC_CONV_OP_DIRECT 3
typedef struct { void* p; int cs, co, C, N, H, W, f32; } cc_slice;
typedef struct {
  int kind;
  char name[128];
  cc_slice in, out, res;
  const void* w; const float* bias; int k, stride, groups, act; const float* slope;
  const float* pre; int pre_h, pre_w;
  const void* w2; const float* bias2; int act2, k0; cc_slice part, out2; int store1;
  int BN, BK, lTW, lTH, lTN, s2, stages, b_res, grid, num_tiles;
  int BNn, narrow_tiles;
  int out_ns;
} cc_conv_op;
/* Launches the conv *op describes.  A kind other than GEMM, CHAIN or DIRECT, a NULL input, weight or output pointer, a slice
 * whose extent is not the conv's, a shape the chosen kernel does not take or a pair the kernel cannot chain (see conv_gemm.cu
 * conv_gemm_chain_build) fails with CC_ERR_INVALID before anything is launched. */
int cc_conv(const cc_conv_op* op, void* stream);

/* ---- YOLOv9 detector (replaces detection/yolov9.py: class YOLOv9, :298-458) ---- */
typedef struct cc_yolo cc_yolo;

/* size: "t"|"s"|"c"|"e" as the reference defines them (detection/yolov9.py:461-464), or "t@16"|"m@16": the zero-padded
 * equivalents of t and m (every width a multiple of 16; same function) whose weights the host produces from the
 * reference's by scattering them into the padded layout (clearcam_b200/detection/padding.py `pad_state_dict`).  Literal
 * "m" is not accepted by the plan builder (widths 60/90/184 break the 16-byte slice alignment); literal "t" runs with its
 * 24-channel convs on the generic CUDA-core kernel.
 * Weights: n host fp32 tensors in PyTorch layout, named with the reference's state-dict keys with `.list.`
 * elided, e.g. "model.0.conv.weight", "model.2.cv2.0.cv1.conv.bias", "model.22.cv2.0.2.weight"
 * (what safe_load/load_state_dict consume at detection/yolov9.py:372-373).  They are repacked to the kernel
 * layout and uploaded once; the host pointers are not retained. */
int cc_yolo_create(const char* size, int n_tensors, const char* const* names, const float* const* h_data,
                   const int64_t* numels, cc_yolo** out);
/* Same with options.  CC_YOLO_FP32_ACCURATE: the fp32-accurate mode — activations stored in fp32, every conv as six
 * bf16 plane products of a 3-way split of both operands on the same wgmma kernel (fp32 accumulation), exact SiLU.  The
 * reference computes in fp32 end to end (SURVEY.md §2.1); this is the mode whose boxes / scores are compared with the fp32
 * oracle at the north-star tolerance.  Costs ~6x the tensor work and 2x the activation bytes of the default (bf16) mode. */
#define CC_YOLO_FP32_ACCURATE 1
int cc_yolo_create_ex(const char* size, int flags, int n_tensors, const char* const* names, const float* const* h_data,
                      const int64_t* numels, cc_yolo** out);
int cc_yolo_destroy(cc_yolo* h);

/* Frame formats (the frame_fmt argument of the detector entry points and cc_letterbox):
 *   CC_FRAME_BGR_U8  [B,Hf,Wf,3] HWC BGR uint8 (clearcam.py:582, ffmpeg -pix_fmt bgr24);
 *   CC_FRAME_BGR_F32 [B,Hf,Wf,3] HWC BGR float32 (test/run_mot.py:33);
 *   CC_FRAME_I420_U8 [B,Hf*3/2,Wf] uint8 planar YUV 4:2:0 (ffmpeg -pix_fmt yuv420p, OpenCV I420): the Y plane Hf x Wf, then
 *                    U and V, each (Hf/2) x (Wf/2); Hf and Wf must be even.  Converted to BGR on the device exactly as
 *                    cv2.cvtColor(yuv, COLOR_YUV2BGR_I420) does (BT.601 limited range, 20-bit fixed point, nearest chroma);
 *   CC_FRAME_RGB_U8  [h,w,3] HWC RGB uint8, in the frame tables of the crop entry points only (cc_clip_preprocess_frames,
 *                    cc_jpeg_encode_crops_frames, cc_jpeg_coeffs_frames, cc_jpeg_crops_decoded_frames); every other entry
 *                    point refuses it.
 * Any other code, or an odd Hf / Wf with I420, fails with CC_ERR_INVALID before anything is launched. */
#define CC_FRAME_BGR_U8 0
#define CC_FRAME_BGR_F32 1
#define CC_FRAME_I420_U8 2
#define CC_FRAME_RGB_U8 3

/* YOLOv9.__call__ (detection/yolov9.py:375-388) for a batch of same-shape frames.
 * d_frames: B frames of format frame_fmt, Hf x Wf pixels each.
 * d_out: [B,300,6] fp32 rows [x1,y1,x2,y2,conf,class] in frame pixels, descending conf, suppressed rows all-zero.
 * d_raw: optional [B,84,A] fp32 tap of the head output (xc,yc,w,h,80 class probs) for parity tests, or NULL.
 * A plan (buffers, TMA descriptors) is built and cached on the first call for each (dtype,B,Hf,Wf,res) — the
 * analogue of jit_infer's per-shape TinyJit cache (utils/helpers.py:214-221); later calls only launch kernels. */
int cc_yolo_forward(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, float* d_out,
                    float* d_raw, void* stream);
/* Frames of different shapes and formats in one forward.  Every camera whose frames letterbox to the same net input
 * (720p, 1080p, 1440p and 2160p all give 384 x 640 at res 640) runs in one batch: the letterbox reads a per-frame table,
 * the conv stack is that of a uniform batch of the net shape, and scale_boxes takes each frame's own geometry.
 * cc_frame: data = device pointer to one frame (CC_FRAME_BGR_U8 [h,w,3] or CC_FRAME_I420_U8 [h*3/2,w], h and w even), or
 * NULL for a padding row (letterboxed as zeros; its output rows mean nothing).  At most CC_MAX_FRAMES frames per call. */
#define CC_MAX_FRAMES 128
typedef struct { const void* data; int fmt; int h; int w; } cc_frame;
/* The net input extent (the letterboxed extent rounded up to a multiple of 32) of an Hf x Wf frame at `res`: the key under
 * which frames can share a batch.  Host only: needs no GPU. */
int cc_yolo_net_shape(int frame_fmt, int Hf, int Wf, int res, int* net_h, int* net_w);
/* cc_yolo_forward over a table of B frames (HOST array, read during the call only) that share one net shape; row b of
 * d_out [B,300,6] is frame b's detections in its own pixels, as cc_yolo_forward of a batch of frames of its shape and
 * format would give it at that row.  d_raw: optional [B,84,A] head tap.  Mixed net shapes, CC_FRAME_BGR_F32 or
 * CC_FRAME_RGB_U8 frames, odd I420 sides, no frame at all or B > CC_MAX_FRAMES fail with CC_ERR_INVALID before anything is launched.  Plans are
 * cached per (B, net shape, res); the letterbox and the postprocess take the table as a kernel parameter on every call and
 * the CUDA graph covers the launches between them, so a different table every call still replays the graph. */
int cc_yolo_forward_frames(cc_yolo* h, const cc_frame* frames, int B, int res, float* d_out, float* d_raw, void* stream);
int cc_yolo_workspace_bytes_frames(cc_yolo* h, const cc_frame* frames, int B, int res, size_t* bytes);

/* plan facts: letterboxed net input size, anchors, kernel launches per forward, algorithmic conv FLOPs,
 * bytes of activation workspace */
int cc_yolo_plan_info(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int* net_h, int* net_w, int* anchors,
                      int* launches, double* conv_flops, double* act_bytes);

/* Workspace.  Every cached plan of a handle carves its activations out of ONE device workspace (size of the largest plan;
 * at most 16 plans are kept, least recently used goes first), so a process that sees many batch sizes / frame shapes does
 * not accumulate buffers.  By default the library owns it and grows it on demand (a growth frees and reallocates: it
 * synchronises the device once, and the plans of the old workspace are rebuilt on their next use).  A caller that wants no
 * allocation after start-up sizes it with cc_yolo_workspace_bytes for its largest shape and hands it over with
 * cc_yolo_set_workspace (256-byte aligned device memory, owned by the caller; d_workspace = NULL returns to the
 * library-owned one); a plan that does not fit a caller-owned workspace fails with CC_ERR_INVALID.  The plans of one
 * handle share the memory: run them in stream order (one stream per handle). */
int cc_yolo_workspace_bytes(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, size_t* bytes);
int cc_yolo_set_workspace(cc_yolo* h, void* d_workspace, size_t bytes);

/* measurement: per-op device time of one forward (CUDA events between launches on `stream`; synchronises).
 * Up to `cap` entries of ms / algorithmic conv FLOPs / algorithmic HBM bytes / kernel kind / op name (pointers valid
 * while h lives). */
int cc_yolo_profile(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, float* d_out, int cap,
                    float* ms, double* flops, double* bytes, const char** kinds, const char** names, int* n_ops, void* stream);

/* measurement: in-situ device timeline of one forward, no events between the launches (so programmatic dependent launch
 * overlaps exactly as in production).  For op i, host_ns[12i..12i+11] = globaltimer ns of (first CTA entered, grid
 * dependency released, last CTA exited; then of CTA 0: first operands landed, all MMAs issued, first accumulator complete,
 * last epilogue group done, exit; then four stamps inside the first staging pass of its first tile) for the tensor-core conv launches, zeros for the other kernels.  Synchronises. */
int cc_yolo_trace(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, float* d_out, int cap,
                  unsigned long long* host_ns, const char** kinds, const char** names, double* flops, int* n_ops, void* stream);

/* Conv op taps, for tests that check every conv launch of a plan in place, one op at a time.
 * cc_yolo_op_conv describes op i of the cached plan of this shape (built on first use, as cc_yolo_forward would) and returns
 * the plan's op count (a cc_conv_op, see above, with the tiling as built); out == NULL only returns the count, an i outside
 * [0, count) fails with CC_ERR_INVALID.
 * cc_yolo_run_ops launches ops [first, last) of that plan on `stream` exactly as a forward launches them, without a CUDA
 * graph; d_frames, d_out and d_raw are a cc_yolo_forward call's.  Nothing synchronises. */
int cc_yolo_op_conv(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int i, cc_conv_op* out);
/* Operand taps, for tests that check every launch of a plan in place: what op i of a plan reads and writes, for every op,
 * convs included.  Each operand is a slice of type cc_slice, whose f32 field mirrors type == CC_OP_F32, with an element type and ns, the
 * elements ("pixels") from one image to the next (0: dense, H * W).  A row-major matrix of R rows of C values per image is
 * N images of H = 1, W = R pixels of cs values.  An operand with p == NULL is the call's own input (frames, images, token ids,
 * faces), output or raw tap, with its extent filled in (an output's cs is its row width; the call picks the row stride).
 * Operand order per kind (in: what the op reads; out: what it writes; [x]: only when present):
 *   conv_gemm, conv_direct  in: in, [res], [pre], [part]   out: [out] (a stored first output), [out2] (a chained 1x1)
 *                           (the weights are in the cc_*_op_conv descriptor of the same op)
 *   letterbox          in: frames (u8 [B,Hf,Wf,3], f32 for CC_FRAME_BGR_F32, u8 [B,Hf*3/2,Wf,1] for I420)  out: net input
 *   stem, stem_tc      in: net input (the letterbox's output, or the call's frames), w (f32 [Cout][3][3][3], (kh, kw, RGB)
 *                      order, before any packing), bias (f32 [Cout])   out: the first map
 *   avgpool2_pad, avgmax_pool, maxpool5, upsample2   in: in   out: out
 *   spp3               in: channels [co, co + c1) of the concat buffer   out: channels [co + c1, co + 4 c1)
 *   cbfuse             in: src_0 .. src_{n-1}, last   out: out
 *   split_planes       in: in (f32)   out: the dense bf16 planes [N,H,W][6C]
 *   finish_f32         in: acc (dense f32), bias, [res]   out: out.  Scalar: act
 *   decode             in: box_0..2 (f32 [B,h,w,64]), cls_0..2 (f32 [B,h,w,80])   out: pred (f32 [B,1,A,6]), raw tap
 *                      (p NULL, f32 [B,84,A,1]).  Scalar: conf_thr
 *   postprocess        in: pred   out: detections (p NULL, f32 [B,1,max_det,6]).  Scalars: max_det, iou_thr, scale_boxes'
 *                      pad_x, pad_y, gain, clip_w, clip_h (do_scale = 0: none)
 *   patchify           in: images (p NULL, f32 [B,3,S,S] as [B,3S,S,1])   out: patches (bf16 [B,1,Pn,Kpad]).  Scalar: patch
 *   embed_ln_pre       in: stream (f32 [B,1,L,W]), cls (f32 [1,1,1,W]), pos ([1,1,L,W]), gamma, beta ([W])   out: stream
 *   text_embed         in: ids (p NULL, i32 [B,1,L,1]), tok ([1,1,vocab,W]), pos ([1,1,L,W])   out: stream (f32 [B,1,L,W]),
 *                      EOT rows (i32 [B,1,1,1]: b * L + the EOT's position)
 *   layernorm          in: x, gamma, beta, [row index (i32 [B,1,1,1])]   out: bf16 rows.  x is the rows read: every row of
 *                      the stream ([B,1,L,W]), token 0 of each image ([B,1,1,W], ns = L), or with a row index the whole stream
 *   attention          in: qkv (bf16 [B,1,L,3*heads*64])   out: ctx (bf16 [B,1,L,heads*64]), [the wgmma kernel's V^T
 *                      scratch (bf16 [B,heads*64,Lpad,1])].  Scalar: causal
 *   l2norm             in: embeddings (f32 [B,1,1,D])   out: the call's output rows (p NULL, [B,1,1,D]).  Scalar: eps
 *   face_pack          in: faces (p NULL, u8 [B,112,112,3])   out: bf16 [B,112,112,16] (channels 3..15 zero)
 * Same contract as cc_yolo_op_conv: the op count, out == NULL only counts, an i outside [0, count) fails. */
#define CC_OP_U8 0
#define CC_OP_BF16 1
#define CC_OP_F32 2
#define CC_OP_I32 3
#define CC_OP_IO_MAX 8
typedef struct { cc_slice s; int type; int ns; } cc_operand;
typedef struct {
  char kind[32];
  char name[128];
  int n_in, n_out;
  cc_operand in[CC_OP_IO_MAX], out[CC_OP_IO_MAX];
  int causal;                                  /* attention */
  float eps;                                   /* l2norm */
  float conf_thr;                              /* decode */
  int max_det; float iou_thr;                  /* postprocess */
  int do_scale; float pad_x, pad_y, gain, clip_w, clip_h;
  int act;                                     /* finish_f32 */
  int patch;                                   /* patchify */
} cc_op_io;
int cc_yolo_op_io(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int i, cc_op_io* out);
int cc_yolo_run_ops(cc_yolo* h, const void* d_frames, int frame_fmt, int B, int Hf, int Wf, int res, int first, int last,
                    float* d_out, float* d_raw, void* stream);

/* parity tap: after a forward, copy the output of graph layer `layer` (index into the reference's self.model list,
 * detection/yolov9.py:303-371) to dense fp32 [B,H,W,C].  d_dst == NULL only queries C/H/W (C = 0: no tensor). */
int cc_yolo_layer_output(cc_yolo* h, int frame_fmt, int B, int Hf, int Wf, int res, int layer, float* d_dst, int* C,
                         int* H, int* W, void* stream);

/* kernel-level taps (parity tests) */
/* postprocess tail (detection/yolov9.py:449-458) [+ scale_boxes :406-421 when do_scale]: d_pred [B,A,6] ->
 * d_out [B,max_det,6] */
int cc_detect_postprocess(const float* d_pred, int B, int A, int max_det, float iou_thr, int do_scale, float pad_x,
                          float pad_y, float gain, float clip_w, float clip_h, float* d_out, void* stream);
/* head of the standalone postprocess(output) (detection/yolov9.py:440-448): d_raw [B, 4+n_classes, A] = xc, yc, w, h, class
 * probabilities -> d_pred [B,A,6] = x1, y1, x2, y2, max probability (0 below conf_thr), first argmax */
int cc_detect_pred_from_raw(const float* d_raw, int B, int n_classes, int A, float conf_thr, float* d_pred, void* stream);
/* DDetect tail (detection/yolov9.py:209-219) + head of postprocess (:440-448): three scales of fp32 logits
 * d_box[i] [B,h,w,64], d_cls[i] [B,h,w,80] (strides 8,16,32) -> d_pred [B,A,6], optional d_raw [B,84,A] */
int cc_detect_decode(const float* const* d_box, const float* const* d_cls, const int* hs, const int* ws, int B,
                     float conf_thr, float* d_pred, float* d_raw, void* stream);
/* YOLOv9.preprocess (detection/yolov9.py:390-404) + resize (utils/helpers.py:127-131): B frames of format frame_fmt,
 * Hin x Win pixels -> letterboxed BGR [B,out_h,out_w,3], float32 for CC_FRAME_BGR_F32, else uint8 (an I420 frame is
 * converted to BGR at each bilinear tap).  d_out == NULL only queries the output size. */
int cc_letterbox(const void* d_in, int frame_fmt, int B, int Hin, int Win, int res, void* d_out, int* out_h, int* out_w,
                 void* stream);
/* The same for a table of B frames sharing one net shape (cc_yolo_forward_frames' rules): frame b is letterboxed into row b
 * of d_out uint8 [B,net_h,net_w,3], its cc_letterbox extent at the top left and zeros past it; a NULL frame gives a zero
 * row.  d_out == NULL only queries net_h / net_w. */
int cc_letterbox_frames(const cc_frame* frames, int B, int res, void* d_out, int* net_h, int* net_w, void* stream);
/* CLIP multi-head attention (models/objects.py:108-118, :157-168), d_head = 64: per (image, head)
 * ctx = softmax(Q K^T / 8 [+ causal mask when causal != 0]) V.  d_qkv: bf16 [B*L, 3*H*64], the fused Q | K | V rows the
 * encoder plans pass; d_ctx: bf16 [B*L, H*64].  impl: 1 = the mma.sync kernel (vit.cu, L <= 704), 2 = the wgmma kernel
 * (attention_tc.cu, L <= 384); there is no automatic choice here.  d_ws: device scratch of *ws_needed bytes (the wgmma
 * kernel's V^T copy; 0 bytes for impl 1), 16-byte aligned.  d_ctx == NULL only writes *ws_needed.  An unknown impl, a bad
 * shape, a sequence the kernel cannot hold or a short workspace fails with CC_ERR_INVALID before anything is launched. */
int cc_attention(const void* d_qkv, int B, int L, int H, int causal, int impl, void* d_ws, size_t ws_bytes, void* d_ctx,
                 size_t* ws_needed, void* stream);

/* The detector's memory-bound kernels as the plan runs them, on caller-owned NHWC slices (ptr, cs, co, C) of N x H x W maps.
 * f32: 0 = bf16 elements, 1 = fp32 (the fp32-accurate mode's activations).  Slices are 16-byte aligned with cs, co and C
 * multiples of 8 channels (of 4 for cc_split_planes / cc_finish_f32).  A bad argument fails with CC_ERR_INVALID before
 * anything is launched.
 * cc_pool op codes, output extent:
 *   CC_POOL_AVG2_PAD  avg_pool2d(2, 1) into an H x W map whose last row and column are zero (ADown / AConv), H, W >= 2;
 *   CC_POOL_AVGMAX    max_pool2d(3, 2, 1) of the stored avg_pool2d(2, 1) map (ADown), H and W even, output H/2 x W/2;
 *   CC_POOL_MAX5      max_pool2d(5, 1, 2) (SPPELAN), H x W;
 *   CC_POOL_UPSAMPLE2 nearest x2 (Upsample), output 2H x 2W. */
#define CC_POOL_AVG2_PAD 0
#define CC_POOL_AVGMAX 1
#define CC_POOL_MAX5 2
#define CC_POOL_UPSAMPLE2 3
int cc_pool(int op, int f32, const void* d_in, int N, int H, int W, int in_cs, int in_co, int C, void* d_out, int out_cs, int out_co,
            void* stream);
/* SPPELAN's three cascaded max_pool2d(5, 1, 2) in one launch, in place in the bf16 concat buffer: channels [co, co + c1)
 * are pooled into [co + c1, co + 2c1), then [co + 2c1, co + 3c1), then [co + 3c1, co + 4c1).  Only where the map fits shared
 * memory (H * W <= 800) and c1 is a multiple of 64; otherwise CC_ERR_INVALID. */
int cc_spp3(void* d_cat, int N, int H, int W, int cs, int co, int c1, void* stream);
/* CBFuse: out = sum_i nearest_resize(src_i, H x W) + last, summed in source order; 1 to 5 sources of C channels each,
 * source i of extent src_h[i] x src_w[i] at (d_src[i], src_cs[i], src_co[i]). */
int cc_cbfuse(int f32, int nsrc, const void* const* d_src, const int* src_h, const int* src_w, const int* src_cs, const int* src_co,
              const void* d_last, int last_cs, int last_co, void* d_out, int out_cs, int out_co, int N, int H, int W, int C,
              void* stream);
/* fp32-accurate mode: an fp32 slice of npix pixels -> dense bf16 [npix][6C] planes [lo | mid | hi | mid | hi | hi], x = hi + mid + lo. */
int cc_split_planes(const float* d_in, int npix, int cs, int co, int C, void* d_out, void* stream);
/* fp32-accurate mode, last pass of a conv: out = [res +] act(acc + bias), act 0 or 1 (exact SiLU); d_acc dense [npix][C];
 * d_bias [C] or NULL; d_res NULL or an fp32 slice. */
int cc_finish_f32(const float* d_acc, const float* d_bias, int act, int npix, int C, float* d_out, int out_cs, int out_co,
                  const float* d_res, int res_cs, int res_co, void* stream);
/* The detector's stem: frame[..., ::-1] / 255 -> conv 3x3 s2 p1 (Cin 3) -> bias -> SiLU.  d_frames [B,H,W,3] BGR, uint8 or
 * float32 (frame_f32); h_w: HOST fp32 [Cout][3][3][3] (PyTorch layout), h_bias: HOST fp32 [Cout], packed exactly as the
 * detector packs them; output slice [B,H/2,W/2] of bf16 or fp32 (out_f32).  impl 1 = the tensor-core stem (stem_tc: uint8 frames,
 * bf16 output, Cout 16, 32 or 64), 2 = the CUDA-core stem_kernel.  d_ws: *ws_needed bytes of device scratch for the packed
 * weights (16-byte aligned); d_out == NULL only writes *ws_needed. */
int cc_stem(const void* d_frames, int frame_f32, int B, int H, int W, const float* h_w, const float* h_bias, int Cout, void* d_out,
            int out_cs, int out_co, int out_f32, int impl, void* d_ws, size_t ws_bytes, size_t* ws_needed, void* stream);
/* One conv of the fp32-accurate mode, as the detector runs it: the six-plane split of the fp32 input slice, one GEMM per hi x hi
 * input-channel segment (at most 48 k16 steps each) accumulated in fp32, the cross-product GEMM, then [res +] act(acc + bias).
 * h_w: HOST fp32 [Cout][Cin][k][k], h_bias: HOST fp32 [Cout] or NULL; k 1 (stride 1) or 3 (stride 1 or 2); act 0 or 1; Cin and Cout
 * multiples of 16; d_in / d_res / d_out fp32 slices (cs, co multiples of 4).  d_ws: *ws_needed bytes of device scratch (planes,
 * partial sums, packed weights; 16-byte aligned); d_out == NULL only writes *ws_needed. */
int cc_conv2d_fp32_accurate(const float* d_in, int N, int Hin, int Win, int in_cs, int in_co, int Cin, const float* h_w,
                            const float* h_bias, int Cout, int k, int stride, int act, const float* d_res, int res_cs, int res_co,
                            float* d_out, int out_cs, int out_co, void* d_ws, size_t ws_bytes, size_t* ws_needed, void* stream);

/* The CLIP encoders' row kernels as the plans run them (one warp per row, fp32 statistics).  LayerNorm uses eps 1e-5 and takes
 * the widths W = 128 x {1, 2, 3, 4, 5, 6, 8, 10, 12}.  A bad argument fails with CC_ERR_INVALID before anything is launched.
 * cc_patchify: d_x fp32 [B,3,S,S] -> d_out bf16 [B*(S/p)^2][Kpad] (16-byte aligned), row b*(S/p)^2 + gy*(S/p) + gx holding
 *   x[b, c, gy*p + r, gx*p + s] in column c*p^2 + r*p + s and zeros in [3p^2, Kpad); S a multiple of p, Kpad a multiple of 8
 *   and >= 3p^2. */
int cc_patchify(const float* d_x, int B, int S, int p, int Kpad, void* d_out, void* stream);
/* In place on the fp32 stream d_x [B*L][W]: token 0 of every image becomes cls, every token t gets pos[t] added, then each row
 *   is LayerNorm'ed with d_gamma / d_beta (ln_pre).  Token 0's input rows are not read.  All pointers 16-byte aligned. */
int cc_clip_embed_ln(float* d_x, const float* d_cls, const float* d_pos, const float* d_gamma, const float* d_beta, int B, int L, int W,
                     void* stream);
/* d_out bf16 [rows][W] (dense, 8-byte aligned): row r = LayerNorm(x row src) * gamma + beta, with src = d_row_idx[r] when
 *   d_row_idx is not NULL (ln_final at the EOT rows; the indices must be rows of d_x) and r * row_stride otherwise (1: every row,
 *   L: token 0 of each image for ln_post).  d_x, d_gamma, d_beta 16-byte aligned. */
int cc_layernorm_bf16(const float* d_x, int rows, int W, long long row_stride, const int32_t* d_row_idx, const float* d_gamma,
                      const float* d_beta, void* d_out, void* stream);
/* d_x fp32 [B*L][W] = tok[id][:] + pos[t][:] for id = d_ids[b*L + t] clamped to [0, vocab) (an id below 0 reads row 0, one at or
 *   above vocab reads row vocab - 1); d_eot_row[b] = b*L + the first position of the largest raw id of row b (the EOT token).
 *   W a multiple of 4; d_tok, d_pos, d_x 16-byte aligned. */
int cc_text_embed(const int32_t* d_ids, const float* d_tok, const float* d_pos, int B, int L, int W, int vocab, float* d_x,
                  int32_t* d_eot_row, void* stream);
/* d_out[r*out_stride + c] = d_in[r*D + c] / (||d_in row r|| + eps), out_stride >= D, eps >= 0 (the image tower uses 1e-8, the
 *   text tower 0, which gives NaN for a zero row as the reference does). */
int cc_l2norm(const float* d_in, int rows, int D, float eps, float* d_out, long long out_stride, void* stream);

/* ---- CLIP image/text encoder (replaces class OpenCLIP, models/objects.py:21-186) ---- */
typedef struct cc_clip cc_clip;
typedef struct cc_clip_config {
  int image_size, patch;                     /* 224, 14 (ViT-L/14 as in the reference) or 224, 32 (ViT-B/32) */
  int v_width, v_layers, v_heads, v_mlp;     /* vision tower: 1024, 24, 16, 4096 (models/objects.py:50-69) */
  int embed_dim;                             /* 768 (models/objects.py:55) */
  int t_width, t_layers, t_heads, t_mlp;     /* text tower: 768, 12, 12, 3072 (models/objects.py:29-47) */
  int vocab, ctx;                            /* 49408, 77 */
} cc_clip_config;

/* Weights: host fp32 tensors named with the reference's attribute paths: "visual_conv1.weight", "class_embedding",
 * "positional_embedding", "ln_pre.weight", "resblocks_img.0.in_proj_weight", "resblocks_img.0.mlp_c_fc.bias",
 * "ln_post.bias", "proj", "token_embedding.weight", "positional_embedding_text", "resblocks.0.attn_out_proj_weight",
 * "ln_final.weight", "text_projection" ... (what load_state_dict consumes at models/objects.py:91-92). */
int cc_clip_create(const cc_clip_config* cfg, int n_tensors, const char* const* names, const float* const* h_data,
                   const int64_t* numels, cc_clip** out);
int cc_clip_destroy(cc_clip* h);
/* OpenCLIP.precompute_embedding (models/objects.py:94-133): d_x [B,3,S,S] fp32 normalised -> L2-normalised
 * embeddings written to d_out[b*out_row_stride .. +embed_dim) (out_row_stride in floats, 0 = embed_dim; a stride /
 * offset lets the kernel write straight into this rank's slice of an all-gather buffer). */
int cc_clip_encode_image(cc_clip* h, const float* d_x, int B, float* d_out, long long out_row_stride, void* stream);
/* encode_text (models/objects.py:145-186), batched: d_ids [B,ctx] int32 ([49406]+BPE+[49407], zero padded). */
int cc_clip_encode_text(cc_clip* h, const int32_t* d_ids, int B, float* d_out, long long out_row_stride, void* stream);
/* Workspace of the CLIP plans, same contract as cc_yolo_workspace_bytes / cc_yolo_set_workspace (text != 0: text tower). */
int cc_clip_workspace_bytes(cc_clip* h, int text, int B, size_t* bytes);
int cc_clip_set_workspace(cc_clip* h, void* d_workspace, size_t bytes);
/* per-op device timing of one encode (text != 0: text tower). */
int cc_clip_profile(cc_clip* h, int text, const void* d_in, int B, float* d_out, int cap, float* ms, double* flops,
                    const char** names, int* n_ops, double* total_flops, void* stream);
/* Conv op taps of the CLIP plans (text != 0: text tower), with cc_yolo_op_conv's contract: cc_clip_op_conv describes op i of
 * the cached plan of batch B and returns the op count (out == NULL only counts; an i outside [0, count) fails); a GEMM is
 * reported as CC_CONV_OP_GEMM (a linear over R rows as a 1x1 conv of N = 1, H = 1, W = R; the patch embedding with out_ns),
 * any other op as CC_CONV_OP_NONE, both with cc_clip_profile's op name.  cc_clip_run_ops launches ops [first, last) exactly
 * as an encode launches them; d_in, d_out and out_row_stride are those of cc_clip_encode_image / cc_clip_encode_text.
 * Nothing synchronises. */
int cc_clip_op_conv(cc_clip* h, int text, int B, int i, cc_conv_op* out);
/* The operand tap of the CLIP plans (cc_yolo_op_io). */
int cc_clip_op_io(cc_clip* h, int text, int B, int i, cc_op_io* out);
int cc_clip_run_ops(cc_clip* h, int text, const void* d_in, int B, int first, int last, float* d_out, long long out_row_stride,
                    void* stream);
/* ---- AdaFace IR-50 face embedder (replaces class ADAFACE, models/adaface.py:24-96) ---- */
typedef struct cc_face cc_face;
/* Weights: host fp32 tensors of the folded network that clearcam_b200/models/adaface.py `fold_state_dict` makes from the
 * reference's state dict (every BatchNorm and the input normalisation folded in float64):
 *   "stem.w" [64][3][3][3] (input channels in the uint8 image's order), "stem.cls" [9][64], "stem.slope" [64];
 *   "body.<i>.c0.w" [D][3][3][Cin], "body.<i>.c0.cls" [9][D], "body.<i>.c0.slope" [D], "body.<i>.c1.w" [D][3][3][D],
 *   "body.<i>.c1.b" [D], and for a block with a stride or a width change "body.<i>.sc.w" [D][Cin], "body.<i>.sc.b" [D];
 *   "linear.w" [512][7*7*512] (columns in NHWC order), "linear.b" [512].
 * They are rounded to bf16 and uploaded once; the host pointers are not retained. */
int cc_face_create(int n_tensors, const char* const* names, const float* const* h_data, const int64_t* numels, cc_face** out);
int cc_face_destroy(cc_face* h);
/* ADAFACE.__call__ (models/adaface.py:79-96) for B faces: d_faces uint8 [B,112,112,3] (the image as the reference receives
 * it; the channel flip of :81 happens inside) -> L2-normalised embeddings at d_out[b*out_row_stride .. +512) (0 = 512).
 * Face b's row is what the reference's call on face b alone returns (its norm is over its own row). */
int cc_face_embed(cc_face* h, const uint8_t* d_faces, int B, float* d_out, long long out_row_stride, void* stream);
/* Workspace of the face plans, same contract as cc_clip_workspace_bytes / cc_clip_set_workspace. */
int cc_face_workspace_bytes(cc_face* h, int B, size_t* bytes);
int cc_face_set_workspace(cc_face* h, void* d_workspace, size_t bytes);
/* Parity tap: runs the plan of batch B up to `layer` (0: conv0 -> bn0 -> PReLU, 1..24: the output of block layer-1, 25: the
 * linear -> bn2 output before the L2 norm) and writes that map as dense fp32 NHWC [B,H,W,C] to d_dst.  d_dst = NULL only
 * reports C, H, W. */
int cc_face_layer_output(cc_face* h, const uint8_t* d_faces, int B, int layer, float* d_dst, int* C, int* H, int* W, void* stream);
/* Conv op taps of the face plans, as cc_clip_op_conv / cc_clip_run_ops: op names "pack", "stem", "body.<i>.c0", "body.<i>.sc"
 * (the 1x1 shortcut, run as a 3x3 whose only nonzero tap is the centre), "body.<i>.c1", "linear" (a 1x1 conv of N = 1,
 * H = 1, W = B over the 7x7x512 map as one row per face) and "l2norm".  d_faces and d_out are those of cc_face_embed
 * (d_out rows of 512 floats). */
int cc_face_op_conv(cc_face* h, int B, int i, cc_conv_op* out);
/* The operand tap of the face plans (cc_yolo_op_io). */
int cc_face_op_io(cc_face* h, int B, int i, cc_op_io* out);
int cc_face_run_ops(cc_face* h, const uint8_t* d_faces, int B, int first, int last, float* d_out, void* stream);

/* ---- BlazeFace face detector (replaces class BlazeFace, models/blazeface.py:62-232), fp32 ---- */
typedef struct cc_blazeface cc_blazeface;
/* Weights: the reference's own host fp32 tensors under its key names (models/blazeface.safetensors): "conv_tiny.weight"
 * [24][3][5][5], "backbone_tiny.list.<i>.conv0_tiny.weight" [C][1][3][3] / ".conv1_tiny.weight" [Cout][Cin][1][1] (i = 0..30)
 * and their biases, "final.conv{0,1}_tiny.*", "{classifier,regressor}_{8,16}_tiny.*" and "anchors" [896][4].  Uploaded
 * once; the host pointers are not retained. */
int cc_blazeface_create(int n_tensors, const char* const* names, const float* const* h_data, const int64_t* numels,
                        cc_blazeface** out);
int cc_blazeface_destroy(cc_blazeface* h);
/* The workspace a forward of B images needs, and the caller-owned buffer (256-byte aligned) that every later forward uses.
 * cc_blazeface_forward allocates nothing: a missing or smaller workspace fails with CC_ERR_INVALID. */
int cc_blazeface_workspace_bytes(cc_blazeface* h, int B, size_t* bytes);
int cc_blazeface_set_workspace(cc_blazeface* h, void* d_workspace, size_t bytes);
/* BlazeFace.__call__ (:153-175) for B images at once.  frames[b]: a device uint8 [h,w,3] image (format CC_FRAME_BGR_U8; its
 * channels are used in the order given, as the reference does), any size, any number of images.  Writes the forward's raw
 * outputs d_boxes [B,896,16] (16-byte aligned) and d_scores [B,896], and d_dets [B,896,17]: row b is exactly what the
 * reference's call on image b alone returns, every anchor in score order, rows under 0.85 or suppressed zeroed, then *256,
 * the pads off the box columns and everything divided by the scale.  No allocation and no host synchronisation. */
int cc_blazeface_forward(cc_blazeface* h, const cc_frame* frames, int B, float* d_boxes, float* d_scores, float* d_dets,
                         void* stream);
/* The decode, order, suppression and scaling of cc_blazeface_forward alone, on given head outputs d_boxes [B,896,16] and
 * d_scores [B,896]; h_sizes: host int32 [B][2] (height, width) of the images they stand for. */
int cc_blazeface_decode(cc_blazeface* h, const float* d_boxes, const float* d_scores, int B, const int32_t* h_sizes, float* d_dets,
                        void* stream);
/* The detection img_to_face uses (models/objects.py:283-284, detections[detections[:, 0] != 0][0]) for B images at once:
 * d_first [B,17] gets, for each image, the first row of d_dets [B,896,17] whose column 0 != 0 as numpy compares it (-0.0
 * counts as zero, NaN as non-zero), bit for bit, or a zero row when there is none.  Works on any B >= 1. */
int cc_blazeface_first(const float* d_dets, int B, float* d_first, void* stream);

/* ---- img_to_face's image arithmetic (models/objects.py:263-354), byte for byte with cv2 ---- */
/* The pre-resize of B images: frames[b] a device uint8 [h,w,3] image (CC_FRAME_BGR_U8, channels used as given) ->
 * d_out [B,640,640,3]: cv2.resize(INTER_LINEAR) to a long side of 640, then cv2.copyMakeBorder's centred zero border. */
int cc_face_canvas(const cc_frame* frames, int B, uint8_t* d_out, void* stream);
/* One face of cc_face_align: the original device image src [h,w,3], the crop [y1:y2, x1:x2], the size of the rotated image
 * and the two forward matrices as the reference computes them (rot: cv2.getRotationMatrix2D with the canvas growth;
 * transform: the float32 eye transform, given as its float32 values). */
typedef struct {
  const void* src; int h, w;
  int x1, y1, x2, y2;
  int rot_w, rot_h;
  double rot[6], transform[6];
} cc_face_warp;
/* d_out [K,112,112,3]: face k is cv2.cvtColor(cv2.warpAffine(cv2.warpAffine(src[y1:y2, x1:x2], rot, (rot_w, rot_h)),
 * transform, (112, 112)), COLOR_RGB2BGR), pixel for pixel.  A crop outside its image fails with CC_ERR_INVALID before
 * anything is launched. */
int cc_face_align(const cc_face_warp* faces, int K, uint8_t* d_out, void* stream);
/* The same two operations on the images of a padded batch, as the device JPEG decoders write them (cc_jpeg_decode_frames,
 * cc_jpeg_crops_decoded_frames): d_slots uint8 [n_slots, Hmax, Wmax, 3], image k in the h x w corner of slot h_slot[k]
 * (host int32 [K]), rows Wmax * 3 bytes apart, slots Hmax * Wmax * 3 bytes apart.  The slots hold BGR pixels (cv2.imread,
 * cv2.imdecode); each is read as the RGB image cv2.cvtColor(slot, COLOR_BGR2RGB) that img_to_face receives
 * (clearcam.py:1228-1241, 671-678), so result k equals cc_face_canvas / cc_face_align on that contiguous RGB copy, byte for
 * byte.  Canvas: h_sizes host int32 [B][2] (height, width).  Align: faces[k].src is not read; faces[k].h and .w are the image's
 * size within its slot.  Bad arguments (NULL pointers, B or K < 1, a slot index outside the batch, an image larger than a
 * slot, a crop outside its image) fail with CC_ERR_INVALID before anything is launched. */
int cc_face_canvas_slots(const uint8_t* d_slots, int n_slots, int Hmax, int Wmax, const int32_t* h_slot, const int32_t* h_sizes,
                         int B, uint8_t* d_out, void* stream);
int cc_face_align_slots(const uint8_t* d_slots, int n_slots, int Hmax, int Wmax, const int32_t* h_slot, const cc_face_warp* faces,
                        int K, uint8_t* d_out, void* stream);

/* ObjectFinder.search inner loop (models/objects.py:365-376): d_scores[q*N + n] = <d_index[n,:], d_q[q,:]>, fp32. */
int cc_search_scores(const float* d_index, int N, int D, const float* d_q, int Q, float* d_scores, void* stream);

/* ObjectFinder.search with the selection on the device (models/objects.py:365-390): every index row n belongs to group
 * d_group[n] in [0, G) — the rows of one object id share a group, a row without an object id has its own — and rows with
 * d_mask[n] == 0 are skipped (camera / date filter; NULL = no filter).  Per group the best-scoring row is kept, and the k
 * best groups are written in descending score order to d_rows[k] (index row, -1 past the last match) / d_scores[k]; an
 * exact tie goes to the lower row.  d_workspace: 8 * max(G,1) bytes of device scratch.  Only the k winners cross PCIe. */
int cc_search_topk(const float* d_index, int N, int D, const float* d_q, const int32_t* d_group, const uint8_t* d_mask, int G, int k,
                   void* d_workspace, int32_t* d_rows, float* d_scores, void* stream);

/* Object crops of device frames.  frames: HOST array of n_frames cc_frame rows (read during the call only) of any shapes,
 * CC_FRAME_BGR_U8, CC_FRAME_RGB_U8 or CC_FRAME_I420_U8 (h, w even); rects: HOST int32 [K,5] = frame, x1, y1, x2, y2 in
 * pixels, r[0] indexing the table and the rect lying inside its own frame (validated, passed as kernel arguments: no copy,
 * no sync).  A batch of n frames of one shape and format is n rows.  Crop k of any output is what the same call gives for
 * that crop alone.  A NULL frame, another format, an odd I420 side or a rect that is empty or outside its own frame fails
 * with CC_ERR_INVALID before anything is launched.
 *
 * Crop + ObjectFinder.preprocess on the device, for objects cut out of frames already resident for the detector:
 * frame[y1:y2, x1:x2] (clearcam.py:396) -> RGB (models/objects.py:249) -> cv2.resize((size,size), INTER_CUBIC) -> /255 ->
 * (x-0.5)/0.5 -> CHW (models/objects.py:237-242).  An RGB frame is taken as is, a BGR frame has its channels swapped, an
 * I420 frame is converted as cv2.cvtColor(frame, COLOR_YUV2RGB_I420) and then cropped.  d_out: device float32
 * [K,3,size,size] — the tensor cc_clip_encode_image takes. */
int cc_clip_preprocess_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int size, float* d_out,
                              void* stream);

/* Object thumbnails on the device: baseline JPEG of frame crops, byte for byte the file cv2.imwrite(path, crop) writes at
 * IMWRITE_JPEG_QUALITY `quality` (`VideoCapture.save_object`, clearcam.py:373-399): 4:2:0, integer DCT, Annex K tables,
 * JFIF 1.01 header; oracle/jpeg.py states the arithmetic.  frames and rects as above; the crop is encoded as the BGR image
 * cv2 would see (RGB frames are swapped, I420 frames converted as cv2.cvtColor(COLOR_YUV2BGR_I420) and then cropped).
 * quality: 0..100 (0 acts as 1); a crop side over 65535 fails.
 * cc_jpeg_bound: worst-case bytes of one encoded w x h crop (every code at its longest, every byte stuffed, headers, EOI).
 * cc_jpeg_encode_crops_frames: crop k is written to d_out + out_offsets[k] (HOST int64 [K]; each region [offset, offset +
 * cc_jpeg_bound) inside the out_bytes of d_out, none overlapping: the prefix sum of the bounds needs no sync) and its
 * length to d_lengths[k] (device int64 [K]).  d_workspace: *ws_needed bytes of device scratch, 256-byte aligned.
 * d_out == NULL only writes *ws_needed.  Nothing is allocated and nothing synchronises; a bad argument fails with
 * CC_ERR_INVALID before anything is launched.
 * cc_jpeg_coeffs_frames (parity tap): the quantised coefficients of every 8x8 block of every crop, int16 [n_blocks][64]
 * in zigzag order: crop by crop, MCU by MCU (Y0 Y1 Y2 Y3 Cb Cr), dummy blocks included.  d_coef == NULL only writes
 * *n_blocks; otherwise d_coef is 4-byte aligned. */
int cc_jpeg_bound(int w, int h, int64_t* bytes);
int cc_jpeg_encode_crops_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int quality, uint8_t* d_out,
                                int64_t out_bytes, const int64_t* out_offsets, int64_t* d_lengths, void* d_workspace,
                                size_t ws_bytes, size_t* ws_needed, void* stream);
int cc_jpeg_coeffs_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int quality, int16_t* d_coef,
                          int64_t* n_blocks, void* stream);

/* JPEG files -> BGR uint8 on the device, pixel for pixel what cv2.imdecode(buf, IMREAD_COLOR) returns (libjpeg-turbo 3.1:
 * islow IDCT, fancy upsampling, table-driven YCbCr -> BGR); oracle/jpeg_decode.py states the arithmetic.  Replaces the host
 * decodes of stored thumbnails (clearcam.py:272-279) and of search-by-image uploads (models/objects.py:244-251).
 * Decoded on the device: baseline and extended sequential Huffman (SOF0 / SOF1), 8-bit, one scan holding every component,
 * 1 component (grey, replicated to B, G and R) or 3 with luma sampling 1x1, 2x1, 1x2 or 2x2 and chroma 1x1 (4:4:4, 4:2:2,
 * 4:4:0, 4:2:0), any DQT / DHT tables, restart intervals, APPn / COM skipped.  Every other file gets a status and is left to
 * the caller (cv2 on the host): CC_JPEG_UNSUPPORTED for progressive, arithmetic, lossless, 12-bit, 4:1:1, CMYK / Adobe RGB,
 * several scans, an Exif orientation other than 1, a missing Huffman table, or coefficients outside the range where every
 * libjpeg-turbo IDCT agrees; CC_JPEG_CORRUPT for a malformed header (a marker libjpeg does not know included), an invalid
 * Huffman code, wrong RSTn markers or a scan that ends before its last MCU.
 * cc_jpeg_table_bytes: bytes of one image's entry in the parse table.
 * cc_jpeg_parse (host only): K files at h_data + offsets[k], lengths[k] bytes (all HOST int64 [K], inside data_bytes) ->
 * h_table (K entries, 16-byte aligned), h_sizes [K,2] = width, height (0 where the header did not say), h_status [K] and
 * h_blocks [K] (8x8 blocks of each decoded image, 0 for the others).  A file never makes it fail; the entries also place
 * each image's intermediates in the workspace, so a table belongs to its own set of K files.
 * cc_jpeg_decode_frames: d_data holds the same bytes as h_data and d_table the same bytes as h_table.  outs (HOST [K],
 * read during the call only): image k, when its status is OK, is written as BGR uint8 [h, w, 3] at outs[k].data (device),
 * rows outs[k].pitch bytes apart, e.g. a device frame buffer a detector call reads, or slot k of a padded batch [K, Hmax,
 * Wmax, 3] (pitch 3 Wmax); nothing else is written.  d_status [K] (device int32) receives the final status: the parse
 * status, or CC_JPEG_CORRUPT / CC_JPEG_UNSUPPORTED found on the device, in which case that image's destination is left as
 * it was and the other images are unaffected.  d_coef: NULL, or device int16 [sum of h_blocks][64], 16-byte aligned, that
 * receives the dequantisation input (zigzag order, block by block in scan order, image after image): the coefficient tap.
 * d_workspace: *ws_needed bytes of device scratch, 256-byte aligned; outs == NULL only writes *ws_needed (which depends
 * on whether d_coef is NULL).  Nothing is allocated and nothing synchronises; a bad argument fails with CC_ERR_INVALID
 * before anything is launched, among them a parsed image whose destination is NULL, is not the image's h x w, has a pitch
 * below 3 w or overlaps another such destination; the destinations of images the parse did not accept are not read.
 * cc_jpeg_crops_decoded_frames: for the crops of cc_jpeg_encode_crops_frames (same frames, rects and quality), the pixels
 * cv2.imdecode(cv2.imencode(".jpg", crop, quality)) gives: the encoder's transform, then the decoder's reconstruction, with
 * no entropy coding between them (the coefficients are the file's content).  Crop k goes to rows 0..h-1, columns 0..w-1 of
 * slot k of d_out [K, Hmax, Wmax, 3], and d_status [K] (device int32) gets CC_JPEG_OK, or CC_JPEG_UNSUPPORTED where the
 * coefficients leave the range in which every libjpeg-turbo IDCT agrees (that slot is then not written; decode the file
 * with cv2).  d_out == NULL only writes *ws_needed; workspace as above. */
#define CC_JPEG_OK 0
#define CC_JPEG_UNSUPPORTED 1
#define CC_JPEG_CORRUPT 2
size_t cc_jpeg_table_bytes(void);
int cc_jpeg_parse(const uint8_t* h_data, int64_t data_bytes, const int64_t* offsets, const int64_t* lengths, int K, void* h_table,
                  int32_t* h_sizes, int32_t* h_status, int64_t* h_blocks);
typedef struct { void* data; int64_t pitch; int32_t h; int32_t w; } cc_jpeg_dest;
int cc_jpeg_decode_frames(const uint8_t* d_data, const void* h_table, const void* d_table, int K, const cc_jpeg_dest* outs,
                          int32_t* d_status, int16_t* d_coef, void* d_workspace, size_t ws_bytes, size_t* ws_needed,
                          void* stream);
int cc_jpeg_crops_decoded_frames(const cc_frame* frames, int n_frames, const int32_t* rects, int K, int quality, uint8_t* d_out,
                                 int Hmax, int Wmax, int32_t* d_status, void* d_workspace, size_t ws_bytes, size_t* ws_needed,
                                 void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Tracker that consumes the detector rows (host code, no GPU): ocsort_tracker/ocsort.py:163-308 `OCSort`, with
 * association.py and kalmanfilter.py.  One handle per camera (clearcam.py:239 `ocsort.OCSort(max_age=100)`).
 * cc_ocsort_create arguments = OCSort.__init__'s (ocsort.py:164-165; det_thresh is per update call as in :177).
 * Track ids start at 1 per handle (the reference shares one class-level counter between cameras and resets it whenever
 * any tracker is constructed, ocsort.py:177 — ids there are only unique per camera between such resets). */
typedef struct cc_ocsort* cc_ocsort_t;
int cc_ocsort_create(int max_age, int min_hits, double iou_threshold, int delta_t, double inertia, int use_byte, cc_ocsort_t* out);
int cc_ocsort_destroy(cc_ocsort_t h);
/* OCSort.update(output_results, det_thresh) (ocsort.py:177-308).  rows: host float32 [n,6] = x1,y1,x2,y2,score,class
 * (the detector's (300,6) block as is; zero rows are ignored by the score gates).  out: host float64 [cap,9] =
 * tl_x, tl_y, w, h, score, class_id, track_id, tracklet_len, speed — the STrack fields clearcam.py:583-621 reads —
 * in the reference's order (newest track first).  *n_out = rows written; error if it would exceed cap. */
int cc_ocsort_update(cc_ocsort_t h, const float* rows, int n, float det_thresh, double* out, int cap, int* n_out);
/* The same for B cameras in one call: hs[B] (NULL entries skipped), rows [B,n,6], det_thresh [B], out [B,cap,9], n_out [B]. */
int cc_ocsort_update_batch(cc_ocsort_t* hs, int B, const float* rows, int n, const float* det_thresh, double* out, int cap,
                           int* n_out);
int cc_ocsort_num_tracks(cc_ocsort_t h);

/* ---------------------------------------------------------------------------------------------------------------
 * The same tracker on the GPU, bit for bit (track ids included): a handle owns `slots` camera trackers on the current
 * device, and one cc_ocsort_gpu_update launch steps up to CC_MAX_FRAMES of them, one CTA per camera, on rows that stay
 * on the device.  Slot calls are stream-ordered on the stream given (use one stream per handle); nothing synchronises
 * except cc_ocsort_gpu_num_tracks (which waits for `stream`, then reads the count) and cc_ocsort_gpu_destroy.
 *
 * cc_ocsort_gpu_configure: (re)starts slot `slot` as cc_ocsort_create(max_age, ...) would, with room for `capacity`
 * tracks (storage is reused when the capacity is unchanged); delta_t may not exceed the handle's max_delta_t.
 * cc_ocsort_gpu_grow: keeps the slot's tracks and raises its room to `capacity` (a smaller value does nothing).
 *
 * cc_ocsort_gpu_update: job b steps slot jobs[b].slot on the device rows d_rows [n,6] (as cc_ocsort_update's rows) at
 * det_thresh; each slot at most once per call.  Per job b: d_out [B,cap,9] float64 rows as cc_ocsort_update writes them,
 * d_count[b], d_status[b] = CC_TRACK_*:
 *   OK         the frame was applied, d_count[b] rows written;
 *   NEEDS_ROOM the slot lacks room for the tracks this frame may add: nothing changed, d_count[b] = the capacity needed
 *              (cc_ocsort_gpu_grow, then step the camera again);
 *   BAD_CLASS  a detection inside the score gates has a class id that is not an integer in 0..CC_OCSORT_CLASSES-1:
 *              nothing changed, d_count[b] = 0;
 *   OVERFLOW   more than cap rows: the frame was applied (as cc_ocsort_update does), d_count[b] = the row count, only
 *              cap rows written.
 * Nothing is written in d_out past a job's rows.  Bad arguments (unconfigured or repeated slot, n outside
 * 0..CC_OCSORT_MAX_ROWS, NULL rows, B outside 1..CC_MAX_FRAMES) fail with CC_ERR_INVALID before the launch. */
typedef struct cc_ocsort_gpu cc_ocsort_gpu;
typedef struct { const float* d_rows; int n; int slot; float det_thresh; int reserved; } cc_track_job;
#define CC_OCSORT_CLASSES 80
#define CC_OCSORT_MAX_ROWS 1024
#define CC_TRACK_OK 0
#define CC_TRACK_NEEDS_ROOM 1
#define CC_TRACK_BAD_CLASS 2
#define CC_TRACK_OVERFLOW 3
#define CC_TRACK_BAD_BOX 4              /* cc_ocsort_gpu_update_runs only */
int cc_ocsort_gpu_create(int slots, int max_delta_t, cc_ocsort_gpu** out);
int cc_ocsort_gpu_destroy(cc_ocsort_gpu* h);
int cc_ocsort_gpu_configure(cc_ocsort_gpu* h, int slot, int max_age, int min_hits, double iou_threshold, int delta_t,
                            double inertia, int use_byte, int capacity, void* stream);
int cc_ocsort_gpu_free(cc_ocsort_gpu* h, int slot, void* stream);
int cc_ocsort_gpu_grow(cc_ocsort_gpu* h, int slot, int capacity, void* stream);
int cc_ocsort_gpu_capacity(cc_ocsort_gpu* h, int slot, int* capacity);
int cc_ocsort_gpu_num_tracks(cc_ocsort_gpu* h, int slot, int* n, void* stream);
int cc_ocsort_gpu_update(cc_ocsort_gpu* h, const cc_track_job* jobs, int B, double* d_out, int cap, int* d_count,
                         int* d_status, void* stream);

/* Runs: several consecutive frames of one camera per job, e.g. a run of a recorded video, in one launch per stage.  Each
 * job's CTA applies frames 0..frames-1 in order, exactly as that many cc_ocsort_gpu_update calls would, and stops at the
 * first frame whose status is not CC_TRACK_OK.
 * cc_track_run: device rows [frames,n,6] (frame f at d_rows + f*n*6; n <= CC_OCSORT_MAX_ROWS), frames 1..frames_max
 * (frames_max <= CC_MAX_FRAMES), slot, det_thresh.
 * cc_ocsort_gpu_update_runs: per job b and frame f, row b*frames_max + f of d_out [B,frames_max,cap,9], d_count
 * [B,frames_max] (as cc_ocsort_gpu_update's d_out and d_count), d_live [B,frames_max] the live tracks after the frame and
 * d_ids [B,frames_max,id_cap] their ids (slot order; what the events of that frame read), id_cap >= every job's slot
 * capacity.  d_done[b] = frames applied with status OK, d_status[b] = the status of frame d_done[b] (CC_TRACK_OK when
 * every frame was); its count, live and ids are written too.  NEEDS_ROOM and BAD_CLASS leave the slot as frame
 * d_done[b] - 1 left it (grow, then run the rest from there); OVERFLOW applied that frame.  BAD_BOX: frame d_done[b] - 1
 * was applied (status OK, counted in d_done) but one of its target boxes is not finite or beyond 2^60, which the
 * events reject; the run stops after it so that its events run before the tracker goes on (run the rest from d_done[b]
 * once they have).  Nothing is written past a
 * job's last frame.  Bad arguments (as cc_ocsort_gpu_update, frames outside 1..frames_max, id_cap below a slot's
 * capacity) fail with CC_ERR_INVALID before the launch.  A one-frame run gives what cc_ocsort_gpu_update gives. */
typedef struct { const float* d_rows; int n; int frames; int slot; float det_thresh; } cc_track_run;
int cc_ocsort_gpu_update_runs(cc_ocsort_gpu* h, const cc_track_run* runs, int B, int frames_max, double* d_out, int cap, int* d_count,
                              int32_t* d_ids, int id_cap, int* d_live, int* d_done, int* d_status, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Object events on the tracker handle: what run_inference does with the targets (clearcam.py:586-621), per camera on the
 * device — the class filter, tracklet_len < 1, the pred_occs clock and save_object's rectangle with its 100-px gate, the
 * motion gate speed < 2.5, the zone test (point_not_in_polygon in float64, exactly as written there) with `outside` and
 * the non-zone-alert rule, the (k,7) preds rows and the new / new-in-zone bookkeeping.  clearcam_b200/events.py is the
 * host form and documents the choices (one clock reading per camera-step; non-finite boxes are errors).
 *
 * cc_ocsort_gpu_events_configure: the events of tracker slot `slot` (configured with cc_ocsort_gpu_configure): zone_xy
 * [n_vertices,2] float64 fractions of the frame (n_vertices 0 = no zone, at most CC_EVENT_MAX_VERTICES, finite),
 * outside / non_zone_alert as 0/1, class_mask 3 words of bits for class ids 0..79 (NULL = every class), room for
 * `capacity` track ids.  Clears the slot's event state (pred_occs, object_set, object_set_zone), as does
 * cc_ocsort_gpu_configure; cc_ocsort_gpu_free frees it.  cc_ocsort_gpu_events_grow keeps the state and raises the room.
 *
 * cc_ocsort_gpu_events: job b (a cc_ocsort_gpu_update job table; only .slot is read) runs the events of jobs[b].slot on
 * row b of that call's outputs d_trk_out [B,trk_cap,9], d_trk_count, d_trk_status, queued after it on the same stream,
 * for a frame of frame_wh[2b] x frame_wh[2b+1] pixels at clock now[b] (seconds).  Outputs per job b: d_preds [B,cap,7]
 * float64, d_flags [B,cap] uint8 (bit 0 new, bit 1 new_in_zone), d_saves [B,cap,6] int64 (track_id, class_id, x1, y1,
 * x2, y2), d_counts[b] preds rows and d_counts[B+b] save rows, d_status[b] = CC_EVENT_*:
 *   OK         the step was applied;
 *   NEEDS_ROOM the slot's event storage lacks room: nothing changed, d_counts[b] = the capacity needed
 *              (cc_ocsort_gpu_events_grow, then run the events of that camera again on the same tracker rows);
 *   BAD_BOX    a target past the class filter and tracklet_len has a box that is not finite or beyond 2^60: nothing changed;
 *   NOT_RUN    the tracker's status for the job was not CC_TRACK_OK: nothing changed;
 *   BAD_ORDER  the tracker's ids are not in the strictly ascending slot order the state relies on: nothing changed.
 * Nothing is written past a job's rows.  Bad arguments (a slot without tracker or events, a repeated slot, B outside
 * 1..CC_MAX_FRAMES, cap < trk_cap, a frame side < 1, a non-finite clock, NULL pointers) fail with CC_ERR_INVALID before
 * the launch. */
#define CC_EVENT_MAX_VERTICES 256
#define CC_EVENT_OK 0
#define CC_EVENT_NEEDS_ROOM 1
#define CC_EVENT_BAD_BOX 2
#define CC_EVENT_NOT_RUN 3
#define CC_EVENT_BAD_ORDER 4
int cc_ocsort_gpu_events_configure(cc_ocsort_gpu* h, int slot, const double* zone_xy, int n_vertices, int outside,
                                   int non_zone_alert, const uint32_t* class_mask, int capacity, void* stream);
int cc_ocsort_gpu_events_grow(cc_ocsort_gpu* h, int slot, int capacity, void* stream);
int cc_ocsort_gpu_events(cc_ocsort_gpu* h, const cc_track_job* jobs, int B, const int* frame_wh, const double* now,
                         const double* d_trk_out, int trk_cap, const int* d_trk_count, const int* d_trk_status, double* d_preds,
                         uint8_t* d_flags, int64_t* d_saves, int cap, int* d_counts, int* d_status, void* stream);

int cc_ocsort_gpu_events_set_non_zone_alert(cc_ocsort_gpu* h, int slot, int non_zone_alert, void* stream);

/* cc_ocsort_gpu_events_runs: the events of a cc_ocsort_gpu_update_runs call (same runs and frames_max; only .slot and
 * .frames are read), queued after it: job b applies frames 0..d_trk_done[b]-1 in order, frame f on row b*frames_max+f of
 * d_trk_out / d_trk_count / d_trk_ids / d_trk_live, for a picture of frame_wh[2i] x frame_wh[2i+1] at clock now[i], i the
 * frame's index in the job-major list of every job's frames.  Outputs per frame at row b*frames_max+f: d_preds
 * [B,frames_max,cap,7], d_flags [B,frames_max,cap], d_saves [B,frames_max,cap,6], d_counts [2,B,frames_max] (preds rows,
 * save rows) as cc_ocsort_gpu_events writes them; d_done[b] frames applied, d_status[b] the CC_EVENT_* of frame d_done[b]
 * (NOT_RUN when the tracker stopped there, OK when every frame was applied).  NEEDS_ROOM leaves the slot's entries as
 * frame d_done[b]-1 left them: grow, then run the events again from that frame on the same tracker rows.  Bad arguments
 * fail with CC_ERR_INVALID before anything is launched. */
int cc_ocsort_gpu_events_runs(cc_ocsort_gpu* h, const cc_track_run* runs, int B, int frames_max, const int* frame_wh, const double* now,
                              const double* d_trk_out, int trk_cap, const int* d_trk_count, const int32_t* d_trk_ids, int id_cap,
                              const int* d_trk_live, const int* d_trk_done, double* d_preds, uint8_t* d_flags, int64_t* d_saves, int cap,
                              int* d_counts, int* d_done, int* d_status, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Alerts on the tracker handle: the adds of run_inference (clearcam.py:612-620) behind the object events, the object
 * counter, the firing loop of process_frame (:465-499) and the description alerts of clip_latest_img (:1289-1307).
 * clearcam_b200/alerts.py is the host form and documents the choices (one clock and one local time per step; a missing
 * weekday entry is inactive; alerts with max 0 and description alerts keep no counts; the warm-up counts steps; the
 * similarity's fixed summation order; a camera the caller leaves out of a step — the reference's gate when none of its
 * alerts is active — keeps its counts and its warm-up count until its next step).
 *
 * cc_alert: one alert.  classes: bits for the class ids 0..79 it counts; max: 0 = none (it never fires on counts);
 * window: seconds > 0, already resolved (None -> 60 when is_notif, else 1); flags CC_ALERT_*; with CC_ALERT_SCHED the
 * alert is active on the weekdays of `days` (bit 0 Monday) when start - window < time of day < end; threshold: the
 * similarity a description alert must exceed (+inf: never); last_det: the clock of its last firing.
 *
 * cc_ocsort_gpu_alerts_configure: the n alerts of tracker slot `slot`, in order (at most CC_ALERT_MAX_ALERTS);
 * desc_emb [n,dim] float32 host rows (only rows of CC_ALERT_DESC alerts are read; NULL when there are none); keep[i] >= 0
 * makes alert i keep the counts and last_det of the slot's current alert keep[i] (same max, classes and CC_ALERT_DESC),
 * rows of alerts without CC_ALERT_DESC are neither read nor checked;
 * -1 (or keep NULL) starts it empty at its own last_det.  The object counter, the warm-up count and alerts_on stay.
 * cc_ocsort_gpu_configure clears the counter and the warm-up (init_cam); cc_ocsort_gpu_free frees the alerts.
 * cc_ocsort_gpu_alerts_set_on: the camera's alerts_on (1 after configure).  cc_ocsort_gpu_alerts_counts: the object
 * counter, int64 [80] per class id (waits for `stream`); cc_ocsort_gpu_alerts_reset_counts zeroes it.
 * cc_ocsort_gpu_events_set_non_zone_alert changes a slot's non_zone_alert without touching its event state.
 *
 * cc_ocsort_gpu_alerts: job b (a cc_ocsort_gpu_update job table; only .slot is read) runs the alerts of jobs[b].slot on
 * row b of a cc_ocsort_gpu_events launch's outputs (d_preds [B,cap,7], d_flags [B,cap], its d_counts and d_status),
 * queued after it on the same stream, at clock now[b] and local time local[2b] (seconds of day), local[2b+1] (weekday,
 * 0 = Monday).  Outputs: d_fired [B,CC_ALERT_MAX_ALERTS] the indices of the alerts that fired, in order; d_res[b] their
 * number and d_res[B+b] = CC_ALERT_*: OK, or NOT_RUN when the events' status was not CC_EVENT_OK (nothing changed; run
 * the alerts again after the events).
 *
 * cc_ocsort_gpu_describe: job b matches rows[b] object embeddings of slot slots[b] (consecutive rows of d_emb [N,dim]
 * float32, jobs in order) against its description alerts at clock now[b], local time local[2b..2b+1].  Outputs per row:
 * d_hit the index of the alert that fired (-1 none), d_sim [N,CC_ALERT_MAX_ALERTS] float32 similarities (NaN for alerts
 * without a description).
 *
 * Bad arguments (a slot without alerts, a repeated slot, B outside 1..CC_MAX_FRAMES, a clock or time of day that is not
 * finite, a weekday outside 0..6, a description width that differs from the slot's, NULL pointers; for configure a
 * bad alert or keep entry) fail with CC_ERR_INVALID before anything is launched or changed. */
#define CC_ALERT_MAX_ALERTS 64
#define CC_ALERT_MAX_COUNT 1024
#define CC_ALERT_ON 1
#define CC_ALERT_ZONE 2
#define CC_ALERT_DESC 4
#define CC_ALERT_SCHED 8
#define CC_ALERT_OK 0
#define CC_ALERT_NOT_RUN 1
typedef struct {
  uint32_t classes[3];
  int max, flags, days, reserved[2];
  double window, start, end, threshold, last_det;
} cc_alert;
int cc_ocsort_gpu_alerts_configure(cc_ocsort_gpu* h, int slot, const cc_alert* alerts, int n, const float* desc_emb, int dim,
                                   const int* keep, void* stream);
int cc_ocsort_gpu_alerts_set_on(cc_ocsort_gpu* h, int slot, int on, void* stream);
int cc_ocsort_gpu_alerts_counts(cc_ocsort_gpu* h, int slot, int64_t* counts, void* stream);
int cc_ocsort_gpu_alerts_reset_counts(cc_ocsort_gpu* h, int slot, void* stream);
int cc_ocsort_gpu_alerts(cc_ocsort_gpu* h, const cc_track_job* jobs, int B, const double* now, const double* local,
                         const double* d_preds, const uint8_t* d_flags, int cap, const int* d_ev_counts, const int* d_ev_status,
                         int* d_fired, int* d_res, void* stream);
int cc_ocsort_gpu_describe(cc_ocsort_gpu* h, const int* slots, const int* rows, int B, const double* now, const double* local,
                           const float* d_emb, int dim, int* d_hit, float* d_sim, void* stream);

/* Runs.  cc_ocsort_gpu_alerts_runs: the alerts of a cc_ocsort_gpu_events_runs call (same runs and frames_max), queued
 * after it: job b applies frames 0..d_ev_done[b]-1 in order, frame f on row b*frames_max+f of d_preds, d_flags and
 * d_ev_counts [2,B,frames_max], at clock now[i] and local time local[2i..2i+1], i the frame's index in the job-major list.
 * Outputs: d_fired [B,frames_max,CC_ALERT_MAX_ALERTS] and d_nfired [B,frames_max] per frame, d_done[b] frames applied,
 * d_status[b] OK, or NOT_RUN when the events stopped before the last frame.
 * cc_ocsort_gpu_describe_runs: job b matches the saves of frames[b] frames of slot slots[b]: rows[i] rows of d_emb for
 * frame i of the job-major list (consecutive, frame after frame, job after job), frame i at clock now[i] and local time
 * local[2i..2i+1].  The frames are matched in order, each row as cc_ocsort_gpu_describe would at its frame's clock; outputs
 * per row as there.  Bad arguments fail with CC_ERR_INVALID before anything is launched. */
int cc_ocsort_gpu_alerts_runs(cc_ocsort_gpu* h, const cc_track_run* runs, int B, int frames_max, const double* now, const double* local,
                              const double* d_preds, const uint8_t* d_flags, int cap, const int* d_ev_counts, const int* d_ev_done,
                              int* d_fired, int* d_nfired, int* d_done, int* d_status, void* stream);
int cc_ocsort_gpu_describe_runs(cc_ocsort_gpu* h, const int* slots, const int* frames, int B, const int* rows, const double* now,
                                const double* local, const float* d_emb, int dim, int* d_hit, float* d_sim, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CLEARCAM_B200_H */
