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

#define CC_ABI_VERSION 1

int cc_version(void);
const char* cc_last_error(void);
/* number of SMs of the current device if it is sm_90 (H100), else <0 */
int cc_device_check(void);

/* activation codes */
#define CC_ACT_NONE 0
#define CC_ACT_SILU 1      /* x*sigmoid(x): detection/yolov9.py:38 */
#define CC_ACT_GELU_TANH 2 /* tinygrad Tensor.gelu(): models/objects.py:125,179 */

/* ---- kernel-level ops (used by the graphs below and exposed for the parity tests) ---- */

/* Conv2d(bias) [+act] [+residual], k in {1,3}, stride in {1,2}, pad = k/2, NHWC bf16 in, bf16|fp32 out.
 * Replaces nn.Conv2d + .silu() of detection/yolov9.py:33-38 (and the bare nn.Conv2d of :173,:186,:224).
 * d_w: bf16 [Cout][k][k][Cin/groups]; d_bias: fp32 [Cout] or NULL; d_res: same dtype/shape class as out or NULL.
 * impl: 0 = auto (wgmma implicit GEMM when the shape allows, else direct), 1 = force wgmma, 2 = force direct.
 * bn: wgmma N-tile upper bound (0 = heuristic). */
int cc_conv2d(const void* d_in, int N, int Hin, int Win, int in_cs, int in_co, int Cin,
              const void* d_w, const float* d_bias, int Cout, int k, int stride, int groups,
              void* d_out, int out_cs, int out_co, int out_f32, int act,
              const void* d_res, int res_cs, int res_co, int impl, int bn, void* stream);

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

/* YOLOv9.__call__ (detection/yolov9.py:375-388) for a batch of same-shape frames.
 * d_frames: [B,Hf,Wf,3] HWC **BGR**, uint8 (is_f32=0, clearcam.py:582) or float32 (is_f32=1, test/run_mot.py:33).
 * d_out: [B,300,6] fp32 rows [x1,y1,x2,y2,conf,class] in frame pixels, descending conf, suppressed rows all-zero.
 * d_raw: optional [B,84,A] fp32 tap of the head output (xc,yc,w,h,80 class probs) for parity tests, or NULL.
 * A plan (buffers, TMA descriptors) is built and cached on the first call for each (dtype,B,Hf,Wf,res) — the
 * analogue of jit_infer's per-shape TinyJit cache (utils/helpers.py:214-221); later calls only launch kernels. */
int cc_yolo_forward(cc_yolo* h, const void* d_frames, int is_f32, int B, int Hf, int Wf, int res, float* d_out,
                    float* d_raw, void* stream);
/* plan facts: letterboxed net input size, anchors, kernel launches per forward, algorithmic conv FLOPs,
 * bytes of activation workspace */
int cc_yolo_plan_info(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, int* net_h, int* net_w, int* anchors,
                      int* launches, double* conv_flops, double* act_bytes);

/* Workspace.  Every cached plan of a handle carves its activations out of ONE device workspace (size of the largest plan;
 * at most 16 plans are kept, least recently used goes first), so a process that sees many batch sizes / frame shapes does
 * not accumulate buffers.  By default the library owns it and grows it on demand (a growth frees and reallocates: it
 * synchronises the device once, and the plans of the old workspace are rebuilt on their next use).  A caller that wants no
 * allocation after start-up sizes it with cc_yolo_workspace_bytes for its largest shape and hands it over with
 * cc_yolo_set_workspace (256-byte aligned device memory, owned by the caller; d_workspace = NULL returns to the
 * library-owned one); a plan that does not fit a caller-owned workspace fails with CC_ERR_INVALID.  The plans of one
 * handle share the memory: run them in stream order (one stream per handle). */
int cc_yolo_workspace_bytes(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, size_t* bytes);
int cc_yolo_set_workspace(cc_yolo* h, void* d_workspace, size_t bytes);

/* measurement: per-op device time of one forward (CUDA events between launches on `stream`; synchronises).
 * Up to `cap` entries of ms / algorithmic conv FLOPs / algorithmic HBM bytes / kernel kind / op name (pointers valid
 * while h lives). */
int cc_yolo_profile(cc_yolo* h, const void* d_frames, int is_f32, int B, int Hf, int Wf, int res, float* d_out, int cap,
                    float* ms, double* flops, double* bytes, const char** kinds, const char** names, int* n_ops, void* stream);

/* measurement: in-situ device timeline of one forward, no events between the launches (so programmatic dependent launch
 * overlaps exactly as in production).  For op i, host_ns[12i..12i+11] = globaltimer ns of (first CTA entered, grid
 * dependency released, last CTA exited; then of CTA 0: first operands landed, all MMAs issued, first accumulator complete,
 * last epilogue group done, exit; then four stamps inside the first staging pass of its first tile) for the tensor-core conv launches, zeros for the other kernels.  Synchronises. */
int cc_yolo_trace(cc_yolo* h, const void* d_frames, int is_f32, int B, int Hf, int Wf, int res, float* d_out, int cap,
                  unsigned long long* host_ns, const char** kinds, const char** names, double* flops, int* n_ops, void* stream);

/* parity tap: after a forward, copy the output of graph layer `layer` (index into the reference's self.model list,
 * detection/yolov9.py:303-371) to dense fp32 [B,H,W,C].  d_dst == NULL only queries C/H/W (C = 0: no tensor). */
int cc_yolo_layer_output(cc_yolo* h, int is_f32, int B, int Hf, int Wf, int res, int layer, float* d_dst, int* C,
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
/* YOLOv9.preprocess (detection/yolov9.py:390-404) + resize (utils/helpers.py:127-131): [B,Hin,Win,3] -> letterboxed
 * [B,out_h,out_w,3], same dtype.  d_out == NULL only queries the output size. */
int cc_letterbox(const void* d_in, int is_f32, int B, int Hin, int Win, int res, void* d_out, int* out_h, int* out_w,
                 void* stream);

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
/* ObjectFinder.search inner loop (models/objects.py:365-376): d_scores[q*N + n] = <d_index[n,:], d_q[q,:]>, fp32. */
int cc_search_scores(const float* d_index, int N, int D, const float* d_q, int Q, float* d_scores, void* stream);

/* ObjectFinder.search with the selection on the device (models/objects.py:365-390): every index row n belongs to group
 * d_group[n] in [0, G) — the rows of one object id share a group, a row without an object id has its own — and rows with
 * d_mask[n] == 0 are skipped (camera / date filter; NULL = no filter).  Per group the best-scoring row is kept, and the k
 * best groups are written in descending score order to d_rows[k] (index row, -1 past the last match) / d_scores[k]; an
 * exact tie goes to the lower row.  d_workspace: 8 * max(G,1) bytes of device scratch.  Only the k winners cross PCIe. */
int cc_search_topk(const float* d_index, int N, int D, const float* d_q, const int32_t* d_group, const uint8_t* d_mask, int G, int k,
                   void* d_workspace, int32_t* d_rows, float* d_scores, void* stream);

/* Crop + ObjectFinder.preprocess on the device, for objects cut out of frames already resident for the detector:
 * frame[y1:y2, x1:x2] (clearcam.py:396) -> BGR->RGB when bgr != 0 (models/objects.py:249) -> cv2.resize((size,size),
 * INTER_CUBIC) -> /255 -> (x-0.5)/0.5 -> CHW (models/objects.py:237-242).  d_frames: device uint8 [n_frames,H,W,3];
 * rects: HOST int32 [K,5] = frame, x1, y1, x2, y2 (validated, passed as kernel arguments: no copy, no sync);
 * d_out: device float32 [K,3,size,size] — the tensor cc_clip_encode_image takes. */
int cc_clip_preprocess(const uint8_t* d_frames, int n_frames, int H, int W, const int32_t* rects, int K, int size, int bgr,
                       float* d_out, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* CLEARCAM_B200_H */
