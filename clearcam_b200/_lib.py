"""ctypes binding of libclearcam_b200.so (C-ABI declared in include/clearcam_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, a CCError is raised
(the reference's callers catch exceptions and supervise restarts themselves, clearcam.py:543-546).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# CC_LIB: developer override used for same-box A/B runs of two builds (tools/ab.py); production loads the in-tree library
LIB_PATH = os.environ.get("CC_LIB") or os.path.join(_HERE, "libclearcam_b200.so")


class CCError(RuntimeError):
    pass


# frames per cc_yolo_forward_frames / cc_letterbox_frames call (CC_MAX_FRAMES in include/clearcam_b200.h); the crop entry
# points' tables (cc_*_frames of the JPEG encoder and the CLIP preprocess) have no such limit
CC_MAX_FRAMES = 128


class cc_frame(ctypes.Structure):
    """One row of a frame table: device pointer (None = padding row), CC_FRAME_* code, height, width in pixels."""
    _fields_ = [("data", ctypes.c_void_p), ("fmt", ctypes.c_int), ("h", ctypes.c_int), ("w", ctypes.c_int)]


class cc_jpeg_dest(ctypes.Structure):
    """One destination of cc_jpeg_decode_frames: device pointer, row pitch in bytes, height, width in pixels."""
    _fields_ = [("data", ctypes.c_void_p), ("pitch", ctypes.c_int64), ("h", ctypes.c_int32), ("w", ctypes.c_int32)]


class cc_track_job(ctypes.Structure):
    """One row of a tracker job table (cc_ocsort_gpu_update): device rows [n,6], their count, slot, threshold."""
    _fields_ = [("rows", ctypes.c_void_p), ("n", ctypes.c_int), ("slot", ctypes.c_int), ("det_thresh", ctypes.c_float),
                ("reserved", ctypes.c_int)]


class cc_track_run(ctypes.Structure):
    """One row of a tracker run table (cc_ocsort_gpu_update_runs): device rows [frames,n,6], n, frames, slot, threshold."""
    _fields_ = [("rows", ctypes.c_void_p), ("n", ctypes.c_int), ("frames", ctypes.c_int), ("slot", ctypes.c_int),
                ("det_thresh", ctypes.c_float)]


class cc_slice(ctypes.Structure):
    """An NHWC slice as cc_yolo_op_conv reports it: device pointer, channels per pixel, first channel, channels, N, H, W, fp32."""
    _fields_ = [("p", ctypes.c_void_p)] + [(n, ctypes.c_int) for n in ("cs", "co", "C", "N", "H", "W", "f32")]


class cc_conv_op(ctypes.Structure):
    """One op of a detector plan as cc_yolo_op_conv describes it (include/clearcam_b200.h); `in_` is the header's `in`."""
    _fields_ = ([("kind", ctypes.c_int), ("name", ctypes.c_char * 128), ("in_", cc_slice), ("out", cc_slice), ("res", cc_slice),
                 ("w", ctypes.c_void_p), ("bias", ctypes.c_void_p)]
                + [(n, ctypes.c_int) for n in ("k", "stride", "groups", "act")]
                + [("pre", ctypes.c_void_p), ("pre_h", ctypes.c_int), ("pre_w", ctypes.c_int), ("w2", ctypes.c_void_p),
                   ("bias2", ctypes.c_void_p), ("act2", ctypes.c_int), ("k0", ctypes.c_int), ("part", cc_slice), ("out2", cc_slice),
                   ("store1", ctypes.c_int)]
                + [(n, ctypes.c_int) for n in ("BN", "BK", "lTW", "lTH", "lTN", "s2", "stages", "b_res", "grid", "num_tiles")])


# cc_conv_op kinds (CC_CONV_OP_* in include/clearcam_b200.h)
CC_CONV_OP_NONE, CC_CONV_OP_GEMM, CC_CONV_OP_CHAIN, CC_CONV_OP_DIRECT = 0, 1, 2, 3

# cc_ocsort_gpu_update statuses (CC_TRACK_* in include/clearcam_b200.h)
CC_TRACK_OK, CC_TRACK_NEEDS_ROOM, CC_TRACK_BAD_CLASS, CC_TRACK_OVERFLOW, CC_TRACK_BAD_BOX = 0, 1, 2, 3, 4
# cc_ocsort_gpu_events statuses (CC_EVENT_* in include/clearcam_b200.h)
CC_EVENT_OK, CC_EVENT_NEEDS_ROOM, CC_EVENT_BAD_BOX, CC_EVENT_NOT_RUN, CC_EVENT_BAD_ORDER = 0, 1, 2, 3, 4
CC_EVENT_MAX_VERTICES = 256
# cc_ocsort_gpu_alerts: limits, cc_alert flags and statuses (CC_ALERT_* in include/clearcam_b200.h)
CC_ALERT_MAX_ALERTS, CC_ALERT_MAX_COUNT = 64, 1024
CC_ALERT_ON, CC_ALERT_ZONE, CC_ALERT_DESC, CC_ALERT_SCHED = 1, 2, 4, 8
CC_ALERT_OK, CC_ALERT_NOT_RUN = 0, 1


class cc_alert(ctypes.Structure):
    """One alert of cc_ocsort_gpu_alerts_configure: class mask, max, CC_ALERT_* flags, weekday bits (Monday = bit 0),
    resolved window, schedule start / end (seconds of day), description threshold, last_det."""
    _fields_ = [("classes", ctypes.c_uint32 * 3), ("max", ctypes.c_int), ("flags", ctypes.c_int), ("days", ctypes.c_int),
                ("reserved", ctypes.c_int * 2)] + [(n, ctypes.c_double) for n in ("window", "start", "end", "threshold", "last_det")]

_lib = None

_vp = ctypes.c_void_p
_i = ctypes.c_int
_f = ctypes.c_float
_SIGS = {
    "cc_version": (_i, []),
    "cc_last_error": (ctypes.c_char_p, []),
    "cc_device_check": (_i, []),
    "cc_conv2d": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _vp]),
    "cc_conv2d_chain": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _i, _i, _i,
                             _vp, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "cc_yolo_create": (_i, [ctypes.c_char_p, _i, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_vp),
                            ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(_vp)]),
    "cc_yolo_create_ex": (_i, [ctypes.c_char_p, _i, _i, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_vp),
                               ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(_vp)]),
    "cc_yolo_destroy": (_i, [_vp]),
    "cc_yolo_forward": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "cc_yolo_workspace_bytes": (_i, [_vp, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_size_t)]),
    "cc_yolo_set_workspace": (_i, [_vp, _vp, ctypes.c_size_t]),
    "cc_clip_workspace_bytes": (_i, [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]),
    "cc_clip_set_workspace": (_i, [_vp, _vp, ctypes.c_size_t]),
    "cc_yolo_plan_info": (_i, [_vp, _i, _i, _i, _i, _i, ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i),
                               ctypes.POINTER(_i), ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]),
    "cc_yolo_profile": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _i, ctypes.POINTER(_f), ctypes.POINTER(ctypes.c_double),
                             ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_i), _vp]),
    "cc_yolo_trace": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _i, ctypes.POINTER(ctypes.c_ulonglong), ctypes.POINTER(ctypes.c_char_p),
                           ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_double), ctypes.POINTER(_i), _vp]),
    "cc_yolo_op_conv": (_i, [_vp, _i, _i, _i, _i, _i, _i, ctypes.POINTER(cc_conv_op)]),
    "cc_yolo_run_ops": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "cc_yolo_layer_output": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, ctypes.POINTER(_i), ctypes.POINTER(_i),
                                  ctypes.POINTER(_i), _vp]),
    "cc_detect_postprocess": (_i, [_vp, _i, _i, _i, _f, _i, _f, _f, _f, _f, _f, _vp, _vp]),
    "cc_detect_pred_from_raw": (_i, [_vp, _i, _i, _i, _f, _vp, _vp]),
    "cc_detect_decode": (_i, [ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_i), ctypes.POINTER(_i), _i, _f,
                              _vp, _vp, _vp]),
    "cc_clip_create": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_vp), ctypes.POINTER(ctypes.c_int64),
                            ctypes.POINTER(_vp)]),
    "cc_clip_destroy": (_i, [_vp]),
    "cc_clip_encode_image": (_i, [_vp, _vp, _i, _vp, ctypes.c_longlong, _vp]),
    "cc_clip_encode_text": (_i, [_vp, _vp, _i, _vp, ctypes.c_longlong, _vp]),
    "cc_clip_profile": (_i, [_vp, _i, _vp, _i, _vp, _i, ctypes.POINTER(_f), ctypes.POINTER(ctypes.c_double),
                             ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_i), ctypes.POINTER(ctypes.c_double), _vp]),
    "cc_conv2d_prelu": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _i, _vp]),
    "cc_face_create": (_i, [_i, ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_vp), ctypes.POINTER(ctypes.c_int64),
                            ctypes.POINTER(_vp)]),
    "cc_face_destroy": (_i, [_vp]),
    "cc_face_embed": (_i, [_vp, _vp, _i, _vp, ctypes.c_longlong, _vp]),
    "cc_face_workspace_bytes": (_i, [_vp, _i, ctypes.POINTER(ctypes.c_size_t)]),
    "cc_face_set_workspace": (_i, [_vp, _vp, ctypes.c_size_t]),
    "cc_face_layer_output": (_i, [_vp, _vp, _i, _i, _vp, ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i), _vp]),
    "cc_search_scores": (_i, [_vp, _i, _i, _vp, _i, _vp, _vp]),
    "cc_search_topk": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "cc_clip_preprocess": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp]),
    "cc_clip_preprocess_frames": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp]),
    "cc_ocsort_create": (_i, [_i, _i, ctypes.c_double, _i, ctypes.c_double, _i, ctypes.POINTER(_vp)]),
    "cc_ocsort_destroy": (_i, [_vp]),
    "cc_ocsort_update": (_i, [_vp, _vp, _i, _f, _vp, _i, ctypes.POINTER(_i)]),
    "cc_ocsort_update_batch": (_i, [_vp, _i, _vp, _i, _vp, _vp, _i, _vp]),
    "cc_ocsort_num_tracks": (_i, [_vp]),
    "cc_ocsort_gpu_create": (_i, [_i, _i, ctypes.POINTER(_vp)]),
    "cc_ocsort_gpu_destroy": (_i, [_vp]),
    "cc_ocsort_gpu_configure": (_i, [_vp, _i, _i, _i, ctypes.c_double, _i, ctypes.c_double, _i, _i, _vp]),
    "cc_ocsort_gpu_free": (_i, [_vp, _i, _vp]),
    "cc_ocsort_gpu_grow": (_i, [_vp, _i, _i, _vp]),
    "cc_ocsort_gpu_capacity": (_i, [_vp, _i, ctypes.POINTER(_i)]),
    "cc_ocsort_gpu_num_tracks": (_i, [_vp, _i, ctypes.POINTER(_i), _vp]),
    "cc_ocsort_gpu_update": (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "cc_ocsort_gpu_events_configure": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _i, _vp]),
    "cc_ocsort_gpu_events_grow": (_i, [_vp, _i, _i, _vp]),
    "cc_ocsort_gpu_events": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "cc_ocsort_gpu_events_set_non_zone_alert": (_i, [_vp, _i, _i, _vp]),
    "cc_ocsort_gpu_alerts_configure": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _vp]),
    "cc_ocsort_gpu_alerts_set_on": (_i, [_vp, _i, _i, _vp]),
    "cc_ocsort_gpu_alerts_counts": (_i, [_vp, _i, _vp, _vp]),
    "cc_ocsort_gpu_alerts_reset_counts": (_i, [_vp, _i, _vp]),
    "cc_ocsort_gpu_alerts": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "cc_ocsort_gpu_describe": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "cc_ocsort_gpu_update_runs": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "cc_ocsort_gpu_events_runs": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp,
                                       _vp]),
    "cc_ocsort_gpu_alerts_runs": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cc_ocsort_gpu_describe_runs": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "cc_letterbox": (_i, [_vp, _i, _i, _i, _i, _i, _vp, ctypes.POINTER(_i), ctypes.POINTER(_i), _vp]),
    "cc_yolo_net_shape": (_i, [_i, _i, _i, _i, ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    "cc_yolo_forward_frames": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    "cc_yolo_workspace_bytes_frames": (_i, [_vp, _vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]),
    "cc_letterbox_frames": (_i, [_vp, _i, _i, _vp, ctypes.POINTER(_i), ctypes.POINTER(_i), _vp]),
    "cc_attention": (_i, [_vp, _i, _i, _i, _i, _i, _vp, ctypes.c_size_t, _vp, ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_pool": (_i, [_i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "cc_spp3": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp]),
    "cc_cbfuse": (_i, [_i, _i, ctypes.POINTER(_vp), ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i),
                       _vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "cc_split_planes": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "cc_finish_f32": (_i, [_vp, _vp, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp]),
    "cc_stem": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _i, _vp, _i, _i, _i, _i, _vp, ctypes.c_size_t,
                     ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_conv2d_pre": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp, _i, _i, _i, _i, _vp, _i, _vp]),
    "cc_conv2d_fp32_accurate": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp,
                                     ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_patchify": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "cc_clip_embed_ln": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "cc_layernorm_bf16": (_i, [_vp, _i, _i, ctypes.c_longlong, _vp, _vp, _vp, _vp, _vp]),
    "cc_text_embed": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "cc_l2norm": (_i, [_vp, _i, _i, _f, _vp, ctypes.c_longlong, _vp]),
    "cc_jpeg_bound": (_i, [_i, _i, ctypes.POINTER(ctypes.c_int64)]),
    "cc_jpeg_encode_crops": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, ctypes.c_int64, _vp, _vp, _vp, ctypes.c_size_t,
                                  ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_jpeg_encode_crops_frames": (_i, [_vp, _i, _vp, _i, _i, _vp, ctypes.c_int64, _vp, _vp, _vp, ctypes.c_size_t,
                                         ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_jpeg_coeffs": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, ctypes.POINTER(ctypes.c_int64), _vp]),
    "cc_jpeg_table_bytes": (ctypes.c_size_t, []),
    "cc_jpeg_parse": (_i, [_vp, ctypes.c_int64, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "cc_jpeg_decode": (_i, [_vp, _vp, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_jpeg_decode_frames": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_jpeg_crops_decoded": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, ctypes.c_size_t,
                                   ctypes.POINTER(ctypes.c_size_t), _vp]),
    "cc_jpeg_crops_decoded_frames": (_i, [_vp, _i, _vp, _i, _i, _vp, _i, _i, _vp, _vp, ctypes.c_size_t,
                                          ctypes.POINTER(ctypes.c_size_t), _vp]),
}


def lib():
    """Load (once) and return the ctypes handle; raises CCError when the library was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CCError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(h, name, None)
            if fn is None and os.environ.get("CC_LIB"):
                continue              # an older build under A/B comparison may lack newer entry points
            if fn is None:
                raise CCError(f"{LIB_PATH} does not export {name}: rebuild it (python -c 'import __graft_entry__ as g; g.build()')")
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().cc_last_error()
        raise CCError(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")


def declared_symbols():
    return sorted(_SIGS)


def ptr(t):
    """Device/host pointer of a torch tensor (or None)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr(stream=None):
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return ctypes.c_void_p(s.cuda_stream)
