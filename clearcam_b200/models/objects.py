"""Drop-in for the reference's `models/objects.py` CLIP part on H100 (same names and call signatures).

    from clearcam_b200.models.objects import ObjectFinder
    finder = ObjectFinder(); finder.init_clip(weights=..., arch="ViT-L/14")
    emb  = finder.model.precompute_embedding(x).numpy()            # x (B,3,224,224) float32  (clearcam.py:1285)
    temb = finder.model._encode_text("ferrari f40", realize=True)  # (768,)                   (clearcam.py:667)
    hits = finder.search("ferrari f40", top_k=10)                  # [(path, score)]          (models/objects.py:356)

Mirrors class OpenCLIP (/root/reference/models/objects.py:21-143), encode_text (:145-186) and ObjectFinder's CLIP
methods (:189-206, :237-251, :356-421), and the face embedder's (`init_face`, `turn_off_face`, `adaface`,
`preprocess_face` for 112x112 faces, face search; :207-217, :253-261) and the BlazeFace face detector (`blazeface`,
models/blazeface.py) with face alignment (`img_to_face`, :263-354, and the batched `faces_from_images`), and the
faces of object saves (`encode_embed_faces_frames`, clearcam.py:1228-1241) and of uploads (`embed_face_images`,
clearcam.py:671-678).  All arithmetic runs in libclearcam_b200.so; there is no CPU fallback.

Additions: `arch=` (the reference hard-codes ViT-L/14; "ViT-B/32" runs the same kernels), explicit `weights=`
(the reference downloads from HuggingFace, :91), `encode_text_batch`, a contiguous device index for search, and
`gather=` to all-gather embeddings across ranks (NCCL) straight from the kernel's output slice.
"""
from __future__ import annotations

import ctypes
import os
import pickle
from typing import Dict, List, NamedTuple, Optional

import numpy as np
import torch

from .._lib import CCError, Handle, check, create, lib, ptr, stream_ptr
from ..detection.yolov9 import DeviceResult, _as_tensor, load_weights_arg
from .. import ops
from ..pixfmt import BGR24, CC_FRAME_BGR_U8, CC_FRAME_I420_U8, CC_FRAME_RGB_U8, check_pix_fmt, yuv420p_size
from ..utils.clip_tokenizer import SimpleTokenizer
from ..utils.helpers import batch_bucket

# (image_size, patch, v_width, v_layers, v_heads, v_mlp, embed_dim, t_width, t_layers, t_heads, t_mlp, vocab, ctx)
ARCHS = {
    "ViT-L/14": (224, 14, 1024, 24, 16, 4096, 768, 768, 12, 12, 3072, 49408, 77),   # models/objects.py:29-69
    "ViT-B/32": (224, 32, 768, 12, 12, 3072, 512, 512, 12, 8, 2048, 49408, 77),
    "ViT-tiny": (64, 16, 128, 2, 2, 512, 64, 128, 2, 2, 512, 49408, 77),
}


class _ClipConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("image_size", "patch", "v_width", "v_layers", "v_heads", "v_mlp", "embed_dim",
                                            "t_width", "t_layers", "t_heads", "t_mlp", "vocab", "ctx")]


def event_img_info(name: str) -> dict:
    """clearcam.event_img_info (clearcam.py:1193): "{ts}_{objid}_{cls}" -> fields used by search dedupe."""
    parts = name.split("_")
    return {"ts": parts[0], "object_id": parts[1] if len(parts) > 1 else None, "class": parts[2] if len(parts) > 2 else None}


class OpenCLIP(Handle):
    _destroy = "cc_clip_destroy"

    def __init__(self, base_path="data/cameras", weights=None, arch: str = "ViT-L/14"):
        self.base_path = base_path
        self.arch = arch
        self.cfg = ARCHS[arch]
        self.embed_dim = self.cfg[6]
        self.image_size = self.cfg[0]
        self.ctx = self.cfg[12]
        self.tokenizer = SimpleTokenizer()
        self.load_weights(load_weights_arg(weights, "https://huggingface.co/roryclear/CLIP-ViT-L-14-laion2B-s32B-b82K/resolve/main/"
                                                    "CLIP-ViT-L-14-laion2B-s32B-b82K.safetensors"))

    def load_weights(self, state_dict) -> None:
        tensors = lambda: {k: v for k, v in state_dict.items() if k != "attn_mask"}     # noqa: E731
        self._adopt(create("cc_clip_create", tensors, ctypes.byref(_ClipConfig(*self.cfg))))

    # ---- image tower
    @staticmethod
    def _as_device(x, dtype) -> torch.Tensor:
        return _as_tensor(x).to("cuda", dtype, non_blocking=True).contiguous()

    def embed_into(self, x, out: torch.Tensor, row0: int = 0, stream=None) -> None:
        """precompute_embedding writing rows [row0, row0+B) of `out` ([N, embed_dim] fp32 CUDA) in place."""
        t = self._as_device(x, torch.float32)
        B = t.shape[0]
        assert t.shape[1:] == (3, self.image_size, self.image_size), f"expected (B,3,{self.image_size},{self.image_size})"
        assert out.is_cuda and out.dtype == torch.float32 and out.stride(-1) == 1
        dst = out[row0:row0 + B]
        check(lib().cc_clip_encode_image(self._h, ptr(t), B, ctypes.c_void_p(dst.data_ptr()), out.stride(0), stream_ptr(stream)),
              "cc_clip_encode_image")

    def precompute_embedding(self, x, gather: bool = False):
        """(B,3,224,224) float32 normalised -> DeviceResult (B,embed_dim), L2-normalised (models/objects.py:94-133).
        gather=True (torch.distributed initialised, NCCL): returns the all-gathered (world*B, embed_dim) index;
        the final kernel writes this rank's rows directly into the gather buffer (in-place all-gather)."""
        t = self._as_device(x, torch.float32)
        B = t.shape[0]
        if gather:
            import torch.distributed as dist
            world, rank = dist.get_world_size(), dist.get_rank()
            full = torch.empty(world * B, self.embed_dim, device="cuda", dtype=torch.float32)
            self.embed_into(t, full, rank * B)
            dist.all_gather_into_tensor(full, full[rank * B:(rank + 1) * B])
            return DeviceResult(full)
        out = torch.empty(B, self.embed_dim, device="cuda", dtype=torch.float32)
        self.embed_into(t, out, 0)
        return DeviceResult(out)

    # ---- text tower
    def tokenize(self, query: str) -> List[int]:
        tokens = [49406] + self.tokenizer.encode(query) + [49407]          # models/objects.py:136-138
        if len(tokens) > self.ctx:
            raise CCError(f"query has {len(tokens) - 2} BPE tokens; the reference does not truncate (max {self.ctx - 2})")
        return tokens + [0] * (self.ctx - len(tokens))                      # :139

    def encode_text_batch(self, queries: List[str]):
        ids = torch.tensor([self.tokenize(q) for q in queries], dtype=torch.int32).cuda()
        out = torch.empty(len(queries), self.embed_dim, device="cuda", dtype=torch.float32)
        check(lib().cc_clip_encode_text(self._h, ptr(ids), len(queries), ptr(out), 0, stream_ptr()), "cc_clip_encode_text")
        return DeviceResult(out)

    def encode_token_ids(self, ids):
        t = self._as_device(ids, torch.int32)
        out = torch.empty(t.shape[0], self.embed_dim, device="cuda", dtype=torch.float32)
        check(lib().cc_clip_encode_text(self._h, ptr(t), t.shape[0], ptr(out), 0, stream_ptr()), "cc_clip_encode_text")
        return DeviceResult(out)

    def _encode_text(self, query, realize=False):
        """models/objects.py:135-143: one query -> (embed_dim,) ; numpy when realize=True."""
        r = DeviceResult(self.encode_text_batch([query]).tensor[0])
        return r.numpy() if realize else r

    def profile(self, x=None, ids=None):
        cap = 1024
        ms = (ctypes.c_float * cap)(); fl = (ctypes.c_double * cap)(); names = (ctypes.c_char_p * cap)()
        n = ctypes.c_int(); tot = ctypes.c_double()
        if x is not None:
            t = self._as_device(x, torch.float32); text = 0
        else:
            t = self._as_device(ids, torch.int32); text = 1
        out = torch.empty(t.shape[0], self.embed_dim, device="cuda", dtype=torch.float32)
        check(lib().cc_clip_profile(self._h, text, ptr(t), t.shape[0], ptr(out), cap, ms, fl, names, ctypes.byref(n),
                                    ctypes.byref(tot), stream_ptr()), "cc_clip_profile")
        return [{"name": names[i].decode(), "ms": ms[i], "flops": fl[i]} for i in range(n.value)], tot.value


def search_scores(index, queries) -> torch.Tensor:
    """index (N,D), queries (Q,D) fp32 -> (Q,N) dot products on device (models/objects.py:373 per pair)."""
    idx = OpenCLIP._as_device(index, torch.float32)
    q = OpenCLIP._as_device(queries, torch.float32)
    if q.dim() == 1:
        q = q.unsqueeze(0)
    N, D = idx.shape
    out = torch.empty(q.shape[0], N, device="cuda", dtype=torch.float32)
    check(lib().cc_search_scores(ptr(idx), N, D, ptr(q), q.shape[0], ptr(out), stream_ptr()), "cc_search_scores")
    return out


def _device_crops(frames, rects, bgr: bool, pix_fmt: str):
    """The frame / rect conventions of `ObjectFinder.preprocess_device` and `encode_crops`: frames uint8 [n,H,W,3] / [H,W,3]
    (bgr24, or RGB when not `bgr`) or [n,H*3/2,W] / [H*3/2,W] (yuv420p), host or device; rects K rows of (frame, x1, y1,
    x2, y2) or (x1, y1, x2, y2).  -> (contiguous device frames [n,...], their frame table, int32 rects [K,5]); the table
    points into the frames, so it is used while they live."""
    t = _as_tensor(frames)
    if check_pix_fmt(pix_fmt) == BGR24:
        if t.dim() == 3:
            t = t.unsqueeze(0)
        if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[-1] != 3:
            raise ValueError("frames must be uint8 [n,H,W,3]")
        fmt = CC_FRAME_BGR_U8 if bgr else CC_FRAME_RGB_U8
    else:
        if t.dim() == 2:
            t = t.unsqueeze(0)
        if t.dtype != torch.uint8 or t.dim() != 3:
            raise ValueError(f"yuv420p frames must be uint8 [n,H*3/2,W], got {t.dtype} {tuple(t.shape)}")
        yuv420p_size(t.shape)
        fmt = CC_FRAME_I420_U8
    t = t.to("cuda", non_blocking=True).contiguous()
    r = np.asarray(rects, np.int32).reshape(-1, np.shape(rects)[-1] if len(rects) else 5)
    if r.shape[1] == 4:
        r = np.concatenate([np.zeros((len(r), 1), np.int32), r], 1)
    return t, ops.batch_table(t, fmt), np.ascontiguousarray(r, np.int32)


class FaceSaves(NamedTuple):
    """The faces of a batch of object saves (`process_latest_face`, clearcam.py:1228-1241)."""
    rows: List[int]                         # the saves whose img_to_face found a face, in save order
    files: List[bytes]                      # each face's JPEG, as cv2.imwrite writes the 112x112 BGR face
    embeddings: Optional[DeviceResult]      # (f,512): row j is adaface(face j)


class ObjectFinder:
    """CLIP half of the reference's ObjectFinder (models/objects.py:188-206, 237-251, 356-421)."""

    def __init__(self, base_path="data/cameras"):
        self.base_path = base_path
        self.image_embeddings: Dict[str, np.ndarray] = {}
        self.face_embeddings: Dict[str, np.ndarray] = {}
        self.image_paths = {}
        self.face_paths = {}
        self.clip = False
        self.face = False
        self.jit_cache = {}
        # is_face -> (paths, device tensor [N,D], per-row search metadata, identities of the cached values): the device
        # copies of image_embeddings and face_embeddings
        self._index = {}
        self.model: Optional[OpenCLIP] = None
        self.blazeface = None
        self.adaface = None           # ADAFACE once init_face ran: adaface(img) -> (1,512), as the reference calls it

    def init_clip(self, weights=None, arch: str = "ViT-L/14"):
        if self.clip:
            return
        self.clip = True
        self.model = OpenCLIP(weights=weights, arch=arch)
        s = self.model.image_size
        for _ in range(2):                                                  # prewarm = build the cached plans (:204-205)
            self.model._encode_text("text here", realize=True)
            self.model.precompute_embedding(torch.rand(1, 3, s, s)).numpy()

    def turn_off_clip(self):
        self.clip = False
        self.model = None

    def init_face(self, weights=None, detector=None):
        """models/objects.py:211-215: the AdaFace embedder, from the reference's state dict / safetensors path, or the
        reference's file when None; and the BlazeFace detector (`blazeface(img)` -> (896,17)) from `detector` (a state dict
        or safetensors path), or from the reference's models/blazeface.safetensors when that file exists.  Without either,
        `blazeface` stays None."""
        if self.face:
            return
        from .adaface import ADAFACE
        from .blazeface import WEIGHTS_PATH, BlazeFace
        self.adaface = ADAFACE(weights)
        if detector is not None or os.path.exists(WEIGHTS_PATH):
            self.blazeface = BlazeFace(detector)
        self.face = True

    def turn_off_face(self):
        self.face = False
        self.blazeface = None
        self.adaface = None

    def embed_faces(self, faces):
        """uint8 [B,112,112,3] faces (host or device) -> device (B,512): row b is `adaface(faces[b])`, in one batched call."""
        if self.adaface is None:
            raise CCError("the face embedder is off: call init_face() first")
        return self.adaface.embed(faces)

    def preprocess_face(self, img):
        """models/objects.py:253-261: an uploaded file (bytes) or a stored path under data/cameras -> the RGB image when it is
        already a 112x112 face.  Other sizes raise: the reference routes them through `img_to_face`, which
        `embed_face_images` does for a batch of uploads."""
        import cv2
        if type(img) == bytes:
            img = cv2.imdecode(np.frombuffer(img, np.uint8), cv2.IMREAD_COLOR)
        else:
            img = cv2.imread(f"data/cameras{img}")
        img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        if img.shape != (112, 112, 3):
            raise CCError(f"preprocess_face: a {img.shape[1]}x{img.shape[0]} image needs face detection and alignment "
                          "(img_to_face), which uploads do not go through yet; only 112x112 faces are accepted")
        return img

    def faces_from_images(self, images):
        """`img_to_face` for many images at once: images are uint8 [h,w,3] (host or device, any sizes, as the reference's
        call receives them) -> (device uint8 [K,112,112,3], rows): rows[i] is the index of image i's face in the batch, or
        None where `img_to_face(images[i])` returns None.  One canvas launch, one BlazeFace forward, one read of the
        detections for the host geometry, one alignment launch; the faces go to `embed_faces` without leaving the device."""
        from .blazeface import _images, align_faces, face_canvas, face_geometry, first_detections
        self._need_detector()
        ims = _images(images)
        canvas = face_canvas(ims)
        first = first_detections(self.blazeface.detect(canvas)).cpu().numpy()      # the host geometry needs one row per image
        jobs, rows = [], []
        for i, t in enumerate(ims):
            g = face_geometry(first[i:i + 1], t.shape[0], t.shape[1])
            rows.append(None if g is None else len(jobs))
            if g is not None:
                jobs.append((t, g))
        return align_faces(jobs), rows

    def _need_detector(self):
        if self.blazeface is None:
            raise CCError("face detection is off: init_face(detector=...) builds BlazeFace from its weights, or from the "
                          "reference's models/blazeface.safetensors when that file exists")

    def _queue_first(self, slots, index, sizes):
        """Queue img_to_face's detection for the (height, width) corners of slots[index] of a padded BGR batch, each read
        as its RGB image: canvas, BlazeFace on a batch padded to batch_bucket, first kept row -> device [len(index),17]."""
        from .blazeface import face_canvas_slots, first_detections
        n = len(index)
        canvas = face_canvas_slots(slots, index, sizes, rows=batch_bucket(n))
        return first_detections(self.blazeface.detect(canvas)[:n])

    @staticmethod
    def _align_slots(slots, index, sizes, first):
        """The rest of img_to_face for those images, given their first rows on the host: the reference's geometry on the
        host, then one alignment launch -> (device uint8 [f,112,112,3] BGR faces, per image its face's row or None)."""
        from .blazeface import align_faces_slots, face_geometry
        jobs, rows = [], []
        for i, (slot, hw) in enumerate(zip(index, sizes)):
            g = face_geometry(first[i:i + 1], *hw)
            rows.append(None if g is None else len(jobs))
            if g is not None:
                jobs.append((slot, hw, g))
        return align_faces_slots(slots, jobs), rows

    def img_to_face(self, orig):
        """models/objects.py:263-354: an HWC uint8 image -> the aligned 112x112 face (numpy uint8, BGR order as the
        reference returns it), or None.  Raises CCError when BlazeFace is not built."""
        faces, rows = self.faces_from_images([orig])
        return None if rows[0] is None else faces[rows[0]].cpu().numpy()

    def preprocess(self, img):
        """models/objects.py:237-242 (host, cv2): RGB HWC uint8 -> (3,S,S) float32 in [-1,1]."""
        import cv2
        s = self.model.image_size if self.model is not None else 224
        img = cv2.resize(img, (s, s), interpolation=cv2.INTER_CUBIC)
        img = img.astype(np.float32) / 255.0
        img = (img - 0.5) / 0.5
        return np.transpose(img, (2, 0, 1))

    def preprocess_clip(self, img):
        import cv2
        if type(img) == bytes:
            img = cv2.imdecode(np.frombuffer(img, np.uint8), cv2.IMREAD_COLOR)
        else:
            img = cv2.imread(f"data/cameras{img}")
        img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        return [self.preprocess(img)]

    # ---- objects cut out of frames that are already on the device (SURVEY.md §8f N3)
    @staticmethod
    def crop_rect(box_xyxy, W: int, H: int, min_side: int = 100):
        """`save_object`'s rectangle (clearcam.py:381-395): the box grown to twice its size about its centre in integer
        arithmetic, clamped to the frame; None when a side is under 100 px ("too small")."""
        x1, y1, x2, y2 = (int(v) for v in box_xyxy)
        cx, cy = (x1 + x2) // 2, (y1 + y2) // 2
        hw, hh = (x2 - x1) // 2 * 2, (y2 - y1) // 2 * 2
        nx1, nx2 = max(0, min(cx - hw, W)), max(0, min(cx + hw, W))
        ny1, ny2 = max(0, min(cy - hh, H)), max(0, min(cy + hh, H))
        if (ny2 - ny1) < min_side or (nx2 - nx1) < min_side:
            return None
        return nx1, ny1, nx2, ny2

    def preprocess_device(self, frames, rects, bgr: bool = True, size: Optional[int] = None, rows: Optional[int] = None,
                          pix_fmt: str = BGR24):
        """frames: uint8 [n,H,W,3] or [H,W,3] (host or device; BGR as the cameras deliver them), rects: K rows of
        (frame, x1, y1, x2, y2) or (x1, y1, x2, y2) -> DeviceResult (K,3,S,S) float32, bit-identical to
        `preprocess(cv2.cvtColor(frame[y1:y2, x1:x2], BGR2RGB))` with OpenCV's own bicubic — without leaving the GPU.
        pix_fmt="yuv420p": frames are uint8 [n,H*3/2,W] or [H*3/2,W] (H, W even; rects in pixels), and the result is
        bit-identical to the same crop of `cv2.cvtColor(frame, COLOR_YUV2RGB_I420)` (`bgr` does not apply)."""
        t, table, r = _device_crops(frames, rects, bgr, pix_fmt)
        s = size or (self.model.image_size if self.model is not None else 224)
        # rows > K: the result is allocated with `rows` images, the first K filled and the rest zero (batch padding)
        out = torch.empty(len(r), 3, s, s, device="cuda", dtype=torch.float32) if not rows or rows <= len(r) else \
            torch.zeros(rows, 3, s, s, device="cuda", dtype=torch.float32)
        check(lib().cc_clip_preprocess_frames(table, len(table), r.ctypes.data, len(r), s, ptr(out), stream_ptr(None)),
              "cc_clip_preprocess_frames")
        return DeviceResult(out)

    def embed_crops(self, frames, rects, bgr: bool = True, pix_fmt: str = BGR24):
        """Detector frame -> embeddings of its objects in one device pass: crop + preprocess + `precompute_embedding`
        (the reference goes through cv2.imwrite / cv2.imread and the host, clearcam.py:398, 274-276).  `pix_fmt` as in
        `preprocess_device` (CameraBatch.device_frame returns a camera's frame in its own format)."""
        k = len(rects)
        if k == 0:
            return DeviceResult(torch.empty(0, self.model.embed_dim, device="cuda", dtype=torch.float32))
        # the number of objects differs from frame to frame: pad the batch to a bucket size so the encoder keeps a small,
        # bounded set of plans; the padded rows are dropped
        x = self.preprocess_device(frames, rects, bgr, rows=batch_bucket(k), pix_fmt=pix_fmt)
        return DeviceResult(self.model.precompute_embedding(x).tensor[:k])

    def encode_crops(self, frames, rects, quality: int = 95, bgr: bool = True, pix_fmt: str = BGR24) -> List[bytes]:
        """Detector frame -> the JPEG file of each object crop, encoded on the device: element k is byte for byte what
        `cv2.imwrite(path, frame[y1:y2, x1:x2])` writes at IMWRITE_JPEG_QUALITY `quality` (`save_object`,
        clearcam.py:373-399).  frames / rects / bgr / pix_fmt as in `preprocess_device`; a yuv420p frame gives the file of
        the same crop of `cv2.cvtColor(frame, COLOR_YUV2BGR_I420)`.  Only the encoded bytes cross PCIe."""
        if not 0 <= int(quality) <= 100:
            raise ValueError(f"quality must be in 0..100 (cv2's range), got {quality}")
        t, table, r = _device_crops(frames, rects, bgr, pix_fmt)
        return ops.jpeg_collect(*ops.jpeg_encode_crops_frames(table, r, quality)) if len(r) else []

    def embed_images(self, items):
        """The batched device form of `run_clip`'s `preprocess_clip` + `precompute_embedding` (clearcam.py:671-678,
        models/objects.py:244-251): items are `bytes` (an uploaded file) or the reference's paths relative to data/cameras
        (stored thumbnails) -> DeviceResult (K, embed_dim).  The files are decoded on the device (ops.jpeg_decode), then
        cropped, resized and normalised by cc_clip_preprocess_frames and embedded in one batch.  A file the device reports as
        unsupported or corrupt is decoded by cv2 on the host and joins the same batch; where cv2 returns None this raises as
        the reference's cvtColor does."""
        k = len(items)
        if k == 0:
            return DeviceResult(torch.empty(0, self.model.embed_dim, device="cuda", dtype=torch.float32))
        out, sizes = self._decode_items(items)
        rects = [(i, 0, 0, w, h) for i, (w, h) in enumerate(sizes)]
        x = self.preprocess_device(out, rects, bgr=True, rows=batch_bucket(k))
        return DeviceResult(self.model.precompute_embedding(x).tensor[:k])

    @staticmethod
    def _decode_items(items):
        """Uploaded files (`bytes`) or paths relative to data/cameras -> (device uint8 [k,Hmax,Wmax,3], image i in the
        top-left corner of slot i as cv2.imdecode gives it, [(w, h)] per image).  The device decodes what it can
        (ops.JpegBatch); a file it reports as unsupported or corrupt is decoded by cv2 on the host and copied into its slot;
        where cv2 returns None this raises as the reference's cvtColor does."""
        import cv2
        files = []
        for it in items:
            if type(it) == bytes:
                files.append(it)
            else:
                try:
                    with open(f"data/cameras{it}", "rb") as f:
                        files.append(f.read())
                except OSError:
                    files.append(b"")                   # cv2.imread gives None: raised below
        batch = ops.JpegBatch(files)
        host = {}

        def host_decode(i):
            img = cv2.imdecode(np.frombuffer(files[i], np.uint8), cv2.IMREAD_COLOR) if files[i] else None
            cv2.cvtColor(img, cv2.COLOR_BGR2RGB)        # raises on None exactly as preprocess_clip does
            host[i] = img

        for i in np.flatnonzero(batch.status != ops.JPEG_OK):
            host_decode(int(i))
        sizes = [(int(w), int(h)) for w, h in batch.sizes]
        for i, img in host.items():
            sizes[i] = (img.shape[1], img.shape[0])
        hmax, wmax = max(h for _, h in sizes), max(w for w, _ in sizes)
        out, status = batch.decode(hmax=hmax, wmax=wmax)
        late = [i for i in np.flatnonzero(status.cpu().numpy() != ops.JPEG_OK) if int(i) not in host]
        for i in late:
            host_decode(int(i))
        for i, img in host.items():
            out[i, :img.shape[0], :img.shape[1]] = torch.from_numpy(img).to(out.device)
        return out, sizes

    def embed_face_images(self, items):
        """The batched `run_clip(..., is_face=True)` face embedding (clearcam.py:671-678: preprocess_face, then adaface):
        items are `bytes` (an uploaded file) or the reference's paths relative to data/cameras -> (DeviceResult (n,512), rows):
        rows[i] is item i's row, or None where the reference's img_to_face finds no face (run_clip then returns no hits).
        The files are decoded as in `embed_images`.  A 112x112 image is embedded as the RGB image preprocess_face returns
        it; any other size goes through img_to_face on the device-decoded batch (canvas, BlazeFace, one read of the first
        detections for the host geometry, alignment), and all faces are embedded in one batch."""
        if self.adaface is None:
            raise CCError("the face embedder is off: call init_face() first")
        if not len(items):
            return DeviceResult(torch.empty(0, 512, device="cuda", dtype=torch.float32)), []
        out, sizes = self._decode_items(items)
        other = [i for i, wh in enumerate(sizes) if wh != (112, 112)]
        hw = [(sizes[i][1], sizes[i][0]) for i in other]
        aligned, arow = None, {}
        if other:
            self._need_detector()
            aligned, got = self._align_slots(out, other, hw, self._queue_first(out, other, hw).cpu().numpy())
            arow = dict(zip(other, got))
        rows, pick = [], []                                  # pick: (aligned face row) or (-1 - slot of a 112x112 image)
        for i in range(len(items)):
            r = arow.get(i, -1 - i)
            rows.append(None if r is None else len(pick))
            if r is not None:
                pick.append(r)
        if not pick:
            return DeviceResult(torch.empty(0, 512, device="cuda", dtype=torch.float32)), rows
        faces = torch.empty(len(pick), 112, 112, 3, dtype=torch.uint8, device="cuda")
        at = [j for j, r in enumerate(pick) if r >= 0]
        if at:
            faces[at] = aligned[[pick[j] for j in at]]
        at = [j for j, r in enumerate(pick) if r < 0]
        if at:                                               # preprocess_face's cvtColor(BGR2RGB) of a 112x112 upload
            faces[at] = out[[-1 - pick[j] for j in at], :112, :112].flip(-1)
        return DeviceResult(self.adaface.embed(faces)), rows

    def encode_embed_crops(self, frames, rects, quality: int = 95, bgr: bool = True, pix_fmt: str = BGR24):
        """Detector frame -> (the JPEG file of each object crop, exactly as `encode_crops` returns them, and DeviceResult
        (K, embed_dim): the embeddings `clip_latest_img` stores for those files).  The reference writes the crop with
        cv2.imwrite, reads the file back and embeds the decoded pixels (clearcam.py:272-279, 1278-1287); here the decoded
        pixels come from the encoder's quantised coefficients on the device (ops.jpeg_crops_decoded_frames), with no host
        round trip, and are embedded in one batch (a crop whose coefficients the device leaves to cv2 is decoded from its
        file on the host).  `encode_embed_frames` over the table of this batch."""
        if not 0 <= int(quality) <= 100:
            raise ValueError(f"quality must be in 0..100 (cv2's range), got {quality}")
        t, table, r = _device_crops(frames, rects, bgr, pix_fmt)
        return self._encode_embed(table, r, quality)[:2]

    def encode_embed_frames(self, frames, pix_fmts, rects, quality: int = 95):
        """`encode_embed_crops` for the objects of many frames of different shapes and formats in one call (the saves of
        every camera of a step): frames is a list of device frames, each [H,W,3] bgr24 or [H*3/2,W] yuv420p as its
        pix_fmts entry says (one format for all, or one per frame); rects: K rows (frame index into `frames`, x1, y1, x2,
        y2) -> (files, DeviceResult (K, embed_dim) or None).  File k is exactly what `encode_crops` writes for crop k of
        its frame alone, and embedding k what `encode_embed_crops` stores for it, in a batch padded to batch_bucket(K).
        Embeddings are None when CLIP is not initialised (the reference writes the thumbnails either way); then only the
        encoder runs, and the host waits twice, for the lengths and for the bytes.
        With CLIP, one encoder call, one crops-decoded call, one preprocess and one CLIP forward over all K crops are queued before
        anything is read; then the host waits twice, whatever the number of frames or crops: once for the files' lengths
        and the decoded crops' statuses together, once for the files' bytes.  A crop whose coefficients the device leaves
        to cv2 (CC_JPEG_UNSUPPORTED, which only very low qualities reach) is decoded from its file on the host; the
        preprocess then runs again over those crops only, and the CLIP forward is repeated on the same padded batch."""
        if not 0 <= int(quality) <= 100:
            raise ValueError(f"quality must be in 0..100 (cv2's range), got {quality}")
        table, sizes = ops.frame_table(frames, pix_fmts)
        return self._encode_embed(table, ops.table_rects(rects, sizes), quality)[:2]

    def encode_embed_faces_frames(self, frames, pix_fmts, rects, person, quality: int = 95):
        """`encode_embed_frames` and the faces of the person saves among the crops in the same call (`process_latest_face`,
        clearcam.py:1228-1241, on the thumbnail that save_object wrote and the queue read back as RGB): person is one bool per
        rect -> (files, embeddings, faces).  files and embeddings are exactly what `encode_embed_frames` returns; faces is a
        FaceSaves: the rects whose img_to_face finds a face, each face's JPEG as cv2.imwrite writes it at `quality`, and
        DeviceResult (f,512) of adaface(face); None when the face leg is off (`face` false).  Raises CCError before anything
        is queued when the face leg is on without a detector.
        The crops-decoded pixels (ops.jpeg_crops_decoded_frames) feed both legs.  Queued before the first read: the encoder,
        the decoded pixels, the CLIP preprocess and forward, and over the person crops the face canvas, BlazeFace and the
        first kept detection.  The host then waits once for the thumbnails' lengths, the decode statuses and the first rows
        together, runs the reference's face geometry, and queues the alignment, the faces' encoder and the AdaFace batch;
        it waits a second time for the thumbnails' bytes and the faces' lengths, and a third for the faces' bytes, whatever
        the number of frames, saves or faces.  A crop whose coefficients the device leaves to cv2 is decoded from its file on
        the host as in `encode_embed_frames`, and its face detection is run again (more waits, at very low qualities only)."""
        if not 0 <= int(quality) <= 100:
            raise ValueError(f"quality must be in 0..100 (cv2's range), got {quality}")
        table, sizes = ops.frame_table(frames, pix_fmts)
        r = ops.table_rects(rects, sizes)
        person = np.asarray(person, bool).reshape(-1)
        if len(person) != len(r):
            raise ValueError(f"{len(person)} person flags for {len(r)} rects")
        if self.face:
            self._need_detector()
        return self._encode_embed(table, r, quality, person if self.face else None)

    def _encode_embed(self, table, r, quality, person=None):
        """-> (files, CLIP embeddings or None, FaceSaves or None); person: None (no face leg) or one bool per rect."""
        K = len(r)
        persons = [] if person is None else [int(i) for i in np.flatnonzero(person)]
        none = lambda dim: DeviceResult(torch.empty(0, dim, device="cuda", dtype=torch.float32))   # noqa: E731
        no_faces = None if person is None else FaceSaves([], [], none(512))
        if K == 0:
            return [], (None if self.model is None else none(self.model.embed_dim)), no_faces
        out, lengths, offsets = ops.jpeg_encode_crops_frames(table, r, quality)
        if self.model is None and not persons:
            return ops.jpeg_collect(out, lengths, offsets), None, no_faces
        pix, status = ops.jpeg_crops_decoded_frames(table, r, quality)
        crops = [(i, 0, 0, int(x2 - x1), int(y2 - y1)) for i, (_, x1, y1, x2, y2) in enumerate(r)]
        hw = [(int(y2 - y1), int(x2 - x1)) for _, x1, y1, x2, y2 in r]
        x = emb = None
        if self.model is not None:
            x = self.preprocess_device(pix, crops, bgr=True, rows=batch_bucket(K)).tensor
            emb = self.model.precompute_embedding(x).tensor
        first = self._queue_first(pix, persons, [hw[i] for i in persons]) if persons else torch.empty(0, 17, device="cuda")
        lens, st, first = ops.read_together(lengths, status, first)                # host wait 1
        thumbs = ops.jpeg_gather(out, lengths, offsets, lens)
        files = None
        bad = [int(i) for i in np.flatnonzero(st != ops.JPEG_OK)]
        if bad:
            import cv2                                  # coefficients outside the range every libjpeg-turbo IDCT agrees on
            files = ops.jpeg_split(thumbs.cpu().numpy(), lens)
            for i in bad:
                img = cv2.imdecode(np.frombuffer(files[i], np.uint8), cv2.IMREAD_COLOR)
                pix[i, :img.shape[0], :img.shape[1]] = torch.from_numpy(img).to(pix.device)
            if x is not None:
                x[torch.tensor(bad, device=x.device)] = self.preprocess_device(pix, [crops[i] for i in bad], bgr=True).tensor
                emb = self.model.precompute_embedding(x).tensor
            redo = [j for j, i in enumerate(persons) if i in bad]
            if redo:
                first[redo] = self._queue_first(pix, [persons[j] for j in redo], [hw[persons[j]] for j in redo]).cpu().numpy()
        emb = None if emb is None else DeviceResult(emb[:K])
        if person is None:
            return (ops.jpeg_split(thumbs.cpu().numpy(), lens) if files is None else files), emb, None  # host wait 2
        faces, got = self._align_slots(pix, persons, [hw[i] for i in persons], first)
        rows = [i for i, g in zip(persons, got) if g is not None]
        if not rows:
            return (ops.jpeg_split(thumbs.cpu().numpy(), lens) if files is None else files), emb, no_faces
        from ..pixfmt import CC_FRAME_BGR_U8
        fout, flengths, foffsets = ops.jpeg_encode_crops_frames(ops.batch_table(faces, CC_FRAME_BGR_U8),
                                                                [(j, 0, 0, 112, 112) for j in range(len(rows))], quality)
        femb = DeviceResult(self.adaface.embed(faces))
        if files is None:
            flat, flens = ops.read_together(thumbs, flengths)                    # host wait 2
            files = ops.jpeg_split(flat, lens)
        else:
            flens = flengths.cpu().numpy()
        return files, emb, FaceSaves(rows, ops.jpeg_collect(fout, flengths, foffsets, flens), femb)   # host wait 3

    def _device_index(self, is_face=False):
        """Contiguous device copy of `image_embeddings` (`face_embeddings` when is_face) plus, per row, what `search`
        filters and groups on — rebuilt whenever a key OR the array stored under a key changes (the fingerprint holds the
        identity of every value, so an embedding replaced under an existing path is seen).  Returns (paths, device [N,D],
        meta)."""
        embeddings = self.face_embeddings if is_face else self.image_embeddings
        keys = [k for k, v in embeddings.items() if v is not None]
        fp = tuple(id(embeddings[k]) for k in keys)
        cached = self._index.get(is_face)
        if cached is None or cached[0] != keys or cached[3] != fp:
            mat = np.concatenate([np.asarray(embeddings[k], np.float32).reshape(1, -1) for k in keys]) if keys \
                else np.zeros((0, self.model.embed_dim if self.model else 1), np.float32)
            n = len(keys)
            norm = np.array([k.replace("\\", "/") for k in keys], dtype=str) if n else np.zeros(0, dtype=str)
            jpg = np.zeros(n, bool)
            truthy = np.zeros(n, bool)
            group = np.arange(n, dtype=np.int32)             # a row without an object id is its own group
            first = {}
            for i, k in enumerate(keys):
                filename = os.path.basename(k)
                if not filename.lower().endswith(".jpg"):     # models/objects.py:370: only .jpg rows are candidates
                    continue
                jpg[i] = True
                oid = event_img_info(filename.split(".jpg")[0])["object_id"] if "_" in filename else None
                if oid is not None:
                    group[i] = first.setdefault(oid, i)       # group id = first row of that object id
                    truthy[i] = bool(oid)
            meta = {"norm": norm, "jpg": jpg, "truthy": truthy, "group": torch.from_numpy(group).cuda(),
                    "ident": torch.arange(n, dtype=torch.int32, device="cuda"),
                    "work": torch.empty(max(n, 1), dtype=torch.int64, device="cuda")}
            self._index[is_face] = (keys, torch.from_numpy(mat).cuda(), meta, fp)
        return self._index[is_face][:3]

    def search(self, query=None, top_k=10, cam_name=None, timestamp=None, text_embedding=None, is_face=False):
        """models/objects.py:356-390 — same filtering, best score per object id, descending order, top_k — with the N dot
        products, the per-object maximum and the top-k selection in one device pass over the contiguous index
        (cc_search_topk): only the k winners come back over PCIe.  (An exact score tie goes to the earlier index row.)
        is_face=True searches `face_embeddings` with the embedding given (`adaface(img).numpy()` in run_clip), under the
        same filters; as in the reference, its date filter looks for "/objects/<date>/" in the stored path."""
        if not (self.face_embeddings if is_face else self.image_embeddings):
            print("No embeddings available.")
            return []
        if text_embedding is None:
            text_embedding = self.model._encode_text(query).numpy()
        keys, index, meta = self._device_index(is_face)
        n = len(keys)
        if n == 0 or top_k <= 0:
            return []
        mask = meta["jpg"]
        if cam_name:
            mask = mask & (np.char.find(meta["norm"], f"/cameras/{cam_name}/") >= 0)
        if timestamp:
            mask = mask & ((np.char.find(meta["norm"], f"/objects/{timestamp}/") >= 0) | (np.char.find(meta["norm"], "/objects/video/") >= 0))
        # the reference groups by object id only when some candidate has a (non-empty) one (:377)
        group = meta["group"] if bool((meta["truthy"] & mask).any()) else meta["ident"]
        dmask = None if bool(mask.all()) else torch.from_numpy(np.ascontiguousarray(mask.astype(np.uint8))).cuda()
        q = torch.from_numpy(np.ascontiguousarray(np.asarray(text_embedding, np.float32).reshape(-1))).cuda()
        k = int(min(top_k, n))
        rows = torch.empty(k, dtype=torch.int32, device="cuda")
        scores = torch.empty(k, dtype=torch.float32, device="cuda")
        check(lib().cc_search_topk(ptr(index), n, index.shape[1], ptr(q), ptr(group), ptr(dmask), n, k, ptr(meta["work"]), ptr(rows),
                                   ptr(scores), stream_ptr()), "cc_search_topk")
        rows, scores = rows.cpu().numpy(), scores.cpu().numpy()
        return [(keys[r], float(sc)) for r, sc in zip(rows, scores) if r >= 0]

    def _load_all_embeddings(self, face=False):
        """models/objects.py:392-421: merge every <cam>/objects/<date>/embeddings.pkl into image_embeddings."""
        valid, target = set(), (self.face_embeddings if face else self.image_embeddings)
        if not os.path.isdir(self.base_path):
            return
        for cam in os.listdir(self.base_path):
            objects = os.path.join(self.base_path, cam, "faces" if face else "objects")
            if not os.path.isdir(objects):
                continue
            for date in os.listdir(objects):
                cache = os.path.join(objects, date, "embeddings.pkl")
                if not os.path.exists(cache):
                    continue
                with open(cache, "rb") as f:
                    emb = pickle.load(f).get("embeddings", {})
                valid.update(emb.keys())
                target.update(emb)
        for k in set(target.keys()) - valid:
            del target[k]
        self._index.pop(face, None)
