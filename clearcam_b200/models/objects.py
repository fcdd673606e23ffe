"""Drop-in for the reference's `models/objects.py` CLIP part on H100 (same names and call signatures).

    from clearcam_b200.models.objects import ObjectFinder
    finder = ObjectFinder(); finder.init_clip(weights=..., arch="ViT-L/14")
    emb  = finder.model.precompute_embedding(x).numpy()            # x (B,3,224,224) float32  (clearcam.py:1285)
    temb = finder.model._encode_text("ferrari f40", realize=True)  # (768,)                   (clearcam.py:667)
    hits = finder.search("ferrari f40", top_k=10)                  # [(path, score)]          (models/objects.py:356)

Mirrors class OpenCLIP (/root/reference/models/objects.py:21-143), encode_text (:145-186) and ObjectFinder's CLIP
methods (:189-206, :237-251, :356-421), and the face embedder's (`init_face`, `turn_off_face`, `adaface`,
`preprocess_face` for 112x112 faces, face search; :207-217, :253-261).  Face detection and alignment (BlazeFace,
`img_to_face`, :263-354) are not built yet.  All arithmetic runs in libclearcam_b200.so; there is no CPU fallback.

Additions: `arch=` (the reference hard-codes ViT-L/14; "ViT-B/32" runs the same kernels), explicit `weights=`
(the reference downloads from HuggingFace, :91), `encode_text_batch`, a contiguous device index for search, and
`gather=` to all-gather embeddings across ranks (NCCL) straight from the kernel's output slice.
"""
from __future__ import annotations

import ctypes
import os
import pickle
from typing import Dict, List, Optional

import numpy as np
import torch

from .._lib import CCError, check, lib, ptr, stream_ptr
from ..detection.yolov9 import DeviceResult, _to_host_fp32, fetch, safe_load
from ..pixfmt import BGR24, check_pix_fmt, yuv420p_size
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


class OpenCLIP:
    def __init__(self, base_path="data/cameras", weights=None, arch: str = "ViT-L/14"):
        self.base_path = base_path
        self.arch = arch
        self.cfg = ARCHS[arch]
        self.embed_dim = self.cfg[6]
        self.image_size = self.cfg[0]
        self.ctx = self.cfg[12]
        self.tokenizer = SimpleTokenizer()
        self._h = None
        if weights is None:
            weights = safe_load(fetch("https://huggingface.co/roryclear/CLIP-ViT-L-14-laion2B-s32B-b82K/resolve/main/"
                                      "CLIP-ViT-L-14-laion2B-s32B-b82K.safetensors"))
        elif isinstance(weights, (str, os.PathLike)):
            weights = safe_load(weights)
        self.load_weights(weights)

    def load_weights(self, state_dict) -> None:
        L = lib()
        if L.cc_device_check() <= 0:
            raise CCError("clearcam_b200 needs an H100 (sm_90) GPU: " + L.cc_last_error().decode())
        items = [(k, _to_host_fp32(v)) for k, v in state_dict.items() if k != "attn_mask"]
        names = (ctypes.c_char_p * len(items))(*[k.encode() for k, _ in items])
        ptrs = (ctypes.c_void_p * len(items))(*[a.ctypes.data for _, a in items])
        nums = (ctypes.c_int64 * len(items))(*[a.size for _, a in items])
        cfg = _ClipConfig(*self.cfg)
        h = ctypes.c_void_p()
        check(L.cc_clip_create(ctypes.byref(cfg), len(items), names, ptrs, nums, ctypes.byref(h)), "cc_clip_create")
        if self._h is not None:
            L.cc_clip_destroy(self._h)
        self._h = h

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                lib().cc_clip_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- image tower
    @staticmethod
    def _as_device(x, dtype) -> torch.Tensor:
        if isinstance(x, DeviceResult):
            x = x.tensor
        if not isinstance(x, torch.Tensor):
            if hasattr(x, "numpy") and not isinstance(x, np.ndarray):
                x = x.numpy()
            x = torch.from_numpy(np.ascontiguousarray(x))
        return x.to("cuda", dtype, non_blocking=True).contiguous()

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
    (bgr24) or [n,H*3/2,W] / [H*3/2,W] (yuv420p), host or device; rects K rows of (frame, x1, y1, x2, y2) or (x1, y1, x2,
    y2).  -> (contiguous device frames [n,...], H, W, the C-ABI src_fmt (0 RGB, 1 BGR, 2 I420), int32 rects [K,5])."""
    t = frames.tensor if isinstance(frames, DeviceResult) else frames
    if not isinstance(t, torch.Tensor):
        t = torch.from_numpy(np.ascontiguousarray(t))
    if check_pix_fmt(pix_fmt) == BGR24:
        if t.dim() == 3:
            t = t.unsqueeze(0)
        if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[-1] != 3:
            raise ValueError("frames must be uint8 [n,H,W,3]")
        H, W, src_fmt = t.shape[1], t.shape[2], 1 if bgr else 0
    else:
        if t.dim() == 2:
            t = t.unsqueeze(0)
        if t.dtype != torch.uint8 or t.dim() != 3:
            raise ValueError(f"yuv420p frames must be uint8 [n,H*3/2,W], got {t.dtype} {tuple(t.shape)}")
        (H, W), src_fmt = yuv420p_size(t.shape), 2
    t = t.to("cuda", non_blocking=True).contiguous()
    r = np.asarray(rects, np.int32).reshape(-1, np.shape(rects)[-1] if len(rects) else 5)
    if r.shape[1] == 4:
        r = np.concatenate([np.zeros((len(r), 1), np.int32), r], 1)
    return t, H, W, src_fmt, np.ascontiguousarray(r, np.int32)


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

    def init_face(self, weights=None):
        """models/objects.py:211-215 without BlazeFace (face detection is not built yet): the AdaFace embedder, from the
        reference's state dict / safetensors path, or the reference's file when None."""
        if self.face:
            return
        from .adaface import ADAFACE
        self.adaface = ADAFACE(weights)
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
        already a 112x112 face.  Other sizes need face detection and alignment (`img_to_face`), which is not built yet."""
        import cv2
        if type(img) == bytes:
            img = cv2.imdecode(np.frombuffer(img, np.uint8), cv2.IMREAD_COLOR)
        else:
            img = cv2.imread(f"data/cameras{img}")
        img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        if img.shape != (112, 112, 3):
            raise CCError(f"preprocess_face: a {img.shape[1]}x{img.shape[0]} image needs face detection and alignment "
                          "(img_to_face), which is not built yet; only 112x112 faces are accepted")
        return img

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
        t, H, W, src_fmt, r = _device_crops(frames, rects, bgr, pix_fmt)
        s = size or (self.model.image_size if self.model is not None else 224)
        # rows > K: the result is allocated with `rows` images, the first K filled and the rest zero (batch padding)
        out = torch.empty(len(r), 3, s, s, device="cuda", dtype=torch.float32) if not rows or rows <= len(r) else \
            torch.zeros(rows, 3, s, s, device="cuda", dtype=torch.float32)
        check(lib().cc_clip_preprocess(ptr(t), t.shape[0], H, W, r.ctypes.data, len(r), s, src_fmt, ptr(out), stream_ptr(None)),
              "cc_clip_preprocess")
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
        from .. import ops
        if not 0 <= int(quality) <= 100:
            raise ValueError(f"quality must be in 0..100 (cv2's range), got {quality}")
        t, _, _, src_fmt, r = _device_crops(frames, rects, bgr, pix_fmt)
        return ops.jpeg_encode_crops(t, r, quality, src_fmt)

    def embed_images(self, items):
        """The batched device form of `run_clip`'s `preprocess_clip` + `precompute_embedding` (clearcam.py:671-678,
        models/objects.py:244-251): items are `bytes` (an uploaded file) or the reference's paths relative to data/cameras
        (stored thumbnails) -> DeviceResult (K, embed_dim).  The files are decoded on the device (ops.jpeg_decode), then
        cropped, resized and normalised by cc_clip_preprocess and embedded in one batch.  A file the device reports as
        unsupported or corrupt is decoded by cv2 on the host and joins the same batch; where cv2 returns None this raises as
        the reference's cvtColor does."""
        import cv2
        from .. import ops
        k = len(items)
        if k == 0:
            return DeviceResult(torch.empty(0, self.model.embed_dim, device="cuda", dtype=torch.float32))
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
        rects = [(i, 0, 0, w, h) for i, (w, h) in enumerate(sizes)]
        x = self.preprocess_device(out, rects, bgr=True, rows=batch_bucket(k))
        return DeviceResult(self.model.precompute_embedding(x).tensor[:k])

    def encode_embed_crops(self, frames, rects, quality: int = 95, bgr: bool = True, pix_fmt: str = BGR24):
        """Detector frame -> (the JPEG file of each object crop, exactly as `encode_crops` returns them, and DeviceResult
        (K, embed_dim): the embeddings `clip_latest_img` stores for those files).  The reference writes the crop with
        cv2.imwrite, reads the file back and embeds the decoded pixels (clearcam.py:272-279, 1278-1287); here the decoded
        pixels come from the encoder's quantised coefficients on the device (ops.jpeg_crops_decoded), with no host round
        trip, and are embedded in one batch (a crop whose coefficients the device leaves to cv2 is decoded from its file on
        the host)."""
        from .. import ops
        files = self.encode_crops(frames, rects, quality, bgr, pix_fmt)
        k = len(files)
        if k == 0:
            return files, DeviceResult(torch.empty(0, self.model.embed_dim, device="cuda", dtype=torch.float32))
        t, _, _, src_fmt, r = _device_crops(frames, rects, bgr, pix_fmt)
        pix, status = ops.jpeg_crops_decoded(t, r, quality, src_fmt)
        for i in np.flatnonzero(status.cpu().numpy() != ops.JPEG_OK):
            import cv2                                  # coefficients outside the range every libjpeg-turbo IDCT agrees on
            img = cv2.imdecode(np.frombuffer(files[i], np.uint8), cv2.IMREAD_COLOR)
            pix[i, :img.shape[0], :img.shape[1]] = torch.from_numpy(img).to(pix.device)
        crops = [(i, 0, 0, int(x2 - x1), int(y2 - y1)) for i, (_, x1, y1, x2, y2) in enumerate(r)]
        x = self.preprocess_device(pix, crops, bgr=True, rows=batch_bucket(k))
        return files, DeviceResult(self.model.precompute_embedding(x).tensor[:k])

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
        from .. import ops
        if not 0 <= int(quality) <= 100:
            raise ValueError(f"quality must be in 0..100 (cv2's range), got {quality}")
        frames = list(frames)
        table, sizes = ops.frame_table(frames, pix_fmts)
        r = ops.table_rects(rects, sizes)
        K = len(r)
        if K == 0:
            return [], (None if self.model is None else
                        DeviceResult(torch.empty(0, self.model.embed_dim, device="cuda", dtype=torch.float32)))
        out, lengths, offsets = ops.jpeg_encode_launch_frames(table, len(frames), r, quality, frames[0].device)
        if self.model is None:
            return ops.jpeg_collect(out, lengths, lengths.cpu().numpy(), offsets), None
        pix, status = ops.jpeg_crops_decoded_frames(frames, pix_fmts, r, quality, table=(table, r))
        crops = [(i, 0, 0, int(x2 - x1), int(y2 - y1)) for i, (_, x1, y1, x2, y2) in enumerate(r)]
        x = self.preprocess_device(pix, crops, bgr=True, rows=batch_bucket(K)).tensor
        emb = self.model.precompute_embedding(x).tensor
        got = torch.cat([lengths, status.long()]).cpu().numpy()                 # host wait 1
        files = ops.jpeg_collect(out, lengths, got[:K], offsets)                # host wait 2
        bad = [int(i) for i in np.flatnonzero(got[K:] != ops.JPEG_OK)]
        if bad:
            import cv2                                  # coefficients outside the range every libjpeg-turbo IDCT agrees on
            for i in bad:
                img = cv2.imdecode(np.frombuffer(files[i], np.uint8), cv2.IMREAD_COLOR)
                pix[i, :img.shape[0], :img.shape[1]] = torch.from_numpy(img).to(pix.device)
            x[torch.tensor(bad, device=x.device)] = self.preprocess_device(pix, [crops[i] for i in bad], bgr=True).tensor
            emb = self.model.precompute_embedding(x).tensor
        return files, DeviceResult(emb[:K])

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
