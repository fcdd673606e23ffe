"""clearcam_b200 — H100-native (sm_90a) YOLOv9 + CLIP hot path behind the reference's Python signatures."""
from ._lib import CCError, lib, LIB_PATH  # noqa: F401
