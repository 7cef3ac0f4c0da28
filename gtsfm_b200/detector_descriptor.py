"""SuperPoint detector-descriptor plugin.

Drop-in for gtsfm/frontend/detector_descriptor/superpoint.py:32-93 (`SuperPointDetectorDescriptor`): same constructor
arguments, same `detect_and_describe(image) -> (Keypoints, (N, 256) float32)` contract, same post-processing order
(mask filter, then `Keypoints.get_top_k` i.e. numpy argpartition, gtsfm/.../superpoint.py:87-91), lazily created
device state so the object stays picklable (tests/frontend/detector/test_detector_base.py:51-56).

All arithmetic runs in libgtsfm_b200.so (CUDA, sm_90a); this file only moves numpy buffers across the C ABI.  The one
deliberate difference from the reference data flow: descriptors are sampled on the GPU only for the keypoints that
survive the host-side mask / top-k selection, instead of for every detection (identical values, 3x less D2H at 5000 of
17000 keypoints).
"""
from __future__ import annotations

import threading
from pathlib import Path
from typing import Optional, Tuple, Union

import numpy as np

from . import _lib, weights
from .gtsfm_api import DetectorDescriptorBase, Image, Keypoints

KEYPOINT_THRESHOLD = 0.005  # thirdparty/.../superpoint.py:104-110 default_config
NMS_RADIUS = 4
REMOVE_BORDERS = 4
DESC_DIM = 256


class SuperPointEngine:
    """Thin host object over the C ABI (one context, one set of uploaded weights)."""

    def __init__(self, state_dict, device: int = 0, ctx: Optional[_lib.Context] = None):
        self.ctx = ctx or _lib.Context(device)
        blob = weights.pack_superpoint(weights.load_state_dict(state_dict))
        self.ctx.check(self.ctx.lib.b2_superpoint_set_weights(self.ctx.handle, _lib.ptr(blob), blob.size), "superpoint_set_weights")
        self.h2d_bytes = 0  # bytes this engine copied host->device / device->host (bench.py's e2e accounting)
        self.d2h_bytes = 0
        self.map_token = 0  # dense descriptor map left by the last detect (describe refuses any other)
        self.lock = threading.RLock()  # detect + describe of one image form one critical section (shared plugin, threads)

    @staticmethod
    def capacity(h: int, w: int) -> int:
        """Upper bound on NMS survivors: radius-4 maxima are >= 5 apart in Chebyshev distance."""
        return ((h // 8) * 8 // 5 + 1) * ((w // 8) * 8 // 5 + 1)

    def detect(self, image_u8: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        img = np.ascontiguousarray(image_u8)
        if img.dtype != np.uint8:
            raise ValueError("image must be uint8")
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else img.shape[2]
        cap = self.capacity(h, w)
        xy = np.empty((cap, 2), np.float32)
        sc = np.empty(cap, np.float32)
        n = _lib.C.c_int(0)
        tok = _lib.C.c_uint64(0)
        rc = self.ctx.lib.b2_superpoint_detect_host(self.ctx.handle, _lib.ptr(img), h, w, ch, KEYPOINT_THRESHOLD, NMS_RADIUS,
                                                    REMOVE_BORDERS, _lib.ptr(xy), _lib.ptr(sc), cap, _lib.C.byref(n), _lib.C.byref(tok))
        self.ctx.check(rc, "superpoint_detect")
        self.map_token = tok.value
        k = min(n.value, cap)
        self.h2d_bytes += img.nbytes
        self.d2h_bytes += k * 12 + 4
        return xy[:k].copy(), sc[:k].copy()

    def describe(self, xy: np.ndarray, map_token: Optional[int] = None) -> np.ndarray:
        """Samples the dense map of the detect call that issued `map_token` (default: this engine's last detect); raises
        B200Error if another image has been detected on the context in between."""
        xy = np.ascontiguousarray(xy, np.float32)
        out = np.empty((len(xy), DESC_DIM), np.float32)
        tok = self.map_token if map_token is None else int(map_token)
        self.ctx.check(self.ctx.lib.b2_superpoint_describe_host(self.ctx.handle, tok, _lib.ptr(xy), len(xy), _lib.ptr(out)), "superpoint_describe")
        self.h2d_bytes += xy.nbytes
        self.d2h_bytes += out.nbytes
        return out


class B200SuperPointDetectorDescriptor(DetectorDescriptorBase):
    """SuperPoint on hand-written sm_90a kernels behind GTSfM's DetectorDescriptorBase."""

    def __init__(self, max_keypoints: int = 5000, use_cuda: bool = True, weights_path: Union[Path, str, dict, None] = None,
                 device: int = 0) -> None:
        super().__init__(max_keypoints=max_keypoints)
        if weights_path is None:
            raise FileNotFoundError("SuperPoint weights_path is required (a superpoint_v1.pth-style checkpoint)")
        if not isinstance(weights_path, dict) and not Path(weights_path).exists():
            raise FileNotFoundError(  # same failure as gtsfm/.../superpoint.py:50-54
                f"SuperPoint weights not found at {weights_path}. Please run 'bash scripts/download_model_weights.sh' from the repo root.")
        self._use_cuda = use_cuda  # kept for signature compatibility; this plugin has no CPU path
        self._weights = weights_path
        self._device = device
        self._engine: Optional[SuperPointEngine] = None  # lazy, never pickled

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> SuperPointEngine:
        if self._engine is None:
            self._engine = SuperPointEngine(self._weights, self._device)
        return self._engine

    def detect_and_describe(self, image: Image) -> Tuple[Keypoints, np.ndarray]:
        eng = self._ensure_engine()
        arr = image.value_array
        if arr.ndim == 3 and arr.shape[2] not in (3, 4):
            raise ValueError("Input image dimensions are wrong")  # gtsfm/utils/images.py:39-40
        with eng.lock:  # the dense map lives in the context between the two C calls
            xy, sc = eng.detect(arr)
            token = eng.map_token
            keypoints = Keypoints(xy, scales=None, responses=sc)
            if getattr(image, "mask", None) is not None:
                keypoints, _ = keypoints.filter_by_mask(image.mask)
            keypoints, _ = keypoints.get_top_k(self.max_keypoints)
            if len(keypoints) == 0:
                return keypoints, np.zeros((0, DESC_DIM), np.float32)
            descriptors = eng.describe(np.asarray(keypoints.coordinates, np.float32), token)
        return keypoints, descriptors
