"""SuperPoint, SIFT, ORB and D2-Net detector-descriptor plugins.

Drop-in for gtsfm/frontend/detector_descriptor/superpoint.py:32-93 (`SuperPointDetectorDescriptor`): same constructor
arguments, same `detect_and_describe(image) -> (Keypoints, (N, 256) float32)` contract, same post-processing order
(mask filter, then `Keypoints.get_top_k` i.e. numpy argpartition, gtsfm/.../superpoint.py:87-91), lazily created
device state so the object stays picklable (tests/frontend/detector/test_detector_base.py:51-56).

All arithmetic runs in libgtsfm_b200.so (CUDA, sm_90a); this file only moves numpy buffers across the C ABI.  The one
deliberate difference from the reference data flow: descriptors are sampled on the GPU only for the keypoints that
survive the host-side mask / top-k selection, instead of for every detection (identical values, 3x less D2H at 5000 of
17000 keypoints).

`B200SIFTDetectorDescriptor` is the drop-in for gtsfm/frontend/detector_descriptor/sift.py:24-55 (`SIFTDetectorDescriptor`):
cv2.SIFT_create() with its defaults, restated in csrc/sift.cu.  Its one deliberate difference: an image without keypoints
gives (empty Keypoints, (0, 128) float32) where the reference raises a TypeError.

`B200ORBDetectorDescriptor` is the drop-in for gtsfm/frontend/detector_descriptor/orb.py (`ORBDetectorDescriptor`):
cv2.ORB_create() with its defaults, restated in csrc/orb.cu.

`B200D2NetDetectorDescriptor` is the drop-in for gtsfm/frontend/detector_descriptor/d2net.py (`D2NetDetDesc`), single scale, restated
in csrc/d2net.cu.
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


SIFT_DESC_DIM = 128
SIFT_WORKSPACE_BUDGET = 4 << 30  # bytes of device workspace one batched call may use (csrc/sift.cu: ~151 H W per image)


class SiftEngine:
    """cv2.SIFT_create() defaults on csrc/sift.cu: host calls (every keypoint, as cv2 returns them) and batched device calls
    (the max_keypoints largest responses, uint8 descriptors left on the GPU for TwoWayEngine.match_batched_dev)."""

    DESC_DIM = SIFT_DESC_DIM
    WORKSPACE_PER_PIXEL = 151  # device workspace bytes per image pixel of a batched call
    HOST_CALL, BATCHED_CALL, IMAGE_T = "b2_sift_detect_host", "b2_sift_detect_batched_dev", _lib.SiftImage

    def __init__(self, device: int = 0, ctx: Optional[_lib.Context] = None, capacity: int = 8192):
        self.ctx = ctx or _lib.Context(device)
        self.capacity = capacity  # first guess of the host call's output size; grown to the count the library reports
        self.lock = threading.RLock()

    def detect_and_describe(self, image: np.ndarray, mask: Optional[np.ndarray] = None):
        """Host uint8 image (H, W) / (H, W, 3) / (H, W, 4) and optional (H, W) mask -> (keypoint records
        `_lib.SIFT_KEYPOINT_DTYPE`, (N, 128) uint8 descriptors), every keypoint in cv2's order."""
        img = np.ascontiguousarray(image)
        if img.dtype != np.uint8:
            raise ValueError("image must be uint8")
        if img.ndim == 3 and img.shape[2] not in (3, 4) or img.ndim not in (2, 3):
            raise ValueError("Input image dimensions are wrong")
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else img.shape[2]
        m = None
        if mask is not None:
            if mask.shape[:2] != (h, w):
                raise ValueError("mask must have the image's height and width")
            m = np.ascontiguousarray(mask != 0, np.uint8)
        with self.lock:
            while True:
                cap = self.capacity
                kp = np.empty(cap, _lib.SIFT_KEYPOINT_DTYPE)
                desc = np.empty((cap, self.DESC_DIM), np.uint8)
                n = _lib.C.c_int(0)
                rc = getattr(self.ctx.lib, self.HOST_CALL)(self.ctx.handle, _lib.ptr(img), h, w, ch, _lib.ptr(m), _lib.ptr(kp),
                                                           _lib.ptr(desc), cap, _lib.C.byref(n))
                if rc == _lib.SIFT_CAPACITY:
                    self.capacity = n.value
                    continue
                self.ctx.check(rc, self.HOST_CALL[3:])
                return kp[: n.value].copy(), desc[: n.value].copy()

    @classmethod
    def images_per_call(cls, h: int, w: int) -> int:
        return int(max(1, min(64, SIFT_WORKSPACE_BUDGET // (cls.WORKSPACE_PER_PIXEL * h * w))))

    def extract_many(self, images, masks=None, max_keypoints: int = 5000):
        """images: sequence of same-shape CUDA uint8 tensors (H, W) / (H, W, C), rows may be pitched (stride(0) >= W C, unit
        inner strides); masks: None or a per-image sequence of CUDA (H, W) uint8 tensors / None.  -> list of (keypoint records
        as a (n, 6) float32 view [x, y, size, angle, response, octave bits], (n, DESC_DIM) uint8 descriptors, total before
        top-k)."""
        import torch

        if len(images) == 0:
            return []
        shape = tuple(images[0].shape)
        if any(tuple(x.shape) != shape for x in images):
            raise ValueError("extract_many takes images of one shape")
        h, w = shape[:2]
        ch = 1 if len(shape) == 2 else shape[2]
        masks = [None] * len(images) if masks is None else list(masks)
        dev = images[0].device
        per = self.images_per_call(h, w)
        out = []
        with self.lock:
            for c0 in range(0, len(images), per):
                idx = range(c0, min(len(images), c0 + per))
                st = (self.IMAGE_T * len(idx))()
                keep = []
                pitch = None
                for s, i in enumerate(idx):
                    x = images[i]
                    if x.dtype != torch.uint8:
                        raise ValueError("images must be uint8")
                    if x.stride(-1) != 1 or (x.dim() == 3 and x.stride(1) != ch):
                        x = x.contiguous()
                    p = x.stride(0)
                    if pitch is None:
                        pitch = p
                    elif p != pitch:
                        x = x.contiguous()
                        if x.stride(0) != pitch:
                            raise ValueError("images of one call must share a row pitch")
                    m = masks[i]
                    if m is not None:
                        m = (m != 0).to(torch.uint8).contiguous()
                    kp = torch.empty((max_keypoints, 6), dtype=torch.float32, device=dev)
                    desc = torch.empty((max_keypoints, self.DESC_DIM), dtype=torch.uint8, device=dev)
                    keep.append((x, m, kp, desc))
                    st[s] = self.IMAGE_T(x.data_ptr(), 0 if m is None else m.data_ptr(), int(max_keypoints), kp.data_ptr(),
                                         desc.data_ptr(), 0, 0)
                stream = torch.cuda.current_stream(dev).cuda_stream
                rc = getattr(self.ctx.lib, self.BATCHED_CALL)(self.ctx.handle, st, len(idx), h, w, ch, int(pitch),
                                                              _lib.C.c_void_p(stream))
                self.ctx.check(rc, self.BATCHED_CALL[3:])
                for s, (_, _, kp, desc) in enumerate(keep):
                    n = st[s].out_n
                    out.append((kp[:n], desc[:n], st[s].out_total))
        return out


class B200SIFTDetectorDescriptor(DetectorDescriptorBase):
    """cv2 SIFT (default parameters) on hand-written sm_90a kernels behind GTSfM's DetectorDescriptorBase."""

    def __init__(self, max_keypoints: int = 5000, device: int = 0) -> None:
        super().__init__(max_keypoints=max_keypoints)
        self._device = device
        self._engine: Optional[SiftEngine] = None  # lazy, never pickled

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> SiftEngine:
        if self._engine is None:
            self._engine = SiftEngine(self._device)
        return self._engine

    def detect_and_describe(self, image: Image) -> Tuple[Keypoints, np.ndarray]:
        arr = image.value_array
        if arr.ndim == 3 and arr.shape[2] not in (3, 4):
            raise ValueError("Input image dimensions are wrong")  # gtsfm/utils/images.py:39-40
        kp, desc = self._ensure_engine().detect_and_describe(arr, getattr(image, "mask", None))
        if len(kp) == 0:
            return Keypoints(np.zeros((0, 2))), np.zeros((0, SIFT_DESC_DIM), np.float32)
        keypoints = Keypoints(np.stack([kp["x"], kp["y"]], 1).astype(np.float64), scales=kp["size"].astype(np.float64),
                              responses=kp["response"].astype(np.float64))
        keypoints, sel = keypoints.get_top_k(self.max_keypoints)  # gtsfm/.../sift.py:53-54
        return keypoints, desc[sel].astype(np.float32)


ORB_DESC_DIM = 32


class OrbEngine(SiftEngine):
    """cv2.ORB_create() defaults on csrc/orb.cu, with SiftEngine's calls: `detect_and_describe` returns every keypoint (level by
    level, response descending, then y, x), `extract_many` leaves (n, 32) uint8 descriptors on the GPU, which
    b2_mnn_match_batched_dev takes as they are (u8, dim 32)."""

    DESC_DIM = ORB_DESC_DIM
    WORKSPACE_PER_PIXEL = 40
    HOST_CALL, BATCHED_CALL, IMAGE_T = "b2_orb_detect_host", "b2_orb_detect_batched_dev", _lib.OrbImage

    def __init__(self, device: int = 0, ctx: Optional[_lib.Context] = None, capacity: int = 1024):
        super().__init__(device, ctx, capacity)


class B200ORBDetectorDescriptor(DetectorDescriptorBase):
    """cv2 ORB (default parameters) on hand-written sm_90a kernels behind GTSfM's DetectorDescriptorBase; the drop-in for
    gtsfm/frontend/detector_descriptor/orb.py (`ORBDetectorDescriptor`).  Its one deliberate difference: an image without
    keypoints gives (empty Keypoints, (0, 32) uint8) where the reference raises a TypeError."""

    def __init__(self, max_keypoints: int = 5000, device: int = 0) -> None:
        super().__init__(max_keypoints=max_keypoints)
        self._device = device
        self._engine: Optional[OrbEngine] = None  # lazy, never pickled

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> OrbEngine:
        if self._engine is None:
            self._engine = OrbEngine(self._device)
        return self._engine

    def detect_and_describe(self, image: Image) -> Tuple[Keypoints, np.ndarray]:
        arr = image.value_array
        if arr.ndim == 3 and arr.shape[2] not in (3, 4):
            raise ValueError("Input image dimensions are wrong")  # gtsfm/utils/images.py:39-40
        kp, desc = self._ensure_engine().detect_and_describe(arr, getattr(image, "mask", None))
        return orb_keypoints(kp, desc, self.max_keypoints)


def orb_keypoints(kp: np.ndarray, desc: np.ndarray, max_keypoints: int) -> Tuple[Keypoints, np.ndarray]:
    """ORB keypoint records and descriptors -> the reference's (Keypoints(coordinates, scales=size, responses), uint8
    descriptors) after get_top_k (gtsfm/.../orb.py:51-57)."""
    if len(kp) == 0:
        return Keypoints(np.zeros((0, 2))), np.zeros((0, ORB_DESC_DIM), np.uint8)
    keypoints = Keypoints(np.stack([kp["x"], kp["y"]], 1).astype(np.float64), scales=kp["size"].astype(np.float64),
                          responses=kp["response"].astype(np.float64))
    keypoints, sel = keypoints.get_top_k(max_keypoints)
    return keypoints, desc[sel]


D2NET_DESC_DIM = 512
D2NET_MAX_EDGE_PX, D2NET_MAX_SUM_EDGES_PX = 1600, 2800  # gtsfm/.../d2net.py:22-23
D2NET_MODEL_SUBPATH = Path("thirdparty") / "d2net" / "weights" / "d2_tf.pth"


def default_d2net_model_path() -> Path:
    """The reference's default (gtsfm/.../d2net.py:29): thirdparty/d2net/weights/d2_tf.pth under the root of the GTSfM checkout,
    found from the importable `gtsfm` package.  Without one, the same relative path under the working directory."""
    try:
        import importlib.util

        spec = importlib.util.find_spec("gtsfm")
    except (ImportError, ValueError):
        spec = None
    if spec is not None and spec.origin:
        return Path(spec.origin).resolve().parent.parent / D2NET_MODEL_SUBPATH
    return Path.cwd() / D2NET_MODEL_SUBPATH


class D2NetEngine:
    """Single-scale D2-Net on csrc/d2net.cu: host calls and batched device calls (descriptors left on the GPU for
    TwoWayEngine.match_batched_dev)."""

    def __init__(self, state_dict, device: int = 0, ctx: Optional[_lib.Context] = None):
        self.ctx = ctx or _lib.Context(device)
        blob = weights.pack_d2net(weights.load_d2net(state_dict))
        self.ctx.check(self.ctx.lib.b2_d2net_set_weights(self.ctx.handle, _lib.ptr(blob), blob.size), "d2net_set_weights")
        self.lock = threading.RLock()

    @staticmethod
    def check_image(img: np.ndarray) -> np.ndarray:
        img = np.ascontiguousarray(img)
        if img.dtype != np.uint8:
            raise ValueError("D2-Net takes uint8 images")
        if img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] not in (1, 3)):
            raise ValueError("D2-Net takes gray (H, W) / (H, W, 1) or RGB (H, W, 3) images")
        h, w = img.shape[:2]
        if max(h, w) > D2NET_MAX_EDGE_PX or h + w > D2NET_MAX_SUM_EDGES_PX:
            raise ValueError(f"image {h}x{w} is over D2-Net's size limits (longer edge 1600, edges summing to 2800): the reference "
                             "resizes such images with scipy.misc.imresize, which current scipy no longer has")
        if min(h, w) < 8:
            raise ValueError("D2-Net needs images of at least 8 x 8 pixels")
        return img

    def detect_and_describe(self, image: np.ndarray, max_keypoints: int = 5000):
        """Host uint8 image -> ((K, 2) float32 (x, y), (K,) float32 scores, (K, 512) float32 descriptors), score-ordered."""
        img = self.check_image(image)
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else img.shape[2]
        xy = np.empty((max_keypoints, 2), np.float32)
        sc = np.empty(max_keypoints, np.float32)
        desc = np.empty((max_keypoints, D2NET_DESC_DIM), np.float32)
        n, total = _lib.C.c_int(0), _lib.C.c_int(0)
        with self.lock:
            rc = self.ctx.lib.b2_d2net_detect_host(self.ctx.handle, _lib.ptr(img), h, w, ch, int(max_keypoints), _lib.ptr(xy), _lib.ptr(sc),
                                                   _lib.ptr(desc), _lib.C.byref(n), _lib.C.byref(total))
        self.ctx.check(rc, "d2net_detect_host")
        k = n.value
        return xy[:k].copy(), sc[:k].copy(), desc[:k].copy()

    def extract_many(self, images, max_keypoints: int = 5000):
        """images: same-shape CUDA uint8 tensors (H, W) / (H, W, 1) / (H, W, 3), rows may be pitched.  -> list of
        ((n, 2) xy, (n,) scores, (n, 512) descriptors) CUDA float32 tensors and the count before the top-k."""
        import torch

        if len(images) == 0:
            return []
        shape = tuple(images[0].shape)
        if any(tuple(x.shape) != shape for x in images):
            raise ValueError("extract_many takes images of one shape")
        h, w = shape[:2]
        ch = 1 if len(shape) == 2 else shape[2]
        self.check_image(np.empty((h, w, ch), np.uint8))  # the size limits, before any device work
        dev = images[0].device
        out = []
        with self.lock:
            for c0 in range(0, len(images), 64):
                idx = range(c0, min(len(images), c0 + 64))
                st = (_lib.D2NetImage * len(idx))()
                keep, pitch = [], None
                for s, i in enumerate(idx):
                    x = images[i]
                    if x.dtype != torch.uint8:
                        raise ValueError("images must be uint8")
                    if x.stride(-1) != 1 or (x.dim() == 3 and x.stride(1) != ch):
                        x = x.contiguous()
                    if pitch is None:
                        pitch = x.stride(0)
                    elif x.stride(0) != pitch:
                        x = x.contiguous()
                        if x.stride(0) != pitch:
                            raise ValueError("images of one call must share a row pitch")
                    xy = torch.empty((max_keypoints, 2), dtype=torch.float32, device=dev)
                    sc = torch.empty(max_keypoints, dtype=torch.float32, device=dev)
                    desc = torch.empty((max_keypoints, D2NET_DESC_DIM), dtype=torch.float32, device=dev)
                    keep.append((x, xy, sc, desc))
                    st[s] = _lib.D2NetImage(x.data_ptr(), int(max_keypoints), xy.data_ptr(), sc.data_ptr(), desc.data_ptr(), 0, 0)
                stream = torch.cuda.current_stream(dev).cuda_stream
                rc = self.ctx.lib.b2_d2net_detect_batched_dev(self.ctx.handle, st, len(idx), h, w, ch, int(pitch), _lib.C.c_void_p(stream))
                self.ctx.check(rc, "d2net_detect_batched_dev")
                for s, (_, xy, sc, desc) in enumerate(keep):
                    n = st[s].out_n
                    out.append((xy[:n], sc[:n], desc[:n], st[s].out_total))
        return out


class B200D2NetDetectorDescriptor(DetectorDescriptorBase):
    """Single-scale D2-Net on hand-written sm_90a kernels: the drop-in for gtsfm/.../d2net.py `D2NetDetDesc`.

    Same outputs: float32 (x, y) coordinates and responses (no scales), (K, 512) float32 descriptors, the max_keypoints best
    scores first.  Like the reference it ignores `image.mask` and runs single-scale only.  Images whose longer edge is over
    1600 pixels or whose edges sum to over 2800 raise ValueError: the reference resizes them with scipy.misc.imresize, which
    its pinned scipy no longer has, so it cannot process them either.  RGBA and non-uint8 input raise ValueError."""

    def __init__(self, max_keypoints: int = 5000, model_path: Union[Path, str, dict, None] = None, device: int = 0) -> None:
        super().__init__(max_keypoints=max_keypoints)
        model_path = default_d2net_model_path() if model_path is None else model_path
        if not isinstance(model_path, dict) and not Path(model_path).exists():
            raise FileNotFoundError(  # same failure as gtsfm/.../d2net.py:46-50
                f"D2-Net weights not found at {model_path}. Please run 'bash scripts/download_model_weights.sh' from the repo root.")
        self._model_path = model_path
        self._device = device
        self._engine: Optional[D2NetEngine] = None  # lazy, never pickled

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> D2NetEngine:
        if self._engine is None:
            self._engine = D2NetEngine(self._model_path, self._device)
        return self._engine

    def detect_and_describe(self, image: Image) -> Tuple[Keypoints, np.ndarray]:
        arr = D2NetEngine.check_image(image.value_array)
        xy, sc, desc = self._ensure_engine().detect_and_describe(arr, self.max_keypoints)
        return Keypoints(coordinates=xy, responses=sc), desc
