"""LightGlue / SuperGlue / two-way matcher plugins.

Drop-ins for gtsfm/frontend/matcher/lightglue_matcher.py:24-112 (`LightGlueMatcher`),
gtsfm/frontend/matcher/superglue_matcher.py:30-115 (`SuperGlueMatcher`) and gtsfm/frontend/matcher/twoway_matcher.py
(`TwoWayMatcher`): same `match(...)` signature, argument meaning, errors and output dtypes ((K, 2) int64 for LightGlue,
uint32 for SuperGlue, rows ascending in column 0; uint32 rows ordered by distance for the two-way matcher).
All arithmetic runs in libgtsfm_b200.so; lazily created device state keeps the objects picklable
(tests/frontend/matcher/test_matcher_base.py:102-107).
"""
from __future__ import annotations

from enum import Enum
from pathlib import Path
from typing import Optional, Tuple, Union

import numpy as np

from . import _lib, weights
from .gtsfm_api import Keypoints, MatcherBase

DESC_DIM = 256


class LightGlueEngine:
    def __init__(self, state_dict, device: int = 0, ctx: Optional[_lib.Context] = None, feature_cache: Optional[bool] = None):
        self.ctx = ctx or _lib.Context(device)
        if feature_cache is not None:
            self.ctx.set_option("feature_cache", 1 if feature_cache else 0)
        blob = weights.pack_lightglue(weights.load_state_dict(state_dict))
        self.ctx.check(self.ctx.lib.b2_lightglue_set_weights(self.ctx.handle, _lib.ptr(blob), blob.size), "lightglue_set_weights")
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def match(self, kp0, desc0, kp1, desc1, depth_confidence=0.95, width_confidence=0.99, filter_threshold=0.1,
              prune_min_kpts=-1, return_scores=False, fp16_attention=False):
        kp0 = np.ascontiguousarray(kp0, np.float32)
        kp1 = np.ascontiguousarray(kp1, np.float32)
        desc0 = np.ascontiguousarray(desc0, np.float32)
        desc1 = np.ascontiguousarray(desc1, np.float32)
        n0, n1 = len(kp0), len(kp1)
        cap = max(1, min(n0, n1))
        out = np.empty((cap, 2), np.int64)
        sc = np.empty(cap, np.float32)
        k, stop = _lib.C.c_int(0), _lib.C.c_int(0)
        prm = _lib.LightGlueParams(depth_confidence, width_confidence, filter_threshold, prune_min_kpts, 1 if fp16_attention else 0)
        sent0 = self.ctx.h2d_bytes()
        rc = self.ctx.lib.b2_lightglue_match_host(self.ctx.handle, _lib.ptr(kp0), _lib.ptr(desc0), n0, _lib.ptr(kp1),
                                                  _lib.ptr(desc1), n1, _lib.C.byref(prm), _lib.ptr(out), _lib.ptr(sc),
                                                  _lib.C.byref(k), _lib.C.byref(stop))
        self.ctx.check(rc, "lightglue_match")
        self.last_stop = stop.value
        self.h2d_bytes += self.ctx.h2d_bytes() - sent0  # feature arrays the library already holds are not re-sent
        self.d2h_bytes += k.value * (16 + 4) + 8
        if return_scores:
            return out[: k.value].copy(), sc[: k.value].copy()
        return out[: k.value].copy()

    def layer_trace(self):
        """The per-layer state the last match call recorded under set_option("lightglue_trace", 1): one dict per active side
        and layer, in the order recorded (include/gtsfm_b200.h, b2_lightglue_trace_get)."""
        lib, h = self.ctx.lib, self.ctx.handle
        recs = []
        for i in range(lib.b2_lightglue_trace_count(h)):
            meta = np.zeros(8, np.int32)
            self.ctx.check(lib.b2_lightglue_trace_get(h, i, _lib.ptr(meta), None, None, None, None, None), "lightglue_trace_get")
            pair, side, layer, n, heads, unconf, kept, stop = (int(v) for v in meta)
            x, ind = np.empty((n, DESC_DIM), np.float32), np.empty(n, np.int32)
            conf, mat = np.empty(n if heads else 0, np.float32), np.empty(n if heads else 0, np.float32)
            keep = np.empty(kept if heads else 0, np.int32)
            self.ctx.check(lib.b2_lightglue_trace_get(h, i, _lib.ptr(meta), _lib.ptr(x), _lib.ptr(ind), _lib.ptr(conf), _lib.ptr(mat),
                                                      _lib.ptr(keep)), "lightglue_trace_get")
            recs.append(dict(pair=pair, side=side, layer=layer, n=n, heads=bool(heads), unconf=unconf, kept=kept, stop=bool(stop), x=x,
                             ind=ind, conf=conf, mat=mat, keep=keep))
        return recs


class B200LightGlueMatcher(MatcherBase):
    """LightGlue on hand-written sm_90a kernels behind GTSfM's MatcherBase.

    `cpu_semantics=True` (default) reproduces what the reference computes on its CPU front-end (pruning attempted at
    every layer, lightglue.py:339-344) and is what the parity fixtures pin; False uses the reference's CUDA+flash
    pruning threshold of 1536 keypoints.

    `feature_cache=True` (opt-in, default off) lets the library keep device copies of the host feature arrays it is handed,
    keyed by (host address, size) and validated by a hash of the full contents: an image matched against many partners is
    uploaded once.  It only helps callers that pass the SAME numpy buffers repeatedly (a sequential in-process loop);
    under Dask every task unpickles fresh arrays and the default - copy on every call, like the reference - is what runs.
    """

    def __init__(self, features: str = "superpoint", use_cuda: bool = True, weights_path: Union[Path, str, dict, None] = None,
                 device: int = 0, cpu_semantics: bool = True, feature_cache: bool = False, fp16_attention: bool = False):
        super().__init__()
        if features != "superpoint":
            raise ValueError(f"Unsupported features: {features} (this build serves the SuperPoint LightGlue only)")
        if weights_path is None:
            raise FileNotFoundError("LightGlue weights_path is required (superpoint_lightglue_v0-1_arxiv.pth-style checkpoint)")
        if not isinstance(weights_path, dict) and not Path(weights_path).exists():
            raise FileNotFoundError(f"LightGlue weights not found at {weights_path}")
        self._use_cuda = use_cuda
        self._features = features
        self._weights = weights_path
        self._device = device
        self._cpu_semantics = cpu_semantics
        self._feature_cache = bool(feature_cache)
        self._fp16_attention = bool(fp16_attention)  # opt-in: the reference's CUDA numerics (fp16 flash SDPA), ~2x faster attention
        self._engine: Optional[LightGlueEngine] = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> LightGlueEngine:
        if self._engine is None:
            self._engine = LightGlueEngine(self._weights, self._device, feature_cache=self._feature_cache)
        return self._engine

    def match(self, keypoints_i1: Keypoints, keypoints_i2: Keypoints, descriptors_i1: np.ndarray, descriptors_i2: np.ndarray,
              im_shape_i1: Tuple[int, int, int], im_shape_i2: Tuple[int, int, int]) -> np.ndarray:
        if keypoints_i1.responses is None or keypoints_i2.responses is None:
            raise ValueError("Responses for keypoints required for LightGlue.")  # lightglue_matcher.py:78-79
        if len(keypoints_i1) == 0 or len(keypoints_i2) == 0:
            return np.zeros((0, 2), np.int64)
        if descriptors_i1.shape[1] != DESC_DIM or descriptors_i2.shape[1] != DESC_DIM:
            raise AssertionError("LightGlue(superpoint) expects 256-dimensional descriptors")  # lightglue.py:509-510
        eng = self._ensure_engine()
        return eng.match(keypoints_i1.coordinates, descriptors_i1, keypoints_i2.coordinates, descriptors_i2,
                         prune_min_kpts=-1 if self._cpu_semantics else 1536, fp16_attention=self._fp16_attention)


SUPERGLUE_DESC_DIM = 256
DEFAULT_NUM_SINKHORN_ITERATIONS = 20  # superglue_matcher.py:27
SUPERGLUE_MATCH_THRESHOLD = 0.2  # thirdparty/.../superglue.py:201


class SuperGlueEngine:
    def __init__(self, state_dict, device: int = 0, ctx: Optional[_lib.Context] = None):
        self.ctx = ctx or _lib.Context(device)
        blob = weights.pack_superglue(weights.load_state_dict(state_dict))
        self.ctx.check(self.ctx.lib.b2_superglue_set_weights(self.ctx.handle, _lib.ptr(blob), blob.size), "superglue_set_weights")
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def match(self, kp0, sc0, desc0, kp1, sc1, desc1, shape0, shape1, sinkhorn_iters=DEFAULT_NUM_SINKHORN_ITERATIONS,
              match_threshold=SUPERGLUE_MATCH_THRESHOLD, return_scores=False):
        arrs = [np.ascontiguousarray(a, np.float32) for a in (kp0, sc0, desc0, kp1, sc1, desc1)]
        n0, n1 = len(arrs[0]), len(arrs[3])
        cap = max(1, min(n0, n1))
        out = np.empty((cap, 2), np.uint32)
        sc = np.empty(cap, np.float32)
        k = _lib.C.c_int(0)
        rc = self.ctx.lib.b2_superglue_match_host(self.ctx.handle, _lib.ptr(arrs[0]), _lib.ptr(arrs[1]), _lib.ptr(arrs[2]), n0, int(shape0[0]),
                                                  int(shape0[1]), _lib.ptr(arrs[3]), _lib.ptr(arrs[4]), _lib.ptr(arrs[5]), n1, int(shape1[0]),
                                                  int(shape1[1]), int(sinkhorn_iters), float(match_threshold), _lib.ptr(out), _lib.ptr(sc),
                                                  _lib.C.byref(k))
        self.ctx.check(rc, "superglue_match")
        self.h2d_bytes += sum(a.nbytes for a in arrs)
        self.d2h_bytes += k.value * 12 + 4
        if return_scores:
            return out[: k.value].copy(), sc[: k.value].copy()
        return out[: k.value].copy()

    def layer_trace(self):
        """The arrays the last match call recorded under set_option("superglue_trace", 1), in the order recorded
        (include/gtsfm_b200.h, b2_superglue_trace_get): one dict per record with `kind` "x" (layer -1 .. 17), "md" or "Z"."""
        lib, h = self.ctx.lib, self.ctx.handle
        recs = []
        for i in range(lib.b2_superglue_trace_count(h)):
            meta = np.zeros(5, np.int32)
            self.ctx.check(lib.b2_superglue_trace_get(h, i, _lib.ptr(meta), None), "superglue_trace_get")
            layer, side, n, kind, cols = (int(v) for v in meta)
            v = np.empty((n, cols), np.float32)
            self.ctx.check(lib.b2_superglue_trace_get(h, i, _lib.ptr(meta), _lib.ptr(v)), "superglue_trace_get")
            recs.append(dict(layer=layer, side=side, n=n, kind=("x", "md", "Z")[kind], v=v))
        return recs


class B200SuperGlueMatcher(MatcherBase):
    """SuperGlue on hand-written sm_90a kernels behind GTSfM's MatcherBase (gtsfm/frontend/matcher/superglue_matcher.py:30-115)."""

    def __init__(self, use_cuda: bool = True, use_outdoor_model: bool = True, weights_path: Union[Path, str, dict, None] = None, device: int = 0):
        super().__init__()
        if weights_path is None:
            raise FileNotFoundError("SuperGlue weights_path is required (a superglue_outdoor.pth-style checkpoint)")
        if not isinstance(weights_path, dict) and not Path(weights_path).exists():
            raise FileNotFoundError(f"SuperGlue weights not found at {weights_path}")
        self._use_cuda = use_cuda
        self._config = {"descriptor_dim": SUPERGLUE_DESC_DIM, "weights": "outdoor" if use_outdoor_model else "indoor",
                        "sinkhorn_iterations": DEFAULT_NUM_SINKHORN_ITERATIONS}
        self._weights = weights_path
        self._device = device
        self._engine: Optional[SuperGlueEngine] = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> SuperGlueEngine:
        if self._engine is None:
            self._engine = SuperGlueEngine(self._weights, self._device)
        return self._engine

    def match(self, keypoints_i1: Keypoints, keypoints_i2: Keypoints, descriptors_i1: np.ndarray, descriptors_i2: np.ndarray,
              im_shape_i1: Tuple[int, int, int], im_shape_i2: Tuple[int, int, int]) -> np.ndarray:
        if keypoints_i1.responses is None or keypoints_i2.responses is None:
            raise ValueError("Responses for keypoints required for SuperGlue")  # superglue_matcher.py:78-79
        if len(keypoints_i1) == 0 or len(keypoints_i2) == 0:
            return np.zeros((0, 2), np.uint32)
        if descriptors_i1.shape[1] != SUPERGLUE_DESC_DIM or descriptors_i2.shape[1] != SUPERGLUE_DESC_DIM:
            raise Exception("Superglue pretrained network only works on 256 dimensional descriptors")  # :81-82
        eng = self._ensure_engine()
        return eng.match(keypoints_i1.coordinates, keypoints_i1.responses, descriptors_i1, keypoints_i2.coordinates,
                         keypoints_i2.responses, descriptors_i2, im_shape_i1, im_shape_i2, self._config["sinkhorn_iterations"])


class MatchingDistanceType(Enum):
    """gtsfm/frontend/matcher/twoway_matcher.py:17-21."""

    HAMMING = 1
    EUCLIDEAN = 2


class TwoWayEngine:
    """Mutual-nearest-neighbour matching on k_mnn_top2 (csrc/mnn.cu).  `ratio=None`: no ratio test."""

    def __init__(self, device: int = 0, ctx: Optional[_lib.Context] = None):
        self.ctx = ctx or _lib.Context(device)

    def _check(self, rc: int, what: str) -> None:
        if rc == _lib.MNN_ERR_RATIO:
            raise ValueError("the ratio test needs at least 2 descriptors per image (cv2 knnMatch(k=2) found one neighbour)")
        self.ctx.check(rc, what)

    def match(self, desc0: np.ndarray, desc1: np.ndarray, ratio: Optional[float] = None, return_dist: bool = False):
        """Host arrays (float32 or uint8, no NaN) -> (K, 2) int64 rows (i0, i1) ordered by (0 -> 1 distance, i0)."""
        dt = 1 if desc0.dtype == np.uint8 and desc1.dtype == np.uint8 else 0
        npd = np.uint8 if dt else np.float32
        d0, d1 = np.ascontiguousarray(desc0, npd), np.ascontiguousarray(desc1, npd)
        dim = d0.shape[1] if d0.ndim == 2 else d1.shape[1]
        n0, n1 = len(d0), len(d1)
        cap = max(1, min(n0, n1))
        out = np.empty((cap, 2), np.int64)
        dist = np.empty(cap, np.float32)
        k = _lib.C.c_int(0)
        rc = self.ctx.lib.b2_mnn_match_host(self.ctx.handle, _lib.ptr(d0), n0, _lib.ptr(d1), n1, int(dim), dt,
                                            -1.0 if ratio is None else float(ratio), _lib.ptr(out), _lib.ptr(dist), _lib.C.byref(k))
        self._check(rc, "mnn_match_host")
        if return_dist:
            return out[: k.value].copy(), dist[: k.value].copy()
        return out[: k.value].copy()

    def match_batched_dev(self, pairs, ratio: Optional[float] = None, return_dist: bool = False):
        """pairs: sequence of (desc0, desc1) CUDA tensors (float32 or uint8, [n][dim]).  -> list of device int64 (K, 2) tensors
        (and float32 distances), one library call per (dim, dtype) group of pairs."""
        import torch

        groups = {}
        for i, (a, b) in enumerate(pairs):
            dim = a.shape[1] if a.dim() == 2 else b.shape[1]
            dt = 1 if a.dtype == torch.uint8 and b.dtype == torch.uint8 else 0
            groups.setdefault((int(dim), dt), []).append(i)
        res = [None] * len(pairs)
        for (dim, dt), idx in groups.items():
            tdt = torch.uint8 if dt else torch.float32
            ins, outs, st = [], [], (_lib.MnnPair * len(idx))()
            for s, i in enumerate(idx):
                a, b = (x.to(tdt).reshape(-1, dim).contiguous() for x in pairs[i])
                cap = max(1, min(len(a), len(b)))
                m = torch.empty((cap, 2), dtype=torch.int64, device=a.device)
                d = torch.empty(cap, dtype=torch.float32, device=a.device)
                ins.append((a, b))
                outs.append((m, d))
                st[s] = _lib.MnnPair(a.data_ptr(), len(a), b.data_ptr(), len(b), m.data_ptr(), d.data_ptr(), 0)
            stream = torch.cuda.current_stream(ins[0][0].device).cuda_stream
            rc = self.ctx.lib.b2_mnn_match_batched_dev(self.ctx.handle, st, len(idx), dim, dt,
                                                       -1.0 if ratio is None else float(ratio), _lib.C.c_void_p(stream))
            self._check(rc, "mnn_match_batched_dev")
            for s, i in enumerate(idx):
                m, d = outs[s]
                kk = st[s].out_k
                res[i] = (m[:kk], d[:kk]) if return_dist else m[:kk]
        return res


class B200TwoWayMatcher(MatcherBase):
    """Drop-in for gtsfm/frontend/matcher/twoway_matcher.py (`TwoWayMatcher`): mutual nearest neighbours under cv2's L2
    distance with an optional ratio test, on hand-written sm_90a kernels.  Integer-valued descriptors of dimension <= 258
    (cv2 SIFT, ORB, BRISK) give cv2's indices, order and distances bit for bit; other float descriptors can differ from cv2
    on near-ties."""

    def __init__(self, distance_type: MatchingDistanceType = MatchingDistanceType.EUCLIDEAN, ratio_test_threshold: Optional[float] = None,
                 device: int = 0):
        super().__init__()
        if distance_type is not MatchingDistanceType.EUCLIDEAN:
            raise NotImplementedError("B200TwoWayMatcher implements the EUCLIDEAN distance only")
        self._distance_type = distance_type
        self._ratio_test_threshold = ratio_test_threshold
        self._device = device
        self._engine: Optional[TwoWayEngine] = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> TwoWayEngine:
        if self._engine is None:
            self._engine = TwoWayEngine(self._device)
        return self._engine

    def match(self, keypoints_i1: Keypoints, keypoints_i2: Keypoints, descriptors_i1: np.ndarray, descriptors_i2: np.ndarray,
              im_shape_i1: Tuple[int, int, int], im_shape_i2: Tuple[int, int, int]) -> np.ndarray:
        if descriptors_i1.size == 0 or descriptors_i2.size == 0:
            return np.array([])  # the reference's return value (twoway_matcher.py:72-73)
        v1 = np.nonzero(~np.isnan(descriptors_i1).any(axis=1))[0]
        v2 = np.nonzero(~np.isnan(descriptors_i2).any(axis=1))[0]
        if len(v1) == 0 or len(v2) == 0:
            return np.array([])
        m = self._ensure_engine().match(descriptors_i1[v1], descriptors_i2[v2], self._ratio_test_threshold)
        if len(m) == 0:
            return np.array([])
        return np.stack([v1[m[:, 0]], v2[m[:, 1]]], 1).astype(np.uint32)
