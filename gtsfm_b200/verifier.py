"""RANSAC verifier plugin.

Drop-in for gtsfm/frontend/verifier/ransac.py:51-111 (`Ransac`, an `OpencvVerifierBase`): same constructor, same
`verify(...) -> (Rot3 | None, Unit3 | None, (K', 2) rows of match_indices, inlier ratio)` contract, same guards and
failure tuple (gtsfm/frontend/verifier/opencv_verifier_base.py:70-79, verifier_base.py:60-64), same threshold
convention (thr_px / max(fx) on calibrated points for E, thr_px on pixels for F).  The arithmetic the reference
delegates to OpenCV runs in libgtsfm_b200.so (CUDA).
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

from . import _lib
from .gtsfm_api import Keypoints, Rot3, Unit3, VerifierBase

RANSAC_SUCCESS_PROB = 0.999999  # ransac.py:22
E_MAX_ITERS = 1000  # cv2.findEssentialMat default maxIters (ransac.py:74-81 does not pass one)
F_MAX_ITERS = 1000000  # ransac.py:23 (the library caps the hypothesis budget, adaptive termination applies)
DEFAULT_SEED = 0x5EED


def normalize_coordinates(coordinates: np.ndarray, intrinsics) -> np.ndarray:
    """gtsfm/utils/features.py:41-51 without the per-point Python loop when the model is distortion-free."""
    k1 = intrinsics.k1() if hasattr(intrinsics, "k1") else 0.0
    k2 = intrinsics.k2() if hasattr(intrinsics, "k2") else 0.0
    c = np.asarray(coordinates, np.float64)
    if len(c) == 0:
        return np.zeros((0, 2))
    if k1 == 0.0 and k2 == 0.0 and hasattr(intrinsics, "px"):
        K = intrinsics.K()
        return np.stack([(c[:, 0] - K[0, 2]) / K[0, 0], (c[:, 1] - K[1, 2]) / K[1, 1]], -1)
    return np.vstack([intrinsics.calibrate(x[:2].reshape(2, 1)).ravel() for x in c])


class RansacEngine:
    def __init__(self, device: int = 0, ctx: Optional[_lib.Context] = None):
        self.ctx = ctx or _lib.Context(device)
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def essential(self, x1, x2, threshold, confidence=RANSAC_SUCCESS_PROB, max_iters=E_MAX_ITERS, seed=DEFAULT_SEED):
        x1 = np.ascontiguousarray(x1, np.float64)
        x2 = np.ascontiguousarray(x2, np.float64)
        k = len(x1)
        E, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
        mask = np.zeros(max(k, 1), np.uint8)
        n = _lib.C.c_int(0)
        prm = _lib.RansacParams(threshold, confidence, max_iters, seed)
        rc = self.ctx.lib.b2_ransac_essential_host(self.ctx.handle, _lib.ptr(x1), _lib.ptr(x2), k, _lib.C.byref(prm), _lib.ptr(E),
                                                   _lib.ptr(mask), _lib.C.byref(n), _lib.ptr(R), _lib.ptr(t))
        self.ctx.check(rc, "ransac_essential")
        self.h2d_bytes += x1.nbytes + x2.nbytes
        self.d2h_bytes += k + 8 * 21 + 4
        if rc == 1:
            return None, mask[:k], None, None
        return E.reshape(3, 3), mask[:k], R.reshape(3, 3), t

    def fundamental(self, x1, x2, threshold, confidence=RANSAC_SUCCESS_PROB, max_iters=F_MAX_ITERS, seed=DEFAULT_SEED):
        x1 = np.ascontiguousarray(x1, np.float64)
        x2 = np.ascontiguousarray(x2, np.float64)
        k = len(x1)
        F = np.zeros(9)
        mask = np.zeros(max(k, 1), np.uint8)
        n = _lib.C.c_int(0)
        prm = _lib.RansacParams(threshold, confidence, min(max_iters, 2**31 - 1), seed)
        rc = self.ctx.lib.b2_ransac_fundamental_host(self.ctx.handle, _lib.ptr(x1), _lib.ptr(x2), k, _lib.C.byref(prm), _lib.ptr(F),
                                                     _lib.ptr(mask), _lib.C.byref(n))
        self.ctx.check(rc, "ransac_fundamental")
        self.h2d_bytes += x1.nbytes + x2.nbytes
        self.d2h_bytes += k + 8 * 9 + 4
        if rc == 1:
            return None, mask[:k]
        return F.reshape(3, 3), mask[:k]

    def recover_pose(self, E, x1, x2):
        E = np.ascontiguousarray(E, np.float64)
        x1 = np.ascontiguousarray(x1, np.float64)
        x2 = np.ascontiguousarray(x2, np.float64)
        R, t = np.zeros(9), np.zeros(3)
        good = _lib.C.c_int(0)
        rc = self.ctx.lib.b2_recover_pose_host(self.ctx.handle, _lib.ptr(E), _lib.ptr(x1), _lib.ptr(x2), len(x1), _lib.ptr(R), _lib.ptr(t),
                                               _lib.C.byref(good))
        self.ctx.check(rc, "recover_pose")
        return R.reshape(3, 3), t, good.value


class B200Ransac(VerifierBase):
    """5-point / 8-point RANSAC on sm_90a kernels behind GTSfM's VerifierBase."""

    def __init__(self, use_intrinsics_in_verification: bool, estimation_threshold_px: float, device: int = 0, seed: int = DEFAULT_SEED) -> None:
        super().__init__(use_intrinsics_in_verification, estimation_threshold_px)
        self._device = device
        self._seed = seed
        self._engine: Optional[RansacEngine] = None

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_engine"] = None
        return st

    def _ensure_engine(self) -> RansacEngine:
        if self._engine is None:
            self._engine = RansacEngine(self._device)
        return self._engine

    def verify(self, keypoints_i1: Keypoints, keypoints_i2: Keypoints, match_indices: np.ndarray, camera_intrinsics_i1,
               camera_intrinsics_i2) -> Tuple[Optional[Rot3], Optional[Unit3], np.ndarray, float]:
        if match_indices.shape[0] < self._min_matches:  # opencv_verifier_base.py:70-71
            return self._failure_result
        eng = self._ensure_engine()
        idx1 = match_indices[:, 0].astype(np.int64)
        idx2 = match_indices[:, 1].astype(np.int64)
        if self._use_intrinsics_in_verification:
            if match_indices.shape[0] < 6:  # opencv_verifier_base.py:77-79
                return self._failure_result
            n1 = normalize_coordinates(np.asarray(keypoints_i1.coordinates)[idx1], camera_intrinsics_i1)
            n2 = normalize_coordinates(np.asarray(keypoints_i2.coordinates)[idx2], camera_intrinsics_i2)
            fx = max(camera_intrinsics_i1.K()[0, 0], camera_intrinsics_i2.K()[0, 0])
            E, mask, R, t = eng.essential(n1, n2, self._estimation_threshold_px / fx, seed=self._seed)
            if E is None:
                return self._failure_result
        else:
            p1 = np.asarray(keypoints_i1.coordinates, np.float64)[idx1]
            p2 = np.asarray(keypoints_i2.coordinates, np.float64)[idx2]
            F, mask = eng.fundamental(p1, p2, self._estimation_threshold_px, seed=self._seed)
            if F is None:
                return self._failure_result
            E = camera_intrinsics_i2.K().T @ F @ camera_intrinsics_i1.K()  # utils/verification.py:99-112
            inl = mask.ravel() == 1
            n1 = normalize_coordinates(p1[inl], camera_intrinsics_i1)
            n2 = normalize_coordinates(p2[inl], camera_intrinsics_i2)
            R, t, _ = eng.recover_pose(E, n1, n2)
        inlier_idxs = np.where(mask.ravel() == 1)[0]
        v_corr_idxs = match_indices[inlier_idxs]
        inlier_ratio_est_model = float(np.mean(mask))
        return Rot3(R), Unit3(t), v_corr_idxs, inlier_ratio_est_model
