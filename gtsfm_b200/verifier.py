"""RANSAC verifier plugin.

Drop-in for gtsfm/frontend/verifier/ransac.py:51-111 (`Ransac`, an `OpencvVerifierBase`): same constructor, same
`verify(...) -> (Rot3 | None, Unit3 | None, (K', 2) rows of match_indices, inlier ratio)` contract, same guards and
failure tuple (gtsfm/frontend/verifier/opencv_verifier_base.py:70-79, verifier_base.py:60-64), same threshold
convention (thr_px / max(fx) on calibrated points for E, thr_px on pixels for F).  The arithmetic the reference
delegates to OpenCV runs in libgtsfm_b200.so (CUDA).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

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


def pinhole_cal(intrinsics) -> Optional[Tuple[float, float, float]]:
    """(f, u0, v0) when `intrinsics` is a distortion-free pinhole model with one focal length and no skew, which is what the
    device calibrates with (`k_rs_gather` computes the same (u - u0) / f in double as `normalize_coordinates`); else None."""
    k1 = intrinsics.k1() if hasattr(intrinsics, "k1") else 0.0
    k2 = intrinsics.k2() if hasattr(intrinsics, "k2") else 0.0
    if k1 != 0.0 or k2 != 0.0 or not hasattr(intrinsics, "px"):
        return None
    K = np.asarray(intrinsics.K(), np.float64)
    if K[0, 0] != K[1, 1] or K[0, 1] != 0.0 or not K[0, 0] > 0.0:
        return None
    return float(K[0, 0]), float(K[0, 2]), float(K[1, 2])


def ransac_problem(k: int, mode: int, threshold: float, max_iters: int, mask=None, kp1=None, kp2=None, matches=None, x1=None,
                   x2=None, cal1=(1.0, 0.0, 0.0), cal2=(1.0, 0.0, 0.0)) -> "_lib.RansacProblem":
    """One b2_ransac_problem.  Array arguments are device tensors or addresses; the caller keeps them alive over the call."""
    p = _lib.RansacProblem()
    p.kp1, p.kp2, p.matches, p.x1, p.x2, p.mask = (_lib.ptr(a) for a in (kp1, kp2, matches, x1, x2, mask))
    p.k, p.mode, p.max_iters, p.threshold = int(k), int(mode), int(min(max_iters, 2**31 - 1)), float(threshold)
    p.cal1[:], p.cal2[:] = [float(c) for c in cal1], [float(c) for c in cal2]
    return p


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

    def verify_batched_dev(self, problems: Sequence["_lib.RansacProblem"], confidence=RANSAC_SUCCESS_PROB, seed=DEFAULT_SEED,
                           stream=None):
        """b2_ransac_verify_batched_dev: every problem of the list in one call -> ctypes array of b2_ransac_result.
        `stream`: a raw CUDA stream handle (None / 0: the legacy default stream)."""
        n = len(problems)
        arr = (_lib.RansacProblem * max(n, 1))(*problems)
        res = (_lib.RansacResult * max(n, 1))()
        prm = _lib.RansacParams(0.0, confidence, 0, seed)
        rc = self.ctx.lib.b2_ransac_verify_batched_dev(self.ctx.handle, arr, n, _lib.C.byref(prm), res, _lib.C.c_void_p(stream or 0))
        self.ctx.check(rc, "ransac_verify_batched_dev")
        self.d2h_bytes += n * _lib.C.sizeof(_lib.RansacResult)
        return res

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

    def verify_many(self, items: Sequence[tuple]) -> List[Tuple[Optional[Rot3], Optional[Unit3], np.ndarray, float]]:
        """`verify` for a list of its argument tuples in ONE library call: `verify_many(items)[i]` is what
        `verify(*items[i])` returns (rows and ratio equal; the pose equal for E, and for F up to the rounding of
        E = K2^T F K1, which the device forms itself).  Keypoints and rows are uploaded once per distinct array and the
        device gathers and calibrates them; a pair whose intrinsics are not a plain pinhole model (distortion, two focal
        lengths) is normalised on the host as in `verify` (E) or verified on its own (F)."""
        out: list = [None] * len(items)
        live = []
        for i, (kp1, kp2, rows, _, _) in enumerate(items):
            n = rows.shape[0]
            if n < self._min_matches or (self._use_intrinsics_in_verification and n < 6):  # opencv_verifier_base.py:70-79
                out[i] = self._failure_result
            else:
                live.append(i)
        if not live:
            return out
        import torch

        eng = self._ensure_engine()
        dev = torch.device("cuda", self._device)
        uploaded = {}

        def up(a: np.ndarray, dtype):  # one device copy per distinct host array
            key = (id(a), dtype)
            if key not in uploaded:
                uploaded[key] = (a, torch.from_numpy(np.ascontiguousarray(a, dtype)).to(dev))
            return uploaded[key][1]

        mode = 0 if self._use_intrinsics_in_verification else 1
        batch, problems = [], []
        masks = torch.zeros(sum(items[i][2].shape[0] for i in live) + 1, dtype=torch.uint8, device=dev)
        off = 0
        for i in live:
            kp1, kp2, rows, intr1, intr2 = items[i]
            k = rows.shape[0]
            c1, c2 = pinhole_cal(intr1), pinhole_cal(intr2)
            xy1, xy2 = np.asarray(kp1.coordinates), np.asarray(kp2.coordinates)
            gather = xy1.dtype == np.float32 and xy2.dtype == np.float32 and c1 is not None and c2 is not None
            if mode == 1 and (c1 is None or c2 is None):
                out[i] = self.verify(*items[i])
                continue
            thr = self._estimation_threshold_px / max(intr1.K()[0, 0], intr2.K()[0, 0]) if mode == 0 else self._estimation_threshold_px
            args = dict(mask=masks[off:off + k], cal1=c1 or (1.0, 0.0, 0.0), cal2=c2 or (1.0, 0.0, 0.0))
            if gather:
                args.update(kp1=up(xy1, np.float32), kp2=up(xy2, np.float32), matches=up(rows, np.int64))
            else:
                idx1, idx2 = rows[:, 0].astype(np.int64), rows[:, 1].astype(np.int64)
                if mode == 0:
                    p1, p2 = normalize_coordinates(xy1[idx1], intr1), normalize_coordinates(xy2[idx2], intr2)
                else:
                    p1, p2 = xy1.astype(np.float64)[idx1], xy2.astype(np.float64)[idx2]
                args.update(x1=up(p1, np.float64), x2=up(p2, np.float64))
            problems.append(ransac_problem(k, mode, thr, E_MAX_ITERS if mode == 0 else F_MAX_ITERS, **args))
            batch.append((i, off))
            off += k
        res = eng.verify_batched_dev(problems, seed=self._seed, stream=torch.cuda.current_stream(dev).cuda_stream)
        masks_h = masks.cpu().numpy()
        for (i, o), r in zip(batch, res):
            if r.status != 0:
                out[i] = self._failure_result
                continue
            rows = items[i][2]
            mask = masks_h[o:o + rows.shape[0]]
            out[i] = (Rot3(np.array(r.R).reshape(3, 3)), Unit3(np.array(r.t)), rows[np.where(mask == 1)[0]], float(np.mean(mask)))
        return out


LMEDS_E_CONFIDENCE = 0.999  # cv2.findEssentialMat's default prob (lmeds.py:36-41 passes none)
LMEDS_F_CONFIDENCE = 0.99  # cv2.findFundamentalMat's default confidence (lmeds.py:58-62)
LMEDS_MAX_ITERS = 1000  # cv2's default maxIters for both


def lmeds_params(e_confidence: float = LMEDS_E_CONFIDENCE, f_confidence: float = LMEDS_F_CONFIDENCE) -> "_lib.LmedsParams":
    prm = _lib.LmedsParams()
    prm.confidence[:] = [float(e_confidence), float(f_confidence)]
    return prm


def lmeds_verify_batched_dev(ctx: "_lib.Context", problems: Sequence["_lib.RansacProblem"], params=None, stream=None):
    """b2_lmeds_verify_batched_dev: every problem of the list in one call -> ctypes array of b2_ransac_result.
    `stream`: a raw CUDA stream handle (None / 0: the legacy default stream)."""
    n = len(problems)
    arr = (_lib.RansacProblem * max(n, 1))(*problems)
    res = (_lib.RansacResult * max(n, 1))()
    prm = params if params is not None else lmeds_params()
    rc = ctx.lib.b2_lmeds_verify_batched_dev(ctx.handle, arr, n, _lib.C.byref(prm), res, _lib.C.c_void_p(stream or 0))
    ctx.check(rc, "lmeds_verify_batched_dev")
    return res


class B200LMEDS(VerifierBase):
    """cv2's LMeDS (gtsfm/frontend/verifier/lmeds.py, `LMEDS`) on sm_90a kernels behind GTSfM's VerifierBase.

    Same constructor as the reference; `estimation_threshold_px` is accepted and not used, as there: the inlier threshold
    comes from the best model's median error.  E (5-point) on calibrated points with cv2's defaults (prob 0.999, 1000
    iterations), or F (7-point) on pixels (confidence 0.99); the inlier mask is cv2's bit for bit on the scenes
    tests/test_lmeds_cpu.py checks, and the pose is recovered on the device as for `B200Ransac`."""

    def __init__(self, use_intrinsics_in_verification: bool, estimation_threshold_px: float, device: int = 0) -> None:
        super().__init__(use_intrinsics_in_verification, estimation_threshold_px)
        self._device = device
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
        return self.verify_many([(keypoints_i1, keypoints_i2, match_indices, camera_intrinsics_i1, camera_intrinsics_i2)])[0]

    def verify_many(self, items: Sequence[tuple]) -> List[Tuple[Optional[Rot3], Optional[Unit3], np.ndarray, float]]:
        """`verify` for a list of its argument tuples in ONE library call.  Keypoints and rows are uploaded once per
        distinct array and the device gathers and calibrates them; a pair whose intrinsics are not a plain pinhole model
        is normalised on the host (E), or has its pose recovered from E = K2^T F K1 on the host (F)."""
        out: list = [None] * len(items)
        live = []
        for i, (kp1, kp2, rows, _, _) in enumerate(items):
            n = rows.shape[0]
            if n < self._min_matches or (self._use_intrinsics_in_verification and n < 6):  # opencv_verifier_base.py:70-79
                out[i] = self._failure_result
            else:
                live.append(i)
        if not live:
            return out
        import torch

        eng = self._ensure_engine()
        dev = torch.device("cuda", self._device)
        uploaded = {}

        def up(a: np.ndarray, dtype):  # one device copy per distinct host array
            key = (id(a), dtype)
            if key not in uploaded:
                uploaded[key] = (a, torch.from_numpy(np.ascontiguousarray(a, dtype)).to(dev))
            return uploaded[key][1]

        mode = 0 if self._use_intrinsics_in_verification else 1
        batch, problems = [], []
        masks = torch.zeros(sum(items[i][2].shape[0] for i in live) + 1, dtype=torch.uint8, device=dev)
        off = 0
        for i in live:
            kp1, kp2, rows, intr1, intr2 = items[i]
            k = rows.shape[0]
            c1, c2 = pinhole_cal(intr1), pinhole_cal(intr2)
            xy1, xy2 = np.asarray(kp1.coordinates), np.asarray(kp2.coordinates)
            pinhole = c1 is not None and c2 is not None
            gather = xy1.dtype == np.float32 and xy2.dtype == np.float32 and pinhole
            args = dict(mask=masks[off:off + k], cal1=c1 or (1.0, 0.0, 0.0), cal2=c2 or (1.0, 0.0, 0.0))
            if gather:
                args.update(kp1=up(xy1, np.float32), kp2=up(xy2, np.float32), matches=up(rows, np.int64))
            else:
                idx1, idx2 = rows[:, 0].astype(np.int64), rows[:, 1].astype(np.int64)
                if mode == 0:
                    p1, p2 = normalize_coordinates(xy1[idx1], intr1), normalize_coordinates(xy2[idx2], intr2)
                else:
                    p1, p2 = xy1.astype(np.float64)[idx1], xy2.astype(np.float64)[idx2]
                args.update(x1=up(p1, np.float64), x2=up(p2, np.float64))
            problems.append(ransac_problem(k, mode, 0.0, LMEDS_MAX_ITERS, **args))
            batch.append((i, off, pinhole))
            off += k
        res = lmeds_verify_batched_dev(eng.ctx, problems, stream=torch.cuda.current_stream(dev).cuda_stream)
        masks_h = masks.cpu().numpy()
        for (i, o, pinhole), r in zip(batch, res):
            if r.status != 0:
                out[i] = self._failure_result
                continue
            kp1, kp2, rows, intr1, intr2 = items[i]
            mask = masks_h[o:o + rows.shape[0]]
            inl = np.where(mask == 1)[0]
            R, t = np.array(r.R).reshape(3, 3), np.array(r.t)
            if mode == 1 and not pinhole:  # utils/verification.py:99-112 with the full K, pose on the host-normalised inliers
                E = intr2.K().T @ np.array(r.model).reshape(3, 3) @ intr1.K()
                n1 = normalize_coordinates(np.asarray(kp1.coordinates, np.float64)[rows[inl, 0]], intr1)
                n2 = normalize_coordinates(np.asarray(kp2.coordinates, np.float64)[rows[inl, 1]], intr2)
                R, t, _ = eng.recover_pose(E, n1, n2)
            out[i] = (Rot3(R), Unit3(t), rows[inl], float(np.mean(mask)))
        return out
