"""TEST INFRASTRUCTURE — fp64 NumPy restatement of cv2's LMeDS estimator (never shipped).

What the reference's ``LMEDS`` verifier (gtsfm/frontend/verifier/lmeds.py, config verifier/lmeds_5pt.yaml) delegates to
``cv2.findEssentialMat(..., method=cv2.LMEDS)`` / ``cv2.findFundamentalMat(..., cv2.FM_LMEDS)``: OpenCV's
``LMeDSPointSetRegistrator::run``.  OpenCV's source is not part of this repository; every rule below is pinned against
cv2 itself (4.13.0 here) by tests/test_lmeds_cpu.py, and each carries the cv2 behaviour it was checked against.

* RNG: cv::RNG multiply-with-carry, ``state = (state & 0xffffffff) * 4164903690 + (state >> 32)``, ``next()`` = low 32
  bits, seeded with 2^64 - 1 once per call; ``uniform(0, n) = next() % n``.
* Subsets: m = 5 (E) / 7 (F) indices drawn in order, an index repeating an earlier one is drawn again.  F (points cast
  to float32 first) rejects a subset whose last point is collinear with two earlier ones in either image (FLT_EPSILON
  test) and draws a new one, at most 1000 attempts; running out stops the sampling (on the first subset: no model).
* Iterations: ``max(3, RANSACUpdateNumIters(confidence, 0.45, m, maxIters))``, no early stop: 134 for E at 0.999,
  300 for F at 0.99 (maxIters 1000).
* Models: every real root of the 5-point problem on the double points (E), the 7-point solver with F33 = 1 (F); the
  minimal solvers are the host build of gtsfm_b200/csrc/ransac_math.cuh (``build_shim``), which is what the device runs.
* Errors: squared Sampson (E) / max of the two squared epipolar-line distances (F) in double, cast to float32.
* Median: the ``count // 2``-th smallest float error, ordered by bit pattern as int32.  A model replaces the best
  only if its median is strictly lower, in visiting order (subset, then solution).
* Mask: ``sigma = max(0.001, 2.5 * 1.4826 * (1 + 5 / (count - m)) * sqrt(minMedian))``; inliers ``err <= float32(sigma^2)``.
  E returns the best model whatever the inlier count; F fails below m inliers.
"""
from __future__ import annotations

import ctypes
import shutil
import subprocess
from pathlib import Path
from typing import Callable, Optional

import numpy as np

MAX_SOL = 10  # solution slots per subset (the device's layout)
E_CONFIDENCE, F_CONFIDENCE = 0.999, 0.99  # cv2.findEssentialMat prob / findFundamentalMat confidence defaults
MAX_ITERS = 1000


def build_shim(out_dir: Path) -> ctypes.CDLL:
    """g++ build of tests/cpp/lmeds_shim.cpp (-DB2_FIVEPT_QR: the 5-point variant libgtsfm_b200.so compiles)."""
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    so = Path(out_dir) / "lmeds_shim.so"
    src = Path(__file__).resolve().parent.parent / "tests" / "cpp" / "lmeds_shim.cpp"
    subprocess.run([cxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-DB2_FIVEPT_QR", str(src), "-o", str(so)], check=True)
    lib = ctypes.CDLL(str(so))
    vp, i, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.lm_solve.argtypes = [i, vp, vp, vp]
    lib.lm_solve.restype = i
    lib.lm_fivept_sampled.argtypes = [vp, vp, vp]
    lib.lm_fivept_sampled.restype = i
    lib.lm_fivept_poly.argtypes = [vp, vp, vp]
    lib.lm_fivept_poly.restype = i
    lib.lm_poly_roots.argtypes = [vp, i, vp]
    lib.lm_poly_roots.restype = i
    lib.lm_subsets.argtypes = [vp, vp, i, i, i, vp]
    lib.lm_subsets.restype = i
    lib.lm_niters.argtypes = [d, i, i]
    lib.lm_niters.restype = i
    lib.lm_errors.argtypes = [i, vp, vp, vp, i, vp]
    return lib


def _p(a: np.ndarray):
    return ctypes.c_void_p(a.ctypes.data)


def shim_solver(lib) -> Callable[[int, np.ndarray, np.ndarray], np.ndarray]:
    """-> solve(mode, a (m,2), b (m,2)) -> (n, 9) models, through the shim."""
    def solve(mode, a, b):
        out = np.zeros((MAX_SOL, 9))
        n = lib.lm_solve(mode, _p(np.ascontiguousarray(a, np.float64)), _p(np.ascontiguousarray(b, np.float64)), _p(out))
        return out[:n]
    return solve


# ---- sampler ------------------------------------------------------------------------------------------------------

class CvRNG:
    """cv::RNG: 64-bit multiply-with-carry."""

    def __init__(self, state: int = 2**64 - 1):
        self.state = state

    def next(self) -> int:
        self.state = ((self.state & 0xFFFFFFFF) * 4164903690 + (self.state >> 32)) & 0xFFFFFFFFFFFFFFFF
        return self.state & 0xFFFFFFFF

    def uniform(self, n: int) -> int:
        return self.next() % n


def collinear_last(p: np.ndarray) -> bool:
    """cv2's haveCollinearPoints on float32 points (m, 2): the last point against every pair of earlier ones."""
    p = np.asarray(p, np.float32)
    i = len(p) - 1
    eps = float(np.finfo(np.float32).eps)
    for j in range(i):
        dx1, dy1 = float(p[j, 0] - p[i, 0]), float(p[j, 1] - p[i, 1])  # float32 differences, as cv2's Point2f
        for k in range(j):
            dx2, dy2 = float(p[k, 0] - p[i, 0]), float(p[k, 1] - p[i, 1])
            if abs(dx2 * dy1 - dy2 * dx1) <= eps * (abs(dx1) + abs(dy1) + abs(dx2) + abs(dy2)):
                return True
    return False


def subsets(x1: np.ndarray, x2: np.ndarray, mode: int, niters: int) -> np.ndarray:
    """(n_drawn, m) index table; n_drawn < niters when a subset ran out of its 1000 attempts (F)."""
    k, m = len(x1), (5 if mode == 0 else 7)
    rng = CvRNG()
    out = []
    for _ in range(niters):
        for _attempt in range(1000):
            s: list = []
            while len(s) < m:
                v = rng.uniform(k)
                if v not in s:
                    s.append(v)
            if mode == 0 or not (collinear_last(x1[s]) or collinear_last(x2[s])):
                break
        else:
            break
        out.append(s)
    return np.array(out, np.int32).reshape(-1, m)


def niters(confidence: float, m: int, max_iters: int = MAX_ITERS) -> int:
    """max(3, cv2's RANSACUpdateNumIters(confidence, 0.45, m, max_iters))."""
    num = np.log(max(1.0 - confidence, np.finfo(float).tiny))
    denom = 1.0 - (1.0 - 0.45) ** m
    if denom < np.finfo(float).tiny:
        n = 0
    else:
        ld = np.log(denom)
        n = max_iters if (ld >= 0 or -num >= max_iters * (-ld)) else int(np.floor(num / ld + 0.5))
    return max(n, 3)


# ---- errors and the median -----------------------------------------------------------------------------------------

def errors(mode: int, M: np.ndarray, x1: np.ndarray, x2: np.ndarray) -> np.ndarray:
    """cv2's computeError as float32, with its operation order (each product and sum rounded once)."""
    E = np.asarray(M, np.float64).ravel()
    a1, b1, a2, b2 = x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1]
    with np.errstate(divide="ignore", invalid="ignore"):
        if mode == 0:
            e0 = E[0] * a1 + E[1] * b1 + E[2]
            e1 = E[3] * a1 + E[4] * b1 + E[5]
            e2 = E[6] * a1 + E[7] * b1 + E[8]
            t0 = E[0] * a2 + E[3] * b2 + E[6]
            t1 = E[1] * a2 + E[4] * b2 + E[7]
            r = a2 * e0 + b2 * e1 + e2
            return (r * r / (e0 * e0 + e1 * e1 + t0 * t0 + t1 * t1)).astype(np.float32)
        a = E[0] * a1 + E[1] * b1 + E[2]
        b = E[3] * a1 + E[4] * b1 + E[5]
        c = E[6] * a1 + E[7] * b1 + E[8]
        s2 = 1.0 / (a * a + b * b)
        d2 = a2 * a + b2 * b + c
        a = E[0] * a2 + E[3] * b2 + E[6]
        b = E[1] * a2 + E[4] * b2 + E[7]
        c = E[2] * a2 + E[5] * b2 + E[8]
        s1 = 1.0 / (a * a + b * b)
        d1 = a1 * a + b1 * b + c
        u, v = d1 * d1 * s1, d2 * d2 * s2
        return np.where(u < v, v, u).astype(np.float32)


def median(err: np.ndarray) -> np.float32:
    """The len // 2-th smallest float32 error, ordered as int32 bit patterns (cv2's nth_element on int*)."""
    bits = np.ascontiguousarray(err, np.float32).view(np.int32)
    return np.partition(bits, len(bits) // 2)[len(bits) // 2:len(bits) // 2 + 1].view(np.float32)[0]


def sigma(min_median: float, count: int, m: int) -> float:
    return max(2.5 * 1.4826 * (1 + 5.0 / (count - m)) * np.sqrt(min_median), 0.001)


# ---- the estimator -------------------------------------------------------------------------------------------------

def lmeds(x1: np.ndarray, x2: np.ndarray, mode: int, solve: Callable, confidence: Optional[float] = None,
          max_iters: int = MAX_ITERS) -> dict:
    """LMeDSPointSetRegistrator::run for count > m.  x1 / x2: (k, 2) double, calibrated (E) or pixels (F; cast to float32
    here).  -> dict with the index table, per-slot solution counts / models / medians (NaN: empty slot), the chosen slot,
    the minimum median, sigma, the threshold, the mask, its count, the model and ``ok``."""
    m = 5 if mode == 0 else 7
    if confidence is None:
        confidence = E_CONFIDENCE if mode == 0 else F_CONFIDENCE
    x1 = np.asarray(x1, np.float64)
    x2 = np.asarray(x2, np.float64)
    if mode == 1:
        x1, x2 = x1.astype(np.float32).astype(np.float64), x2.astype(np.float32).astype(np.float64)
    k = len(x1)
    out = dict(ok=False, model=None, mask=np.zeros(k, np.uint8), count=0, slot=-1, min_median=None, sigma=None, thr=None)
    if k <= m:
        raise ValueError("lmeds: count must exceed the minimal sample (cv2's count <= m branches are not restated)")
    n_it = niters(confidence, m, max_iters)
    idx = subsets(x1, x2, mode, n_it)
    nsol = np.zeros(len(idx), np.int32)
    models = np.zeros((len(idx), MAX_SOL, 9))
    med = np.full((len(idx), MAX_SOL), np.nan, np.float32)
    best, best_med = -1, np.inf
    for s, sub in enumerate(idx):
        sols = solve(mode, x1[sub], x2[sub])
        nsol[s] = len(sols)
        for j, M in enumerate(sols):
            models[s, j] = M
            med[s, j] = median(errors(mode, M, x1, x2))
            if float(med[s, j]) < best_med:  # strict: earlier slots win ties; NaN and inf are never taken
                best, best_med = s * MAX_SOL + j, float(med[s, j])
    out.update(idx=idx, n_drawn=len(idx), niters=n_it, nsol=nsol, models=models, medians=med)
    if best < 0:
        return out
    M = models[best // MAX_SOL, best % MAX_SOL]
    sg = sigma(best_med, k, m)
    thr = np.float32(sg * sg)
    err = errors(mode, M, x1, x2)
    mask = (err <= thr).astype(np.uint8)
    cnt = int(mask.sum())
    out.update(slot=best, min_median=best_med, sigma=sg, thr=thr, mask=mask, count=cnt, model=M.reshape(3, 3),
               ok=(mode == 0 or cnt >= m))
    return out


# ---- cv2 itself, driven as the reference drives it -------------------------------------------------------------------

def cv2_lmeds(x1: np.ndarray, x2: np.ndarray, mode: int):
    """-> (model (3, 3) | None, mask (k,) uint8) from cv2, as gtsfm/frontend/verifier/lmeds.py calls it."""
    import cv2

    if mode == 0:
        M, mask = cv2.findEssentialMat(np.asarray(x1, np.float64), np.asarray(x2, np.float64), np.eye(3), method=cv2.LMEDS)
    else:
        M, mask = cv2.findFundamentalMat(np.asarray(x1, np.float64), np.asarray(x2, np.float64), method=cv2.FM_LMEDS)
    mask = np.zeros(len(x1), np.uint8) if mask is None else mask.ravel().astype(np.uint8)
    if M is None or M.shape != (3, 3):
        return None, mask
    return M, mask


def probe_scene(seed: int, k: int, outlier_frac: float = 0.5):
    """Calibrated two-view scene: points ~ N(0, 1) + (0, 0, 6), R = Rodrigues(N(0, 0.1^2)), t = (1, 0.1, 0.05), outliers
    N(0, 0.5^2) on x2, then 1e-3 noise on x1 and on x2.  -> (x1, x2) (k, 2) normalised coordinates."""
    import cv2

    rng = np.random.default_rng(seed)
    X = rng.normal(size=(k, 3)) + [0, 0, 6]
    R = cv2.Rodrigues(rng.normal(size=3) * 0.1)[0]
    t = np.array([1.0, 0.1, 0.05])
    x1 = X[:, :2] / X[:, 2:]
    Y = X @ R.T + t
    x2 = Y[:, :2] / Y[:, 2:]
    n_out = int(round(k * outlier_frac))
    x2[:n_out] = rng.normal(size=(n_out, 2)) * 0.5
    x1 = x1 + rng.normal(size=x1.shape) * 1e-3
    x2 = x2 + rng.normal(size=x2.shape) * 1e-3
    return x1, x2
