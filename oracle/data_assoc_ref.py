"""fp64 NumPy restatement of data association's triangulation (gtsfm/data_association/data_assoc.py:205-273,
point3d_initializer.py:139-295, utils/reprojection.py, utils/tracks.py:83-103) for the two modes the configs use,
NO_RANSAC and RANSAC_SAMPLE_UNIFORM, and Cal3Bundler cameras without distortion.

gtsam.triangulatePoint3(cameras, measurements, rank_tol=1e-9, optimize=True) is twoview_ba_ref's DLT and point LM over n
views: the DLT takes the right singular vector of the full 2n x 4 system, the LM sums the n views' residuals, and the call
fails (RuntimeError in the reference) when the DLT rank is below 3, the point is at infinity, or it lies behind a camera
after refinement.  As for the two-view path, these are gtsam's documented defaults, not a live gtsam run.

RANSAC_SAMPLE_UNIFORM draws min(num_hypotheses, C(n, 2)) pairs without replacement.  Where that is every pair the result
does not depend on the draw order (up to exact ties, which go to the lower pair index); otherwise the draw is the keyed
permutation of csrc/data_assoc_math.cuh, restated here in uint64 (`sample_pairs`).
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle import twoview_ba_ref as tv

SUCCESS, CHEIRALITY_FAILURE, INLIERS_UNDERCONSTRAINED, POSES_UNDERCONSTRAINED, EXCEEDS_REPROJ_THRESH, LOW_TRIANGULATION_ANGLE = range(6)
NO_RANSAC, SAMPLE_UNIFORM = "NO_RANSAC", "RANSAC_SAMPLE_UNIFORM"
MAX_TRACK_REPROJ_ERROR = float(np.finfo(np.float32).max)
NUM_SAMPLES_PER_RANSAC_HYPOTHESIS = 2

_M64 = (1 << 64) - 1


def num_ransac_hypotheses(min_inlier_ratio=0.1, confidence=0.9999, dyn_num_hypotheses_multiplier=3.0, min_num_hypotheses=0,
                          max_num_hypotheses=2 ** 63 - 1) -> int:
    """TriangulationOptions.num_ransac_hypotheses()."""
    dyn = int((np.log(1 - confidence) / np.log(1 - min_inlier_ratio ** NUM_SAMPLES_PER_RANSAC_HYPOTHESIS)) * dyn_num_hypotheses_multiplier)
    return max(min(max_num_hypotheses, dyn), min_num_hypotheses)


# ---- the sampler (data_assoc_math.cuh), uint64 arithmetic ---------------------------------------------------------------
def mix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xbf58476d1ce4e5b9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94d049bb133111eb)
        x = x ^ (x >> np.uint64(31))
    return x


def sampler_key(seed: int, track: int) -> np.uint64:
    with np.errstate(over="ignore"):
        return mix64(np.uint64(seed & _M64) ^ mix64(np.uint64(track) + np.uint64(0x9e3779b97f4a7c15)))


def sample_pairs(seed: int, track: int, pairs: int, hyps: int) -> np.ndarray:
    """Pair index of every hypothesis h < hyps of the track at input position `track` with `pairs` = C(n, 2) pairs."""
    h = np.arange(hyps, dtype=np.uint64)
    if hyps >= pairs:
        return h.astype(np.int64)
    bits = 1
    while (1 << bits) < pairs:
        bits += 1
    half = np.uint64((bits + 1) // 2)
    mask = np.uint64((1 << int(half)) - 1)
    key = sampler_key(seed, track)
    x = h.copy()
    todo = np.ones(len(x), bool)
    while todo.any():
        L, R = x[todo] >> half, x[todo] & mask
        with np.errstate(over="ignore"):
            for r in range(4):
                F = mix64(key ^ (np.uint64(r) * np.uint64(0xd6e8feb86659fd93)) ^ R) & mask
                L, R = R, L ^ F
        x[todo] = (L << half) | R
        todo = x >= np.uint64(pairs)
    return x.astype(np.int64)


def pair_of(p: int, n: int) -> Tuple[int, int]:
    """Pair index -> (k1, k2) in itertools.combinations(range(n), 2) order."""
    a = 0
    while p >= n - 1 - a:
        p -= n - 1 - a
        a += 1
    return a, a + 1 + p


# ---- triangulatePoint3 over n views -------------------------------------------------------------------------------------
def camera(R, t, f, u0, v0):
    """(R_wTi, t_wTi, cal = (f, k1, k2, u0, v0)) as twoview_ba_ref takes cameras."""
    return np.asarray(R, float).reshape(3, 3), np.asarray(t, float).reshape(3), np.array([f, 0.0, 0.0, u0, v0], float)


def dlt_n(cams, uvs) -> Optional[np.ndarray]:
    """triangulateDLT: the right singular vector of the smallest singular value of the 2n x 4 system -> point, or None
    when the rank (singular values above 1e-9) is below 3 or the point is at infinity."""
    rows = []
    for c, uv in zip(cams, uvs):
        P = tv.projection_matrix(*c)
        rows += [uv[0] * P[2] - P[0], uv[1] * P[2] - P[1]]
    _, s, Vt = np.linalg.svd(np.array(rows))
    if int(np.sum(s > tv.DLT_RANK_TOL)) < 3:
        return None
    v = Vt[3]
    X = v[:3] / v[3]
    return X if np.all(np.isfinite(X)) else None


def triangulate_point3(cams, uvs) -> Optional[np.ndarray]:
    """gtsam.triangulatePoint3(rank_tol=1e-9, optimize=True) -> point, or None where it raises."""
    X = dlt_n(cams, uvs)
    if X is None:
        return None
    X = tv.refine_point(list(cams), [np.asarray(u, float) for u in uvs], X)
    for R, t, _ in cams:
        if not (R.T @ (X - t))[2] > 0.0:
            return None
    return X


def reproj_errors(cams: Dict[int, tuple], X, meas) -> np.ndarray:
    """compute_point_reprojection_errors' errors: NaN for a missing camera or a depth <= 0 (projectSafe)."""
    out = np.full(len(meas), np.nan)
    for k, (i, uv) in enumerate(meas):
        c = cams.get(i)
        if c is None:
            continue
        pr, z, *_ = tv.project(c[0], c[1], c[2], X)
        if z > 0.0:
            out[k] = np.sqrt((uv[0] - pr[0]) ** 2 + (uv[1] - pr[1]) ** 2)
    return out


def max_triangulation_angle(cams: Dict[int, tuple], X, images) -> float:
    angles = []
    for i1, i2 in itertools.combinations(images, 2):
        a, b = X - cams[i1][1], X - cams[i2][1]
        a, b = a / np.linalg.norm(a), b / np.linalg.norm(b)
        angles.append(float(np.rad2deg(np.arccos(np.clip(np.dot(a, b), -1, 1)))))
    return max(angles)


@dataclass
class TrackResult:
    exit_code: int
    point: Optional[np.ndarray]  # None unless the n-view triangulation ran
    avg_error: Optional[float]
    inliers: np.ndarray  # bool (n,)


def ransac_inliers(cams: Dict[int, tuple], meas, num_hypotheses: int, thr: float, seed: int, track_index: int) -> np.ndarray:
    """Point3dInitializer.execute_ransac_variant for RANSAC_SAMPLE_UNIFORM."""
    n = len(meas)
    pairs = list(itertools.combinations(range(n), 2))
    hyps = min(num_hypotheses, len(pairs))
    best_votes, best_err, best = 0, MAX_TRACK_REPROJ_ERROR, np.zeros(n, bool)
    for p in sample_pairs(seed, track_index, len(pairs), hyps):
        k1, k2 = pairs[p]
        (i1, uv1), (i2, uv2) = meas[k1], meas[k2]
        if cams.get(i1) is None or cams.get(i2) is None:
            continue
        X = triangulate_point3([cams[i1], cams[i2]], [uv1, uv2])
        if X is None:
            continue
        errors = reproj_errors(cams, X, meas)
        is_inlier = errors < thr
        inlier_errors = errors[is_inlier]
        if inlier_errors.size > 0:
            avg, votes = inlier_errors.mean(), int(is_inlier.sum())
            if votes > best_votes or (votes == best_votes and avg < best_err):
                best_votes, best_err, best = votes, avg, is_inlier
    return best


def triangulate_track(cams: Dict[int, tuple], meas: Sequence[Tuple[int, np.ndarray]], mode: str, num_hypotheses: int, thr: float,
                      min_angle: float, seed: int = 0, track_index: int = 0) -> TrackResult:
    """Point3dInitializer.triangulate for one track; `cams` maps image index -> camera (absent or None: no pose)."""
    n = len(meas)
    if mode == SAMPLE_UNIFORM:
        inl = ransac_inliers(cams, meas, num_hypotheses, thr, seed, track_index)
    elif mode == NO_RANSAC:
        inl = np.ones(n, bool)
    else:
        raise ValueError(f"mode {mode!r} is not restated")
    idx = np.flatnonzero(inl)
    if len(idx) < 2:
        return TrackResult(INLIERS_UNDERCONSTRAINED, None, None, inl)
    sub = [meas[k] for k in idx]
    with_cam = [(i, uv) for i, uv in sub if cams.get(i) is not None]
    if len(with_cam) < 2:
        return TrackResult(POSES_UNDERCONSTRAINED, None, None, inl)
    X = triangulate_point3([cams[i] for i, _ in with_cam], [uv for _, uv in with_cam])
    if X is None:
        return TrackResult(CHEIRALITY_FAILURE, None, None, inl)
    errors = reproj_errors(cams, X, sub)
    avg = float("nan") if np.isnan(errors).all() else float(np.nanmean(errors))
    if not np.all(errors < thr):
        return TrackResult(EXCEEDS_REPROJ_THRESH, X, avg, inl)
    if max_triangulation_angle(cams, X, [i for i, _ in sub]) < min_angle:
        return TrackResult(LOW_TRIANGULATION_ANGLE, X, avg, inl)
    return TrackResult(SUCCESS, X, avg, inl)


# ---- arrays ---------------------------------------------------------------------------------------------------------------
def cams_dict(cams: np.ndarray, valid: np.ndarray) -> Dict[int, tuple]:
    """[num_images][15] (R 9, t 3, f, u0, v0) and validity -> {image: camera}."""
    return {i: camera(c[:9], c[9:12], c[12], c[13], c[14]) for i, c in enumerate(np.asarray(cams, float)) if valid[i]}


def run_arrays(track_off, meas_cam, meas_uv, cams, valid, mode: str, num_hypotheses: int, thr: float, min_angle: float,
               seed: int = 0, tracks: Optional[Sequence[int]] = None):
    """The reference's loop over the tracks of a packed batch (all, or the positions `tracks`) -> (exit (T,) int8,
    point (T, 3), avg (T,), inlier (M,) uint8) in the device's layout (NaN for None; rows not in `tracks` stay NaN / 0)."""
    track_off = np.asarray(track_off, np.int64)
    T = len(track_off) - 1
    cd = cams_dict(cams, valid)
    ex, pt, avg = np.full(T, -1, np.int8), np.full((T, 3), np.nan), np.full(T, np.nan)
    inl = np.zeros(track_off[-1], np.uint8)
    for t in (range(T) if tracks is None else tracks):
        a, b = track_off[t], track_off[t + 1]
        meas = [(int(meas_cam[m]), np.asarray(meas_uv[m], float)) for m in range(a, b)]
        r = triangulate_track(cd, meas, mode, num_hypotheses, thr, min_angle, seed, t)
        ex[t] = r.exit_code
        if r.point is not None:
            pt[t] = r.point
        if r.avg_error is not None:
            avg[t] = r.avg_error
        inl[a:b] = r.inliers
    return ex, pt, avg, inl


def pack_tracks(tracks: List[List[Tuple[int, Sequence[float]]]]):
    """[[(image, uv), ...], ...] -> (track_off (T+1,) int64, meas_cam (M,) int32, meas_uv (M, 2) float64)."""
    off = np.zeros(len(tracks) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in tracks])
    cam = np.fromiter((i for t in tracks for i, _ in t), np.int32, count=int(off[-1]))
    uv = np.array([uv for t in tracks for _, uv in t], np.float64).reshape(-1, 2)
    return off, cam, uv
