"""Restatement of gtsfm/frontend/matcher/twoway_matcher.py (`TwoWayMatcher.match`) over cv2.BFMatcher(NORM_L2): NaN rows
dropped and indices remapped, one-way matching in both directions (knnMatch k = 2 with `m1.distance <= ratio * m2.distance`
in Python floats, or match without a ratio test), stable sort by distance, mutual check in 1 -> 2 dict order.  Also returns
the cv2 distance of every kept 1 -> 2 match (DMatch.distance), which the reference computes but does not return."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np


def _oneway(d1: np.ndarray, d2: np.ndarray, ratio: Optional[float]):
    import cv2

    bf = cv2.BFMatcher(normType=cv2.NORM_L2, crossCheck=False)
    if ratio is not None:
        matches = []
        for pair in bf.knnMatch(d1, d2, k=2):
            m1, m2 = pair  # ValueError with fewer than two candidates, as in the reference
            if m1.distance <= ratio * m2.distance:
                matches.append(m1)
    else:
        matches = bf.match(d1, d2)
    matches = sorted(matches, key=lambda m: m.distance)
    return {m.queryIdx: (m.trainIdx, m.distance) for m in matches}


def twoway_match(desc1: np.ndarray, desc2: np.ndarray, ratio: Optional[float] = None) -> Tuple[np.ndarray, np.ndarray]:
    """-> (matches, distances): (K, 2) uint32 rows in the reference's order and their float32 cv2 distances, or
    (np.array([]), empty float32) when there is no match (the reference's return value)."""
    empty = (np.array([]), np.zeros(0, np.float32))
    if desc1.size == 0 or desc2.size == 0:
        return empty
    v1 = np.nonzero(~np.isnan(desc1).any(axis=1))[0]
    v2 = np.nonzero(~np.isnan(desc2).any(axis=1))[0]
    m12 = _oneway(desc1[v1], desc2[v2], ratio)
    m21 = _oneway(desc2[v2], desc1[v1], ratio)
    rows = [(i1, i2, d) for i1, (i2, d) in m12.items() if i2 in m21 and m21[i2][0] == i1]
    if not rows:
        return empty
    m = np.array([(i1, i2) for i1, i2, _ in rows], dtype=np.uint32)
    m[:, 0] = v1[m[:, 0]]
    m[:, 1] = v2[m[:, 1]]
    return m, np.array([d for _, _, d in rows], np.float32)


def u8_distances(q: np.ndarray, t: np.ndarray) -> np.ndarray:
    """The exact path's arithmetic in NumPy: integer norms and dot products, d^2 = |a|^2 + |b|^2 - 2 a.b, then
    float32(sqrt(float32(d^2))).  -> [len(q)][len(t)] float32."""
    qi, ti = q.astype(np.int64), t.astype(np.int64)
    d2 = (qi * qi).sum(1)[:, None] + (ti * ti).sum(1)[None, :] - 2 * qi @ ti.T
    return np.sqrt(d2.astype(np.float32))


def top2(dist: np.ndarray):
    """cv2's batchDistance insertion rule for K = 2: order by (float distance, train index). -> (best, d1, d2)."""
    n = dist.shape[1]
    order = np.lexsort((np.broadcast_to(np.arange(n), dist.shape), dist), axis=1)
    best = order[:, 0]
    rows = np.arange(len(dist))
    d1 = dist[rows, best]
    d2 = dist[rows, order[:, 1]] if n > 1 else np.full(len(dist), np.inf, np.float32)
    return best, d1, d2


def twoway_from_distances(d12: np.ndarray, ratio: Optional[float] = None):
    """The reference's selection on a given 1 -> 2 distance matrix (its transpose is the 2 -> 1 one). -> (matches, dists)."""
    b12, a12, s12 = top2(d12)
    b21, a21, s21 = top2(np.ascontiguousarray(d12.T))
    ok12 = np.ones(len(b12), bool) if ratio is None else a12.astype(np.float64) <= ratio * s12.astype(np.float64)
    ok21 = np.ones(len(b21), bool) if ratio is None else a21.astype(np.float64) <= ratio * s21.astype(np.float64)
    i = np.nonzero(ok12 & ok21[b12] & (b21[b12] == np.arange(len(b12))))[0]
    i = i[np.lexsort((i, a12[i]))]
    return np.stack([i, b12[i]], 1).astype(np.uint32), a12[i]
