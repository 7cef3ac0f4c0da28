"""NumPy statement of GTSfM's cycle-consistent rotation view-graph filter (CycleConsistentRotationViewGraphEstimator.run,
gtsfm/view_graph_estimator/cycle_consistent_rotation_estimator.py:80-157, 224-240; graph.py:92-149;
geometry_comparisons.py:137-159, 226-241), in two forms:

  run_literal     the reference's loop restated line by line (dict adjacency, set intersections, one scipy rotvec and one
                  np.median / np.amin per edge); what oracle/make_golden_view_graph.py pins against the reference's code
  run_vectorised  the same result for graphs of ~10^6 triplets: triplets from a sorted sparse adjacency, batched 3 x 3
                  products, one batched scipy rotvec, per-edge segments by a lexsort

Both take edges (E, 2) with i1 < i2 and R (E, 3, 3) with R[e] = i2Ri1 of edge e, and return (keep (E,) bool, aggregate (E,)
float64, NaN for an edge in no triplet, num_cycles (E,) int).  An edge is kept when aggregate < threshold or when it is in
no triplet.
"""
from __future__ import annotations

from collections import defaultdict
from typing import Dict, List, Tuple

import numpy as np
from scipy.spatial.transform import Rotation

MEDIAN, MIN = "MEDIAN_EDGE_ERROR", "MIN_EDGE_ERROR"
ERROR_THRESHOLD = 7.0


def cycle_error_deg(R01: np.ndarray, R12: np.ndarray, R02: np.ndarray) -> float:
    """compute_cyclic_rotation_error(i1Ri0=R01, i2Ri1=R12, i2Ri0=R02): the angle of i2Ri0.between(i2Ri1).compose(i1Ri0)."""
    C = (R02.T @ R12) @ R01
    return float(np.rad2deg(np.linalg.norm(Rotation.from_matrix(C).as_rotvec())))


def triplets_literal(edges) -> List[Tuple[int, int, int]]:
    """extract_cyclic_triplets_from_edges, sorted (the reference's order comes from a set and is not used)."""
    adj = defaultdict(set)
    for a, b in edges:
        adj[a].add(b)
        adj[b].add(a)
    out = set()
    for a, b in edges:
        a, b = min(a, b), max(a, b)
        for c in adj[a] & adj[b]:
            out.add(tuple(sorted((a, b, c))))
    return sorted(out)


def _aggregate(errors: List[float], criterion: str) -> float:
    if criterion == MIN:
        return float(np.amin(errors))
    if criterion == MEDIAN:
        return float(np.median(errors))
    raise ValueError(f"unknown criterion {criterion!r}")


def run_literal(edges, R, criterion: str = MEDIAN, threshold: float = ERROR_THRESHOLD):
    edges = [(int(a), int(b)) for a, b in np.asarray(edges).reshape(-1, 2)]
    rot: Dict[Tuple[int, int], np.ndarray] = {e: np.asarray(r, np.float64) for e, r in zip(edges, np.asarray(R).reshape(-1, 3, 3))}
    per_edge = defaultdict(list)
    for i0, i1, i2 in triplets_literal(edges):
        err = cycle_error_deg(rot[(i0, i1)], rot[(i1, i2)], rot[(i0, i2)])
        for e in ((i0, i1), (i1, i2), (i0, i2)):
            per_edge[e].append(err)
    agg = np.array([_aggregate(per_edge[e], criterion) if e in per_edge else np.nan for e in edges], np.float64)
    ncyc = np.array([len(per_edge.get(e, ())) for e in edges], np.int64)
    keep = (ncyc == 0) | (agg < threshold)
    return keep, agg, ncyc


def triplets_vectorised(edges) -> np.ndarray:
    """(T, 3) sorted triplets, rows in lexicographic order: for every edge (i, j) and every k > j adjacent to j, the
    triplet (i, j, k) when (i, k) is an edge."""
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    if len(e) == 0:
        return np.zeros((0, 3), np.int64)
    nodes, inv = np.unique(e, return_inverse=True)
    s = inv.reshape(-1, 2)
    n = len(nodes)
    s = s[np.lexsort((s[:, 1], s[:, 0]))]
    keys = s[:, 0] * n + s[:, 1]
    indptr = np.searchsorted(s[:, 0], np.arange(n + 1))
    deg = indptr[s[:, 1] + 1] - indptr[s[:, 1]]
    first = np.repeat(indptr[s[:, 1]], deg)
    within = np.arange(int(deg.sum())) - np.repeat(np.cumsum(deg) - deg, deg)
    src = np.repeat(np.arange(len(s)), deg)
    i, j, k = s[src, 0], s[src, 1], s[first + within, 1]
    q = i * n + k
    pos = np.minimum(np.searchsorted(keys, q), len(keys) - 1)
    ok = keys[pos] == q
    t = np.stack([i[ok], j[ok], k[ok]], 1)
    t = t[np.lexsort((t[:, 2], t[:, 1], t[:, 0]))]
    return nodes[t]


def edge_index(edges, a, b) -> np.ndarray:
    """Row of edge (a[t], b[t]) in `edges` for every t (each must be an edge)."""
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    span = int(e.max()) + 1
    keys = e[:, 0] * span + e[:, 1]
    order = np.argsort(keys, kind="stable")
    q = np.asarray(a, np.int64) * span + np.asarray(b, np.int64)
    idx = order[np.searchsorted(keys[order], q)]
    assert np.array_equal(keys[idx], q)
    return idx


def triplet_errors(edges, R, T) -> np.ndarray:
    """Cycle errors (degrees) of triplets T (t, 3), batched."""
    R = np.asarray(R, np.float64).reshape(-1, 3, 3)
    if len(T) == 0:
        return np.zeros(0)
    e01, e12, e02 = (edge_index(edges, T[:, x], T[:, y]) for x, y in ((0, 1), (1, 2), (0, 2)))
    C = np.matmul(np.matmul(R[e02].transpose(0, 2, 1), R[e12]), R[e01])
    return np.rad2deg(np.linalg.norm(Rotation.from_matrix(C).as_rotvec(), axis=1))


def run_vectorised(edges, R, criterion: str = MEDIAN, threshold: float = ERROR_THRESHOLD):
    if criterion not in (MEDIAN, MIN):
        raise ValueError(f"unknown criterion {criterion!r}")
    edges = np.asarray(edges, np.int64).reshape(-1, 2)
    E = len(edges)
    T = triplets_vectorised(edges)
    err = triplet_errors(edges, R, T)
    if len(T):
        ids = np.concatenate([edge_index(edges, T[:, x], T[:, y]) for x, y in ((0, 1), (1, 2), (0, 2))])
    else:
        ids = np.zeros(0, np.int64)
    vals = np.tile(err, 3)
    order = np.lexsort((vals, ids))  # NaN sorts last within an edge
    ids, vals = ids[order], vals[order]
    ncyc = np.bincount(ids, minlength=E)
    start = np.cumsum(ncyc) - ncyc
    agg = np.full(E, np.nan)
    has = ncyc > 0
    st, m = start[has], ncyc[has]
    nan = np.isnan(vals[st + m - 1])
    if criterion == MIN:
        a = vals[st]
    else:
        hi = vals[st + m // 2]
        lo = vals[st + np.maximum(m // 2 - 1, 0)]
        a = np.where(m % 2 == 1, hi, (lo + hi) / 2.0)
    agg[has] = np.where(nan, np.nan, a)
    keep = (ncyc == 0) | (agg < threshold)
    return keep, agg, ncyc
