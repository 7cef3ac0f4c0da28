"""NumPy statement of 1DSfM's outlier rejection (gtsfm/averaging/translation/averaging_1dsfm.py:127-315, with gtsam's
MFAS::computeOutlierWeights per projection direction), the oracle of csrc/mfas.cu.

MFAS is stated twice:
  * `mfas_literal`: gtsam's algorithm as written, on 64-bit keys, dicts and sorted sets (one direction);
  * `order_vectorised`: dense node ids, NumPy arrays, one argmax per step (fast enough for a few thousand nodes).
For one direction d, edge (k1, k2) with unit measurement m has weight w = (mx*dx + my*dy) + mz*dz and points k1 -> k2
when w >= 0, else k2 -> k1; |w| is added to the destination's in-sum and the source's out-sum, edges in std::map order.
Until no node is left: a node with in-sum < 1e-8 is picked if there is one, else the node of largest (out + 1) / (in + 1);
both ties go to the lowest key (gtsam takes the first in its unordered_map's hash order, which cannot be reproduced).  The
picked node's edges are subtracted from its remaining neighbours.  Edge s -> t's outlier weight is |w| if t was removed
before s, else 0.

`outlier_weight_sums` adds each edge's outlier weights over the directions in order, as the reference's Python loop
does, `inlier_mask` applies the threshold, and `split_outputs` rebuilds compute_inliers' three outputs.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

MAX_PROJECTION_DIRECTIONS = 2000  # averaging_1dsfm.py:51
OUTLIER_WEIGHT_THRESHOLD = 0.125  # averaging_1dsfm.py:52
SOURCE_IN_WEIGHT = 1e-8           # gtsam MFAS.cpp: a source has inWeightSum below this
SAMPLE_INPUT_MEASUREMENTS = "SAMPLE_INPUT_MEASUREMENTS"
SAMPLE_WITH_INPUT_DENSITY = "SAMPLE_WITH_INPUT_DENSITY"
SAMPLE_WITH_UNIFORM_DENSITY = "SAMPLE_WITH_UNIFORM_DENSITY"


def C(i: int) -> int:  # symbol_shorthand.A: camera translation keys
    return (ord("a") << 56) | int(i)


def L(j: int) -> int:  # symbol_shorthand.B: landmark keys
    return (ord("b") << 56) | int(j)


def unit3(v) -> np.ndarray:
    """gtsam.Unit3(v).point3(): Eigen's normalized(), v / sqrt((x*x + y*y) + z*z), row by row."""
    v = np.asarray(v, np.float64)
    v2 = np.atleast_2d(v)
    n = np.sqrt((v2[:, 0] * v2[:, 0] + v2[:, 1] * v2[:, 1]) + v2[:, 2] * v2[:, 2])
    return (v2 / n[:, None]).reshape(v.shape)


def sample_directions(method: str, measurements: np.ndarray, num: int = MAX_PROJECTION_DIRECTIONS) -> np.ndarray:
    """__sample_projection_directions (averaging_1dsfm.py:127-155) on NumPy's global RNG: (K, 3)."""
    measurements = np.asarray(measurements, np.float64).reshape(-1, 3)
    if method == SAMPLE_INPUT_MEASUREMENTS:
        n = len(measurements)
        return measurements[np.random.choice(n, min(n, num), replace=False)].reshape(-1, 3)
    if method == SAMPLE_WITH_UNIFORM_DENSITY:
        return unit3(np.random.normal(size=(num, 3)))  # sampling.sample_random_directions
    raise ValueError(f"sampling method {method!r} is not restated here (the KDE sampler is the reference's own)")


def edge_weights(meas: np.ndarray, d: np.ndarray) -> np.ndarray:
    """w = m . d as (mx*dx + my*dy) + mz*dz for every row of meas (E, 3)."""
    meas = np.asarray(meas, np.float64).reshape(-1, 3)
    return (meas[:, 0] * d[0] + meas[:, 1] * d[1]) + meas[:, 2] * d[2]


# ---- measurements and dense ids -------------------------------------------------------------------------------------------
def measurements_from_dicts(w_i2Ui1: Dict, w_iUj_tracks: Dict) -> List[Tuple[int, int, np.ndarray]]:
    """_binary_measurements_from_dict (averaging_1dsfm.py:157-179): (key1, key2, unit vector), cameras then tracks."""
    out = [(C(i2), C(i1), np.asarray(v, np.float64)) for (i1, i2), v in w_i2Ui1.items()]
    out += [(C(i), L(j), np.asarray(v, np.float64)) for (j, i), v in w_iUj_tracks.items()]
    return out


def dense_problem(measurements: Sequence[Tuple[int, int, np.ndarray]]):
    """Measurements -> (keys (V,) uint64 sorted, ea, eb (E,) int32 dense ids in map order, meas (E, 3), perm (E,)):
    edge e of the map is measurement perm[e].  ValueError for a self edge or a node pair given twice."""
    k1 = np.array([m[0] for m in measurements], np.uint64)
    k2 = np.array([m[1] for m in measurements], np.uint64)
    keys = np.unique(np.concatenate([k1, k2]))
    a, b = np.searchsorted(keys, k1).astype(np.int32), np.searchsorted(keys, k2).astype(np.int32)
    if np.any(a == b):
        raise ValueError("a measurement from a node to itself")
    lo, hi = np.minimum(a, b).astype(np.int64), np.maximum(a, b).astype(np.int64)
    if len(np.unique(lo * len(keys) + hi)) != len(a):
        raise ValueError("the same node pair is measured twice")
    perm = np.lexsort((b, a))
    meas = np.array([m[2] for m in measurements], np.float64).reshape(-1, 3)
    return keys, a[perm], b[perm], meas[perm], perm


# ---- MFAS, literally ----------------------------------------------------------------------------------------------------------
def mfas_literal(measurements: Sequence[Tuple[int, int, np.ndarray]], d) -> Tuple[List[int], Dict[Tuple[int, int], float]]:
    """gtsam MFAS(measurements, d): (ordering as keys, computeOutlierWeights() as {(key1, key2): weight})."""
    dx, dy, dz = (float(x) for x in np.asarray(d, np.float64).reshape(3))
    weights: Dict[Tuple[int, int], float] = {}
    for k1, k2, m in measurements:  # std::map<KeyPair, double>
        mx, my, mz = (float(x) for x in m)
        weights[(int(k1), int(k2))] = (mx * dx + my * dy) + mz * dz
    graph: Dict[int, dict] = {}
    for (k1, k2) in sorted(weights):  # graphFromEdges, in map order
        w = weights[(k1, k2)]
        s, t = (k1, k2) if w >= 0 else (k2, k1)
        for k in (s, t):
            graph.setdefault(k, {"in": 0.0, "out": 0.0, "in_nb": set(), "out_nb": set()})
        graph[t]["in_nb"].add(s)
        graph[t]["in"] += abs(w)
        graph[s]["out_nb"].add(t)
        graph[s]["out"] += abs(w)

    def weight(x, y):
        return weights[(x, y)] if (x, y) in weights else weights[(y, x)]

    ordering: List[int] = []
    while graph:
        nodes = sorted(graph)
        sources = [k for k in nodes if graph[k]["in"] < SOURCE_IN_WEIGHT]
        if sources:
            sel = sources[0]
        else:
            sel, best = None, -np.inf
            for k in nodes:
                r = (graph[k]["out"] + 1.0) / (graph[k]["in"] + 1.0)
                if sel is None or r > best:
                    sel, best = k, r
        for nb in sorted(graph[sel]["in_nb"]):  # removeNodeFromGraph
            graph[nb]["out"] -= abs(weight(nb, sel))
            graph[nb]["out_nb"].discard(sel)
        for nb in sorted(graph[sel]["out_nb"]):
            graph[nb]["in"] -= abs(weight(sel, nb))
            graph[nb]["in_nb"].discard(sel)
        del graph[sel]
        ordering.append(sel)
    pos = {k: i for i, k in enumerate(ordering)}
    out: Dict[Tuple[int, int], float] = {}
    for (k1, k2), w in sorted(weights.items()):
        s, t = (k1, k2) if w >= 0 else (k2, k1)
        out[(k1, k2)] = abs(w) if pos[t] < pos[s] else 0.0
    return ordering, out


# ---- MFAS, vectorised -------------------------------------------------------------------------------------------------------
def incidence(V: int, ea: np.ndarray, eb: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Each node's incident edges in map order: (inc_off (V+1,), inc_edge (2E,)) int32."""
    E = len(ea)
    nodes = np.concatenate([ea, eb]).astype(np.int64)
    eids = np.concatenate([np.arange(E), np.arange(E)])
    o = np.lexsort((eids, nodes))
    off = np.zeros(V + 1, np.int64)
    np.cumsum(np.bincount(nodes, minlength=V), out=off[1:])
    return off.astype(np.int32), eids[o].astype(np.int32)


def _pick_key(inn, out):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(inn < SOURCE_IN_WEIGHT, np.inf, (out + 1.0) / (inn + 1.0))


def order_vectorised(V: int, ea, eb, meas, d, inc=None) -> Tuple[np.ndarray, np.ndarray]:
    """One direction on dense ids: (order (V,) node removed at each step, violated (E,) bool)."""
    ea, eb = np.asarray(ea, np.int64), np.asarray(eb, np.int64)
    w = edge_weights(meas, np.asarray(d, np.float64).reshape(3))
    aw = np.abs(w)
    src, dst = np.where(w >= 0, ea, eb), np.where(w >= 0, eb, ea)
    inn, out = np.zeros(V), np.zeros(V)
    np.add.at(inn, dst, aw)  # element by element in map order: each node's sums add in gtsam's order
    np.add.at(out, src, aw)
    off, inc_edge = incidence(V, ea, eb) if inc is None else inc
    key = _pick_key(inn, out)
    pos = np.full(V, -1, np.int64)
    order = np.empty(V, np.int64)
    for step in range(V):
        u = int(np.argmax(key))  # the first maximum: the lowest id; removed nodes hold -inf
        pos[u], order[step], key[u] = step, u, -np.inf
        idx = inc_edge[off[u]:off[u + 1]]
        v = np.where(ea[idx] == u, eb[idx], ea[idx])
        live = pos[v] < 0
        idx, v = idx[live], v[live]
        u_src = src[idx] == u
        inn[v[u_src]] -= aw[idx[u_src]]
        out[v[~u_src]] -= aw[idx[~u_src]]
        key[v] = _pick_key(inn[v], out[v])
    return order, pos[dst] < pos[src]


def outlier_weight_sums(V: int, ea, eb, meas, dirs, form: str = "vectorised", keys=None) -> np.ndarray:
    """Each edge's sum over the directions, in order, of its outlier weight (the reference's Python-float loop)."""
    dirs = np.asarray(dirs, np.float64).reshape(-1, 3)
    s = np.zeros(len(ea))
    if form == "vectorised":
        inc = incidence(V, np.asarray(ea), np.asarray(eb))
        for d in dirs:
            _, bad = order_vectorised(V, ea, eb, meas, d, inc)
            s = s + np.where(bad, np.abs(edge_weights(meas, d)), 0.0)
        return s
    keys = np.arange(V, dtype=np.uint64) if keys is None else keys
    ms = [(int(keys[a]), int(keys[b]), m) for a, b, m in zip(ea, eb, np.asarray(meas).reshape(-1, 3))]
    for d in dirs:
        _, ow = mfas_literal(ms, d)
        s = s + np.array([ow[(k1, k2)] for k1, k2, _ in ms])
    return s


def inlier_mask(weight_sum: np.ndarray, K: int) -> np.ndarray:
    return np.asarray(weight_sum) / K < OUTLIER_WEIGHT_THRESHOLD


def split_outputs(w_i2Ui1: Dict, w_iUj_tracks: Dict, inlier_meas: np.ndarray):
    """compute_inliers' outputs (averaging_1dsfm.py:298-315) from the inlier flag of each measurement, in
    measurements_from_dicts order: (inlier camera dict, inlier track dict, inlier cameras)."""
    nc = len(w_i2Ui1)
    cams, tracks, inlier_cameras = {}, {}, set()
    for f, ((i1, i2), v) in zip(inlier_meas[:nc], w_i2Ui1.items()):
        if f:
            cams[(i1, i2)] = v
            inlier_cameras.update((i1, i2))
    for f, ((j, i), v) in zip(inlier_meas[nc:], w_iUj_tracks.items()):
        if f and i in inlier_cameras:
            tracks[(j, i)] = v
    return cams, tracks, inlier_cameras


def compute_inliers(w_i2Ui1: Dict, w_iUj_tracks: Dict, dirs: np.ndarray, form: str = "vectorised"):
    """compute_inliers on given directions: (the three outputs, the per-edge sums in map order)."""
    ms = measurements_from_dicts(w_i2Ui1, w_iUj_tracks)
    if not ms:
        return ({}, {}, set()), np.zeros(0)
    keys, ea, eb, meas, perm = dense_problem(ms)
    s = outlier_weight_sums(len(keys), ea, eb, meas, dirs, form, keys)
    inl = np.empty(len(ms), bool)
    inl[perm] = inlier_mask(s, len(dirs))
    return split_outputs(w_i2Ui1, w_iUj_tracks, inl), s


# the reference's Test1dsfmAllOutliers (tests/averaging/translation/test_averaging_1dsfm.py:233-303)
ALL_OUTLIERS_WRI = [
    [[-0.382164, 0.89195, 0.241612], [-0.505682, 0.0169854, -0.862553], [-0.773458, -0.451815, 0.444551]],
    [[-0.453335, 0.886803, -0.0898219], [-0.27425, -0.234656, -0.93259], [-0.8481, -0.398142, 0.349584]],
    [[-0.385656, 0.90387, -0.18517], [0.125519, -0.147431, -0.981076], [-0.914065, -0.4016, -0.0565954]],
    [[-0.359387, 0.898029, -0.253744], [0.253506, -0.167734, -0.95268], [-0.898096, -0.406706, -0.167375]],
    [[-0.342447, 0.898333, -0.275186], [0.0881727, -0.260874, -0.961338], [-0.935391, -0.353471, 0.0101272]]]
ALL_OUTLIERS_U = {(0, 1): [0.967948, -0.0290259, 0.24947], (0, 2): [0.906879, -0.000610539, 0.42139],
                  (0, 3): [0.937168, -0.0161865, 0.348502], (0, 4): [-0.975139, 0.0133109, -0.221193],
                  (1, 2): [0.990186, 0.0188153, 0.138484], (1, 3): [0.986072, -0.00746304, 0.166149],
                  (1, 4): [-0.996558, 0.00911097, -0.0823996], (2, 3): [0.990546, -0.0294894, 0.133976],
                  (2, 4): [0.998932, -0.0300599, -0.035099], (3, 4): [0.994791, -0.033332, -0.0963361]}


def all_outliers_inputs():
    """get_valid_measurements_in_world_frame on the reference test's inputs: {(i1, i2): Unit3(wRi2 * i2Ui1)}.  With uniform
    sampling, seed 0 and K = 2000, the reference rejects every edge to camera 4."""
    out = {}
    for (i1, i2), u in ALL_OUTLIERS_U.items():
        R, p = np.array(ALL_OUTLIERS_WRI[i2]), unit3(np.array(u))
        out[(i1, i2)] = unit3((R[:, 0] * p[0] + R[:, 1] * p[1]) + R[:, 2] * p[2])
    return out
