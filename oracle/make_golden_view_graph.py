"""Writes the fixtures of the cycle-consistent rotation view-graph filter (oracle/view_graph_ref.py):

    tests/golden/view_graph_scenes.npz     seeded scenes: world rotations, relative rotations with 0.5-2 degrees of noise
        and 10-30 % random outlier edges, on exhaustive and k-nearest-neighbour graphs, a tree (no triangle), one
        triangle, two triangles sharing an edge (an even count), disconnected components, sparse large image indices,
        and cycles near 180 degrees
    tests/golden/view_graph_lund_door.npz  lund-door's pairs that pass inlier support, with their post-ISP rotations, from
        tests/golden/twoview_report_lund_door.npz

    python -m oracle.make_golden_view_graph --reference /path/to/gtsfm-checkout

Each scene is stored under "<name>/": edges (E, 2) int32, R (E, 3, 3); and per run "<name>/<run>/": keep, aggregate,
num_cycles, for the runs of RUNS (both criteria at the default threshold, and a non-default threshold).

Before writing, the restatement is pinned against the reference's own code, run from the checkout's sources under a
stand-in for Rot3: CycleConsistentRotationViewGraphEstimator.run and its aggregation, extract_cyclic_triplets_from_edges,
create_adjacency_list, compute_cyclic_rotation_error and compute_relative_rotation_angle (see _pin_against_reference).
"""
from __future__ import annotations

import argparse
import ast
import types
from pathlib import Path

import numpy as np
from scipy.spatial.transform import Rotation

from oracle import view_graph_ref as ref

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"
OUT_SCENES = GOLDEN / "view_graph_scenes.npz"
OUT_LUND = GOLDEN / "view_graph_lund_door.npz"
RUNS = {"median_7": (ref.MEDIAN, 7.0), "min_7": (ref.MIN, 7.0), "median_3": (ref.MEDIAN, 3.0), "min_2_5": (ref.MIN, 2.5)}


# ---- graphs and rotations (also used by the tests to make seeded graphs) -----------------------------------------------
def exhaustive_edges(n: int) -> np.ndarray:
    i, j = np.triu_indices(n, 1)
    return np.stack([i, j], 1).astype(np.int32)


def knn_edges(n: int, k: int, seed: int) -> np.ndarray:
    """Each of n points on the unit sphere joined to its k nearest: the union of those pairs, (i1 < i2), sorted."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, 3))
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    nn = np.empty((n, k), np.int64)
    for s in range(0, n, 1024):  # blocks keep the n x n similarity out of memory
        d = x[s:s + 1024] @ x.T
        d[np.arange(len(d)), np.arange(s, s + len(d))] = -np.inf
        nn[s:s + 1024] = np.argpartition(-d, k, axis=1)[:, :k]
    a = np.repeat(np.arange(n), k)
    e = np.stack([np.minimum(a, nn.ravel()), np.maximum(a, nn.ravel())], 1)
    return np.unique(e, axis=0).astype(np.int32)


def relative_rotations(edges, seed: int, noise_deg=(0.5, 2.0), outlier_frac: float = 0.2) -> np.ndarray:
    """i2Ri1 = i2Rw wRi1 of random world rotations, each times a rotation of noise_deg degrees about a random axis; a
    fraction outlier_frac of the edges gets a uniformly random rotation instead."""
    edges = np.asarray(edges, np.int64).reshape(-1, 2)
    rng = np.random.default_rng(seed)
    nodes, inv = np.unique(edges, return_inverse=True)
    wR = Rotation.random(len(nodes), random_state=rng.integers(2 ** 31)).as_matrix()
    inv = inv.reshape(-1, 2)
    R = np.matmul(wR[inv[:, 1]].transpose(0, 2, 1), wR[inv[:, 0]])
    axis = rng.normal(size=(len(edges), 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    ang = np.radians(rng.uniform(noise_deg[0], noise_deg[1], len(edges)))
    R = np.matmul(Rotation.from_rotvec(axis * ang[:, None]).as_matrix(), R)
    out = rng.random(len(edges)) < outlier_frac
    if out.any():
        R[out] = Rotation.random(int(out.sum()), random_state=rng.integers(2 ** 31)).as_matrix()
    return R


def _near_180(seed: int):
    """An exhaustive 8-node graph whose outlier edges are the consistent rotation turned by 179-180 degrees, so the cycles
    through one of them sit near 180 degrees."""
    e = exhaustive_edges(8)
    R = relative_rotations(e, seed, (0.0, 0.05), 0.0)
    rng = np.random.default_rng(seed + 1)
    for idx, deg in zip(rng.choice(len(e), 6, replace=False), (179.0, 179.9, 179.99, 179.999, 180.0, 179.5)):
        a = rng.normal(size=3)
        R[idx] = Rotation.from_rotvec(a / np.linalg.norm(a) * np.radians(deg)).as_matrix() @ R[idx]
    return e, R


def scenes() -> dict:
    out = {}
    for name, n, frac, seed in (("exhaustive_12", 12, 0.1, 1), ("exhaustive_25", 25, 0.3, 2)):
        e = exhaustive_edges(n)
        out[name] = (e, relative_rotations(e, seed, outlier_frac=frac))
    for name, n, k, frac, seed in (("knn_60_k6", 60, 6, 0.2, 3), ("knn_200_k10", 200, 10, 0.3, 4)):
        e = knn_edges(n, k, seed)
        out[name] = (e, relative_rotations(e, seed, outlier_frac=frac))
    rng = np.random.default_rng(5)
    parent = np.array([rng.integers(0, i) for i in range(1, 30)])
    e = np.stack([parent, np.arange(1, 30)], 1).astype(np.int32)
    out["tree_30"] = (e, relative_rotations(e, 5, outlier_frac=0.2))
    e = np.array([[0, 1], [1, 2], [0, 2]], np.int32)
    out["triangle"] = (e, relative_rotations(e, 6, outlier_frac=0.0))
    e = np.array([[0, 1], [0, 2], [1, 2], [1, 3], [2, 3]], np.int32)
    out["two_triangles"] = (e, relative_rotations(e, 7, noise_deg=(2.0, 4.0), outlier_frac=0.0))
    a, b = exhaustive_edges(7), knn_edges(30, 5, 8) + 100
    e = np.concatenate([a, b, [[50, 60], [60, 70]]]).astype(np.int32)
    out["disconnected"] = (e, relative_rotations(e, 8, outlier_frac=0.15))
    ids = np.sort(np.random.default_rng(9).choice(10 ** 6, 40, replace=False))
    e = ids[knn_edges(40, 6, 9)].astype(np.int32)
    out["sparse_large_ids"] = (e, relative_rotations(e, 9, outlier_frac=0.2))
    out["near_180"] = _near_180(10)
    return out


def lund_edges():
    """(edges, R): lund-door's pairs that pass inlier support, with the rotation their post-ISP report carries."""
    d = np.load(GOLDEN / "twoview_report_lund_door.npz")
    edges, R = [], []
    for a, b in d["pairs"]:
        key = f"{a}_{b}"
        if not bool(d[f"{key}/isp_ok"]):
            continue
        post = bool(d[f"{key}/ba"]) and bool(d[f"{key}/post_pose"])
        edges.append((int(a), int(b)))
        R.append(d[f"{key}/R_post"] if post else d[f"{key}/R_pre"])
    return np.array(edges, np.int32), np.array(R, np.float64)


def _store(arrays: dict, name: str, edges, R) -> None:
    arrays[f"{name}/edges"] = np.asarray(edges, np.int32)
    arrays[f"{name}/R"] = np.asarray(R, np.float64)
    for run, (crit, thr) in RUNS.items():
        keep, agg, ncyc = ref.run_literal(edges, R, crit, thr)
        k2, a2, n2 = ref.run_vectorised(edges, R, crit, thr)
        assert np.array_equal(keep, k2) and np.array_equal(ncyc, n2) and np.allclose(agg, a2, rtol=1e-12, atol=1e-12, equal_nan=True)
        arrays[f"{name}/{run}/keep"], arrays[f"{name}/{run}/aggregate"], arrays[f"{name}/{run}/num_cycles"] = keep, agg, ncyc.astype(np.int32)
        print(f"{name} {run}: {len(edges)} edges, {int(ncyc.sum()) // 3} triplets, kept {int(keep.sum())}")


# ---- pinning against the reference ------------------------------------------------------------------------------------
class _Rot3:
    def __init__(self, R=None):
        self.R = np.eye(3) if R is None else np.asarray(R, float)

    def between(self, o):
        return _Rot3(self.R.T @ o.R)

    def compose(self, o):
        return _Rot3(self.R @ o.R)

    def matrix(self):
        return self.R


def _module_body(path: Path, ns: dict, skip=()) -> dict:
    """Executes a module's top-level definitions (not its imports, nor the names in `skip`) in `ns`."""
    tree = ast.parse(path.read_text())
    for node in tree.body:
        if isinstance(node, (ast.Import, ast.ImportFrom)):
            continue
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id in skip for t in node.targets):
            continue
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in skip:
            continue
        exec(compile(ast.Module([node], []), str(path), "exec"), ns)
    return ns


def _reference(reference: Path) -> types.SimpleNamespace:
    import logging
    import time
    import typing
    from collections import defaultdict
    from enum import Enum

    g = reference / "gtsfm"
    base = {"np": np, "Rotation": Rotation, "defaultdict": defaultdict, "Enum": Enum, "time": time, "Path": Path, "Rot3": _Rot3,
            "Unit3": object, "Pose3": object, "Cal3Bundler": object, "Keypoints": object, "TwoViewEstimationReport": object,
            "AnnotatedGraph": typing.Dict, "ImageIndexPairs": typing.List, "logger": logging.getLogger("view_graph_pin"),
            **{k: getattr(typing, k) for k in typing.__all__}}
    graph = dict(base)
    for fn in ("create_adjacency_list", "extract_cyclic_triplets_from_edges"):
        src = ast.parse((g / "utils/graph.py").read_text())
        node = next(n for n in src.body if isinstance(n, ast.FunctionDef) and n.name == fn)
        exec(compile(ast.Module([node], []), str(g / "utils/graph.py"), "exec"), graph)
    comp = dict(base)
    src = ast.parse((g / "utils/geometry_comparisons.py").read_text())
    for node in src.body:
        if isinstance(node, ast.FunctionDef) and node.name in ("compute_relative_rotation_angle", "compute_cyclic_rotation_error"):
            exec(compile(ast.Module([node], []), str(g / "utils/geometry_comparisons.py"), "exec"), comp)
    est = dict(base, ViewGraphEstimatorBase=object, graph_utils=types.SimpleNamespace(**graph), comp_utils=types.SimpleNamespace(**comp))
    _module_body(g / "view_graph_estimator/cycle_consistent_rotation_estimator.py", est, skip=("logger",))
    return types.SimpleNamespace(graph=graph, comp=comp, est=est)


class _Report:
    R_error_deg = None


def _pin_against_reference(reference: Path, cases: dict) -> None:
    """The restatement equals the reference's code, run from the checkout's sources under a Rot3 stand-in."""
    r = _reference(reference)
    Est, Crit = r.est["CycleConsistentRotationViewGraphEstimator"], r.est["EdgeErrorAggregationCriterion"]
    assert r.est["ERROR_THRESHOLD"] == ref.ERROR_THRESHOLD
    for name, (edges, R) in cases.items():
        pairs = [(int(a), int(b)) for a, b in edges]
        t_ref = sorted(r.graph["extract_cyclic_triplets_from_edges"](pairs))
        assert t_ref == ref.triplets_literal(pairs) == [tuple(int(v) for v in t) for t in ref.triplets_vectorised(edges)], name
        adj = r.graph["create_adjacency_list"](pairs)
        assert all(b in adj[a] and a in adj[b] for a, b in pairs)
        rot = {p: _Rot3(m) for p, m in zip(pairs, R)}
        err_ref = [r.comp["compute_cyclic_rotation_error"](rot[(i0, i1)], rot[(i1, i2)], rot[(i0, i2)]) for i0, i1, i2 in t_ref]
        assert err_ref == [ref.cycle_error_deg(R[pairs.index((i0, i1))], R[pairs.index((i1, i2))], R[pairs.index((i0, i2))])
                           for i0, i1, i2 in t_ref], name
        if t_ref:
            assert np.allclose(ref.triplet_errors(edges, R, np.array(t_ref)), err_ref, rtol=1e-12, atol=1e-12)
        reports = {p: _Report() for p in pairs}
        for run, (crit, thr) in RUNS.items():
            est = Est(Crit(crit), thr)
            kept = est.run(dict(rot), {}, [], {}, [], reports)
            keep, agg, ncyc = ref.run_literal(edges, R, crit, thr)
            assert kept == {p for p, k in zip(pairs, keep) if k}, (name, run)
            per_edge = {}
            for (i0, i1, i2), err in zip(t_ref, err_ref):
                for e in ((i0, i1), (i1, i2), (i0, i2)):
                    per_edge.setdefault(e, []).append(err)
            aggregate = getattr(est, "_CycleConsistentRotationViewGraphEstimator__aggregate_errors_for_edge")
            a_ref = np.array([aggregate(per_edge[p]) if p in per_edge else np.nan for p in pairs])
            assert np.allclose(agg, a_ref, rtol=1e-12, atol=1e-12, equal_nan=True), (name, run)
            assert np.array_equal(ncyc, [len(per_edge.get(p, ())) for p in pairs])
    print(f"restatement equals the reference's run, triplet extraction and cycle error on {len(cases)} graphs")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, required=True, help="a GTSfM checkout (the pinned functions)")
    a = ap.parse_args()
    cases = scenes()
    lund = lund_edges()
    _pin_against_reference(a.reference, {**cases, "lund_door": lund})
    arrays = {}
    for name, (e, R) in cases.items():
        _store(arrays, name, e, R)
    arrays["names"] = np.array(list(cases))
    arrays["runs"] = np.array(list(RUNS))
    np.savez_compressed(OUT_SCENES, **arrays)
    print(OUT_SCENES)
    arrays = {}
    _store(arrays, "lund_door", *lund)
    arrays["runs"] = np.array(list(RUNS))
    np.savez_compressed(OUT_LUND, **arrays)
    print(OUT_LUND)


if __name__ == "__main__":
    main()
