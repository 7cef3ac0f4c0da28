"""Cycle-consistent rotation view-graph estimator on the device.

Drop-in for gtsfm/view_graph_estimator/cycle_consistent_rotation_estimator.py (`CycleConsistentRotationViewGraphEstimator`):
same constructor arguments, and `run(...) -> Set[Tuple[int, int]]` with the reference's signature and result.  Every
triplet of edges (i0, i1), (i1, i2), (i0, i2) gets the cycle error |rotvec(i2Ri0^T i2Ri1 i1Ri0)| in degrees, each edge the
median or the minimum of the errors of its triplets, and an edge is kept when that aggregate is below `error_threshold`
or when it is in no triplet.  Triplet extraction, the errors and the aggregation run in libgtsfm_b200.so
(`b2_viewgraph_cycle_filter_host`, csrc/view_graph.cu) in fp64.  With GTSfM installed the class subclasses the
reference's ViewGraphEstimatorBase and overrides `run` only, so `create_computation_graph` and `compute_metrics` are the
reference's own.  The debug plots the reference writes under `output_dir` are not produced: the argument is accepted and
ignored (logged once).
"""
from __future__ import annotations

import logging
from pathlib import Path
from typing import Dict, Optional, Set, Tuple

import numpy as np

from . import _lib
from .gtsfm_api import EdgeErrorAggregationCriterion, ViewGraphEstimatorBase

logger = logging.getLogger(__name__)

ERROR_THRESHOLD = 7.0  # cycle_consistent_rotation_estimator.py:28
_CRITERIA = {EdgeErrorAggregationCriterion.MEDIAN_EDGE_ERROR.value: _lib.VG_MEDIAN,
             EdgeErrorAggregationCriterion.MIN_EDGE_ERROR.value: _lib.VG_MIN}


def _criterion_name(c) -> str:
    name = getattr(c, "value", c)
    if not isinstance(name, str) or name not in _CRITERIA:
        raise ValueError(f"unknown edge error aggregation criterion {c!r}; expected one of {sorted(_CRITERIA)}")
    return name


def _matrix(R) -> np.ndarray:
    if R is None:
        raise ValueError("a relative rotation is None; drop the edge before the view-graph estimator")
    m = np.asarray(R.matrix() if hasattr(R, "matrix") else R, np.float64)
    if m.shape != (3, 3):
        raise ValueError(f"a relative rotation must be 3 x 3, not {m.shape}")
    return m


class B200CycleConsistentRotationViewGraphEstimator(ViewGraphEstimatorBase):
    """`edge_error_aggregation_criterion`: the reference's EdgeErrorAggregationCriterion or its name ("MEDIAN_EDGE_ERROR",
    "MIN_EDGE_ERROR").  `ctx`: a library context, or a DeviceFrontEnd whose context to share; by default the estimator
    creates its own on `device` at the first call.  After `run`, `last_edge_errors` maps each edge in a triplet to its
    aggregate (the reference's per_edge_aggregate_error) and `last_num_cycles` each input edge to its triplet count."""

    def __init__(self, edge_error_aggregation_criterion, error_threshold: float = ERROR_THRESHOLD, device: int = 0, ctx=None) -> None:
        name = _criterion_name(edge_error_aggregation_criterion)
        self._edge_error_aggregation_criterion = EdgeErrorAggregationCriterion(name)
        self._error_threshold = float(error_threshold)
        if np.isnan(self._error_threshold):
            raise ValueError("error_threshold is NaN")
        self._device = device
        self._ctx = getattr(ctx, "ctx", ctx)
        self._warned_output_dir = False
        self.last_edge_errors: Dict[Tuple[int, int], float] = {}
        self.last_num_cycles: Dict[Tuple[int, int], int] = {}

    def __getstate__(self):  # device state is created lazily on the worker, like the other plugins
        d = dict(self.__dict__)
        d["_ctx"] = None
        return d

    def _context(self) -> _lib.Context:
        if self._ctx is None:
            self._ctx = _lib.Context(self._device)
        return self._ctx

    def run(self, i2Ri1_dict, i2Ui1_dict, calibrations, corr_idxs_i1i2, keypoints, two_view_reports,
            output_dir: Optional[Path] = None) -> Set[Tuple[int, int]]:
        """Edges of the view graph: the subset of the keys of `i2Ri1_dict` whose rotations are cycle-consistent.  The other
        arguments are unused, as in the reference.  Raises ValueError for an edge with i1 >= i2 or a negative index, and
        for a missing or non-finite rotation."""
        if output_dir and not self._warned_output_dir:
            logger.info("B200CycleConsistentRotationViewGraphEstimator: output_dir is ignored (no debug plots)")
            self._warned_output_dir = True
        keys = [(int(i1), int(i2)) for i1, i2 in i2Ri1_dict]
        self.last_edge_errors, self.last_num_cycles = {}, {}
        if not keys:
            return set()
        edges, R = self.arrays(i2Ri1_dict)
        keep, agg, ncyc = self.filter_arrays(edges, R)
        self.last_num_cycles = {e: int(c) for e, c in zip(keys, ncyc)}
        self.last_edge_errors = {e: float(a) for e, a, c in zip(keys, agg, ncyc) if c > 0}
        return {e for e, k in zip(keys, keep) if k}

    @staticmethod
    def arrays(i2Ri1_dict) -> Tuple[np.ndarray, np.ndarray]:
        """{(i1, i2): rotation} -> (edges (E, 2) int32, R (E, 3, 3) float64), checked as `run` documents."""
        edges = np.empty((len(i2Ri1_dict), 2), np.int32)
        R = np.empty((len(i2Ri1_dict), 3, 3), np.float64)
        for e, ((i1, i2), rot) in enumerate(i2Ri1_dict.items()):
            if not 0 <= i1 < i2 or i2 >= 2 ** 31:
                raise ValueError(f"edge ({i1}, {i2}): indices must satisfy 0 <= i1 < i2 < 2^31")
            edges[e] = i1, i2
            R[e] = _matrix(rot)
        if not np.isfinite(R).all():
            raise ValueError("relative rotations must be finite")
        return edges, R

    def filter_arrays(self, edges: np.ndarray, R: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The device call on arrays: -> (keep (E,) bool, aggregate (E,) float64, NaN for an edge in no triplet,
        num_cycles (E,) int32), in input order."""
        edges = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
        R = np.ascontiguousarray(R, np.float64).reshape(-1, 3, 3)
        n = len(edges)
        keep, agg, ncyc = np.zeros(n, np.uint8), np.empty(n, np.float64), np.empty(n, np.int32)
        if n == 0:
            return keep.astype(bool), agg, ncyc
        ctx = self._context()
        prm = _lib.ViewGraphParams(_CRITERIA[self._edge_error_aggregation_criterion.value], 0, self._error_threshold)
        rc = ctx.lib.b2_viewgraph_cycle_filter_host(ctx.handle, _lib.ptr(edges), _lib.ptr(R), n, _lib.C.byref(prm), _lib.ptr(keep),
                                                    _lib.ptr(agg), _lib.ptr(ncyc), None)
        ctx.check(rc, "viewgraph_cycle_filter")
        return keep.astype(bool), agg, ncyc


def debug_triplets(ctx: "_lib.Context", edges: np.ndarray, R: np.ndarray, capacity: Optional[int] = None):
    """Test-only: every triplet (sorted node ids) and its cycle error in degrees, as the device computes them, in no order."""
    edges = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
    R = np.ascontiguousarray(R, np.float64).reshape(-1, 3, 3)
    cap = int(capacity if capacity is not None else 4 * len(edges) + 16)
    nodes, err, count = np.zeros((cap, 3), np.int32), np.zeros(cap, np.float64), _lib.C.c_int64(0)
    rc = ctx.lib.b2_debug_viewgraph_triplets_host(ctx.handle, _lib.ptr(edges), _lib.ptr(R), len(edges), cap, _lib.ptr(nodes), _lib.ptr(err),
                                                  _lib.C.byref(count), None)
    ctx.check(rc, "debug_viewgraph_triplets")
    if count.value > cap:
        return debug_triplets(ctx, edges, R, int(count.value))
    return nodes[:count.value], err[:count.value], int(count.value)
