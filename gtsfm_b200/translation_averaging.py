"""1DSfM's outlier rejection on the device.

Drop-in for gtsfm/averaging/translation/averaging_1dsfm.py (`TranslationAveraging1DSFM`): the reference's constructor
arguments plus `device` and `ctx`.  With GTSfM installed the class subclasses the reference's and overrides
`compute_inliers` only, so `run_translation_averaging` (track selection, landmark directions, TranslationRecovery,
metrics) stays the reference's own.  The projection directions come from the reference's own sampler on NumPy's global
RNG, as in a reference run; the MFAS ordering of every direction and the per-edge sum of the outlier weights come from
one fp64 call into libgtsfm_b200.so (`b2_mfas_outlier_weights_host`, csrc/mfas.cu).  Where gtsam breaks a tie in the
hash order of an unordered_map, the device takes the lowest key (DESIGN.md).

Without GTSfM the mirror in gtsfm_api.py restates the SAMPLE_INPUT_MEASUREMENTS and SAMPLE_WITH_UNIFORM_DENSITY samplers;
SAMPLE_WITH_INPUT_DENSITY raises ValueError and `run_translation_averaging` is unavailable.
"""
from __future__ import annotations

from typing import Any, Dict, Set, Tuple

import numpy as np

from . import _lib
from .gtsfm_api import TranslationAveraging1DSFM

OUTLIER_WEIGHT_THRESHOLD = 0.125  # averaging_1dsfm.py:52


def _vectors(values) -> np.ndarray:
    """Unit3 objects (or 3-vectors) -> (n, 3) float64, each as its point3()."""
    out = np.empty((len(values), 3))
    for k, v in enumerate(values):
        out[k] = v.point3() if hasattr(v, "point3") else np.asarray(v, np.float64).reshape(3)
    return out


def dense_edges(w_i2Ui1_dict: Dict, w_iUj_dict_tracks: Dict):
    """The reference's measurements (camera pair (i1, i2) -> edge (C(i2), C(i1)); track measurement (j, i) -> edge
    (C(i), L(j))) on dense node ids in key order (cameras, then landmarks).  -> (num_nodes, edge_a, edge_b (E,) int32 in
    map order, perm (E,): edge e is measurement perm[e], cameras first).  ValueError for a self edge, a node pair measured
    twice, or an index outside [0, 2^56)."""
    cam = np.array([(i2, i1) for (i1, i2) in w_i2Ui1_dict], np.int64).reshape(-1, 2)
    trk = np.array([(i, j) for (j, i) in w_iUj_dict_tracks], np.int64).reshape(-1, 2)
    for x in (cam, trk):
        if x.size and (x.min() < 0 or x.max() >= 2 ** 56):
            raise ValueError("camera and track indices must lie in [0, 2^56)")
    cams = np.unique(np.concatenate([cam.ravel(), trk[:, 0]]))
    lmks = np.unique(trk[:, 1])
    a = np.concatenate([np.searchsorted(cams, cam[:, 0]), np.searchsorted(cams, trk[:, 0])]).astype(np.int64)
    b = np.concatenate([np.searchsorted(cams, cam[:, 1]), len(cams) + np.searchsorted(lmks, trk[:, 1])]).astype(np.int64)
    if np.any(a == b):
        raise ValueError("a camera pair (i, i): an edge from a node to itself")
    V = len(cams) + len(lmks)
    if len(np.unique(np.minimum(a, b) * V + np.maximum(a, b))) != len(a):
        raise ValueError("a camera pair is given twice, as (i1, i2) and (i2, i1)")
    if V >= 2 ** 30:
        raise ValueError("more than 2^30 nodes")
    perm = np.lexsort((b, a))
    return V, a[perm].astype(np.int32), b[perm].astype(np.int32), perm


def outlier_weights_arrays(ctx: "_lib.Context", V: int, edge_a, edge_b, meas, dirs, order: bool = False, violated: bool = False):
    """The device call on arrays: V nodes, edges (edge_a, edge_b) strictly increasing in (a, b), meas (E, 3) unit vectors,
    dirs (K, 3).  -> weight_sum (E,) float64, the sum over directions in order of each edge's outlier weight; with `order`
    also (K, V) int32, the node removed at each step; with `violated` also (K, ceil(E/32)) uint32, the violated-edge bits."""
    ea = np.ascontiguousarray(edge_a, np.int32).reshape(-1)
    eb = np.ascontiguousarray(edge_b, np.int32).reshape(-1)
    m = np.ascontiguousarray(meas, np.float64).reshape(-1, 3)
    d = np.ascontiguousarray(dirs, np.float64).reshape(-1, 3)
    E, K = len(ea), len(d)
    if len(eb) != E or len(m) != E:
        raise ValueError("edge_a, edge_b and meas do not agree in size")
    s = np.zeros(E)
    o = np.zeros((K, V), np.int32) if order else None
    w = np.zeros((K, (E + 31) // 32), np.uint32) if violated else None
    rc = ctx.lib.b2_mfas_outlier_weights_host(ctx.handle, int(V), E, _lib.ptr(ea), _lib.ptr(eb), _lib.ptr(m), K, _lib.ptr(d), _lib.ptr(s),
                                              None if o is None else _lib.ptr(o), None if w is None else _lib.ptr(w), None)
    ctx.check(rc, "mfas_outlier_weights")
    if not (order or violated):
        return s
    return (s,) + ((o,) if order else ()) + ((w,) if violated else ())


class B200TranslationAveraging1DSFM(TranslationAveraging1DSFM):
    """`ctx`: a library context, or a DeviceFrontEnd whose context to share; by default one is created on `device` at
    the first call."""

    def __init__(self, robust_measurement_noise: bool = True, use_tracks_for_averaging: bool = True, reject_outliers: bool = True,
                 projection_sampling_method=TranslationAveraging1DSFM.ProjectionSamplingMethod.SAMPLE_WITH_UNIFORM_DENSITY,
                 max_delayed_calls: int = 16, use_all_tracks_for_averaging: bool = False, use_relative_camera_poses: bool = True,
                 device: int = 0, ctx: Any = None) -> None:
        if isinstance(projection_sampling_method, str):
            projection_sampling_method = self.ProjectionSamplingMethod(projection_sampling_method)
        super().__init__(robust_measurement_noise=robust_measurement_noise, use_tracks_for_averaging=use_tracks_for_averaging,
                         reject_outliers=reject_outliers, projection_sampling_method=projection_sampling_method,
                         max_delayed_calls=max_delayed_calls, use_all_tracks_for_averaging=use_all_tracks_for_averaging,
                         use_relative_camera_poses=use_relative_camera_poses)
        self._device = device
        self._ctx = getattr(ctx, "ctx", ctx)

    def __getstate__(self):  # device state is created lazily on the worker, like the other plugins
        d = dict(self.__dict__)
        d["_ctx"] = None
        return d

    def _context(self) -> _lib.Context:
        if self._ctx is None:
            self._ctx = _lib.Context(self._device)
        return self._ctx

    def projection_directions(self, w_i2Ui1_dict: Dict, w_iUj_dict_tracks: Dict) -> np.ndarray:
        """The reference's __sample_projection_directions on its combined measurement list (consumes NumPy's global RNG
        as a reference run does): (K, 3)."""
        combined = list(w_i2Ui1_dict.values()) + list(w_iUj_dict_tracks.values())
        return _vectors(self._TranslationAveraging1DSFM__sample_projection_directions(combined)).reshape(-1, 3)

    def compute_inliers(self, w_i2Ui1_dict: Dict, w_iUj_dict_tracks: Dict) -> Tuple[Dict, Dict, Set[int]]:
        """The reference's (inlier camera directions, inlier track directions, inlier cameras)."""
        dirs = self.projection_directions(w_i2Ui1_dict, w_iUj_dict_tracks)
        if len(dirs) == 0:  # the reference's batching fails the same way: range() with a step of 0
            raise ValueError("no projection directions: SAMPLE_INPUT_MEASUREMENTS without any measurement")
        V, ea, eb, perm = dense_edges(w_i2Ui1_dict, w_iUj_dict_tracks)
        values = list(w_i2Ui1_dict.values()) + list(w_iUj_dict_tracks.values())
        if not values:
            return {}, {}, set()
        meas = _vectors(values)[perm]
        s = outlier_weights_arrays(self._context(), V, ea, eb, meas, dirs)
        inlier = np.empty(len(values), bool)
        inlier[perm] = s / len(dirs) < OUTLIER_WEIGHT_THRESHOLD
        nc = len(w_i2Ui1_dict)
        cams, tracks, inlier_cameras = {}, {}, set()
        for f, ((i1, i2), v) in zip(inlier[:nc], w_i2Ui1_dict.items()):
            if f:
                cams[(i1, i2)] = v
                inlier_cameras.update((i1, i2))
        for f, ((j, i), v) in zip(inlier[nc:], w_iUj_dict_tracks.items()):
            if f and i in inlier_cameras:  # a track measurement is kept only when its camera has an inlier camera pair
                tracks[(j, i)] = v
        return cams, tracks, inlier_cameras
