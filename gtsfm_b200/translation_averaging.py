"""1DSfM's outlier rejection and translation recovery on the device.

Drop-in for gtsfm/averaging/translation/averaging_1dsfm.py (`TranslationAveraging1DSFM`): the reference's constructor
arguments plus `device` and `ctx`.  With GTSfM installed the class subclasses the reference's and overrides
`compute_inliers` and `__run_averaging` only, so `run_translation_averaging` (track selection, landmark directions,
metrics) stays the reference's own.
- Outlier rejection: the projection directions come from the reference's own sampler on NumPy's global RNG, as in a
  reference run; the MFAS ordering of every direction and the per-edge sum of the outlier weights come from one fp64 call
  into libgtsfm_b200.so (`b2_mfas_outlier_weights_host`, csrc/mfas.cu).  Where gtsam breaks a tie in the hash order of an
  unordered_map, the device takes the lowest key (DESIGN.md).
- Translation recovery: gtsam's TranslationRecovery (Huber LM over one Point3 per camera and landmark) runs as one fp64
  call (`b2_translation_recovery_host`, csrc/translation_recovery.cu).  gtsam draws the initial values from its
  process-wide std::mt19937(42), never reseeded; this module keeps one mirror of that stream per process
  (`reseed_translation_rng` resets it), so consecutive calls in one process continue it as gtsam's do.  Nodes joined by
  zero translations share one value, as TranslationRecovery merges them (`merge_same_translation`).  Relative pose
  priors (i2Ti1_priors) and problems over the "ba_workspace_mb" budget run the reference's method, logged once; such a
  call starts gtsam's own generator where it stands, which after a device call is not where a reference run's would be
  (DESIGN.md §3).

Without GTSfM the mirror in gtsfm_api.py restates the SAMPLE_INPUT_MEASUREMENTS and SAMPLE_WITH_UNIFORM_DENSITY samplers;
SAMPLE_WITH_INPUT_DENSITY raises ValueError and `run_translation_averaging` is unavailable.  `recover_translations` is the
recovery's dict entry point, which needs no GTSfM.
"""
from __future__ import annotations

import logging
from typing import Any, Dict, List, Optional, Set, Tuple

import numpy as np

from . import _lib
from .gtsfm_api import HAVE_GTSFM_1DSFM, TranslationAveraging1DSFM

logger = logging.getLogger(__name__)

OUTLIER_WEIGHT_THRESHOLD = 0.125  # averaging_1dsfm.py:52
NOISE_MODEL_SIGMA = 0.01          # averaging_1dsfm.py:55, Isotropic.Sigma(2, 0.01) on the 3-vector error
HUBER_LOSS_K = 1.3                # averaging_1dsfm.py:56
PRIOR_SIGMA = 0.01                # TranslationRecovery::addPrior's priorNoiseModel, Isotropic::Sigma(3, 0.01)
LM_MAX_ITERS = 100                # LevenbergMarquardtParams().maxIterations
DEFAULT_WORKSPACE_MB = 4096       # b2_context's "ba_workspace_mb" default

_logged_fallback = False


class _Mt19937Uniform:
    """std::uniform_real_distribution<double>(-1, 1) on std::mt19937, as libstdc++ draws it: two 32-bit words per value,
    (w0 + w1 2^32) / 2^64 in double (just below 1 if it rounds to 1), mapped to 2 c - 1.  NumPy's legacy-seeded MT19937
    emits std::mt19937's words."""

    def __init__(self, seed: int):
        self._bg = np.random.MT19937()
        self._bg._legacy_seeding(seed)

    def draws(self, n: int) -> np.ndarray:
        w = self._bg.random_raw(2 * n).astype(np.float64).reshape(-1, 2)
        c = (w[:, 0] + w[:, 1] * 4294967296.0) / 18446744073709551616.0
        c = np.where(c >= 1.0, np.nextafter(1.0, 0.0), c)
        return 2.0 * c + -1.0


_rng: Optional[_Mt19937Uniform] = None


def reseed_translation_rng(seed: int = 42) -> None:
    """Restart this process's mirror of gtsam's kRandomNumberGenerator, as a fresh process would have it (tests)."""
    global _rng
    _rng = _Mt19937Uniform(seed)


def random_points(n: int) -> np.ndarray:
    """n Point3(u(), u(), u()) from the process-wide stream, (n, 3).  g++ evaluates the constructor's arguments right to
    left, so z takes the first draw of each point."""
    if _rng is None:
        reseed_translation_rng()
    return _rng.draws(3 * n).reshape(-1, 3)[:, ::-1].copy()


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

    def _TranslationAveraging1DSFM__run_averaging(self, num_images: int, w_i2Ui1_dict: Dict, w_i2Ui1_dict_tracks: Dict, wRi_list: List,
                                                  i2Ti1_priors: Dict, absolute_pose_priors: List, scale_factor: float) -> List[Optional[np.ndarray]]:
        """The reference's __run_averaging with TranslationRecovery on the device: the translation of every camera with a
        rotation that appears in an edge, None for the others."""
        why = None
        if len(i2Ti1_priors) > 0:
            why = "relative pose priors (i2Ti1_priors)"
        else:
            _, _, nodes, C, L, ea, eb, _ = reduced_problem(w_i2Ui1_dict, w_i2Ui1_dict_tracks)
            if len(ea) and not 0 < recovery_workspace_bytes(C, L, ea, eb) <= _budget_mb(self._ctx) << 20:
                why = "a problem over the ba_workspace_mb budget"
        if why is not None:
            if not HAVE_GTSFM_1DSFM:
                raise ValueError(f"{why} needs the reference's TranslationRecovery, and GTSfM is not installed")
            global _logged_fallback
            if not _logged_fallback:
                logger.info("B200TranslationAveraging1DSFM: %s is not served on the device; running the reference's method", why)
                _logged_fallback = True
            out = super()._TranslationAveraging1DSFM__run_averaging(num_images, w_i2Ui1_dict, w_i2Ui1_dict_tracks, wRi_list,
                                                                    i2Ti1_priors, absolute_pose_priors, scale_factor)
            if len(i2Ti1_priors) == 0:  # gtsam drew one Point3 per solved node from its stream: keep the mirror in step
                random_points(len(nodes))
            return out
        wti = recover_translations(self._context(), w_i2Ui1_dict, w_i2Ui1_dict_tracks, self._robust_measurement_noise, scale_factor)
        return [wti[i] if wRi_list[i] is not None and i in wti else None for i in range(num_images)]

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


def translation_graph(w_i2Ui1_dict: Dict, w_iUj_dict_tracks: Dict):
    """TranslationRecovery's graph on dense node ids: camera pair (i1, i2) -> edge (C(i2), C(i1), w_i2Ui1) first, then track
    measurement (j, i) -> (C(i), L(j), w_iUj), in the dicts' order.  -> (cameras (C,) sorted camera indices, tracks (L,)
    sorted track ids, edge_a, edge_b (E,) int32 with cameras 0..C-1 then landmarks, meas (E, 3))."""
    cam = np.array([(i2, i1) for (i1, i2) in w_i2Ui1_dict], np.int64).reshape(-1, 2)
    trk = np.array([(i, j) for (j, i) in w_iUj_dict_tracks], np.int64).reshape(-1, 2)
    cams = np.unique(np.concatenate([cam.ravel(), trk[:, 0]]))
    tracks = np.unique(trk[:, 1])
    if len(cams) + len(tracks) >= 2 ** 30:
        raise ValueError("more than 2^30 nodes")
    a = np.concatenate([np.searchsorted(cams, cam[:, 0]), np.searchsorted(cams, trk[:, 0])]).astype(np.int32)
    b = np.concatenate([np.searchsorted(cams, cam[:, 1]), len(cams) + np.searchsorted(tracks, trk[:, 1])]).astype(np.int32)
    meas = _vectors(list(w_i2Ui1_dict.values()) + list(w_iUj_dict_tracks.values()))
    return cams, tracks, a, b, meas


def initial_values(edge_a, edge_b, num_nodes: int) -> np.ndarray:
    """initializeRandomly: a, then b, of every edge in order; each node's first appearance draws its Point3 from the
    process-wide stream.  -> (num_nodes, 3)."""
    order = np.stack([np.asarray(edge_a), np.asarray(edge_b)], 1).ravel()
    first, idx = np.unique(order, return_index=True)
    if len(first) != num_nodes:
        raise ValueError("a node without an edge")
    x = np.empty((num_nodes, 3))
    x[order[np.sort(idx)]] = random_points(num_nodes)
    return x


def recovery_workspace_bytes(num_cameras: int, num_landmarks: int, edge_a, edge_b) -> int:
    """b2_translation_recovery_workspace_bytes: the call's device workspace (0 for invalid input)."""
    ea = np.ascontiguousarray(edge_a, np.int32)
    eb = np.ascontiguousarray(edge_b, np.int32)
    return int(_lib.load().b2_translation_recovery_workspace_bytes(int(num_cameras), int(num_landmarks), len(ea), _lib.ptr(ea), _lib.ptr(eb)))


def recover_arrays(ctx: "_lib.Context", num_cameras: int, num_landmarks: int, edge_a, edge_b, meas, init, huber_k: float = HUBER_LOSS_K,
                   scale: float = 1.0, sigma: float = NOISE_MODEL_SIGMA, prior_sigma: float = PRIOR_SIGMA, max_iters: int = LM_MAX_ITERS,
                   trace: bool = False) -> dict:
    """The device call on arrays: nodes 0..C-1 cameras, C..C+L-1 landmarks; edges (edge_a, edge_b, meas (E, 3)) in the
    reference's order; init (C + L, 3).  huber_k 0: no robust model.  -> dict of x (C + L, 3), final_error, iterations
    and, with `trace`, trace and trials."""
    ea = np.ascontiguousarray(edge_a, np.int32).reshape(-1)
    eb = np.ascontiguousarray(edge_b, np.int32).reshape(-1)
    m = np.ascontiguousarray(meas, np.float64).reshape(-1, 3)
    x0 = np.ascontiguousarray(init, np.float64).reshape(-1, 3)
    C, L, E = int(num_cameras), int(num_landmarks), len(ea)
    if len(eb) != E or len(m) != E or len(x0) != C + L:
        raise ValueError("edge_a, edge_b, meas and init do not agree in size")
    prm = _lib.TrParams(sigma=float(sigma), huber_k=float(huber_k), prior_sigma=float(prior_sigma), scale=float(scale),
                        max_iters=int(max_iters))
    out = np.empty_like(x0)
    res = _lib.BaResult()
    tr = np.zeros(prm.max_iters + 2) if trace else None
    cap = 64 * (prm.max_iters + 2) if trace else 0
    trials = np.zeros(cap, np.int32) if trace else None
    rc = ctx.lib.b2_translation_recovery_host(ctx.handle, C, L, E, _lib.ptr(ea), _lib.ptr(eb), _lib.ptr(m), _lib.ptr(x0), _lib.C.byref(prm),
                                              _lib.ptr(out), _lib.C.byref(res), _lib.ptr(tr), _lib.ptr(trials), cap, None)
    ctx.check(rc, "translation_recovery")
    d = dict(x=out, final_error=float(res.final_error), iterations=int(res.iterations))
    if trace:
        d["trace"] = tr[:res.trace_len].copy()
        d["trials"] = trials[:min(res.trials, cap)].copy()
    return d


def _budget_mb(ctx) -> int:
    return ctx.options.get("ba_workspace_mb", DEFAULT_WORKSPACE_MB) if ctx is not None else DEFAULT_WORKSPACE_MB


ZERO_TRANSLATION_TOL = 1e-9  # Unit3::equals' default tolerance, against Unit3(0, 0, 0)


def merge_same_translation(num_nodes: int, edge_a, edge_b, meas):
    """TranslationRecovery::run's zero-translation sets: nodes joined by a measurement equal to Unit3(0, 0, 0) (every
    component within 1e-9) share one translation; edges inside a set leave the graph, the others join the sets'
    representatives.  -> (root (num_nodes,) each node's representative, its lowest id; keep (E,) the edges that stay)."""
    ea, eb = np.asarray(edge_a, np.int64), np.asarray(edge_b, np.int64)
    parent = np.arange(num_nodes)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for e in np.nonzero(np.all(np.abs(np.asarray(meas).reshape(-1, 3)) <= ZERO_TRANSLATION_TOL, axis=1))[0]:
        ra, rb = find(ea[e]), find(eb[e])
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    root = np.array([find(x) for x in range(num_nodes)], np.int64)
    return root, root[ea] != root[eb]


def reduced_problem(w_i2Ui1_dict: Dict, w_iUj_dict_tracks: Dict):
    """The problem TranslationRecovery solves: translation_graph without the zero-translation sets' inner edges, on the
    sets' representatives.  -> (cameras (C,), root (V,), nodes (the solved nodes, ascending, cameras first), C', L',
    edge_a, edge_b (E',) on nodes' compact ids, meas (E', 3))."""
    cams, tracks, ea, eb, meas = translation_graph(w_i2Ui1_dict, w_iUj_dict_tracks)
    root, keep = merge_same_translation(len(cams) + len(tracks), ea, eb, meas)
    a, b = root[ea[keep]], root[eb[keep]]
    nodes = np.unique(np.concatenate([a, b]))
    nc = int(np.sum(nodes < len(cams)))
    return (cams, root, nodes, nc, len(nodes) - nc, np.searchsorted(nodes, a).astype(np.int32), np.searchsorted(nodes, b).astype(np.int32),
            meas[keep])


def recover_translations(ctx: "_lib.Context", w_i2Ui1_dict: Dict, w_iUj_dict_tracks: Dict, robust_measurement_noise: bool = True,
                         scale_factor: float = 1.0) -> Dict[int, np.ndarray]:
    """TranslationRecovery().run(measurements, scale_factor) on the reference's direction dicts ((i1, i2) -> w_i2Ui1 and
    (j, i) -> w_iUj, Unit3 or 3-vectors): {camera index: its translation} for every camera of an edge.  Nodes joined by
    zero translations share one value; with no other edge, every set sits at the origin.  Draws the initial values of
    the solved nodes from the process-wide stream.  ValueError for a problem over the "ba_workspace_mb" budget (checked
    before any draw) or that the device refuses."""
    cams, root, nodes, C, L, ea, eb, meas = reduced_problem(w_i2Ui1_dict, w_iUj_dict_tracks)
    if len(root) == 0:
        return {}
    x = np.full((len(root), 3), np.nan)
    if len(ea):
        need = recovery_workspace_bytes(C, L, ea, eb)
        if not 0 < need <= _budget_mb(ctx) << 20:
            raise ValueError(f"the translation recovery needs {need} bytes of device workspace, over the ba_workspace_mb budget")
        x0 = initial_values(ea, eb, C + L)
        try:
            out = recover_arrays(ctx, C, L, ea, eb, meas, x0, huber_k=HUBER_LOSS_K if robust_measurement_noise else 0.0, scale=scale_factor)
        except _lib.B200Error as e:
            raise ValueError(str(e)) from e
        x[nodes] = out["x"]
    else:
        x[np.unique(root)] = 0.0
    x = x[root]  # a set without an edge to the solve has no value (gtsam would raise)
    return {int(i): x[k].copy() for k, i in enumerate(cams) if np.all(np.isfinite(x[k]))}
