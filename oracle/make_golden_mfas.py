"""Writes the fixtures of 1DSfM's outlier rejection (oracle/mfas_ref.py):

    tests/golden/mfas_scenes.npz     seeded kNN camera graphs with 10-30 % outlier directions, with and without track
        landmarks, under each of the three sampling methods; a single edge, a tree, disconnected components; weights of
        exactly 0 and below 1e-8; a graph of exact ratio ties; no measurement; one direction
    tests/golden/mfas_lund_door.npz  lund-door's post-ISP i2Ui1 (tests/golden/twoview_report_lund_door.npz) in perturbed
        ground-truth rotations with camera 11 without one, and the 672 tracks of tests/golden/data_assoc_lund_door.npz through
        the reference's track selection and landmark directions, under SAMPLE_INPUT_MEASUREMENTS (onedsfm_front_end.yaml)

    python -m oracle.make_golden_mfas --reference /path/to/gtsfm-checkout

Stored per scene, under "<name>/": cam_keys (nc, 2) (i1, i2) and cam_vecs (nc, 3), trk_keys (nt, 2) (j, i) and trk_vecs
(nt, 3), in dict order; the sampling method; the directions dirs (K, 3) the reference's sampler drew after np.random.seed(0);
the dense problem V, edge_a, edge_b, meas (map order) and perm (edge e is measurement perm[e]); weight_sum (E,) in map
order; and the outputs inlier_cam (nc,), inlier_trk (nt,), inlier_cameras.

Before writing, every scene is run through the reference's own TranslationAveraging1DSFM.compute_inliers (and, for
lund-door, get_valid_measurements_in_world_frame, _select_tracks_for_averaging and _get_landmark_directions), from the
checkout's sources under stand-ins: gtsam.MFAS is mfas_ref.mfas_literal, Unit3 normalises as Eigen does, symbol_shorthand
builds the 64-bit keys, Rot3 and Cal3Bundler provide rotate and calibrate, Dask's delayed / compute are the identity and
get_client raises ValueError.  The reference's own per-edge sums (its defaultdict) and outputs must equal the restatement's.
"""
from __future__ import annotations

import argparse
import sys
import types
import typing
from collections import defaultdict
from enum import Enum
from pathlib import Path

import numpy as np

from oracle import mfas_ref as mr
from oracle.make_golden_data_assoc import _module_body, lund_matches

ROOT = Path(__file__).resolve().parents[1]
OUT_SCENES = ROOT / "tests/golden/mfas_scenes.npz"
OUT_LUND = ROOT / "tests/golden/mfas_lund_door.npz"
METHODS = (mr.SAMPLE_INPUT_MEASUREMENTS, mr.SAMPLE_WITH_UNIFORM_DENSITY, mr.SAMPLE_WITH_INPUT_DENSITY)


# ---- scenes -------------------------------------------------------------------------------------------------------------------
def knn_graph(rng, n, k, outlier_frac, n_landmarks=0, views=(2, 5)):
    """Camera centres in a ring with height; pairs (i1 < i2) of each camera's k nearest; w_i2Ui1 the true direction from
    c_i2 to c_i1, a random one for `outlier_frac` of them.  Landmarks seen by 2-5 cameras: w_iUj from c_i to X_j."""
    a = 2 * np.pi * np.arange(n) / n
    c = np.stack([10 * np.cos(a), rng.normal(0, 1.0, n), 10 * np.sin(a)], 1) + rng.normal(0, 0.3, (n, 3))
    dist = np.linalg.norm(c[:, None] - c[None], axis=2)
    pairs = sorted({(min(i, j), max(i, j)) for i in range(n) for j in np.argsort(dist[i])[1:k + 1]})
    cam = {}
    for i1, i2 in pairs:
        v = c[i1] - c[i2]
        cam[(int(i1), int(i2))] = mr.unit3(rng.normal(size=3) if rng.random() < outlier_frac else v)
    trk = {}
    for j in range(n_landmarks):
        X = rng.normal(0, 4.0, 3)
        for i in sorted(rng.choice(n, rng.integers(views[0], views[1] + 1), replace=False)):
            v = X - c[i]
            trk[(j, int(i))] = mr.unit3(rng.normal(size=3) if rng.random() < outlier_frac else v)
    return cam, trk


def scenes(seed=0):
    rng = np.random.default_rng(seed)
    out = {}
    for m, tag in zip(METHODS, ("input", "uniform", "kde")):
        out[f"knn_{tag}"] = (m, *knn_graph(rng, 24, 4, 0.2))
        out[f"knn_tracks_{tag}"] = (m, *knn_graph(rng, 18, 4, 0.25, n_landmarks=20))
    out["knn_outliers_10"] = (mr.SAMPLE_WITH_UNIFORM_DENSITY, *knn_graph(rng, 30, 5, 0.1))
    out["knn_outliers_30"] = (mr.SAMPLE_INPUT_MEASUREMENTS, *knn_graph(rng, 30, 5, 0.3, n_landmarks=15))
    out["single_edge"] = (mr.SAMPLE_WITH_UNIFORM_DENSITY, {(0, 1): mr.unit3(np.array([0.3, -0.2, 0.9]))}, {})
    tree = {(int(p), int(i)): mr.unit3(rng.normal(size=3)) for i in range(1, 12) for p in [rng.integers(0, i)]}
    out["tree"] = (mr.SAMPLE_WITH_UNIFORM_DENSITY, tree, {})
    c1, t1 = knn_graph(rng, 10, 3, 0.2, n_landmarks=6)
    c2, _ = knn_graph(rng, 8, 3, 0.2)
    out["disconnected"] = (mr.SAMPLE_INPUT_MEASUREMENTS, {**c1, **{(i1 + 20, i2 + 20): v for (i1, i2), v in c2.items()}}, t1)
    # exact zeros: axis directions, each perpendicular to the directions the sampler draws from the others; and a weight
    # of about 1e-9 from a measurement a hair off the y-z plane
    ax = [np.array(v, float) for v in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (-1, 0, 0), (0, -1, 0))]
    zero = {(i1, i2): ax[(i1 + 2 * i2) % 5] for i1 in range(6) for i2 in range(i1 + 1, 6) if (i1 + i2) % 3}
    zero[(0, 3)] = mr.unit3(np.array([1e-9, 1.0, 0.5]))
    out["zero_weights"] = (mr.SAMPLE_INPUT_MEASUREMENTS, zero, {(0, 1): ax[2], (0, 4): mr.unit3(np.array([-1e-9, 0.0, 1.0]))})
    # a directed 4-cycle and a 6-cycle of unit weights along +-x: with d = +-x every node has in = out = 1, all ratios tie
    tie = {(0, 1): ax[0], (1, 2): ax[0], (2, 3): ax[0], (0, 3): ax[3], (4, 5): ax[3], (5, 6): ax[3], (6, 7): ax[3],
           (7, 8): ax[3], (8, 9): ax[3], (4, 9): ax[0], (1, 5): ax[1]}
    out["ratio_ties"] = (mr.SAMPLE_INPUT_MEASUREMENTS, tie, {})
    out["empty"] = (mr.SAMPLE_WITH_UNIFORM_DENSITY, {}, {})  # with no measurement to sample from, the reference raises
    out["one_direction"] = (mr.SAMPLE_INPUT_MEASUREMENTS, {(2, 5): mr.unit3(np.array([0.1, 0.2, -0.97]))}, {})
    return out


def large_scene(n, k=30, per_cam=12, seed=7):
    """A kNN camera graph of n cameras with 20 % outlier directions, and landmarks: each camera starts per_cam / 4 tracks
    seen by 3-6 of its neighbours, about per_cam track directions per camera (the reference's 12 per camera).  For the
    device tests and profiles/bench_mfas.py: too large for the literal oracle."""
    rng = np.random.default_rng(seed)
    c = rng.normal(0, 10, (n, 3))
    from scipy.spatial import cKDTree

    _, nb = cKDTree(c).query(c, k + 1)
    pairs = np.unique(np.sort(np.stack([np.repeat(np.arange(n), k), nb[:, 1:].ravel()], 1), axis=1), axis=0)
    cam = {(int(a), int(b)): mr.unit3(c[a] - c[b]) for a, b in pairs}
    trk, j = {}, 0
    for i in range(n):
        for _ in range(per_cam // 4):
            X = c[i] + rng.normal(0, 3, 3)
            for v in set(nb[i, :rng.integers(3, 7)].tolist()):
                trk[(j, v)] = mr.unit3(X - c[v])
            j += 1
    for key in list(cam)[:: 5]:
        cam[key] = mr.unit3(rng.normal(size=3))
    return cam, trk



# ---- the reference's own code under stand-ins ---------------------------------------------------------------------------------
class _Unit3:
    def __init__(self, p=None):
        self._p = mr.unit3(np.asarray(p, float).reshape(3))

    def point3(self):
        return self._p


class _Rot3:
    def __init__(self, R):
        self.R = np.asarray(R, float).reshape(3, 3)

    def rotate(self, p):  # Eigen's R * p: column by column
        p = np.asarray(p, float)
        return (self.R[:, 0] * p[0] + self.R[:, 1] * p[1]) + self.R[:, 2] * p[2]


class _Cal3Bundler:
    def __init__(self, f, u0, v0):
        self.f, self.u0, self.v0 = f, u0, v0

    def calibrate(self, uv):
        return np.array([(uv[0] - self.u0) / self.f, (uv[1] - self.v0) / self.f])


class _Binary:
    def __init__(self, k1, k2, m, noise=None):
        self.k = (int(k1), int(k2))
        self.m = m

    def key1(self):
        return self.k[0]

    def key2(self):
        return self.k[1]

    def measured(self):
        return self.m


class _MFAS:
    def __init__(self, measurements, d):
        self.ms = [(b.key1(), b.key2(), b.measured().point3()) for b in measurements]
        self.d = d.point3()

    def computeOutlierWeights(self):  # noqa: N802 - gtsam's name
        return mr.mfas_literal(self.ms, self.d)[1]


class _Anything:  # stands in for names that appear only in annotations and unused defaults
    def __getattr__(self, name):
        return self

    def __getitem__(self, k):
        return self

    def __call__(self, *a, **k):
        return self


class _Sums(defaultdict):  # the reference's outlier_weights_sum, kept for the pin
    last = None

    def __init__(self, *a):
        super().__init__(*a)
        _Sums.last = self


def _no_client():
    raise ValueError("no Dask client")


def _reference(reference: Path):
    g = reference / "gtsfm"
    any_ = _Anything()
    base = {"np": np, "Enum": Enum, **{k: getattr(typing, k) for k in typing.__all__}}
    conv = _module_body(g / "utils/coordinate_conversions.py", dict(base, Unit3=_Unit3))
    from scipy import stats

    sampling = _module_body(g / "utils/sampling.py", dict(base, Unit3=_Unit3, stats=stats,
                                                           conversion_utils=types.SimpleNamespace(**conv)))
    st = _module_body(g / "common/sfm_track.py", dict(base))
    gtsam = types.SimpleNamespace(noiseModel=any_, MFAS=_MFAS, Values=any_)
    ns = dict(base, gtsam=gtsam, MFAS=_MFAS, BinaryMeasurementUnit3=_Binary, BinaryMeasurementsUnit3=list, Unit3=_Unit3, Rot3=_Rot3,
              Point3=lambda x, y, z: np.array([x, y, z], float), Pose3=any_, BinaryMeasurementPoint3=any_, BinaryMeasurementsPoint3=any_,
              TranslationRecovery=any_, symbol_shorthand=types.SimpleNamespace(A=mr.C, B=mr.L),
              TranslationAveragingBase=type("TranslationAveragingBase", (), {"__init__": lambda self, r=True: setattr(
                  self, "_robust_measurement_noise", r)}),
              dask=types.SimpleNamespace(delayed=lambda f: f, compute=lambda *xs: xs), get_client=_no_client,
              defaultdict=_Sums, DefaultDict=typing.DefaultDict, gtsfm_types=any_, logger_utils=types.SimpleNamespace(get_logger=lambda: any_),
              metrics_utils=any_, sampling_utils=types.SimpleNamespace(**sampling), PosePrior=any_, SfmTrack2d=st["SfmTrack2d"],
              GtsfmMetric=any_, GtsfmMetricsGroup=any_, AnnotatedGraph=any_, ImageIndexPair=any_, ImageIndexPairs=any_, align=any_,
              transform=any_, time=__import__("time"), timeit=__import__("timeit"))
    return _module_body(g / "averaging/translation/averaging_1dsfm.py", ns), st


def _method(r, m):
    return r["TranslationAveraging1DSFM"].ProjectionSamplingMethod(m)


def solve(r, method, cam, trk):
    """The reference's compute_inliers and the restatement on the same directions: both must agree."""
    obj = r["TranslationAveraging1DSFM"](projection_sampling_method=_method(r, method))  # np.random.seed(0)
    cu = {k: _Unit3(v) for k, v in cam.items()}
    tu = {k: _Unit3(v) for k, v in trk.items()}
    cam, trk = {k: u.point3() for k, u in cu.items()}, {k: u.point3() for k, u in tu.items()}  # as the Unit3s hold them
    combined = list(cu.values()) + list(tu.values())
    dirs = np.array([d.point3() for d in obj._TranslationAveraging1DSFM__sample_projection_directions(combined)]).reshape(-1, 3)
    obj = r["TranslationAveraging1DSFM"](projection_sampling_method=_method(r, method))  # the same draw again, inside the call
    _Sums.last = None
    ref_cam, ref_trk, ref_ic = obj.compute_inliers(cu, tu)
    (my_cam, my_trk, my_ic), s = mr.compute_inliers(cam, trk, dirs, form="literal")
    assert set(ref_cam) == set(my_cam) and set(ref_trk) == set(my_trk) and ref_ic == my_ic
    p = {}
    if cam or trk:
        keys, ea, eb, meas, perm = mr.dense_problem(mr.measurements_from_dicts(cam, trk))
        ref_sum = np.array([_Sums.last[(int(keys[a]), int(keys[b]))] for a, b in zip(ea, eb)]) if len(dirs) else np.zeros(len(ea))
        assert np.array_equal(ref_sum, s), "the reference's own sums differ from the restatement's"
        assert np.array_equal(mr.outlier_weight_sums(len(keys), ea, eb, meas, dirs), s), "vectorised != literal"
        p = dict(V=np.array(len(keys)), edge_a=ea, edge_b=eb, meas=meas, perm=perm)
    inl_c = np.array([k in my_cam for k in cam], bool)
    inl_t = np.array([k in my_trk for k in trk], bool)
    return dict(cam_keys=np.array(list(cam), np.int64).reshape(-1, 2), cam_vecs=np.array(list(cam.values()), float).reshape(-1, 3),
                trk_keys=np.array(list(trk), np.int64).reshape(-1, 2), trk_vecs=np.array(list(trk.values()), float).reshape(-1, 3),
                method=np.array(method), dirs=dirs, weight_sum=s, inlier_cam=inl_c, inlier_trk=inl_t,
                inlier_cameras=np.array(sorted(my_ic), np.int64), **p)


def lund_inputs(r, st, seed=5):
    """lund-door through the reference's get_valid_measurements_in_world_frame, _select_tracks_for_averaging and
    _get_landmark_directions: -> (w_i2Ui1 dict, w_iUj dict) of unit vectors."""
    z = np.load(ROOT / "tests/golden/twoview_report_lund_door.npz")
    _, _, cams = lund_matches()
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(seed)
    wRi = []
    for i in range(12):
        dR = Rotation.from_rotvec(rng.normal(0, np.radians(1.0), 3)).as_matrix()
        wRi.append(_Rot3(dR @ cams[i, :9].reshape(3, 3)))
    wRi[11] = None  # the last camera: only ever i2, so its pairs drop out and no track direction needs its rotation
    i2Ui1 = {(int(a) - 1, int(b) - 1): _Unit3(z[f"{a}_{b}/t_post"]) if bool(z[f"{a}_{b}/post_pose"]) else None
             for a, b in z["pairs"] if bool(z[f"{a}_{b}/isp_ok"])}  # no pose after BA: the reference's None, skipped
    da = np.load(ROOT / "tests/golden/data_assoc_lund_door.npz")
    off, mc, uv = da["uniform_10px_100/track_off"], da["uniform_10px_100/meas_cam"], da["uniform_10px_100/meas_uv"]
    SfmTrack2d, SfmMeasurement = st["SfmTrack2d"], st["SfmMeasurement"]
    tracks = [SfmTrack2d([SfmMeasurement(int(mc[m]), uv[m]) for m in range(off[t], off[t + 1])]) for t in range(len(off) - 1)]
    assert len(tracks) == 672
    intr = [_Cal3Bundler(*cams[i, 12:]) for i in range(12)]
    obj = r["TranslationAveraging1DSFM"](projection_sampling_method=_method(r, mr.SAMPLE_INPUT_MEASUREMENTS))
    w_cam, valid = r["get_valid_measurements_in_world_frame"](i2Ui1, wRi)
    sel = obj._select_tracks_for_averaging(tracks, valid, intr)
    w_trk = obj._get_landmark_directions(sel, intr, wRi)
    return {k: v.point3() for k, v in w_cam.items()}, {k: v.point3() for k, v in w_trk.items()}, len(sel)


def _store(path, results):
    arrays = {"names": np.array(list(results))}
    for name, res in results.items():
        arrays.update({f"{name}/{k}": v for k, v in res.items()})
        print(name, len(res["cam_keys"]), len(res["trk_keys"]), len(res["dirs"]), int((~res["inlier_cam"]).sum()), "camera outliers")
    np.savez_compressed(path, **arrays)
    print(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, required=True, help="a GTSfM checkout (the pinned functions)")
    args = ap.parse_args()
    r, st = _reference(args.reference)
    results = {name: solve(r, m, cam, trk) for name, (m, cam, trk) in scenes().items()}
    cam, trk, nsel = lund_inputs(r, st)
    print(f"lund-door: {len(cam)} camera directions, {nsel} selected tracks, {len(trk)} track directions")
    lund = {"lund_door": solve(r, mr.SAMPLE_INPUT_MEASUREMENTS, cam, trk)}
    print(f"restatement equals the reference's compute_inliers (outputs and per-edge sums) on {len(results) + 1} scenes")
    _store(OUT_SCENES, results)
    _store(OUT_LUND, lund)


if __name__ == "__main__":
    sys.exit(main())
