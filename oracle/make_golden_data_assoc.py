"""Writes the fixtures of data association's triangulation (oracle/data_assoc_ref.py):

    tests/golden/data_assoc_scenes.npz     seeded scenes: cameras (R_wTi, t_wTi, f, u0, v0) on a ring around the points,
        some without a pose, and tracks of points seen by random subsets of the cameras, with pixel noise and optional
        outlier measurements
    tests/golden/data_assoc_lund_door.npz  lund-door's tracks: the union-find of the post-ISP correspondences of its 66
        pairs (tests/golden/twoview_report_lund_door.npz), triangulated in the ground-truth world cameras with a seeded
        perturbation and one camera dropped, under deep_front_end.yaml's options and under NO_RANSAC

    python -m oracle.make_golden_data_assoc --reference /path/to/gtsfm-checkout

Stored per scene, under "<name>/": track_off, meas_cam, meas_uv, cams, cam_valid, the options (mode 0 NO_RANSAC /
1 RANSAC_SAMPLE_UNIFORM, num_hypotheses, threshold, min_angle, seed) and the oracle's exit, point, avg, inlier.

Before writing, the restatement is pinned against the reference's own code, run from the checkout's sources
(_pin_against_reference): DataAssociation.run_triangulation, Point3dInitializer.triangulate / execute_ransac_variant,
compute_point_reprojection_errors, get_max_triangulation_angle, SfmTrack2d, and DsfTracksEstimator.run for the lund-door
tracks.  Stand-ins: gtsam.triangulatePoint3 is the restatement (raising RuntimeError where it fails), cameras provide
projectSafe and pose().translation(), camera sets and Point2Vector are lists, SfmTrack / Unit3 / DSFMapIndexPair are
small classes, Dask's delayed / compute are the identity, and np.random.choice returns the restated sampler's draw.
"""
from __future__ import annotations

import argparse
import ast
import itertools
import logging
import sys
import time
import types
import typing
from collections import Counter
from dataclasses import dataclass
from enum import Enum
from pathlib import Path

import numpy as np

from oracle import data_assoc_ref as da

ROOT = Path(__file__).resolve().parents[1]
OUT_SCENES = ROOT / "tests/golden/data_assoc_scenes.npz"
OUT_LUND = ROOT / "tests/golden/data_assoc_lund_door.npz"
# deep_front_end.yaml's data association: RANSAC_SAMPLE_UNIFORM, 10 px, max_num_hypotheses 100
CONFIG_HYPS = da.num_ransac_hypotheses(max_num_hypotheses=100)


def look_at(centre, target):
    z = target - centre
    z = z / np.linalg.norm(z)
    x = np.cross([0.0, 1.0, 0.0], z)
    x = x / np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], 1)  # columns: camera axes in the world (R_wTi)


def ring_cameras(rng, n, radius=10.0, f=600.0, u0=320.0, v0=240.0):
    cams = np.zeros((n, 15))
    for i in range(n):
        a = 2 * np.pi * i / n + rng.normal(0, 0.02)
        c = np.array([radius * np.cos(a), rng.normal(0, 0.5), radius * np.sin(a)])
        cams[i, :9] = look_at(c, rng.normal(0, 0.3, 3)).ravel()
        cams[i, 9:12] = c
        cams[i, 12:] = f, u0, v0
    return cams


def project(cam, X):
    R, t = cam[:9].reshape(3, 3), cam[9:12]
    pc = R.T @ (X - t)
    return np.array([cam[13] + cam[12] * pc[0] / pc[2], cam[14] + cam[12] * pc[1] / pc[2]]), pc[2]


def make_tracks(rng, cams, lengths, noise=0.5, outlier_frac=0.0, behind=False):
    tracks = []
    for n in lengths:
        X = rng.normal(0, 1.5, 3)
        imgs = rng.choice(len(cams), size=n, replace=False)
        t = []
        for i in imgs:
            uv, _ = project(cams[i], X)
            uv = uv + rng.normal(0, noise, 2)
            if rng.random() < outlier_frac:
                uv = uv + rng.uniform(30, 200, 2) * rng.choice([-1, 1], 2)
            t.append((int(i), uv))
        if behind:  # the point mirrored through the first camera: behind it, in front of none of the others' ray
            i0 = t[0][0]
            Xb = 2 * cams[i0, 9:12] - X
            t = [(i, project(cams[i], Xb)[0] + rng.normal(0, noise, 2)) for i, _ in t]
        tracks.append(t)
    return tracks


def geometric_lengths(rng, T, p=0.35, lo=2, hi=40):
    return np.clip(lo + rng.geometric(p, T) - 1, lo, hi)


def scenes(seed=0):
    rng = np.random.default_rng(seed)
    out = {}

    def add(name, cams, valid, tracks, mode, hyps=CONFIG_HYPS, thr=10.0, min_angle=0.0, s=7):
        off, cam, uv = da.pack_tracks(tracks)
        out[name] = dict(track_off=off, meas_cam=cam, meas_uv=uv, cams=cams, cam_valid=np.asarray(valid, np.uint8),
                         options=np.array([1.0 if mode == da.SAMPLE_UNIFORM else 0.0, hyps, thr, min_angle, s]))

    cams = ring_cameras(rng, 60)
    valid = np.ones(60, np.uint8)
    clean = make_tracks(rng, cams, list(range(2, 41)) + list(geometric_lengths(rng, 200)))
    add("clean_uniform", cams, valid, clean, da.SAMPLE_UNIFORM)
    add("clean_no_ransac", cams, valid, clean, da.NO_RANSAC)
    for frac in (0.1, 0.3):
        tr = make_tracks(rng, cams, list(geometric_lengths(rng, 250, 0.25)), outlier_frac=frac)
        add(f"outliers_{int(frac * 100)}", cams, valid, tr, da.SAMPLE_UNIFORM)
    boundary = make_tracks(rng, cams, [14] * 12 + [15] * 12 + [16] * 4, outlier_frac=0.2)
    add("boundary_14_15", cams, valid, boundary, da.SAMPLE_UNIFORM, hyps=91)  # C(14, 2) = 91: 14 exhaustive, 15 sampled
    add("boundary_config", cams, valid, boundary, da.SAMPLE_UNIFORM)
    missing = valid.copy()
    missing[rng.choice(60, 15, replace=False)] = 0
    tr = make_tracks(rng, cams, list(geometric_lengths(rng, 200, 0.3)), outlier_frac=0.1)
    add("missing_uniform", cams, missing, tr, da.SAMPLE_UNIFORM)
    add("missing_no_ransac", cams, missing, tr, da.NO_RANSAC)
    add("missing_no_ransac_inf", cams, missing, tr, da.NO_RANSAC, thr=np.inf)
    tr = make_tracks(rng, cams, [2, 3, 4, 5] * 10, behind=True)
    add("behind", cams, valid, tr, da.NO_RANSAC, thr=np.inf)
    add("behind_uniform", cams, valid, tr, da.SAMPLE_UNIFORM, thr=np.inf)
    coinc = cams.copy()
    coinc[1:6, 9:12] = coinc[0, 9:12]  # cameras 0-5 share a centre: their DLT is rank-deficient
    tr = [[(i, project(coinc[i], np.array([0.3, 0.1, 0.2]) * k)[0]) for i in range(6)] for k in range(1, 8)]
    tr += make_tracks(rng, coinc, [3, 4, 6] * 5)
    add("coincident_centres", coinc, valid, tr, da.NO_RANSAC, thr=np.inf)
    add("coincident_centres_uniform", coinc, valid, tr, da.SAMPLE_UNIFORM)
    tr = make_tracks(rng, cams, list(geometric_lengths(rng, 150, 0.4)))
    add("min_angle", cams, valid, tr, da.SAMPLE_UNIFORM, min_angle=30.0)
    add("min_angle_no_ransac", cams, valid, tr, da.NO_RANSAC, thr=np.inf, min_angle=60.0)
    add("inf_threshold", cams, valid, make_tracks(rng, cams, list(geometric_lengths(rng, 100)), outlier_frac=0.2),
        da.SAMPLE_UNIFORM, thr=np.inf)
    add("empty", cams, valid, [], da.SAMPLE_UNIFORM)
    add("all_missing", cams, np.zeros(60, np.uint8), make_tracks(rng, cams, [2, 3, 7]), da.SAMPLE_UNIFORM)
    return out


def solve(sc):
    o = sc["options"]
    mode = da.SAMPLE_UNIFORM if o[0] else da.NO_RANSAC
    return da.run_arrays(sc["track_off"], sc["meas_cam"], sc["meas_uv"], sc["cams"], sc["cam_valid"], mode, int(o[1]), float(o[2]),
                         float(o[3]), int(o[4]))


# ---- lund-door -------------------------------------------------------------------------------------------------------------
def lund_matches():
    """{(i1, i2): post-ISP correspondence rows (k1, k2)} of the pairs that pass inlier support, and every image's keypoints,
    with 0-based image indices."""
    z = np.load(ROOT / "tests/golden/twoview_report_lund_door.npz")
    kps = [z[f"kp_{i}"].astype(np.float64) for i in range(1, 13)]
    matches, cams = {}, np.zeros((12, 15))
    for a, b in z["pairs"]:
        key = f"{a}_{b}"
        cams[a - 1], cams[b - 1] = z[f"{key}/cam1"], z[f"{key}/cam2"]
        if bool(z[f"{key}/isp_ok"]):
            matches[(int(a) - 1, int(b) - 1)] = z[f"{key}/isp/v_corr_idxs"].astype(np.int64)
    return matches, kps, cams


def union_find_tracks(matches, kps):
    """DsfTracksEstimator.run: the connected components of the (image, keypoint) pairs joined by the correspondences, each
    a track of its measurements, without the tracks that hold two measurements of one image.  Tracks are ordered by
    their smallest (image, keypoint), measurements by (image, keypoint)."""
    parent = {}

    def find(x):
        while parent.setdefault(x, x) != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for (i1, i2), rows in matches.items():
        for k1, k2 in rows:
            a, b = find((i1, int(k1))), find((i2, int(k2)))
            if a != b:
                parent[max(a, b)] = min(a, b)
    sets = {}
    for x in list(parent):
        sets.setdefault(find(x), []).append(x)
    tracks = []
    for members in sorted(sorted(m) for m in sets.values()):
        if len({i for i, _ in members}) == len(members):
            tracks.append([(i, kps[i][k]) for i, k in members])
    return tracks


def lund_scenes(seed=3):
    matches, kps, cams = lund_matches()
    tracks = union_find_tracks(matches, kps)
    rng = np.random.default_rng(seed)
    from scipy.spatial.transform import Rotation

    pert = cams.copy()  # standing in for averaging's output: 0.2 degrees and 1 cm of noise per camera, camera 6 dropped
    for i in range(12):
        dR = Rotation.from_rotvec(rng.normal(0, np.radians(0.2), 3)).as_matrix()
        pert[i, :9] = (dR @ cams[i, :9].reshape(3, 3)).ravel()
        pert[i, 9:12] = cams[i, 9:12] + rng.normal(0, 0.01, 3)
    valid = np.ones(12, np.uint8)
    valid[6] = 0
    off, cam, uv = da.pack_tracks(tracks)
    base = dict(track_off=off, meas_cam=cam, meas_uv=uv, cams=pert, cam_valid=valid)
    return {"uniform_10px_100": dict(base, options=np.array([1.0, CONFIG_HYPS, 10.0, 0.0, 0])),
            "no_ransac_10px": dict(base, options=np.array([0.0, CONFIG_HYPS, 10.0, 0.0, 0]))}, matches, kps


# ---- the reference's own code under stand-ins ---------------------------------------------------------------------------------
def _module_body(path: Path, ns: dict, names=None, skip=()) -> dict:
    """Executes a module's top-level definitions (not its imports; only `names` when given; not `skip`) in `ns`."""
    for node in ast.parse(path.read_text()).body:
        if isinstance(node, (ast.Import, ast.ImportFrom)):
            continue
        name = node.name if isinstance(node, (ast.FunctionDef, ast.ClassDef)) else \
            next((t.id for t in getattr(node, "targets", []) if isinstance(t, ast.Name)), None)
        if (names is not None and name not in names) or name in skip:
            continue
        exec(compile(ast.Module([node], []), str(path), "exec"), ns)
    return ns


class _Unit3:
    def __init__(self, p):
        p = np.asarray(p, float)
        self._p = p / np.linalg.norm(p)

    def point3(self):
        return self._p


class _Pose:
    def __init__(self, t):
        self._t = t

    def translation(self):
        return self._t


class _Camera:
    """PinholeCameraCal3Bundler without distortion: projectSafe (uv, depth > 0) and pose().translation()."""

    def __init__(self, c):
        self.c = da.camera(c[:9], c[9:12], c[12], c[13], c[14])

    def projectSafe(self, p):  # noqa: N802 - gtsam's name
        uv, z, *_ = da.tv.project(*self.c, np.asarray(p, float))
        return uv, bool(z > 0.0)

    def pose(self):
        return _Pose(self.c[1])

    def calibration(self):
        return None


class _SfmTrack:
    def __init__(self, p):
        self.p, self.m = np.asarray(p, float), []

    def addMeasurement(self, i, uv):  # noqa: N802
        self.m.append((int(i), np.asarray(uv, float)))

    def numberMeasurements(self):  # noqa: N802
        return len(self.m)

    def measurement(self, k):
        return self.m[k]

    def point3(self):
        return self.p


def _triangulate_point3(cameras, measurements, rank_tol, optimize):
    assert rank_tol == da.tv.DLT_RANK_TOL and optimize
    X = da.triangulate_point3([c.c for c in cameras], [np.asarray(u, float) for u in measurements])
    if X is None:
        raise RuntimeError("triangulation failed")
    return X


class _DSFMapIndexPair:
    def __init__(self):
        self.parent = {}

    def _find(self, x):
        while self.parent.setdefault(x, x) != x:
            x = self.parent[x]
        return x

    def merge(self, a, b):
        ra, rb = self._find(a), self._find(b)
        if ra != rb:
            self.parent[ra] = rb

    def sets(self):
        out = {}
        for x in list(self.parent):
            out.setdefault(self._find(x), set()).add(x)
        return out


class _IndexPair(tuple):
    def __new__(cls, i, j):
        return super().__new__(cls, (int(i), int(j)))

    def i(self):
        return self[0]

    def j(self):
        return self[1]


def _reference(reference: Path, draw):
    g = reference / "gtsfm"
    log = logging.getLogger("data_assoc_pin")
    log.setLevel(logging.ERROR)  # the reference warns once per skipped camera
    base = {"np": np, "itertools": itertools, "sys": sys, "Enum": Enum, "time": time, "Counter": Counter, "dataclass": dataclass,
            "logger": log, **{k: getattr(typing, k) for k in typing.__all__}}
    st = _module_body(g / "common/sfm_track.py", dict(base))
    gtsam = types.SimpleNamespace(triangulatePoint3=_triangulate_point3, Point2Vector=list, SfmTrack=_SfmTrack, Unit3=_Unit3,
                                  PinholeCameraCal3Bundler=_Camera, DSFMapIndexPair=_DSFMapIndexPair, IndexPair=_IndexPair,
                                  IndexPairSetAsArray=sorted)
    gtsfm_types = types.SimpleNamespace(get_camera_set_class_for_calibration=lambda cal: list, CAMERA_TYPE=object,
                                        CAMERA_SET_TYPE=object)
    common = dict(base, gtsam=gtsam, gtsfm_types=gtsfm_types, SfmTrack=_SfmTrack, Unit3=_Unit3, PinholeCameraCal3Bundler=_Camera,
                  SfmMeasurement=st["SfmMeasurement"], SfmTrack2d=st["SfmTrack2d"], CAMERA_TYPE=object)
    reproj = _module_body(g / "utils/reprojection.py", dict(common))
    geom = _module_body(g / "utils/geometry_comparisons.py", dict(common), names={"compute_relative_unit_translation_angle"})
    mvs = _module_body(g / "densify/mvs_utils.py", dict(common, geometry_utils=types.SimpleNamespace(**geom)),
                       names={"calculate_triangulation_angle_in_degrees"})
    tracks = _module_body(g / "utils/tracks.py", dict(common, calculate_triangulation_angle_in_degrees=mvs["calculate_triangulation_angle_in_degrees"]),
                          names={"get_max_triangulation_angle"})
    np_proxy = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith("__")})
    np_proxy.random = types.SimpleNamespace(choice=draw)
    p3d = _module_body(g / "data_association/point3d_initializer.py", dict(common, np=np_proxy,
                                                                            reproj_utils=types.SimpleNamespace(**reproj)), skip=("logger",))
    assoc = _module_body(g / "data_association/data_assoc.py", dict(
        common, GTSFMProcess=object, UiMetadata=object, Delayed=object, GtsfmData=object, Image=object, PosePrior=object,
        GtsfmMetric=object, GtsfmMetricsGroup=object, io_utils=None, track_utils=None, os=None,
        dask_delayed=lambda f: f, dask_compute=lambda *xs: xs, Point3dInitializer=p3d["Point3dInitializer"],
        TriangulationExitCode=p3d["TriangulationExitCode"], TriangulationOptions=p3d["TriangulationOptions"]), skip=("logger",))
    dsf = _module_body(g / "data_association/dsf_tracks_estimator.py", dict(common, TracksEstimatorBase=object, Keypoints=object),
                       skip=("logger",))
    # triangulate() imports gtsfm.utils.tracks inside the function
    mods = {"gtsfm": types.ModuleType("gtsfm"), "gtsfm.utils": types.ModuleType("gtsfm.utils"),
            "gtsfm.utils.tracks": types.ModuleType("gtsfm.utils.tracks")}
    mods["gtsfm.utils.tracks"].get_max_triangulation_angle = tracks["get_max_triangulation_angle"]
    mods["gtsfm"].utils, mods["gtsfm.utils"].tracks = mods["gtsfm.utils"], mods["gtsfm.utils.tracks"]
    return types.SimpleNamespace(st=st, p3d=p3d, assoc=assoc, dsf=dsf, modules=mods)


def _pin_scene(r, state, name, sc, res):
    o = sc["options"]
    mode = r.p3d["TriangulationSamplingMode"]("RANSAC_SAMPLE_UNIFORM" if o[0] else "NO_RANSAC")
    opts = r.p3d["TriangulationOptions"](mode, reproj_error_threshold=float(o[2]), min_triangulation_angle=float(o[3]),
                                         max_num_hypotheses=int(o[1]))
    assert opts.num_ransac_hypotheses() == int(o[1]) or not o[0], name
    state["seed"] = int(o[4])
    off = sc["track_off"]
    tracks = [r.st["SfmTrack2d"]([r.st["SfmMeasurement"](int(sc["meas_cam"][m]), sc["meas_uv"][m]) for m in range(off[t], off[t + 1])])
              for t in range(len(off) - 1)]
    cameras = {i: _Camera(c) for i, c in enumerate(sc["cams"]) if sc["cam_valid"][i]}
    ex, pt, avg, inl = res
    DA = r.assoc["DataAssociation"]
    state["track"] = 0
    s_ref, e_ref, c_ref = DA(min_track_len=2, triangulation_options=opts).run_triangulation(cameras, tracks)
    if not cameras or not tracks:  # the reference returns empty lists (so does B200DataAssociation.run_triangulation)
        assert (s_ref, e_ref, c_ref) == ([], [], []), name
        return
    assert [c.value for c in c_ref] == ex.tolist(), name
    init = r.p3d["Point3dInitializer"](cameras, opts)
    for t, tr in enumerate(tracks):
        a, b = off[t], off[t + 1]
        if o[0]:
            state["track"] = t
            assert np.array_equal(init.execute_ransac_variant(tr), inl[a:b].astype(bool)), (name, t)
        if e_ref[t] is None or np.isnan(e_ref[t]):
            assert np.isnan(avg[t]), (name, t)
        else:
            assert abs(e_ref[t] - avg[t]) <= 1e-12 * max(1.0, abs(avg[t])), (name, t)
        if s_ref[t] is not None:
            assert np.allclose(s_ref[t].point3(), pt[t], rtol=1e-12, atol=1e-12), (name, t)
            kept = [m[0] for m in s_ref[t].m]
            assert kept == [int(sc["meas_cam"][m]) for m in range(a, b) if inl[m]], (name, t)


def _pin_against_reference(reference: Path, cases: dict, results: dict, matches, kps) -> None:
    """The restatement equals the reference's code, run from the checkout's sources under the stand-ins above."""
    state = {"seed": 0, "track": 0}

    def draw(n, size, replace, p):  # np.random.choice in sample_ransac_hypotheses: the restated sampler's draw
        assert not replace and np.allclose(p, 1.0 / n)
        out = da.sample_pairs(state["seed"], state["track"], n, size)
        state["track"] += 1
        return out

    r = _reference(reference, draw)
    assert r.p3d["SVD_DLT_RANK_TOL"] == da.tv.DLT_RANK_TOL and r.p3d["MAX_TRACK_REPROJ_ERROR"] == da.MAX_TRACK_REPROJ_ERROR
    saved = {k: sys.modules.get(k) for k in r.modules}
    sys.modules.update(r.modules)
    try:
        for name, sc in cases.items():
            _pin_scene(r, state, name, sc, results[name])
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    # DsfTracksEstimator.run on lund-door's correspondences: the same tracks as the union-find (as sets)
    kp = [types.SimpleNamespace(coordinates=k) for k in kps]
    ref_tracks = r.dsf["DsfTracksEstimator"]().run(matches, kp)
    mine = union_find_tracks(matches, kps)
    key = lambda t: sorted((int(i), float(uv[0]), float(uv[1])) for i, uv in t)  # noqa: E731
    assert sorted(key([(m.i, m.uv) for m in t.measurements]) for t in ref_tracks) == sorted(key(t) for t in mine)
    print(f"restatement equals the reference's run_triangulation, RANSAC and DSF tracks on {len(cases)} scenes "
          f"({len(mine)} lund-door tracks)")


def _store(path, cases, results):
    arrays = {}
    for name, sc in cases.items():
        ex, pt, avg, inl = results[name]
        arrays.update({f"{name}/{k}": v for k, v in dict(sc, exit=ex, point=pt, avg=avg, inlier=inl).items()})
        print(name, len(sc["track_off"]) - 1, np.bincount(ex.astype(np.int64), minlength=6) if len(ex) else [])
    np.savez_compressed(path, **arrays)
    print(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, required=True, help="a GTSfM checkout (the pinned functions)")
    args = ap.parse_args()
    cases = scenes()
    lund, matches, kps = lund_scenes()
    every = {**cases, **{f"lund_door_{k}": v for k, v in lund.items()}}
    results = {name: solve(sc) for name, sc in every.items()}
    _pin_against_reference(args.reference, every, results, matches, kps)
    _store(OUT_SCENES, cases, results)
    _store(OUT_LUND, lund, {k: results[f"lund_door_{k}"] for k in lund})


if __name__ == "__main__":
    main()
