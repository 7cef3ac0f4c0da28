"""Writes the fixtures of the global bundle adjustment (oracle/global_ba_ref.py):

    tests/golden/global_ba_scenes.npz     seeded scenes of 2-60 cameras: noisy tracks of 2-40 views with 10 % outlier
        measurements (Huber active), k1 / k2 starting at 0 and non-zero, a camera without a track, points behind a camera,
        HUBER and NONE, the Karcher gauge and the first-pose prior, sigma 1 and 2, exactly two cameras
    tests/golden/global_ba_lund_door.npz  the 672 tracks of tests/golden/data_assoc_lund_door.npz (uniform RANSAC at
        10 px) that triangulated, with their inlier measurements, in the valid cameras perturbed by seeded pose and focal
        noise

    python -m oracle.make_golden_global_ba [--reference /path/to/gtsfm-checkout]

Stored per scene, under "<name>/": the inputs cams (C, 17), points (N, 3), track_off (N + 1,), meas_cam (M,), meas_uv
(M, 2), params [noise_sigma, huber_k, gauge, max_iters, karcher_beta, pose_prior_sigma, f_sigma, k_sigma, k_sigma];
and the oracle's outputs cams_out, points_out, reproj_err, final_error, iterations, trace and trials (1 accepted,
0 rejected, 2 rejected with the lambda search stopped, -1 not positive definite).

With --reference, every scene first goes through the reference's own BundleAdjustmentOptimizer.run_ba and
run_ba_stage_with_filtering with its graph builders (gtsfm/bundle/bundle_adjustment.py), loaded from the checkout under
stand-ins: the factors and noise models record what they are given, Values is a dict, LevenbergMarquardtOptimizer runs
global_ba_ref on the recorded graph, and graph.error is global_ba_ref.cost.  GtsfmData (to_values, from_values,
filter_landmarks) is a stand-in here too: gtsfm/common/gtsfm_data.py imports gtsam, open3d-backed IO and the
reprojection utilities at module level, so it is not loaded; DESIGN.md lists it as unpinned.  The script asserts that
the reference's stage loop hands the input data to every stage, and that its outputs equal the restatement's.
"""
from __future__ import annotations

import argparse
import types
from pathlib import Path

import numpy as np

from oracle import global_ba_ref as gb
from oracle import twoview_ba_ref as tv

ROOT = Path(__file__).resolve().parents[1]
OUT_SCENES = ROOT / "tests/golden/global_ba_scenes.npz"
OUT_LUND = ROOT / "tests/golden/global_ba_lund_door.npz"
THRESHOLDS = (10.0, 5.0, 3.0)


def look_at(eye, target, up=np.array([0.0, -1.0, 0.0])):
    """wRc of a camera at `eye` whose optical axis (its z) points at `target`."""
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], 1)


def make_scene(seed, C, N, views=(2, 8), outlier=0.1, noise_px=0.7, dist=False, no_track_cam=False, behind=0,
               pose_noise=0.01, focal_noise=0.02, radius=6.0):
    """C cameras on an arc around the origin looking at it, N points near the origin, tracks of `views` measurements with
    `outlier` of them displaced by 20-60 px; the cameras and points perturbed.  -> dict of the problem arrays."""
    rng = np.random.default_rng(seed)
    cams = np.zeros((C, 17))
    for a in range(C):
        ang = 2.0 * np.pi * a / max(C, 3) * 0.5 - 0.8
        eye = np.array([radius * np.sin(ang), 0.5 * rng.normal(), -radius * np.cos(ang)])
        cams[a, :9] = look_at(eye, 0.2 * rng.normal(size=3)).ravel()
        cams[a, 9:12] = eye
        k1, k2 = (rng.uniform(-0.08, 0.08), rng.uniform(-0.02, 0.02)) if dist else (0.0, 0.0)
        cams[a, 12:] = [rng.uniform(450, 650), k1, k2, 320.0, 240.0]
    pts = rng.normal(size=(N, 3)) * 1.2
    ncam = C - 1 if no_track_cam else C
    toff, mcam, uv = [0], [], []
    for j in range(N):
        k = int(rng.integers(views[0], min(views[1], ncam) + 1))
        for a in sorted(rng.choice(ncam, size=k, replace=False)):
            u, *_ = tv.project(cams[a, :9].reshape(3, 3), cams[a, 9:12], cams[a, 12:], pts[j])
            u = u + rng.normal(size=2) * noise_px
            if rng.random() < outlier:
                ang = rng.uniform(0, 2 * np.pi)
                u = u + rng.uniform(20, 60) * np.array([np.cos(ang), np.sin(ang)])
            mcam.append(a)
            uv.append(u)
        toff.append(len(mcam))
    cams_n = cams.copy()
    for a in range(C):
        R, t = tv.retract_pose(cams[a, :9].reshape(3, 3), cams[a, 9:12], rng.normal(size=6) * pose_noise)
        cams_n[a, :9], cams_n[a, 9:12] = R.ravel(), t
        cams_n[a, 12] *= 1.0 + focal_noise * rng.normal()
    pts_n = pts + rng.normal(size=pts.shape) * 0.01
    for j in range(behind):  # a point moved behind its first camera
        a = mcam[toff[j]]
        R, t = cams_n[a, :9].reshape(3, 3), cams_n[a, 9:12]
        pc = R.T @ (pts_n[j] - t)
        pts_n[j] = t + R @ np.array([pc[0], pc[1], -0.5])
    return dict(cams=cams_n, points=pts_n, track_off=np.array(toff, np.int64), meas_cam=np.array(mcam, np.int32),
                meas_uv=np.array(uv, float))


def params_array(p: gb.Params):
    return np.array([p.noise_sigma, p.huber_k, p.gauge, p.max_iters, p.karcher_beta, p.pose_prior_sigma, *p.cal_prior_sigma])


def params_from(a) -> gb.Params:
    return gb.Params(float(a[0]), float(a[1]), int(a[2]), int(a[3]), float(a[4]), float(a[5]), tuple(float(x) for x in a[6:9]))


SCENE_SPECS = {
    # name: (make_scene kwargs, Params kwargs)
    "huber_k0_c8": (dict(seed=1, C=8, N=150), dict(noise_sigma=1.0)),
    "huber_dist_c12": (dict(seed=2, C=12, N=220, dist=True), dict(noise_sigma=2.0)),
    "none_prior_c10": (dict(seed=3, C=10, N=160, outlier=0.0), dict(noise_sigma=1.0, huber_k=0.0, gauge=gb.FIRST_POSE_PRIOR)),
    "huber_prior_c6": (dict(seed=4, C=6, N=90, dist=True), dict(noise_sigma=2.0, gauge=gb.FIRST_POSE_PRIOR)),
    "no_track_cam_c7": (dict(seed=5, C=7, N=120, no_track_cam=True), dict(noise_sigma=1.0)),
    "behind_c9": (dict(seed=6, C=9, N=140, behind=4), dict(noise_sigma=1.0)),
    "two_cams": (dict(seed=7, C=2, N=80, views=(2, 2)), dict(noise_sigma=1.0)),
    "three_cams_none": (dict(seed=8, C=3, N=60, outlier=0.0), dict(noise_sigma=2.0, huber_k=0.0)),
    "long_tracks_c60": (dict(seed=9, C=60, N=400, views=(2, 40), dist=True), dict(noise_sigma=1.0)),
}


def scenes():
    out = {}
    for name, (sk, pk) in SCENE_SPECS.items():
        sc = make_scene(**sk)
        sc["params"] = params_array(gb.Params(**pk))
        out[name] = sc
    return out


def lund_scene(seed=11):
    z = np.load(ROOT / "tests/golden/data_assoc_lund_door.npz")
    g = lambda k: z["uniform_10px_100/" + k]  # noqa: E731
    off, cam, uvs, cams15, valid, ex, pt, inl = (g(k) for k in ("track_off", "meas_cam", "meas_uv", "cams", "cam_valid", "exit",
                                                              "point", "inlier"))
    vidx = np.flatnonzero(valid)
    remap = -np.ones(len(valid), np.int64)
    remap[vidx] = np.arange(len(vidx))
    toff, mcam, uv, pts = [0], [], [], []
    for t in range(len(off) - 1):
        if ex[t] != 0:
            continue
        for m in range(off[t], off[t + 1]):
            if inl[m]:
                mcam.append(remap[cam[m]])
                uv.append(uvs[m])
        toff.append(len(mcam))
        pts.append(pt[t])
    rng = np.random.default_rng(seed)
    cams = np.zeros((len(vidx), 17))
    for a, i in enumerate(vidx):
        R, t = tv.retract_pose(cams15[i, :9].reshape(3, 3), cams15[i, 9:12], rng.normal(size=6) * np.r_[[0.002] * 3, [0.02] * 3])
        cams[a, :9], cams[a, 9:12] = R.ravel(), t
        cams[a, 12:] = [cams15[i, 12] * (1.0 + 0.01 * rng.normal()), 0.0, 0.0, cams15[i, 13], cams15[i, 14]]
    return dict(cams=cams, points=np.array(pts), track_off=np.array(toff, np.int64), meas_cam=np.array(mcam, np.int32),
                meas_uv=np.array(uv, float), params=params_array(gb.Params(noise_sigma=1.0)))


def solve(sc):
    r = gb.adjust(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"], params_from(sc["params"]))
    return dict(cams_out=r.cams, points_out=r.pts, reproj_err=r.reproj_err, final_error=np.array(r.final_error),
                iterations=np.array(r.iterations), trace=np.array(r.trace), trials=np.array(r.trials, np.int32))


# ---- the reference's own stage loop under stand-ins ------------------------------------------------------------------
class _Rec:
    """A factor or noise model stand-in: records its constructor arguments."""

    def __init__(self, kind, *args):
        self.kind, self.args = kind, args


class _Graph(list):
    def push_back(self, f):
        self.extend(f) if isinstance(f, _Graph) else self.append(f)

    def error(self, values):
        return values.final_error


class _Values(dict):
    final_error = 0.0

    def insert(self, k, v):
        self[k] = v


def _standin_data(sc):
    """A GtsfmData stand-in over the scene's arrays: the calls run_ba_stage_with_filtering makes."""
    C = len(sc["cams"])

    class Cam:
        def __init__(self, a):
            self.a = a

        def calibration(self):
            return types.SimpleNamespace(dim=lambda: 3, kind="Cal3Bundler")

        def pose(self):
            return ("pose", self.a)

    class Track:
        def __init__(self, j):
            self.j = j

        def numberMeasurements(self):  # noqa: N802
            return int(sc["track_off"][self.j + 1] - sc["track_off"][self.j])

        def measurement(self, k):
            m = sc["track_off"][self.j] + k
            return int(sc["meas_cam"][m]), sc["meas_uv"][m]

        def point3(self):
            return sc["points"][self.j]

    class Data:
        calls = []

        def __init__(self, tag="input"):
            self.tag = tag

        def number_tracks(self):
            return len(sc["track_off"]) - 1

        def get_valid_camera_indices(self):
            return list(range(C))

        def get_camera(self, i):
            return Cam(i)

        def cameras(self):
            return {i: Cam(i) for i in range(C)}

        def get_track(self, j):
            return Track(j)

        def to_values(self, shared_calib=False):
            Data.calls.append(("to_values", self.tag))
            return _Values()

        @classmethod
        def from_values(cls, values, initial_data, shared_calib=False):
            Data.calls.append(("from_values", initial_data.tag))
            d = cls("optimized")
            d.result = values.result
            return d

        def filter_landmarks(self, thresh):
            mask = gb.valid_mask(self.result.reproj_err, sc["track_off"], thresh)
            d = Data("filtered")
            d.result = self.result
            return d, [bool(v) for v in mask]

    return Data


def _reference(reference: Path, sc):
    from oracle.make_golden_data_assoc import _module_body

    prm = params_from(sc["params"])
    Data = _standin_data(sc)
    graphs = []

    class LM:
        def __init__(self, graph, values, params):
            graphs.append(graph)
            self.values_ = values

        def optimize(self):
            r = gb.adjust(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"], prm)
            v = _Values()
            v.result, v.final_error = r, r.final_error
            return v

    lmp = types.SimpleNamespace(setVerbosityLM=lambda *a: None, setOrderingType=lambda *a: None, setMaxIterations=lambda *a: None)
    gtsam = types.SimpleNamespace(LevenbergMarquardtParams=lambda: lmp, LevenbergMarquardtOptimizer=LM,
                                  KarcherMeanFactorPose3=lambda *a: _Rec("karcher", *a),
                                  Marginals=lambda *a: types.SimpleNamespace(marginalCovariance=lambda k: None))
    noise = types.SimpleNamespace(Sigma=lambda d, s: _Rec("isotropic", d, s))
    gtsfm_types = types.SimpleNamespace(
        get_sfm_factor_for_calibration=lambda cal: (lambda *a: _Rec("sfm", *a)),
        get_prior_factor_for_calibration=lambda cal: (lambda *a: _Rec("cal_prior", *a)),
        get_noise_model_for_calibration=lambda cal, focal_sigma, dist_sigma, pp_sigma, skew_sigma: _Rec("diag", focal_sigma, dist_sigma))
    from enum import Enum
    from typing import Dict, List, Optional, Sequence, Tuple

    ns = dict(np=np, Enum=Enum, Dict=Dict, List=List, Optional=Optional, Sequence=Sequence, Tuple=Tuple, gtsam=gtsam,
              NonlinearFactorGraph=_Graph, Values=_Values, Isotropic=noise, Robust=lambda m, n: _Rec("robust", m, n),
              mEstimator=types.SimpleNamespace(Huber=lambda k: _Rec("huber", k)), PriorFactorPose3=lambda *a: _Rec("pose_prior", *a),
              PriorFactorPoint3=lambda *a: _Rec("point_prior", *a), BetweenFactorPose3=lambda *a: _Rec("between", *a),
              X=lambda i: ("x", i), P=lambda j: ("p", j), K=lambda i: ("k", i), GtsfmData=Data, gtsfm_types=gtsfm_types,
              gtsfm_data=types.SimpleNamespace(), logger=types.SimpleNamespace(info=lambda *a: None, warning=lambda *a: None,
                                                                                 error=lambda *a: None), time=__import__("time"))
    body = _module_body(reference / "gtsfm/bundle/bundle_adjustment.py", ns,
                        names={"RobustBAMode", "CAM_POSE3_DOF", "IMG_MEASUREMENT_DIM", "POINT3_DOF", "BundleAdjustmentOptimizer"})
    opt = body["BundleAdjustmentOptimizer"](
        reproj_error_thresholds=list(THRESHOLDS), robust_ba_mode="HUBER" if prm.huber_k > 0 else "NONE",
        measurement_noise_sigma=prm.noise_sigma, robust_noise_basin=prm.huber_k if prm.huber_k > 0 else 1.345,
        use_karcher_mean_factor=prm.gauge == gb.KARCHER, cam_pose3_prior_noise_sigma=prm.pose_prior_sigma,
        calibration_prior_focal_sigma=prm.cal_prior_sigma[0], calibration_prior_dist_sigma=prm.cal_prior_sigma[1])
    optimized, filtered, mask = opt.run_ba(Data(), [], {})
    # the graph the reference built, against the restatement's
    g = graphs[-1]
    sfm = [f for f in g if f.kind == "sfm"]
    M = len(sc["meas_cam"])
    assert len(sfm) == M and [f.args[2] for f in sfm] == [("x", int(a)) for a in sc["meas_cam"]]
    assert [f.args[3][1] for f in sfm] == list(np.repeat(np.arange(len(sc["track_off"]) - 1), np.diff(sc["track_off"])))
    nm = sfm[0].args[1]
    if prm.huber_k > 0:
        assert nm.kind == "robust" and nm.args[0].args == (prm.huber_k,) and nm.args[1].args == (2, prm.noise_sigma)
    else:
        assert nm.kind == "isotropic" and nm.args == (2, prm.noise_sigma)
    gauge = [f for f in g if f.kind in ("karcher", "pose_prior")]
    assert len(gauge) == 1 and gauge[0].kind == ("karcher" if prm.gauge == gb.KARCHER else "pose_prior")
    if prm.gauge == gb.KARCHER:
        assert gauge[0].args[1:] == (6, 1000) and list(gauge[0].args[0]) == [("x", a) for a in range(len(sc["cams"]))]
    cal = [f for f in g if f.kind == "cal_prior"]
    assert len(cal) == len(sc["cams"]) and all(f.args[2].args == prm.cal_prior_sigma[:2] for f in cal)
    # every stage optimised the input data, and the result is the last stage's
    assert Data.calls == [("to_values", "input"), ("from_values", "input")] * len(THRESHOLDS), Data.calls
    return optimized.result, mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, default=None)
    a = ap.parse_args()
    for path, scs in ((OUT_SCENES, scenes()), (OUT_LUND, {"lund_door": lund_scene()})):
        out = {}
        for name, sc in scs.items():
            res = solve(sc)
            if a.reference is not None:
                r, mask = _reference(a.reference, sc)
                assert r.iterations == res["iterations"] and np.array_equal(r.trials, res["trials"])
                assert np.array_equal(r.cams, res["cams_out"]) and np.array_equal(r.pts, res["points_out"])
                assert r.final_error == float(res["final_error"])
                assert np.array_equal(mask, gb.valid_mask(res["reproj_err"], sc["track_off"], THRESHOLDS[-1]))
            print(f"{name}: C {len(sc['cams'])} N {len(sc['points'])} M {len(sc['meas_cam'])} its {int(res['iterations'])} "
                  f"trials {len(res['trials'])} cost {res['trace'][0]:.6g} -> {float(res['final_error']):.6g}")
            for k, v in {**sc, **res}.items():
                out[f"{name}/{k}"] = v
        np.savez_compressed(path, **out)
        print("wrote", path)


if __name__ == "__main__":
    main()
