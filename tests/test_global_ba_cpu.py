"""Global bundle adjustment without a GPU: oracle/global_ba_ref.py against its fixtures and against scipy's minimiser of
the explicit robust cost, the Karcher gauge, the reference's stage loop, the host build of csrc/twoview_math.cuh's
projection Jacobians, and the plugin's fallback rules, pickling and config."""
from __future__ import annotations

import os
import pickle
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import global_ba_ref as gb  # noqa: E402
from oracle import twoview_ba_ref as tv  # noqa: E402
from oracle.make_golden_global_ba import lund_scene, make_scene, params_from, scenes  # noqa: E402


def load_scenes(path):
    z = np.load(path)
    out = {}
    for k in z.files:
        name, key = k.split("/")
        out.setdefault(name, {})[key] = z[k]
    return out


SCENES = load_scenes(ROOT / "tests/golden/global_ba_scenes.npz")
LUND = load_scenes(ROOT / "tests/golden/global_ba_lund_door.npz")
ALL = {**SCENES, **LUND}
INPUTS = ("cams", "points", "track_off", "meas_cam", "meas_uv", "params")


def run(sc, **kw):
    p = params_from(sc["params"])
    for k, v in kw.items():
        setattr(p, k, v)
    return gb.adjust(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"], p)


@pytest.mark.parametrize("name", sorted(ALL))
def test_oracle_matches_fixture(name):
    sc = ALL[name]
    r = run(sc)
    assert r.iterations == sc["iterations"]
    np.testing.assert_array_equal(r.trials, sc["trials"])
    np.testing.assert_allclose(r.trace, sc["trace"], rtol=1e-12)
    np.testing.assert_allclose(r.cams, sc["cams_out"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(r.pts, sc["points_out"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(r.reproj_err, sc["reproj_err"], rtol=1e-10, atol=1e-10, equal_nan=True)
    assert r.final_error == pytest.approx(float(sc["final_error"]), rel=1e-12)


def test_fixture_inputs_are_the_generator_s():
    gen = {**scenes(), "lund_door": lund_scene()}
    assert sorted(gen) == sorted(ALL)
    for name, sc in gen.items():
        for k in INPUTS:
            np.testing.assert_array_equal(sc[k], ALL[name][k])


def test_fixtures_cover_the_cases():
    p = {n: params_from(s["params"]) for n, s in SCENES.items()}
    assert {x.huber_k > 0 for x in p.values()} == {True, False}
    assert {x.gauge for x in p.values()} == {gb.KARCHER, gb.FIRST_POSE_PRIOR}
    assert {x.noise_sigma for x in p.values()} == {1.0, 2.0}
    assert any(len(s["cams"]) == 2 for s in SCENES.values())
    assert max(len(s["cams"]) for s in SCENES.values()) == 60
    assert max(np.diff(s["track_off"]).max() for s in SCENES.values()) >= 30
    assert any(np.any(s["cams"][:, 13] != 0) for s in SCENES.values()) and any(np.all(s["cams"][:, 13] == 0) for s in SCENES.values())
    assert any(len(np.unique(s["meas_cam"])) < len(s["cams"]) for s in SCENES.values())  # a camera without a track
    # Huber is active: some whitened residual at the result lies outside the basin
    hub = [n for n in SCENES if p[n].huber_k > 0]
    assert any(np.nanmax(SCENES[n]["reproj_err"]) / p[n].noise_sigma > p[n].huber_k for n in hub)


def test_oracle_converges_to_scipy_minimum():
    """Run to convergence, the oracle's optimum is a minimum of the explicit robust cost that scipy's minimiser, started
    there, keeps (first-pose prior, so the optimum is isolated)."""
    from scipy.optimize import least_squares

    sc = make_scene(seed=21, C=4, N=40, views=(2, 4), outlier=0.1, dist=True)
    prm = gb.Params(noise_sigma=1.0, gauge=gb.FIRST_POSE_PRIOR, max_iters=500, rel_tol=0.0, abs_tol=0.0)
    r = gb.adjust(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"], prm)
    pr = gb.Problem(sc["cams"].copy(), sc["track_off"], sc["meas_cam"], sc["meas_uv"], prm)
    C, N = len(sc["cams"]), len(sc["points"])
    base = r.cams

    def unpack(x):
        cams = gb.retract(base, x[:9 * C])
        return cams, x[9 * C:].reshape(N, 3)

    def resid(x):
        cams, pts = unpack(x)
        uv, z, _, _ = gb.project_meas(cams, pts, pr)
        d = (uv - pr.uv) / prm.noise_sigma
        e = np.linalg.norm(d, axis=1)
        rho = np.where(e <= prm.huber_k, 0.5 * e * e, prm.huber_k * (e - 0.5 * prm.huber_k))
        f = (np.sqrt(2.0 * rho) / np.maximum(e, 1e-300))[:, None] * d
        ci = 1.0 / np.asarray(prm.cal_prior_sigma)
        fc = ((cams[:, 12:15] - pr.cam0[:, 12:15]) * ci).ravel()
        fp = gb._pose_prior_err(cams[0], pr.cam0[0], 1.0 / prm.pose_prior_sigma)
        return np.concatenate([f.ravel(), fc, fp])

    x0 = np.concatenate([np.zeros(9 * C), r.pts.ravel()])  # scipy starts at the oracle's optimum and cannot improve it
    sol = least_squares(resid, x0, xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=5000, method="trf", x_scale="jac")
    cams_s, pts_s = unpack(sol.x)
    c_s = gb.cost(cams_s, pts_s, pr)
    assert r.final_error == pytest.approx(c_s, rel=1e-9)
    for a in range(C):
        dR = r.cams[a, :9].reshape(3, 3).T @ cams_s[a, :9].reshape(3, 3)
        assert np.linalg.norm(tv.so3_log(dR)) < 1e-7


def test_karcher_term_is_beta_ones_kron_identity():
    sc = SCENES["huber_k0_c8"]
    pr = gb.Problem(sc["cams"].copy(), sc["track_off"], sc["meas_cam"], sc["meas_uv"], params_from(sc["params"]))
    a = gb.reduced_system(sc["cams"], sc["points"], pr, 1e-3)
    b = gb.reduced_system(sc["cams"], sc["points"], pr, 1e-3, karcher=False)
    C = len(sc["cams"])
    K = np.zeros((C, 9, C, 9))
    K[:, :6, :, :6] = np.eye(6)[None, :, None, :]
    np.testing.assert_allclose(a[0] - b[0], 1000.0 * K.reshape(9 * C, 9 * C), rtol=0, atol=1e-7)
    np.testing.assert_array_equal(a[1], b[1])


def test_karcher_pose_updates_sum_to_zero():
    """Every accepted step's pose updates sum to ~0: the Karcher factor's beta |sum d_i|^2 dominates that direction."""
    sc = SCENES["huber_dist_c12"]
    r = run(sc)
    for dc in r.steps:
        d = dc.reshape(-1, 9)[:, :6]
        assert np.linalg.norm(d.sum(0)) <= 1e-6 * max(1.0, np.linalg.norm(d))


def test_karcher_result_does_not_depend_on_camera_order():
    """The Karcher gauge has no anchor camera: relabelling the cameras relabels the problem, and LM takes the same path.
    The reduced system's elimination order changes with the labels, and the scale direction is fixed by the damping only,
    so the paths agree to the problem's conditioning rather than to round-off."""
    sc = SCENES["huber_k0_c8"]
    C = len(sc["cams"])
    perm = np.roll(np.arange(C), 3)  # new camera a is old camera perm[a]
    inv = np.argsort(perm)
    r0 = run(sc)
    r1 = gb.adjust(sc["cams"][perm], sc["points"], sc["track_off"], inv[sc["meas_cam"]], sc["meas_uv"], params_from(sc["params"]))
    assert r1.iterations == r0.iterations
    np.testing.assert_allclose(r1.trace[:3], r0.trace[:3], rtol=1e-9)
    assert r1.final_error == pytest.approx(r0.final_error, rel=1e-6)


REFERENCE = Path(os.environ.get("GTSFM_REFERENCE", "")) if os.environ.get("GTSFM_REFERENCE") else None


@pytest.mark.skipif(REFERENCE is None or not (REFERENCE / "gtsfm/bundle/bundle_adjustment.py").exists(),
                    reason="set GTSFM_REFERENCE to a GTSfM checkout")
def test_reference_stage_loop_optimises_the_input_every_stage():
    """The reference's run_ba hands `initial_data` to every stage, so [10, 5, 3] is one optimisation filtered at 3 px
    (make_golden_global_ba._reference asserts the calls)."""
    from oracle.make_golden_global_ba import _reference

    sc = SCENES["three_cams_none"]
    r, mask = _reference(REFERENCE, sc)
    assert r.iterations == sc["iterations"]
    np.testing.assert_array_equal(mask, gb.valid_mask(sc["reproj_err"], sc["track_off"], 3.0))


def test_valid_mask_rule():
    err = np.array([1.0, 2.9, 3.0, 0.5, np.nan, 0.1])
    off = np.array([0, 2, 4, 6])
    np.testing.assert_array_equal(gb.valid_mask(err, off, 3.0), [True, False, False])
    np.testing.assert_array_equal(gb.valid_mask(err, off, 3.5), [True, True, False])


PROJ_CASES = [
    (np.array([0.1, -0.2, 0.3]), np.array([0.5, -0.2, -3.0]), np.array([520.0, 0.0, 0.0, 320.0, 240.0]), np.array([0.3, 0.4, 2.0])),
    (np.array([-0.3, 0.1, 0.05]), np.array([1.0, 0.2, -2.0]), np.array([610.0, -0.07, 0.015, 300.0, 200.0]), np.array([-0.5, 0.2, 3.5])),
]


def test_host_build_jacobians_against_central_differences(tmp_path):
    """tests/cpp/test_twoview_math.cpp (twoview_math.cuh on the host): the projection with k1, k2 and its Jacobians equal the
    oracle's and central differences of the projection under the retraction."""
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    exe = tmp_path / "twoview_math"
    subprocess.run([cxx, "-O2", "-std=c++17", "-x", "c++", str(ROOT / "tests/cpp/test_twoview_math.cpp"), "-o", str(exe)], check=True)
    lines = []
    for w, t, cal, p in PROJ_CASES:
        R = tv.so3_exp(w)
        lines.append("proj " + " ".join(f"{v:.17g}" for v in np.concatenate([R.ravel(), t, cal, p])))
    out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.split("\n")
    for (w, t, cal, p), line in zip(PROJ_CASES, out):
        v = np.array(line.split(), float)
        R = tv.so3_exp(w)
        uv, z, Jc, Jp = gb.project_meas(np.concatenate([R.ravel(), t, cal])[None], p[None], gb.Problem(
            np.zeros((1, 17)), [0, 1], [0], np.zeros((1, 2)), gb.Params()))
        np.testing.assert_allclose(v[1:3], uv[0], rtol=1e-13)
        np.testing.assert_allclose(v[3:21].reshape(2, 9), Jc[0], rtol=1e-11, atol=1e-9)
        np.testing.assert_allclose(v[21:27].reshape(2, 3), Jp[0], rtol=1e-11, atol=1e-9)
        h = 1e-6
        for i in range(9):
            d = np.zeros(9)
            d[i] = h
            up = [tv.retract_pose(R, t, d[:6]), tv.retract_pose(R, t, -d[:6])]
            cp, cm = cal.copy(), cal.copy()
            cp[:3] += d[6:]
            cm[:3] -= d[6:]
            fd = (tv.project(*up[0], cp, p)[0] - tv.project(*up[1], cm, p)[0]) / (2 * h)
            np.testing.assert_allclose(v[3:21].reshape(2, 9)[:, i], fd, rtol=1e-6, atol=1e-4)
        for i in range(3):
            d = np.zeros(3)
            d[i] = h
            fd = (tv.project(R, t, cal, p + d)[0] - tv.project(R, t, cal, p - d)[0]) / (2 * h)
            np.testing.assert_allclose(v[21:27].reshape(2, 3)[:, i], fd, rtol=1e-6, atol=1e-4)


# ---- the plugin ------------------------------------------------------------------------------------------------------
from gtsfm_b200 import bundle_adjustment as ba  # noqa: E402
from gtsfm_b200.gtsfm_api import HAVE_GTSFM_BA  # noqa: E402


def test_plugin_params_follow_the_reference_fields():
    o = ba.B200BundleAdjustmentOptimizer(reproj_error_thresholds=[10, 5, 3], robust_ba_mode="HUBER", measurement_noise_sigma=1.0)
    p = o.device_params()
    assert (p.noise_sigma, p.huber_k, p.gauge, p.max_iters, p.karcher_beta) == (1.0, 1.345, 0, 100, 1000.0)
    assert tuple(p.cal_prior_sigma) == (20.0, 0.1, 0.1)
    p = ba.B200BundleAdjustmentOptimizer(use_karcher_mean_factor=False, max_iterations=7, robust_noise_basin=2.0).device_params()
    assert (p.huber_k, p.gauge, p.max_iters, p.pose_prior_sigma) == (0.0, 1, 7, 0.1)


@pytest.mark.parametrize("kw", [dict(use_gnc=True), dict(robust_ba_mode="GMC"), dict(shared_calib=True), dict(use_pose_prior=True),
                                dict(use_first_point_prior=True), dict(use_calibration_prior=False)])
def test_plugin_unserved_settings_raise_without_gtsfm(kw):
    o = ba.B200BundleAdjustmentOptimizer(**kw)
    assert o.unserved() is not None
    with pytest.raises(ValueError):
        o.device_params()
    if not HAVE_GTSFM_BA:
        with pytest.raises(ValueError):
            o.run_ba_stage_with_filtering(object(), [], {}, 3.0)


def test_plugin_relative_pose_priors_are_not_served():
    o = ba.B200BundleAdjustmentOptimizer()
    assert o.unserved({(0, 1): object()}) == "relative_pose_priors"
    assert o.unserved({}) is None


def test_plugin_pickles_without_its_context():
    o = ba.B200BundleAdjustmentOptimizer(robust_ba_mode="HUBER", device=1)
    o.ctx = object()
    o2 = pickle.loads(pickle.dumps(o))
    assert o2.ctx is None and o2.device == 1 and o2._robust_ba_mode == o._robust_ba_mode


def test_plugin_size_checks_before_any_device_call():
    o = ba.B200BundleAdjustmentOptimizer()
    with pytest.raises(ValueError):
        o.adjust_arrays(np.zeros((2, 17)), np.zeros((3, 3)), [0, 2, 4], [0, 1, 0, 1], np.zeros((4, 2)))


def test_config_swaps_in_the_plugin_with_the_reference_fields():
    import yaml

    cfg = yaml.safe_load((ROOT / "configs/deep_front_end_b200_ba.yaml").read_text())
    assert cfg["defaults"][0] == "deep_front_end_b200_data_assoc"
    m = cfg["cluster_optimizer"]["multiview_optimizer"]["bundle_adjustment_module"]
    assert m["_target_"] == "gtsfm_b200.bundle_adjustment.B200BundleAdjustmentOptimizer"
    args = {k: v for k, v in m.items() if k != "_target_"}
    assert args == dict(reproj_error_thresholds=[10, 5, 3], robust_ba_mode="HUBER", shared_calib=False, cam_pose3_prior_noise_sigma=0.1,
                        calibration_prior_focal_sigma=20.0, measurement_noise_sigma=1.0)
    o = ba.B200BundleAdjustmentOptimizer(**args)
    assert o.unserved() is None and o.device_params().noise_sigma == 1.0
