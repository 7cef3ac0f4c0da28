"""Global bundle adjustment on the device (b2_bundle_adjust_host) against oracle/global_ba_ref.py: every fixture scene,
a 200-camera scene generated here, repeated calls, the workspace bound, the argument checks and the plugin's array
entry point."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import global_ba_ref as gb  # noqa: E402
from oracle import twoview_ba_ref as tv  # noqa: E402
from oracle.make_golden_global_ba import make_scene, params_from  # noqa: E402

pytestmark = pytest.mark.gpu


def load_scenes(path):
    z = np.load(path)
    out = {}
    for k in z.files:
        name, key = k.split("/")
        out.setdefault(name, {})[key] = z[k]
    return out


ALL = {**load_scenes(ROOT / "tests/golden/global_ba_scenes.npz"), **load_scenes(ROOT / "tests/golden/global_ba_lund_door.npz")}


@pytest.fixture(scope="module")
def ctx():
    from gtsfm_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


def optimizer(prm: gb.Params, ctx):
    from gtsfm_b200.bundle_adjustment import B200BundleAdjustmentOptimizer

    return B200BundleAdjustmentOptimizer(robust_ba_mode="HUBER" if prm.huber_k > 0 else "NONE", measurement_noise_sigma=prm.noise_sigma,
                                         robust_noise_basin=prm.huber_k if prm.huber_k > 0 else 1.345,
                                         use_karcher_mean_factor=prm.gauge == gb.KARCHER, cam_pose3_prior_noise_sigma=prm.pose_prior_sigma,
                                         calibration_prior_focal_sigma=prm.cal_prior_sigma[0],
                                         calibration_prior_dist_sigma=prm.cal_prior_sigma[1], max_iterations=prm.max_iters, ctx=ctx)


def device(sc, ctx):
    prm = params_from(sc["params"])
    return optimizer(prm, ctx).adjust_arrays(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"], trace=True)


def rot_err(A, B):
    return max(np.linalg.norm(tv.so3_log(A[a, :9].reshape(3, 3).T @ B[a, :9].reshape(3, 3))) for a in range(len(A)))


def check_against(d, ref, toff):
    """d: the device's outputs; ref: dict of cams_out, points_out, reproj_err, final_error, iterations, trace, trials."""
    assert d["iterations"] == int(ref["iterations"])
    np.testing.assert_array_equal(d["trials"], ref["trials"])
    # the damped reduced system is ill-conditioned along the scale direction (no factor fixes the scale), so the solve's
    # rounding shows in the cost at ~1e-8 relative; DESIGN.md §3 records the observed agreement
    np.testing.assert_allclose(d["trace"], ref["trace"], rtol=1e-7)
    assert d["final_error"] == pytest.approx(float(ref["final_error"]), rel=1e-7)
    assert rot_err(d["cams"], ref["cams_out"]) < 1e-6
    # translations, f, k1, k2 and points to 1e-6 of their column's magnitude (a coordinate near 0 has no relative scale)
    scale = np.abs(ref["cams_out"][:, 9:15]).max(0)
    assert np.all(np.abs(d["cams"][:, 9:15] - ref["cams_out"][:, 9:15]) <= 1e-6 * scale)
    assert np.all(np.abs(d["points"] - ref["points_out"]) <= 1e-6 * np.abs(ref["points_out"]).max(0))
    near = 0
    for thr in (10.0, 5.0, 3.0):
        e, r = d["reproj_err"], ref["reproj_err"]
        hair = np.logical_or.reduceat(np.abs(r - thr) < 1e-6, toff[:-1])
        near += int(hair.sum())
        vd, vr = gb.valid_mask(e, toff, thr), gb.valid_mask(r, toff, thr)
        assert np.array_equal(vd[~hair], vr[~hair])
    assert near <= max(1, len(toff) // 100)


STRICT = sorted(n for n, s in ALL.items() if not np.any(s["trials"] == -1))
INDETERMINATE = sorted(n for n, s in ALL.items() if np.any(s["trials"] == -1))


@pytest.mark.parametrize("name", STRICT)
def test_fixture_scene(name, ctx):
    """Scenes whose damped systems all factor: the same trials, trace, result and masks as the oracle."""
    sc = ALL[name]
    check_against(device(sc, ctx), sc, sc["track_off"])


@pytest.mark.parametrize("name", INDETERMINATE)
def test_fixture_scene_with_indeterminate_trials(name, ctx):
    """Scenes where LM drives lambda so low that the damped reduced system is singular to working precision along the
    scale direction (no factor fixes the scale): whether such a trial's Cholesky fails depends on rounding, so the trial
    sequences of two correct implementations may part there.  The device must still converge to the oracle's cost."""
    sc = ALL[name]
    d = device(sc, ctx)
    print(name, d["iterations"], int(sc["iterations"]), d["final_error"], float(sc["final_error"]))
    np.testing.assert_allclose(d["trace"][:3], sc["trace"][:3], rtol=1e-6)
    assert d["final_error"] == pytest.approx(float(sc["final_error"]), rel=1e-4)


def test_200_camera_scene(ctx):
    sc = make_scene(seed=31, C=200, N=3000, views=(2, 12), dist=True)
    prm = gb.Params(noise_sigma=1.0, max_iters=15)
    r = gb.adjust(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"], prm)
    d = optimizer(prm, ctx).adjust_arrays(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"], trace=True)
    ref = dict(cams_out=r.cams, points_out=r.pts, reproj_err=r.reproj_err, final_error=r.final_error, iterations=r.iterations,
               trace=np.array(r.trace), trials=np.array(r.trials, np.int32))
    check_against(d, ref, sc["track_off"])


def test_repeated_calls_are_bit_identical(ctx):
    sc = ALL["long_tracks_c60"]
    a, b = device(sc, ctx), device(sc, ctx)
    for k in ("cams", "points", "reproj_err", "trace", "trials"):
        assert np.array_equal(a[k], b[k], equal_nan=True), k
    assert a["final_error"] == b["final_error"]


def test_workspace_bound(ctx):
    from gtsfm_b200 import _lib
    from gtsfm_b200.bundle_adjustment import B200BundleAdjustmentOptimizer

    sc = ALL["long_tracks_c60"]
    c = _lib.Context(0)
    try:
        c.set_option("ba_workspace_mb", 1)
        o = B200BundleAdjustmentOptimizer(robust_ba_mode="HUBER", measurement_noise_sigma=1.0, ctx=c)
        assert not o.fits(len(sc["cams"]), sc["track_off"])  # the plugin falls back to the reference
        with pytest.raises(_lib.B200Error, match="ba_workspace_mb"):
            o.adjust_arrays(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"])
        c.set_option("ba_workspace_mb", 4096)
        assert o.fits(len(sc["cams"]), sc["track_off"])
    finally:
        c.close()


def _call(ctx, cams, pts, off, cam, uv, prm=None):
    from gtsfm_b200 import _lib

    prm = prm or optimizer(gb.Params(noise_sigma=1.0), None).device_params()
    cams = np.ascontiguousarray(cams, float)
    pts = np.ascontiguousarray(pts, float)
    off = np.ascontiguousarray(off, np.int64)
    cam = np.ascontiguousarray(cam, np.int32)
    uv = np.ascontiguousarray(uv, float)
    co, po, err, res = np.empty_like(cams), np.empty_like(pts), np.empty(len(cam)), _lib.BaResult()
    return ctx.lib.b2_bundle_adjust_host(ctx.handle, len(cams), _lib.ptr(cams), len(pts), _lib.ptr(pts), _lib.ptr(off), _lib.ptr(cam),
                                         _lib.ptr(uv), _lib.C.byref(prm), _lib.ptr(co), _lib.ptr(po), _lib.ptr(err), _lib.C.byref(res),
                                         None, None, 0, None)


def test_argument_checks(ctx):
    sc = ALL["three_cams_none"]
    cams, pts, off, cam, uv = (sc[k].copy() for k in ("cams", "points", "track_off", "meas_cam", "meas_uv"))
    assert _call(ctx, cams, pts, off, cam, uv) == 0
    bad = cam.copy()
    bad[0] = 3
    assert _call(ctx, cams, pts, off, bad, uv) == -2
    bad[0] = -1
    assert _call(ctx, cams, pts, off, bad, uv) == -2
    c2 = cams.copy()
    c2[1, 12] = 0.0
    assert _call(ctx, c2, pts, off, cam, uv) == -2
    p2 = pts.copy()
    p2[3, 1] = np.nan
    assert _call(ctx, cams, p2, off, cam, uv) == -2
    u2 = uv.copy()
    u2[5, 0] = np.inf
    assert _call(ctx, cams, pts, off, cam, u2) == -2
    o2 = off.copy()
    o2[2] = o2[1]  # track 1 without a measurement
    assert _call(ctx, cams, pts, o2, cam, uv) == -2
    dup = cam.copy()
    dup[off[0] + 1] = dup[off[0]]  # two measurements of track 0 in one camera
    assert _call(ctx, cams, pts, off, dup, uv) == -2


def test_plugin_adjust_arrays_equals_the_direct_call(ctx):
    from gtsfm_b200 import _lib

    sc = ALL["huber_prior_c6"]
    prm = params_from(sc["params"])
    o = optimizer(prm, ctx)
    d = o.adjust_arrays(sc["cams"], sc["points"], sc["track_off"], sc["meas_cam"], sc["meas_uv"])
    p = o.device_params()
    cams = np.ascontiguousarray(sc["cams"])
    pts = np.ascontiguousarray(sc["points"])
    co, po, err, res = np.empty_like(cams), np.empty_like(pts), np.empty(len(sc["meas_cam"])), _lib.BaResult()
    rc = ctx.lib.b2_bundle_adjust_host(ctx.handle, len(cams), _lib.ptr(cams), len(pts), _lib.ptr(pts), _lib.ptr(sc["track_off"]),
                                       _lib.ptr(np.ascontiguousarray(sc["meas_cam"], np.int32)), _lib.ptr(sc["meas_uv"]), _lib.C.byref(p),
                                       _lib.ptr(co), _lib.ptr(po), _lib.ptr(err), _lib.C.byref(res), None, None, 0, None)
    assert rc == 0
    assert np.array_equal(d["cams"], co) and np.array_equal(d["points"], po) and np.array_equal(d["reproj_err"], err, equal_nan=True)
    assert d["final_error"] == res.final_error and d["iterations"] == res.iterations
