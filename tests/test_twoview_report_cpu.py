"""CPU suite for the two-view reports: the NumPy oracle (oracle/twoview_report_ref.py) against the committed fixtures, the
report field list, and the host build of the device maths (csrc/twoview_eval.cuh) against the oracle."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import make_golden_twoview_report as mg
from oracle import twoview_report_ref as ref

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"


@pytest.fixture(scope="module", params=["scenes", "lund_door"])
def fixture(request):
    d = np.load(GOLDEN / f"twoview_report_{request.param}.npz")
    names = [str(n) for n in d["names"]] if "names" in d else [f"{a}_{b}" for a, b in d["pairs"]]
    return d, names


def _check_report(d, name, stage, r):
    assert np.array_equal(np.asarray(r["v_corr_idxs"]).reshape(-1, 2), d[f"{name}/{stage}/v_corr_idxs"]), (name, stage)
    for f, v, none in zip(ref.SCALARS, d[f"{name}/{stage}/scalars"], d[f"{name}/{stage}/none"]):
        if none:
            assert r[f] is None, (name, stage, f)
        else:
            assert r[f] is not None and (float(r[f]) == v or (np.isnan(v) and np.isnan(float(r[f])))), (name, stage, f, r[f], v)
    if f"{name}/{stage}/mask" in d:
        assert np.array_equal(r["v_corr_idxs_inlier_mask_gt"], d[f"{name}/{stage}/mask"])
        assert np.array_equal(r["reproj_error_gt_model"], d[f"{name}/{stage}/d2"], equal_nan=True)
    else:
        assert r["v_corr_idxs_inlier_mask_gt"] is None and r["reproj_error_gt_model"] is None


def test_oracle_reproduces_fixtures(fixture):
    d, names = fixture
    for name in names:
        pre, post, isp, ok = mg.unit_reports(mg.load_unit(d, name))
        assert ok == bool(d[f"{name}/isp_ok"])
        for stage, r in (("pre", pre), ("post", post), ("isp", isp)):
            _check_report(d, name, stage, r)


def test_fixture_covers_the_cases():
    d = np.load(GOLDEN / "twoview_report_scenes.npz")
    u = {str(n): mg.load_unit(d, str(n)) for n in d["names"]}
    assert not bool(u["verification_failed"]["ver_ok"])
    assert np.isnan(u["one_camera_missing"]["cam2"]).all()
    assert bool(u["ba_keeps_nothing"]["ba"]) and u["ba_keeps_nothing"]["pmask"].sum() == 0
    assert not bool(d["isp_ratio/isp_ok"]) and d["isp_ratio/pre/scalars"][1] < 0.1
    assert not bool(d["isp_count/isp_ok"]) and bool(u["isp_count"]["ba"]) and 0 < u["isp_count"]["pmask"].sum() < 15
    assert not bool(u["below_min_inliers"]["ba"]) and u["below_min_inliers"]["vmask"].sum() < 15
    assert abs(d["rotation_170/pre/scalars"][4] - 170.0) < 1e-6
    for name in ("near_thr_above", "near_thr_below"):
        d2, thr = d[f"{name}/pre/d2"], float(u[name]["thr"])
        assert np.min(np.abs(d2 / thr ** 2 - 1.0)) < 1e-9


def test_quirks():
    """ISP failure keeps the post-BA rows in its report with every other field at its default; without BA the post-BA
    report is a copy of the pre-BA one; the ISP-failure report's ratio is None."""
    d = np.load(GOLDEN / "twoview_report_scenes.npz")
    pre, post, isp, ok = mg.unit_reports(mg.load_unit(d, "isp_count"))
    assert not ok and isp["num_inliers_est_model"] == 0 and np.array_equal(isp["v_corr_idxs"], post["v_corr_idxs"])
    assert all(isp[f] is None for f in ref.FIELDS if f not in ("v_corr_idxs", "num_inliers_est_model"))
    pre, post, isp, ok = mg.unit_reports(mg.load_unit(d, "below_min_inliers"))
    same = [(a is None and b is None) or (a is not None and b is not None and np.array_equal(np.asarray(a, float), np.asarray(b, float),
                                                                                          equal_nan=True))
            for a, b in ((post[f], pre[f]) for f in ref.FIELDS)]
    assert post is not pre and all(same)
    pre, post, isp, ok = mg.unit_reports(mg.load_unit(d, "verification_failed"))
    assert pre["num_inliers_gt_model"] == 0 and np.isnan(pre["inlier_ratio_gt_model"]) and pre["R_error_deg"] is None


def test_report_fields_match_fixture():
    from gtsfm_b200.gtsfm_api import TwoViewEstimationReport

    for f in ("scenes", "lund_door"):
        assert tuple(str(x) for x in np.load(GOLDEN / f"twoview_report_{f}.npz")["fields"]) == ref.FIELDS
    assert tuple(TwoViewEstimationReport.__dataclass_fields__) == ref.FIELDS
    r = TwoViewEstimationReport(v_corr_idxs=np.zeros((0, 2)), num_inliers_est_model=0)
    assert all(getattr(r, f) is None for f in ref.FIELDS[2:])


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    exe = tmp_path_factory.mktemp("te") / "test_twoview_eval"
    subprocess.run([cxx, "-O2", "-std=c++17", "-x", "c++", str(ROOT / "tests/cpp/test_twoview_eval.cpp"), "-o", str(exe)], check=True)

    def run(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return [np.array(line.split(), float) for line in out.strip().splitlines()]

    return run


def _f(a):
    return " ".join(repr(float(v)) for v in np.ravel(a))


def _rot(rng, deg):
    from scipy.spatial.transform import Rotation

    a = rng.normal(size=3)
    return Rotation.from_rotvec(a / np.linalg.norm(a) * np.radians(deg)).as_matrix()


def test_host_maths_equal_oracle(shim):
    rng = np.random.default_rng(3)
    cams = [((_rot(rng, rng.uniform(0, 180)), rng.normal(size=3), rng.uniform(400, 900), rng.uniform(300, 400), rng.uniform(200, 300)),
             (_rot(rng, rng.uniform(0, 180)), rng.normal(size=3), rng.uniform(400, 900), 320.0, 240.0)) for _ in range(20)]
    out = shim([f"F {_f(a[0])} {_f(a[1])} {_f(b[0])} {_f(b[1])} {_f(a[2:])} {_f(b[2:])}" for a, b in cams])
    for (a, b), F in zip(cams, out):
        R, t = ref.gt_relative(a, b)
        F_ref = ref.gt_fundamental(R, t, a[2:], b[2:])
        assert np.allclose(F.reshape(3, 3), F_ref, rtol=1e-12, atol=1e-12 * np.abs(F_ref).max())
        x1, x2 = rng.uniform(0, 800, (10, 2)), rng.uniform(0, 800, (10, 2))
        d2 = shim([f"samp {_f(F_ref)} {_f(p)} {_f(q)}" for p, q in zip(x1, x2)])
        assert np.allclose(np.concatenate(d2), ref.sampson_sq(x1, x2, F_ref), rtol=1e-12, atol=0)


@pytest.mark.parametrize("deg", [0.0, 1e-7, 1e-3, 0.5, 45.0, 90.0, 170.0, 179.9, 179.9999, 180.0])
def test_host_rotation_angle(shim, deg):
    rng = np.random.default_rng(int(deg * 1000) % 2 ** 31)
    Rb = _rot(rng, rng.uniform(0, 180))
    Ra = _rot(rng, deg) @ Rb if deg > 0 else Rb.copy()
    got = shim([f"rot {_f(Ra)} {_f(Rb)}"])[0][0]
    assert abs(got - ref.rotation_angle_deg(Ra, Rb)) < 1e-9 and abs(got - deg) < 1e-9


@pytest.mark.parametrize("deg", [0.0, 1e-3, 30.0, 179.0, 180.0])
def test_host_unit_angle(shim, deg):
    rng = np.random.default_rng(7)
    a = rng.normal(size=3)
    b = _rot(rng, 0.0) @ a if deg == 0 else None
    if b is None:
        axis = np.cross(a, rng.normal(size=3))
        from scipy.spatial.transform import Rotation

        b = Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.radians(deg)).as_matrix() @ a * 2.5
    got = shim([f"unit {_f(a)} {_f(b)}"])[0][0]
    assert abs(got - ref.unit_angle_deg(a, b)) < 1e-6 and abs(got - deg) < 1e-5
