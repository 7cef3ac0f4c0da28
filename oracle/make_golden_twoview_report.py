"""Writes the fixtures of the two-view reports (oracle/twoview_report_ref.py):

    tests/golden/twoview_report_lund_door.npz  lund-door's 66 pairs: the keypoints of lund_door_images.npz, the verified
        and post-BA rows and poses of twoview_ba_lund_door.npz, and the ground-truth cameras of the reference's
        tests/data/set1_lund_door/data.mat as OlssonLoader decomposes them (loader/olsson_loader.py:75-100), intrinsics
        rescaled to the fixture's 760-pixel frames (loader/loader_base.py:202-240)
    tests/golden/twoview_report_scenes.npz     seeded scenes of make_golden_twoview_ba.synthetic_scene with their true pose
        as the ground truth, and the cases: verification failure, one camera without ground truth, BA that keeps no rows,
        inlier-support failure by ratio and by count, fewer verified rows than min_num_inliers_est_model (post-BA = pre-BA),
        an estimate 170 degrees off, and rows within 1e-9 relative of the threshold

    python -m oracle.make_golden_twoview_report --reference /path/to/gtsfm-checkout

Each pair ("unit") is stored under "<name>/": kp1, kp2 (float32 pixels), putative (k, 2), ver_ok, vmask (k,), R_pre, t_pre,
ba (bundle adjustment ran), post_pose (the BA has an estimate), R_post, t_post, pmask (k,) (the rows BA kept), cam1, cam2
((15,) = R_wTi, t_wTi, f, u0, v0; NaN when absent), thr, min_inliers, min_ratio; and the oracle's reports: for stage in
pre, post, isp: <stage>/v_corr_idxs, <stage>/scalars (SCALARS order, NaN for None), <stage>/none (which SCALARS are None),
<stage>/mask and <stage>/d2 (present when not None), and isp_ok.

The golden maker also pins the restatement against the reference's own functions where they run without gtsam or dask:
their sources are taken from the checkout and run under minimal stand-ins for Rot3 / Unit3 / EssentialMatrix (see
_pin_against_reference).  run_inlier_support and the report assembly of run_2view are restated, not pinned.
"""
from __future__ import annotations

import argparse
import ast
from pathlib import Path

import numpy as np

from oracle import make_golden_twoview_ba as tvb
from oracle import twoview_ba_ref as ba
from oracle import twoview_report_ref as ref

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"
OUT_LUND = GOLDEN / "twoview_report_lund_door.npz"
OUT_SCENES = GOLDEN / "twoview_report_scenes.npz"


def _cam_vec(cam):
    if cam is None:
        return np.full(15, np.nan)
    R, t, f, u0, v0 = cam
    return np.concatenate([np.asarray(R, float).ravel(), np.asarray(t, float).ravel(), [f, u0, v0]])


def cam_from_vec(v):
    """(15,) fixture vector -> (R_wTi, t_wTi, f, u0, v0), or None (NaN)."""
    v = np.asarray(v, float)
    if np.isnan(v).any():
        return None
    return v[:9].reshape(3, 3), v[9:12], float(v[12]), float(v[13]), float(v[14])


def unit_reports(u: dict):
    """The oracle's three reports of a fixture unit (dict of its arrays)."""
    post = None
    if bool(u["ba"]):
        post = (u["R_post"] if bool(u["post_pose"]) else None, u["t_post"] if bool(u["post_pose"]) else None, u["pmask"])
    return ref.run_2view_reports(u["kp1"], u["kp2"], u["putative"], bool(u["ver_ok"]), u["vmask"], u["R_pre"], u["t_pre"], post,
                                 cam_from_vec(u["cam1"]), cam_from_vec(u["cam2"]), float(u["thr"]), int(u["min_inliers"]),
                                 float(u["min_ratio"]))


def load_unit(d, name: str) -> dict:
    """A fixture unit's inputs as a dict (lund-door keeps each image's keypoints once, as kp_<image>)."""
    u = {key: d[f"{name}/{key}"] for key in UNIT_KEYS if f"{name}/{key}" in d}
    if "kp1" not in u:
        i1, i2 = (int(x) for x in name.split("_"))
        u["kp1"], u["kp2"] = d[f"kp_{i1}"], d[f"kp_{i2}"]
    return u


UNIT_KEYS = ("kp1", "kp2", "putative", "ver_ok", "vmask", "R_pre", "t_pre", "ba", "post_pose", "R_post", "t_post", "pmask", "cam1",
             "cam2", "thr", "min_inliers", "min_ratio")


def _store(arrays: dict, name: str, u: dict, skip=()) -> None:
    for key, v in u.items():
        if key not in skip:
            arrays[f"{name}/{key}"] = np.asarray(v)
    pre, post, isp, ok = unit_reports(u)
    arrays[f"{name}/isp_ok"] = np.array(ok)
    for stage, r in (("pre", pre), ("post", post), ("isp", isp)):
        arrays[f"{name}/{stage}/v_corr_idxs"] = np.asarray(r["v_corr_idxs"], np.int64).reshape(-1, 2)
        arrays[f"{name}/{stage}/scalars"] = np.array([np.nan if r[f] is None else float(r[f]) for f in ref.SCALARS])
        arrays[f"{name}/{stage}/none"] = np.array([r[f] is None for f in ref.SCALARS])
        if r["v_corr_idxs_inlier_mask_gt"] is not None:
            arrays[f"{name}/{stage}/mask"] = np.asarray(r["v_corr_idxs_inlier_mask_gt"], bool)
            arrays[f"{name}/{stage}/d2"] = np.asarray(r["reproj_error_gt_model"], float)


def _unit(kp1, kp2, putative, ver_ok, vmask, R_pre, t_pre, post, cam1, cam2, thr=4.0, min_inliers=15, min_ratio=0.1):
    k = len(putative)
    R_post, t_post, pmask = post if post is not None else (None, None, np.zeros(k, bool))
    return dict(kp1=np.asarray(kp1, np.float32), kp2=np.asarray(kp2, np.float32), putative=np.asarray(putative, np.int64).reshape(-1, 2),
                ver_ok=np.array(bool(ver_ok)), vmask=np.asarray(vmask, np.uint8), R_pre=np.asarray(R_pre if R_pre is not None else np.full((3, 3), np.nan)),
                t_pre=np.asarray(t_pre if t_pre is not None else np.full(3, np.nan)), ba=np.array(post is not None),
                post_pose=np.array(R_post is not None), R_post=np.asarray(R_post if R_post is not None else np.full((3, 3), np.nan)),
                t_post=np.asarray(t_post if t_post is not None else np.full(3, np.nan)), pmask=np.asarray(pmask, np.uint8),
                cam1=_cam_vec(cam1), cam2=_cam_vec(cam2), thr=np.array(float(thr)), min_inliers=np.array(int(min_inliers)),
                min_ratio=np.array(float(min_ratio)))


def _post_ba(uv1, uv2, rows, cal1, cal2, R0, t0):
    """The two-view BA of the oracle before inlier support: -> (R | None, t | None, kept-row mask over the k rows)."""
    r = ba._bundle_adjust_pair(uv1, uv2, np.asarray(rows, np.int64), cal1, cal2, np.asarray(R0, float), np.asarray(t0, float),
                               0.5, np.inf, 0.0, ba.LM_MAX_ITERS)
    mask = np.zeros(len(uv1), bool)
    mask[r.rows] = True
    return (r.R, r.t, mask) if r.ok else (None, None, mask)


# ---- lund-door --------------------------------------------------------------------------------------------------------
def lund_cameras(reference: Path):
    """{image (1-based, as the fixtures): (R_wTi, t_wTi, f, u0, v0)} from data.mat, as OlssonLoader decomposes it, with the
    intrinsics rescaled to 760 pixels on the short side (get_downsampling_factor_per_axis + Cal3Bundler rescale)."""
    import scipy.io
    import scipy.linalg

    P = scipy.io.loadmat(str(reference / "tests/data/set1_lund_door/data.mat"))["P"][0]

    def decompose(M):  # verification.py:22-51
        Q, m4 = M[:3, :3], M[:, 3]
        wtc = np.linalg.inv(-Q) @ m4
        K, cRw = scipy.linalg.rq(Q)
        T = np.diag(np.sign(np.diag(K)))
        return K @ T, (T @ cRw).T, wtc

    K0 = decompose(P[0])[0]
    from PIL import Image

    w, h = Image.open(reference / "tests/data/set1_lund_door/images/DSC_0001.JPG").size
    assert min(h, w) > 760
    if min(h, w) == h:
        new_h = 760
        new_w = int(np.round(w * (new_h / float(h))))
    else:
        new_w = 760
        new_h = int(np.round(h * (new_w / float(w))))
    su, sv = new_w / w, new_h / h
    f, u0, v0 = min(K0[0, 0], K0[1, 1]) * su, K0[0, 2] * su, K0[1, 2] * sv
    cams = {}
    for i in range(len(P)):
        _, wRc, wtc = decompose(P[i])
        cams[i + 1] = (wRc, wtc, f, u0, v0)
    return cams, (new_h, new_w)


def make_lund(reference: Path) -> None:
    kps, pairs, rows, cal = tvb.lund_inputs()
    fx = np.load(GOLDEN / "twoview_ba_lund_door.npz")
    cams, shape = lund_cameras(reference)
    assert shape == np.load(GOLDEN / "lund_door_images.npz")["gray_1"].shape, shape
    arrays = {"pairs": np.array(pairs), **{f"kp_{i}": k.astype(np.float32) for i, k in kps.items()}}
    for p in pairs:
        key = f"{p[0]}_{p[1]}"
        m = rows[p]
        ok = bool(fx[f"{key}/ok"])
        vmask = np.zeros(len(m), bool)
        vmask[fx[f"{key}/verified"]] = True
        post = None
        if ok and vmask.sum() >= 15:
            post = _post_ba(kps[p[0]][m[:, 0]].astype(np.float64), kps[p[1]][m[:, 1]].astype(np.float64), np.flatnonzero(vmask),
                            cal, cal, fx[f"{key}/R0"], fx[f"{key}/t0"])
        u = _unit(kps[p[0]], kps[p[1]], m, ok, vmask, fx[f"{key}/R0"] if ok else None, fx[f"{key}/t0"] if ok else None, post,
                  cams[p[0]], cams[p[1]])
        _store(arrays, key, u, skip=("kp1", "kp2"))
        pre = arrays[f"{key}/pre/scalars"]
        print(f"{key}: verified {int(vmask.sum())} R_err {pre[4]:.3f} U_err {pre[5]:.3f} gt inliers {pre[2]:.0f}")
    arrays["fields"] = np.array(ref.FIELDS)
    np.savez_compressed(OUT_LUND, **arrays)
    print(OUT_LUND)


# ---- seeded scenes ----------------------------------------------------------------------------------------------------
def _scene_unit(seed, n, ba_on=True, ver_ok=True, drop_cam2=False, R_off_deg=0.0, thr=4.0, min_inliers=15, min_ratio=0.1,
                **kw):
    s = tvb.synthetic_scene(seed, n, **kw)
    k = s["k"]
    vmask = np.zeros(k, bool)
    vmask[s["verified"]] = True
    R_pre = s["R0"] if R_off_deg == 0.0 else tvb._rot([0.3, 1.0, -0.2], R_off_deg) @ s["R_true"]
    post = None
    if ba_on and ver_ok and vmask.sum() >= min_inliers:
        post = _post_ba(s["uv1"], s["uv2"], s["verified"], s["cal1"], s["cal2"], R_pre, s["t0"])
    Rt, tt = s["R_true"], s["t_true"]
    cam1 = (np.eye(3), np.zeros(3), *s["cal1"])
    cam2 = None if drop_cam2 else (Rt.T, -Rt.T @ tt, *s["cal2"])  # wTi2 with wTi2.between(wTi1) = (R_true, t_true)
    put = np.stack([np.arange(k), np.arange(k)], 1)
    return _unit(s["uv1"], s["uv2"], put, ver_ok, vmask if ver_ok else np.zeros(k, bool), R_pre if ver_ok else None,
                 s["t0"] if ver_ok else None, post, cam1, cam2, thr, min_inliers, min_ratio)


SCENES = {
    "clean_40": dict(seed=1, n=40, noise_px=0.0, perturb_deg=0.0),
    "noisy_60": dict(seed=2, n=60),
    "outliers10_120": dict(seed=3, n=120, outlier_frac=0.1),
    "outliers30_200": dict(seed=4, n=200, outlier_frac=0.3),
    "outliers20_1000": dict(seed=6, n=1000, outlier_frac=0.2),
    "no_ba_300": dict(seed=12, n=300, outlier_frac=0.1, ba_on=False),
    "verification_failed": dict(seed=13, n=50, ver_ok=False),
    "one_camera_missing": dict(seed=14, n=80, outlier_frac=0.1, drop_cam2=True),
    "ba_keeps_nothing": dict(seed=9, n=50, n_front=0),
    "isp_ratio": dict(seed=10, n=20, n_unverified=400),
    "isp_count": dict(seed=15, n=18, outlier_frac=0.3, n_unverified=4),
    "below_min_inliers": dict(seed=8, n=12),
    "rotation_170": dict(seed=16, n=100, outlier_frac=0.1, R_off_deg=170.0, ba_on=False),
    "rotation_179_9": dict(seed=17, n=60, R_off_deg=179.9, ba_on=False),
}


def _near_threshold(arrays: dict, name: str, base: dict, rel: float) -> None:
    """`base` with the threshold moved so that one verified row's squared distance is within |rel| of thr^2."""
    pre = ref.run_2view_reports(base["kp1"], base["kp2"], base["putative"], True, base["vmask"], base["R_pre"], base["t_pre"], None,
                                cam_from_vec(base["cam1"]), cam_from_vec(base["cam2"]))[0]
    d2 = pre["reproj_error_gt_model"]
    j = int(np.argsort(d2)[len(d2) // 2])
    u = dict(base, thr=np.array(np.sqrt(d2[j] * (1.0 + rel))), ba=np.array(False))
    _store(arrays, name, u)
    print(f"{name}: thr^2 / d2 - 1 = {u['thr'] ** 2 / d2[j] - 1:.3g}")


def make_scenes() -> None:
    arrays = {}
    names = []
    for name, kw in SCENES.items():
        u = _scene_unit(**kw)
        _store(arrays, name, u)
        names.append(name)
        print(f"{name}: ver {int(u['vmask'].sum())} ba {bool(u['ba'])} post rows {int(u['pmask'].sum())} isp_ok "
              f"{bool(arrays[name + '/isp_ok'])} R_err {arrays[name + '/pre/scalars'][4]:.6g}")
    base = _scene_unit(seed=18, n=80, outlier_frac=0.1, ba_on=False)
    for name, rel in (("near_thr_above", 5e-10), ("near_thr_below", -5e-10)):
        _near_threshold(arrays, name, base, rel)
        names.append(name)
    arrays["names"] = np.array(names)
    arrays["fields"] = np.array(ref.FIELDS)
    np.savez_compressed(OUT_SCENES, **arrays)
    print(OUT_SCENES)


# ---- pinning against the reference ------------------------------------------------------------------------------------
class _Rot3:
    def __init__(self, R):
        self.R = np.asarray(R, float)

    def between(self, o):
        return _Rot3(self.R.T @ o.R)

    def matrix(self):
        return self.R


class _Unit3:
    def __init__(self, v):
        self.v = np.asarray(v, float) / np.linalg.norm(v)

    def point3(self):
        return self.v


class _Essential:
    def __init__(self, R, U):
        u = U.point3()
        self.E = np.array([[0.0, -u[2], u[1]], [u[2], 0.0, -u[0]], [-u[1], u[0], 0.0]]) @ R.matrix()

    def matrix(self):
        return self.E


class _Cal:
    def __init__(self, f, u0, v0):
        self._K = np.array([[f, 0.0, u0], [0.0, f, v0], [0.0, 0.0, 1.0]])

    def K(self):
        return self._K


def _functions(path: Path, names, ns: dict) -> dict:
    tree = ast.parse(path.read_text())
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module([node], []), str(path), "exec"), ns)
    return ns


def _pin_against_reference(reference: Path) -> None:
    """The restatement equals the reference's functions, run from the checkout's sources under stand-ins."""
    import types

    from scipy.spatial.transform import Rotation

    from gtsfm_b200.gtsfm_api import TwoViewEstimationReport

    g = reference / "gtsfm"
    ns = {"np": np, "Optional": __import__("typing").Optional, "Tuple": __import__("typing").Tuple, "Rotation": Rotation,
          "Rot3": _Rot3, "Unit3": _Unit3, "EssentialMatrix": _Essential, "TwoViewEstimationReport": TwoViewEstimationReport,
          "CALIBRATION_TYPE": object}
    _functions(g / "utils/features.py", {"convert_to_homogenous_coordinates", "convert_to_epipolar_lines", "point_line_dotproduct"}, ns)
    ns["feature_utils"] = types.SimpleNamespace(**{k: ns[k] for k in ("convert_to_epipolar_lines", "point_line_dotproduct")})
    _functions(g / "utils/verification.py", {"compute_epipolar_distances_sq_sampson", "essential_to_fundamental_matrix"}, ns)
    _functions(g / "utils/geometry_comparisons.py", {"compute_relative_rotation_angle", "compute_relative_unit_translation_angle"}, ns)
    _functions(g / "two_view_estimator.py", {"_masked_nanmean", "generate_two_view_report"}, ns)
    rng = np.random.default_rng(0)
    for trial in range(50):
        R = tvb._rot(rng.normal(size=3), rng.uniform(0, 180))
        t = rng.normal(size=3)
        c1, c2 = (rng.uniform(400, 900), rng.uniform(300, 400), rng.uniform(200, 300)), (rng.uniform(400, 900), 320.0, 240.0)
        F_ref = ns["essential_to_fundamental_matrix"](_Essential(_Rot3(R), _Unit3(t)), _Cal(*c1), _Cal(*c2))
        F = ref.gt_fundamental(R, t, c1, c2)
        assert np.allclose(F, F_ref, rtol=1e-12, atol=1e-15 * np.abs(F_ref).max()), (F, F_ref)
        x1, x2 = rng.uniform(0, 800, (30, 2)), rng.uniform(0, 800, (30, 2))
        assert np.allclose(ref.sampson_sq(x1, x2, F), ns["compute_epipolar_distances_sq_sampson"](x1, x2, F), rtol=1e-13, atol=0)
        Ra = tvb._rot(rng.normal(size=3), rng.uniform(0, 180))
        assert ref.rotation_angle_deg(Ra, R) == ns["compute_relative_rotation_angle"](_Rot3(Ra), _Rot3(R))
        assert ref.unit_angle_deg(t, x1[0].tolist() + [1.0]) == ns["compute_relative_unit_translation_angle"](_Unit3(t), _Unit3(x1[0].tolist() + [1.0]))
        d2 = rng.uniform(0, 40, 25)
        d2[rng.integers(0, 25, 3)] = np.nan
        mask = d2 < 16.0
        rows = rng.integers(0, 100, (25, 2))
        a = ref.generate_two_view_report(0.3, rows, 1.0, 2.0, mask, d2)
        b = ns["generate_two_view_report"](0.3, rows, 1.0, 2.0, mask, d2)
        for f in ref.FIELDS:
            x, y = a[f], getattr(b, f)
            assert (x is None and y is None) or np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True), f
        for inv in (False, True):
            x, y = ref.masked_nanmean(d2, mask, inv), ns["_masked_nanmean"](d2, mask, inv)
            assert x == y or (np.isnan(x) and np.isnan(y))
    b = ns["generate_two_view_report"](0.0, np.zeros((0, 2), np.int64))
    a = ref.generate_two_view_report(0.0, np.zeros((0, 2), np.int64))
    assert all((a[f] is None and getattr(b, f) is None) or np.array_equal(np.asarray(a[f]), np.asarray(getattr(b, f)), equal_nan=True)
               for f in ref.FIELDS)
    print("restatement equals the reference's Sampson, F, angle, _masked_nanmean and generate_two_view_report")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, required=True, help="a GTSfM checkout (data.mat and the pinned functions)")
    a = ap.parse_args()
    _pin_against_reference(a.reference)
    make_scenes()
    make_lund(a.reference)


if __name__ == "__main__":
    main()
