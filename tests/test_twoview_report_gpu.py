"""GPU suite for the two-view reports: k_tv_eval (b2_twoview_eval_batched_dev) against the NumPy oracle on both fixtures,
batch independence, and the reports B200TwoViewBatch.run returns."""
import math

import numpy as np
import pytest
import torch

from oracle import make_golden_twoview_report as mg
from oracle import twoview_report_ref as ref

pytestmark = pytest.mark.gpu

GOLDEN = __import__("pathlib").Path(__file__).resolve().parent / "golden"
REL, ABS = 1e-9, 1e-12


@pytest.fixture(scope="module")
def fe():
    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFrontEnd

    return DeviceFrontEnd(syn.superpoint_state_dict(0), max_keypoints=64)


def _load(which):
    d = np.load(GOLDEN / f"twoview_report_{which}.npz")
    names = [str(n) for n in d["names"]] if "names" in d else [f"{a}_{b}" for a, b in d["pairs"]]
    return d, names


def _units(d, names):
    """-> [(name, stage, EvalUnit, ratio, rows_host)] of every fixture stage with ground truth and an evaluation."""
    from gtsfm_b200.pipeline import EvalUnit

    out = []
    for name in names:
        u = mg.load_unit(d, name)
        c1, c2 = mg.cam_from_vec(u["cam1"]), mg.cam_from_vec(u["cam2"])
        if not bool(u["ver_ok"]):
            continue
        kp1, kp2 = torch.from_numpy(np.ascontiguousarray(u["kp1"])).cuda(), torch.from_numpy(np.ascontiguousarray(u["kp2"])).cuda()
        m = torch.from_numpy(u["putative"]).cuda()
        put = u["putative"]
        ratio = float(u["vmask"].sum()) / len(put)
        out.append((name, "pre", EvalUnit(kp1, kp2, m, torch.from_numpy(u["vmask"]).cuda(), (u["R_pre"], u["t_pre"]), c1, c2), ratio,
                    put[u["vmask"].astype(bool)]))
        if bool(u["ba"]):
            pose = (u["R_post"], u["t_post"]) if bool(u["post_pose"]) else None
            out.append((name, "post", EvalUnit(kp1, kp2, m, torch.from_numpy(u["pmask"]).cuda(), pose, c1, c2), ratio,
                        put[u["pmask"].astype(bool)]))
    return out


def _compare(d, name, stage, rep, near):
    """A device report against the fixture's; -> the number of rows within REL of the threshold whose mask differs."""
    exp = {f: (None if none else v) for f, v, none in zip(ref.SCALARS, d[f"{name}/{stage}/scalars"], d[f"{name}/{stage}/none"])}
    assert np.array_equal(rep.v_corr_idxs, d[f"{name}/{stage}/v_corr_idxs"])
    thr2 = float(d[f"{name}/thr"]) ** 2
    flips = 0
    if f"{name}/{stage}/mask" in d:
        d2, mask = d[f"{name}/{stage}/d2"], d[f"{name}/{stage}/mask"]
        assert rep.reproj_error_gt_model is not None
        fin = np.isfinite(d2)
        assert np.array_equal(np.isnan(rep.reproj_error_gt_model), np.isnan(d2))
        assert np.all(np.abs(rep.reproj_error_gt_model[fin] - d2[fin]) <= REL * np.abs(d2[fin]) + ABS), (name, stage)
        diff = rep.v_corr_idxs_inlier_mask_gt != mask
        assert np.all(np.abs(d2[diff] / thr2 - 1.0) < REL), (name, stage)
        flips += int(diff.sum())
        near[0] += int(diff.sum())
        n_in = int(rep.v_corr_idxs_inlier_mask_gt.sum())
        assert rep.num_inliers_gt_model == n_in and rep.inlier_ratio_gt_model == n_in / len(rep.v_corr_idxs)
    else:
        assert rep.reproj_error_gt_model is None and rep.v_corr_idxs_inlier_mask_gt is None
        assert rep.num_inliers_gt_model == exp["num_inliers_gt_model"] and math.isnan(rep.inlier_ratio_gt_model)
    for f in ("inlier_avg_reproj_error_gt_model", "outlier_avg_reproj_error_gt_model"):
        a, b = getattr(rep, f), exp[f]
        if flips == 0:
            assert (math.isnan(a) and math.isnan(b)) or abs(a - b) <= REL * abs(b) + ABS, (name, stage, f, a, b)
    for f in ("R_error_deg", "U_error_deg"):
        a, b = getattr(rep, f), exp[f]
        assert (a is None) == (b is None), (name, stage, f)
        if a is not None:
            assert abs(a - b) < 1e-5, (name, stage, f, a, b)
    assert rep.num_inliers_est_model == exp["num_inliers_est_model"] and rep.inlier_ratio_est_model == exp["inlier_ratio_est_model"]


@pytest.mark.parametrize("which", ["scenes", "lund_door"])
def test_eval_matches_oracle(fe, which):
    from gtsfm_b200.two_view import _stage_report

    d, names = _load(which)
    units = _units(d, names)
    res = fe.evaluate_many([u[2] for u in units], 4.0) if which == "lund_door" else None
    near = [0]
    # scenes carry their own thresholds: one call per threshold
    if res is None:
        res = [None] * len(units)
        for thr in sorted({float(d[f"{u[0]}/thr"]) for u in units}):
            idx = [i for i, u in enumerate(units) if float(d[f"{u[0]}/thr"]) == thr]
            for i, r in zip(idx, fe.evaluate_many([units[i][2] for i in idx], thr)):
                res[i] = r
    for (name, stage, unit, ratio, rows), ev in zip(units, res):
        _compare(d, name, stage, _stage_report(rows, ratio, unit.pose, ev), near)
    assert near[0] <= 2


def _key(r):
    res, d2, inl = r
    return (res.num_rows, res.num_inliers_gt, res.no_gt, res.no_rows, np.float64(res.inlier_avg_reproj_error_gt).tobytes(),
            np.float64(res.outlier_avg_reproj_error_gt).tobytes(), np.float64(res.R_error_deg).tobytes(),
            np.float64(res.U_error_deg).tobytes(), d2.numpy().tobytes(), inl.numpy().tobytes())


def test_batches_equal_one_at_a_time(fe):
    d, names = _load("lund_door")
    units = [u[2] for u in _units(d, names)]
    single = [_key(fe.evaluate_many([u])[0]) for u in units]
    for b in (1, 8, 33):
        got = []
        for c0 in range(0, len(units), b):
            got += [_key(r) for r in fe.evaluate_many(units[c0:c0 + b])]
        assert got == single, b


def _lund_batch():
    from gtsfm_b200.pipeline import DeviceFeatures

    d, names = _load("lund_door")
    kps = {i: torch.from_numpy(np.ascontiguousarray(d[f"kp_{i}"])).cuda() for i in range(1, 13)}
    feats = {i: DeviceFeatures(k, torch.zeros(len(k), device="cuda"), torch.zeros((len(k), 1), device="cuda"), (0, 0))
             for i, k in kps.items()}
    pairs = [tuple(int(x) for x in p) for p in d["pairs"]]
    putative = {p: torch.from_numpy(d[f"{p[0]}_{p[1]}/putative"]).cuda() for p in pairs}
    cams = {}
    for p in pairs:
        cams[p[0]] = mg.cam_from_vec(d[f"{p[0]}_{p[1]}/cam1"])
        cams[p[1]] = mg.cam_from_vec(d[f"{p[0]}_{p[1]}/cam2"])
    from oracle.make_golden_twoview_ba import lund_inputs

    cal = lund_inputs()[3]
    return d, feats, pairs, putative, cams, {i: cal for i in range(1, 13)}


def _dict(rep):
    return {f: getattr(rep, f) for f in ref.FIELDS}


@pytest.mark.parametrize("ba", [False, True])
def test_run_reports_equal_oracle_on_its_own_outputs(fe, ba):
    """B200TwoViewBatch.run with ground truth: every report equals the oracle's run_2view_reports on the rows and poses the
    device produced; without ground truth R, U, rows and ratio are those of the run with it, and the estimated-model
    fields are filled; a mesh raises."""
    from gtsfm_b200.two_view import B200TwoViewBatch

    d, feats, pairs, putative, cams, intr = _lund_batch()
    tvb = B200TwoViewBatch(fe, 4.0, bundle_adjust_2view=ba)
    with pytest.raises(ValueError):
        tvb.run(feats, pairs[:2], intr, putative, gt_cameras=cams, gt_scene_mesh=object())
    cams_missing = dict(cams)
    cams_missing[12] = None  # pairs with image 12 have no ground truth
    res = tvb.run(feats, pairs, intr, putative, gt_cameras=cams_missing)
    plain = tvb.run(feats, pairs, intr, putative)
    near = 0
    for p in pairs:
        r, q = res[p], plain[p]
        assert (r.i2Ri1 is None) == (q.i2Ri1 is None) and np.array_equal(r.v_corr_idxs, q.v_corr_idxs)
        assert r.v_corr_idxs.dtype == q.v_corr_idxs.dtype and r.inlier_ratio_est_model == q.inlier_ratio_est_model
        if r.i2Ri1 is not None:
            assert np.array_equal(r.i2Ri1.matrix(), q.i2Ri1.matrix()) and np.array_equal(r.i2Ui1.point3(), q.i2Ui1.point3())
        assert q.pre_ba_report is not None and q.pre_ba_report.num_inliers_est_model == q.pre_ba_report.v_corr_idxs.shape[0]
        assert q.pre_ba_report.R_error_deg is None and q.pre_ba_report.num_inliers_gt_model == 0
        assert np.array_equal(r.putative_corr_idxs, d[f"{p[0]}_{p[1]}/putative"])
        # the oracle on the device's own rows and poses
        pre = r.pre_ba_report
        m = r.putative_corr_idxs
        ok = pre.num_inliers_est_model > 0 or r.inlier_ratio_est_model > 0
        row_of = {tuple(x): j for j, x in enumerate(m)}
        vmask = np.zeros(len(m), bool)
        vmask[[row_of[tuple(x)] for x in pre.v_corr_idxs]] = True
        post = None
        if ba and ok and vmask.sum() >= 15:
            pm = np.zeros(len(m), bool)
            pm[[row_of[tuple(x)] for x in r.post_ba_report.v_corr_idxs]] = True
            post = (None, None, pm)
        c1, c2 = cams_missing.get(p[0]), cams_missing.get(p[1])
        # without BA the returned pose is the pre-BA estimate, so the oracle gets it and the pose errors are compared too
        R_pre, t_pre = (r.i2Ri1.matrix(), r.i2Ui1.point3()) if (not ba and r.i2Ri1 is not None) else (None, None)
        e_pre, e_post, e_isp, e_ok = ref.run_2view_reports(d[f"kp_{p[0]}"], d[f"kp_{p[1]}"], m, ok, vmask, R_pre, t_pre, post, c1, c2)
        for got, exp in ((r.pre_ba_report, e_pre), (r.post_ba_report, e_post), (r.post_isp_report, e_isp)):
            g = _dict(got)
            assert np.array_equal(g["v_corr_idxs"], exp["v_corr_idxs"])
            assert g["num_inliers_est_model"] == exp["num_inliers_est_model"]
            assert (g["inlier_ratio_est_model"] is None) == (exp["inlier_ratio_est_model"] is None)
            if exp["reproj_error_gt_model"] is None:
                assert g["reproj_error_gt_model"] is None and g["num_inliers_gt_model"] == exp["num_inliers_gt_model"]
            else:
                a, b = g["reproj_error_gt_model"], exp["reproj_error_gt_model"]
                assert np.all(np.abs(a - b) <= REL * np.abs(b) + ABS)
                near += int((g["v_corr_idxs_inlier_mask_gt"] != exp["v_corr_idxs_inlier_mask_gt"]).sum())
            if not ba:
                for f in ("R_error_deg", "U_error_deg"):
                    assert (g[f] is None) == (exp[f] is None), (p, f)
                    if g[f] is not None:
                        assert abs(g[f] - exp[f]) < 1e-5, (p, f, g[f], exp[f])
        assert (r.post_isp_report.inlier_ratio_est_model is None) == (not e_ok)
    assert near <= 2


def test_launch_count_grows_by_one_per_chunk(fe):
    from gtsfm_b200.two_view import MATCH_BATCH, B200TwoViewBatch

    d, feats, pairs, putative, cams, intr = _lund_batch()
    tvb = B200TwoViewBatch(fe, 4.0)
    tvb.run(feats, pairs[:8], intr, putative)  # the verification lane exists from here on
    ctx = fe._vctx
    n0 = ctx.launch_count()
    tvb.run(feats, pairs, intr, putative)
    n1 = ctx.launch_count()
    tvb.run(feats, pairs, intr, putative, gt_cameras=cams)
    n2 = ctx.launch_count()
    chunks = (len(pairs) + MATCH_BATCH - 1) // MATCH_BATCH
    assert (n2 - n1) - (n1 - n0) == chunks
