"""NumPy statement of the two-view reports GTSfM's run_2view returns per pair (pre_ba_report, post_ba_report,
post_isp_report) and of their ground-truth metrics: the contract of csrc/twoview_eval.cu and of the report assembly in
gtsfm_b200/two_view.py.

    run_2view                         gtsfm/two_view_estimator.py:350-481
    __get_2view_report_from_results   gtsfm/two_view_estimator.py:290-344
    _masked_nanmean                   gtsfm/two_view_estimator.py:654-660
    generate_two_view_report          gtsfm/two_view_estimator.py:663-702
    compute_relative_pose_metrics     gtsfm/two_view_estimator.py:705-731
    compute_correspondence_metrics    gtsfm/utils/metrics.py:38-96 (Sampson branch; a mesh is out of scope)
    epipolar_inlier_correspondences   gtsfm/utils/metrics.py:99-129
    essential_to_fundamental_matrix   gtsfm/utils/verification.py:115
    compute_epipolar_distances_sq_sampson  gtsfm/utils/verification.py:172-216
    compute_relative_rotation_angle / _unit_translation_angle  gtsfm/utils/geometry_comparisons.py:137-180
    InlierSupportProcessor.run_inlier_support  gtsfm/frontend/inlier_support_processor.py:39-95

A ground-truth camera is (R_wTi (3, 3), t_wTi (3,), f, u0, v0): gtsam's PinholeCameraCal3Bundler with k1 = k2 = 0.  A
report is a dict over FIELDS (TwoViewEstimationReport's fields, gtsfm/common/two_view_estimation_report.py:43-56, in
order), None where the reference leaves None.
"""
from __future__ import annotations

import warnings
from typing import Optional, Sequence, Tuple

import numpy as np
from scipy.spatial.transform import Rotation

# TwoViewEstimationReport's fields and defaults, in declaration order
FIELDS = ("v_corr_idxs", "num_inliers_est_model", "inlier_ratio_est_model", "num_inliers_gt_model", "inlier_ratio_gt_model",
          "v_corr_idxs_inlier_mask_gt", "R_error_deg", "U_error_deg", "i2Ri1", "i2Ui1", "reproj_error_gt_model",
          "inlier_avg_reproj_error_gt_model", "outlier_avg_reproj_error_gt_model")
SCALARS = ("num_inliers_est_model", "inlier_ratio_est_model", "num_inliers_gt_model", "inlier_ratio_gt_model", "R_error_deg",
           "U_error_deg", "inlier_avg_reproj_error_gt_model", "outlier_avg_reproj_error_gt_model")


def empty_report(v_corr_idxs, num_inliers_est_model) -> dict:
    """TwoViewEstimationReport(v_corr_idxs=..., num_inliers_est_model=...) with every other field at its default (None)."""
    r = {f: None for f in FIELDS}
    r["v_corr_idxs"], r["num_inliers_est_model"] = v_corr_idxs, num_inliers_est_model
    return r


def gt_relative(cam1, cam2) -> Tuple[np.ndarray, np.ndarray]:
    """wTi2.between(wTi1) = wTi2^-1 wTi1 -> (R, t)."""
    R1, t1 = np.asarray(cam1[0], float), np.asarray(cam1[1], float)
    R2, t2 = np.asarray(cam2[0], float), np.asarray(cam2[1], float)
    return R2.T @ R1, R2.T @ (t1 - t2)


def k_inv(cal) -> np.ndarray:
    f, u0, v0 = (float(c) for c in cal)
    return np.array([[1.0 / f, 0.0, -u0 / f], [0.0, 1.0 / f, -v0 / f], [0.0, 0.0, 1.0]])


def gt_fundamental(R, t, cal1, cal2) -> np.ndarray:
    """EssentialMatrix(R, Unit3(t)).matrix() = [t / |t|]x R, then K2^-T E K1^-1 (verification.py:115)."""
    u = np.asarray(t, float) / np.linalg.norm(t)
    S = np.array([[0.0, -u[2], u[1]], [u[2], 0.0, -u[0]], [-u[1], u[0], 0.0]])
    return k_inv(cal2).T @ (S @ np.asarray(R, float)) @ k_inv(cal1)


def sampson_sq(x1: np.ndarray, x2: np.ndarray, F: np.ndarray) -> np.ndarray:
    """compute_epipolar_distances_sq_sampson for (n, 2) coordinates (not None: callers pass n > 0)."""
    h1 = np.hstack([x1, np.ones((len(x1), 1))])
    h2 = np.hstack([x2, np.ones((len(x2), 1))])
    l2 = h1 @ F.T  # convert_to_epipolar_lines(x1, F)
    l1 = h2 @ F    # convert_to_epipolar_lines(x2, F.T)
    den = np.sum(np.square(l1[:, :2]), axis=1) + np.sum(np.square(l2[:, :2]), axis=1)
    return np.square(np.sum(h1 * l1, axis=1)) / den


def rotation_angle_deg(Ra, Rb) -> Optional[float]:
    """compute_relative_rotation_angle: |rotvec(Ra.between(Rb))| in degrees (scipy, through a quaternion)."""
    if Ra is None or Rb is None:
        return None
    rel = np.asarray(Ra, float).T @ np.asarray(Rb, float)
    return float(np.rad2deg(np.linalg.norm(Rotation.from_matrix(rel).as_rotvec())))


def unit_angle_deg(a, b) -> Optional[float]:
    """compute_relative_unit_translation_angle of Unit3(a), Unit3(b)."""
    if a is None or b is None:
        return None
    ua, ub = np.asarray(a, float) / np.linalg.norm(a), np.asarray(b, float) / np.linalg.norm(b)
    return float(np.rad2deg(np.arccos(np.clip(np.dot(ua, ub), -1, 1))))


def masked_nanmean(model, mask, invert_mask: bool = False) -> float:
    """_masked_nanmean (two_view_estimator.py:654-660)."""
    if model is not None and mask is not None and len(mask) > 0:
        final_mask = np.logical_not(mask) if invert_mask else mask
        if np.any(final_mask):
            with warnings.catch_warnings():  # an all-NaN selection is NaN, as np.nanmean warns
                warnings.simplefilter("ignore", RuntimeWarning)
                return float(np.nanmean(model[final_mask]))
    return float("nan")


def generate_two_view_report(inlier_ratio_est_model, v_corr_idxs, R_error_deg=None, U_error_deg=None,
                             v_corr_idxs_inlier_mask_gt=None, reproj_error_gt_model=None) -> dict:
    """generate_two_view_report (two_view_estimator.py:663-702)."""
    if v_corr_idxs_inlier_mask_gt is not None and reproj_error_gt_model is not None:
        num_inliers_gt_model = np.count_nonzero(v_corr_idxs_inlier_mask_gt)
        inlier_ratio_gt_model = (np.count_nonzero(v_corr_idxs_inlier_mask_gt) / v_corr_idxs.shape[0]
                                 if len(v_corr_idxs) > 0 else 0.0)
        inlier_avg = masked_nanmean(reproj_error_gt_model, v_corr_idxs_inlier_mask_gt)
        outlier_avg = masked_nanmean(reproj_error_gt_model, v_corr_idxs_inlier_mask_gt, invert_mask=True)
    else:
        num_inliers_gt_model = 0
        inlier_ratio_gt_model = float("nan")
        inlier_avg = float("nan")
        outlier_avg = float("nan")
    r = empty_report(v_corr_idxs, v_corr_idxs.shape[0])
    r.update(inlier_ratio_est_model=inlier_ratio_est_model, num_inliers_gt_model=num_inliers_gt_model,
             inlier_ratio_gt_model=inlier_ratio_gt_model, v_corr_idxs_inlier_mask_gt=v_corr_idxs_inlier_mask_gt,
             R_error_deg=R_error_deg, U_error_deg=U_error_deg, reproj_error_gt_model=reproj_error_gt_model,
             inlier_avg_reproj_error_gt_model=inlier_avg, outlier_avg_reproj_error_gt_model=outlier_avg)
    return r


def stage_report(kp1, kp2, rows: np.ndarray, ratio: float, R, t, cam1, cam2, thr_px: float) -> dict:
    """__get_2view_report_from_results: `rows` (n, 2) indices into kp1 / kp2; R, t the stage's estimate (None: none)."""
    if cam1 is not None and cam2 is not None:
        Rg, tg = gt_relative(cam1, cam2)
        R_err, U_err = rotation_angle_deg(R, Rg), unit_angle_deg(t, tg)
        if rows.size == 0:
            mask, d2 = None, None
        else:
            F = gt_fundamental(Rg, tg, cam1[2:], cam2[2:])
            x1 = np.asarray(kp1, np.float64)[rows[:, 0]]
            x2 = np.asarray(kp2, np.float64)[rows[:, 1]]
            with np.errstate(divide="ignore", invalid="ignore"):
                d2 = sampson_sq(x1, x2, F)
            mask = d2 < thr_px ** 2
    else:
        R_err, U_err, mask, d2 = None, None, None, None
    return generate_two_view_report(ratio, rows, R_err, U_err, mask, d2)


def inlier_support(report: dict, v_corr_idxs, min_num_inliers: int, min_ratio: float) -> Tuple[bool, dict]:
    """run_inlier_support's decision and report: -> (success, post_isp_report)."""
    fail = empty_report(v_corr_idxs, 0)
    if report["inlier_ratio_est_model"] < min_ratio:
        return False, fail
    if report["num_inliers_est_model"] > 0 and report["num_inliers_est_model"] < min_num_inliers:
        return False, fail
    return True, dict(report)


def run_2view_reports(kp1, kp2, putative: np.ndarray, verified_ok: bool, vmask: Optional[np.ndarray], R_pre, t_pre,
                      post: Optional[Tuple], cam1, cam2, thr_px: float = 4.0, min_num_inliers: int = 15,
                      min_ratio: float = 0.1) -> Tuple[dict, dict, dict, bool]:
    """The three reports of one pair.  `putative` (k, 2) match rows; `vmask` (k,) the verifier's inlier mask; `post`: the
    two-view BA's (R | None, t | None, kept-row mask (k,)) when bundle adjustment ran for the pair (bundle_adjust_2view and
    at least min_num_inliers verified rows), else None.  -> (pre_ba, post_ba, post_isp, isp success)."""
    putative = np.asarray(putative, np.int64).reshape(-1, 2)
    k = len(putative)
    if verified_ok:
        rows = putative[np.asarray(vmask, bool)]
        ratio = float(len(rows)) / float(k)
    else:  # verifier_base.py:60-64 / opencv_verifier_base.py:70-79
        rows, ratio, R_pre, t_pre = np.zeros((0, 2), np.int64), 0.0, None, None
    pre = stage_report(kp1, kp2, rows, ratio, R_pre, t_pre, cam1, cam2, thr_px)
    if post is not None:
        R_post, t_post, pmask = post
        post_rows = putative[np.asarray(pmask, bool)]
        post_ba = stage_report(kp1, kp2, post_rows, ratio, R_post, t_post, cam1, cam2, thr_px)  # the pre-BA ratio (:426)
    else:
        post_rows, post_ba = rows, dict(pre)  # dataclasses.replace(pre_ba_report)
    ok, post_isp = inlier_support(post_ba, post_rows, min_num_inliers, min_ratio)
    return pre, post_ba, post_isp, ok
