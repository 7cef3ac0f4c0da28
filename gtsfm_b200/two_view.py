"""Batched two-view seam (SURVEY.md §8f rank 1): the device half of `TwoViewEstimator.run_2view` for a shard of pairs.

The reference runs, per pair and per Dask task (gtsfm/two_view_estimator.py:350-481, 846-886): `normalize_coordinates`
(a Python loop of gtsam calls over every keypoint, gtsfm/utils/features.py:41-51), `cv2.findEssentialMat` +
`cv2.recoverPose` (gtsfm/frontend/verifier/ransac.py:74-81, gtsfm/utils/verification.py:83) and then hands the inliers
to triangulation / bundle adjustment on the CPU.  Here a whole shard of pairs is walked on one GPU with every keypoint
and match tensor resident in HBM: calibration, hypothesis generation, scoring, local optimisation, the inlier mask
and the cheirality vote are the kernels of csrc/ransac.cu (`b2_ransac_verify_batched_dev`: one call per matched chunk of
up to 8 pairs, every stage launched once for the chunk), chunk c's verification runs on its own stream under chunk c+1's
matching, and only what the CPU back half consumes leaves the device: the verified rows
of the match array, R, t and the inlier ratio - exactly the `VerifierBase.verify` tuple (verifier_base.py:67-90).

With `bundle_adjust_2view=True` each chunk's verification is followed, on the same stream, by the rest of `run_2view`
(:410-450): triangulation, the two-view bundle adjustment and the inlier-support thresholds (csrc/twoview_ba.cu,
`b2_twoview_ba_batched_dev`), and the rows, R and t handed back are the refined ones.  Off by default.

Every result also carries run_2view's three reports (pre_ba_report, post_ba_report, post_isp_report, :375-450) and the
putative rows.  Their estimated-model fields are assembled on the host from what the chunk brings back anyway; with
ground-truth cameras for both images of a pair, their ground-truth metrics (Sampson distances under the ground-truth F,
the inlier mask, its averages, the pose errors) come from csrc/twoview_eval.cu, one launch per chunk on the verification
lane behind the chunk's verification (and refinement).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace
from typing import Dict, Iterable, List, Mapping, Optional, Sequence, Tuple

import numpy as np
import torch

from .gtsfm_api import Rot3, TwoViewEstimationReport, Unit3
from .pipeline import DeviceFeatures, DeviceFrontEnd, EvalUnit, RefineOptions
from .verifier import DEFAULT_SEED

MIN_MATCHES_E = 6  # opencv_verifier_base.py:77-79
MATCH_BATCH = 8    # pairs per lock-step LightGlue batch (the library maximum)


@dataclass
class TwoViewResult:
    i2Ri1: Optional[Rot3]
    i2Ui1: Optional[Unit3]
    v_corr_idxs: np.ndarray  # (n, 2) rows of the putative match array that survived verification (host)
    inlier_ratio_est_model: float
    num_putative: int
    # run_2view's reports (gtsfm/products/two_view_result.py) and the putative rows (host)
    pre_ba_report: Optional[TwoViewEstimationReport] = None
    post_ba_report: Optional[TwoViewEstimationReport] = None
    post_isp_report: Optional[TwoViewEstimationReport] = None
    putative_corr_idxs: Optional[np.ndarray] = None

    def valid(self) -> bool:
        return self.i2Ri1 is not None and self.i2Ui1 is not None


def _failure(num_putative: int) -> TwoViewResult:  # verifier_base.py:60-64
    return TwoViewResult(None, None, np.zeros((0, 2), np.int64), 0.0, num_putative)


def _refined_failure(ratio: float, num_putative: int) -> TwoViewResult:  # inlier_support_processor.py failure_result
    return TwoViewResult(None, None, np.array([], np.uint64), ratio, num_putative)


@dataclass
class ReportOptions:
    """What the reports need beyond the chunk: ground-truth cameras {image: (R_wTi, t_wTi, f, u0, v0)} (None: none), the
    Sampson threshold of a correct correspondence, and the inlier-support thresholds (inlier_support_processor.py)."""
    gt_cameras: Optional[Mapping[int, tuple]] = None
    eval_threshold_px: float = 4.0
    min_num_inliers_est_model: int = 15
    min_inlier_ratio_est_model: float = 0.1

    def cams(self, pair) -> Tuple[Optional[tuple], Optional[tuple]]:
        if not self.gt_cameras:
            return None, None
        return self.gt_cameras.get(pair[0]), self.gt_cameras.get(pair[1])


def gt_camera(cam) -> Optional[tuple]:
    """A ground-truth camera as (R_wTi (3, 3), t_wTi (3,), f, u0, v0): from that tuple, or from a gtsam
    PinholeCameraCal3Bundler (distortion must be zero).  None stays None."""
    if cam is None:
        return None
    if hasattr(cam, "pose") and hasattr(cam, "calibration"):
        pose, cal = cam.pose(), cam.calibration()
        if cal.k1() != 0.0 or cal.k2() != 0.0:
            raise ValueError("ground-truth cameras with lens distortion are not supported")
        return (np.asarray(pose.rotation().matrix(), np.float64), np.asarray(pose.translation(), np.float64).ravel(),
                float(cal.fx()), float(cal.px()), float(cal.py()))
    R, t, f, u0, v0 = cam
    return (np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3), float(f), float(u0), float(v0))


class B200TwoViewBatch:
    """match (optional) -> calibrate -> RANSAC-5pt (or LMedS-5pt) -> recoverPose for a list of pairs, device-resident.

    `intrinsics[i]` = (f, u0, v0) of image i (Cal3Bundler without distortion: what GTSfM's deep front-end configs use).
    `method`: "ransac" (the reference's Ransac verifier) or "lmeds" (its LMEDS verifier; the threshold and seed are unused).
    `bundle_adjust_2view`: also triangulate, bundle-adjust and apply inlier support on the device, with the reference's
    TwoViewEstimator / InlierSupportProcessor arguments below (sift_front_end sets the triangulation threshold to 100).
    `eval_threshold_px`: the Sampson distance below which a correspondence is correct under the ground truth
    (TwoViewEstimator's corr_metric_dist_threshold; the configs' eval_threshold_px).
    """

    def __init__(self, front_end: DeviceFrontEnd, estimation_threshold_px: float = 4.0, seed: int = DEFAULT_SEED,
                 method: str = "ransac", bundle_adjust_2view: bool = False, ba_reproj_error_threshold: float = 0.5,
                 min_num_inliers_est_model: int = 15, min_inlier_ratio_est_model: float = 0.1,
                 triangulation_reproj_error_threshold: float = float("inf"), eval_threshold_px: float = 4.0):
        if method not in ("ransac", "lmeds"):
            raise ValueError(f"verification method must be 'ransac' or 'lmeds', not {method!r}")
        if not eval_threshold_px > 0.0:
            raise ValueError(f"eval_threshold_px must be > 0, not {eval_threshold_px!r}")
        self.fe = front_end
        self.threshold_px = float(estimation_threshold_px)
        self.seed = int(seed)
        self.method = method
        self.refine = RefineOptions(ba_reproj_error_threshold, min_num_inliers_est_model, min_inlier_ratio_est_model,
                                    triangulation_reproj_error_threshold) if bundle_adjust_2view else None
        self.report = ReportOptions(None, float(eval_threshold_px), int(min_num_inliers_est_model), float(min_inlier_ratio_est_model))

    def report_options(self, gt_cameras=None, gt_scene_mesh=None) -> ReportOptions:
        if gt_scene_mesh is not None:
            raise ValueError("mesh-based ground-truth metrics are not supported; pass gt_scene_mesh=None (Sampson metrics)")
        cams = None if gt_cameras is None else {i: gt_camera(c) for i, c in gt_cameras.items()}
        return replace(self.report, gt_cameras=cams)

    def run(self, features: Mapping[int, DeviceFeatures], pairs: Iterable[Tuple[int, int]], intrinsics: Mapping[int, Sequence[float]],
            putative: Optional[Mapping[Tuple[int, int], torch.Tensor]] = None, gt_cameras: Optional[Mapping[int, object]] = None,
            gt_scene_mesh=None) -> Dict[Tuple[int, int], TwoViewResult]:
        """`putative[(i1, i2)]`: (k, 2) int64 device tensor of match indices; matched here with LightGlue when absent.
        `gt_cameras[i]`: image i's ground-truth camera, (R_wTi, t_wTi, f, u0, v0) or a gtsam PinholeCameraCal3Bundler; a
        pair with a camera missing (or None) gets no ground-truth metrics.  A mesh (`gt_scene_mesh`) raises ValueError."""
        rep = self.report_options(gt_cameras, gt_scene_mesh)
        out: Dict[Tuple[int, int], TwoViewResult] = {}
        pending = []  # chunks in flight on the verification stream
        pairs = list(pairs)
        for c0 in range(0, len(pairs), MATCH_BATCH):
            chunk = pairs[c0:c0 + MATCH_BATCH]
            todo = [pr for pr in chunk if putative is None or pr not in putative]
            matched = dict(zip(todo, self.fe.match_batch([(features[i1], features[i2]) for i1, i2 in todo])))
            prs, items = [], []
            for i1, i2 in chunk:
                m = putative[(i1, i2)] if (i1, i2) not in matched else matched[(i1, i2)][0]
                k = int(m.shape[0])
                if k < MIN_MATCHES_E:
                    out[(i1, i2)] = _with_reports(_failure(k), m.cpu().numpy().astype(np.int64), rep)
                    continue
                prs.append((i1, i2))
                items.append((features[i1], features[i2], m, intrinsics[i1], intrinsics[i2]))
            if items:  # this chunk's verification: one call on its own stream / thread under the next chunk's matching
                pending.append(submit_chunk(self.fe, prs, items, self.threshold_px, self.seed, self.method, self.refine, rep))
            while len(pending) > 1:
                self._collect_chunk(pending.pop(0), out)
        for p in pending:
            self._collect_chunk(p, out)
        return out

    @classmethod
    def _collect_chunk(cls, chunk: "_Chunk", out) -> None:
        verified = chunk.vfut.result()
        refined = chunk.rfut.result() if chunk.rfut is not None else [None] * len(chunk.prs)
        evals = chunk.efut.result() if chunk.efut is not None else []
        # the chunk's putative rows and masks cross PCIe in one copy each; each pair's rows are host slices of them
        ks = [int(m.shape[0]) for m in chunk.ms]
        cuts = np.cumsum([0] + ks)
        put = torch.cat([m.reshape(-1, 2).to(torch.int64) for m in chunk.ms]).cpu().numpy()
        vmask = torch.cat([v[4] for v in verified]).cpu().numpy().astype(bool)
        pmask = torch.cat(chunk.post_masks).cpu().numpy().astype(bool) if chunk.post_masks is not None else None
        for j, (pair, v, r) in enumerate(zip(chunk.prs, verified, refined)):
            m = put[cuts[j]:cuts[j + 1]]
            vm = vmask[cuts[j]:cuts[j + 1]]
            res = cls._collect_one(m, v, vm) if chunk.rfut is None else cls._collect_refined(m, v, r)
            ev = {st: evals[u] for (jj, st), u in chunk.units.items() if jj == j}
            pm = pmask[cuts[j]:cuts[j + 1]] if pmask is not None else None
            out[pair] = _with_reports(res, m, chunk.rep, v, vm, r, pm, ev)

    @staticmethod
    def _collect_refined(m, verified, refined) -> TwoViewResult:
        k = len(m)
        if verified[0] is None:
            return _failure(k)
        ratio = float(verified[3]) / float(k)  # the ratio from before BA (two_view_estimator.py:426)
        R, t, rows, _ = refined
        if R is None:
            return _refined_failure(ratio, k)
        return TwoViewResult(Rot3(R), Unit3(t), rows.cpu().numpy().astype(np.int64), ratio, k)  # only the final rows cross PCIe

    @staticmethod
    def _collect_one(m, result, vm) -> TwoViewResult:
        E, R, t, n_inl, _ = result
        k = len(m)
        if E is None:
            return _failure(k)
        return TwoViewResult(Rot3(R), Unit3(t), m[vm], float(n_inl) / float(k), k)


@dataclass
class _Chunk:
    """A chunk in flight on the verification lane: its pairs and putative rows, the Futures of its verification,
    refinement (None: off) and evaluation (None: no ground truth in the chunk), the report options, the post-BA row masks
    refinement writes (None: off), and {(pair position, stage): evaluation unit}."""
    prs: list
    ms: list
    vfut: object
    rfut: object
    efut: object
    rep: ReportOptions
    post_masks: Optional[List[torch.Tensor]]
    units: Dict[Tuple[int, str], int]


def submit_chunk(fe: DeviceFrontEnd, prs, items, threshold_px: float, seed: int, method: str, refine: Optional[RefineOptions],
                 rep: Optional[ReportOptions] = None) -> _Chunk:
    """Queue one chunk's verification (and, with `refine`, its refinement right behind it, and with ground-truth cameras
    for some pair, its reports' evaluation behind that) on the verification lane.  -> the chunk `_collect_chunk` takes."""
    rep = rep or ReportOptions()
    vfut = fe.verify_many_async(items, threshold_px, seed, method)
    post_masks, rfut = None, None
    if refine is not None:
        lane = fe._verify_lane()
        with torch.cuda.stream(lane.stream):  # zero-filled on the stream the kernels use
            post_masks = [torch.zeros(int(it[2].shape[0]), dtype=torch.uint8, device=fe.device) for it in items]
        rfut = lane.pool.submit(lambda: fe.refine_many(items, vfut.result(), refine, lane.ctx, lane.stream, out_masks=post_masks))
    units: Dict[Tuple[int, str], int] = {}
    wanted = [(j, *rep.cams(pr)) for j, pr in enumerate(prs)]
    wanted = [(j, c1, c2) for j, c1, c2 in wanted if c1 is not None and c2 is not None]
    efut = None
    if wanted:
        def make_units() -> List[EvalUnit]:  # on the lane's thread, once verification (and refinement) are done
            ver = vfut.result()
            ref = rfut.result() if rfut is not None else None
            us: List[EvalUnit] = []
            for j, c1, c2 in wanted:
                a, b, m = items[j][:3]
                E, R, t, _, mask = ver[j]
                if E is None:
                    continue  # no rows: no ground-truth mask, and no estimate to compare
                units[(j, "pre")] = len(us)
                us.append(EvalUnit(a.kp, b.kp, m, mask, (R, t), c1, c2))
                r = ref[j][3] if ref is not None else None
                if r is not None and r.bundle_adjusted:
                    units[(j, "post")] = len(us)
                    pose = None if r.indeterminate else (np.array(r.R), np.array(r.t))
                    us.append(EvalUnit(a.kp, b.kp, m, post_masks[j], pose, c1, c2))
            return us

        efut = fe.evaluate_many_async(make_units, rep.eval_threshold_px)
    return _Chunk(prs, [it[2] for it in items], vfut, rfut, efut, rep, post_masks, units)


def _stage_report(rows: np.ndarray, ratio: float, pose, ev) -> TwoViewEstimationReport:
    """__get_2view_report_from_results + generate_two_view_report (two_view_estimator.py:290-344, 663-702) from the
    stage's rows and, with ground truth, its evaluation (b2_twoview_eval_result, distances, mask)."""
    R_err = U_err = mask = d2 = None
    n_gt, ratio_gt, avg_in, avg_out = 0, math.nan, math.nan, math.nan
    if ev is not None and not ev[0].no_gt:
        r, dist, inl = ev
        if pose is not None:
            R_err, U_err = float(r.R_error_deg), float(r.U_error_deg)
        if not r.no_rows:
            d2, mask = dist.numpy().copy(), inl.numpy().astype(bool)
            n_gt, ratio_gt = int(r.num_inliers_gt), int(r.num_inliers_gt) / rows.shape[0]
            avg_in, avg_out = float(r.inlier_avg_reproj_error_gt), float(r.outlier_avg_reproj_error_gt)
    return TwoViewEstimationReport(v_corr_idxs=rows, num_inliers_est_model=rows.shape[0], inlier_ratio_est_model=ratio,
                                   num_inliers_gt_model=n_gt, inlier_ratio_gt_model=ratio_gt, v_corr_idxs_inlier_mask_gt=mask,
                                   R_error_deg=R_err, U_error_deg=U_err, reproj_error_gt_model=d2,
                                   inlier_avg_reproj_error_gt_model=avg_in, outlier_avg_reproj_error_gt_model=avg_out)


def _with_reports(res: TwoViewResult, putative: np.ndarray, rep: ReportOptions, verified=None, vm=None, refined=None,
                  pm=None, ev=None) -> TwoViewResult:
    """`res` with run_2view's three reports (:375-450) and the putative rows.  `verified`: verify_many()'s tuple (None:
    fewer than 6 matches), `vm` its mask on the host; `refined`: refine_many()'s tuple (None: refinement off), `pm` the
    post-BA row mask; `ev` {stage: evaluate_many() entry}."""
    ev = ev or {}
    k = len(putative)
    if verified is not None and verified[0] is not None:
        pre_rows, ratio, pre_pose = putative[vm], float(verified[3]) / float(k), (verified[1], verified[2])
    else:
        pre_rows, ratio, pre_pose = np.zeros((0, 2), np.int64), 0.0, None
    pre = _stage_report(pre_rows, ratio, pre_pose, ev.get("pre"))
    r = refined[3] if refined is not None else None
    if r is not None and r.bundle_adjusted:  # :412-438
        post_rows = putative[pm]
        post = _stage_report(post_rows, ratio, None if r.indeterminate else (r.R, r.t), ev.get("post"))
    else:  # :439-443
        post_rows, post = pre_rows, replace(pre)
    # InlierSupportProcessor.run_inlier_support (inlier_support_processor.py:39-95)
    n = post.num_inliers_est_model
    if post.inlier_ratio_est_model < rep.min_inlier_ratio_est_model or (n > 0 and n < rep.min_num_inliers_est_model):
        isp = TwoViewEstimationReport(v_corr_idxs=post_rows, num_inliers_est_model=0)
    else:
        isp = replace(post)
    return replace(res, pre_ba_report=pre, post_ba_report=post, post_isp_report=isp, putative_corr_idxs=putative)
