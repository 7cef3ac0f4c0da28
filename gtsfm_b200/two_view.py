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
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Iterable, Mapping, Optional, Sequence, Tuple

import numpy as np
import torch

from .gtsfm_api import Rot3, Unit3
from .pipeline import DeviceFeatures, DeviceFrontEnd, RefineOptions
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


def _failure(num_putative: int) -> TwoViewResult:  # verifier_base.py:60-64
    return TwoViewResult(None, None, np.zeros((0, 2), np.int64), 0.0, num_putative)


def _refined_failure(ratio: float, num_putative: int) -> TwoViewResult:  # inlier_support_processor.py failure_result
    return TwoViewResult(None, None, np.array([], np.uint64), ratio, num_putative)


class B200TwoViewBatch:
    """match (optional) -> calibrate -> RANSAC-5pt (or LMedS-5pt) -> recoverPose for a list of pairs, device-resident.

    `intrinsics[i]` = (f, u0, v0) of image i (Cal3Bundler without distortion: what GTSfM's deep front-end configs use).
    `method`: "ransac" (the reference's Ransac verifier) or "lmeds" (its LMEDS verifier; the threshold and seed are unused).
    `bundle_adjust_2view`: also triangulate, bundle-adjust and apply inlier support on the device, with the reference's
    TwoViewEstimator / InlierSupportProcessor arguments below (sift_front_end sets the triangulation threshold to 100).
    """

    def __init__(self, front_end: DeviceFrontEnd, estimation_threshold_px: float = 4.0, seed: int = DEFAULT_SEED,
                 method: str = "ransac", bundle_adjust_2view: bool = False, ba_reproj_error_threshold: float = 0.5,
                 min_num_inliers_est_model: int = 15, min_inlier_ratio_est_model: float = 0.1,
                 triangulation_reproj_error_threshold: float = float("inf")):
        if method not in ("ransac", "lmeds"):
            raise ValueError(f"verification method must be 'ransac' or 'lmeds', not {method!r}")
        self.fe = front_end
        self.threshold_px = float(estimation_threshold_px)
        self.seed = int(seed)
        self.method = method
        self.refine = RefineOptions(ba_reproj_error_threshold, min_num_inliers_est_model, min_inlier_ratio_est_model,
                                    triangulation_reproj_error_threshold) if bundle_adjust_2view else None

    def run(self, features: Mapping[int, DeviceFeatures], pairs: Iterable[Tuple[int, int]], intrinsics: Mapping[int, Sequence[float]],
            putative: Optional[Mapping[Tuple[int, int], torch.Tensor]] = None) -> Dict[Tuple[int, int], TwoViewResult]:
        """`putative[(i1, i2)]`: (k, 2) int64 device tensor of match indices; matched here with LightGlue when absent."""
        out: Dict[Tuple[int, int], TwoViewResult] = {}
        pending = []  # (pairs, matches, future) of a chunk in flight on the verification stream
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
                    out[(i1, i2)] = _failure(k)
                    continue
                prs.append((i1, i2))
                items.append((features[i1], features[i2], m, intrinsics[i1], intrinsics[i2]))
            if items:  # this chunk's verification: one call on its own stream / thread under the next chunk's matching
                pending.append(submit_chunk(self.fe, prs, items, self.threshold_px, self.seed, self.method, self.refine))
            while len(pending) > 1:
                self._collect_chunk(pending.pop(0), out)
        for p in pending:
            self._collect_chunk(p, out)
        return out

    @classmethod
    def _collect_chunk(cls, chunk, out) -> None:
        prs, ms, fut, rfut = chunk
        if rfut is None:
            for pair, m, r in zip(prs, ms, fut.result()):
                cls._collect_one(pair, m, r, out)
            return
        for pair, m, v, r in zip(prs, ms, fut.result(), rfut.result()):
            cls._collect_refined(pair, m, v, r, out)

    @staticmethod
    def _collect_refined(pair, m, verified, refined, out) -> None:
        k = int(m.shape[0])
        if verified[0] is None:
            out[pair] = _failure(k)
            return
        ratio = float(verified[3]) / float(k)  # the ratio from before BA (two_view_estimator.py:426)
        R, t, rows, _ = refined
        if R is None:
            out[pair] = _refined_failure(ratio, k)
            return
        out[pair] = TwoViewResult(Rot3(R), Unit3(t), rows.cpu().numpy().astype(np.int64), ratio, k)  # only the final rows cross PCIe

    @staticmethod
    def _collect_one(pair, m, result, out) -> None:
        E, R, t, n_inl, mask = result
        k = int(m.shape[0])
        if E is None:
            out[pair] = _failure(k)
            return
        keep = mask.bool()
        rows = m[keep].cpu().numpy().astype(np.int64)  # only the verified rows cross PCIe
        out[pair] = TwoViewResult(Rot3(R), Unit3(t), rows, float(n_inl) / float(k), k)


def submit_chunk(fe: DeviceFrontEnd, prs, items, threshold_px: float, seed: int, method: str, refine: Optional[RefineOptions]):
    """Queue one chunk's verification (and, with `refine`, its refinement right behind it) on the verification lane.
    -> the chunk entry `_collect_chunk` takes."""
    vfut = fe.verify_many_async(items, threshold_px, seed, method)
    return prs, [it[2] for it in items], vfut, fe.refine_many_async(items, vfut, refine) if refine is not None else None
