"""fp64 NumPy restatement of the reference's global bundle adjustment (gtsfm/bundle/bundle_adjustment.py:148-410 with
common/gtsfm_data.py:511-528 and 839-881), built on twoview_ba_ref's pieces (Pose3 retraction and logmap, the LM
constants).

The graph, with shared_calib False and cameras_to_model = every valid camera in sorted order:
  * one GeneralSFMFactor2<Cal3Bundler>(uv, Isotropic.Sigma(2, sigma) [Robust(Huber(k))], X(i), P(j), K(i)) per
    measurement; a point at depth <= 0 contributes a zero residual and zero Jacobians (the factor's cheirality branch);
  * the gauge: KarcherMeanFactorPose3(all X, 6, beta) - error 0, linearised as a constant JacobianFactor with sqrt(beta) I6
    on every pose key and b = 0 - or a PriorFactorPose3 on the first camera's input pose (error -Logmap(x^-1 prior), the
    Jacobian gtsam's PriorFactor writes, I);
  * one PriorFactor<Cal3Bundler> per camera on its input (f, k1, k2): error x - prior, Jacobian I, diagonal sigmas.
LM is gtsam.LevenbergMarquardtParams()'s: lambda 1e-5 scaled by 10, lambdaUpperBound 1e5, relative and absolute error
tolerance 1e-5, minModelFidelity 1e-3, damping lambda I on every unknown, a damped system whose Cholesky fails is a
rejected trial.  The damped normal equations are solved as the device does: every point's 3 x 3 block is eliminated
first and the dense reduced camera system (9 unknowns per camera) is factored by Cholesky.

Cameras are rows (C, 17): R (9, row-major wRc), t (3), f, k1, k2, u0, v0.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from oracle import twoview_ba_ref as tv

KARCHER, FIRST_POSE_PRIOR = 0, 1
KARCHER_BETA = 1000.0  # KarcherMeanFactorPose3(keys, 6, 1000) (bundle_adjustment.py:231)


@dataclass
class Params:
    noise_sigma: float = 2.0            # measurement_noise_sigma
    huber_k: float = 1.345              # robust_noise_basin; 0: robust_ba_mode NONE
    gauge: int = KARCHER
    max_iters: int = tv.LM_MAX_ITERS
    karcher_beta: float = KARCHER_BETA
    pose_prior_sigma: float = 0.1       # cam_pose3_prior_noise_sigma
    cal_prior_sigma: tuple = (20.0, 0.1, 0.1)  # calibration_prior_focal_sigma, _dist_sigma, _dist_sigma
    rel_tol: float = tv.LM_REL_TOL      # test hooks (run to convergence); gtsam's defaults otherwise
    abs_tol: float = tv.LM_ABS_TOL


@dataclass
class Problem:
    cam0: np.ndarray     # (C, 17) input cameras (the calibration priors and the first-pose prior)
    toff: np.ndarray     # (N + 1,)
    mcam: np.ndarray     # (M,)
    uv: np.ndarray       # (M, 2)
    prm: Params
    mtrk: np.ndarray = field(init=False)

    def __post_init__(self):
        self.toff = np.asarray(self.toff, np.int64)
        self.mcam = np.asarray(self.mcam, np.int64)
        self.uv = np.asarray(self.uv, float).reshape(-1, 2)
        self.mtrk = np.repeat(np.arange(len(self.toff) - 1), np.diff(self.toff))


def project_meas(cams: np.ndarray, pts: np.ndarray, pr: Problem):
    """Every measurement's projection -> uv (M, 2), depth (M,), J over its camera's 9 unknowns (M, 2, 9), J over its point
    (M, 2, 3): tv.project_many's formulas with per-measurement cameras."""
    R = cams[pr.mcam, :9].reshape(-1, 3, 3)
    t = cams[pr.mcam, 9:12]
    f, k1, k2, u0, v0 = (cams[pr.mcam, 12 + i] for i in range(5))
    pc = np.einsum("mji,mj->mi", R, pts[pr.mtrk] - t)  # R^T (p - t)
    z = pc[:, 2]
    x, y = pc[:, 0] / z, pc[:, 1] / z
    r = x * x + y * y
    g = 1.0 + k1 * r + k2 * r * r
    uv = np.stack([u0 + f * g * x, v0 + f * g * y], 1)
    dg = 2.0 * (k1 + 2.0 * k2 * r)
    A00, A01, A11 = f * (g + dg * x * x), f * dg * x * y, f * (g + dg * y * y)
    iz = 1.0 / z
    D = np.stack([np.stack([A00 * iz, A01 * iz, -(A00 * x + A01 * y) * iz], -1),
                  np.stack([A01 * iz, A11 * iz, -(A01 * x + A11 * y) * iz], -1)], 1)  # (M, 2, 3)
    Jw = np.stack([D[:, :, 1] * pc[:, None, 2] - D[:, :, 2] * pc[:, None, 1], D[:, :, 2] * pc[:, None, 0] - D[:, :, 0] * pc[:, None, 2],
                   D[:, :, 0] * pc[:, None, 1] - D[:, :, 1] * pc[:, None, 0]], -1)
    q = np.stack([x, y], 1)
    Jcal = np.stack([g[:, None] * q, (f * r)[:, None] * q, (f * r * r)[:, None] * q], -1)
    Jc = np.concatenate([Jw, -D, Jcal], 2)
    Jp = np.einsum("mkj,mij->mki", D, R)  # D R^T
    return uv, z, Jc, Jp


def _robust_loss(e, k):
    return 0.5 * e * e if k <= 0 else np.where(e <= k, 0.5 * e * e, k * (e - 0.5 * k))


def _robust_weight(e, k):
    return np.ones_like(e) if k <= 0 else np.where(e <= k, 1.0, k / np.maximum(e, k))


def _pose_prior_err(cam, cam0, inv):
    """-Logmap(x^-1 prior) / sigma."""
    R, t = cam[:9].reshape(3, 3), cam[9:12]
    R0, t0 = cam0[:9].reshape(3, 3), cam0[9:12]
    return -tv.se3_log(R.T @ R0, R.T @ (t0 - t)) * inv


def _cal_inv(pr):
    return 1.0 / np.asarray(pr.prm.cal_prior_sigma, float)


def prior_cost(cams, pr: Problem) -> float:
    e = (cams[:, 12:15] - pr.cam0[:, 12:15]) * _cal_inv(pr)
    c = 0.5 * float(np.sum(e * e))
    if pr.prm.gauge == FIRST_POSE_PRIOR:
        ep = _pose_prior_err(cams[0], pr.cam0[0], 1.0 / pr.prm.pose_prior_sigma)
        c += 0.5 * float(ep @ ep)
    return c


def reproj_errors(cams, pts, pr: Problem) -> np.ndarray:
    """|project - uv| per measurement, NaN where the point is not in front of the camera (projectSafe)."""
    uv, z, _, _ = project_meas(cams, pts, pr)
    e = np.linalg.norm(uv - pr.uv, axis=1)
    return np.where(z > 0.0, e, np.nan)


def cost(cams, pts, pr: Problem) -> float:
    """graph.error: the robust reprojection losses, the priors; the Karcher factor's error is 0."""
    uv, z, _, _ = project_meas(cams, pts, pr)
    e = np.linalg.norm(uv - pr.uv, axis=1) / pr.prm.noise_sigma
    return float(np.sum(np.where(z > 0.0, _robust_loss(e, pr.prm.huber_k), 0.0))) + prior_cost(cams, pr)


def linearise(cams, pts, pr: Problem):
    """The whitened, reweighted rows of every reprojection factor: sqrt(w) Jc / sigma, sqrt(w) Jp / sigma, sqrt(w) r / sigma."""
    uv, z, Jc, Jp = project_meas(cams, pts, pr)
    s = pr.prm.noise_sigma
    front = z > 0.0
    r = np.where(front[:, None], (uv - pr.uv) / s, 0.0)
    w = _robust_weight(np.linalg.norm(r, axis=1), pr.prm.huber_k)
    sw = np.sqrt(w)
    Jc = np.where(front[:, None, None], Jc, 0.0) * (sw / s)[:, None, None]
    Jp = np.where(front[:, None, None], Jp, 0.0) * (sw / s)[:, None, None]
    return Jc, Jp, r * sw[:, None]


def reduced_system(cams, pts, pr: Problem, lam: float, lin=None, karcher=True):
    """-> (S (9C, 9C) damped reduced camera system, b (9C,) its gradient, per track L (N, 3, 3) and z (N, 3), W (M, 3, 9),
    the linearisation) or None when a point block is not positive definite.  `karcher` False leaves the Karcher term out
    (a test hook)."""
    C, N = len(cams), len(pr.toff) - 1
    Jc, Jp, r = lin if lin is not None else linearise(cams, pts, pr)
    Hpp = np.zeros((N, 3, 3))
    gp = np.zeros((N, 3))
    np.add.at(Hpp, pr.mtrk, np.einsum("mki,mkj->mij", Jp, Jp))
    np.add.at(gp, pr.mtrk, np.einsum("mki,mk->mi", Jp, r))
    Hpp += lam * np.eye(3)
    if not (np.all(np.isfinite(Hpp)) and np.all(np.isfinite(gp))):
        return None
    try:
        L = np.linalg.cholesky(Hpp)
    except np.linalg.LinAlgError:
        return None
    Hpc = np.einsum("mki,mkj->mij", Jp, Jc)  # (M, 3, 9)
    W = np.linalg.solve(L[pr.mtrk], Hpc)
    z = np.linalg.solve(L, gp[:, :, None])[:, :, 0]
    S = np.zeros((9 * C, 9 * C))
    b = np.zeros(9 * C)
    S4 = S.reshape(C, 9, C, 9)
    np.add.at(S4, (pr.mcam, slice(None), pr.mcam), np.einsum("mki,mkj->mij", Jc, Jc))
    np.add.at(b.reshape(C, 9), pr.mcam, np.einsum("mki,mk->mi", Jc, r) - np.einsum("mki,mk->mi", W, z[pr.mtrk]))
    for j in range(N):  # - W_a^T W_b over every pair of the track's measurements
        ms = np.arange(pr.toff[j], pr.toff[j + 1])
        Wj = W[ms].transpose(1, 0, 2).reshape(3, -1)  # (3, 9 k)
        blk = (Wj.T @ Wj).reshape(len(ms), 9, len(ms), 9)
        cj = pr.mcam[ms]
        S4[cj[:, None], :, cj[None, :], :] -= blk.transpose(0, 2, 1, 3)
    if karcher and pr.prm.gauge == KARCHER:
        P = np.zeros((C, 9, C, 9))
        P[:, :6, :, :6] = np.eye(6)[None, :, None, :]
        S += pr.prm.karcher_beta * P.reshape(9 * C, 9 * C)
    ci = _cal_inv(pr)
    for a in range(C):
        S[9 * a + 6:9 * a + 9, 9 * a + 6:9 * a + 9] += np.diag(ci * ci)
        b[9 * a + 6:9 * a + 9] += (cams[a, 12:15] - pr.cam0[a, 12:15]) * ci * ci
    if pr.prm.gauge == FIRST_POSE_PRIOR:
        inv = 1.0 / pr.prm.pose_prior_sigma
        S[:6, :6] += np.eye(6) * inv * inv
        b[:6] += _pose_prior_err(cams[0], pr.cam0[0], inv) * inv
    S += lam * np.eye(9 * C)
    return S, b, L, z, W, (Jc, Jp, r)


def retract(cams, dc):
    out = cams.copy()
    for a in range(len(cams)):
        d = dc[9 * a:9 * a + 9]
        R, t = tv.retract_pose(cams[a, :9].reshape(3, 3), cams[a, 9:12], d[:6])
        out[a, :9], out[a, 9:12] = R.ravel(), t
        out[a, 12:15] += d[6:]
    return out


def step(cams, pts, pr: Problem, lam: float, lin=None):
    """One damped solve -> (candidate cams, candidate points, linearised decrease, old linearised cost, dc) or None when the
    damped system is not positive definite (a rejected trial)."""
    sys_ = reduced_system(cams, pts, pr, lam, lin)
    if sys_ is None:
        return None
    S, b, L, z, W, (Jc, Jp, r) = sys_
    if not (np.all(np.isfinite(S)) and np.all(np.isfinite(b))):
        return None
    try:
        Ls = np.linalg.cholesky(S)
    except np.linalg.LinAlgError:
        return None
    dc = -np.linalg.solve(Ls.T, np.linalg.solve(Ls, b))
    C = len(cams)
    dcm = dc.reshape(C, 9)
    y = z.copy()
    np.add.at(y, pr.mtrk, np.einsum("mij,mj->mi", W, dcm[pr.mcam]))
    dp = -np.linalg.solve(np.transpose(L, (0, 2, 1)), y[:, :, None])[:, :, 0]
    Jd = np.einsum("mkj,mj->mk", Jc, dcm[pr.mcam]) + np.einsum("mkj,mj->mk", Jp, dp[pr.mtrk])
    lin_dec = -float(np.sum(r * Jd) + 0.5 * np.sum(Jd * Jd))
    old = 0.5 * float(np.sum(r * r))
    ci = _cal_inv(pr)
    e = (cams[:, 12:15] - pr.cam0[:, 12:15]) * ci
    jd = dcm[:, 6:] * ci
    lin_dec -= float(np.sum(e * jd) + 0.5 * np.sum(jd * jd))
    old += 0.5 * float(np.sum(e * e))
    if pr.prm.gauge == FIRST_POSE_PRIOR:
        inv = 1.0 / pr.prm.pose_prior_sigma
        ep = _pose_prior_err(cams[0], pr.cam0[0], inv)
        jd = dcm[0, :6] * inv
        lin_dec -= float(ep @ jd + 0.5 * jd @ jd)
        old += 0.5 * float(ep @ ep)
    else:  # the Karcher factor: linearised error 0 at dx = 0, 0.5 beta |sum_i d_i|^2 at the step
        s = dcm[:, :6].sum(0)
        lin_dec -= 0.5 * pr.prm.karcher_beta * float(s @ s)
    return retract(cams, dc), pts + dp, lin_dec, old, dc


@dataclass
class Result:
    cams: np.ndarray
    pts: np.ndarray
    reproj_err: np.ndarray
    final_error: float
    iterations: int
    trace: List[float]
    trials: List[int]        # 1 accepted, 0 rejected, 2 rejected and the lambda search stopped, -1 not positive definite
    steps: List[np.ndarray]  # dc of every accepted trial (test hook)


def adjust(cams, pts, toff, mcam, uv, prm: Optional[Params] = None) -> Result:
    """gtsam's LevenbergMarquardtOptimizer::optimize on the graph above (twoview_ba_ref._lm's schedule, with the trials
    recorded)."""
    prm = prm or Params()
    cams = np.array(cams, float).reshape(-1, 17)
    pts = np.array(pts, float).reshape(-1, 3)
    pr = Problem(cams.copy(), toff, mcam, uv, prm)
    err = cost(cams, pts, pr)
    trace, trials, steps = [err], [], []
    lam, its, new = tv.LM_LAMBDA0, 0, err
    if err > 0.0:
        while True:
            cur = new
            lin = linearise(cams, pts, pr)
            while True:
                st = step(cams, pts, pr, lam, lin)
                success = stop = False
                if st is not None:
                    cn, pn, lin_dec, old, dc = st
                    if lin_dec >= 0.0:
                        e_new = cost(cn, pn, pr)
                        dcost = cur - e_new
                        success = dcost / lin_dec > tv.LM_MIN_FIDELITY if lin_dec > np.finfo(float).eps * old else True
                        stop = abs(dcost) < prm.rel_tol * cur
                trials.append(-1 if st is None else 1 if success else 2 if stop else 0)
                if success:
                    cams, pts, lam, its, new = cn, pn, lam / tv.LM_FACTOR, its + 1, e_new
                    steps.append(dc)
                    break
                if stop:
                    break
                lam *= tv.LM_FACTOR
                if lam >= tv.LM_LAMBDA_MAX:
                    break
            trace.append(new)
            dec = cur - new
            converged = dec / cur <= prm.rel_tol or dec <= prm.abs_tol or new <= 0.0
            if not (its < prm.max_iters and not converged and np.isfinite(cur)):
                break
    return Result(cams, pts, reproj_errors(cams, pts, pr), new, its, trace, trials, steps)


def valid_mask(reproj_err: np.ndarray, toff: np.ndarray, thresh: float) -> np.ndarray:
    """GtsfmData.__validate_track per track: every error < thresh and none NaN."""
    ok = np.where(np.isnan(reproj_err), False, reproj_err < thresh)
    return np.logical_and.reduceat(ok, np.asarray(toff[:-1], np.int64)) if len(toff) > 1 else np.zeros(0, bool)
