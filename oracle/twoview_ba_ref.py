"""fp64 NumPy restatement of the reference's per-pair refinement after verification (gtsfm/two_view_estimator.py:350-481).

For a verified pair with at least `min_num_inliers` verified rows (:412): triangulate every verified correspondence in
the cameras Pose3() / Pose3(R, U)^-1 (:241-252) with gtsam.triangulatePoint3(rank_tol=1e-9, optimize=True)
(data_association/point3d_initializer.py:221-295, NO_RANSAC), run the two-view bundle adjustment the reference builds
(bundle/bundle_adjustment.py:148-345 with the constructor arguments of two_view_estimator.py:86-99), reject the pair when
the Hessian at the optimum is indeterminate (:566-579), keep the tracks whose reprojection errors are all below 0.5 px
(common/gtsfm_data.py:839-881), and apply the inlier-support thresholds (frontend/inlier_support_processor.py).

gtsam is not a dependency of this project, so the constants below are gtsam 4.2's documented defaults, restated from
its sources (nonlinear/LevenbergMarquardtParams.h, geometry/triangulation.h, linear/LossFunctions.cpp).  They are NOT
pinned against a live gtsam run; DESIGN.md §11 lists what that leaves open.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

# gtsam.LevenbergMarquardtParams() defaults; maxIterations is set to 100 by the reference (two_view_estimator.py:60)
LM_LAMBDA0 = 1e-5
LM_FACTOR = 10.0           # useFixedLambdaFactor = true: lambda *= 10 on a rejected step, /= 10 on an accepted one
LM_LAMBDA_MAX = 1e5        # lambdaUpperBound; lambdaLowerBound = 0
LM_REL_TOL = 1e-5          # relativeErrorTol
LM_ABS_TOL = 1e-5          # absoluteErrorTol
LM_MIN_FIDELITY = 1e-3     # minModelFidelity
LM_MAX_ITERS = 100
# gtsam/geometry/triangulation.h optimize(): the point refinement of triangulatePoint3(..., optimize=True)
TRI_LAMBDA0 = 1.0
TRI_ABS_TOL = 1.0
DLT_RANK_TOL = 1e-9        # point3d_initializer.py SVD_DLT_RANK_TOL
# the factor graph (two_view_estimator.py:86-99, bundle_adjustment.py:148-345, common/types.py:113-132)
HUBER_K = 1.345
POSE_PRIOR_SIGMA = 0.1
POINT_PRIOR_SIGMA = 0.1
CAL_PRIOR_SIGMA = 1e-5     # f, k1, k2 of Cal3Bundler
# the indeterminate-system test that stands in for gtsam.Marginals throwing: a Cholesky pivot of the undamped Hessian at
# the optimum (points eliminated first) at or below this fraction of the unknown's own diagonal entry
INDETERMINATE_PIVOT = 1e-10


def skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def so3_exp(w):
    """Rot3::Expmap (Rodrigues; first order below theta^2 = eps, as gtsam's SO3 ExpmapFunctor)."""
    th2 = float(w @ w)
    W = skew(w)
    if th2 <= np.finfo(float).eps:
        return np.eye(3) + W
    th = np.sqrt(th2)
    return np.eye(3) + (np.sin(th) / th) * W + ((1.0 - np.cos(th)) / th2) * (W @ W)


def so3_log(R):
    """SO3::Logmap away from theta = pi (gtsam's normal and near-zero branches)."""
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    tr3 = tr - 3.0
    if tr3 < -1e-6:
        th = np.arccos(np.clip((tr - 1.0) / 2.0, -1.0, 1.0))
        mag = th / (2.0 * np.sin(th))
    else:
        mag = 0.5 - tr3 / 12.0 + tr3 * tr3 / 60.0
    return mag * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])


def se3_v(w, v):
    """The translation of Pose3::Expmap([w, v]): V(w) v, with V's series below theta = 1e-4 (gtsam writes the same
    quantity as (w x v - R (w x v) + w (w . v)) / theta^2)."""
    th2 = float(w @ w)
    wv = np.cross(w, v)
    wwv = np.cross(w, wv)
    if th2 < 1e-8:
        a, b = 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0
    else:
        th = np.sqrt(th2)
        a, b = (1.0 - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)
    return v + a * wv + b * wwv


def se3_log(R, t):
    """Pose3::Logmap -> [w, u] (Agrawal06iros eq. 14, as gtsam writes it)."""
    w = so3_log(R)
    th = np.linalg.norm(w)
    if th < 1e-10:
        return np.concatenate([w, t])
    W = skew(w / th)
    WT = W @ t
    u = t - (0.5 * th) * WT + (1.0 - th / (2.0 * np.tan(0.5 * th))) * (W @ WT)
    return np.concatenate([w, u])


def retract_pose(R, t, d):
    """Pose3::retract = compose(Expmap(d)): R Exp(w), t + R V(w) v."""
    return R @ so3_exp(d[:3]), t + R @ se3_v(d[:3], d[3:])


def project(R, t, cal, p):
    """PinholeCamera<Cal3Bundler>(Pose3(R, t), cal = (f, k1, k2, u0, v0)).project(p) with its Jacobians in gtsam's
    conventions (pose: right perturbation [w, v]).  -> uv, depth, J_pose (2, 6), J_point (2, 3), J_cal (2, 3)."""
    pc = R.T @ (p - t)
    z = pc[2]
    x, y = pc[0] / z, pc[1] / z
    f, k1, k2, u0, v0 = cal
    r = x * x + y * y
    g = 1.0 + k1 * r + k2 * r * r
    uv = np.array([u0 + f * g * x, v0 + f * g * y])
    dg = 2.0 * (k1 + 2.0 * k2 * r)
    Duv_pn = f * np.array([[g + dg * x * x, dg * x * y], [dg * x * y, g + dg * y * y]])
    Dpn_pc = np.array([[1.0 / z, 0.0, -x / z], [0.0, 1.0 / z, -y / z]])
    Duv_pc = Duv_pn @ Dpn_pc
    J_pose = np.hstack([Duv_pc @ skew(pc), -Duv_pc])
    J_point = Duv_pc @ R.T
    J_cal = np.array([[g * x, f * r * x, f * r * r * x], [g * y, f * r * y, f * r * r * y]])
    return uv, z, J_pose, J_point, J_cal


def huber_weight(e):
    return 1.0 if e <= HUBER_K else HUBER_K / e


def huber_loss(e):
    return 0.5 * e * e if e <= HUBER_K else HUBER_K * (e - 0.5 * HUBER_K)


def projection_matrix(R, t, cal):
    """camera.cameraProjectionMatrix(): K [R^T | -R^T t] for the camera Pose3(R, t)."""
    K = np.array([[cal[0], 0.0, cal[3]], [0.0, cal[0], cal[4]], [0.0, 0.0, 1.0]])
    return K @ np.hstack([R.T, (-R.T @ t)[:, None]])


def dlt(P0, P1, uv0, uv1):
    """triangulateDLT: the right singular vector of the smallest singular value of the 4 x 4 DLT matrix.
    -> (point | None when the rank (singular values above 1e-9) is below 3 or the point is at infinity)."""
    A = np.stack([uv0[0] * P0[2] - P0[0], uv0[1] * P0[2] - P0[1], uv1[0] * P1[2] - P1[0], uv1[1] * P1[2] - P1[1]])
    _, s, Vt = np.linalg.svd(A)
    if int(np.sum(s > DLT_RANK_TOL)) < 3:
        return None
    v = Vt[3]
    X = v[:3] / v[3]
    return X if np.all(np.isfinite(X)) else None


def _lm(cost, step, x, lambda0, abs_tol, max_iters=LM_MAX_ITERS, trace: Optional[list] = None):
    """gtsam's LevenbergMarquardtOptimizer::optimize on a problem given by `cost(x)` and `step(x, lam)` -> (x + dx, the
    linearized cost decrease, the undamped linearized cost at dx = 0), or None when the damped system is not positive
    definite.  -> (x, successful iterations, final lambda).  `trace` gets the cost before the first and after every
    outer iteration."""
    err = cost(x)
    if trace is not None:
        trace.append(err)
    lam, its = lambda0, 0
    if err <= 0.0:
        return x, its, lam
    new = err
    while True:
        cur = new
        while True:  # tryLambda until it returns true
            st = step(x, lam)
            success, stop = False, False
            if st is not None:
                x_new, lin, old_lin = st
                if lin >= 0.0:
                    e_new = cost(x_new)
                    dc = cur - e_new
                    if lin > np.finfo(float).eps * old_lin:
                        success = dc / lin > LM_MIN_FIDELITY
                    else:
                        success = True
                    if abs(dc) < LM_REL_TOL * cur:
                        stop = True
            if success:
                x, lam, its = x_new, lam / LM_FACTOR, its + 1
                break
            if stop:
                break
            lam *= LM_FACTOR
            if lam >= LM_LAMBDA_MAX:
                break
        new = cost(x)
        if trace is not None:
            trace.append(new)
        dec = cur - new
        converged = (dec / cur <= LM_REL_TOL) or (dec <= abs_tol) or (new <= 0.0)
        if not (its < max_iters and not converged and np.isfinite(cur)):
            return x, its, lam


def refine_point(cams, uvs, X):
    """triangulateNonlinear: LM (lambda0 1, absolute tolerance 1) on sum 0.5 |project - uv|^2 over the two cameras; a
    point behind a camera gives that camera the residual (2f, 2f) and a zero Jacobian (TriangulationFactor)."""

    def resid(p):
        out = []
        for (R, t, cal), uv in zip(cams, uvs):
            pr, z, _, Jp, _ = project(R, t, cal, p)
            if z <= 0.0:
                out.append((np.full(2, 2.0 * cal[0]), np.zeros((2, 3))))
            else:
                out.append((pr - uv, Jp))
        return out

    def cost(p):
        return sum(0.5 * float(r @ r) for r, _ in resid(p))

    def step(p, lam):
        rs = resid(p)
        H = sum(J.T @ J for _, J in rs) + lam * np.eye(3)
        g = sum(J.T @ r for r, J in rs)
        if not (np.all(np.isfinite(H)) and np.all(np.isfinite(g))):
            return None
        try:
            L = np.linalg.cholesky(H)
        except np.linalg.LinAlgError:
            return None
        d = -np.linalg.solve(L.T, np.linalg.solve(L, g))
        lin = -sum(float(r @ (J @ d)) + 0.5 * float((J @ d) @ (J @ d)) for r, J in rs)
        return p + d, lin, sum(0.5 * float(r @ r) for r, _ in rs)

    return _lm(cost, step, X, TRI_LAMBDA0, TRI_ABS_TOL)[0]


def triangulate(cams, uv0, uv1, reproj_thr=np.inf, min_angle_deg=0.0):
    """Point3dInitializer.triangulate (NO_RANSAC) for one correspondence -> point or None (dropped)."""
    P = [projection_matrix(*c) for c in cams]
    X = dlt(P[0], P[1], uv0, uv1)
    if X is None:
        return None
    X = refine_point(cams, (uv0, uv1), X)
    errs = []
    for (R, t, cal), uv in zip(cams, (uv0, uv1)):
        pr, z, *_ = project(R, t, cal, X)
        if not z > 0.0:  # GTSAM_THROW_CHEIRALITY_EXCEPTION: the point must be in front of every camera
            return None
        errs.append(np.linalg.norm(pr - uv))
    if not all(e < reproj_thr for e in errs):
        return None
    r0, r1 = X - cams[0][1], X - cams[1][1]
    c = float(r0 @ r1) / (np.linalg.norm(r0) * np.linalg.norm(r1))
    if np.degrees(np.arccos(np.clip(c, -1.0, 1.0))) < min_angle_deg:
        return None
    return X


def project_many(R, t, cal, P):
    """`project` for (n, 3) points at once -> uv (n, 2), depth (n,), J over the camera's 9 unknowns [pose, f, k1, k2]
    (n, 2, 9), J over the point (n, 2, 3)."""
    pc = (P - t) @ R
    z = pc[:, 2]
    x, y = pc[:, 0] / z, pc[:, 1] / z
    f, k1, k2, u0, v0 = cal
    r = x * x + y * y
    g = 1.0 + k1 * r + k2 * r * r
    uv = np.stack([u0 + f * g * x, v0 + f * g * y], 1)
    dg = 2.0 * (k1 + 2.0 * k2 * r)
    A = f * np.stack([np.stack([g + dg * x * x, dg * x * y], -1), np.stack([dg * x * y, g + dg * y * y], -1)], 1)  # (n, 2, 2)
    iz = 1.0 / z
    Dpn = np.zeros((len(P), 2, 3))
    Dpn[:, 0, 0] = iz
    Dpn[:, 1, 1] = iz
    Dpn[:, 0, 2] = -x * iz
    Dpn[:, 1, 2] = -y * iz
    D = A @ Dpn  # (n, 2, 3)
    S = np.zeros((len(P), 3, 3))
    S[:, 0, 1], S[:, 0, 2], S[:, 1, 2] = -pc[:, 2], pc[:, 1], -pc[:, 0]
    S[:, 1, 0], S[:, 2, 0], S[:, 2, 1] = pc[:, 2], -pc[:, 1], pc[:, 0]
    Jc = np.concatenate([D @ S, -D, np.stack([np.stack([g * x, f * r * x, f * r * r * x], -1),
                                              np.stack([g * y, f * r * y, f * r * r * y], -1)], 1)], 2)
    Jp = D @ R.T
    return uv, z, Jc, Jp


def _huber_w(e):
    return np.where(e <= HUBER_K, 1.0, HUBER_K / np.maximum(e, HUBER_K))


def _huber_loss(e):
    return np.where(e <= HUBER_K, 0.5 * e * e, HUBER_K * (e - 0.5 * HUBER_K))


def _terms(s: "BAState", pr: "BAProblem"):
    """Per camera c: whitened residuals r (n, 2), J over the camera's unknowns (n, 2, 9), J over the point (n, 2, 3) and
    Huber weights (n,); a point behind the camera contributes zero (GeneralSFMFactor2's cheirality branch)."""
    out = []
    for c in range(2):
        uv, z, Jc, Jp = project_many(s.R[c], s.t[c], s.cal[c], s.pts)
        front = z > 0.0
        r = np.where(front[:, None], uv - pr.uv[:, c], 0.0)
        Jc = np.where(front[:, None, None], Jc, 0.0)
        Jp = np.where(front[:, None, None], Jp, 0.0)
        out.append((r, Jc, Jp, _huber_w(np.linalg.norm(r, axis=1))))
    return out


def _prior_terms(s: "BAState", pr: "BAProblem"):
    """(whitened error, Jacobian over the 18 camera unknowns) of the pose prior and the calibration priors; the point prior
    is handled with its point."""
    terms = []
    e = se3_log(s.R[0], s.t[0]) / POSE_PRIOR_SIGMA  # PriorFactor: -Local(x, identity) = Logmap(x), Jacobian I
    J = np.zeros((6, 18))
    J[:, :6] = np.eye(6) / POSE_PRIOR_SIGMA
    terms.append((e, J))
    for c in range(2):
        e = (s.cal[c][:3] - pr.cal0[c][:3]) / CAL_PRIOR_SIGMA
        J = np.zeros((3, 18))
        J[:, 9 * c + 6:9 * c + 9] = np.eye(3) / CAL_PRIOR_SIGMA
        terms.append((e, J))
    return terms


@dataclass
class BAState:
    R: List[np.ndarray]   # wRc of the two cameras
    t: List[np.ndarray]   # wtc
    cal: List[np.ndarray]  # (f, k1, k2, u0, v0)
    pts: np.ndarray       # (n, 3)


@dataclass
class BAProblem:
    uv: np.ndarray        # (n, 2, 2): measurement of track j in camera c
    pt0: np.ndarray       # the first track's initial point (PriorFactorPoint3)
    cal0: List[np.ndarray]  # the calibrations' initial values (the calibration priors)


def ba_cost(s: BAState, pr: BAProblem) -> float:
    c = 0.0
    for r, _, _, _ in _terms(s, pr):
        c += float(np.sum(_huber_loss(np.linalg.norm(r, axis=1))))
    for e, _ in _prior_terms(s, pr):
        c += 0.5 * float(e @ e)
    ep = (s.pts[0] - pr.pt0) / POINT_PRIOR_SIGMA
    return c + 0.5 * float(ep @ ep)


def _blocks(s: BAState, pr: BAProblem, lam: float, terms):
    """Hcc (18, 18) without priors, gc (18,), per-track Hpp (n, 3, 3) (+ lam I, + the first point's prior), gp (n, 3), Hcp
    (n, 18, 3)."""
    n = len(s.pts)
    Hcc, gc = np.zeros((18, 18)), np.zeros(18)
    Hpp = np.zeros((n, 3, 3)) + lam * np.eye(3)
    gp, Hcp = np.zeros((n, 3)), np.zeros((n, 18, 3))
    for c, (r, Jc, Jp, w) in enumerate(terms):
        sl = slice(9 * c, 9 * c + 9)
        Hcc[sl, sl] += np.einsum("n,nki,nkj->ij", w, Jc, Jc)
        gc[sl] += np.einsum("n,nki,nk->i", w, Jc, r)
        Hpp += np.einsum("n,nki,nkj->nij", w, Jp, Jp)
        gp += np.einsum("n,nki,nk->ni", w, Jp, r)
        Hcp[:, sl] += np.einsum("n,nki,nkj->nij", w, Jc, Jp)
    Hpp[0] += np.eye(3) / POINT_PRIOR_SIGMA ** 2
    gp[0] += (s.pts[0] - pr.pt0) / POINT_PRIOR_SIGMA ** 2
    return Hcc, gc, Hpp, gp, Hcp


def ba_step(s: BAState, pr: BAProblem, lam: float):
    """One damped solve with the points eliminated (Gauss-Newton with Huber reweighting, w J^T J and w J^T r per factor,
    damped by lam I) -> (candidate state, linearized cost decrease, undamped linearized cost at 0), or None when the
    system is not positive definite."""
    terms = _terms(s, pr)
    Hcc, gc, Hpp, gp, Hcp = _blocks(s, pr, lam, terms)
    if not all(np.all(np.isfinite(x)) for x in (Hcc, gc, Hpp, gp, Hcp)):
        return None  # the device's Cholesky fails on a non-finite pivot: the same outcome
    S, b = Hcc + lam * np.eye(18), gc.copy()
    old = 0.0
    for e, J in _prior_terms(s, pr):
        S += J.T @ J
        b += J.T @ e
        old += 0.5 * float(e @ e)
    try:
        L = np.linalg.cholesky(Hpp)
        W = np.linalg.solve(L, np.transpose(Hcp, (0, 2, 1)))  # L^-1 Hpc  (n, 3, 18)
        z = np.linalg.solve(L, gp[:, :, None])[:, :, 0]
        S -= np.einsum("nki,nkj->ij", W, W)
        b -= np.einsum("nki,nk->i", W, z)
        Ls = np.linalg.cholesky(S)
    except np.linalg.LinAlgError:
        return None
    if not np.all(np.isfinite(Ls)):
        return None
    dc = -np.linalg.solve(Ls.T, np.linalg.solve(Ls, b))
    # back-substitution through the point blocks' Cholesky factors, as the device does (Hpp of a point near infinity is
    # close to singular along its ray: a general solve may give up where the factors still exist)
    y = np.linalg.solve(L, (gp + np.einsum("nij,i->nj", Hcp, dc))[:, :, None])
    dp = -np.linalg.solve(np.transpose(L, (0, 2, 1)), y)[:, :, 0]
    if not np.all(np.isfinite(dp)):
        return None
    # linearized decrease: -sum_f w (r . J d + |J d|^2 / 2)
    lin = 0.0
    for e, J in _prior_terms(s, pr):
        Jd = J @ dc
        lin -= float(e @ Jd) + 0.5 * float(Jd @ Jd)
    for c, (r, Jc, Jp, w) in enumerate(terms):
        Jd = Jc @ dc[9 * c:9 * c + 9] + np.einsum("nkj,nj->nk", Jp, dp)
        lin -= float(np.sum(w * (np.sum(r * Jd, 1) + 0.5 * np.sum(Jd * Jd, 1))))
        old += 0.5 * float(np.sum(w * np.sum(r * r, 1)))
    ep = (s.pts[0] - pr.pt0) / POINT_PRIOR_SIGMA
    Jd = dp[0] / POINT_PRIOR_SIGMA
    lin -= float(ep @ Jd) + 0.5 * float(Jd @ Jd)
    old += 0.5 * float(ep @ ep)
    R, t, cal = [], [], []
    for c in range(2):
        d = dc[9 * c:9 * c + 9]
        Rc, tc = retract_pose(s.R[c], s.t[c], d[:6])
        R.append(Rc), t.append(tc)
        cal.append(np.concatenate([s.cal[c][:3] + d[6:], s.cal[c][3:]]))
    return BAState(R, t, cal, s.pts + dp), lin, old


def _pivots_ok(A, ref_diag) -> bool:
    """Cholesky of A: every pivot (before its square root) above INDETERMINATE_PIVOT * ref_diag and finite."""
    A = np.array(A, float)
    n = len(A)
    for k in range(n):
        piv = A[k, k] - A[k, :k] @ A[k, :k]
        if not (np.isfinite(piv) and piv > INDETERMINATE_PIVOT * ref_diag[k]):
            return False
        A[k, k] = np.sqrt(piv)
        for i in range(k + 1, n):
            A[i, k] = (A[i, k] - A[i, :k] @ A[k, :k]) / A[k, k]
    return True


def indeterminate(s: BAState, pr: BAProblem) -> bool:
    """Cholesky of the undamped Hessian at `s`, points first: a pivot at or below INDETERMINATE_PIVOT times the unknown's
    diagonal entry in the full Hessian (or not finite) stands for gtsam.Marginals' IndeterminantLinearSystemException."""
    Hcc, _, Hpp, _, Hcp = _blocks(s, pr, 0.0, _terms(s, pr))
    for e, J in _prior_terms(s, pr):
        Hcc += J.T @ J
    for j in range(len(s.pts)):
        if not _pivots_ok(Hpp[j], np.diag(Hpp[j])):
            return True
    S = Hcc - np.einsum("nik,nkl,njl->ij", Hcp, np.linalg.inv(Hpp), Hcp)
    return not _pivots_ok(S, np.diag(Hcc))


def bundle_adjust(s: BAState, pr: BAProblem, max_iters: int = LM_MAX_ITERS, trace: Optional[list] = None):
    """gtsam LM with the default schedule on the two-view graph.  -> (state, successful iterations)."""
    x, its, _ = _lm(lambda x: ba_cost(x, pr), lambda x, lam: ba_step(x, pr, lam), s, LM_LAMBDA0, LM_ABS_TOL, max_iters, trace)
    return x, its


@dataclass
class PairResult:
    ok: bool                     # False: (None, None, empty) - the pair fails
    R: Optional[np.ndarray]      # i2Ri1
    t: Optional[np.ndarray]      # unit i2ti1
    rows: np.ndarray             # indices into the pair's putative match rows that survive, ascending
    num_tracks: int = 0          # triangulated tracks
    iterations: int = 0
    trace: List[float] = field(default_factory=list)
    ran_ba: bool = False
    track_rows: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))  # rows that were bundle-adjusted
    track_err: np.ndarray = field(default_factory=lambda: np.zeros(0))  # their larger reprojection error at the optimum


def refine_pair(uv1, uv2, verified: np.ndarray, k_putative: int, cal1, cal2, R0, t0, ba_reproj_thr=0.5, min_inliers=15,
                min_ratio=0.1, tri_reproj_thr=np.inf, min_tri_angle=0.0, max_iters=LM_MAX_ITERS, verified_ok=True) -> PairResult:
    """The reference's run_2view after verification, for one pair.

    uv1 / uv2: (k, 2) pixel coordinates of the putative match rows; `verified`: ascending indices of the verified rows
    (empty when verification failed, `verified_ok` False); cal = (f, u0, v0); R0, t0: verification's i2Ri1 and unit i2ti1.
    """
    ratio = len(verified) / k_putative if (verified_ok and k_putative > 0) else 0.0
    res = PairResult(verified_ok, R0 if verified_ok else None, t0 if verified_ok else None, np.asarray(verified, np.int64))
    if verified_ok and len(verified) >= min_inliers:
        res = _bundle_adjust_pair(uv1, uv2, np.asarray(verified, np.int64), cal1, cal2, np.asarray(R0, float),
                                  np.asarray(t0, float), ba_reproj_thr, tri_reproj_thr, min_tri_angle, max_iters)
    # InlierSupportProcessor with num_inliers_est_model = len(v_corr_idxs) and the pre-BA ratio (:426)
    n = len(res.rows)
    if ratio < min_ratio or (0 < n < min_inliers):
        return PairResult(False, None, None, np.zeros(0, np.int64), res.num_tracks, res.iterations, res.trace, res.ran_ba,
                          res.track_rows, res.track_err)
    return res


def _bundle_adjust_pair(uv1, uv2, rows, cal1, cal2, R0, t0, ba_thr, tri_thr, min_angle, max_iters) -> PairResult:
    K = [np.array([cal1[0], 0.0, 0.0, cal1[1], cal1[2]]), np.array([cal2[0], 0.0, 0.0, cal2[1], cal2[2]])]
    cams = [(np.eye(3), np.zeros(3), K[0]), (R0.T, -R0.T @ t0, K[1])]  # Pose3(), Pose3(R, U)^-1
    keep, pts = [], []
    for i in rows:
        X = triangulate(cams, np.asarray(uv1[i], float), np.asarray(uv2[i], float), tri_thr, min_angle)
        if X is not None:
            keep.append(i)
            pts.append(X)
    if not keep:
        return PairResult(True, R0, t0, np.zeros(0, np.int64), 0, 0, [], False)
    keep = np.array(keep, np.int64)
    pts = np.array(pts)
    uv = np.stack([np.asarray(uv1, float)[keep], np.asarray(uv2, float)[keep]], 1)
    s0 = BAState([cams[0][0], cams[1][0]], [cams[0][1], cams[1][1]], [K[0].copy(), K[1].copy()], pts)
    pr = BAProblem(uv, pts[0].copy(), [K[0].copy(), K[1].copy()])
    trace: List[float] = []
    s, its = bundle_adjust(s0, pr, max_iters, trace)
    if indeterminate(s, pr):
        return PairResult(False, None, None, np.zeros(0, np.int64), len(keep), its, trace, True)
    err = np.zeros(len(keep))
    for c in range(2):
        pr_uv, z, _, _ = project_many(s.R[c], s.t[c], s.cal[c], s.pts)
        err = np.maximum(err, np.where(z > 0.0, np.linalg.norm(pr_uv - uv[:, c], axis=1), np.inf))
    valid = err < ba_thr
    if not valid.any():  # no camera left in the filtered result: the initial pose (two_view_estimator.py:276-278)
        return PairResult(True, R0, t0, np.zeros(0, np.int64), len(keep), its, trace, True, keep, err)
    R = s.R[1].T @ s.R[0]  # wTi2.between(wTi1)
    t = s.R[1].T @ (s.t[0] - s.t[1])
    return PairResult(True, R, t / np.linalg.norm(t), keep[valid], len(keep), its, trace, True, keep, err)

