"""NumPy statement of 1DSfM's translation recovery: gtsam's TranslationRecovery::run(measurements, scale) as the reference's
averaging_1dsfm.py:__run_averaging calls it (csrc/translation_recovery.cu and translation_math.cuh restate it on the device).

The graph, in the reference's measurement order (every camera pair (i1, i2) -> (C(i2), C(i1), w_i2Ui1) first, then every
track measurement (j, i) -> (C(i), L(j), w_iUj)):
  - TranslationFactor(a, b, m): error normalize(x_b - x_a) - m, Jacobians -N (a) and +N (b), N gtsam's normalize()
    derivative; Isotropic.Sigma(2, 0.01) whitens by 1 / sigma whatever its declared dimension, and Robust(Huber(1.3))
    reweights on the norm of the whole whitened 3-vector;
  - addPrior: PriorFactor<Point3>(a_0, 0, Isotropic(3, 0.01)) and PriorFactor<Point3>(b_0, scale m_0, edge 0's model);
  - initializeRandomly: a then b of every edge in order, a new key gets Point3(u(), u(), u()) from gtsam's process-wide
    std::mt19937(42) with uniform_real_distribution(-1, 1); g++ evaluates the arguments right to left, so z takes the first
    draw;
  - LevenbergMarquardtParams() defaults (twoview_ba_ref's constants), lambda I damping on every unknown.
`step` eliminates the landmarks (3 x 3 blocks) and solves the reduced camera system by a dense Cholesky, as the device does;
`dense_step` solves the same damped system over every unknown at once, which the tests compare it against.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import scipy.linalg as sla

from oracle import twoview_ba_ref as tv

SIGMA = 0.01          # averaging_1dsfm.py NOISE_MODEL_SIGMA
HUBER_K = 1.3         # averaging_1dsfm.py HUBER_LOSS_K
PRIOR_SIGMA = 0.01    # TranslationRecovery::addPrior's default priorNoiseModel, Isotropic::Sigma(3, 0.01)
MAX_ITERS = 100       # LevenbergMarquardtParams().maxIterations


class Mt19937Uniform:
    """std::uniform_real_distribution<double>(-1, 1) on std::mt19937(seed), as libstdc++ draws it: two 32-bit words per
    value, (w0 + w1 2^32) / 2^64 in double, mapped to 2 c - 1.  NumPy's legacy-seeded MT19937 emits std::mt19937's words."""

    def __init__(self, seed: int = 42):
        self.bg = np.random.MT19937()
        self.bg._legacy_seeding(seed)

    def __call__(self) -> float:
        w0, w1 = (float(w) for w in self.bg.random_raw(2))
        c = (w0 + w1 * 4294967296.0) / 18446744073709551616.0
        if c >= 1.0:
            c = float(np.nextafter(1.0, 0.0))
        return 2.0 * c + -1.0

    def point3(self) -> np.ndarray:
        z = self()
        y = self()
        x = self()
        return np.array([x, y, z])


def initialise(ea, eb, V: int, u: Mt19937Uniform) -> np.ndarray:
    """initializeRandomly: every node in order of first appearance (a, then b, of each edge) draws its Point3."""
    x = np.full((V, 3), np.nan)
    seen = np.zeros(V, bool)
    for a, b in zip(ea, eb):
        for n in (int(a), int(b)):
            if not seen[n]:
                seen[n] = True
                x[n] = u.point3()
    return x


@dataclass
class Problem:
    C: int
    L: int
    ea: np.ndarray     # (E,) node ids: cameras 0..C-1, landmarks C..C+L-1
    eb: np.ndarray
    meas: np.ndarray   # (E, 3)
    sigma: float = SIGMA
    huber_k: float = HUBER_K  # 0: no robust model
    prior_sigma: float = PRIOR_SIGMA
    scale: float = 1.0
    max_iters: int = MAX_ITERS

    def __post_init__(self):
        self.ea = np.asarray(self.ea, np.int64)
        self.eb = np.asarray(self.eb, np.int64)
        self.meas = np.asarray(self.meas, np.float64).reshape(-1, 3)
        self.lmk = (self.ea >= self.C) | (self.eb >= self.C)           # landmark edges
        self.lidx = np.where(self.eb >= self.C, self.eb, self.ea)[self.lmk] - self.C
        self.lcam = np.where(self.eb >= self.C, self.ea, self.eb)[self.lmk]
        self.lsgn = np.where(self.eb >= self.C, 1.0, -1.0)[self.lmk]   # the landmark is b (+N) or a (-N)
        self.priors = [(int(self.ea[0]), np.zeros(3), 1.0 / self.prior_sigma, 0.0),
                       (int(self.eb[0]), self.scale * self.meas[0], 1.0 / self.sigma, self.huber_k)]


def _loss(e, k):
    return np.where(e <= k, 0.5 * e * e, k * (e - 0.5 * k)) if k > 0 else 0.5 * e * e


def _weight(e, k):
    return np.where(e <= k, 1.0, k / np.maximum(e, 1e-300)) if k > 0 else np.ones_like(e)


def _norm(v):
    return np.sqrt(v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2])


def edge_errors(x, pr: Problem, jac: bool = False):
    """Whitened errors (E, 3) of every TranslationFactor at x and, with jac, the whitened Jacobians in b (E, 3, 3)."""
    d = x[pr.eb] - x[pr.ea]
    e = (d / _norm(d)[:, None] - pr.meas) / pr.sigma
    if not jac:
        return e
    x2, y2, z2 = d[:, 0] ** 2, d[:, 1] ** 2, d[:, 2] ** 2
    xy, xz, yz = d[:, 0] * d[:, 1], d[:, 0] * d[:, 2], d[:, 1] * d[:, 2]
    H = np.stack([y2 + z2, -xy, -xz, -xy, x2 + z2, -yz, -xz, -yz, x2 + y2], 1) / ((x2 + y2 + z2) ** 1.5)[:, None]
    return e, H.reshape(-1, 3, 3) / pr.sigma


def _prior(pr: Problem, k: int, x):
    """prior k at x: (node, whitened error, sqrt of its IRLS weight, Jacobian scale)."""
    n, t, inv, hk = pr.priors[k]
    e = (x[n] - t) * inv
    return n, e, float(np.sqrt(_weight(np.array(_norm(e)), hk))), inv


def cost(x, pr: Problem) -> float:
    c = float(np.sum(_loss(_norm(edge_errors(x, pr)), pr.huber_k)))
    for k in range(2):
        n, e, _, _ = _prior(pr, k, x)
        c += 0.5 * float(e @ e) if k == 0 else float(_loss(np.array(_norm(e)), pr.priors[1][3]))
    return c


def linearise(x, pr: Problem):
    """-> (M (E, 3, 3), r (E, 3)): sqrt(w) J_b and sqrt(w) e of every edge, J_a = -M."""
    e, M = edge_errors(x, pr, jac=True)
    sw = np.sqrt(_weight(_norm(e), pr.huber_k))
    return sw[:, None, None] * M, sw[:, None] * e


def _prior_hg(pr: Problem, x, V):
    """The priors at x: (h (V,) onto each node's diagonal, g (V, 3) onto its gradient)."""
    h, g = np.zeros(V), np.zeros((V, 3))
    for k in range(2):
        n, e, sw, inv = _prior(pr, k, x)
        j = sw * inv
        h[n] += j * j
        g[n] += j * (sw * e)
    return h, g


def _lin_dec(x, pr: Problem, lin, dx):
    """The linearised decrease of the step dx and the undamped linearised cost at dx = 0."""
    M, r = lin
    jd = np.einsum("eij,ej->ei", M, dx[pr.eb] - dx[pr.ea])
    dec = -float(np.sum(r * jd + 0.5 * jd * jd))
    old = 0.5 * float(np.sum(r * r))
    for k in range(2):
        n, e, sw, inv = _prior(pr, k, x)
        rr, jj = sw * e, sw * inv * dx[n]
        dec -= float(rr @ jj + 0.5 * jj @ jj)
        old += 0.5 * float(rr @ rr)
    return dec, old


def step(x, pr: Problem, lam: float, lin):
    """One damped trial by the landmark-eliminating Schur solve.  -> (candidate, linearised decrease, old linearised cost,
    dx), or None when a damped block or the reduced system is not positive definite."""
    C, L = pr.C, pr.L
    V = C + L
    M, r = lin
    MtM = np.einsum("eki,ekj->eij", M, M)
    Mtr = np.einsum("eki,ek->ei", M, r)
    h, gp = _prior_hg(pr, x, V)
    lm = pr.lmk
    Hl = np.zeros((L, 3, 3))
    gl = np.zeros((L, 3))
    np.add.at(Hl, pr.lidx, MtM[lm])
    np.add.at(gl, pr.lidx, pr.lsgn[:, None] * Mtr[lm])
    Hl += (h[C:] + lam)[:, None, None] * np.eye(3)
    gl += gp[C:]
    try:
        Lf = np.linalg.cholesky(Hl) if L else np.zeros((0, 3, 3))
    except np.linalg.LinAlgError:
        return None
    z = np.linalg.solve(Lf, gl[..., None])[..., 0] if L else gl
    W = np.linalg.solve(Lf[pr.lidx], -MtM[lm]) if L else np.zeros((0, 3, 3))  # L^-1 H_lc per landmark edge
    # the reduced camera system, block (a, b) at Sb[a, b]
    Sb = np.zeros((C, C, 3, 3))
    cc = ~lm
    a, b = pr.ea[cc], pr.eb[cc]
    np.add.at(Sb, (a, a), MtM[cc])
    np.add.at(Sb, (b, b), MtM[cc])
    np.add.at(Sb, (a, b), -MtM[cc])
    np.add.at(Sb, (b, a), -MtM[cc])
    np.add.at(Sb, (pr.lcam, pr.lcam), MtM[lm])
    order = np.argsort(pr.lidx, kind="stable")
    cnt = np.bincount(pr.lidx, minlength=L)
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    xs, ys = [], []
    for k in np.unique(cnt):  # all (x, y) pairs of every landmark with k edges
        ls = np.nonzero(cnt == k)[0]
        if k == 0:
            continue
        base = start[ls][:, None, None]
        ii, jj = np.meshgrid(np.arange(k), np.arange(k), indexing="ij")
        xs.append((base + ii).ravel())
        ys.append((base + jj).ravel())
    if xs:
        px, py = order[np.concatenate(xs)], order[np.concatenate(ys)]
        np.add.at(Sb, (pr.lcam[px], pr.lcam[py]), -np.einsum("pki,pkj->pij", W[px], W[py]))
    S = Sb.transpose(0, 2, 1, 3).reshape(3 * C, 3 * C)
    S[np.diag_indices(3 * C)] += np.repeat(h[:C], 3) + lam
    g = np.zeros((C, 3))
    np.add.at(g, pr.ea[pr.ea < C], -Mtr[pr.ea < C])
    np.add.at(g, pr.eb[pr.eb < C], Mtr[pr.eb < C])
    np.add.at(g, pr.lcam, -np.einsum("eki,ek->ei", W, z[pr.lidx]) if L else np.zeros((0, 3)))
    g += gp[:C]
    try:
        Lc = np.linalg.cholesky(S)
    except np.linalg.LinAlgError:
        return None
    dc = sla.solve_triangular(Lc.T, sla.solve_triangular(Lc, -g.ravel(), lower=True), lower=False).reshape(C, 3)
    dx = np.zeros((V, 3))
    dx[:C] = dc
    if L:
        y = z.copy()
        np.add.at(y, pr.lidx, np.einsum("eij,ej->ei", W, dc[pr.lcam]))
        dx[C:] = -np.linalg.solve(np.swapaxes(Lf, 1, 2), y[..., None])[..., 0]
    dec, old = _lin_dec(x, pr, lin, dx)
    return x + dx, dec, old, dx


def dense_step(x, pr: Problem, lam: float, lin):
    """The same damped system over all 3 (C + L) unknowns, solved at once (the tests' check of the Schur solve)."""
    V = pr.C + pr.L
    M, r = lin
    E = len(pr.ea)
    J = np.zeros((3 * E, 3 * V))
    for e in range(E):
        J[3 * e:3 * e + 3, 3 * pr.eb[e]:3 * pr.eb[e] + 3] = M[e]
        J[3 * e:3 * e + 3, 3 * pr.ea[e]:3 * pr.ea[e] + 3] = -M[e]
    h, gp = _prior_hg(pr, x, V)
    H = J.T @ J + np.diag(np.repeat(h, 3) + lam)
    g = J.T @ r.ravel() + gp.ravel()
    dx = np.linalg.solve(H, -g).reshape(V, 3)
    dec, old = _lin_dec(x, pr, lin, dx)
    return x + dx, dec, old, dx


@dataclass
class Result:
    x: np.ndarray
    final_error: float
    iterations: int
    trace: List[float]
    trials: List[int] = field(default_factory=list)  # 1 accepted, 0 rejected, 2 rejected and stopped, -1 not positive definite


def recover(pr: Problem, init, solver=step) -> Result:
    """gtsam's LevenbergMarquardtOptimizer::optimize on the graph from `init` (V, 3)."""
    x = np.array(init, float).reshape(-1, 3)
    err = cost(x, pr)
    trace, trials = [err], []
    lam, its, new = tv.LM_LAMBDA0, 0, err
    if err > 0.0:
        while True:
            cur = new
            lin = linearise(x, pr)
            while True:
                st = solver(x, pr, lam, lin)
                success = stop = False
                if st is not None:
                    xn, dec, old, _ = st
                    if dec >= 0.0:
                        e_new = cost(xn, pr)
                        dcost = cur - e_new
                        success = dcost / dec > tv.LM_MIN_FIDELITY if dec > np.finfo(float).eps * old else True
                        stop = abs(dcost) < tv.LM_REL_TOL * cur
                trials.append(-1 if st is None else 1 if success else 2 if stop else 0)
                if success:
                    x, lam, its, new = xn, lam / tv.LM_FACTOR, its + 1, e_new
                    break
                if stop:
                    break
                lam *= tv.LM_FACTOR
                if lam >= tv.LM_LAMBDA_MAX:
                    break
            trace.append(new)
            dec = cur - new
            converged = dec / cur <= tv.LM_REL_TOL or dec <= tv.LM_ABS_TOL or new <= 0.0
            if not (its < pr.max_iters and not converged and np.isfinite(cur)):
                break
    return Result(x, new, its, trace, trials)


ZERO_TOL = 1e-9  # Unit3::equals' default tolerance, against Unit3(0, 0, 0)


def merge_same_translation(V: int, ea, eb, meas):
    """TranslationRecovery::run's zero-translation handling: a DSF over the nodes joined by a measurement equal to
    Unit3(0, 0, 0) (every component within 1e-9), whose nodes share one translation, and the edges between different
    sets, which the graph keeps (on the sets' representatives).  -> (root (V,), keep (E,) bool)."""
    ea, eb = np.asarray(ea, np.int64), np.asarray(eb, np.int64)
    parent = list(range(V))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for e in np.nonzero(np.all(np.abs(np.asarray(meas).reshape(-1, 3)) <= ZERO_TOL, axis=1))[0]:
        ra, rb = find(int(ea[e])), find(int(eb[e]))
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    root = np.array([find(x) for x in range(V)], np.int64)
    return root, root[ea] != root[eb]


def run(C: int, L: int, ea, eb, meas, u: Mt19937Uniform, huber_k: float = HUBER_K, scale: float = 1.0, max_iters: int = MAX_ITERS):
    """TranslationRecovery::run(measurements, scale) on dense nodes (cameras 0..C-1, then landmarks): merge the
    zero-translation sets, drop the edges inside a set, solve the rest from initializeRandomly's values; with no edge
    left every set sits at the origin.  Each node takes its set's value; a set without an edge to the solve has none
    (NaN; gtsam would raise).  -> dict of x (V, 3), root, nodes (the reduced problem's nodes, ascending), and when
    there is a solve problem (on nodes' compact ids), init and result."""
    V = C + L
    ea, eb = np.asarray(ea, np.int64), np.asarray(eb, np.int64)
    meas = np.asarray(meas, float).reshape(-1, 3)
    root, keep = merge_same_translation(V, ea, eb, meas)
    a, b = root[ea[keep]], root[eb[keep]]
    nodes = np.unique(np.concatenate([a, b]))
    x = np.full((V, 3), np.nan)
    out = dict(root=root, nodes=nodes)
    if len(nodes):
        Cr = int(np.sum(nodes < C))
        pr = Problem(Cr, len(nodes) - Cr, np.searchsorted(nodes, a), np.searchsorted(nodes, b), meas[keep], huber_k=huber_k, scale=scale,
                     max_iters=max_iters)
        init = initialise(pr.ea, pr.eb, len(nodes), u)
        res = recover(pr, init)
        x[nodes] = res.x
        out.update(problem=pr, init=init, result=res)
    elif len(ea):
        x[np.unique(root[np.concatenate([ea, eb])])] = 0.0
    out["x"] = x[root]
    return out
