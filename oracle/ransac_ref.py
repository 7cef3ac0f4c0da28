"""TEST INFRASTRUCTURE — fp64 NumPy restatement of the RANSAC verifier's stages (gtsfm_b200/csrc/ransac.cu), never shipped.

Written from the algorithms, not from the kernels: the counter-based sampler (SplitMix64), the squared Sampson and
symmetric epipolar-line errors, MSAC scoring, the normalised 8-point algorithm (Hartley 1997) with NumPy's eigen and
singular value decompositions, the top-8 candidate selection across batches with its confidence bound, the iterated
least-squares local optimisation, the pick, the inlier mask and the cheirality vote by linear triangulation.

The device works in fp64 with fixed-order reductions, so most stages replay exactly (integers, selections, masks away
from the threshold) or to within a few ulps; what does not (eigenvectors from a different eigen-solver) is held to a
bound the tests derive and state.
"""
from __future__ import annotations

import ctypes
import shutil
import subprocess
from dataclasses import dataclass, field
from pathlib import Path
from typing import List, Optional, Sequence

import numpy as np

from oracle.verifier_ref import sampson_sq

MAX_SOL = 10  # solution slots per sample
TOP = 8  # candidates handed to the local optimisation
LO_ITERS = 6
MIN_LO_POINTS = 8
BIG = 1e300  # cost of an empty slot / invalid candidate
SQRT2 = 1.4142135623730951

_U64 = np.uint64
_GOLDEN = _U64(0x9E3779B97F4A7C15)


def build_shim(out_dir: Path, qr: bool = True) -> ctypes.CDLL:
    """g++ build of tests/cpp/ransac_shim.cpp, the host build of ransac_math.cuh behind a C ABI (-DB2_FIVEPT_QR: the
    5-point variant libgtsfm_b200.so compiles)."""
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    so = Path(out_dir) / "ransac_shim.so"
    src = Path(__file__).resolve().parent.parent / "tests" / "cpp" / "ransac_shim.cpp"
    subprocess.run([cxx, "-O2", "-std=c++17", "-shared", "-fPIC", *(["-DB2_FIVEPT_QR"] if qr else []), str(src), "-o", str(so)], check=True)
    lib = ctypes.CDLL(str(so))
    vp, i, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64
    lib.shim_sample_distinct.argtypes = [u64, u64, i, i, i, vp]
    lib.shim_error.argtypes = [i, vp, vp, vp, i, vp]
    lib.shim_eightpt.argtypes = [vp, vp, vp]
    lib.shim_eightpt.restype = i
    lib.shim_fivept.argtypes = [vp, vp, vp]
    lib.shim_fivept.restype = i
    return lib


# ---- sampler ------------------------------------------------------------------------------------------------------

def splitmix64(state: np.ndarray):
    """One SplitMix64 step on a uint64 array of states -> (next states, outputs), wrapping arithmetic."""
    with np.errstate(over="ignore"):
        z = state + _GOLDEN
        nxt = z.copy()
        z = (z ^ (z >> _U64(30))) * _U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> _U64(27))) * _U64(0x94D049BB133111EB)
    return nxt, z ^ (z >> _U64(31))


def sample_distinct(seed: int, streams: Sequence[int], n: int, m: int) -> np.ndarray:
    """m distinct indices in [0, n) per stream: draw SplitMix64 % n, redraw on a repeat.  -> int64 [len(streams)][m]."""
    streams = np.asarray(streams, np.uint64)
    with np.errstate(over="ignore"):
        st = _U64(seed) * _U64(0xD1342543DE82EF95) + streams * _U64(0x2545F4914F6CDD1D) + _U64(0x1234567)
    out = np.full((len(streams), m), -1, np.int64)
    for i in range(m):
        todo = np.ones(len(streams), bool)
        while todo.any():
            st[todo], v = splitmix64(st[todo])
            v = (v % _U64(n)).astype(np.int64)
            rows = np.flatnonzero(todo)
            dup = (out[rows, :i] == v[:, None]).any(1)
            out[rows[~dup], i] = v[~dup]
            todo[rows[~dup]] = False
    return out


# ---- errors and scoring ---------------------------------------------------------------------------------------------

def epiline_sq(F: np.ndarray, x1: np.ndarray, x2: np.ndarray) -> np.ndarray:
    """Larger of the two squared point-to-epipolar-line distances (pixels for F)."""
    p1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    p2 = np.concatenate([x2, np.ones((len(x2), 1))], 1)
    l2, l1 = p1 @ F.T, p2 @ F  # epipolar lines in image 2 / image 1
    d2 = np.sum(p2 * l2, 1) ** 2 / (l2[:, 0] ** 2 + l2[:, 1] ** 2 + 1e-300)
    d1 = np.sum(p1 * l1, 1) ** 2 / (l1[:, 0] ** 2 + l1[:, 1] ** 2 + 1e-300)
    return np.maximum(d1, d2)


def error(mode: int, M: np.ndarray, x1: np.ndarray, x2: np.ndarray) -> np.ndarray:
    """mode 0: squared Sampson distance (E), 1: symmetric epiline distance (F)."""
    M = np.asarray(M, np.float64).reshape(3, 3)
    return sampson_sq(M, x1, x2) if mode == 0 else epiline_sq(M, x1, x2)


def msac(err: np.ndarray, thr2: float):
    """-> (MSAC cost sum(min(e, thr2)) with e < thr2 as the inlier test, inlier count)."""
    inl = err < thr2
    return float(np.sum(np.where(inl, err, thr2))), int(inl.sum())


# ---- hypotheses ---------------------------------------------------------------------------------------------------

def _hartley(x: np.ndarray):
    """centroid and scale sqrt(2) / mean distance to it, or None when the points coincide."""
    c = x.mean(0)
    d = np.sqrt(((x - c) ** 2).sum(1)).sum()
    if d < 1e-12:
        return None
    return c, SQRT2 * len(x) / d


def _design_rows(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """rows q with q . vec(F) = b^T F a (F row-major)."""
    one = np.ones(len(a))
    return np.stack([b[:, 0] * a[:, 0], b[:, 0] * a[:, 1], b[:, 0], b[:, 1] * a[:, 0], b[:, 1] * a[:, 1], b[:, 1], a[:, 0], a[:, 1], one], 1)


def _linear_fit(x1: np.ndarray, x2: np.ndarray, essential: bool, rank2_normalised: bool = False) -> Optional[np.ndarray]:
    """Hartley-normalised least squares: smallest eigenvector of sum q q^T, denormalised, projected onto the essential
    (singular values 1, 1, 0) or rank-2 manifold, unit Frobenius norm.  rank2_normalised: F is made rank 2 before it is
    denormalised (the 8-point hypotheses) instead of after (the local optimisation)."""
    n1, n2 = _hartley(x1), _hartley(x2)
    if n1 is None or n2 is None:
        return None
    (c1, s1), (c2, s2) = n1, n2
    Q = _design_rows((x1 - c1) * s1, (x2 - c2) * s2)
    w, V = np.linalg.eigh(Q.T @ Q)
    Fn = V[:, 0].reshape(3, 3)
    T1 = np.array([[s1, 0, -s1 * c1[0]], [0, s1, -s1 * c1[1]], [0, 0, 1.0]])
    T2 = np.array([[s2, 0, -s2 * c2[0]], [0, s2, -s2 * c2[1]], [0, 0, 1.0]])
    if rank2_normalised:
        U, sv, Vt = np.linalg.svd(Fn)
        F = T2.T @ (U @ np.diag([sv[0], sv[1], 0.0]) @ Vt) @ T1
    else:
        U, sv, Vt = np.linalg.svd(T2.T @ Fn @ T1)
        F = U @ np.diag([1.0, 1.0, 0.0] if essential else [sv[0], sv[1], 0.0]) @ Vt
    nrm = np.linalg.norm(F)
    if not nrm > 1e-300:
        return None
    return F / nrm


def eightpt(x1: np.ndarray, x2: np.ndarray) -> Optional[np.ndarray]:
    """Normalised 8-point F of 8 correspondences (rank 2, unit norm; sign arbitrary), None when degenerate."""
    return _linear_fit(np.asarray(x1, np.float64), np.asarray(x2, np.float64), essential=False, rank2_normalised=True)


def essential_residuals(E: np.ndarray):
    """-> (|norm - 1|, max |2 E E^T E - tr(E E^T) E|): the essential-matrix identities of a unit-norm E."""
    E = np.asarray(E, np.float64).reshape(3, 3)
    EEt = E @ E.T
    return abs(np.linalg.norm(E) - 1.0), float(np.abs(2 * EEt @ E - np.trace(EEt) * E).max())


# ---- selection ----------------------------------------------------------------------------------------------------

@dataclass
class Candidate:
    model: np.ndarray
    cost: float
    ninl: int
    valid: bool = True


def invalid() -> Candidate:
    return Candidate(np.zeros(9), BIG, 0, False)


def select(cands: List[Candidate], models: np.ndarray, cost: np.ndarray, ninl: np.ndarray) -> List[Candidate]:
    """Merge one batch into the running list: the TOP lowest (cost, index) among the valid candidates (index j - TOP, so
    earlier arrivals win ties) and the batch's non-empty slots (index = slot)."""
    pool = [(c.cost, j - TOP, c) for j, c in enumerate(cands) if c.valid]
    live = np.flatnonzero(cost < 1e299)
    order = live[np.lexsort((live, cost[live]))][:TOP]
    pool += [(float(cost[i]), int(i), None) for i in order]
    pool.sort(key=lambda e: (e[0], e[1]))
    out = []
    for c, i, cand in pool[:TOP]:
        out.append(cand if cand is not None else Candidate(np.array(models[i], np.float64), c, int(ninl[i])))
    return out + [invalid() for _ in range(TOP - len(out))]


def samples_needed(ninl: int, k: int, m: int, confidence: float) -> float:
    """Standard RANSAC bound log(1 - confidence) / log(1 - w^m) for inlier ratio w = ninl / k."""
    pw = (ninl / k) ** m
    if pw >= 1.0:
        return 1.0
    if pw <= 0.0:
        return 1e300
    return float(np.log(1.0 - confidence) / np.log(1.0 - pw))


def more_flag(best: Candidate, k: int, m: int, confidence: float, done_after: int) -> int:
    """The device's 'not enough samples yet' flag after a batch (1 without a valid candidate)."""
    if not best.valid:
        return 1
    return int(samples_needed(best.ninl, k, m, confidence) > done_after)


@dataclass
class Schedule:
    batches: List[int] = field(default_factory=list)  # samples per sampling batch
    extension: int = 0  # samples of the E extension stage when enqueued (0: not enqueued)


def schedule(mode: int, max_iters: int, batch: int, best_ninl_after, k: int, confidence: float) -> Schedule:
    """The host loop: batches of min(batch, remaining) samples, stopping early when the bound of the best candidate after
    a batch (best_ninl_after(b) -> ninl, or None when invalid) is met; the E extension is enqueued only when the whole
    budget ran and max_iters <= 4096."""
    hard_cap = 65536 if mode == 0 else 262144
    max_iters = min(max(max_iters, 1), hard_cap)
    m = 5 if mode == 0 else 8
    out, done = Schedule(), 0
    while done < max_iters:
        n = min(batch, max_iters - done)
        out.batches.append(n)
        done += n
        if done >= max_iters:
            break
        ni = best_ninl_after(len(out.batches) - 1)
        if ni is not None and done >= samples_needed(ni, k, m, confidence):
            break
    if mode == 0 and done >= max_iters and max_iters <= 4096:
        out.extension = min(4 * max_iters, batch)
    return out


# ---- local optimisation, pick, mask -------------------------------------------------------------------------------

def refine(mode: int, x1: np.ndarray, x2: np.ndarray, thr2: float, cand: Candidate) -> Candidate:
    """Iterated least-squares refit from one candidate: support at 4x, 2x, then 1x thr2; a refit is kept only when its MSAC
    cost at thr2 is lower; the loop ends when fewer than 8 points are selected, or on a non-improving refit from the third
    iteration on."""
    if not cand.valid:
        return cand
    M, cur, ninl = np.array(cand.model, np.float64), cand.cost, cand.ninl
    for it in range(LO_ITERS):
        sel2 = thr2 * (4.0 if it == 0 else (2.0 if it == 1 else 1.0))
        inl = error(mode, M, x1, x2) < sel2
        if inl.sum() < MIN_LO_POINTS:
            break
        F = _linear_fit(x1[inl], x2[inl], essential=mode == 0)
        if F is None:
            break
        c, ni = msac(error(mode, F, x1, x2), thr2)
        if not c < cur:
            if it >= 2:
                break
            continue
        M, cur, ninl = F.ravel(), c, ni
    return Candidate(M, cur, ninl, True)


def pick(cands: Sequence[Candidate]) -> Optional[int]:
    """Index of the valid candidate with the lowest cost, ties to the lower rank (None: no valid candidate)."""
    b = None
    for j, c in enumerate(cands):
        if c.valid and (b is None or c.cost < cands[b].cost):
            b = j
    return b


# ---- cheirality vote ----------------------------------------------------------------------------------------------

def cheirality(R: np.ndarray, t: np.ndarray, x1: np.ndarray, x2: np.ndarray, dist: float = 50.0, margin: float = 1e-9):
    """Linear triangulation under P1 = [I|0], P2 = [R|t] (smallest eigenvector of the 4 x 4 normal equations), in front
    of both cameras and closer than `dist`.  -> (ok [k] bool, ambiguous [k] bool): ambiguous marks points whose depths lie
    within `margin` (relative) of 0 or dist, or whose two smallest eigenvalues are too close to fix the eigenvector."""
    R, t = np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).ravel()
    k = len(x1)
    if k == 0:
        return np.zeros(0, bool), np.zeros(0, bool)
    rows = np.zeros((k, 4, 4))
    rows[:, 0, 0] = -1
    rows[:, 0, 2] = x1[:, 0]
    rows[:, 1, 1] = -1
    rows[:, 1, 2] = x1[:, 1]
    rows[:, 2, :3] = x2[:, :1] * R[2] - R[0]
    rows[:, 2, 3] = x2[:, 0] * t[2] - t[0]
    rows[:, 3, :3] = x2[:, 1:2] * R[2] - R[1]
    rows[:, 3, 3] = x2[:, 1] * t[2] - t[1]
    A = np.einsum("kri,krj->kij", rows, rows)
    w, V = np.linalg.eigh(A)
    X = V[:, :, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        P = X[:, :3] / X[:, 3:]
        z1 = P[:, 2]
        z2 = P @ R[2] + t[2]
    ok = (np.abs(X[:, 3]) >= 1e-300) & (z1 > 0) & (z1 < dist) & (z2 > 0) & (z2 < dist)
    scale = 1.0 + np.abs(z1) + np.abs(z2)
    near = np.minimum.reduce([np.abs(z1), np.abs(z1 - dist), np.abs(z2), np.abs(z2 - dist)]) < margin * scale * dist
    gap = (w[:, 1] - w[:, 0]) < 1e-10 * np.abs(w[:, 3])
    return ok, near | gap | ~np.isfinite(scale)


def votes(cands21: np.ndarray, x1: np.ndarray, x2: np.ndarray):
    """Cheirality votes of the four decompositions (R1,t), (R2,t), (R1,-t), (R2,-t) given as R1 [9], R2 [9], t [3].
    -> (votes [4], ambiguous counts [4])."""
    c = np.asarray(cands21, np.float64)
    R1, R2, t = c[:9], c[9:18], c[18:21]
    v, a = [], []
    for R, sg in ((R1, 1), (R2, 1), (R1, -1), (R2, -1)):
        ok, amb = cheirality(R, sg * t, x1, x2)
        v.append(int(ok.sum()))
        a.append(int(amb.sum()))
    return np.array(v), np.array(a)


def vote_winner(tot: Sequence[int]) -> int:
    """First maximum, in the order (R1,t), (R2,t), (R1,-t), (R2,-t)."""
    b = 0
    for c in range(1, 4):
        if tot[c] > tot[b]:
            b = c
    return b
