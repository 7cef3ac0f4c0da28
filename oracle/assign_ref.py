"""TEST INFRASTRUCTURE — fp64 NumPy restatements of the matchers' assignment step (never shipped).

* ``log_optimal_transport`` restates superglue.py:141-170 (oracle/superglue_ref.py:60-74), norm = -log(M + N).
* ``double_log_softmax`` restates the score of sigmoid_log_double_softmax, lightglue.py:265-277
  (oracle/lightglue_ref.py:107-119): log_softmax over rows + over columns + logsigmoid(z0) + logsigmoid(z1).
* ``mutual_filter`` restates the mutual arg-max + threshold of superglue.py:266-276 and lightglue.py:302-318
  (oracle/superglue_ref.py:96-101, oracle/lightglue_ref.py:176-183); like torch.max it takes the first maximum.

tests/test_assign_ref_cpu.py pins them to the oracle's torch functions run in float64.
"""
from __future__ import annotations

import numpy as np


def lse(x: np.ndarray, axis: int) -> np.ndarray:
    m = x.max(axis, keepdims=True)
    return (np.log(np.exp(x - m).sum(axis, keepdims=True)) + m).squeeze(axis)


def logsigmoid(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, np.float64)
    return np.minimum(z, 0.0) - np.log1p(np.exp(-np.abs(z)))


def log_optimal_transport(Z: np.ndarray, alpha: float, iters: int):
    """-> (scores [M + 1][N + 1], u [M + 1], v [N + 1], amax_r, amax_c): amax_r / amax_c bound |x| of every term that entered a
    row / column logsumexp in any iteration."""
    m, n = Z.shape
    z = np.empty((m + 1, n + 1))
    z[:m, :n] = Z
    z[:m, n] = alpha
    z[m, :] = alpha
    norm = -np.log(float(m + n))
    log_mu = np.concatenate([np.full(m, norm), [np.log(float(n)) + norm]])
    log_nu = np.concatenate([np.full(n, norm), [np.log(float(m)) + norm]])
    u, v = np.zeros(m + 1), np.zeros(n + 1)
    zmax = np.abs(z).max()
    amax_r = amax_c = 0.0
    for _ in range(iters):
        amax_r = max(amax_r, zmax + np.abs(v).max())
        u = log_mu - lse(z + v[None, :], 1)
        amax_c = max(amax_c, zmax + np.abs(u).max())
        v = log_nu - lse(z + u[:, None], 0)
    return z + u[:, None] + v[None, :] - norm, u, v, amax_r, amax_c


def double_log_softmax(sim: np.ndarray, z0: np.ndarray, z1: np.ndarray):
    """-> (scores [M][N], row logsumexp [M], column logsumexp [N])."""
    s = np.asarray(sim, np.float64)
    lr, lc = lse(s, 1), lse(s, 0)
    return (s - lr[:, None]) + (s - lc[None, :]) + (logsigmoid(z0)[:, None] + logsigmoid(z1)[None, :]), lr, lc


def mutual_filter(core: np.ndarray, threshold: float):
    """-> (rows i ascending, matches0[i], exp(max_j core[i])) of the mutual, above-threshold row maxima."""
    a0, a1 = core.argmax(1), core.argmax(0)
    mx0 = core[np.arange(core.shape[0]), a0]
    mutual = a1[a0] == np.arange(core.shape[0])
    valid = mutual & (np.where(mutual, np.exp(mx0), 0.0) > threshold)
    rows = np.nonzero(valid)[0]
    return rows, a0[rows], np.exp(mx0[rows])
