"""CPU suite: oracle/ransac_ref.py (the fp64 NumPy restatement the verifier's stage tests replay against) pinned to the
host build of gtsfm_b200/csrc/ransac_math.cuh, through the small C shim tests/cpp/ransac_shim.cpp."""
import ctypes

import numpy as np
import pytest

from oracle import ransac_ref as rr
from oracle import verifier_ref as vr


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return rr.build_shim(tmp_path_factory.mktemp("shim"))


@pytest.mark.parametrize("seed,n,m", [(0x5EED, 1000, 5), (1, 8, 8), (2**64 - 1, 9, 8), (12345, 70000, 5), (7, 5, 5), (3, 2**31 - 1, 8)])
def test_sampler_exact(shim, seed, n, m):
    """sample_distinct: the same integers as the host build, including small n (many redraws) and wrapping seeds."""
    count, stream0 = 3000, 2**40 - 17
    host = np.zeros((count, m), np.int32)
    shim.shim_sample_distinct(seed, stream0, count, n, m, _p(host))
    ref = rr.sample_distinct(seed, np.arange(count, dtype=np.uint64) + np.uint64(stream0), n, m)
    assert np.array_equal(ref, host)
    assert all(len(set(r)) == m for r in ref.tolist()) and ref.min() >= 0 and ref.max() < n


@pytest.mark.parametrize("mode", [0, 1])
def test_error_metrics_ulp(shim, mode):
    """Squared Sampson (E) and symmetric epiline (F) error: within a few ulps of the host build on a scene with inliers,
    outliers and points near the epipoles."""
    kp1, kp2, _, K, R, t, _ = vr.synthetic_two_view(4, 4000, 0.5)
    if mode == 0:
        x1, x2 = vr.calibrate(kp1, *K), vr.calibrate(kp2, *K)
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        M = tx @ R
    else:
        x1, x2 = kp1, kp2
        Kinv = np.linalg.inv(np.array([[K[0], 0, K[1]], [0, K[0], K[2]], [0, 0, 1]]))
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        M = Kinv.T @ tx @ R @ Kinv
    M = np.ascontiguousarray(M / np.linalg.norm(M)).ravel()
    host = np.zeros(len(x1))
    shim.shim_error(mode, _p(M), _p(np.ascontiguousarray(x1)), _p(np.ascontiguousarray(x2)), len(x1), _p(host))
    ref = rr.error(mode, M, x1, x2)
    # The residual r = x2^T M x1 sums 9 products in a different order: its error is <= 9 eps T, T = |x2|^T |M| |x1|.
    # Squared and divided by a denominator good to a few eps: rel(e) <= 2 * 9 eps T / |r| + 8 eps.
    eps = np.finfo(float).eps
    h1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    h2 = np.concatenate([x2, np.ones((len(x2), 1))], 1)
    T = np.einsum("ki,ij,kj->k", np.abs(h2), np.abs(M.reshape(3, 3)), np.abs(h1))
    r = np.abs(np.einsum("ki,ij,kj->k", h2, M.reshape(3, 3), h1))
    bound = 18 * eps * T / np.maximum(r, 1e-300) + 8 * eps
    rel = np.abs(ref - host) / np.maximum(np.abs(host), 1e-300)
    assert np.all(rel <= bound), (rel.max(), np.max(rel / bound))
    assert np.median(rel) < 4 * eps


def test_eightpt_matches_host_build(shim):
    """The NumPy 8-point F equals the host build's on the same samples, up to sign; degenerate samples give none."""
    kp1, kp2, *_ = vr.synthetic_two_view(6, 500, 0.7)
    idx = rr.sample_distinct(0x5EED, np.arange(400, dtype=np.uint64), len(kp1), 8)
    worst = 0.0
    for s in idx:
        a, b = np.ascontiguousarray(kp1[s]), np.ascontiguousarray(kp2[s])
        F = np.zeros(9)
        assert shim.shim_eightpt(_p(a), _p(b), _p(F)) == 1
        Fr = rr.eightpt(a, b).ravel()
        worst = max(worst, min(np.abs(F - Fr).max(), np.abs(F + Fr).max()))
        assert abs(np.linalg.det(F.reshape(3, 3))) < 1e-12 and abs(np.linalg.norm(F) - 1) < 1e-14
    # eigenvectors of two solvers (Jacobi to off-diagonal mass 1e-30 relative, LAPACK): measured worst ~1e-11 on pixels
    assert worst < 1e-8, worst
    a = np.repeat([[640.0, 480.0]], 8, 0)  # coincident (and exactly representable, so the centroid is exact)
    F = np.zeros(9)
    assert shim.shim_eightpt(_p(np.ascontiguousarray(a)), _p(np.ascontiguousarray(kp2[:8])), _p(F)) == 0
    assert rr.eightpt(a, kp2[:8]) is None


def test_selection_ties_and_schedule():
    """The restated selection keeps earlier candidates on ties and fills invalid slots; the schedule enqueues the
    extension only for E with the whole budget spent and max_iters <= 4096."""
    models = np.arange(30 * 9, dtype=float).reshape(30, 9)
    cost = np.full(30, 5.0)
    cost[[3, 17]] = 1e300
    c0 = rr.select([rr.invalid()] * 8, models, cost, np.ones(30, int))
    assert [int(c.model[0] // 9) for c in c0] == [0, 1, 2, 4, 5, 6, 7, 8]
    c1 = rr.select(c0, models + 1000, cost, np.ones(30, int))
    assert all(a is b for a, b in zip(c0, c1))
    few = rr.select([rr.invalid()] * 8, models[:3], np.array([2.0, 1e300, 1.0]), np.ones(3, int))
    assert [c.valid for c in few] == [True, True] + [False] * 6 and few[0].cost == 1.0
    assert rr.schedule(0, 5000, 1000, lambda b: None, 100, 0.99).batches == [1000] * 5
    assert rr.schedule(0, 4096, 1000, lambda b: None, 100, 0.99).extension == 1000
    assert rr.schedule(0, 4097, 16384, lambda b: None, 100, 0.99).extension == 0
    assert rr.schedule(1, 5000, 1000, lambda b: 100, 100, 0.99).batches == [1000]
