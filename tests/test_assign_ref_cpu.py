"""CPU: the fp64 assignment restatements of oracle/assign_ref.py (the yardstick of tests/test_assign_gpu.py) agree with the
oracle's torch functions run in float64."""
import numpy as np
import pytest
import torch

from oracle import assign_ref, lightglue_ref, superglue_ref


@pytest.fixture
def float64_default():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)  # the oracle builds norm / log_mu from Python floats
    yield
    torch.set_default_dtype(old)


@pytest.mark.parametrize("iters", [0, 1, 20])
@pytest.mark.parametrize("M,N,alpha", [(7, 5, 1.0), (40, 3, -5.0), (33, 70, 8.0)])
def test_log_optimal_transport_pinned(float64_default, M, N, alpha, iters):
    Z = np.random.default_rng(M * N + iters).standard_normal((M, N)) * 3
    want = superglue_ref.log_optimal_transport(torch.from_numpy(Z), torch.tensor(alpha), iters).numpy()
    got, u, v, _, _ = assign_ref.log_optimal_transport(Z, alpha, iters)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got[:M, :N], Z + u[:M, None] + v[None, :N] + np.log(M + N), rtol=0, atol=1e-12)


@pytest.mark.parametrize("M,N", [(1, 1), (6, 9), (50, 20)])
def test_double_log_softmax_pinned(float64_default, M, N):
    rng = np.random.default_rng(M + 100 * N)
    D = 8
    a0, a1 = rng.standard_normal((M, D)) * 2, rng.standard_normal((N, D)) * 2
    z0, z1 = rng.standard_normal(M) * 30, rng.standard_normal(N) * 30
    # final_proj passes the first D features through (its output is divided by 256 ** 0.25 again), matchability reads the last
    w = np.zeros((D + 1, D + 1))
    w[:D, :D] = np.eye(D) * 256 ** 0.25
    mw = np.zeros((1, D + 1))
    mw[0, D] = 1.0
    sd = {"log_assignment.0.final_proj.weight": w, "log_assignment.0.final_proj.bias": np.zeros(D + 1),
          "log_assignment.0.matchability.weight": mw, "log_assignment.0.matchability.bias": np.zeros(1)}
    d0 = torch.from_numpy(np.hstack([a0, z0[:, None]]))
    d1 = torch.from_numpy(np.hstack([a1, z1[:, None]]))
    want = lightglue_ref.log_assignment(sd, 0, d0, d1).numpy()[:M, :N]
    got, lr, lc = assign_ref.double_log_softmax(a0 @ a1.T, z0, z1)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-10)
    np.testing.assert_allclose(assign_ref.logsigmoid(z0), torch.nn.functional.logsigmoid(torch.from_numpy(z0)).numpy(), rtol=0, atol=1e-14)


def test_mutual_filter_takes_the_first_maximum_like_torch():
    rng = np.random.default_rng(3)
    core = np.round(rng.standard_normal((60, 40)), 1)  # many exact ties
    core[:, 7] = core[:, 3]  # duplicated column: rows maximal at 3 tie with 7
    core[11] = core[5]  # duplicated row
    rows, cols, sc = assign_ref.mutual_filter(core, 0.2)
    t = torch.from_numpy(core)
    mx0, a0 = t.max(1)
    _, a1 = t.max(0)
    mutual = torch.arange(t.shape[0]) == a1[a0]
    valid = mutual & (torch.where(mutual, mx0.exp(), mx0.new_tensor(0)) > 0.2)
    want = torch.where(valid)[0].numpy()
    assert np.array_equal(rows, want) and np.array_equal(cols, a0.numpy()[want])
    np.testing.assert_allclose(sc, mx0.exp().numpy()[want], rtol=1e-15)
    assert 11 not in rows.tolist() or 5 not in rows.tolist()
