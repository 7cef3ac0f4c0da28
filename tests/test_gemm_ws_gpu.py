"""GPU: the batched wgmma split-fp16 GEMM (k_gemm_ws) at ragged shapes, through b2_debug_gemm_host, against fp64 NumPy.

Shapes cover an 8-row and a 1-row last row tile (M = 5000, 129, 1), fewer tiles than SMs, a column tile cut at N = 64, 200
and 130 (130 has no 16-byte aligned rows, so the epilogue takes its per-element path), and K from one to eight 64-wide
chunks.  A timed-out pipeline wait raises through the error flag.

Tolerance: split-fp16 operands carry 22 significand bits and the dropped lo * lo product is 2^-22 relative, so the result is
off by a few 2^-22 of sum_k |a_k b_k|; fp32 accumulation adds far less at these K.  The bound is 16 * 2^-22 of that sum.
It is checked to be tight enough to matter: a plain fp16 GEMM (hi planes only) must exceed it at every shape."""
import numpy as np
import pytest

from gtsfm_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K", [64, 256, 512])
@pytest.mark.parametrize("N", [64, 130, 200, 768])
@pytest.mark.parametrize("M", [1, 8, 129, 5000])
def test_gemm_ws_matches_fp64(b200_ctx, M, N, K):
    rng = np.random.default_rng(1000 * M + 10 * N + K)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    C = np.full((M, N), np.nan, np.float32)
    rc = b200_ctx.lib.b2_debug_gemm_host(b200_ctx.handle, 1, _lib.ptr(A), _lib.ptr(B), _lib.ptr(bias), _lib.ptr(C), M, N, K)
    b200_ctx.check(rc, "b2_debug_gemm_host")
    want = A.astype(np.float64) @ B.astype(np.float64).T + bias
    bound = 16 * 2.0 ** -22 * (np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T) + 2.0 ** -22 * np.abs(bias)
    hi_only = A.astype(np.float16).astype(np.float64) @ B.astype(np.float16).astype(np.float64).T + bias
    assert (np.abs(hi_only - want) > bound).any(), "the bound does not tell split-fp16 from plain fp16 at this shape"
    assert np.isfinite(C).all()
    err = np.abs(C - want)
    assert (err <= bound).all(), (M, N, K, float(err.max()), float((err / bound).max()))
