"""GPU: the column-segment epilogue of the wgmma GEMM (k_gemm_ws) that writes LightGlue's attention operands.

- Self attention: one launch writes rotated q, rotated k and v as head-major split planes.  It must equal, bit for bit, the
  unfused sequence: the same GEMM with an fp32 output, then rotary (lightglue.py:58-65) with round-to-nearest fp32 products
  and sums, then the split into fp16 hi and unscaled lo (hi = fp16(clamp(x)), lo = fp16(clamp(x) - hi)).
- Cross attention: [to_qk; to_v] as one N = 512 launch must equal two separate N = 256 launches, bit for bit.

M covers a single row, half a row tile, one whole row tile, ragged last row tiles of 1 row (129, 257) and the default
workload's 5000 keypoints; cos / sin are random.  The unfused GEMM runs through b2_debug_linear_host (one problem, fp32
output)."""
import ctypes

import numpy as np
import pytest

from gtsfm_b200 import _lib

pytestmark = pytest.mark.gpu

K = 256


def _operands(M, nseg, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = (rng.standard_normal((256 * nseg, K)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(256 * nseg).astype(np.float32)
    return A, B, bias


def _segments(ctx, A, B, bias, nseg, rot_mask=0, cs=None, sn=None, separate=0):
    M = A.shape[0]
    hi = np.zeros((nseg, 4, M, 64), np.uint16)
    lo = np.zeros((nseg, 4, M, 64), np.uint16)
    rc = ctx.lib.b2_debug_gemm_segments_host(ctx.handle, _lib.ptr(A), _lib.ptr(B), _lib.ptr(bias), M, K, nseg, rot_mask, _lib.ptr(cs),
                                             _lib.ptr(sn), separate, _lib.ptr(hi), _lib.ptr(lo))
    ctx.check(rc, "b2_debug_gemm_segments_host")
    return hi, lo


def _split_unscaled(x):
    x = np.clip(x, np.float32(-65504.0), np.float32(65504.0))
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi.view(np.uint16), lo.view(np.uint16)


@pytest.mark.parametrize("M", [1, 64, 128, 129, 257, 5000])
def test_rotary_segments_equal_fp32_gemm_then_rotary_and_split(b200_ctx, M):
    A, B, bias = _operands(M, 3, 7 + M)
    rng = np.random.default_rng(100 + M)
    ang = rng.uniform(-np.pi, np.pi, (M, 32))
    cs, sn = np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)
    C = np.full((M, 768), np.nan, np.float32)
    launch = _lib.LinearLaunch(path=1, k1=K, bias=_lib.ptr(bias).value, scale=1.0)
    prob = _lib.LinearProblem(a1=_lib.ptr(A).value, lda1=K, b=_lib.ptr(B).value, ldb=K, c=_lib.ptr(C).value, ldc=768, m=M, n=768)
    rc = b200_ctx.lib.b2_debug_linear_host(b200_ctx.handle, ctypes.byref(launch), ctypes.byref(prob), 1)
    b200_ctx.check(rc, "b2_debug_linear_host")
    hi, lo = _segments(b200_ctx, A, B, bias, 3, rot_mask=3, cs=cs, sn=sn)
    for s in range(3):
        x = C[:, 256 * s:256 * (s + 1)].reshape(M, 4, 32, 2)
        if s < 2:  # (t * cos) + (rotate_half(t) * sin): every float32 product and sum rounds on its own, as __fmul_rn / __fadd_rn
            c, sn_ = cs[:, None, :], sn[:, None, :]
            x0, x1 = x[..., 0], x[..., 1]
            x = np.stack([x0 * c + (-x1) * sn_, x1 * c + x0 * sn_], -1)
        want_hi, want_lo = _split_unscaled(np.ascontiguousarray(x.reshape(M, 4, 64).transpose(1, 0, 2)))
        assert np.array_equal(hi[s], want_hi), (M, s, int((hi[s] != want_hi).sum()))
        assert np.array_equal(lo[s], want_lo), (M, s, int((lo[s] != want_lo).sum()))


@pytest.mark.parametrize("M", [1, 129, 5000])
def test_merged_qk_v_launch_equals_two_launches(b200_ctx, M):
    A, B, bias = _operands(M, 2, 11 + M)
    merged = _segments(b200_ctx, A, B, bias, 2)
    separate = _segments(b200_ctx, A, B, bias, 2, separate=1)
    for got, want in zip(merged, separate):
        assert np.array_equal(got, want)
