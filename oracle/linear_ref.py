"""fp64 restatement of the shared linear (`run_linear` in gtsfm_b200/csrc/linear.cuh) and the error bound its kernels meet.

One launch computes, per output element,

    out = act((acc + bias) * scale) + resid,    acc = [A1 | A2] B^T,    act = identity, ReLU or exact (erf) GELU,

and may write `out` as fp32 and / or as split fp16 planes: hi = fp16(clamp(out, +-65504)) and lo = fp16((clamp(out) - hi) * 2^11)
(scaled lo, the GEMM operand format) or lo = fp16(clamp(out) - hi) (unscaled lo, the attention operand format).  Head-major
outputs are [ceil(N / 64)][M][64]: column j of row i at [j // 64][i][j % 64].

Error bound of one launch on the wgmma path (k_gemm_ws), with S = sum_k |a_k b_k| over the launch's K_l columns:
  - operand split: each operand carries 22 significand bits (hi + lo * 2^-11) and the dropped lo * lo product is 2^-22 relative,
    so a product is off by a few 2^-22 of |a_k b_k|:                                             16 * 2^-22 * S
  - accumulation: the tensor core's fp32 accumulator truncates instead of rounding; one truncation (< 2^-23 relative of a
    partial sum <= S) per k16 MMA:                                                              (K_l / 16) * 2^-23 * S
    This assumes one truncation per MMA; it is consistent with the -4e-5 retrieval.cu records at K = 4096 .. 8448 but has not
    been checked on its own.
  - combining the two accumulators, fmaf(acc1, 2^-11, acc0):                                     2^-23 * S
  - each fp32 epilogue operation rounds once, 2^-23 relative of its result: + bias (|acc + bias|), * scale (|y|), + resid
    (|act(y)| + |resid|).  The GEMM terms are multiplied by |scale|.
  - GELU: its slope is below 1.13 in magnitude, so the error of y grows by at most 1.13; erff and its multiply chain add
    2^-20 |GELU(y)| + 2^-23 |y|.
On the SIMT path (k_gemm_nt, one fmaf per k in fp32) the GEMM terms are K_l * 2^-23 * S instead; the epilogue terms are the same.
K walked in chunks (one launch per chunk, each adding the previous output as its residual) adds the bounds of its launches:
an error in the residual passes through the add unchanged."""
from __future__ import annotations

import numpy as np
import torch

H_MAX = 65504.0
GELU_SLOPE = 1.13  # max |GELU'(x)| = 1.1289 (at x = 1.4142 ...)


def linear64(a1, b, *, a2=None, bias=None, scale=1.0, relu=False, gelu=False, resid=None) -> np.ndarray:
    """act(([a1 | a2] b^T + bias) * scale) + resid in float64."""
    a = np.asarray(a1, np.float64)
    if a2 is not None:
        a = np.concatenate([a, np.asarray(a2, np.float64)], 1)
    y = a @ np.asarray(b, np.float64).T
    if bias is not None:
        y = y + np.asarray(bias, np.float64)[: y.shape[1]]
    y = y * float(scale)
    if relu:
        y = np.maximum(y, 0.0)
    if gelu:
        y = gelu64(y)
    if resid is not None:
        y = y + np.asarray(resid, np.float64)
    return y


def gelu64(x) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1.0 + torch.erf(torch.from_numpy(x / np.sqrt(2.0))).numpy())


def split_planes(x, unscaled: bool = False):
    """fp32 values -> (hi, lo) fp16 bit patterns (uint16), as the kernels' epilogues write them.  numpy's float16 cast rounds
    to nearest even, like __float2half_rn; the differences below are exact in float32."""
    x = np.clip(np.asarray(x, np.float32), np.float32(-H_MAX), np.float32(H_MAX))
    hi = x.astype(np.float16)
    d = x - hi.astype(np.float32)
    lo = (d if unscaled else d * np.float32(2048.0)).astype(np.float16)
    return hi.view(np.uint16), lo.view(np.uint16)


def join_planes(hi, lo, unscaled: bool = False) -> np.ndarray:
    """(hi, lo) bit patterns -> the float64 value they stand for."""
    h = np.asarray(hi, np.uint16).view(np.float16).astype(np.float64)
    l = np.asarray(lo, np.uint16).view(np.float16).astype(np.float64)
    return h + (l if unscaled else l * 2.0 ** -11)


def head_major_elems(m: int, n: int) -> int:
    """Elements of a head-major [ceil(n / 64)][m][64] buffer."""
    return -(-n // 64) * m * 64


def to_head_major(x, fill=0) -> np.ndarray:
    """[m][n] -> [ceil(n / 64)][m][64]; the columns past n of the last head hold `fill`."""
    x = np.asarray(x)
    m, n = x.shape
    heads = -(-n // 64)
    out = np.full((m, heads * 64), fill, x.dtype)
    out[:, :n] = x
    return np.ascontiguousarray(out.reshape(m, heads, 64).transpose(1, 0, 2))


def from_head_major(h, n: int) -> np.ndarray:
    """[ceil(n / 64)][m][64] (or its flat buffer with m given by the size) -> [m][n]."""
    h = np.asarray(h)
    heads = -(-n // 64)
    h = h.reshape(heads, -1, 64)
    return np.ascontiguousarray(h.transpose(1, 0, 2).reshape(h.shape[1], heads * 64)[:, :n])


def launch_bound(a1, b, *, a2=None, bias=None, scale=1.0, relu=False, gelu=False, resid=None, path=1) -> np.ndarray:
    """Bound on |kernel - linear64| of ONE launch (see the module docstring); path 1 = wgmma, 0 = SIMT."""
    a = np.abs(np.asarray(a1, np.float64))
    if a2 is not None:
        a = np.concatenate([a, np.abs(np.asarray(a2, np.float64))], 1)
    k = a.shape[1]
    s = a @ np.abs(np.asarray(b, np.float64)).T
    gemm = (16 * 2.0 ** -22 + (k / 16) * 2.0 ** -23 + 2.0 ** -23) * s if path == 1 else k * 2.0 ** -23 * s
    t = linear64(a1, b, a2=a2, bias=bias)
    y = t * float(scale)
    e = abs(float(scale)) * (gemm + 2.0 ** -23 * np.abs(t)) + 2.0 ** -23 * np.abs(y)
    if relu:
        y = np.maximum(y, 0.0)
    if gelu:
        g = gelu64(y)
        e = GELU_SLOPE * e + 2.0 ** -20 * np.abs(g) + 2.0 ** -23 * np.abs(y)
        y = g
    if resid is not None:
        e = e + 2.0 ** -23 * (np.abs(y) + np.abs(np.asarray(resid, np.float64)))
    return e


def chunked_bound(a, b, kc: int, *, bias=None, resid=None, path=1) -> np.ndarray:
    """Bound of K walked in chunks of kc columns, chunk c > 0 adding the output of chunk c - 1 as its residual and the bias
    going with the first chunk (megaloc.cu, netvlad.cu, retrieval.cu); `resid`: a residual the first chunk adds."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    total, partial = 0.0, None if resid is None else np.asarray(resid, np.float64)
    for c in range(0, a.shape[1], kc):
        ac, bc = a[:, c:c + kc], b[:, c:c + kc]
        total = total + launch_bound(ac, bc, bias=bias if c == 0 else None, resid=partial, path=path)
        y = linear64(ac, bc, bias=bias if c == 0 else None)
        partial = y if partial is None else partial + y
    return total
