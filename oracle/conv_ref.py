"""fp64 restatement of the shared 3x3 convolution layer (k_conv_ps in gtsfm_b200/csrc/conv_ps.cuh, and the exact-fp32 SIMT
k_conv3x3 beside it) and the error bound its kernels meet.

One layer computes, per output element (NHWC input [H][W][Cin], OIHW weight [Cout][Cin][3][3], padding = dilation d),

    y = act(maxpool(conv(x, w)) + bias),    act = ReLU or identity,    maxpool = optional 2x2/2 (floor, like MaxPool2d(2, 2)),

the pool taken before the bias as the kernels take it (max commutes with adding a per-channel constant), and may write y as
fp32 and / or as split fp16 planes (linear_ref.split_planes: hi = fp16(clamp(y)), lo = fp16((clamp(y) - hi) * 2^11)).

Error bound of the wgmma path, derived like linear_ref.launch_bound with the same terms.  With S = conv(|x|, |w|) over the
K = 9 Cin products of an output pixel:
  - operand split (22 significand bits per operand, the lo * lo product dropped):   16 * 2^-22 * S
  - one truncation of the fp32 accumulator per k16 MMA:                            (K / 16) * 2^-23 * S
  - the fmaf(acc_hl + acc_lh, 2^-11, acc_hh) combine:                               2^-23 * S
On the SIMT path (one fmaf per product) the three are K * 2^-23 * S instead.  With pool the kernel's value is the maximum of
four computed sums, and max is 1-Lipschitz in each argument, so the pooled error is at most the largest of the four pixels'
bounds.  The bias add then rounds once, 2^-23 |maxpool(conv) + bias|.  ReLU is non-expansive."""
from __future__ import annotations

import numpy as np

from oracle.linear_ref import join_planes, split_planes  # noqa: F401  (the plane format of the layer's outputs)

U = 2.0 ** -23


def _taps(x, dilation: int) -> np.ndarray:
    """x [H][W][C] -> [9][H][W][C]: tap t = 3 dy + dx reads x[i + (dy - 1) d][j + (dx - 1) d], zero outside the image."""
    H, W, C = x.shape
    d = dilation
    p = np.zeros((H + 2 * d, W + 2 * d, C), x.dtype)
    p[d:d + H, d:d + W] = x
    return np.stack([p[dy * d:dy * d + H, dx * d:dx * d + W] for dy in range(3) for dx in range(3)])


def _conv(x, w, dilation: int) -> np.ndarray:
    """sum over taps and input channels, float64, no bias: [H][W][Cout]."""
    t = _taps(np.asarray(x, np.float64), dilation)                    # [9][H][W][Cin]
    wt = np.asarray(w, np.float64).reshape(w.shape[0], w.shape[1], 9)  # [Cout][Cin][9]
    return np.einsum("thwc,oct->hwo", t, wt, optimize=True)


def maxpool(y) -> np.ndarray:
    """2x2/2 max-pool of [H][W][C], floor: the last row / column of an odd size is dropped."""
    H, W, C = y.shape
    y = y[:H // 2 * 2, :W // 2 * 2]
    return y.reshape(H // 2, 2, W // 2, 2, C).max(axis=(1, 3))


def conv64(x, w, bias, *, dilation: int = 1, pool: bool = False, relu: bool = True) -> np.ndarray:
    """act(maxpool(conv(x, w)) + bias) in float64, NHWC."""
    y = _conv(x, w, dilation)
    if pool:
        y = maxpool(y)
    y = y + np.asarray(bias, np.float64)
    return np.maximum(y, 0.0) if relu else y


def bound(x, w, bias, *, dilation: int = 1, pool: bool = False, path: int = 1) -> np.ndarray:
    """Bound on |kernel - conv64| per output element (see the module docstring); path 1 = wgmma, 0 = SIMT."""
    k = 9 * w.shape[1]
    s = _conv(np.abs(x), np.abs(w), dilation)
    gemm = (16 * 2.0 ** -22 + (k / 16) * U + U) * s if path == 1 else k * U * s
    y = _conv(x, w, dilation)
    if pool:
        gemm, y = maxpool(gemm), maxpool(y)
    return gemm + U * np.abs(y + np.asarray(bias, np.float64))


def plane_error(y) -> np.ndarray:
    """Bound on |join_planes(split_planes(y)) - y| for |y| <= 65504: hi rounds to nearest, so |y - hi| <= 2^-11 |y| is exact
    in fp32; lo = fp16((y - hi) * 2^11) rounds that once more, 2^-11 relative, or 2^-25 absolute where it is subnormal
    (2^-36 in units of y)."""
    return 2.0 ** -22 * np.abs(np.asarray(y, np.float64)) + 2.0 ** -36
