"""CPU: oracle/conv_ref.py, the fp64 restatement of the shared 3x3 convolution layer that tests/test_conv_ps_gpu.py checks the
kernels against.

- conv64 (shifted taps and an einsum in numpy, pool before the bias) equals torch float64 conv2d + max_pool2d + relu, at odd
  sizes under the pool, sizes below a tile and both dilations.
- torch's fp32 convolution stays inside the wgmma and the SIMT bounds.
- The bound is sharp enough to tell split-fp16 from plain fp16: the fp64 convolution of fp16-rounded operands exceeds it
  somewhere at every call-site case of the GPU test, on that case's data.
- plane_error bounds the split's own rounding across fp16's range, subnormals included."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import conv_ref as cr
from test_conv_ps_gpu import CASES, data


def _torch(x, w, b, dilation, pool, relu, dtype=torch.float64):
    t = F.conv2d(torch.from_numpy(x).to(dtype).permute(2, 0, 1)[None], torch.from_numpy(w).to(dtype), torch.from_numpy(b).to(dtype),
                 padding=dilation, dilation=dilation)
    if pool:
        t = F.max_pool2d(t, 2, 2)
    if relu:
        t = F.relu(t)
    return t[0].permute(1, 2, 0).numpy()


def _layer(rng, H, W, cin, cout, signed=False):
    x = rng.standard_normal((H, W, cin))
    x = (x if signed else np.maximum(x, 0)).astype(np.float32)
    w = (rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    return x, w, rng.standard_normal(cout).astype(np.float32)


SHAPES = [(17, 9, 64, 64), (1, 1, 64, 128), (2, 2, 128, 64), (3, 5, 64, 64), (1, 23, 64, 64), (21, 1, 64, 64), (40, 26, 128, 192)]


@pytest.mark.parametrize("dilation", [1, 2])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("shape,pool", [(s, p) for s in SHAPES for p in (False, True) if not p or min(s[:2]) >= 2],
                         ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else ("pool" if v else "nopool"))
def test_conv64_matches_torch(shape, pool, relu, dilation):
    H, W, cin, cout = shape
    rng = np.random.default_rng(H * 100 + W + cin + 7 * dilation)
    x, w, b = _layer(rng, H, W, cin, cout, signed=True)
    got = cr.conv64(x, w, b, dilation=dilation, pool=pool, relu=relu)
    want = _torch(x, w, b, dilation, pool, relu)
    assert got.shape == want.shape == ((H // 2, W // 2, cout) if pool else (H, W, cout))
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("dilation", [1, 2])
@pytest.mark.parametrize("pool", [False, True])
def test_torch_fp32_is_inside_both_bounds(pool, dilation):
    rng = np.random.default_rng(5 + pool + 2 * dilation)
    x, w, b = _layer(rng, 24, 20, 256, 128)
    want = cr.conv64(x, w, b, dilation=dilation, pool=pool)
    err = np.abs(_torch(x, w, b, dilation, pool, True, torch.float32) - want)
    for path in (1, 0):
        bound = cr.bound(x, w, b, dilation=dilation, pool=pool, path=path)
        r = float((err / bound).max())
        print(f"torch fp32 / bound (path {path}): {r:.4f}")
        assert r < 0.1


@pytest.mark.parametrize("name", list(CASES))
def test_fp16_operands_exceed_the_wgmma_bound(name):
    """A kernel that lost the lo planes (a plain fp16 convolution) would fail the GPU case."""
    _, _, _, _, dil, pool, relu, _ = CASES[name]
    x, w, b = data(name)
    want = cr.conv64(x, w, b, dilation=dil, pool=pool, relu=relu)
    hi_only = cr.conv64(x.astype(np.float16), w.astype(np.float16), b, dilation=dil, pool=pool, relu=relu)
    r = float((np.abs(hi_only - want) / cr.bound(x, w, b, dilation=dil, pool=pool)).max())
    print(f"fp16 operands err/bound {name}: {r:.2f}")
    assert r > 1.0


def test_plane_error_bounds_the_split():
    rng = np.random.default_rng(3)
    mag = 2.0 ** rng.uniform(-40, np.log2(65504.0), 400000)  # fp16's range and far below it
    y = (mag * rng.choice([-1.0, 1.0], mag.size)).astype(np.float32)
    err = np.abs(cr.join_planes(*cr.split_planes(y)) - y.astype(np.float64))
    assert (err <= cr.plane_error(y)).all()
    assert (err > 0.25 * cr.plane_error(y)).any()  # and it is not loose by orders of magnitude


def test_maxpool_drops_the_odd_row_and_column():
    y = np.arange(5 * 7 * 2, dtype=np.float64).reshape(5, 7, 2)
    p = cr.maxpool(y)
    assert p.shape == (2, 3, 2)
    assert np.array_equal(p[..., 0], y[1:4:2, 1:6:2, 0])
