"""CPU: oracle/linear_ref.py, the fp64 restatement of the shared linear that tests/test_gemm_ws_gpu.py checks the kernels against.

- linear64 equals torch float64 (F.linear on torch.cat, exact GELU) in every epilogue mode.
- split_planes reconstructs x to 2^-22 relative across fp16's normal range, saturates at +-65504 with lo = 0, and gives
  hand-computed bits (fp16 subnormals included).
- The head-major helpers round-trip."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import linear_ref as lr


@pytest.mark.parametrize("relu,gelu", [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize("with_a2", [False, True])
def test_linear64_matches_torch(relu, gelu, with_a2):
    rng = np.random.default_rng(3 + 2 * relu + 4 * gelu + with_a2)
    a1 = rng.standard_normal((37, 48))
    a2 = rng.standard_normal((37, 16)) if with_a2 else None
    b = rng.standard_normal((29, 64 if with_a2 else 48))
    bias, resid = rng.standard_normal(29), rng.standard_normal((37, 29))
    got = lr.linear64(a1, b, a2=a2, bias=bias, scale=0.25, relu=relu, gelu=gelu, resid=resid)
    x = torch.from_numpy(a1) if a2 is None else torch.cat([torch.from_numpy(a1), torch.from_numpy(a2)], -1)
    y = F.linear(x, torch.from_numpy(b), torch.from_numpy(bias)) * 0.25
    if relu:
        y = F.relu(y)
    if gelu:
        y = F.gelu(y, approximate="none")
    want = (y + torch.from_numpy(resid)).numpy()
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("unscaled", [False, True])
def test_split_planes_reconstruct_to_2_22(unscaled):
    rng = np.random.default_rng(5)
    mag = 2.0 ** rng.uniform(-14, np.log2(65504.0), 200000)  # fp16's normal range
    x = (mag * rng.choice([-1.0, 1.0], mag.size)).astype(np.float32)
    hi, lo = lr.split_planes(x, unscaled)
    x64 = x.astype(np.float64)
    err = np.abs(lr.join_planes(hi, lo, unscaled) - x64)
    if unscaled:  # lo = x - hi turns subnormal below |x| = 2^-2 (tc.cuh): there its absolute step 2^-24 rules
        assert (err <= np.maximum(2.0 ** -22 * np.abs(x64), 2.0 ** -25)).all()
        x64, err = x64[np.abs(x64) >= 0.25], err[np.abs(x64) >= 0.25]
    rel = err / np.abs(x64)
    assert rel.max() <= 2.0 ** -22, float(rel.max())


@pytest.mark.parametrize("unscaled", [False, True])
def test_split_planes_saturate(unscaled):
    x = np.array([65504.0, 65520.0, 1e6, 3.4e38, np.inf, -65504.0, -7e4, -np.inf], np.float32)
    hi, lo = lr.split_planes(x, unscaled)
    assert hi.tolist() == [0x7BFF] * 5 + [0xFBFF] * 3
    assert lo.tolist() == [0] * 8


def test_split_planes_hand_bits():
    # 1 + 2^-11 + 2^-20 lies just above the tie between 1 and 1 + 2^-10, so hi rounds up to 1 + 2^-10;
    # lo = x - hi = 2^-11 + 2^-20 - 2^-10 = -(2^-11 - 2^-20)
    x = np.float32(1.0 + 2.0 ** -11 + 2.0 ** -20)
    hi, lo = lr.split_planes(np.array([x]))
    assert hex(hi[0]) == hex(0x3C01)  # 1 + 2^-10
    want_lo = np.float16(-(2.0 ** -11 - 2.0 ** -20) * 2048.0).view(np.uint16)  # -(1 - 2^-9), exact in fp16
    assert lo[0] == want_lo == 0xBBFC
    hi_u, lo_u = lr.split_planes(np.array([x]), unscaled=True)
    assert hi_u[0] == 0x3C01
    # -(2^-11 - 2^-20) = -2^-12 (2 - 2^-8): fp16 exponent -12 (biased 3), mantissa 0x3FC
    assert lo_u[0] == 0x8FFC
    # an exact tie rounds to even: 1 + 2^-11 -> hi = 1.0, lo = 2^-11 (scaled: 1.0, unscaled: 0x1000)
    hi, lo = lr.split_planes(np.array([1.0 + 2.0 ** -11], np.float32))
    assert (hi[0], lo[0]) == (0x3C00, 0x3C00)
    hi, lo = lr.split_planes(np.array([1.0 + 2.0 ** -11], np.float32), unscaled=True)
    assert (hi[0], lo[0]) == (0x3C00, 0x1000)
    # fp16 subnormals: 2^-24 is the smallest (0x0001); 3 * 2^-25 is a tie between 0x0001 and 0x0002 -> 0x0002 (even), which
    # leaves -2^-25: scaled lo -2^-14 (0x8400, the smallest normal), unscaled lo a tie between -0 and -2^-24 -> -0 (0x8000)
    v = np.array([2.0 ** -24, 3 * 2.0 ** -25, -(2.0 ** -15)], np.float32)
    hi, lo = lr.split_planes(v)
    assert hi.tolist() == [0x0001, 0x0002, 0x8200]
    assert lo.tolist() == [0, 0x8400, 0]
    assert lr.split_planes(v, unscaled=True)[1].tolist() == [0, 0x8000, 0]
    # 2^-24 + 2^-26: hi = 2^-24 (0x0001), remainder 2^-26 * 2^11 = 2^-15 (subnormal 0x0200); unscaled 2^-26 underflows to 0
    v = np.array([2.0 ** -24 + 2.0 ** -26], np.float32)
    assert [int(t[0]) for t in lr.split_planes(v)] == [0x0001, 0x0200]
    assert [int(t[0]) for t in lr.split_planes(v, unscaled=True)] == [0x0001, 0x0000]


@pytest.mark.parametrize("m,n", [(1, 1), (5, 64), (7, 65), (130, 200), (3, 2304)])
def test_head_major_round_trip(m, n):
    x = np.arange(m * n, dtype=np.float32).reshape(m, n)
    h = lr.to_head_major(x, fill=np.nan)
    assert h.shape == (-(-n // 64), m, 64) and h.size == lr.head_major_elems(m, n)
    assert np.array_equal(lr.from_head_major(h, n), x)
    assert np.array_equal(lr.from_head_major(h.ravel(), n), x)
    j = n - 1
    assert h[j // 64, m - 1, j % 64] == x[m - 1, j]
    assert np.isnan(h[-1, :, n - 64 * (h.shape[0] - 1):]).all()


def test_chunked_bound_adds_launch_bounds():
    rng = np.random.default_rng(9)
    a, b = np.abs(rng.standard_normal((4, 256))), rng.standard_normal((3, 256))
    one = lr.launch_bound(a, b)
    two = lr.chunked_bound(a, b, 128)
    assert (two < one).all()  # fewer truncating MMAs per launch
    assert np.array_equal(lr.chunked_bound(a, b, 256), one)
