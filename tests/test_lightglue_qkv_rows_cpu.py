"""CPU: the row order of LightGlue's self-attention QKV projection on the device (b2_lightglue_qkv_rows).

The device copy of each self block's Wqkv / bqkv is the checkpoint's rows regrouped as [q | k | v], each head-major, so the
projection's epilogue sees both values of a rotary pair.  Applying the regrouped weight and undoing the regrouping on the
output must give the checkpoint's projection exactly, and the regrouped columns must be the q / k / v features the
reference unflattens (lightglue.py:166-167: unflatten(-1, (heads, -1, 3)))."""
import numpy as np

from gtsfm_b200 import _lib, build


def _rows():
    build.build()
    lib = _lib.load()
    rows = np.empty(768, np.int32)
    assert lib.b2_lightglue_qkv_rows(_lib.ptr(rows)) == 0
    return rows


def test_qkv_rows_is_a_permutation_that_round_trips():
    rows = _rows()
    assert np.array_equal(np.sort(rows), np.arange(768))
    rng = np.random.default_rng(3)  # small integers: every sum is exact, whatever order the BLAS kernel adds in
    w = rng.integers(-8, 9, (768, 256)).astype(np.float32)
    b = rng.integers(-8, 9, 768).astype(np.float32)
    x = rng.integers(-8, 9, (37, 256)).astype(np.float32)
    want = x @ w.T + b
    got_permuted = x @ w[rows].T + b[rows]
    undone = np.empty_like(got_permuted)
    undone[:, rows] = got_permuted
    assert np.array_equal(undone.view(np.uint32), want.view(np.uint32))


def test_qkv_rows_group_q_k_v_head_major():
    rows = _rows()
    # the reference's view: feature f = (h * 64 + j) * 3 + t, t = 0 / 1 / 2 for q / k / v
    qkv = np.arange(768).reshape(4, 64, 3)
    for t in range(3):
        assert np.array_equal(rows[256 * t:256 * (t + 1)], qkv[:, :, t].reshape(-1))
