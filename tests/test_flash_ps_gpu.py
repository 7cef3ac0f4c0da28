"""GPU: the batched wgmma split-fp16 flash attention (k_flash_ps) at its edges, through b2_debug_attention_host, against fp64.

Shapes cover a last key tile with 64, 1 and 63 keys, one- and two-tile segments (Nk = 37, 65), a last query block of one
row, a launch with far more (item, key tile) units than SMs (every item cut into several stream-K segments and merged in
the kernel), items that fit one segment whole, 16 problems of different sizes in one launch, and 4 and 12 heads.  Scaled-up
queries make the row maximum grow by more than 2^8 across key tiles, so the lazy rescale of O fires.

Tolerance: q, k, v carry 22 significand bits (hi + unscaled lo) and the dropped lo * lo product is 2^-22 relative, so a
logit is off by a few 2^-22 of scale * sum_d |q_d k_d|; ex2.approx and the hi / lo split of P add about 2^-22 relative.
The bound allows 2^-16 of that logit sum plus 2^-18 relative, on (P |V| + |O|); a plain fp16 attention must exceed it.
The fp16 variant (hi planes only, fp16 P and output) is checked against the fp64 attention of fp16-rounded operands at
2^-9 of (P |V| + |O|).  Two runs of the same launch must agree bit for bit."""
import ctypes

import numpy as np
import pytest

from gtsfm_b200 import _lib

pytestmark = pytest.mark.gpu

_RNG16 = np.random.default_rng(16)

CASES = {
    "nk_mod0": ([300], [192], 4, 1.0),
    "nk_mod1": ([300], [193], 4, 1.0),
    "nk_mod63": ([300], [255], 4, 1.0),
    "one_tile": ([77], [37], 4, 1.0),
    "two_tiles": ([513], [65], 4, 1.0),
    "stream_k_merge": ([1000], [2048], 4, 4.0),
    "batch16": (list(_RNG16.integers(1, 700, 16)), list(_RNG16.integers(1, 400, 16)), 4, 2.0),
    "heads12_whole_items": ([2816], [128], 12, 1.0),
    "heads12_split": ([257, 1369], [1369, 257], 12, 1.0),
}


def _inputs(nq, nk, heads, qmul, seed):
    rng = np.random.default_rng(seed)
    q = [(qmul * rng.standard_normal((heads, n, 64))).astype(np.float32) for n in nq]
    k = [rng.standard_normal((heads, n, 64)).astype(np.float32) for n in nk]
    v = [rng.standard_normal((heads, n, 64)).astype(np.float32) for n in nk]
    return q, k, v


def _run(ctx, q, k, v, scale, single):
    heads = q[0].shape[0]
    nq = np.array([x.shape[1] for x in q], np.int32)
    nk = np.array([x.shape[1] for x in k], np.int32)
    qc, kc, vc = (np.concatenate([x.ravel() for x in a]) for a in (q, k, v))
    o = np.full(int(nq.sum()) * 64 * heads, np.nan, np.float32)
    ip = ctypes.POINTER(ctypes.c_int)
    rc = ctx.lib.b2_debug_attention_host(ctx.handle, len(q), nq.ctypes.data_as(ip), nk.ctypes.data_as(ip), heads, scale,
                                         int(single), _lib.ptr(qc), _lib.ptr(kc), _lib.ptr(vc), _lib.ptr(o))
    ctx.check(rc, "b2_debug_attention_host")
    out, off = [], 0
    for n in nq:
        out.append(o[off:off + n * 64 * heads].reshape(n, heads * 64))
        off += n * 64 * heads
    return out


def _reference(q, k, v, scale):
    """fp64 softmax(scale q k^T) v as [nq][64 heads], plus P |V| and the largest scale * sum_d |q_d k_d| of each row."""
    q, k, v = (x.astype(np.float64) for x in (q, k, v))
    s = scale * np.einsum("hqd,hkd->hqk", q, k)
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    o = np.einsum("hqk,hkd->hqd", p, v)
    pav = np.einsum("hqk,hkd->hqd", p, np.abs(v))
    lsum = (scale * np.einsum("hqd,hkd->hqk", np.abs(q), np.abs(k))).max(-1, keepdims=True)
    to_rows = lambda x: x.transpose(1, 0, 2).reshape(x.shape[1], -1)  # noqa: E731
    return to_rows(o), to_rows(pav), to_rows(np.broadcast_to(lsum, o.shape))


@pytest.mark.parametrize("case", list(CASES))
def test_flash_ps_matches_fp64(b200_ctx, case):
    nq, nk, heads, qmul = CASES[case]
    scale = 0.125
    q, k, v = _inputs(nq, nk, heads, qmul, seed=sum(nq) * 7 + sum(nk))
    got = _run(b200_ctx, q, k, v, scale, single=False)
    again = _run(b200_ctx, q, k, v, scale, single=False)
    told = False
    for z in range(len(q)):
        assert np.array_equal(got[z], again[z]), f"problem {z}: two runs of the same launch differ"
        assert np.isfinite(got[z]).all(), f"problem {z}: non-finite output"
        want, pav, lsum = _reference(q[z], k[z], v[z], scale)
        bound = (2.0 ** -16 * lsum + 2.0 ** -18) * (pav + np.abs(want))
        err = np.abs(got[z] - want)
        assert (err <= bound).all(), (case, z, float(err.max()), float((err / bound).max()))
        f16 = [x.astype(np.float16) for x in (q[z], k[z], v[z])]
        told = told or (np.abs(_reference(*f16, scale)[0] - want) > bound).any()
    assert told, "the bound does not tell split-fp16 from plain fp16 attention at this shape"


@pytest.mark.parametrize("case", ["nk_mod63", "two_tiles", "stream_k_merge", "batch16", "heads12_split"])
def test_flash_ps_fp16_variant(b200_ctx, case):
    nq, nk, heads, qmul = CASES[case]
    scale = 0.125
    q, k, v = _inputs(nq, nk, heads, qmul, seed=sum(nq) * 7 + sum(nk))
    got = _run(b200_ctx, q, k, v, scale, single=True)
    again = _run(b200_ctx, q, k, v, scale, single=True)
    for z in range(len(q)):
        assert np.array_equal(got[z], again[z]), f"problem {z}: two runs of the same launch differ"
        assert np.array_equal(got[z], got[z].astype(np.float16).astype(np.float32)), "output is not fp16"
        want, pav, _ = _reference(*(x.astype(np.float16) for x in (q[z], k[z], v[z])), scale)
        err = np.abs(got[z] - want)
        bound = 2.0 ** -9 * (pav + np.abs(want))
        assert (err <= bound).all(), (case, z, float(err.max()), float((err / bound).max()))
