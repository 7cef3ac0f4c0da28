"""GPU: LightGlue's layer kernels one at a time against NumPy fp64, and its per-layer state (b2_set_option
"lightglue_trace") against the oracle's fp64 replay, layer by layer and side by side, on the single-pair and the lock-step
batched paths.

Kernel level: integer outputs (keep maps, counters, index maps, match rows) are exact.  Float outputs are held to a bound
argued at each test from the fp32 operation count of the kernel (eps = 2^-24, the unit roundoff of fp32).

Network level: the device's x after every layer, and its token confidence / matchability, may differ from the fp64
replay by at most BOUND_FACTOR times the fp32 oracle's own distance from that replay at the same layer and side (the
spread a correct fp32 implementation shows).  Early-exit layer, unconfident counts, keep sets and ind0 / ind1 must be
equal.  Each case's seed is chosen so that every fp64 confidence and matchability lies more than MARGIN from its threshold
(asserted), so the decisions are well defined.  Measured on an H100 SXM (80 GB HBM3, 700 W limit), the largest ratio of
device error to fp32-oracle spread over every case and layer is listed at BOUND_FACTOR.
"""
import ctypes as C

import numpy as np
import pytest
from scipy.special import erf

from gtsfm_b200 import _lib
from gtsfm_b200 import synthetic as syn
from gtsfm_b200.matcher import LightGlueEngine
from oracle import lightglue_ref as ref

EPS = 2.0 ** -24
MARGIN = 1e-5
# Largest measured ratio of device error to fp32-oracle spread, over every case below (H100 SXM 80 GB, 700 W): x 3.7 at
# layer 0 rising to 6.5 at layer 8 (the bench-size pair); conf 12.1 (layer 7 of a 1 x 700 pair, where one rounding of the
# largest value floors the spread), 2-7.8 elsewhere; mat 3.2.  The SIMT path: 2.6.  Bound: 4x the largest.
BOUND_FACTOR = 50.0
# fp16_attention against the fp16-emulating replay: 9.0e-6 measured (conf), bound 4x
FP16_ATOL = 4e-5
LO_SCALE = 2.0 ** -11  # split planes: value = hi + lo * 2^-11


def _i32(a):
    return np.ascontiguousarray(a, np.int32)


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _n(ns):
    return _i32(ns), len(ns)


def _check(ctx, rc, what):
    ctx.check(rc, what)


# ---------------------------------------------------------------------------------------------------------------------
# kernel level
# ---------------------------------------------------------------------------------------------------------------------

PRUNE_NS = [1, 31, 1023, 1024, 1025, 2049, 5000]


def _prune(ctx, ns, conf, mat, thr, keep_thr):
    n, np_ = _n(ns)
    src = np.full(int(n.sum()), -5, np.int32)
    cnt = np.full(4 * ((np_ + 1) // 2), -7, np.int32)
    _check(ctx, ctx.lib.b2_debug_lightglue_prune_host(ctx.handle, np_, _lib.ptr(n), _lib.ptr(conf), _lib.ptr(mat), thr, keep_thr,
                                                      _lib.ptr(src), _lib.ptr(cnt)), "prune")
    return src, cnt.reshape(-1, 4)


@pytest.mark.gpu
def test_prune_plan_counts_and_keep_maps(b200_ctx):
    """Every size around the 1024-row steps (the carry between steps) in one launch, with an empty entry; conf exactly thr
    (not unconfident: `<`; kept: `<=`), mat exactly keep_thr (not kept on its own), NaN conf (neither), all / none kept."""
    rng = np.random.default_rng(0)
    thr, keep_thr = np.float32(0.85), np.float32(1.0 - 0.99)
    ns = PRUNE_NS + [0]
    conf, mat = [], []
    for k, n in enumerate(ns):
        c = rng.uniform(0.6, 1.0, n).astype(np.float32)
        m = rng.uniform(0.0, 0.03, n).astype(np.float32)
        sel = rng.random(n)
        c[sel < 0.05] = thr
        m[(sel > 0.1) & (sel < 0.15)] = keep_thr
        c[(sel > 0.2) & (sel < 0.22)] = np.nan
        if k == 5:  # everything kept
            m[:] = 0.5
        if k == 6:  # nothing kept
            m[:], c[:] = 0.0, 0.95
        conf.append(c), mat.append(m)
    conf, mat = _f32(np.concatenate(conf)), _f32(np.concatenate(mat))
    src, cnt = _prune(b200_ctx, ns, conf, mat, thr, keep_thr)
    o = 0
    for k, n in enumerate(ns):
        c, m = conf[o: o + n], mat[o: o + n]
        keep = np.nonzero((m > keep_thr) | (c <= thr))[0]
        pair, side = divmod(k, 2)
        if n == 0:
            assert cnt[pair, side] == -7 and cnt[pair, 2 + side] == -7, "an empty entry writes no counters"
        else:
            assert cnt[pair, side] == int(np.sum(c < thr)), (n, cnt[pair])
            assert cnt[pair, 2 + side] == len(keep), (n, cnt[pair])
            assert np.array_equal(src[o: o + len(keep)], keep), n
            assert np.all(src[o + len(keep): o + n] == -5), "rows past the kept count are not written"
        o += n
    assert cnt[2, 3] == 2049 and cnt[3, 2] == 0  # the all-kept (entry 5) and none-kept (entry 6) cases


@pytest.mark.gpu
def test_filter_mutual_threshold_and_compaction(b200_ctx):
    """k_lg_filter alone at every size around its 1024-row steps: mutual check, exp(best0) > th (a score exactly at th is
    out), ind0 / ind1 mapping, ordered compaction.  A row without an arg-max (best0 = -inf, index 0 as the arg-max kernels
    write it) never matches, even when mutual under th < 0.  Scores: one expf of an fp32 input, within 2 ulp of fp64."""
    rng = np.random.default_rng(1)
    for m in PRUNE_NS:
        n = m + 3
        a0 = _i32(rng.integers(0, n, m))
        a1 = _i32(rng.integers(0, m, n))
        mut = rng.permutation(m)[: m // 2]
        a1[a0[mut]] = mut  # about half the rows mutual
        best0 = _f32(np.log(rng.uniform(0.05, 1.0, m)))
        best0[rng.random(m) < 0.05] = 0.0  # exp = 1.0 exactly: at th = 1.0, not above it
        best0[rng.random(m) < 0.05] = 0.25  # above 1
        best0[0], a0[0], a1[0] = -np.inf, 0, 0  # row 0: no arg-max, mutual with column 0
        ind0, ind1 = _i32(rng.permutation(10 * m)[:m]), _i32(rng.permutation(10 * n)[:n])
        for th in (np.float32(0.1), np.float32(1.0), np.float32(-1.0)):
            out = np.full((m + 1, 2), -9, np.int64)
            outs = np.full(m + 1, -9, np.float32)
            k = C.c_int(-1)
            _check(b200_ctx, b200_ctx.lib.b2_debug_lightglue_filter_host(
                b200_ctx.handle, m, n, _lib.ptr(best0), _lib.ptr(a0), _lib.ptr(a1), float(th), _lib.ptr(ind0), _lib.ptr(ind1),
                _lib.ptr(out), _lib.ptr(outs), C.byref(k)), "filter")
            e = np.exp(best0.astype(np.float64))
            valid = (a1[a0] == np.arange(m)) & np.isfinite(best0) & (e > th)
            rows = np.nonzero(valid)[0]
            assert k.value == len(rows), (m, th)
            assert np.array_equal(out[: len(rows)], np.stack([ind0[rows], ind1[a0[rows]]], 1)), (m, th)
            assert np.all(out[len(rows):] == -9) and np.all(outs[len(rows):] == -9)
            np.testing.assert_allclose(outs[: len(rows)], e[rows], rtol=6 * EPS, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("path", [1, 2])
def test_argmax_of_nan_rows_stays_in_range(b200_ctx, path):
    """A row whose scores are all NaN (a NaN descriptor reaches the assignment: no entry point rejects non-finite input)
    has no arg-max.  Both the persistent (1) and the multi-launch (2) kernels must write index 0 and best0 = -inf for it,
    never the 0x7fffffff sentinel the filter would then use as a column index.  Arg-max kernels alone: no filter runs."""
    rng = np.random.default_rng(2)
    for M, N in ((7, 40), (300, 1029)):
        sim = _f32(rng.standard_normal((M, N)))
        sim[3] = np.nan
        sim[:, 5] = np.nan
        z0, z1 = _f32(rng.standard_normal(M)), _f32(rng.standard_normal(N))
        for s in (sim, _f32(np.full((M, N), np.nan))):
            best0 = np.zeros(M, np.float32)
            arg0, arg1 = np.full(M, -3, np.int32), np.full(N, -3, np.int32)
            ran = C.c_int(0)
            _check(b200_ctx, b200_ctx.lib.b2_debug_lightglue_argmax_host(
                b200_ctx.handle, path, _lib.ptr(s), M, N, _lib.ptr(z0), _lib.ptr(z1), _lib.ptr(best0), _lib.ptr(arg0), _lib.ptr(arg1),
                C.byref(ran)), "argmax")
            assert ran.value == path
            assert np.all((arg0 >= 0) & (arg0 < N)) and np.all((arg1 >= 0) & (arg1 < M)), (arg0.max(), arg1.max())
            assert arg0[3] == 0 and best0[3] == -np.inf
            if np.isnan(s).all():
                assert np.all(arg0 == 0) and np.all(arg1 == 0) and np.all(best0 == -np.inf)


def _posenc64(kp, wr):
    kp = kp.astype(np.float64)
    size = 1.0 + kp.max(0) - kp.min(0)
    x = (kp - size / 2) / (size.max() / 2)
    proj = x @ wr.astype(np.float64).T
    return np.cos(proj), np.sin(proj), np.abs(x) @ np.abs(wr.astype(np.float64)).T


@pytest.mark.gpu
def test_posenc_table(b200_ctx):
    """k_lg_posenc: bbox normalisation + rotary table, entries of different n in one launch (and an empty one), identical
    keypoints (a bbox of size 1), keypoints on one line.  Bound: the projection x w0 + y w1 carries at most 6 fp32
    roundings (size, shift, scale, two quotients, the dot) each relative to |x w0| + |y w1| =: S, and cosf / sinf add
    2 ulp: |err| <= 8 eps (S + 1)."""
    rng = np.random.default_rng(3)
    wr = _f32(rng.standard_normal((32, 2)) * 1.5)
    kps = [rng.uniform(0, [640, 480], (1, 2)), rng.uniform(0, [640, 480], (32, 2)), rng.uniform(0, [640, 480], (1025, 2)),
           np.zeros((0, 2)), rng.uniform(0, [640, 480], (5000, 2)), np.tile([[123.25, 77.5]], (40, 1)),
           np.stack([np.full(300, 17.0), rng.uniform(0, 480, 300)], 1)]
    kps = [_f32(k) for k in kps]
    n, np_ = _n([len(k) for k in kps])
    tot = int(n.sum())
    kp = _f32(np.concatenate(kps))
    cs, sn = np.full((tot, 32), 7, np.float32), np.full((tot, 32), 7, np.float32)
    ind = np.full(tot, -1, np.int32)
    _check(b200_ctx, b200_ctx.lib.b2_debug_lightglue_posenc_host(b200_ctx.handle, np_, _lib.ptr(n), _lib.ptr(kp), _lib.ptr(wr),
                                                                 _lib.ptr(cs), _lib.ptr(sn), _lib.ptr(ind)), "posenc")
    o = 0
    for k in kps:
        if len(k):
            c64, s64, S = _posenc64(k, wr)
            tol = 8 * EPS * (S + 1)
            assert np.all(np.abs(cs[o: o + len(k)] - c64) <= tol), np.max(np.abs(cs[o: o + len(k)] - c64) / tol)
            assert np.all(np.abs(sn[o: o + len(k)] - s64) <= tol), np.max(np.abs(sn[o: o + len(k)] - s64) / tol)
            assert np.array_equal(ind[o: o + len(k)], np.arange(len(k)))
        o += len(k)


def _ln_gelu64(h, g, b):
    h = h.astype(np.float64)
    mu = h.mean(1, keepdims=True)
    var = ((h - mu) ** 2).mean(1, keepdims=True)
    sd = np.sqrt(var + 1e-5)
    e = (h - mu) / sd * g + b
    return 0.5 * e * (1 + erf(e / np.sqrt(2))), np.abs(h).max(1, keepdims=True) / sd


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [False, True])
def test_ln_gelu(b200_ctx, planes):
    """k_lg_ln_gelu in place and into split planes: rows in {1, 7, 8, 9, 1025} (one warp per row, 8 rows per block) and an
    empty entry in one launch, a constant row (zero variance: only eps keeps it finite) and a row of mean 1e4 with unit
    spread (cancellation).  Bound: mean and variance are warp sums of 512 terms (16 sequential + 5 tree roundings), so
    the centred value is off by <= 32 eps max|h| / sd, scaled by |g|; the affine map, erff and the products add a few
    ulp of the result: |err| <= 32 eps (max|g| max|h| / sd + |y| + 1), plus 2^-22 |y| for the planes' split."""
    rng = np.random.default_rng(4)
    g = _f32(1.0 + 0.1 * rng.standard_normal(512))
    b = _f32(0.05 * rng.standard_normal(512))
    rows = [1, 7, 8, 0, 9, 1025]
    hs = [_f32(rng.standard_normal((r, 512)) * 2) for r in rows]
    hs[2][3] = 0.1  # constant row (0.1 is inexact in fp32: the mean is not exactly the value)
    hs[2][4] = 3.0
    hs[4][0] = _f32(1e4 + rng.standard_normal(512))
    n, np_ = _n(rows)
    h = _f32(np.concatenate(hs))
    h_in = h.copy()
    hi = np.zeros(h.shape, np.float16) if planes else None
    lo = np.zeros(h.shape, np.float16) if planes else None
    _check(b200_ctx, b200_ctx.lib.b2_debug_lightglue_ln_gelu_host(b200_ctx.handle, np_, _lib.ptr(n), _lib.ptr(g), _lib.ptr(b), _lib.ptr(h),
                                                                  _lib.ptr(hi), _lib.ptr(lo)), "ln_gelu")
    y64, ratio = _ln_gelu64(h_in, g, b)
    if planes:
        assert np.array_equal(h, h_in), "the split-plane variant must leave h alone"
        y = hi.astype(np.float64) + lo.astype(np.float64) * LO_SCALE
    else:
        y = h.astype(np.float64)
    tol = 32 * EPS * (np.abs(g).max() * ratio + np.abs(y64) + 1) + (2.0 ** -22 * np.abs(y64) if planes else 0)
    err = np.abs(y - y64)
    assert np.all(err <= tol), (np.unravel_index(np.argmax(err / tol), err.shape), np.max(err / tol))


@pytest.mark.gpu
def test_rowheads(b200_ctx):
    """k_lg_rowheads: head 1 on every entry, head 2 off for one entry, o2 null with zraw set for another, an empty entry,
    saturating logits (+-100: sigmoid underflows / rounds to 1).  Bound: a 256-term dot product with 8 sequential and 5
    tree roundings, |dz| <= 16 eps (sum |w x| + |b|); the sigmoid's slope is at most 1/4 and expf adds 2 ulp:
    |d sigmoid| <= 4 eps (sum |w x| + |b|) + 4 eps."""
    rng = np.random.default_rng(5)
    w1, w2 = _f32(rng.standard_normal(256) * 0.1), _f32(rng.standard_normal(256) * 0.1)
    b1, b2 = _f32([0.3]), _f32([-0.2])
    rows = [9, 1025, 0, 8, 300]
    modes = [7, 5, 7, 0, 3]  # 5: zraw only; 0: head 2 off
    xs = [_f32(rng.standard_normal((r, 256))) for r in rows]
    xs[4][:10] = np.sign(w1) * (100.0 / np.abs(w1).sum())  # logit 1 = +100 + b1
    xs[4][10:20] = -xs[4][:10]  # -100 + b1
    n, np_ = _n(rows)
    x = _f32(np.concatenate(xs))
    tot = int(n.sum())
    o1, o2, zr = (np.full(tot, 5, np.float32) for _ in range(3))
    _check(b200_ctx, b200_ctx.lib.b2_debug_lightglue_rowheads_host(
        b200_ctx.handle, np_, _lib.ptr(n), _lib.ptr(_i32(modes)), _lib.ptr(x), _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2), _lib.ptr(b2),
        _lib.ptr(o1), _lib.ptr(o2), _lib.ptr(zr)), "rowheads")
    x64 = x.astype(np.float64)
    z1, z2 = x64 @ w1 + b1[0], x64 @ w2 + b2[0]
    a1, a2 = np.abs(x64) @ np.abs(w1) + abs(b1[0]), np.abs(x64) @ np.abs(w2) + abs(b2[0])
    sig = lambda z: 0.5 * (1 + np.tanh(z / 2))
    assert np.abs(z1).max() > 90  # the saturating rows are there
    o = 0
    for r, md in zip(rows, modes):
        s = slice(o, o + r)
        assert np.all(np.abs(o1[s] - sig(z1[s])) <= 4 * EPS * a1[s] + 4 * EPS)
        if md & 1 and md & 2:
            assert np.all(np.abs(o2[s] - sig(z2[s])) <= 4 * EPS * a2[s] + 4 * EPS)
        else:
            assert np.all(o2[s] == 5)
        if md & 1 and md & 4:
            assert np.all(np.abs(zr[s] - z2[s]) <= 16 * EPS * a2[s])
        else:
            assert np.all(zr[s] == 5)
        o += r


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [False, True])
def test_gather(b200_ctx, planes):
    """k_lg_gather: count 0, the identity, random monotone maps (what k_lg_prune_plan writes), an empty entry; x, the rotary
    table, ind and (wgmma path) the split planes of x move together; rows past the count are not written.  Exact."""
    rng = np.random.default_rng(6)
    rows = [5, 1025, 0, 300, 2049]
    cnts, srcs = [], []
    for k, r in enumerate(rows):
        if k == 0:
            sel = np.zeros(0, np.int64)
        elif k == 1:
            sel = np.arange(r)
        else:
            sel = np.sort(rng.permutation(r)[: r // 3])
        cnts.append(len(sel)), srcs.append(np.concatenate([sel, np.full(r - len(sel), 0)]))
    n, np_ = _n(rows)
    tot = int(n.sum())
    src, cnt = _i32(np.concatenate(srcs)), _i32(cnts)
    x, cs, sn = _f32(rng.standard_normal((tot, 256))), _f32(rng.standard_normal((tot, 32))), _f32(rng.standard_normal((tot, 32)))
    ind = _i32(rng.integers(0, 1 << 20, tot))
    pl = np.ascontiguousarray(rng.integers(0, 1 << 16, (tot, 2, 256)).astype(np.uint16)) if planes else None
    # the planes of an entry are [2][n][256] (hi then lo): lay each entry out that way
    pl_dev = np.concatenate([pl[o: o + r].transpose(1, 0, 2).reshape(-1) for o, r in zip(np.cumsum([0] + rows[:-1]), rows)]) if planes else None
    x2, cs2, sn2 = np.full_like(x, 3), np.full_like(cs, 3), np.full_like(sn, 3)
    ind2 = np.full_like(ind, -2)
    pl2 = np.full_like(pl_dev, 11) if planes else None
    _check(b200_ctx, b200_ctx.lib.b2_debug_lightglue_gather_host(
        b200_ctx.handle, np_, _lib.ptr(n), _lib.ptr(cnt), _lib.ptr(src), _lib.ptr(x), _lib.ptr(cs), _lib.ptr(sn), _lib.ptr(ind),
        _lib.ptr(pl_dev), _lib.ptr(x2), _lib.ptr(cs2), _lib.ptr(sn2), _lib.ptr(ind2), _lib.ptr(pl2)), "gather")
    o = 0
    for r, c, sr in zip(rows, cnts, srcs):
        g = o + sr[:c]
        assert np.array_equal(x2[o: o + c], x[g]) and np.array_equal(cs2[o: o + c], cs[g]) and np.array_equal(sn2[o: o + c], sn[g])
        assert np.array_equal(ind2[o: o + c], ind[g])
        assert np.all(x2[o + c: o + r] == 3) and np.all(ind2[o + c: o + r] == -2)
        if planes:
            got = pl2[2 * 256 * o: 2 * 256 * (o + r)].reshape(2, r, 256)
            assert np.array_equal(got[:, :c], pl[g].transpose(1, 0, 2)) and np.all(got[:, c:] == 11)
        o += r


# ---------------------------------------------------------------------------------------------------------------------
# network level
# ---------------------------------------------------------------------------------------------------------------------

PROFILES = ["full", "prune", "stop", "sharp"]
SIZES = [(1, 1), (1, 700), (37, 1025), (1024, 1023), (2051, 1500)]
# (profile, n0, n1) -> seed of synthetic_features whose fp64 replay keeps MARGIN from every threshold
SEEDS = {
    ('full', 1, 1): 100,
    ('full', 1, 700): 100,
    ('full', 37, 1025): 100,
    ('full', 1024, 1023): 100,
    ('full', 2051, 1500): 100,
    ('prune', 1, 1): 100,
    ('prune', 1, 700): 102,
    ('prune', 37, 1025): 102,
    ('prune', 1024, 1023): 102,
    ('prune', 2051, 1500): 109,
    ('stop', 1, 1): 100,
    ('stop', 1, 700): 100,
    ('stop', 37, 1025): 100,
    ('stop', 1024, 1023): 100,
    ('stop', 2051, 1500): 102,
    ('sharp', 1, 1): 100,
    ('sharp', 1, 700): 100,
    ('sharp', 37, 1025): 100,
    ('sharp', 1024, 1023): 100,
    ('sharp', 2051, 1500): 102,
}


def _features(seed, n0, n1):
    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(seed, n0, n1)
    return kp0, d0, kp1, d1


def _replay(feats, sd, **kw):
    """fp64 and fp32 traces of the oracle on one pair."""
    t64, t32 = {}, {}
    ref.lightglue_match(*feats[:2], *feats[2:], sd, trace=t64, dtype=np.float64, **kw)
    ref.lightglue_match(*feats[:2], *feats[2:], sd, trace=t32, **kw)
    return t64, t32


def _margin(t64):
    """Distance of the fp64 replay's confidences and matchabilities from the thresholds its decisions compared them with."""
    thr = ref.confidence_thresholds().astype(np.float64)
    keep_thr = np.float32(1 - ref.WIDTH_CONF)
    m = np.inf
    for i in range(ref.N_LAYERS):
        for side in (0, 1):
            if f"t{side}_l{i}" in t64:
                m = min(m, np.abs(t64[f"t{side}_l{i}"] - thr[i]).min(initial=np.inf))
            if f"ma{side}_l{i}" in t64:
                m = min(m, np.abs(t64[f"ma{side}_l{i}"] - keep_thr).min(initial=np.inf))
    return m


def _ratio(dev, r64, r32):
    """Device error over the fp32 oracle's spread from fp64 (floored at one rounding of the largest value)."""
    if r64.size == 0:
        return 0.0
    spread = max(np.abs(r32.astype(np.float64) - r64).max(), EPS * np.abs(r64).max())
    return float(np.abs(dev.astype(np.float64) - r64).max() / spread)


def _compare(recs, pair, t64, t32, bound=None):
    """The trace records of `pair` against the replays: decisions exact, values within BOUND_FACTOR x the fp32 spread (or,
    given `bound`, within that absolute bound).  -> {(kind, layer, side): ratio (or absolute error)}."""
    R = {(r["layer"], r["side"]): r for r in recs if r["pair"] == pair}
    stop = t64["stop"]
    ran = sum(f"desc0_l{l}" in t64 for l in range(ref.N_LAYERS))  # below stop when pruning emptied a side
    assert sorted(R) == [(l, s) for l in range(ran) for s in (0, 1)], (sorted(R), ran)
    out = {}
    for (l, side), r in sorted(R.items()):
        assert np.array_equal(r["ind"], t64[f"ind{side}_l{l}"]), (l, side)
        assert r["n"] == len(t64[f"ind{side}_l{l}"])
        vals = [("x", r["x"], f"desc{side}_l{l}")]
        if r["heads"]:
            vals.append(("conf", r["conf"], f"t{side}_l{l}"))
            if f"ma{side}_l{l}" in t64:
                vals.append(("mat", r["mat"], f"ma{side}_l{l}"))
                assert np.array_equal(r["keep"], t64[f"keep{side}_l{l}"]), (l, side)
            else:  # a side the device does not prune keeps every row
                assert r["kept"] == r["n"] and np.array_equal(r["keep"], np.arange(r["n"]))
            assert r["kept"] == len(r["keep"])
        for kind, dev, key in vals:
            if bound is None:
                v = out[(kind, l, side)] = _ratio(dev, t64[key], t32[key])
                assert v <= BOUND_FACTOR, (kind, l, side, v)
            else:
                v = out[(kind, l, side)] = float(np.abs(dev.astype(np.float64) - t64[key]).max(initial=0))
                assert v <= bound, (kind, l, side, v)
    for l in range(ran):
        if R[(l, 0)]["heads"]:
            assert R[(l, 0)]["unconf"] + R[(l, 1)]["unconf"] == t64[f"unconf_l{l}"], l
        early = ran == stop < ref.N_LAYERS and l == stop - 1
        assert R[(l, 0)]["stop"] == R[(l, 1)]["stop"] == early, (l, stop)
    return out


def _traced_match(eng, feats, **kw):
    eng.ctx.set_option("lightglue_trace", 1)
    try:
        eng.match(*feats, **kw)
        return eng.layer_trace()
    finally:
        eng.ctx.set_option("lightglue_trace", 0)


def _single(ctx, profile, n0, n1, seed, prune_min_kpts=-1, fp16=False, bound=None):
    feats = _features(seed, n0, n1)
    sd = syn.lightglue_state_dict(2, profile)
    t64, t32 = _replay(feats, sd, prune_min_kpts=prune_min_kpts, fp16_attention=fp16)
    assert _margin(t64) > MARGIN, (profile, n0, n1, seed, _margin(t64))
    eng = LightGlueEngine(sd, ctx=ctx)
    recs = _traced_match(eng, feats, prune_min_kpts=prune_min_kpts, fp16_attention=fp16)
    assert eng.last_stop == t64["stop"]
    return _compare(recs, 0, t64, t32, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("profile", PROFILES)
@pytest.mark.parametrize("n0,n1", SIZES)
def test_layers_follow_fp64_replay(b200_ctx, profile, n0, n1):
    _single(b200_ctx, profile, n0, n1, SEEDS[(profile, n0, n1)])


@pytest.mark.gpu
def test_layers_follow_fp64_replay_bench_size(b200_ctx):
    """The pair size and weights bench.py times (5000 x 5000, 'bench': nine layers, nothing pruned)."""
    _single(b200_ctx, "bench", 5000, 5000, 11)


@pytest.mark.gpu
def test_layers_follow_fp64_replay_simt_path():
    ctx = _lib.Context(0)
    try:
        ctx.set_option("force_simt", 1)
        _single(ctx, "prune", 37, 1025, SEEDS[("prune", 37, 1025)])
    finally:
        ctx.close()


@pytest.mark.gpu
def test_layers_follow_fp16_replay_with_fp16_attention(b200_ctx):
    """fp16_attention against the replay's fp16 emulation (operands and result of each attention rounded to fp16): the
    flash kernel's internal rounding of the probabilities cannot be emulated, so values are held to FP16_ATOL absolute;
    'full' weights keep the decisions far from their thresholds."""
    _single(b200_ctx, "full", 300, 350, 5, fp16=True, bound=FP16_ATOL)


BATCH_PROFILE = "prune"
BATCH_PRUNE_MIN = 400
# (seed, n0, n1, encode side 0, encode side 1): sizes, stop layers and prune outcomes differ; sides of at most
# BATCH_PRUNE_MIN rows are never pruned, so (205, 37, 1025) prunes side 1 only; early exits after layers 1, 4, 6 and none
BATCH = [(100, 1, 1, False, False), (202, 1, 700, True, False), (205, 37, 1025, False, False), (102, 1024, 1023, True, True),
         (203, 700, 640, False, True), (200, 3, 2, False, False), (200, 2, 3, True, False), (8, 512, 512, False, False)]


@pytest.mark.gpu
def test_batched_layers_follow_fp64_replay(b200_ctx):
    """One lock-step batch of 8 pairs (b2_lightglue_match_batched_dev), some sides handed in as encodings
    (b2_lightglue_encode_batched_dev): every pair's trace against its own fp64 replay."""
    import torch

    sd = syn.lightglue_state_dict(2, BATCH_PROFILE)
    eng = LightGlueEngine(sd, ctx=b200_ctx)
    lib, h = b200_ctx.lib, b200_ctx.handle
    prm = _lib.LightGlueParams(ref.DEPTH_CONF, ref.WIDTH_CONF, ref.FILTER_TH, BATCH_PRUNE_MIN, 0)
    arr = (_lib.LightGluePair * len(BATCH))()
    keep, reps = [], []
    for i, (seed, n0, n1, e0, e1) in enumerate(BATCH):
        feats = _features(seed, n0, n1)
        t64, t32 = _replay(feats, sd, prune_min_kpts=BATCH_PRUNE_MIN)
        assert _margin(t64) > MARGIN, (seed, _margin(t64))
        reps.append((t64, t32))
        kp0, d0, kp1, d1 = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in feats)
        enc = []
        for kp, d, n, want in ((kp0, d0, n0, e0), (kp1, d1, n1, e1)):
            if not want:
                enc.append(None)
                continue
            blob = torch.empty(lib.b2_lightglue_encoded_bytes(n), dtype=torch.uint8, device="cuda")
            im = (_lib.LightGlueImage * 1)(_lib.LightGlueImage(kp.data_ptr(), d.data_ptr(), n, blob.data_ptr()))
            torch.cuda.synchronize()
            b200_ctx.check(lib.b2_lightglue_encode_batched_dev(h, im, 1, C.byref(prm), None), "encode")
            enc.append(blob)
        cap = max(1, min(n0, n1))
        m = torch.empty((cap, 2), dtype=torch.int64, device="cuda")
        s = torch.empty(cap, dtype=torch.float32, device="cuda")
        keep.append((kp0, d0, kp1, d1, m, s, enc))
        arr[i].kp0, arr[i].desc0, arr[i].n0 = kp0.data_ptr(), d0.data_ptr(), n0
        arr[i].kp1, arr[i].desc1, arr[i].n1 = kp1.data_ptr(), d1.data_ptr(), n1
        arr[i].enc0 = enc[0].data_ptr() if enc[0] is not None else None
        arr[i].enc1 = enc[1].data_ptr() if enc[1] is not None else None
        arr[i].out_matches, arr[i].out_scores = m.data_ptr(), s.data_ptr()
    torch.cuda.synchronize()
    b200_ctx.set_option("lightglue_trace", 1)
    try:
        b200_ctx.check(lib.b2_lightglue_match_batched_dev(h, arr, len(BATCH), C.byref(prm), None), "match_batched_dev")
        torch.cuda.synchronize()
        recs = eng.layer_trace()
    finally:
        b200_ctx.set_option("lightglue_trace", 0)
    for i, (t64, t32) in enumerate(reps):
        assert arr[i].out_stop_layer == t64["stop"], i
        _compare(recs, i, t64, t32)
    stops = {t64["stop"] for t64, _ in reps}
    pruned = [any(f"keep{s}_l{l}" in t64 and len(t64[f"keep{s}_l{l}"]) < len(t64[f"ind{s}_l{l}"]) for l in range(9) for s in (0, 1))
              for t64, _ in reps]
    assert len(stops) >= 3 and 0 < sum(pruned) < len(BATCH), (stops, pruned)


@pytest.mark.gpu
def test_trace_adds_no_launches_and_is_cleared_when_off(b200_ctx):
    feats = _features(5, 300, 350)
    eng = LightGlueEngine(syn.lightglue_state_dict(2, "full"), ctx=b200_ctx)
    l0 = b200_ctx.launch_count()
    eng.match(*feats)
    l1 = b200_ctx.launch_count()
    assert len(_traced_match(eng, feats)) == 18  # nine layers, two sides
    assert b200_ctx.launch_count() - l1 == l1 - l0
    eng.match(*feats)
    assert eng.layer_trace() == []


def _mutated_ffn(gelu_approx="none", eps=1e-5):
    F = ref.F

    def ffn(sd, p, x, msg):
        h = ref._lin(sd, p + "ffn.0", ref.torch.cat([x, msg], -1))
        h = F.layer_norm(h, (h.shape[-1],), ref._w(sd, p + "ffn.1.weight"), ref._w(sd, p + "ffn.1.bias"), eps)
        return x + ref._lin(sd, p + "ffn.3", F.gelu(h, approximate=gelu_approx))

    return ffn


_ROTARY = ref.rotary_table


def _swapped_rotary(sd, kpn):
    c, s = _ROTARY(sd, kpn)
    c, s = c.clone(), s.clone()
    c[:, :2], s[:, :2] = s[:, :2].clone(), c[:, :2].clone()  # frequency 0: sin and cos exchanged
    return c, s


@pytest.mark.parametrize("slip", ["tanh_gelu", "ln_eps_1e-6", "rotary_sin_cos"])
def test_bound_rejects_plausible_slips(monkeypatch, slip):
    """CPU: an fp64 replay with one plausible kernel slip leaves the bound of the network-level tests at some layer, so a
    device with that slip would fail them (the told case of test_flash_ps_gpu.py)."""
    feats = _features(SEEDS[("prune", 37, 1025)], 37, 1025)
    sd = syn.lightglue_state_dict(2, "prune")
    t64, t32 = _replay(feats, sd)
    if slip == "tanh_gelu":
        monkeypatch.setattr(ref, "_ffn", _mutated_ffn(gelu_approx="tanh"))
    elif slip == "ln_eps_1e-6":
        monkeypatch.setattr(ref, "_ffn", _mutated_ffn(eps=1e-6))
    else:
        monkeypatch.setattr(ref, "rotary_table", _swapped_rotary)
    tm = {}
    ref.lightglue_match(*feats[:2], *feats[2:], sd, trace=tm, dtype=np.float64)
    worst = 0.0
    for l in range(min(tm["stop"], t64["stop"])):
        for side in (0, 1):
            a, b = tm[f"desc{side}_l{l}"], t64[f"desc{side}_l{l}"]
            if a.shape == b.shape:
                worst = max(worst, _ratio(a, b, t32[f"desc{side}_l{l}"]))
    assert worst > BOUND_FACTOR, worst
