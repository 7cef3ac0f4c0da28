"""GPU: the shared linear (run_linear: the wgmma split-fp16 k_gemm_ws and the exact-fp32 SIMT k_gemm_nt), through
b2_debug_linear_host, in every mode its callers use, against fp64 (oracle/linear_ref.py) and bit for bit against itself.

Each row of CASES stands for one call site at its mode and shape (N reduced where the real one would need hundreds of MB
on the host, K and the chunk structure kept), beside the M x N x K grid of ragged shapes: an 8-row and a 1-row last row tile,
fewer tiles than SMs, column tiles cut at N = 64, 200 and 130 (130 has no 16-byte aligned rows, so the epilogue takes its
per-element path).  K walked in chunks is composed here, one launch per chunk with the previous output as the residual.

Tolerance (oracle/linear_ref.py derives it term by term): with S = sum_k |a_k b_k| of one launch of K_l columns,
16 * 2^-22 * S for the operand split, (K_l / 16) * 2^-23 * S for the truncating fp32 accumulation (one truncation per k16
MMA; consistent with the -4e-5 retrieval.cu records, not checked on its own), 2^-23 * S for joining the two accumulators,
2^-23 relative for each fp32 epilogue operation and chunk add, and for GELU 1.13 x the error of its input plus
2^-20 |GELU| + 2^-23 |x|.  The SIMT path's GEMM term is K_l * 2^-23 * S.  The bound is checked to be tight enough to matter:
a plain fp16 GEMM (hi planes only) must exceed it on the grid, and a single unchunked K = 8192 launch on retrieval-like data
must exceed the bound of the 256-column chunks that retrieval.cu walks.

Every output is written over sentinels (NaN in fp32, 0x7E01 in planes): pitch padding, and head-major columns past N, must
come back untouched; the entry point itself fails when rows past M are written.  Plane outputs must equal the split of the
same launch's fp32 output, bit for bit."""
import ctypes
import zlib

import numpy as np
import pytest

from gtsfm_b200 import _lib
from oracle import linear_ref as lr

pytestmark = pytest.mark.gpu

PLANE_SENTINEL = 0x7E01
B2_ERR_ARG = -2


class Prob:
    """One problem's host buffers; outputs start filled with sentinels."""

    def __init__(self, a1, b, n, *, a2=None, resid=None, fp32=True, planes=False, ldc=None, ldch=None, hm=False, c=None):
        self.a1, self.b, self.a2, self.resid, self.m, self.n, self.hm = a1, b, a2, resid, a1.shape[0], n, hm
        self.ldc = 0 if hm else (ldc or n)
        self.ldch = 0 if hm else (ldch or n)
        size = lr.head_major_elems(self.m, n) if hm else None
        self.c = c if c is not None else ((np.full(size, np.nan, np.float32) if hm else np.full((self.m, self.ldc), np.nan, np.float32))
                                          if fp32 else None)
        psize = size if hm else self.m * self.ldch
        self.hi = np.full(psize, PLANE_SENTINEL, np.uint16) if planes else None
        self.lo = np.full(psize, PLANE_SENTINEL, np.uint16) if planes else None

    def struct(self):
        def ld(x):
            return 0 if x is None else x.shape[1]

        return _lib.LinearProblem(_lib.ptr(self.a1).value, ld(self.a1), _lib.ptr(self.a2).value, ld(self.a2), _lib.ptr(self.b).value,
                                  ld(self.b), _lib.ptr(self.resid).value, ld(self.resid), _lib.ptr(self.c).value, self.ldc,
                                  _lib.ptr(self.hi).value, _lib.ptr(self.lo).value, self.ldch, self.m, self.n)

    def out(self):
        """fp32 output as [m][n]."""
        return lr.from_head_major(self.c, self.n) if self.hm else self.c[:, :self.n]

    def planes(self):
        if self.hm:
            return lr.from_head_major(self.hi, self.n), lr.from_head_major(self.lo, self.n)
        return self.hi.reshape(self.m, self.ldch)[:, :self.n], self.lo.reshape(self.m, self.ldch)[:, :self.n]


def _call(ctx, probs, *, path=1, k1, k2=0, per_b=False, bias=None, scale=1.0, relu=False, gelu=False, hm=False, unscaled=False,
          in_place=False):
    launch = _lib.LinearLaunch(path, k1, k2, int(per_b), _lib.ptr(bias).value, scale, int(relu), int(gelu), int(hm), int(unscaled),
                               int(in_place))
    arr = (_lib.LinearProblem * len(probs))(*[p.struct() for p in probs])
    return ctx.lib.b2_debug_linear_host(ctx.handle, ctypes.byref(launch), arr, len(probs))


def _run(ctx, probs, **kw):
    rc = _call(ctx, probs, **kw)
    ctx.check(rc, "b2_debug_linear_host")
    return probs


def _check_untouched(p):
    """Sentinels outside rows < m, columns < n came back as they went in."""
    if p.c is not None:
        if p.hm:
            rest = p.c.reshape(-1, p.m, 64)[-1][:, p.n - 64 * (lr.head_major_elems(p.m, p.n) // (64 * p.m) - 1):]
            assert np.isnan(rest).all(), "head-major columns past N written"
        else:
            assert np.isnan(p.c[:, p.n:]).all(), "fp32 pitch padding written"
    if p.hi is not None:
        for x in (p.hi, p.lo):
            if p.hm:
                rest = x.reshape(-1, p.m, 64)[-1][:, p.n - 64 * (x.size // (64 * p.m) - 1):]
            else:
                rest = x.reshape(p.m, p.ldch)[:, p.n:]
            assert (rest == PLANE_SENTINEL).all(), "plane padding written"


def _check_planes(p, unscaled):
    if p.hi is None or p.c is None:
        return
    want_hi, want_lo = lr.split_planes(p.out(), unscaled)
    hi, lo = p.planes()
    assert np.array_equal(hi, want_hi), int((hi != want_hi).sum())
    assert np.array_equal(lo, want_lo), int((lo != want_lo).sum())


def _ratio(name, err, bound):
    r = float((err / bound).max()) if err.size else 0.0
    print(f"err/bound {name}: {r:.4f}")
    return r


# ---- data ----------------------------------------------------------------------------------------------------------------------
def _mat(rng, m, k, kind="normal"):
    x = rng.standard_normal((m, k))
    if kind == "relu":
        x = np.maximum(x, 0.0)
    return x.astype(np.float32)


def _weight(rng, n, k):
    return (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)


def _unit_rows(rng, n, k):
    """Retrieval-like descriptors: unit rows sharing a common component (every similarity around 0.5)."""
    common = rng.standard_normal(k)
    x = common + rng.standard_normal((n, k))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


# ---- single-launch call sites ---------------------------------------------------------------------------------------------------
# name: dict(ms, ns (one per problem, or one for all), k1, k2, per_b, bias, scale, relu, gelu, hm, unscaled, planes, ldc, ldch,
#            resid: None | "sep" | "table" | "inplace", lda1: pitch of A1 (> k1: the unused columns hold NaN), a: data kind)
_M16 = [0, 1, 127, 128, 129, 700, 2048, 0, 1, 127, 128, 129, 700, 2048, 0, 1]
CASES = {
    "lg_ffn0_cat": dict(ms=_M16, ns=512, k1=256, k2=256, bias=True),
    "lg_ffn3_inplace": dict(ms=[700, 129], ns=256, k1=512, bias=True, resid="inplace", planes=True, ldch=256),
    "lg_assign_proj": dict(ms=[700, 301], ns=256, k1=256, bias=True, scale=0.25, planes=True, ldch=256),
    "lg_assign_sim": dict(ms=[700, 1, 129, 300, 64, 1000, 5, 257], ns=[1025, 63, 65, 130, 1, 700, 3, 129], k1=256, per_b=True),
    "sg_qkv": dict(ms=[1000, 77], ns=256, k1=256, bias=True, hm=True, unscaled=True, planes=True),
    "sg_ffn0_relu": dict(ms=[513, 200], ns=512, k1=256, k2=256, bias=True, relu=True, planes=True, ldch=512),
    "ml_patch_embed": dict(ms=[529] * 16, ns=768, k1=640, bias=True, resid="table"),
    "ml_qkv": dict(ms=[530], ns=2304, k1=768, bias=True, hm=True, unscaled=True, planes=True),
    "ml_fc1_gelu": dict(ms=[530], ns=3072, k1=768, bias=True, gelu=True, planes=True, ldch=3072),
    "ml_salad_strided": dict(ms=[530], ns=256, k1=512, lda1=1024, bias=True, a="relu"),
    "ml_cls_rows": dict(ms=[16], ns=512, k1=768, lda1=530 * 768, bias=True, relu=True, planes=True, ldch=512),
    "sg_sim_scale_resid": dict(ms=[300, 129], ns=130, k1=256, bias=True, scale=1 / 16, resid="sep"),
    "sp_convPb": dict(ms=[4800], ns=65, k1=256, ldc=68, bias=True),
    "sat_vec4": dict(ms=[200], ns=128, k1=64, planes=True, a="big"),
    "sat_per_element": dict(ms=[200], ns=128, k1=64, planes=True, ldc=129, ldch=129, a="big"),
}
GRID = {f"grid_M{M}_N{N}_K{K}": dict(ms=[M], ns=N, k1=K, bias=True, hi_only_guard=True)
        for M in (1, 8, 129, 5000) for N in (64, 130, 200, 768) for K in (64, 256, 512)}


def _build(spec, seed, path=1, with_fp32=True, with_planes=None):
    rng = np.random.default_rng(seed)
    ms = spec["ms"]
    ns = spec["ns"] if isinstance(spec["ns"], list) else [spec["ns"]] * len(ms)
    k1, k2 = spec["k1"], spec.get("k2", 0)
    kind = spec.get("a", "normal")
    planes = spec.get("planes", False) if with_planes is None else with_planes
    per_b, hm = spec.get("per_b", False), spec.get("hm", False)
    nmax = max(ns)
    shared_b = _weight(rng, nmax, k1 + k2) * np.float32(40.0 if kind == "big" else 1.0)  # "big": outputs around 8e4
    table = rng.standard_normal((max(ms), nmax)).astype(np.float32)
    probs, data = [], []
    for m, n in zip(ms, ns):
        lda1 = spec.get("lda1", k1)
        a1 = np.full((m, lda1), np.nan, np.float32)
        a1[:, :k1] = _mat(rng, m, k1, "normal" if kind == "big" else kind) * (2000.0 if kind == "big" else 1.0)
        a2 = _mat(rng, m, k2, kind) if k2 else None
        b = _weight(rng, n, k1 + k2) if per_b else shared_b
        resid, c = None, None
        r = spec.get("resid")
        if r == "sep":
            resid = rng.standard_normal((m, n)).astype(np.float32)
        elif r == "table":
            resid = np.ascontiguousarray(table[:m, :n])
        elif r == "inplace":
            ldc = spec.get("ldc") or n
            c = np.full((m, ldc), np.nan, np.float32)
            c[:, :n] = rng.standard_normal((m, n))
            resid = c[:, :n].copy()
        p = Prob(a1, b, n, a2=a2, resid=None if r == "inplace" else resid, fp32=with_fp32, planes=planes and path == 1,
                 ldc=spec.get("ldc"), ldch=spec.get("ldch"), hm=hm, c=c)
        probs.append(p)
        data.append((a1[:, :k1], a2, b if per_b else shared_b[:n], resid))
    bias = rng.standard_normal(nmax).astype(np.float32) if spec.get("bias") else None
    kw = dict(path=path, k1=k1, k2=k2, per_b=per_b, bias=bias, scale=spec.get("scale", 1.0), relu=spec.get("relu", False),
              gelu=spec.get("gelu", False), hm=hm, unscaled=spec.get("unscaled", False), in_place=spec.get("resid") == "inplace")
    return probs, data, kw


def _want(data, kw):
    out = []
    for a1, a2, b, resid in data:
        e = dict(a2=a2, bias=kw["bias"], scale=kw["scale"], relu=kw["relu"], gelu=kw["gelu"], resid=resid)
        out.append((lr.linear64(a1, b, **e), lr.launch_bound(a1, b, path=kw["path"], **e)))
    return out


@pytest.mark.parametrize("name", list(CASES) + list(GRID))
def test_linear_matches_fp64(b200_ctx, name):
    spec = CASES.get(name) or GRID[name]
    probs, data, kw = _build(spec, seed=zlib.crc32(name.encode()))
    _run(b200_ctx, probs, **kw)
    worst = 0.0
    for p, (want, bound), (a1, a2, b, _) in zip(probs, _want(data, kw), data):
        if p.m == 0:
            continue
        got = p.out()
        assert np.isfinite(got).all()
        if spec.get("a") == "big":  # outputs far beyond fp16's range: planes saturate, fp32 keeps the value
            assert np.abs(want).max() > 2 * 65504
            hi, lo = p.planes()
            big = np.abs(got) > 65504
            assert big.any() and (hi[got > 65504] == 0x7BFF).all() and (hi[got < -65504] == 0xFBFF).all() and (lo[big] == 0).all()
        err = np.abs(got - want)
        worst = max(worst, float((err / bound).max()))
        assert (err <= bound).all(), (name, p.m, p.n, float(err.max()), float((err / bound).max()))
        _check_untouched(p)
        _check_planes(p, kw["unscaled"])
        if spec.get("hi_only_guard"):
            hi_only = lr.linear64(a1.astype(np.float16), b.astype(np.float16), bias=kw["bias"])
            assert (np.abs(hi_only - want) > bound).any(), "the bound does not tell split-fp16 from plain fp16 at this shape"
    print(f"err/bound {name}: {worst:.4f}")


# ---- K walked in chunks -----------------------------------------------------------------------------------------------------
# name: (M or None for B = A, N, K, chunk, A kind, resid_in_place, bias, initial residual)
CHUNKED = {
    "ml_fc2_chunks": (530, 768, 3072, 1024, "normal", True, True, True),
    "retrieval_700": (None, 700, 4096, 256, "unit", True, False, False),
    "retrieval_301": (None, 301, 4096, 256, "unit", False, False, False),
    "netvlad_whiten": (16, 256, 8192, 512, "relu", True, True, False),
    "ml_head": (16, 256, 16640, 640, "relu", False, True, False),
}


def _chunked(ctx, a, b, kc, *, bias=None, x0=None, in_place=False, per_b=False, path=1):
    """K in chunks of kc, chunk c adding chunk c - 1's output as its residual (in place or from a separate buffer)."""
    m, n = a.shape[0], b.shape[0]
    prev = x0
    for c0 in range(0, a.shape[1], kc):
        a1, b1 = np.ascontiguousarray(a[:, c0:c0 + kc]), np.ascontiguousarray(b[:, c0:c0 + kc])
        if in_place and prev is not None:
            p = Prob(a1, b1, n, c=prev.copy())
            _run(ctx, [p], path=path, k1=a1.shape[1], bias=bias if c0 == 0 else None, per_b=per_b, in_place=True)
        else:
            p = Prob(a1, b1, n, resid=prev)
            _run(ctx, [p], path=path, k1=a1.shape[1], bias=bias if c0 == 0 else None, per_b=per_b)
        prev = p.c
    return prev


@pytest.mark.parametrize("name", list(CHUNKED))
def test_chunked_k_matches_fp64(b200_ctx, name):
    m, n, k, kc, kind, in_place, with_bias, with_x0 = CHUNKED[name]
    rng = np.random.default_rng(k + n)
    if m is None:
        a = _unit_rows(rng, n, k)
        b = a
    else:
        a, b = _mat(rng, m, k, kind), _weight(rng, n, k)
    bias = rng.standard_normal(n).astype(np.float32) if with_bias else None
    x0 = rng.standard_normal((a.shape[0], n)).astype(np.float32) if with_x0 else None
    got = _chunked(b200_ctx, a, b, kc, bias=bias, x0=x0, in_place=in_place, per_b=m is None)
    want = lr.linear64(a, b, bias=bias, resid=x0)
    bound = lr.chunked_bound(a, b, kc, bias=bias, resid=x0)
    err = np.abs(got - want)
    _ratio(name, err, bound)
    assert (err <= bound).all(), (name, float(err.max()), float((err / bound).max()))


def test_unchunked_long_k_exceeds_the_chunked_bound(b200_ctx):
    """The chunks are needed: one K = 8192 launch on retrieval-like data is off by more than the 256-chunked sum may be."""
    rng = np.random.default_rng(8192)
    a = _unit_rows(rng, 512, 8192)
    p = _run(b200_ctx, [Prob(a, a, 512)], k1=8192)[0]
    want = lr.linear64(a, a)
    err = np.abs(p.out() - want)
    chunked = lr.chunked_bound(a, a, 256)
    print(f"unchunked K = 8192: max err {float(err.max()):.3e}, mean signed err {float((p.out() - want).mean()):.3e}, "
          f"max err / chunked bound {float((err / chunked).max()):.3f}")
    assert (err <= lr.launch_bound(a, a)).all()
    assert (err > chunked).any()


# ---- bit for bit ------------------------------------------------------------------------------------------------------------
def test_batched_problem_equals_alone(b200_ctx):
    spec = CASES["lg_ffn0_cat"]
    probs, data, kw = _build(spec, seed=1)
    _run(b200_ctx, probs, **kw)
    for i in (2, 4, 5, 6, 13):  # M = 127, 129, 700, 2048, 2048
        alone = _run(b200_ctx, [Prob(probs[i].a1, probs[i].b, probs[i].n, a2=probs[i].a2)], **kw)[0]
        assert np.array_equal(alone.c, probs[i].c), i


def test_two_runs_agree(b200_ctx):
    first, _, kw = _build(CASES["lg_ffn0_cat"], seed=2)
    second, _, _ = _build(CASES["lg_ffn0_cat"], seed=2)
    _run(b200_ctx, first, **kw)
    _run(b200_ctx, second, **kw)
    for p, q in zip(first, second):
        assert p.c is None or np.array_equal(p.c, q.c, equal_nan=True)


@pytest.mark.parametrize("epi", ["gelu_resid", "relu_scale_resid", "unscaled", "head_major"])
def test_vec4_epilogue_equals_per_element(b200_ctx, epi):
    """ldc = ldch = ldr = N takes the 16-byte path, N + 1 the per-element path: same values, bit for bit."""
    rng = np.random.default_rng(40)
    m, n, k = 300, 256, 256
    a, b = _mat(rng, m, k), _weight(rng, n, k)
    bias = rng.standard_normal(n).astype(np.float32)
    resid = rng.standard_normal((m, n + 1)).astype(np.float32)
    kw = dict(k1=k, bias=bias, scale=0.25 if epi == "relu_scale_resid" else 1.0, relu=epi == "relu_scale_resid", gelu=epi == "gelu_resid",
              unscaled=epi == "unscaled")
    outs = []
    for ld in (n, n + 1):
        r = np.ascontiguousarray(resid[:, :ld]) if "resid" in epi else None
        p = Prob(a, b, n, resid=r, planes=True, ldc=ld, ldch=ld)
        _run(b200_ctx, [p], **kw)
        _check_untouched(p)
        _check_planes(p, kw["unscaled"])
        outs.append((p.out(), *p.planes()))
    for x, y in zip(*outs):
        assert np.array_equal(x, y)


def test_planes_only_equal_planes_with_fp32(b200_ctx):
    for name in ("sg_qkv", "lg_assign_proj", "ml_fc1_gelu"):
        both, _, kw = _build(CASES[name], seed=5)
        only, _, _ = _build(CASES[name], seed=5, with_fp32=False)
        _run(b200_ctx, both, **kw)
        _run(b200_ctx, only, **kw)
        for p, q in zip(both, only):
            assert q.c is None
            assert np.array_equal(p.hi, q.hi) and np.array_equal(p.lo, q.lo), name


def test_resid_in_place_equals_separate(b200_ctx):
    rng = np.random.default_rng(6)
    m, n, k = 700, 256, 512
    a, b, x = _mat(rng, m, k), _weight(rng, n, k), rng.standard_normal((m, n)).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    sep = _run(b200_ctx, [Prob(a, b, n, resid=x, planes=True)], k1=k, bias=bias)[0]
    inp = _run(b200_ctx, [Prob(a, b, n, c=x.copy(), planes=True)], k1=k, bias=bias, in_place=True)[0]
    assert np.array_equal(sep.c, inp.c) and np.array_equal(sep.hi, inp.hi) and np.array_equal(sep.lo, inp.lo)


@pytest.mark.parametrize("path", [1, 0])
def test_k_segments_equal_one_operand(b200_ctx, path):
    rng = np.random.default_rng(7)
    m, n = 513, 512
    a1, a2, b = _mat(rng, m, 256), _mat(rng, m, 256), _weight(rng, n, 512)
    bias = rng.standard_normal(n).astype(np.float32)
    two = _run(b200_ctx, [Prob(a1, b, n, a2=a2)], path=path, k1=256, k2=256, bias=bias, relu=True)[0]
    one = _run(b200_ctx, [Prob(np.concatenate([a1, a2], 1), b, n)], path=path, k1=512, bias=bias, relu=True)[0]
    assert np.array_equal(two.c, one.c)


@pytest.mark.parametrize("path", [1, 0])
def test_strided_a_equals_contiguous(b200_ctx, path):
    rng = np.random.default_rng(8)
    m, n, k = 530, 256, 512
    wide = np.full((m, 2 * k), np.nan, np.float32)
    wide[:, :k] = _mat(rng, m, k)
    b = _weight(rng, n, k)
    strided = _run(b200_ctx, [Prob(wide, b, n)], path=path, k1=k)[0]
    contiguous = _run(b200_ctx, [Prob(np.ascontiguousarray(wide[:, :k]), b, n)], path=path, k1=k)[0]
    assert np.array_equal(strided.c, contiguous.c)


@pytest.mark.parametrize("path", [1, 0])
def test_head_major_equals_row_major(b200_ctx, path):
    rng = np.random.default_rng(9)
    m, n, k = 77, 200, 256
    a, b = _mat(rng, m, k), _weight(rng, n, k)
    bias = rng.standard_normal(n).astype(np.float32)
    planes = path == 1
    hm = _run(b200_ctx, [Prob(a, b, n, hm=True, planes=planes)], path=path, k1=k, bias=bias, hm=True, unscaled=True)[0]
    rm = _run(b200_ctx, [Prob(a, b, n, planes=planes)], path=path, k1=k, bias=bias, unscaled=True)[0]
    _check_untouched(hm)
    assert np.array_equal(hm.out(), rm.out())
    if planes:
        for x, y in zip(hm.planes(), rm.planes()):
            assert np.array_equal(x, y)


# ---- the SIMT path ----------------------------------------------------------------------------------------------------------
SIMT_CASES = {
    "ragged": dict(ms=[1, 129, 700], ns=[1, 65, 130], k1=256, per_b=True, bias=True),
    "cat_relu_scale_resid": dict(ms=[513, 64], ns=512, k1=256, k2=256, bias=True, relu=True, scale=0.25, resid="sep"),
    "head_major": dict(ms=[1000, 77], ns=200, k1=256, bias=True, hm=True),
}


@pytest.mark.parametrize("name", list(SIMT_CASES))
def test_simt_matches_fp64_and_wgmma(b200_ctx, name):
    spec = SIMT_CASES[name]
    simt, data, kw = _build(spec, seed=11, path=0)
    tc, _, kw1 = _build(spec, seed=11, path=1)
    _run(b200_ctx, simt, **kw)
    _run(b200_ctx, tc, **kw1)
    for p, q, (want, bound0), (_, bound1) in zip(simt, tc, _want(data, kw), _want(data, kw1)):
        err = np.abs(p.out() - want)
        _ratio(f"simt {name}", err, bound0)
        assert (err <= bound0).all(), (name, float((err / bound0).max()))
        assert (np.abs(p.out().astype(np.float64) - q.out()) <= bound0 + bound1).all()
        _check_untouched(p)


# ---- refusals ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path,k1,k2", [(1, 96, 0), (1, 96, 32), (1, 64, 32), (0, 24, 0), (0, 16, 8)])
def test_ragged_k_is_refused(b200_ctx, path, k1, k2):
    rng = np.random.default_rng(12)
    a1 = _mat(rng, 10, k1)
    a2 = _mat(rng, 10, k2) if k2 else None
    p = Prob(a1, _weight(rng, 16, k1 + k2), 16, a2=a2)
    assert _call(b200_ctx, [p], path=path, k1=k1, k2=k2) == B2_ERR_ARG
    assert np.isnan(p.c).all()


def test_too_many_problems_are_refused(b200_ctx):
    rng = np.random.default_rng(13)
    b = _weight(rng, 64, 64)
    probs = [Prob(_mat(rng, 4, 64), b, 64) for _ in range(17)]
    assert _call(b200_ctx, probs, k1=64) == B2_ERR_ARG
    assert _call(b200_ctx, probs[:16], k1=64) == 0


def test_simt_refuses_planes_and_gelu(b200_ctx):
    rng = np.random.default_rng(14)
    a, b = _mat(rng, 8, 64), _weight(rng, 64, 64)
    assert _call(b200_ctx, [Prob(a, b, 64, planes=True)], path=0, k1=64) == B2_ERR_ARG
    assert _call(b200_ctx, [Prob(a, b, 64)], path=0, k1=64, gelu=True) == B2_ERR_ARG
