"""GPU: the SuperGlue and LightGlue assignment step (statistics, mutual arg-max, filter) on both of its code paths, through
b2_debug_superglue_assign_host / b2_debug_lightglue_assign_host, against the fp64 restatements of oracle/assign_ref.py.

Path 1 is the persistent cooperative kernel k_assign_ps<KIND> (assign_ps.cuh), path 2 the multi-launch kernels; path 0
is the matcher's own choice, asserted to be the expected one.  Shapes reach one row / one column, CTAs that own no rows,
a one-row last ring step, columns in a thread's last slot (N around multiples of 1024; SuperGlue's dustbin makes it N + 1),
the persistent kernel's column limits (8191 / 6240), CTA counts 1 .. SM count, ragged pitches and tall matrices.

Every case plants maxima at the edges where an index computation goes wrong: row maxima at columns N - 1, 1023 and 1024,
column maxima at row M - 1 and at the first and last row of every CTA's row block.  Each has a margin of at least 1.0 in the
final score, so its arg-max must be exact.  Exact ties come from columns and rows duplicated bit for bit (in-thread,
in-warp, cross-warp and cross-CTA pairs): the kernels must return the first index, like torch.max, so only the first
duplicate row survives the mutual check.

Bounds (u = 2^-24).  A logsumexp is computed as m + log(sum exp(x - m)) with terms in (0, 1] and a sum >= 1.  Each term
carries a few ulp of the largest magnitude A inside the logsumexp (forming x and x - m, expf), and each addition of a
sequential chain rounds by at most half an ulp of the sum.  The chains are the kernels' own: the multi-launch row pass adds
ceil(n / 32) terms per lane before 5 shuffle levels, k_sg_cols ceil((M + 1) / 8) per warp before 8 partials,
k_lg_col_stats ceil(M / 32) per warp before 32, the persistent kernel at most 8 columns per thread before 10 levels and its
CTA's rows_per rows per column before the cross-CTA merge.  With d the longest chain of either path the bound per
logsumexp is e = u (d + 16 + 4 A).  Sinkhorn adds one such term per half-iteration: logsumexp is 1-Lipschitz in the sup
norm, so errors add and do not grow: eps_u = K e_row + (K - 1) e_col, eps_v = K (e_row + e_col).  A score
((z + u) + v) - norm adds 4 ulp of its magnitudes.  Within a row the u term is common to every score, so the row arg-max
ranks by a quantity off by at most eps_v + rounding (column arg-max: eps_u + rounding); LightGlue likewise ranks a row by
column statistics only.  The bound bites: the fp64 reference on Z rounded to fp16 exceeds it in every case (fp16 rounds
every planted value by 2^-7, and the planted entry dominates its row's logsumexp)."""
import ctypes as C

import numpy as np
import pytest
import torch

from gtsfm_b200 import _lib
from oracle import assign_ref

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LOG_TH = {"sg": 0.2, "lg": 0.1}  # the matchers' default thresholds
PLANT = {"soft": 24.0 + 2.0 ** -7, "sharp": 32.0 + 2.0 ** -7}  # fp16 rounds both by 2^-7


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def fits(kind, N):
    """assign_ps_fits: 8 column slots of 1024 threads, and the ring (+ LightGlue's column constants) in 220 KB."""
    pitch = (N + 31) // 32 * 32
    smem = (3 * 2 * pitch + (3 * N if kind == "lg" else 0)) * 4
    return N + (1 if kind == "sg" else 0) <= 8192 and smem <= 220 * 1024


def chains(kind, M, N, G):
    """Longest sequential summation chain of a row / column logsumexp over both paths (see the module docstring)."""
    aug = 1 if kind == "sg" else 0
    M1, N1 = M + aug, N + aug
    rows_per = -(-M1 // G)
    d_row = max(-(-N1 // 32) + 5, -(-N1 // 1024) + 10)
    d_col = max(-(-M1 // 8) + 8 if kind == "sg" else -(-M // 32) + 32, rows_per + -(-G // 32) + 5)
    return d_row, d_col


def e_lse(d, amax):
    return U * (d + 16 + 4 * amax)


# ---- inputs ----------------------------------------------------------------------------------------------------------------

def make_case(kind, M, N, G, values="soft", seed=0, z_tail=False, ind=False):
    """Score matrix with planted edge maxima and duplicated columns / rows.  -> dict of inputs and what was planted."""
    rng = np.random.default_rng(seed + 7919 * M + 104729 * N + (1 if kind == "lg" else 0))
    Z = rng.standard_normal((M, N)).astype(np.float32)
    z0 = (rng.standard_normal(M) * 2).astype(np.float32)
    z1 = (rng.standard_normal(N) * 2).astype(np.float32)
    if z_tail:  # the logsigmoid tails
        z0 = np.where(rng.random(M) < 0.5, -30.0, 30.0).astype(np.float32)
        z1 = np.where(rng.random(N) < 0.5, -30.0, 30.0).astype(np.float32)
    M1 = M + (1 if kind == "sg" else 0)
    rows_per = -(-M1 // G)
    row_t = [M - 1] + [r for b in range(G) for r in (b * rows_per, min(M1, (b + 1) * rows_per) - 1) if b * rows_per < M1]
    row_t = list(dict.fromkeys(r for r in row_t if r < M))
    col_t = [j for j in (N - 1, 1023, 1024) if j < N]
    free_r, free_c = set(range(M)), set(range(N))
    plant = []

    def take(i, j):
        free_r.discard(i), free_c.discard(j)
        plant.append((i, j))

    for j in col_t:
        rs = [r for r in row_t if r in free_r] or sorted(free_r)
        if not rs or j not in free_c:
            continue
        take(rs[0], j)
    for i in row_t:
        if i in free_r and free_c:
            take(i, sorted(free_c)[int(rng.integers(len(free_c)))])
    col_dup, row_dup, col_ties, row_ties = {}, {}, [], []
    for off in (5, 100, 1024):  # in-warp, cross-warp, in-thread (k -> k + 1) pairs of the row arg-max
        cand = [j for j in sorted(free_c) if j + off in free_c and j + off != j]
        if not cand or len(free_r) < 1:
            continue
        js = cand[len(cand) // 3]
        r = sorted(free_r)[len(free_r) // 2]
        take(r, js)
        free_c.discard(js + off)
        col_dup[js + off] = js
        col_ties.append((r, js, js + off))
    for off in (1, rows_per, 7):  # same step, next CTA's block, another ring step
        cand = [i for i in sorted(free_r) if i + off in free_r and off > 0]
        if not cand or not free_c:
            continue
        rs = cand[len(cand) // 2]
        c = sorted(free_c)[len(free_c) // 2]
        take(rs, c)
        free_r.discard(rs + off)
        row_dup[rs + off] = rs
        row_ties.append((rs, rs + off, c))
    if values == "sharp":  # a diagonal at 20x on the rows / columns left free: most exp terms underflow, as in the "sharp" fixtures
        fr, fc = rng.permutation(np.array(sorted(free_r), np.int64)), rng.permutation(np.array(sorted(free_c), np.int64))
        k = min(len(fr), len(fc))
        Z[fr[:k], fc[:k]] += 20.0
    T = np.float32(PLANT[values])
    for i, j in plant:
        Z[i, j] = T
        z0[i], z1[j] = max(z0[i], 3.0), max(z1[j], 3.0)
    for jd, js in col_dup.items():
        Z[:, jd], z1[jd] = Z[:, js], z1[js]
    for rd, rs in row_dup.items():
        Z[rd, :], z0[rd] = Z[rs, :], z0[rs]
    i0 = i1 = None
    if ind:  # a non-identity, increasing index map, as pruning leaves it
        i0 = np.sort(rng.choice(3 * M, M, replace=False)).astype(np.int32)
        i1 = np.sort(rng.choice(3 * N, N, replace=False)).astype(np.int32)
    return dict(Z=np.ascontiguousarray(Z), z0=z0, z1=z1, plant=plant, col_dup=col_dup, row_dup=row_dup, col_ties=col_ties,
                row_ties=row_ties, ind0=i0, ind1=i1, G=G)


# ---- the kernels -----------------------------------------------------------------------------------------------------------

def run_kernel(ctx, kind, case, path, alpha=1.0, iters=20):
    Z = case["Z"]
    M, N = Z.shape
    k, ran = C.c_int(-1), C.c_int(0)
    best0 = np.full(M, np.nan, np.float32)
    arg0, arg1 = np.full(M, -1, np.int32), np.full(N, -1, np.int32)
    scores = np.full(M, np.nan, np.float32)
    p = _lib.ptr
    if kind == "sg":
        u, v = np.full(M + 1, np.nan, np.float32), np.full(N + 1, np.nan, np.float32)
        out = np.zeros((M, 2), np.uint32)
        rc = ctx.lib.b2_debug_superglue_assign_host(ctx.handle, path, case["G"], p(Z), M, N, alpha, iters, LOG_TH["sg"], p(u), p(v),
                                                    p(best0), p(arg0), p(arg1), p(out), p(scores), C.byref(k), C.byref(ran))
        ctx.check(rc, "b2_debug_superglue_assign_host")
        stats = dict(u=u, v=v)
    else:
        rs, cs = np.full((3, M), np.nan, np.float32), np.full((3, N), np.nan, np.float32)
        out = np.zeros((M, 2), np.int64)
        rc = ctx.lib.b2_debug_lightglue_assign_host(ctx.handle, path, case["G"], p(Z), M, N, p(case["z0"]), p(case["z1"]),
                                                    p(case["ind0"]), p(case["ind1"]), LOG_TH["lg"], p(rs), p(cs), p(best0), p(arg0),
                                                    p(arg1), p(out), p(scores), C.byref(k), C.byref(ran))
        ctx.check(rc, "b2_debug_lightglue_assign_host")
        stats = dict(rmax=rs[0], rlog=rs[1], lsg0=rs[2], cmax=cs[0], clog=cs[1], lsg1=cs[2])
    assert 0 <= k.value <= M
    return dict(stats, best0=best0, arg0=arg0, arg1=arg1, matches=out[:k.value].copy(), scores=scores[:k.value].copy(), path=ran.value)


# ---- the fp64 reference and its bounds -----------------------------------------------------------------------------------

def reference(kind, case, alpha=1.0, iters=20, Z=None):
    Z = case["Z"] if Z is None else Z
    M, N = Z.shape
    if kind == "sg":
        S, u, v, ar, ac = assign_ref.log_optimal_transport(Z.astype(np.float64), alpha, iters)
        S = S[:M, :N]
        d_row, d_col = chains(kind, M, N, case["G"])
        er, ec = e_lse(d_row, ar), e_lse(d_col, ac)
        eps_u, eps_v = iters * er + max(iters - 1, 0) * ec, iters * (er + ec)
        rnd = 4 * U * (np.abs(Z).max() + np.abs(u).max() + np.abs(v).max() + np.log(M + N))
        ref = dict(S=S, u=u, v=v, eps_u=eps_u, eps_v=eps_v, row_b=eps_v + rnd, col_b=eps_u + rnd, score_b=eps_u + eps_v + rnd)
    else:
        S, lr, lc = assign_ref.double_log_softmax(Z, case["z0"], case["z1"])
        l0, l1 = assign_ref.logsigmoid(case["z0"]), assign_ref.logsigmoid(case["z1"])
        rmax, cmax = Z.max(1), Z.max(0)
        d_row, d_col = chains(kind, M, N, case["G"])
        er = e_lse(d_row, np.abs(Z - rmax[:, None]).max())
        ec = e_lse(d_col, np.abs(Z - cmax[None, :]).max())
        e0, e1 = 4 * U * np.abs(l0).max(), 4 * U * np.abs(l1).max()  # 2 ulp
        rnd = 8 * U * (2 * np.abs(Z).max() + np.abs(rmax).max() + np.abs(lr - rmax).max() + np.abs(cmax).max() + np.abs(lc - cmax).max()
                       + np.abs(l0).max() + np.abs(l1).max())
        ref = dict(S=S, lr=lr, lc=lc, l0=l0, l1=l1, er=er, ec=ec, row_b=ec + e1 + rnd, col_b=er + e0 + rnd, score_b=er + ec + e0 + e1 + rnd)
    ref["a0"], ref["a1"] = S.argmax(1), S.argmax(0)  # the first maximum, like torch.max
    ref["best"] = S[np.arange(M), ref["a0"]]
    # top-two margins over distinct columns / rows: a duplicate of the maximum ties exactly and is checked on its own
    Sr = S.copy()
    Sr[:, list(case["col_dup"])] = -np.inf
    Sc = S.copy()
    Sc[list(case["row_dup"]), :] = -np.inf
    ref["row_margin"] = margin(Sr, 1)
    ref["col_margin"] = margin(Sc, 0)
    return ref


def margin(S, axis):
    if S.shape[axis] < 2:
        return np.full(S.shape[1 - axis], np.inf)
    top = -np.partition(-S, 1, axis=axis)
    t0, t1 = np.take(top, 0, axis), np.take(top, 1, axis)
    return np.where(np.isfinite(t1), t0 - t1, np.inf)


# ---- the checks ------------------------------------------------------------------------------------------------------------

def check_stats(kind, case, ref, out):
    if kind == "sg":
        assert np.isfinite(out["u"]).all() and np.isfinite(out["v"]).all()
        du, dv = np.abs(out["u"] - ref["u"]).max(), np.abs(out["v"] - ref["v"]).max()
        assert du <= ref["eps_u"] and dv <= ref["eps_v"], (du, ref["eps_u"], dv, ref["eps_v"])
    else:
        Z = case["Z"]
        assert np.array_equal(out["rmax"], Z.max(1)) and np.array_equal(out["cmax"], Z.max(0)), "max is exact"
        # fminf(z, 0) - log1pf(expf(-|z|)): CUDA documents expf to 2 ulp and log1pf to 1 ulp, and the difference rounds once
        for got, z in ((out["lsg0"], case["z0"]), (out["lsg1"], case["z1"])):
            want = assign_ref.logsigmoid(z)
            ulps = np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32))
            assert ulps.max() <= 4, ("logsigmoid within 4 ulp", float(ulps.max()))
        dr = np.abs(out["rlog"] - (ref["lr"] - out["rmax"])).max()
        dc = np.abs(out["clog"] - (ref["lc"] - out["cmax"])).max()
        assert dr <= ref["er"] and dc <= ref["ec"], (dr, ref["er"], dc, ref["ec"])
    db = np.abs(out["best0"] - ref["best"]).max()
    assert db <= ref["score_b"], (db, ref["score_b"])


def ambiguous(ref):
    return ref["row_margin"] <= 2 * ref["row_b"], ref["col_margin"] <= 2 * ref["col_b"]


def check_argmax(kind, case, ref, out):
    S = ref["S"]
    M, N = S.shape
    amb_r, amb_c = ambiguous(ref)
    assert amb_r.sum() + amb_c.sum() < 0.01 * (M + N), ("too many ambiguous rows / columns", amb_r.sum(), amb_c.sum())
    a0, a1 = out["arg0"], out["arg1"]
    assert ((a0 >= 0) & (a0 < N)).all() and ((a1 >= 0) & (a1 < M)).all()
    bad = np.nonzero(~amb_r & (a0 != ref["a0"]))[0]
    assert len(bad) == 0, ("row arg-max", bad[:10], a0[bad[:10]], ref["a0"][bad[:10]])
    bad = np.nonzero(~amb_c & (a1 != ref["a1"]))[0]
    assert len(bad) == 0, ("column arg-max", bad[:10], a1[bad[:10]], ref["a1"][bad[:10]])
    i = np.nonzero(amb_r)[0]
    assert (S[i, a0[i]] >= ref["best"][i] - 2 * ref["row_b"]).all()
    j = np.nonzero(amb_c)[0]
    assert (S[a1[j], j] >= S[ref["a1"][j], j] - 2 * ref["col_b"]).all()
    for i, j in case["plant"]:  # every planted edge: exact, with a margin of at least 1.0
        assert ref["row_margin"][i] >= 1.0 and ref["col_margin"][j] >= 1.0, ("planted margin", i, j)
        assert a0[i] == j and a1[j] == i, ("planted edge", i, j, a0[i], a1[j])
    for r, js, jd in case["col_ties"]:  # duplicated columns: the first one wins the row
        assert a0[r] == js, ("tie between columns", js, jd, "row", r, "picked", a0[r])
    for rs, rd, c in case["row_ties"]:  # duplicated rows: the first one wins the column, the second is not mutual
        assert a1[c] == rs and a0[rd] == c, ("tie between rows", rs, rd, "column", c, "picked", a1[c])


def check_matches(kind, case, ref, out):
    S = ref["S"]
    M = S.shape[0]
    th = LOG_TH[kind]
    rows, cols, sc = assign_ref.mutual_filter(S, th)
    amb_r, amb_c = ambiguous(ref)
    skip = amb_r | amb_c[ref["a0"]] | (np.abs(ref["best"] - np.log(th)) <= ref["score_b"])
    ind0 = np.arange(M) if case["ind0"] is None else case["ind0"]
    ind1 = np.arange(S.shape[1]) if case["ind1"] is None else case["ind1"]
    m = out["matches"].astype(np.int64)
    assert (np.diff(m[:, 0]) > 0).all(), "match rows ascend"
    pos = np.searchsorted(ind0, m[:, 0])  # back to row indices (ind0 increases)
    assert (pos < M).all() and np.array_equal(ind0[np.minimum(pos, M - 1)], m[:, 0])
    keep = ~skip[pos]
    want_keep = ~skip[rows]
    want = np.stack([ind0[rows], ind1[cols]], 1)[want_keep]
    assert np.array_equal(m[keep], want), ("match list", len(m[keep]), len(want))
    for rs, rd, c in case["row_ties"]:
        assert ind0[rd] not in m[:, 0], ("duplicated row matched", rd)
    e = np.exp(ref["best"][pos])
    assert (np.abs(out["scores"] - e) <= e * np.expm1(ref["score_b"]) + 4 * U).all()
    assert skip.sum() <= 0.02 * M + 2


def check_bites(kind, case, ref, alpha, iters):
    Z16 = case["Z"].astype(np.float16).astype(np.float32)
    r16 = reference(kind, case, alpha, iters, Z=Z16)
    worst = np.abs(r16["best"] - ref["best"]).max() / ref["score_b"]
    if kind == "sg" and iters > 0:
        worst = max(worst, np.abs(r16["u"] - ref["u"]).max() / ref["eps_u"], np.abs(r16["v"] - ref["v"]).max() / ref["eps_v"])
    if kind == "lg":
        worst = max(worst, np.abs(r16["lr"] - ref["lr"]).max() / ref["er"], np.abs(r16["lc"] - ref["lc"]).max() / ref["ec"])
    assert worst > 1.0, "the bound does not tell fp32 from fp16 scores in this case"


def same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a if k != "path")


# ---- cases -----------------------------------------------------------------------------------------------------------------

def _cases():
    c = []
    add = lambda name, M, N, kinds=("sg", "lg"), **kw: c.extend(pytest.param(k, M, N, kw, id=f"{k}-{name}") for k in kinds)
    add("1x1", 1, 1)
    add("1x5000", 1, 5000)
    add("5000x1", 5000, 1)
    add("40x3", 40, 3)  # the superglue_9 shape: most CTAs own no rows
    add("3x700", 3, 700)  # rows_per = 1: one ring step, the prologue commits empty groups
    add("257x1000-G2", 257, 1000, G=2)  # 129 rows per CTA: the last ring step holds one row
    for n in (1022, 1023, 1024, 1025, 2047, 2048):  # the last column of a thread slot, with and without the dustbin
        add(f"300x{n}", 300, n)
    add("300x8191", 300, 8191, kinds=("sg",))  # N + 1 = 8192 fills every slot
    add("300x8192", 300, 8192, kinds=("sg",))
    add("300x6240", 300, 6240, kinds=("lg",))
    add("300x6241", 300, 6241, kinds=("lg",))
    for g in ("1", "7", "sm-4", "sm"):
        add(f"600x1500-G{g}", 600, 1500, G=g)
    add("37x1000", 37, 1000)
    add("100x37", 100, 37)
    add("5000x5000", 5000, 5000, values="sharp")
    add("5000x5000-soft", 5000, 5000, kinds=("lg",))
    add("8000x300", 8000, 300)
    add("257x1000-it0", 257, 1000, kinds=("sg",), iters=0)
    add("257x1000-it1", 257, 1000, kinds=("sg",), iters=1)
    add("300x300-it100", 300, 300, kinds=("sg",), iters=100, values="sharp")
    add("2048x2000-it100", 2048, 2000, kinds=("sg",), iters=100, values="sharp")
    for a in (-5.0, 8.0):
        add(f"600x1500-alpha{a:g}", 600, 1500, kinds=("sg",), alpha=a)
    add("600x1500-z30", 600, 1500, kinds=("lg",), z_tail=True)
    add("3000x2500-filter", 3000, 2500, values="sharp", ind=True)
    return c


@pytest.mark.parametrize("kind,M,N,kw", _cases())
def test_assign_matches_fp64(b200_ctx, kind, M, N, kw):
    kw = dict(kw)
    alpha, iters = kw.pop("alpha", 1.0), kw.pop("iters", 20)
    g = kw.pop("G", "sm")
    sms = sm_count()
    G = {"sm": sms, "sm-4": sms - 4}.get(g, None) or int(g)
    case = make_case(kind, M, N, G, values=kw.get("values", "soft"), z_tail=kw.get("z_tail", False), ind=kw.get("ind", False))
    if kind == "sg":
        case["ind0"] = case["ind1"] = None
    ref = reference(kind, case, alpha, iters)
    check_bites(kind, case, ref, alpha, iters)
    paths = [1, 2] if fits(kind, N) else [2]
    outs = {}
    for path in paths:
        out = run_kernel(b200_ctx, kind, case, path, alpha, iters)
        assert out["path"] == path
        assert same(out, run_kernel(b200_ctx, kind, case, path, alpha, iters)), f"path {path} is not deterministic"
        check_stats(kind, case, ref, out)
        check_argmax(kind, case, ref, out)
        check_matches(kind, case, ref, out)
        outs[path] = out
    auto = run_kernel(b200_ctx, kind, case, 0, alpha, iters)
    assert auto["path"] == (1 if fits(kind, N) else 2), f"the matcher ran path {auto['path']} at N = {N}"
    assert same(auto, outs[auto["path"]])
    if len(outs) == 2:  # the two paths agree with each other
        amb_r, amb_c = ambiguous(ref)
        assert np.array_equal(outs[1]["arg0"][~amb_r], outs[2]["arg0"][~amb_r])
        assert np.array_equal(outs[1]["arg1"][~amb_c], outs[2]["arg1"][~amb_c])
        keys = ("u", "v") if kind == "sg" else ("rlog", "clog")
        bounds = (ref["eps_u"], ref["eps_v"]) if kind == "sg" else (ref["er"], ref["ec"])
        for k, b in zip(keys, bounds):
            assert np.abs(outs[1][k] - outs[2][k]).max() <= 2 * b, k


def test_persistent_path_refuses_too_many_columns(b200_ctx):
    """Forcing the persistent kernel past its column limit is an argument error, not a silent switch of path."""
    M, N = 4, 8192
    Z = np.zeros((M, N), np.float32)
    f = np.zeros(N + 1, np.float32)
    i = np.zeros(N + 1, np.int32)
    k, ran = C.c_int(0), C.c_int(0)
    p = _lib.ptr
    rc = b200_ctx.lib.b2_debug_superglue_assign_host(b200_ctx.handle, 1, 0, p(Z), M, N, 1.0, 1, 0.2, p(f), p(f), p(f), p(i), p(i),
                                                     p(np.zeros((M, 2), np.uint32)), p(f), C.byref(k), C.byref(ran))
    assert rc == -2
