"""GPU: the RANSAC verifier's kernels (gtsfm_b200/csrc/ransac.cu) stage by stage against the fp64 NumPy restatement in
oracle/ransac_ref.py, through the test-only trace entry point b2_debug_ransac_trace_host.

The verifier is fp64, deterministic for a seed and reduces in a fixed order, so the replay is exact where the stage is
discrete (samples, selections, batch counts, flags, masks away from the threshold, vote winners) and bounded where an
eigen-solver or a summation order differs.  Every fixture is generated from a seed."""
import ctypes

import numpy as np
import pytest

from gtsfm_b200 import _lib
from oracle import ransac_ref as rr
from oracle import verifier_ref as vr

pytestmark = pytest.mark.gpu

EPS = np.finfo(float).eps
SEED = 0x5EED
CONF = 0.999999
NEAR = 1e-9  # relative margin around thr^2 inside which an inlier decision may differ between two correct evaluations


def scene(k, ratio, seed=1, mode=0, noise=0.5):
    kp1, kp2, _, K, R, t, is_in = vr.synthetic_two_view(seed, k, ratio, noise_px=noise)
    if mode == 0:
        return np.ascontiguousarray(vr.calibrate(kp1, *K)), np.ascontiguousarray(vr.calibrate(kp2, *K)), 4.0 / K[0], (R, t)
    return np.ascontiguousarray(kp1), np.ascontiguousarray(kp2), 4.0, (R, t)


class Trace:
    """One b2_debug_ransac_trace_host call and its host buffers."""

    def __init__(self, ctx, mode, x1, x2, thr, max_iters, batch, records=1, seed=SEED, models=True):
        k = len(x1)
        self.mode, self.k, self.thr2, self.batch, self.max_iters = mode, k, thr * thr, batch, max_iters
        self.x1, self.x2 = x1, x2
        self.nsol = np.zeros((records, batch), np.int32)
        self.models = np.zeros((records, batch * rr.MAX_SOL, 9)) if models else None
        self.cost = np.zeros((records, batch * rr.MAX_SOL))
        self.ninl = np.zeros((records, batch * rr.MAX_SOL), np.int32)
        self.sel = (_lib.RansacCandidate * (8 * max(records, 1)))()
        self.more = np.zeros(max(records, 1), np.int32)
        tr = _lib.RansacTrace()
        tr.batch, tr.max_records = batch, records
        tr.nsol, tr.models, tr.cost, tr.ninl = (_lib.ptr(self.nsol).value, _lib.ptr(self.models).value if models else None,
                                                _lib.ptr(self.cost).value, _lib.ptr(self.ninl).value)
        tr.selected, tr.more = ctypes.addressof(self.sel), _lib.ptr(self.more).value
        self.model, self.R, self.t = np.zeros(9), np.zeros(9), np.zeros(3)
        self.mask = np.zeros(max(k, 1), np.uint8)
        n = ctypes.c_int(0)
        prm = _lib.RansacParams(thr, CONF, max_iters, seed)
        self.rc = ctx.lib.b2_debug_ransac_trace_host(ctx.handle, mode, _lib.ptr(x1), _lib.ptr(x2), k, ctypes.byref(prm), ctypes.byref(tr),
                                                     _lib.ptr(self.model), _lib.ptr(self.mask), ctypes.byref(n), _lib.ptr(self.R), _lib.ptr(self.t))
        ctx.check(self.rc, "debug_ransac_trace")
        self.tr, self.num_inliers, self.mask = tr, n.value, self.mask[:k]

    def samples(self, r):
        """number of samples of record r (a sampling batch, or the extension after the last batch)"""
        if r < self.tr.batches:
            hard = 65536 if self.mode == 0 else 262144
            return min(self.batch, min(self.max_iters, hard) - r * self.batch)
        return min(4 * self.max_iters, self.batch)

    def selected(self, r):
        return [cand(self.sel[r * 8 + j]) for j in range(8)]


def cand(c):
    return rr.Candidate(np.array(c.model[:]), c.cost, c.ninl, bool(c.valid))


def same_cands(a, b):
    """bit-identical candidate lists (models, costs, counts, validity)"""
    for x, y in zip(a, b):
        assert x.valid == y.valid
        if x.valid:
            assert np.array_equal(x.model, y.model) and x.cost == y.cost and x.ninl == y.ninl


def err_bound(mode, M, x1, x2):
    """per-point relative bound of the error: the residual x2^T M x1 (9 products) is good to 9 eps T, T = |x2|^T |M| |x1|;
    squared and divided by a few-eps denominator: 18 eps T / |r| + 8 eps."""
    h1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    h2 = np.concatenate([x2, np.ones((len(x2), 1))], 1)
    M3 = np.asarray(M).reshape(3, 3)
    T = np.einsum("ki,ij,kj->k", np.abs(h2), np.abs(M3), np.abs(h1))
    r = np.abs(np.einsum("ki,ij,kj->k", h2, M3, h1))
    return 18 * EPS * T / np.maximum(r, 1e-300) + 8 * EPS


def score_check(mode, M, x1, x2, thr2, cost_dev, ninl_dev):
    """MSAC cost / count of model M: count exact away from thr2's margin, cost within the summation and evaluation bound.
    -> (number of near-threshold points, cost error / bound)"""
    e = rr.error(mode, M, x1, x2)
    near = np.abs(e - thr2) <= NEAR * thr2
    c_ref, n_ref = rr.msac(e, thr2)
    assert abs(ninl_dev - n_ref) <= near.sum()
    if not near.any():
        assert ninl_dev == n_ref
    # k-term sum in another order: k eps sum|terms|; each inlier term e_i good to e_i * rel_i; a near point may flip by thr2
    bound = len(e) * EPS * c_ref + np.sum(np.where(e < thr2, e * err_bound(mode, M, x1, x2), 0.0)) + near.sum() * thr2 + 1e-300
    assert abs(cost_dev - c_ref) <= bound, (cost_dev, c_ref, bound)
    return int(near.sum()), abs(cost_dev - c_ref) / bound


# ---- hypotheses ---------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return rr.build_shim(tmp_path_factory.mktemp("shim"))


def test_hypotheses_E_sampler_and_solver(b200_ctx, shim):
    """Every device E of each replayed 5-sample satisfies its constraints, has unit norm and the cubic identity; the true E
    is among the solutions on a noiseless all-inlier scene; the solution count equals the host build's."""
    x1, x2, thr, (R, t) = scene(300, 1.0, seed=11, noise=0.0)
    n = 2000
    tr = Trace(b200_ctx, 0, x1, x2, thr, n, n)
    idx = rr.sample_distinct(SEED, np.arange(n, dtype=np.uint64), len(x1), 5)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    Et = (tx @ R) / np.linalg.norm(tx @ R)
    found, mism, worst = 0, 0, np.zeros(3)
    for s in range(n):
        a, b = x1[idx[s]], x2[idx[s]]
        ns = int(tr.nsol[0, s])
        E = tr.models[0, s * 10:s * 10 + ns]
        h = np.zeros((10, 9))
        mism += shim.shim_fivept(_lib.ptr(np.ascontiguousarray(a)), _lib.ptr(np.ascontiguousarray(b)), _lib.ptr(h)) != ns
        for e in E:
            con = np.abs(np.einsum("ki,ij,kj->k", np.c_[b, np.ones(5)], e.reshape(3, 3), np.c_[a, np.ones(5)])).max()
            dn, cub = rr.essential_residuals(e)
            worst = np.maximum(worst, [con, dn, cub])
        if ns and min(min(np.abs(e - Et.ravel()).max(), np.abs(e + Et.ravel()).max()) for e in E) < 1e-6:
            found += 1
    print(f"E hypotheses: constraint / norm / cubic worst {worst}, true E found {found}/{n}, count mismatches vs host {mism}/{n}")
    # Measured on an H100: constraints 5e-16, norm 3e-16, cubic identity 5e-6 (a root of the degree-10 polynomial found by
    # bisection on a poorly conditioned sample), true E in 1929 / 2000 samples.  The host build gives the same counts, and
    # holds the shipped QR null-space variant to the same 95 % (tests/test_ransac_math_cpu.py).
    assert worst[0] < 1e-12 and worst[1] < 1e-12 and worst[2] < 1e-4, worst
    assert found >= 0.95 * n
    assert mism <= 0.001 * n


def test_hypotheses_F_against_numpy_8pt(b200_ctx):
    """Device F = the NumPy normalised 8-point F of the same sample, up to sign."""
    x1, x2, thr, _ = scene(400, 0.6, seed=12, mode=1)
    n = 1000
    tr = Trace(b200_ctx, 1, x1, x2, thr, n, n)
    idx = rr.sample_distinct(SEED, np.arange(n, dtype=np.uint64), len(x1), 8)
    worst = 0.0
    for s in range(n):
        assert tr.nsol[0, s] == 1
        F = tr.models[0, s * 10]
        Fr = rr.eightpt(x1[idx[s]], x2[idx[s]]).ravel()
        worst = max(worst, min(np.abs(F - Fr).max(), np.abs(F + Fr).max()))
    print(f"F hypotheses: worst |F_dev -+ F_numpy| {worst:.2e} (bound 1e-8)")
    # Jacobi (stops at off-diagonal mass 1e-30 of the diagonal) against LAPACK on 9 x 9 moment matrices of pixel data
    assert worst < 1e-8


def test_degenerate_samples_have_no_solution(b200_ctx):
    """Coincident points: every 8-sample is degenerate, nsol = 0, and the call reports that no model was found."""
    x1, x2 = np.tile([[640.0, 480.0]], (20, 1)), np.tile([[320.0, 240.0]], (20, 1))
    tr = Trace(b200_ctx, 1, x1, x2, 1e-3, 200, 200)
    assert np.all(tr.nsol[0] == 0) and tr.rc == 1 and tr.num_inliers == 0 and not tr.mask.any()


# ---- scoring ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("k", [5, 8, 127, 128, 129, 255, 256, 257, 4096, 70000])
def test_scoring(b200_ctx, mode, k):
    """cost / ninl of every slot recomputed in fp64 on the device's own models."""
    x1, x2, thr, _ = scene(k, 0.5, seed=20 + k % 7, mode=mode)
    n = 16 if k >= 4096 else 64
    tr = Trace(b200_ctx, mode, x1, x2, thr, n, n)
    if k < (5 if mode == 0 else 8):
        assert tr.rc == 1 and tr.tr.records == 0
        return
    near, worst = 0, 0.0
    for s in range(n):
        for j in range(10):
            slot = s * 10 + j
            if j >= tr.nsol[0, s]:
                assert tr.cost[0, slot] == 1e300 and tr.ninl[0, slot] == 0
                continue
            nr, ratio = score_check(mode, tr.models[0, slot], x1, x2, tr.thr2, tr.cost[0, slot], tr.ninl[0, slot])
            near, worst = near + nr, max(worst, ratio)
    print(f"scoring mode {mode} k {k}: worst cost error / bound {worst:.3f}, near-threshold points {near}")
    assert near <= max(1, 1e-4 * k * n)


# ---- selection ----------------------------------------------------------------------------------------------------

def replay_selection(tr):
    """Replay every recorded k_rs_select on the device's own costs and models; -> the replayed final list."""
    m = 5 if tr.mode == 0 else 8
    cands, done = [rr.invalid()] * 8, 0
    for r in range(tr.tr.records):
        n = tr.samples(r)
        cands = rr.select(cands, tr.models[r, :n * 10], tr.cost[r, :n * 10], tr.ninl[r, :n * 10])
        same_cands(tr.selected(r), cands)
        if r < tr.tr.batches:
            done += n
            assert tr.more[r] == rr.more_flag(cands[0], tr.k, m, CONF, done)
        else:
            assert tr.more[r] == -1
    return cands


def check_schedule(tr):
    m = 5 if tr.mode == 0 else 8
    sched = rr.schedule(tr.mode, tr.max_iters, tr.batch,
                        lambda b: tr.selected(b)[0].ninl if tr.selected(b)[0].valid else None, tr.k, CONF)
    assert tr.tr.batches == len(sched.batches)
    if sched.extension:
        assert tr.tr.ext_go == tr.more[tr.tr.batches - 1] == rr.more_flag(tr.selected(tr.tr.batches - 1)[0], tr.k, m, CONF, tr.max_iters)
    else:
        assert tr.tr.ext_go == -1
    return sched


def test_selection_all_ties_across_batches(b200_ctx):
    """Threshold 0, so every point is an outlier (a sample's own points can have a Sampson error of exactly 0, so no
    positive threshold is safe): every slot costs k * 0.  The candidates are the 8 lowest non-empty slots of the first
    batch and stay so across the 5 batches (earlier wins)."""
    x1, x2, _, _ = scene(300, 0.5, seed=30)
    tr = Trace(b200_ctx, 0, x1, x2, 0.0, 5000, 1000, records=5)
    live = tr.cost[0] < 1e299
    assert len(set(tr.cost[:, :][tr.cost < 1e299].tolist())) == 1
    first8 = np.flatnonzero(live)[:8]
    want = [rr.Candidate(tr.models[0, i], tr.cost[0, i], 0) for i in first8]
    for r in range(5):
        same_cands(tr.selected(r), want)
    replay_selection(tr)
    assert tr.tr.batches == 5 and tr.tr.ext_go == -1 and list(tr.more) == [1] * 5
    check_schedule(tr)


@pytest.mark.parametrize("mode,ratio,max_iters,batch,want_batches", [
    (0, 0.3, 5000, 1000, (5, 5)),  # the whole budget in 5 batches
    (0, 0.36, 5000, 1000, (2, 4)),  # the bound is met between batches
    (1, 0.8, 5000, 1000, (1, 1)),  # met after the first batch
])
def test_selection_multi_batch_and_stop(b200_ctx, mode, ratio, max_iters, batch, want_batches):
    x1, x2, thr, _ = scene(500, ratio, seed=31, mode=mode)
    tr = Trace(b200_ctx, mode, x1, x2, thr, max_iters, batch, records=6)
    replay_selection(tr)
    check_schedule(tr)
    same_cands(tr.selected(tr.tr.records - 1), [cand(c) for c in tr.tr.prerefine])
    assert want_batches[0] <= tr.tr.batches <= want_batches[1], tr.tr.batches


@pytest.mark.parametrize("max_iters,ratio,ext", [(4096, 0.3, 1), (4097, 0.3, -1), (1000, 0.8, 0)])
def test_extension_stage(b200_ctx, max_iters, ratio, ext):
    """E extension: enqueued only with max_iters <= 4096; runs (and is replayed) when the bound says the budget fell short."""
    x1, x2, thr, _ = scene(500, ratio, seed=32)
    tr = Trace(b200_ctx, 0, x1, x2, thr, max_iters, 16384, records=2)
    assert tr.tr.ext_go == ext and tr.tr.batches == 1
    sched = check_schedule(tr)
    assert sched.extension == (0 if ext == -1 else min(4 * max_iters, 16384))
    assert tr.tr.records == (2 if ext == 1 else 1)
    final = replay_selection(tr)
    same_cands([cand(c) for c in tr.tr.prerefine], final)


# ---- refinement, pick, mask, pose -----------------------------------------------------------------------------------

REFINE_BOUND = 1e-7  # |refined_dev -+ refined_numpy|: two eigen-solvers (Jacobi to 1e-26 / LAPACK) on normal equations


@pytest.mark.parametrize("mode,k,ratio", [(0, 32768, 0.5), (0, 32769, 0.5), (0, 70000, 0.5), (0, 40000, 0.3), (1, 32769, 0.5),
                                          (0, 1001, 0.6), (1, 5003, 0.6)])
def test_refine_pick_mask_pose(b200_ctx, mode, k, ratio):
    """Local optimisation replayed from the device's pre-refine candidates (k > 32768 runs the flag-word fallback), then
    the pick, the mask / count and, for E, the cheirality vote of the device's own four decompositions."""
    x1, x2, thr, _ = scene(k, ratio, seed=40 + k % 11, mode=mode)
    tr = Trace(b200_ctx, mode, x1, x2, thr, 200, 200, records=0, models=False)
    pre, ref = [cand(c) for c in tr.tr.prerefine], [cand(c) for c in tr.tr.refined]
    worst_m, worst_c, near = 0.0, 0.0, 0
    for p, d in zip(pre, ref):
        assert p.valid == d.valid
        if not d.valid:
            continue
        assert d.cost <= p.cost
        r = rr.refine(mode, x1, x2, tr.thr2, p)
        worst_m = max(worst_m, min(np.abs(d.model - r.model).max(), np.abs(d.model + r.model).max()))
        if d.cost < p.cost:  # a refit was accepted: the stored cost / count are the refit's MSAC score
            nr, ratio_c = score_check(mode, d.model, x1, x2, tr.thr2, d.cost, d.ninl)
            near, worst_c = near + nr, max(worst_c, ratio_c)
        else:
            assert np.array_equal(d.model, p.model) and d.ninl == p.ninl
    print(f"refine mode {mode} k {k}: worst model difference {worst_m:.2e} (bound {REFINE_BOUND}), cost error / bound "
          f"{worst_c:.3f}, near-threshold points {near}")
    assert worst_m < REFINE_BOUND
    # pick: lowest refined cost, ties to the lower rank
    b = rr.pick(ref)
    same_cands([cand(tr.tr.pick)], [ref[b]])
    assert np.array_equal(tr.model, ref[b].model)
    # mask: err < thr2 under the final model, exactly away from the margin; the count is the mask's sum
    e = rr.error(mode, tr.model, x1, x2)
    away = np.abs(e - tr.thr2) > NEAR * tr.thr2
    assert np.array_equal(tr.mask.astype(bool)[away], (e < tr.thr2)[away])
    assert tr.tr.mask_count == tr.num_inliers == int(tr.mask.sum())
    if mode == 0:
        inl = tr.mask.astype(bool)
        v, amb = rr.votes(np.array(tr.tr.pose_cands[:]), x1[inl], x2[inl])
        dev = np.array(tr.tr.votes[:])
        assert np.all(np.abs(dev - v) <= amb), (dev, v, amb)
        assert tr.tr.winner == rr.vote_winner(dev)
        c = np.array(tr.tr.pose_cands[:])
        R, sg = (c[9:18] if tr.tr.winner & 1 else c[:9]), (-1.0 if tr.tr.winner & 2 else 1.0)
        assert np.array_equal(tr.R, R) and np.array_equal(tr.t, sg * c[18:21])


def recover_pose_debug(ctx, E, x1, x2):
    cands, votes, win = np.zeros(21), np.zeros(4, np.int32), ctypes.c_int(-1)
    R, t, good = np.zeros(9), np.zeros(3), ctypes.c_int(0)
    k = len(x1)
    rc = ctx.lib.b2_debug_recover_pose_host(ctx.handle, _lib.ptr(np.ascontiguousarray(E)), _lib.ptr(x1) if k else None,
                                            _lib.ptr(x2) if k else None, k, _lib.ptr(cands), _lib.ptr(votes), ctypes.byref(win),
                                            _lib.ptr(R), _lib.ptr(t), ctypes.byref(good))
    ctx.check(rc, "debug_recover_pose")
    return cands, votes, win.value, R, t, good.value


@pytest.mark.parametrize("k", [0, 1, 127, 128, 129, 5000])
def test_pose_votes(b200_ctx, k):
    """Vote totals of the device's four decompositions equal the NumPy cheirality votes; the winner is the first maximum
    in the order (R1,t), (R2,t), (R1,-t), (R2,-t) (k = 0: all tied, (R1,t) wins); k > 128 spans several CTAs."""
    x1, x2, _, (R, t) = scene(max(k, 1), 1.0, seed=50)
    x1, x2 = x1[:k], x2[:k]
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    E = (tx @ R).ravel() / np.linalg.norm(tx @ R)
    cands, dev, win, Rd, td, good = recover_pose_debug(b200_ctx, E, np.ascontiguousarray(x1), np.ascontiguousarray(x2))
    v, amb = rr.votes(cands, x1, x2)
    assert np.all(np.abs(dev - v) <= amb), (dev, v, amb)
    assert win == rr.vote_winner(dev) and good == dev[win]
    if k == 0:
        assert list(dev) == [0, 0, 0, 0] and win == 0
    R1, R2, tt = cands[:9], cands[9:18], cands[18:]
    assert np.array_equal(Rd, R2 if win & 1 else R1) and np.array_equal(td, -tt if win & 2 else tt)
    if k >= 127:
        assert vr.rot_angle_deg(R, Rd.reshape(3, 3)) < 1e-4 and vr.dir_angle_deg(t, td) < 1e-4  # 0.5 px noise


# ---- contracts ----------------------------------------------------------------------------------------------------

def test_dev_path_bit_identical_to_host_path(b200_ctx):
    """b2_ransac_essential_dev (gather + the caller's stream) = b2_ransac_essential_host on the same calibrated input, bit
    for bit, on a user stream and on the null stream; two calls and two contexts agree exactly."""
    import torch

    from gtsfm_b200.verifier import RansacEngine

    kp1, kp2, _, K, *_ = vr.synthetic_two_view(60, 3001, 0.4)
    kp1f, kp2f = kp1.astype(np.float32), kp2.astype(np.float32)
    rng = np.random.default_rng(60)
    matches = np.stack([rng.permutation(3001), rng.permutation(3001)], 1).astype(np.int64)[:2500]
    cal = np.array([K[0], K[1], K[2]])
    x1 = (kp1f[matches[:, 0]].astype(np.float64) - cal[1:]) / cal[0]
    x2 = (kp2f[matches[:, 1]].astype(np.float64) - cal[1:]) / cal[0]
    thr = 4.0 / K[0]
    eng = RansacEngine(ctx=b200_ctx)
    E_h, mask_h, R_h, t_h = eng.essential(x1, x2, thr)
    dev = torch.device("cuda:0")
    d_kp1, d_kp2, d_m = torch.from_numpy(kp1f).to(dev), torch.from_numpy(kp2f).to(dev), torch.from_numpy(matches).to(dev)
    for stream in (torch.cuda.Stream(), None):
        d_mask = torch.full((len(matches),), 7, dtype=torch.uint8, device=dev)
        E, R, t, n = np.zeros(9), np.zeros(9), np.zeros(3), ctypes.c_int(0)
        prm = _lib.RansacParams(thr, CONF, 1000, 0x5EED)
        rc = b200_ctx.lib.b2_ransac_essential_dev(b200_ctx.handle, _lib.ptr(d_kp1), _lib.ptr(d_kp2), _lib.ptr(d_m), len(matches),
                                                  _lib.ptr(cal), _lib.ptr(cal), ctypes.byref(prm), _lib.ptr(E), _lib.ptr(d_mask),
                                                  ctypes.byref(n), _lib.ptr(R), _lib.ptr(t),
                                                  _lib.ptr(stream.cuda_stream if stream is not None else 0))
        b200_ctx.check(rc, "ransac_essential_dev")
        torch.cuda.synchronize()
        assert rc == 0 and np.array_equal(E, E_h.ravel()) and np.array_equal(R, R_h.ravel()) and np.array_equal(t, t_h)
        assert np.array_equal(d_mask.cpu().numpy(), mask_h) and n.value == int(mask_h.sum())
    again = eng.essential(x1, x2, thr)
    other = _lib.Context(0)
    try:
        third = RansacEngine(ctx=other).essential(x1, x2, thr)
    finally:
        other.close()
    for res in (again, third):
        assert all(np.array_equal(a, b) for a, b in zip(res, (E_h, mask_h, R_h, t_h)))


def test_zero_inlier_result(b200_ctx):
    """No hypothesis with an inlier (threshold 0): the best candidate is still a model, so the verifier returns a pose
    with no inlier rows and ratio 0.  The reference path does not return its failure tuple here either: cv2 finds no
    inliers and its recoverPose then rejects the empty point set, so there is no failure result to copy."""
    import cv2

    from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
    from gtsfm_b200.verifier import B200Ransac

    kp1, kp2, matches, K, *_ = vr.synthetic_two_view(70, 300, 0.5)
    x1, x2 = np.ascontiguousarray(vr.calibrate(kp1, *K)), np.ascontiguousarray(vr.calibrate(kp2, *K))
    tr = Trace(b200_ctx, 0, x1, x2, 0.0, 1000, 1000)
    assert tr.rc == 0 and tr.num_inliers == 0 and tr.tr.mask_count == 0 and not tr.mask.any()
    assert tr.tr.pick.valid == 1 and tr.tr.pick.ninl == 0
    cal = Cal3Bundler(K[0], 0, 0, K[1], K[2])
    R, U, rows, ratio = B200Ransac(True, 0.0).verify(Keypoints(kp1), Keypoints(kp2), matches, cal, cal)
    assert R is not None and U is not None and rows.shape == (0, 2) and ratio == 0.0
    with pytest.raises(cv2.error):
        vr.verify_cv2(kp1, kp2, matches, K, K, True, 0.0)
