"""LMedS verifier on the device (csrc/lmeds.cu): stage by stage against oracle/lmeds_ref.py through the trace entry, end to
end against cv2's golden results (tests/golden/lmeds_scenes.npz, written by oracle/make_golden_lmeds.py), batching, the
plugin, and the launches and synchronisations of one call."""
import ctypes
from pathlib import Path

import numpy as np
import pytest

from gtsfm_b200 import _lib
from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
from gtsfm_b200.verifier import B200LMEDS, lmeds_params, lmeds_verify_batched_dev, ransac_problem
from oracle import lmeds_ref as lr
from oracle import verifier_ref as vr

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "lmeds_scenes.npz"


@pytest.fixture(scope="module")
def ctx():
    return _lib.Context(0)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return lr.build_shim(tmp_path_factory.mktemp("lmeds_shim"))


def _golden():
    g = np.load(GOLDEN)
    return [{k: g[f"s{i}_{k}"] for k in ("mode", "x1", "x2", "K", "model", "mask", "R", "t")} for i in range(int(g["n"]))]


def _trace(ctx, mode, x1, x2, max_iters=1000):
    k = len(x1)
    cap = 1024
    m = 5 if mode == 0 else 7
    tr = _lib.LmedsTrace()
    idx, nsol = np.zeros((cap, m), np.int32), np.zeros(cap, np.int32)
    models, med = np.zeros((cap, 10, 9)), np.zeros(cap * 10, np.float32)
    tr.cap, tr.idx, tr.nsol, tr.models, tr.medians = cap, idx.ctypes.data, nsol.ctypes.data, models.ctypes.data, med.ctypes.data
    res = _lib.RansacResult()
    mask = np.zeros(max(k, 1), np.uint8)
    a, b = np.ascontiguousarray(x1, np.float64), np.ascontiguousarray(x2, np.float64)
    rc = ctx.lib.b2_debug_lmeds_trace_host(ctx.handle, mode, _lib.ptr(a), _lib.ptr(b), k, ctypes.byref(lmeds_params()), max_iters,
                                           ctypes.byref(tr), ctypes.byref(res), _lib.ptr(mask))
    ctx.check(rc, "lmeds_trace")
    n = tr.niters
    return dict(tr=tr, idx=idx[:n], nsol=nsol[:n], models=models[:n], med=med[:n * 10].reshape(n, 10), res=res, mask=mask[:k])


def _rot_deg(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


def _scenes():
    out = [(int(s["mode"]), s["x1"], s["x2"]) for s in _golden()]
    kp1, kp2, _, K, _, _, _ = vr.synthetic_two_view(31, 14000, 0.6)  # larger than the shared-memory copy of the errors
    out.append((1, kp1, kp2))
    out.append((0, vr.calibrate(kp1, *K), vr.calibrate(kp2, *K)))
    return out


@pytest.mark.parametrize("i", range(12))
def test_stages_equal_the_oracle(ctx, shim, i):
    mode, x1, x2 = _scenes()[i]
    d = _trace(ctx, mode, x1, x2)
    o = lr.lmeds(x1, x2, mode, lr.shim_solver(shim))
    assert d["tr"].niters == o["niters"] and d["tr"].drawn == o["n_drawn"]
    assert np.array_equal(d["idx"], o["idx"])
    # lmeds.cu is compiled without FMA contraction, so its solvers round as the host build does (libm's sqrt / division are
    # correctly rounded on both sides): every solution count, solution and median is the host build's.
    nsol_diff = int((d["nsol"] != o["nsol"]).sum())
    same = d["nsol"] == o["nsol"]
    live = ~np.isnan(o["medians"]) & same[:, None]
    far = 0
    for s_ in np.nonzero(same)[0]:
        for j in range(o["nsol"][s_]):
            a_, b_ = d["models"][s_, j], o["models"][s_, j]
            far += np.abs(a_ - b_).max() > 1e-12
    med_diff = int((live & (d["med"] != o["medians"])).sum())
    assert nsol_diff == 0 and far == 0 and med_diff == 0, (nsol_diff, far, med_diff)
    sl = o["slot"]
    if sl >= 0:
        assert np.abs(d["models"][sl // 10, sl % 10] - o["models"][sl // 10, sl % 10]).max() <= 1e-9
    assert d["tr"].slot == o["slot"] and d["tr"].sigma == o["sigma"] and d["tr"].thr == o["thr"]
    assert np.array_equal(d["mask"], o["mask"]) and d["tr"].count == o["count"]


def test_end_to_end_equals_cv2(ctx):
    """The golden scenes: cv2's mask bit for bit, its model to 1e-6 (up to sign), the pose within 0.1 deg of recoverPose's."""
    for i, s in enumerate(_golden()):
        mode, K = int(s["mode"]), tuple(float(v) for v in s["K"])
        d = _trace(ctx, mode, s["x1"], s["x2"])
        assert np.array_equal(d["mask"], s["mask"]), i
        M = np.array(d["res"].model).reshape(3, 3)
        a, b = M / np.linalg.norm(M), s["model"] / np.linalg.norm(s["model"])
        assert min(np.abs(a - b).max(), np.abs(a + b).max()) < 1e-6, i
        # pose through the batched entry (the trace runs with unit calibration)
        k = len(s["x1"])
        x1 = ctx_tensor(s["x1"])
        x2 = ctx_tensor(s["x2"])
        p = ransac_problem(k, mode, 0.0, 1000, x1=x1, x2=x2, cal1=K, cal2=K)
        r = lmeds_verify_batched_dev(ctx, [p])[0]
        assert r.status == 0
        assert _rot_deg(np.array(r.R).reshape(3, 3), s["R"]) < 0.1, i
        t, tc = np.array(r.t), s["t"] / np.linalg.norm(s["t"])
        assert np.degrees(np.arccos(np.clip(t @ tc / np.linalg.norm(t), -1, 1))) < 0.1, i


def ctx_tensor(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, np.float64)).cuda()


def _problem_list():
    import torch

    out, keep = [], []
    for mode, x1, x2 in _scenes()[:10]:
        a, b = ctx_tensor(x1), ctx_tensor(x2)
        m = torch.zeros(len(x1), dtype=torch.uint8, device="cuda")
        keep += [a, b, m]
        out.append(ransac_problem(len(x1), mode, 0.0, 1000, x1=a, x2=b, mask=m, cal1=(800.0, 640.0, 480.0), cal2=(800.0, 640.0, 480.0)))
    return out, keep


def _res(r):
    return (r.status, r.num_inliers, tuple(r.model), tuple(r.R), tuple(r.t))


def test_batched_equals_per_problem_and_any_cut(ctx):
    probs, keep = _problem_list()
    masks = [keep[3 * i + 2] for i in range(len(probs))]
    many = [_res(r) for r in lmeds_verify_batched_dev(ctx, probs)]
    mask_many = [m.cpu().numpy().copy() for m in masks]
    for i, p in enumerate(probs):
        assert _res(lmeds_verify_batched_dev(ctx, [p])[0]) == many[i]
        assert np.array_equal(masks[i].cpu().numpy(), mask_many[i])
    rev = [_res(r) for r in lmeds_verify_batched_dev(ctx, probs[::-1])]
    assert rev[::-1] == many
    ctx.set_option("ransac_workspace_mb", 1)
    try:
        assert [_res(r) for r in lmeds_verify_batched_dev(ctx, probs)] == many
    finally:
        ctx.set_option("ransac_workspace_mb", 1024)


def test_small_problems_fail(ctx):
    import torch

    x = ctx_tensor(np.random.default_rng(0).normal(size=(7, 2)))
    m = torch.ones(7, dtype=torch.uint8, device="cuda")
    probs = [ransac_problem(0, 0, 0.0, 1000, x1=x, x2=x), ransac_problem(5, 0, 0.0, 1000, x1=x, x2=x, mask=m),
             ransac_problem(7, 1, 0.0, 1000, x1=x, x2=x, cal1=(1.0, 0, 0), cal2=(1.0, 0, 0))]
    res = lmeds_verify_batched_dev(ctx, probs)
    assert [r.status for r in res] == [1, 1, 1]
    assert int(m[:5].sum()) == 0


def test_launches_and_one_synchronisation(ctx):
    """A batch of 10 ready problems: subsets, hypotheses, scores, selection, pose = 5 launches and one synchronisation."""
    probs, keep = _problem_list()
    lmeds_verify_batched_dev(ctx, probs)
    n0, s0 = ctx.launch_count(), ctx.ransac_sync_count()
    lmeds_verify_batched_dev(ctx, probs)
    assert ctx.launch_count() - n0 == 5 and ctx.ransac_sync_count() - s0 == 1


def test_bad_arguments_are_refused_before_any_launch(ctx):
    n0 = ctx.launch_count()
    x = ctx_tensor(np.zeros((10, 2)))
    for p in (ransac_problem(10, 2, 0.0, 1000, x1=x, x2=x), ransac_problem(-1, 0, 0.0, 1000, x1=x, x2=x),
              ransac_problem(10, 0, 0.0, 10**6, x1=x, x2=x), ransac_problem(10, 1, 0.0, 1000, x1=x, x2=x, cal1=(0.0, 0, 0))):
        arr = (_lib.RansacProblem * 1)(p)
        res = (_lib.RansacResult * 1)()
        assert ctx.lib.b2_lmeds_verify_batched_dev(ctx.handle, arr, 1, ctypes.byref(lmeds_params()), res, None) == -2
    bad = lmeds_params(1.0, 0.99)
    arr = (_lib.RansacProblem * 1)(ransac_problem(10, 0, 0.0, 1000, x1=x, x2=x))
    assert ctx.lib.b2_lmeds_verify_batched_dev(ctx.handle, arr, 1, ctypes.byref(bad), (_lib.RansacResult * 1)(), None) == -2
    assert ctx.launch_count() == n0


@pytest.mark.parametrize("use_intrinsics", [True, False])
def test_plugin_reference_criteria(use_intrinsics):
    """The reference's verifier criteria on seeded scenes at estimation_threshold_px = 0.5: pose within 2 deg, the inlier
    rows a subset of the matches, verify_many equal to verify; too few matches give the failure tuple."""
    v = B200LMEDS(use_intrinsics_in_verification=use_intrinsics, estimation_threshold_px=0.5)
    items = []
    for seed in range(4):
        kp1, kp2, m, K, R, t, _ = vr.synthetic_two_view(300 + seed, 800, 0.7)
        cal = Cal3Bundler(K[0], 0.0, 0.0, K[1], K[2])
        items.append((Keypoints(kp1.astype(np.float32)), Keypoints(kp2.astype(np.float32)), m.astype(np.int64), cal, cal, R, t))
    many = v.verify_many([it[:5] for it in items])
    for it, got in zip(items, many):
        one = v.verify(*it[:5])
        R_est, U_est, rows, ratio = got
        assert np.array_equal(rows, one[2]) and ratio == one[3]
        assert _rot_deg(R_est.matrix(), it[5]) < 2.0
        assert 0.5 < ratio <= 1.0 and len(rows) == round(ratio * len(it[2]))
    few = items[0][2][:5]
    assert v.verify(items[0][0], items[0][1], few, items[0][3], items[0][4])[0] is None


def test_nan_errors_rank_below_every_number(ctx, shim):
    """A quarter of the points at infinity: their errors are NaN (inf - inf).  cv2 (x86) produces the negative default NaN,
    which its int32 nth_element ranks below every number; the device canonicalises its NaN to that one, so every median,
    the chosen slot and the mask equal the oracle's (whose NumPy arithmetic produces the same NaN as cv2)."""
    for seed in (1, 2):
        x1, x2 = lr.probe_scene(seed, 400, 0.3)
        x1 = x1.copy()
        x1[::4] = np.inf
        d = _trace(ctx, 0, x1, x2)
        o = lr.lmeds(x1, x2, 0, lr.shim_solver(shim))
        live = ~np.isnan(o["medians"])
        assert np.array_equal(np.isnan(d["med"]), ~live)
        assert np.array_equal(d["med"][live], o["medians"][live])
        assert d["tr"].slot == o["slot"] and np.array_equal(d["mask"], o["mask"])
        M, mask = lr.cv2_lmeds(x1, x2, 0) if _have_cv2() else (None, o["mask"])
        assert np.array_equal(d["mask"], mask)


def _have_cv2():
    try:
        import cv2  # noqa: F401
    except ImportError:
        return False
    return True


@pytest.mark.parametrize("use_intrinsics", [True, False])
def test_reference_two_plane_scene(shim, use_intrinsics):
    """test_verifier_base.py:81-100 as test_lmeds.py inherits it (0.5 px), E and F.  Its bar (every row kept, pose within
    2 deg) is not one LMedS meets on 8 points: cv2's own LMEDS keeps 5 of 8 rows for E and 7 for F there, 9.3 and 3.5 deg
    from the true rotation (checked with cv2 4.13 on oracle.verifier_ref.two_planes_scene).  Eight points leave every
    minimal fit a median at the round-off level, so the winner is decided by the solver's last bits.  The plugin is held to
    the restatement instead: its rows are the oracle's inliers and its ratio their share, and at least half the rows stay."""
    uv1, uv2, R, t = vr.two_planes_scene(4, 4)
    matches = np.stack([np.arange(8), np.arange(8)], -1).astype(np.uint32)
    ver = B200LMEDS(use_intrinsics_in_verification=use_intrinsics, estimation_threshold_px=0.5)
    Rc, tc, rows, ratio = ver.verify(Keypoints(uv1), Keypoints(uv2), matches, Cal3Bundler(), Cal3Bundler())
    o = lr.lmeds(uv1, uv2, 0 if use_intrinsics else 1, lr.shim_solver(shim))
    assert Rc is not None and rows.dtype == matches.dtype
    assert np.array_equal(rows, matches[o["mask"] == 1]) and ratio == o["count"] / 8 and len(rows) >= 4


def test_reference_contract_degenerate_and_pickle():
    """test_verifier_base.py:102-146: failure tuple on empty and too-few matches, valid row indices on random input,
    picklability before and after use, the repr the two-view cache keys on."""
    import pickle

    for use_intrinsics in (True, False):
        ver = B200LMEDS(use_intrinsics, 0.5)
        pickle.dumps(ver)
        assert repr(ver) == f"B200LMEDS__use_intrinsics{use_intrinsics}_0.5px"
        rng = np.random.default_rng(0)
        kp1 = Keypoints(rng.uniform(0, 300, (50, 2)))
        kp2 = Keypoints(rng.uniform(0, 300, (60, 2)))
        cal = Cal3Bundler(200, 0, 0, 150, 150)
        for m in (np.zeros((0, 2), np.uint32), np.array([[0, 0], [1, 1], [2, 2], [3, 3], [4, 4]], np.uint32)):
            R, t, rows, ratio = ver.verify(kp1, kp2, m, cal, cal)
            assert R is None and t is None and rows.size == 0 and ratio == 0.0
        matches = np.stack([rng.permutation(50)[:40], rng.permutation(60)[:40]], -1).astype(np.uint32)
        R, t, rows, ratio = ver.verify(kp1, kp2, matches, cal, cal)
        pickle.loads(pickle.dumps(ver))
        if rows.size:
            assert np.all(rows[:, 0] < 50) and np.all(rows[:, 1] < 60)


def test_front_end_method_lmeds(b200_ctx):
    """DeviceFrontEnd.verify_many[_async] and B200TwoViewBatch: the default is RANSAC, unchanged; method="lmeds" gives what
    B200LMEDS.verify_many gives for the same pairs (rows, ratio, pose)."""
    import torch

    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd
    from gtsfm_b200.two_view import B200TwoViewBatch

    feats, intr, pairs, putative, plugin_items = {}, {}, [], {}, []
    for i, (k, ratio) in enumerate([(2000, 0.5), (1200, 0.7), (5, 1.0), (3000, 0.4)]):
        kp1, kp2, _, K, *_ = vr.synthetic_two_view(900 + i, max(k, 6), ratio)
        kp1, kp2 = kp1[:k].astype(np.float32), kp2[:k].astype(np.float32)
        for j, kp in ((2 * i, kp1), (2 * i + 1, kp2)):
            feats[j] = DeviceFeatures(torch.from_numpy(kp).cuda(), torch.zeros(k, device="cuda"), torch.zeros(k, 256, device="cuda"), (960, 1280))
            intr[j] = K
        rows = np.stack([np.arange(k), np.arange(k)], -1).astype(np.int64)
        pairs.append((2 * i, 2 * i + 1))
        putative[(2 * i, 2 * i + 1)] = torch.from_numpy(rows).cuda()
        cal = Cal3Bundler(K[0], 0, 0, K[1], K[2])
        plugin_items.append((Keypoints(kp1), Keypoints(kp2), rows, cal, cal))
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), ctx=b200_ctx)
    items = [(feats[a], feats[b], putative[(a, b)], intr[a], intr[b]) for a, b in pairs]
    default = fe.verify_many(items)
    ransac = fe.verify_many(items, method="ransac")
    lmeds = fe.verify_many(items, method="lmeds")
    lmeds_async = fe.verify_many_async(items, method="lmeds").result()
    ref = B200LMEDS(True, 4.0).verify_many(plugin_items)
    for d, r, l, la, p in zip(default, ransac, lmeds, lmeds_async, ref):
        assert (d[0] is None) == (r[0] is None) and d[3] == r[3] and torch.equal(d[4], r[4])
        assert (l[0] is None) == (p[0] is None) == (la[0] is None)
        assert torch.equal(l[4], la[4])
        if l[0] is not None:
            assert np.array_equal(np.nonzero(l[4].cpu().numpy())[0], p[2][:, 0])
            assert np.array_equal(l[1], p[0].matrix()) and np.allclose(l[2], p[1].point3(), atol=1e-12)
    tv = B200TwoViewBatch(fe, method="lmeds").run(feats, pairs, intr, putative)
    for (a, b), p in zip(pairs, ref):
        got = tv[(a, b)]
        if p[0] is None:
            assert got.i2Ri1 is None
        else:
            assert np.array_equal(got.v_corr_idxs, p[2]) and got.inlier_ratio_est_model == p[3]
    with pytest.raises(ValueError):
        fe.verify_many(items, method="usac")
