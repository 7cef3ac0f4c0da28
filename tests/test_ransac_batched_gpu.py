"""b2_ransac_verify_batched_dev: a batch of image pairs verified in one call gives, for every pair, exactly the bytes the
per-pair entry points give (same seed, same kernels with a table of one problem, fixed-order reductions), whatever else is
in the batch; the F problems also recover their pose on the device; the call costs one pair's launches and one
synchronisation."""
import ctypes

import numpy as np
import pytest
import torch

from gtsfm_b200 import _lib
from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
from gtsfm_b200.verifier import (DEFAULT_SEED, E_MAX_ITERS, F_MAX_ITERS, RANSAC_SUCCESS_PROB, B200Ransac, RansacEngine,
                                 normalize_coordinates, ransac_problem)
from oracle import verifier_ref as vr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class Scene:
    """A seeded two-view scene on the device: float32 keypoints, int64 rows, (f, u0, v0), and the same points as doubles."""

    def __init__(self, seed, k, ratio, thr_px=4.0, kind="plain"):
        kp1, kp2, _, K, self.R, self.t, _ = vr.synthetic_two_view(seed, max(k, 1), ratio)
        kp1, kp2 = kp1[:k].astype(np.float32), kp2[:k].astype(np.float32)
        if kind == "duplicated":  # every correspondence twice
            kp1[1::2], kp2[1::2] = kp1[0:-1:2][: len(kp1[1::2])], kp2[0:-1:2][: len(kp2[1::2])]
        if kind == "identical":  # one correspondence k times: no sample gives a model
            kp1[:], kp2[:] = kp1[0], kp2[0]
        self.k, self.cal, self.thr_px = k, tuple(float(c) for c in K), thr_px
        self.kp1_h, self.kp2_h = kp1, kp2
        self.kp1, self.kp2 = torch.from_numpy(kp1).to(DEV), torch.from_numpy(kp2).to(DEV)
        self.rows = torch.arange(k, device=DEV, dtype=torch.int64)[:, None].repeat(1, 2).contiguous()
        self.mask = torch.zeros(max(k, 1), dtype=torch.uint8, device=DEV)

    def pixels(self):  # what k_rs_gather makes of an F problem: the float32 pixels as doubles
        return np.ascontiguousarray(self.kp1_h, np.float64), np.ascontiguousarray(self.kp2_h, np.float64)

    def calibrated(self):  # what k_rs_gather makes of an E problem
        return np.ascontiguousarray(vr.calibrate(self.kp1_h, *self.cal)), np.ascontiguousarray(vr.calibrate(self.kp2_h, *self.cal))

    def problem(self, mode=0, mask=None):
        thr = self.thr_px / self.cal[0] if mode == 0 else self.thr_px
        return ransac_problem(self.k, mode, thr, E_MAX_ITERS if mode == 0 else F_MAX_ITERS, mask=self.mask if mask is None else mask,
                              kp1=self.kp1, kp2=self.kp2, matches=self.rows, cal1=self.cal, cal2=self.cal)


def result_bytes(r, mask, k):
    return (r.status, r.num_inliers, np.array(r.model), np.array(r.R), np.array(r.t), mask[:k].cpu().numpy().copy())


def same(a, b):
    assert a[0] == b[0] and a[1] == b[1], (a[:2], b[:2])
    for x, y in zip(a[2:], b[2:]):
        assert np.array_equal(x, y)  # raw doubles / bytes, no tolerance


def per_pair_E(ctx, sc, stream=None):
    """b2_ransac_essential_dev on the scene -> the same tuple result_bytes() makes of a batched result"""
    E, R, t, n = np.zeros(9), np.zeros(9), np.zeros(3), ctypes.c_int(0)
    mask = torch.zeros(max(sc.k, 1), dtype=torch.uint8, device=DEV)
    prm = _lib.RansacParams(sc.thr_px / sc.cal[0], RANSAC_SUCCESS_PROB, E_MAX_ITERS, DEFAULT_SEED)
    c = np.asarray(sc.cal, np.float64)
    torch.cuda.synchronize()
    rc = ctx.lib.b2_ransac_essential_dev(ctx.handle, _lib.ptr(sc.kp1), _lib.ptr(sc.kp2), _lib.ptr(sc.rows), sc.k, _lib.ptr(c), _lib.ptr(c),
                                         ctypes.byref(prm), _lib.ptr(E), _lib.ptr(mask), ctypes.byref(n), _lib.ptr(R), _lib.ptr(t),
                                         ctypes.c_void_p(stream or 0))
    ctx.check(rc, "ransac_essential_dev")
    return rc, n.value, E, R, t, mask[: sc.k].cpu().numpy().copy()


def batched(ctx, problems, stream=None):
    torch.cuda.synchronize()
    return RansacEngine(ctx=ctx).verify_batched_dev(problems, stream=stream)


def trace(ctx, mode, x1, x2, thr, max_iters):
    """(sampling rounds, extension flag) of the per-pair path, from the trace entry"""
    tr = _lib.RansacTrace()
    tr.batch, tr.max_records = 16384, 0
    model, R, t, n = np.zeros(9), np.zeros(9), np.zeros(3), ctypes.c_int(0)
    mask = np.zeros(max(len(x1), 1), np.uint8)
    prm = _lib.RansacParams(thr, RANSAC_SUCCESS_PROB, min(max_iters, 2**31 - 1), DEFAULT_SEED)
    rc = ctx.lib.b2_debug_ransac_trace_host(ctx.handle, mode, _lib.ptr(x1), _lib.ptr(x2), len(x1), ctypes.byref(prm), ctypes.byref(tr),
                                            _lib.ptr(model), _lib.ptr(mask), ctypes.byref(n), _lib.ptr(R), _lib.ptr(t))
    ctx.check(rc, "debug_ransac_trace")
    return tr.batches, tr.ext_go


E_SCENES = ([(s, k, r, thr, "plain") for s, (k, r, thr) in enumerate([
    (5, 1.0, 4.0), (6, 1.0, 4.0), (8, 0.9, 4.0), (20, 0.6, 2.0), (60, 0.5, 4.0), (100, 0.3, 4.0), (250, 0.9, 1.0), (500, 0.15, 4.0),
    (500, 0.6, 4.0), (1000, 0.3, 2.0), (1000, 0.8, 4.0), (2000, 0.2, 4.0), (2000, 0.3, 4.0), (2000, 0.9, 4.0), (3000, 0.45, 8.0),
    (5000, 0.3, 4.0), (5000, 0.6, 4.0), (5000, 0.9, 1.0), (777, 0.25, 4.0), (1234, 0.7, 0.5)], start=100)] +
            [(200, 3, 1.0, 4.0, "plain"), (201, 0, 1.0, 4.0, "plain"), (202, 300, 0.0, 0.05, "plain"), (203, 64, 1.0, 4.0, "identical"),
             (204, 400, 0.7, 4.0, "duplicated"), (205, 4, 1.0, 4.0, "plain")])


def test_batched_equals_per_pair_bit_for_bit(b200_ctx):
    scenes = [Scene(*a) for a in E_SCENES]
    assert len(scenes) >= 24
    res = batched(b200_ctx, [sc.problem() for sc in scenes])
    ext, statuses = set(), set()
    for sc, r in zip(scenes, res):
        same(result_bytes(r, sc.mask, sc.k), per_pair_E(b200_ctx, sc))
        statuses.add((r.status, sc.k >= 5))
        if sc.k < 5:
            assert r.status == 1 and r.num_inliers == 0 and not sc.mask[: sc.k].any()
        elif sc.k >= 500:
            ext.add(trace(b200_ctx, 0, *sc.calibrated(), sc.thr_px / sc.cal[0], E_MAX_ITERS)[1])
    assert ext == {0, 1}, "both a scene that runs the extension stage and one that skips it"
    assert (0, True) in statuses and (1, False) in statuses


def host_pose_from_F(eng, F, mask, p1, p2, cal):
    """what the plugin's per-pair path does after b2_ransac_fundamental_host (utils/verification.py:99-112)"""
    c = Cal3Bundler(cal[0], 0, 0, cal[1], cal[2])
    E = c.K().T @ F @ c.K()
    inl = mask == 1
    R, t, _ = eng.recover_pose(E, normalize_coordinates(p1[inl], c), normalize_coordinates(p2[inl], c))
    return R, t


def test_fundamental_problems_equal_the_host_entry_and_recover_pose(b200_ctx):
    eng = RansacEngine(ctx=b200_ctx)
    scenes = [Scene(300, 300, 0.25), Scene(301, 1000, 0.8), Scene(302, 2000, 0.5, thr_px=2.0), Scene(303, 7, 1.0), Scene(304, 8, 1.0)]
    ready = [tuple(torch.from_numpy(a).to(DEV) for a in sc.pixels()) for sc in scenes]
    problems = [sc.problem(mode=1) for sc in scenes]
    for p, (x1, x2) in zip(problems[1::2], ready[1::2]):  # every other problem hands over ready double pixels instead
        p.kp1, p.kp2, p.matches, p.x1, p.x2 = None, None, None, x1.data_ptr(), x2.data_ptr()
    res = batched(b200_ctx, problems)
    rounds = []
    for sc, r in zip(scenes, res):
        p1, p2 = sc.pixels()
        F, mask = eng.fundamental(p1, p2, sc.thr_px)
        got = sc.mask[: sc.k].cpu().numpy()
        assert np.array_equal(got, mask)
        if F is None:
            assert r.status == 1 and not got.any()
            continue
        assert sc.k >= 8
        assert r.status == 0 and np.array_equal(np.array(r.model), F.ravel()) and r.num_inliers == int(mask.sum())
        R, t = host_pose_from_F(eng, F, mask, p1, p2, sc.cal)
        assert np.abs(np.array(r.R).reshape(3, 3) - R).max() < 1e-9 and np.abs(np.array(r.t) - t).max() < 1e-9
        rounds.append(trace(b200_ctx, 1, p1, p2, sc.thr_px, F_MAX_ITERS)[0])
    assert rounds[0] > 1 and rounds[1] == 1, rounds  # ~25 % inliers needs several 16 384-hypothesis rounds, 80 % one
    assert vr.rot_angle_deg(scenes[1].R, np.array(res[1].R).reshape(3, 3)) < 1.5


def test_result_is_independent_of_batch_composition(b200_ctx):
    target = Scene(400, 1500, 0.3)
    alone = per_pair_E(b200_ctx, target)
    others = [Scene(410 + i, 200 + 300 * i, 0.2 + 0.1 * i) for i in range(6)]
    fscene = Scene(420, 600, 0.6)

    def run(problems, at, stream=None):
        target.mask.zero_()
        res = batched(b200_ctx, problems, stream=stream)
        torch.cuda.synchronize()
        same(result_bytes(res[at], target.mask, target.k), alone)
        return res

    run([target.problem()], 0)
    run([target.problem()] + [o.problem() for o in others], 0)
    ref = run([o.problem() for o in others] + [target.problem()], len(others))
    # cut into sub-batches by the workspace budget (an E problem's slices take 3.4 MB + its points)
    first = (ctypes.c_int * 8)()
    probs = [o.problem() for o in others] + [target.problem()]
    arr = (_lib.RansacProblem * len(probs))(*probs)
    assert b200_ctx.lib.b2_ransac_plan(arr, len(probs), 8 << 20, first) >= 3
    b200_ctx.set_option("ransac_workspace_mb", 8)
    try:
        split = run(probs, len(others))
    finally:
        b200_ctx.set_option("ransac_workspace_mb", 1024)
    for a, b in zip(ref, split):
        assert bytes(a) == bytes(b)
    # mixed with F problems, and on a stream of its own
    run([fscene.problem(mode=1), target.problem(), fscene.problem(mode=1, mask=torch.zeros(600, dtype=torch.uint8, device=DEV))], 1)
    st = torch.cuda.Stream(DEV)
    torch.cuda.synchronize()
    run([o.problem() for o in others[:2]] + [target.problem()], 2, stream=st.cuda_stream)


def test_contract_through_the_plugin(golden_dir):
    for use_intrinsics in (True, False):
        ver = B200Ransac(use_intrinsics, 0.5)
        uv1, uv2, R, t = vr.two_planes_scene(4, 4)
        rows8 = np.stack([np.arange(8), np.arange(8)], -1).astype(np.uint32)
        (Rc, tc, rows, ratio), = ver.verify_many([(Keypoints(uv1), Keypoints(uv2), rows8, Cal3Bundler(), Cal3Bundler())])
        assert vr.rot_angle_deg(R, Rc.matrix()) < 2.0 and vr.dir_angle_deg(t, tc.point3()) < 2.0
        assert np.array_equal(rows, rows8) and rows.dtype == rows8.dtype and ratio == 1.0
    fx = np.load(golden_dir / "verifier_argoverse.npz")
    uv1, uv2, K = fx["uv1"], fx["uv2"], fx["K"]
    cal = Cal3Bundler(K[0], 0, 0, K[1], K[2])
    rows = np.stack([np.arange(len(uv1)), np.arange(len(uv1))], -1).astype(np.int64)
    ver = B200Ransac(True, float(fx["thr_px"]))
    (Ra, Ua, _, _), (R5, U5, rows5, ratio5) = ver.verify_many([(Keypoints(uv1), Keypoints(uv2), rows, cal, cal),
                                                              (Keypoints(uv1), Keypoints(uv2), rows[:5], cal, cal)])
    euler, i1ti2 = vr.pose_to_euler_zyx_and_i1ti2(Ra.matrix(), Ua.point3())
    assert np.allclose(euler, fx["euler_zyx_deg_gt"], atol=float(fx["euler_tol_deg"])), euler
    assert np.allclose(i1ti2, fx["i1ti2_gt"], atol=float(fx["t_tol"])), i1ti2
    assert R5 is None and U5 is None and len(rows5) == 0 and ratio5 == 0.0


@pytest.mark.parametrize("use_intrinsics", [True, False])
def test_verify_many_equals_verify_on_a_mixed_list(use_intrinsics):
    ver = B200Ransac(use_intrinsics, 4.0)
    items = []
    for i, (k, ratio, f32) in enumerate([(400, 0.5, True), (3, 1.0, True), (900, 0.7, False), (0, 1.0, True), (1500, 0.35, True), (7, 1.0, False)]):
        kp1, kp2, rows, K, *_ = vr.synthetic_two_view(500 + i, max(k, 1), ratio)
        dt = np.float32 if f32 else np.float64  # float32 keypoints are calibrated on the device, others on the host
        cal = Cal3Bundler(K[0], 0.0 if f32 else 1e-3, 0, K[1], K[2])  # a distorted camera is normalised on the host (E) / verified alone (F)
        items.append((Keypoints(kp1.astype(dt)), Keypoints(kp2.astype(dt)), rows[:k].astype(np.uint32 if i % 2 else np.int64), cal, cal))
    many = ver.verify_many(items)
    assert len(many) == len(items)
    for it, (R, U, rows, ratio) in zip(items, many):
        R1, U1, rows1, ratio1 = ver.verify(*it)
        assert np.array_equal(rows, rows1) and rows.dtype == rows1.dtype and ratio == ratio1
        assert (R is None) == (R1 is None) and (U is None) == (U1 is None)
        if R is not None:
            tol = 0.0 if use_intrinsics else 1e-9
            assert np.abs(R.matrix() - R1.matrix()).max() <= tol and np.abs(U.point3() - U1.point3()).max() <= tol


def test_launches_and_synchronisations_of_a_batch(b200_ctx):
    """One pair: 11 launches (gather, hypotheses / scores / selection of the sampling round and of the extension stage, refine,
    pick, mask, pose).  32 pairs in one call: the same 11, and ONE stream synchronisation."""
    scenes = [Scene(600 + i, 800, 0.3 + 0.02 * (i % 20)) for i in range(32)]
    batched(b200_ctx, [scenes[0].problem()])  # buffers allocated
    n0 = b200_ctx.launch_count()
    batched(b200_ctx, [scenes[0].problem()])
    one = b200_ctx.launch_count() - n0
    n0, s0 = b200_ctx.launch_count(), b200_ctx.ransac_sync_count()
    batched(b200_ctx, [sc.problem() for sc in scenes])
    many, syncs = b200_ctx.launch_count() - n0, b200_ctx.ransac_sync_count() - s0
    assert one == 11 and many <= 2 * one, (one, many)
    assert syncs == 1


def test_bad_arguments_are_refused_before_any_launch(b200_ctx):
    sc = Scene(700, 100, 0.5)
    n0 = b200_ctx.launch_count()
    lib, h = b200_ctx.lib, b200_ctx.handle
    prm = _lib.RansacParams(0.0, RANSAC_SUCCESS_PROB, 0, DEFAULT_SEED)
    res = (_lib.RansacResult * 2)()

    def call(*problems, params=prm):
        arr = (_lib.RansacProblem * len(problems))(*problems)
        return lib.b2_ransac_verify_batched_dev(h, arr, len(problems), ctypes.byref(params), res, None)

    bad = []
    for field, value in (("k", -1), ("mode", 2), ("threshold", -1.0), ("kp1", None), ("matches", None)):
        p = sc.problem()
        setattr(p, field, value)
        bad.append(p)
    p = sc.problem()
    p.cal1[0] = 0.0
    bad.append(p)
    p = sc.problem()
    p.x1 = sc.kp1.data_ptr()  # x1 without x2
    bad.append(p)
    for p in bad:
        assert call(sc.problem(), p) == -2  # B2_ERR_ARG
    assert call(sc.problem(), params=_lib.RansacParams(0.0, 1.5, 0, DEFAULT_SEED)) == -2
    assert lib.b2_ransac_verify_batched_dev(h, None, 0, ctypes.byref(prm), None, None) == 0  # an empty batch is legal
    assert b200_ctx.launch_count() == n0
