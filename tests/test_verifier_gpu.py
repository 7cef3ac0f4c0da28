"""GPU parity for the RANSAC verifier.  USAC cannot be matched bit-for-bit (SURVEY.md §7 hard part 4); the bar is the
reference tests' own criteria (tests/frontend/verifier/test_verifier_base.py, test_ransac.py) plus agreement with the
cv2 results stored in tests/golden/verifier_*.npz."""
import pickle

import numpy as np
import pytest

from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
from gtsfm_b200.verifier import B200Ransac, RansacEngine
from oracle import verifier_ref as vr

pytestmark = pytest.mark.gpu

ROT_TOL_DEG = 2.0  # ROTATION_ANGULAR_ERROR_DEG_THRESHOLD, test_verifier_base.py:24
DIR_TOL_DEG = 2.0


@pytest.mark.parametrize("use_intrinsics", [True, False])
def test_two_plane_scene(use_intrinsics):
    """test_verifier_base.py:81-100 for E (5pt) and F (8pt), thresholds as in test_ransac.py:11-30 (0.5 px)."""
    uv1, uv2, R, t = vr.two_planes_scene(4, 4)
    matches = np.stack([np.arange(8), np.arange(8)], -1).astype(np.uint32)
    ver = B200Ransac(use_intrinsics_in_verification=use_intrinsics, estimation_threshold_px=0.5)
    Rc, tc, rows, ratio = ver.verify(Keypoints(uv1), Keypoints(uv2), matches, Cal3Bundler(), Cal3Bundler())
    assert vr.rot_angle_deg(R, Rc.matrix()) < ROT_TOL_DEG
    assert vr.dir_angle_deg(t, tc.point3()) < DIR_TOL_DEG
    assert np.array_equal(rows, matches) and rows.dtype == matches.dtype
    assert ratio == 1.0


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_agrees_with_cv2_on_seeded_scenes(golden_dir, seed):
    fx = np.load(golden_dir / f"verifier_{seed}.npz")
    kp1, kp2, matches, K, R, t, is_in = vr.synthetic_two_view(seed, int(fx["k"]), float(fx["ratio"]))
    cal = Cal3Bundler(K[0], 0, 0, K[1], K[2])
    ver = B200Ransac(True, 4.0)
    Rc, tc, rows, ratio = ver.verify(Keypoints(kp1), Keypoints(kp2), matches, cal, cal)
    assert vr.rot_angle_deg(R, Rc.matrix()) < 0.5 and vr.dir_angle_deg(t, tc.point3()) < 2.0
    mine = set(rows[:, 0].tolist())
    cv = set(fx["rows_cv"][:, 0].tolist())
    gt = set(np.flatnonzero(is_in).tolist())
    iou = len(mine & cv) / len(mine | cv)
    assert iou > 0.97, f"inlier IoU vs cv2 {iou:.3f}"
    assert len(gt - mine) <= 0.02 * len(gt), "missed true inliers"
    assert abs(ratio - float(fx["ratio_cv"])) < 0.02
    # F path (8-point)
    verF = B200Ransac(False, 4.0)
    Rf, tf, rowsf, ratiof = verF.verify(Keypoints(kp1), Keypoints(kp2), matches, cal, cal)
    assert vr.rot_angle_deg(R, Rf.matrix()) < 1.5
    mf, cvf = set(rowsf[:, 0].tolist()), set(fx["rows_cvF"][:, 0].tolist())
    assert len(mf & cvf) / len(mf | cvf) > 0.95


def test_inlier_definition_and_recover_pose(b200_ctx, golden_dir):
    """mask == (squared Sampson < thr^2) under the returned E; recoverPose matches cv2's R, t for cv2's own E."""
    fx = np.load(golden_dir / "verifier_2.npz")
    kp1, kp2, matches, K, R, t, is_in = vr.synthetic_two_view(2, 1000, 0.8)
    n1, n2 = vr.calibrate(kp1, *K), vr.calibrate(kp2, *K)
    eng = RansacEngine(ctx=b200_ctx)
    thr = 4.0 / K[0]
    E, mask, Rg, tg = eng.essential(n1, n2, thr)
    s = vr.sampson_sq(E, n1, n2)
    assert np.array_equal(mask.astype(bool), s < thr * thr)
    rows = fx["rows_cv"]
    R2, t2, good = eng.recover_pose(fx["E_cv"], n1[rows[:, 0]], n2[rows[:, 1]])
    assert vr.rot_angle_deg(fx["R_cv"], R2) < 1e-3 and vr.dir_angle_deg(fx["t_cv"], t2) < 1e-3
    assert good == len(rows)


def test_contract_degenerate_and_repro():
    """Failure tuple, index validity on random input, picklability, run-to-run identity
    (test_verifier_base.py:102-146, repro test SURVEY.md Appendix B)."""
    ver = B200Ransac(True, 0.5)
    pickle.dumps(ver)
    assert repr(ver) == "B200Ransac__use_intrinsicsTrue_0.5px"
    rng = np.random.default_rng(0)
    kp1 = Keypoints(rng.uniform(0, 300, (50, 2)))
    kp2 = Keypoints(rng.uniform(0, 300, (60, 2)))
    cal = Cal3Bundler(200, 0, 0, 150, 150)
    for m in (np.zeros((0, 2), np.uint32), np.array([[0, 0], [1, 1], [2, 2], [3, 3], [4, 4]], np.uint32)):
        R, t, rows, ratio = ver.verify(kp1, kp2, m, cal, cal)
        assert R is None and t is None and rows.size == 0 and ratio == 0.0
    matches = np.stack([rng.permutation(50)[:40], rng.permutation(60)[:40]], -1).astype(np.uint32)
    R, t, rows, ratio = ver.verify(kp1, kp2, matches, cal, cal)
    pickle.dumps(ver)
    if rows.size:
        assert np.all(rows[:, 0] < 50) and np.all(rows[:, 1] < 60)
    kpa, kpb, m2, K, *_ = vr.synthetic_two_view(9, 400, 0.5)
    cal2 = Cal3Bundler(K[0], 0, 0, K[1], K[2])
    v2 = B200Ransac(True, 4.0)
    first = v2.verify(Keypoints(kpa), Keypoints(kpb), m2, cal2, cal2)
    for _ in range(10):
        again = v2.verify(Keypoints(kpa), Keypoints(kpb), m2, cal2, cal2)
        assert np.array_equal(first[0].matrix(), again[0].matrix()) and np.array_equal(first[2], again[2])


def test_argoverse_known_answer(golden_dir):
    """The reference's known-answer test (tests/frontend/verifier/test_verifier_argoverse.py:72-136) on the CUDA verifier:
    same labelled correspondences, intrinsics, threshold (0.5 px) and tolerances (+-1 deg, +-0.01)."""
    fx = np.load(golden_dir / "verifier_argoverse.npz")
    uv1, uv2, K = fx["uv1"], fx["uv2"], fx["K"]
    cal = Cal3Bundler(K[0], 0, 0, K[1], K[2])
    matches = np.stack([np.arange(len(uv1)), np.arange(len(uv1))], -1).astype(np.int64)
    ver = B200Ransac(use_intrinsics_in_verification=True, estimation_threshold_px=float(fx["thr_px"]))
    R, U, rows, ratio = ver.verify(Keypoints(uv1), Keypoints(uv2), matches, cal, cal)
    assert R is not None
    euler, i1ti2 = vr.pose_to_euler_zyx_and_i1ti2(R.matrix(), U.point3())
    assert np.allclose(euler, fx["euler_zyx_deg_gt"], atol=float(fx["euler_tol_deg"])), euler
    assert np.allclose(i1ti2, fx["i1ti2_gt"], atol=float(fx["t_tol"])), i1ti2
    # 5 correspondences (:119-136): no crash, failure tuple
    R5, U5, rows5, _ = ver.verify(Keypoints(uv1), Keypoints(uv2), matches[:5], cal, cal)
    assert R5 is None and U5 is None and len(rows5) == 0


def test_inlier_iou_and_pose_statistics_over_120_scenes(tmp_path):
    """north_star lists the inlier mask among the outputs to match; cv2's USAC sampler / local optimisation are not part of
    the reference project, so the agreement is STATISTICAL: 120 seeded scenes (K in {200, 500, 1000, 2000}, inlier ratio in
    {0.3, 0.5, 0.8}, 0.5 px noise) through B200Ransac and through cv2 (the oracle), inlier-set IoU and pose error against the
    ground truth for both.  The per-scene distribution is written to the test's temporary directory."""
    import json

    ver = B200Ransac(True, 4.0)
    rows_out = []
    for idx in range(120):
        k = (200, 500, 1000, 2000)[idx % 4]
        ratio = (0.3, 0.5, 0.8)[(idx // 4) % 3]
        kp1, kp2, matches, K, R, t, is_in = vr.synthetic_two_view(1000 + idx, k, ratio)
        cal = Cal3Bundler(K[0], 0, 0, K[1], K[2])
        Rm, tm, rows, _ = ver.verify(Keypoints(kp1), Keypoints(kp2), matches, cal, cal)
        Rc, tc, rows_cv, _, _ = vr.verify_cv2(kp1, kp2, matches, K, K, True, 4.0)
        assert Rm is not None and Rc is not None
        mine, cv, gt = set(rows[:, 0].tolist()), set(rows_cv[:, 0].tolist()), set(np.flatnonzero(is_in).tolist())
        rows_out.append(dict(k=k, ratio=ratio, iou_cv2=len(mine & cv) / max(1, len(mine | cv)), recall_gt=len(mine & gt) / max(1, len(gt)),
                             recall_gt_cv2=len(cv & gt) / max(1, len(gt)), rot_err=vr.rot_angle_deg(R, Rm.matrix()),
                             rot_err_cv2=vr.rot_angle_deg(R, Rc), dir_err=vr.dir_angle_deg(t, tm.point3()), dir_err_cv2=vr.dir_angle_deg(t, tc)))
    iou = np.array([r["iou_cv2"] for r in rows_out])
    rot, rot_cv = np.array([r["rot_err"] for r in rows_out]), np.array([r["rot_err_cv2"] for r in rows_out])
    summary = dict(scenes=len(rows_out), iou_min=float(iou.min()), iou_p05=float(np.percentile(iou, 5)), iou_median=float(np.median(iou)),
                   iou_mean=float(iou.mean()), exact_same_mask=int((iou == 1.0).sum()), rot_err_median=float(np.median(rot)),
                   rot_err_max=float(rot.max()), rot_err_cv2_median=float(np.median(rot_cv)), rot_err_cv2_max=float(rot_cv.max()),
                   recall_gt_min=float(min(r["recall_gt"] for r in rows_out)), recall_gt_cv2_min=float(min(r["recall_gt_cv2"] for r in rows_out)))
    (tmp_path / "ransac_iou.json").write_text(json.dumps(dict(summary=summary, scenes=rows_out), indent=1))
    print(summary)
    # (where the two masks differ most - IoU ~0.9 - it is cv2 that is further from the ground truth: see the per-scene rows)
    assert summary["iou_median"] > 0.99 and summary["iou_p05"] > 0.95 and summary["iou_min"] > 0.85, summary
    assert summary["rot_err_max"] <= summary["rot_err_cv2_max"] + 0.1 and summary["rot_err_median"] <= summary["rot_err_cv2_median"] + 0.02, summary
    assert summary["recall_gt_min"] >= min(0.98, summary["recall_gt_cv2_min"]), summary
