"""GPU: the batched two-view seam (gtsfm_b200/two_view.py) against the ORACLE (oracle/lightglue_ref + the cv2-driven
oracle/verifier_ref), and against the per-pair plugins (same kernels, per-call API)."""
import numpy as np
import pytest
import torch

from gtsfm_b200 import synthetic as syn
from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
from gtsfm_b200.pipeline import DeviceFrontEnd
from gtsfm_b200.two_view import B200TwoViewBatch
from gtsfm_b200.verifier import B200Ransac

pytestmark = pytest.mark.gpu


def test_batch_equals_per_pair_plugins():
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp"), max_keypoints=1024)
    frames, cal = syn.synthetic_sequence(4, 240, 320)
    feats = {i: fe.detect(torch.from_numpy(f).cuda()) for i, f in enumerate(frames)}
    pairs = [(0, 1), (0, 2), (1, 3), (2, 3)]
    intr = {i: cal for i in feats}
    res = B200TwoViewBatch(fe, 4.0).run(feats, pairs, intr)
    assert set(res) == set(pairs)
    ver = B200Ransac(True, 4.0)
    calib = Cal3Bundler(cal[0], 0, 0, cal[1], cal[2])
    n_ok = 0
    for (i1, i2), r in res.items():
        m, _ = fe.match(feats[i1], feats[i2])
        m = m.cpu().numpy()
        assert r.num_putative == len(m)
        k1, k2 = Keypoints(feats[i1].kp.cpu().numpy()), Keypoints(feats[i2].kp.cpu().numpy())
        R, U, v, ratio = ver.verify(k1, k2, m, calib, calib)
        if R is None:
            assert r.i2Ri1 is None and len(r.v_corr_idxs) == 0
            continue
        n_ok += 1
        assert np.array_equal(r.v_corr_idxs, v), "verified rows differ from the per-pair plugin"
        np.testing.assert_allclose(r.i2Ri1.matrix(), R.matrix(), atol=1e-9)
        np.testing.assert_allclose(r.i2Ui1.point3(), U.point3(), atol=1e-9)
        assert abs(r.inlier_ratio_est_model - ratio) < 1e-12
    assert n_ok >= 2, "the synthetic sequence should give verifiable pairs"


def test_batch_matches_the_oracle():
    """Putative matches must be the oracle's LightGlue rows bit for bit; pose / verified rows must agree with what
    cv2.findEssentialMat(USAC_ACCURATE) + recoverPose return for them (OpenCV's RANSAC is not part of the reference project, so the
    verified set is compared by IoU and the pose by angle: the tolerances of tests/test_verifier_gpu.py)."""
    from oracle import lightglue_ref, verifier_ref

    lg_sd = syn.lightglue_state_dict(2, "sharp")
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), lg_sd, max_keypoints=1024)
    frames, cal = syn.synthetic_sequence(4, 240, 320)
    feats = {i: fe.detect(torch.from_numpy(f).cuda()) for i, f in enumerate(frames)}
    pairs = [(0, 1), (0, 2), (1, 3)]
    res = B200TwoViewBatch(fe, 4.0).run(feats, pairs, {i: cal for i in feats})
    n_ok = 0
    for (i1, i2) in pairs:
        a, b = feats[i1], feats[i2]
        kpa, kpb = a.kp.cpu().numpy(), b.kp.cpu().numpy()
        m_ref = lightglue_ref.lightglue_match(kpa, a.desc.cpu().numpy(), kpb, b.desc.cpu().numpy(), lg_sd)
        r = res[(i1, i2)]
        assert r.num_putative == len(m_ref), f"pair {(i1, i2)}: {r.num_putative} putative matches vs oracle {len(m_ref)}"
        m_gpu, _ = fe.match(a, b)
        assert np.array_equal(m_gpu.cpu().numpy(), m_ref)
        R, t, rows, ratio, E = verifier_ref.verify_cv2(kpa.astype(np.float64), kpb.astype(np.float64), m_ref, cal, cal, True, 4.0)
        if R is None:
            continue
        n_ok += 1
        assert r.i2Ri1 is not None
        assert verifier_ref.rot_angle_deg(R, r.i2Ri1.matrix()) < 1.0
        assert verifier_ref.dir_angle_deg(t, r.i2Ui1.point3()) < 5.0
        mine, ref = set(map(tuple, r.v_corr_idxs.tolist())), set(map(tuple, rows.tolist()))
        assert len(mine & ref) / max(1, len(mine | ref)) > 0.9, (len(mine), len(ref))
        assert abs(r.inlier_ratio_est_model - ratio) < 0.08
    assert n_ok >= 2


def test_too_few_matches_is_the_failure_tuple():
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp"), max_keypoints=256)
    frames, cal = syn.synthetic_sequence(2, 120, 160)
    feats = {i: fe.detect(torch.from_numpy(f).cuda()) for i, f in enumerate(frames)}
    put = {(0, 1): torch.zeros((3, 2), dtype=torch.int64, device="cuda")}
    r = B200TwoViewBatch(fe).run(feats, [(0, 1)], {0: cal, 1: cal}, putative=put)[(0, 1)]
    assert r.i2Ri1 is None and r.i2Ui1 is None and r.v_corr_idxs.shape == (0, 2) and r.num_putative == 3


def test_generator_verify_with_equals_two_view_batch():
    """generate_correspondences(..., verify_with=...) = the same matches + the TwoViewResults B200TwoViewBatch gives for them."""
    from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator
    from gtsfm_b200.gtsfm_api import Image

    frames, cal = syn.synthetic_sequence(6, 240, 320)
    graph = [(i, j) for i in range(6) for j in range(i + 1, min(6, i + 4))]  # 12 pairs = two lock-step batches
    gen = B200CorrespondenceGenerator(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp"), max_keypoints=600)
    intr = {i: cal for i in range(6)}
    kps, matches = gen.generate_correspondences(None, [Image(f) for f in frames], graph, verify_with=(intr, 4.0))
    got = gen.last_two_view
    fe, feats = gen._front_end(), gen.last_device_features
    put = {p: torch.from_numpy(matches[p]).cuda() for p in graph}
    want = B200TwoViewBatch(fe, 4.0).run(feats, graph, intr, putative=put)
    assert set(got) == set(graph) and sum(1 for r in got.values() if r.i2Ri1 is not None) >= 10
    for p in graph:
        a, b = got[p], want[p]
        assert a.num_putative == b.num_putative == len(matches[p]) and np.array_equal(a.v_corr_idxs, b.v_corr_idxs)
        assert a.inlier_ratio_est_model == b.inlier_ratio_est_model
        if b.i2Ri1 is None:
            assert a.i2Ri1 is None
        else:
            assert np.array_equal(a.i2Ri1.matrix(), b.i2Ri1.matrix()) and np.array_equal(a.i2Ui1.point3(), b.i2Ui1.point3())
