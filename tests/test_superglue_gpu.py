"""GPU parity: CUDA SuperGlue (C ABI / plugin) vs golden fixtures from the reference and the CPU oracle.
Bar: match indices exact; dtype uint32 (tests/frontend/matcher/test_superglue_matcher.py:41-42)."""
import pickle

import numpy as np
import pytest

from gtsfm_b200 import synthetic as syn
from gtsfm_b200.gtsfm_api import Keypoints
from gtsfm_b200.matcher import B200SuperGlueMatcher, SuperGlueEngine

pytestmark = pytest.mark.gpu


# 12: 2048 x 1900, 13: 5000 x 5000 keypoints (100 MB coupling matrix), 14: 600 x 8300 (more columns than the persistent
# Sinkhorn kernel holds: the multi-launch path)
@pytest.mark.parametrize("seed", [5, 6, 9, 12, 13, 14])
def test_matches_equal_reference_fixture(b200_ctx, golden_dir, seed):
    fx = np.load(golden_dir / f"superglue_{seed}.npz")
    kp0, sc0, d0, kp1, sc1, d1, _ = syn.synthetic_features(seed, int(fx["n0"]), int(fx["n1"]))
    profile = str(fx["profile"]) if "profile" in fx else "full"
    assert seed < 12 or len(fx["matches"]) > 500, "the large fixtures must carry real matches"
    eng = SuperGlueEngine(syn.superglue_state_dict(1, profile), ctx=b200_ctx)
    m, sc = eng.match(kp0, sc0, d0, kp1, sc1, d1, (480, 640, 3), (480, 640, 3), return_scores=True)
    assert m.dtype == np.uint32 and m.shape == fx["matches"].shape, f"{m.shape} vs {fx['matches'].shape}"
    assert np.array_equal(m, fx["matches"])
    np.testing.assert_allclose(sc, fx["mscores"], atol=5e-4)


def test_final_descriptors_match_oracle(b200_ctx):
    from oracle.superglue_ref import superglue_match

    kp0, sc0, d0, kp1, sc1, d1, _ = syn.synthetic_features(31, 150, 170, 300, 400)
    sd = syn.superglue_state_dict(1)
    tr = {}
    ref = superglue_match(kp0, sc0, d0, kp1, sc1, d1, (300, 400, 3), (300, 400, 3), sd, trace=tr)
    eng = SuperGlueEngine(sd, ctx=b200_ctx)
    m = eng.match(kp0, sc0, d0, kp1, sc1, d1, (300, 400, 3), (300, 400, 3))
    assert np.array_equal(m, ref)
    g0 = b200_ctx.debug_fetch("sg_desc0", 150 * 256).reshape(150, 256)
    np.testing.assert_allclose(g0, tr["desc0"].T, atol=1e-4)


def test_plugin_contract(tmp_path, golden_dir):
    wpath = tmp_path / "superglue_outdoor.pth"
    syn.save_pth(syn.superglue_state_dict(1), wpath)
    matcher = B200SuperGlueMatcher(weights_path=wpath)
    pickle.dumps(matcher)
    kp0, sc0, d0, kp1, sc1, d1, _ = syn.synthetic_features(5, 300, 350)
    k0, k1 = Keypoints(kp0, responses=sc0), Keypoints(kp1, responses=sc1)
    m = matcher.match(k0, k1, d0, d1, (480, 640, 3), (480, 640, 3))
    pickle.dumps(matcher)
    assert isinstance(m, np.ndarray) and m.dtype == np.uint32
    assert np.array_equal(m, np.load(golden_dir / "superglue_5.npz")["matches"])
    assert np.all(m[:, 0] < 300) and np.all(m[:, 1] < 350)
    assert len(np.unique(m[:, 0])) == len(m) and len(np.unique(m[:, 1])) == len(m)
    empty = Keypoints(np.zeros((0, 2), np.float32), responses=np.zeros(0, np.float32))
    assert matcher.match(empty, k1, np.zeros((0, 256), np.float32), d1, (480, 640, 3), (480, 640, 3)).size == 0
    with pytest.raises(ValueError):
        matcher.match(Keypoints(kp0), k1, d0, d1, (480, 640, 3), (480, 640, 3))
    with pytest.raises(Exception):
        matcher.match(k0, k1, d0[:, :128], d1, (480, 640, 3), (480, 640, 3))
