"""CPU suite of the two-way matcher: the cv2 restatement and the exact path's integer arithmetic against the goldens written
by the reference's unmodified TwoWayMatcher (oracle/make_golden_twoway.py); the plugin's host-side contract."""
import importlib
import pickle
from pathlib import Path

import numpy as np
import pytest

from oracle import twoway_ref

CASES = ["lund_stored", "sift", "kaze", "orb", "dummy"]
EXACT = ["lund_stored", "sift", "orb"]
RATIOS = [("ratio", 0.8), ("noratio", None)]


def load(golden_dir, name):
    fx = np.load(golden_dir / f"twoway_{name}.npz")
    dt = str(fx["dtype"])
    return fx, fx["desc0"].astype(dt), fx["desc1"].astype(dt)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("tag,ratio", RATIOS)
def test_oracle_vs_golden(golden_dir, name, tag, ratio):
    fx, a, b = load(golden_dir, name)
    m, d = twoway_ref.twoway_match(a, b, ratio)
    assert m.dtype == np.uint32 and np.array_equal(m, fx[f"matches_{tag}"])
    assert np.array_equal(d.view(np.uint32), fx[f"dist_{tag}"].view(np.uint32))


@pytest.mark.parametrize("name", EXACT)
@pytest.mark.parametrize("tag,ratio", RATIOS)
def test_u8_arithmetic_reproduces_cv2(golden_dir, name, tag, ratio):
    """int norms and dot products, d^2 = |a|^2 + |b|^2 - 2 a.b, float32(sqrt(float32(d^2))), then (distance, index) order."""
    fx, a, b = load(golden_dir, name)
    m, d = twoway_ref.twoway_from_distances(twoway_ref.u8_distances(a, b), ratio)
    assert np.array_equal(m, fx[f"matches_{tag}"])
    assert np.array_equal(d.view(np.uint32), fx[f"dist_{tag}"].view(np.uint32))


def test_dummy_golden_is_the_reference_known_answer(golden_dir):
    fx, _, _ = load(golden_dir, "dummy")
    assert np.array_equal(fx["matches_ratio"], [[9, 5], [2, 4], [3, 2], [0, 3]])


def test_plugin_pickles_without_gpu_and_rejects_hamming():
    from gtsfm_b200.matcher import B200TwoWayMatcher, MatchingDistanceType

    m = B200TwoWayMatcher(ratio_test_threshold=0.8)
    m2 = pickle.loads(pickle.dumps(m))
    assert m2._ratio_test_threshold == 0.8 and m2._engine is None
    with pytest.raises(NotImplementedError):
        B200TwoWayMatcher(distance_type=MatchingDistanceType.HAMMING)


def test_sift_overlay_names_existing_classes():
    import yaml

    cfg = yaml.safe_load((Path(__file__).resolve().parent.parent / "configs" / "sift_front_end_b200.yaml").read_text())
    assert cfg["defaults"] == ["sift_front_end", "_self_"]
    co = cfg["cluster_optimizer"]
    matcher = co["correspondence_generator"]["matcher"]["matcher_obj"]
    verifier = co["two_view_estimator"]["two_view_estimator_obj"]["verifier"]
    assert matcher["ratio_test_threshold"] == 0.8
    for target in (matcher["_target_"], verifier["_target_"]):
        mod, cls = target.rsplit(".", 1)
        assert hasattr(importlib.import_module(mod), cls), target
