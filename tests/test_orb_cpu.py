"""CPU suite of the ORB detector-descriptor: the NumPy restatement (oracle/orb_ref.py) against cv2, stage by stage and whole,
the goldens written by the reference's unmodified ORBDetectorDescriptor (oracle/make_golden_orb.py), the probed rBRIEF
pattern, and the plugin's host-side contract."""
import pickle
from pathlib import Path

import numpy as np
import pytest

from oracle import orb_ref

ROOT = Path(__file__).resolve().parent.parent
cv2 = pytest.importorskip("cv2")


def golden(golden_dir, name):
    f = np.load(golden_dir / f"orb_{name}.npz")
    return {k: f[k] for k in orb_ref.FIELDS}, f["desc"], str(f["cv2_version"])


def assert_same(a, da, b, db):
    """Same keypoint set keyed by (octave, x, y), every field equal as float32 bits, identical descriptor bytes."""
    ia, ib = orb_ref.same_keypoints(a, da, b, db)
    for f in orb_ref.FIELDS:
        assert np.array_equal(np.asarray(a[f])[ia].view(np.int32), np.asarray(b[f])[ib].view(np.int32)), f
    assert np.array_equal(da[ia], db[ib])


def random_image(seed, h, w):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w), dtype=np.uint8)
    return cv2.GaussianBlur(img, (0, 0), 0.8 + 0.3 * (seed % 3))


@pytest.mark.parametrize("name", orb_ref.CASES)
def test_restatement_equals_golden(golden_dir, name):
    ref, desc, version = golden(golden_dir, name)
    if cv2.__version__ != version:
        pytest.skip(f"goldens written with cv2 {version}, this is {cv2.__version__}")
    arr, mask = orb_ref.case_image(name, golden_dir)
    got, d = orb_ref.cv2_orb(arr, mask)
    for f in orb_ref.FIELDS:
        assert np.array_equal(got[f], ref[f]), f
    assert np.array_equal(np.zeros((0, 32), np.uint8) if d is None else d, desc)
    mine, dm = orb_ref.orb(arr, mask)
    assert_same(mine, dm, ref, desc)


@pytest.mark.parametrize("seed,h,w", [(0, 480, 640), (1, 333, 517), (2, 701, 299), (3, 160, 160)])
def test_restatement_equals_cv2_on_random_images(seed, h, w):
    arr = random_image(seed, h, w)
    mask = None
    if seed % 2:
        mask = (np.random.default_rng(seed + 10).random((h, w)) < 0.8).astype(np.uint8)
    a, da = orb_ref.orb(arr, mask)
    b, db = orb_ref.cv2_orb(arr, mask)
    assert len(a["x"]) > 0
    assert_same(a, da, b, np.zeros((0, 32), np.uint8) if db is None else db)


def test_output_order_is_level_then_response_then_y_x(golden_dir):
    rec, _ = orb_ref.orb(*orb_ref.case_image("lund_1", golden_dir))
    key = list(zip(rec["octave"], -rec["response"].astype(np.float64), rec["y"], rec["x"]))
    assert key == sorted(key)


def test_features_per_level_and_level_sizes():
    assert orb_ref.features_per_level() == [109, 90, 75, 63, 52, 44, 36, 31]
    assert orb_ref.level_sizes(1135, 760)[7] == (317, 212)


@pytest.mark.parametrize("seed", range(6))
def test_pyramid_is_the_linear_exact_resize_chain(seed):
    h, w = 200 + 37 * seed, 150 + 53 * seed
    img = random_image(seed, h, w)
    levels = orb_ref.pyramid(img)
    prev = img
    for (lh, lw), lv in zip(orb_ref.level_sizes(h, w)[1:], levels[1:]):
        prev = cv2.resize(prev, (lw, lh), interpolation=cv2.INTER_LINEAR_EXACT)
        assert np.array_equal(lv, prev)


@pytest.mark.parametrize("seed", range(4))
def test_fast_score_equals_cv2_response(seed):
    img = random_image(seed, 240, 320)
    score = orb_ref.fast_score(img)
    y, x = orb_ref.fast_nms(score)
    kps = cv2.FastFeatureDetector_create(20, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16).detect(img)
    assert len(kps) > 0
    assert {(int(k.pt[0]), int(k.pt[1])): k.response for k in kps} == {(int(b), int(a)): float(score[a, b]) for a, b in zip(y, x)}


@pytest.mark.parametrize("seed", range(4))
def test_blur_equals_cv2_separable_filter(seed):
    """ORB blurs a sub-matrix of its padded pyramid, which cv2 does with its separable float filter; cv2.GaussianBlur on a
    whole image takes a fixed-point path and differs, so cv2.sepFilter2D is the comparison."""
    img = random_image(seed, 97 + seed, 131)
    k = cv2.getGaussianKernel(7, 2, ktype=cv2.CV_32F)
    assert np.array_equal(orb_ref.gaussian_taps(), k.ravel())
    assert np.array_equal(orb_ref.blur(img), cv2.sepFilter2D(img, -1, k, k, borderType=cv2.BORDER_REFLECT_101))
    assert not np.array_equal(orb_ref.blur(img), cv2.GaussianBlur(img, (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101))


def test_fast_atan2_equals_cv2():
    rng = np.random.default_rng(0)
    y = rng.integers(-200000, 200000, 5000).astype(np.float32)
    x = rng.integers(-200000, 200000, 5000).astype(np.float32)
    y[:50], x[50:100] = 0, 0
    got = orb_ref.fast_atan2(y, x)
    ref = np.array([cv2.fastAtan2(float(a), float(b)) for a, b in zip(y, x)], np.float32)
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))


def test_mask_rule_keeps_keypoints_where_the_carried_mask_is_full(golden_dir):
    """A 0 / 1 mask and a 0 / 255 mask select the same keypoints; on levels > 0 only where the resized mask is 255."""
    arr, _ = orb_ref.case_image("lund_3", golden_dir)
    m = (np.random.default_rng(5).random(arr.shape) < 0.7).astype(np.uint8)
    a, da = orb_ref.orb(arr, m)
    for scale in (1, 255):
        b, db = orb_ref.cv2_orb(arr, m * scale)
        assert_same(a, da, b, db)


def test_pattern_rederived_equals_committed_table():
    from oracle import make_orb_pattern

    committed = orb_ref.load_pattern()
    assert committed.shape == (512, 2) and np.abs(committed).max() <= 13
    assert np.array_equal(make_orb_pattern.probe(), committed)
    assert orb_ref.PATTERN_INC.read_text() == make_orb_pattern.render(committed)


def test_plugin_pickles_without_device_state():
    from gtsfm_b200.detector_descriptor import B200ORBDetectorDescriptor

    p = B200ORBDetectorDescriptor(max_keypoints=300)
    q = pickle.loads(pickle.dumps(p))
    assert q.max_keypoints == 300 and q._engine is None


def test_plugin_top_k_and_empty_results(golden_dir):
    from gtsfm_b200 import _lib
    from gtsfm_b200.detector_descriptor import orb_keypoints

    rec, desc = orb_ref.orb(*orb_ref.case_image("lund_2", golden_dir))
    kp = np.zeros(len(rec["x"]), _lib.SIFT_KEYPOINT_DTYPE)
    for f in orb_ref.FIELDS:
        kp[f] = rec[f]
    for k in (1, 57, 499, 500, 5000):
        keypoints, d = orb_keypoints(kp, desc, k)
        sel = np.arange(len(kp)) if k >= len(kp) else np.argpartition(-rec["response"].astype(np.float64), k)[:k]
        assert set(map(tuple, keypoints.coordinates)) == set(map(tuple, np.stack([rec["x"], rec["y"]], 1)[sel].astype(np.float64)))
        assert d.dtype == np.uint8 and d.shape == (min(k, len(kp)), 32)
    keypoints, d = orb_keypoints(kp[:0], desc[:0], 5000)
    assert keypoints.coordinates.shape == (0, 2) and d.shape == (0, 32) and d.dtype == np.uint8


def test_reference_plugin_restatement_gives_empty_results_without_keypoints(golden_dir):
    c, s, r, d = orb_ref.detect_and_describe(*orb_ref.case_image("flat", golden_dir))
    assert c.shape == (0, 2) and d.shape == (0, 32)


def test_config_targets_exist():
    import importlib

    import yaml

    cfg = yaml.safe_load((ROOT / "configs" / "orb_front_end_b200.yaml").read_text())
    cg = cfg["cluster_optimizer"]["correspondence_generator"]
    for target in (cg["detector_descriptor"]["detector_descriptor_obj"]["_target_"], cg["matcher"]["matcher_obj"]["_target_"]):
        mod, name = target.rsplit(".", 1)
        assert hasattr(importlib.import_module(mod), name)
    assert cg["matcher"]["matcher_obj"]["ratio_test_threshold"] == 0.8
