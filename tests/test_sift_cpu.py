"""CPU suite of the SIFT detector-descriptor: the cv2 restatement against the goldens written by the reference's unmodified
SIFTDetectorDescriptor (oracle/make_golden_sift.py), the parity criterion checked on cv2's own scalar build, and the plugin's
host-side contract."""
import importlib
import pickle
from pathlib import Path

import numpy as np
import pytest

from oracle import sift_ref

ROOT = Path(__file__).resolve().parent.parent


def golden(golden_dir, name):
    f = np.load(golden_dir / f"sift_{name}.npz")
    return {k: f[k] for k in sift_ref.FIELDS}, f["desc"], str(f["cv2_version"])


@pytest.mark.parametrize("name", sift_ref.CASES)
def test_restatement_reproduces_golden(golden_dir, name):
    import cv2

    ref, desc, version = golden(golden_dir, name)
    if cv2.__version__ != version:
        pytest.skip(f"goldens written with cv2 {version}, this is {cv2.__version__}")
    arr, mask = sift_ref.case_image(name, golden_dir)
    got, d = sift_ref.cv2_sift(arr, mask)
    for f in sift_ref.FIELDS:
        assert np.array_equal(got[f], ref[f]), f
    assert np.array_equal(np.zeros((0, 128), np.uint8) if d is None else d.astype(np.uint8), desc)


@pytest.mark.parametrize("i", [1, 2])
def test_cv2_scalar_build_meets_the_parity_bar(golden_dir, i):
    """The bar the GPU path is held to is one cv2 itself meets: its scalar build (no SIMD, no IPP) against its default."""
    import cv2

    ref, desc, version = golden(golden_dir, f"lund_{i}")
    if cv2.__version__ != version:
        pytest.skip(f"goldens written with cv2 {version}, this is {cv2.__version__}")
    opt, ipp = cv2.useOptimized(), cv2.ipp.useIPP()
    try:
        cv2.setUseOptimized(False)
        cv2.ipp.setUseIPP(False)
        got, d = sift_ref.cv2_sift(sift_ref.case_image(f"lund_{i}", golden_dir)[0])
    finally:
        cv2.setUseOptimized(opt)
        cv2.ipp.setUseIPP(ipp)
    p = sift_ref.parity(got, d.astype(np.uint8), ref, desc)
    assert p["a_in_b"] >= 0.99 and p["b_in_a"] >= 0.99 and abs(p["count_ratio"] - 1) <= 0.01 and p["desc_within_1"] >= 0.995, p
    assert p["a_in_b"] < 1.0  # the scalar build is a different float computation, not a copy


def test_correspondence_rejects_other_octaves_and_angles():
    a = {"x": np.array([10.0, 20.0], np.float32), "y": np.array([5.0, 5.0], np.float32), "octave": np.array([1, 2], np.int32),
         "angle": np.array([359.9, 10.0], np.float32)}
    b = {"x": np.array([10.005, 20.0], np.float32), "y": np.array([5.0, 5.0], np.float32), "octave": np.array([1, 3], np.int32),
         "angle": np.array([0.2, 10.0], np.float32)}
    ia, ib = sift_ref.correspond(a, b)
    assert ia.tolist() == [0] and ib.tolist() == [0]


def test_plugin_pickles_without_gpu_and_validates_input():
    from gtsfm_b200.detector_descriptor import B200SIFTDetectorDescriptor, SiftEngine
    from gtsfm_b200.gtsfm_api import Image

    det = B200SIFTDetectorDescriptor(max_keypoints=1234)
    det2 = pickle.loads(pickle.dumps(det))
    assert det2.max_keypoints == 1234 and det2._engine is None
    with pytest.raises(ValueError):  # gtsfm/utils/images.py:39-40, raised before any device work
        det.detect_and_describe(Image(np.zeros((16, 16, 2), np.uint8)))
    assert det._engine is None
    assert SiftEngine.images_per_call(2880, 3840) >= 1 and SiftEngine.images_per_call(760, 1135) <= 64


def test_full_sift_overlay_names_existing_classes():
    import yaml

    cfg = yaml.safe_load((ROOT / "configs" / "sift_front_end_b200_full.yaml").read_text())
    assert cfg["defaults"] == ["sift_front_end_b200", "_self_"]
    det = cfg["cluster_optimizer"]["correspondence_generator"]["detector_descriptor"]["detector_descriptor_obj"]
    assert det["max_keypoints"] == 5000
    mod, cls = det["_target_"].rsplit(".", 1)
    assert hasattr(importlib.import_module(mod), cls), det["_target_"]
