"""CPU suite for the D2-Net detector-descriptor: the oracle against the goldens made by the unmodified reference plugin, the
normalisation table against the reference's preprocess_image steps, weight packing and the plugin's host-side contract."""
import ctypes
import pickle
from pathlib import Path

import numpy as np
import pytest

from gtsfm_b200 import synthetic as syn
from gtsfm_b200 import weights
from oracle import d2net_ref

ROOT = Path(__file__).resolve().parent.parent


def _reference_preprocess(image_u8_hwc):
    """thirdparty/d2net/lib/utils.py preprocess_image(preprocessing='torch') step by step, then the plugin's float32 cast."""
    image = image_u8_hwc.astype(np.float32)
    image = np.transpose(image, [2, 0, 1])
    image /= 255.0
    mean = np.array([0.485, 0.456, 0.406])
    std = np.array([0.229, 0.224, 0.225])
    return ((image - mean.reshape([3, 1, 1])) / std.reshape([3, 1, 1])).astype(np.float32)


def test_norm_table_is_the_reference_preprocessing_bit_for_bit():
    from gtsfm_b200 import _lib, build

    ramp = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)
    want = _reference_preprocess(ramp)[:, 0, :]
    assert np.array_equal(d2net_ref.norm_table().view(np.uint32), want.view(np.uint32))
    lib = ctypes.CDLL(str(build.build()))
    lib.b2_d2net_norm_table.argtypes = [ctypes.c_void_p]
    got = np.empty((3, 256), np.float32)
    assert lib.b2_d2net_norm_table(_lib.ptr(got)) == 0
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    rgb = syn.synthetic_frame(3, 24, 32)
    assert np.array_equal(d2net_ref.preprocess(rgb), _reference_preprocess(rgb))
    gray = rgb[:, :, 0]
    assert np.array_equal(d2net_ref.preprocess(gray), _reference_preprocess(np.repeat(gray[:, :, None], 3, axis=2)))
    assert np.array_equal(d2net_ref.preprocess(gray[:, :, None]), d2net_ref.preprocess(gray))


@pytest.mark.parametrize("name", ["synthetic", "synthetic_top100", "rgb", "odd_crop", "tiny_crop", "flat"])
def test_oracle_matches_golden(name, golden_dir):
    z = np.load(golden_dir / f"d2net_{name}.npz")
    arr = d2net_ref.case_image(name, golden_dir)
    assert tuple(z["shape"]) == arr.shape and int(z["byte_sum"]) == int(arr.astype(np.int64).sum())
    got = d2net_ref.detect_and_describe(arr, syn.d2net_state_dict(int(z["seed"])), int(z["max_keypoints"]))
    # the golden was written on another CPU: convolution sums may round differently, so values get a small tolerance
    assert np.array_equal(got["cij"], z["cij"])
    assert np.abs(got["scores"] - z["scores"]).max(initial=0) <= 1e-5 * max(1.0, float(np.abs(z["scores"]).max(initial=0)))
    assert np.abs(got["xy"] - z["xy"]).max(initial=0) < 1e-3
    k = len(z["desc"])
    assert np.abs(got["desc"][:k] - z["desc"]).max(initial=0) < 1e-5
    assert int(got["total"]) == int(z["total"])


def test_goldens_are_well_formed(golden_dir):
    for name in d2net_ref.CASES:
        z = np.load(golden_dir / f"d2net_{name}.npz")
        n = len(z["scores"])
        assert z["xy"].shape == (n, 2) and z["cij"].shape == (n, 3) and z["desc"].shape[1] == 512
        assert np.all(np.diff(z["scores"].astype(np.float64)) <= 0), name  # ordered by score
        assert bool(z["fp64_same_set"]), name
        assert 0 < float(z["spread_desc"]) < 1e-5 or n == 0, name


def test_blob_order_size_and_checkpoint_file(tmp_path):
    import torch

    sd = syn.d2net_state_dict(7)
    assert list(sd) == weights.D2NET_ORDER
    blob = weights.pack_d2net(sd)
    assert blob.dtype == np.float32 and blob.size == weights.D2NET_BLOB_FLOATS == 7635264
    assert np.array_equal(blob[:1728], sd["dense_feature_extraction.model.0.weight"].ravel())
    assert np.array_equal(blob[-512:], sd["dense_feature_extraction.model.21.bias"])
    path = tmp_path / "d2_tf.pth"
    torch.save({"model": {k: torch.from_numpy(v) for k, v in sd.items()}}, str(path))
    assert np.array_equal(weights.pack_d2net(weights.load_d2net(path)), blob)
    assert np.array_equal(weights.pack_d2net(weights.load_d2net({"model": sd})), blob)
    with pytest.raises(FileNotFoundError):
        weights.load_d2net(tmp_path / "missing.pth")
    with pytest.raises(KeyError):
        weights.pack_d2net({k: v for k, v in sd.items() if not k.endswith("21.bias")})


def test_plugin_contract_without_gpu(tmp_path):
    from gtsfm_b200.detector_descriptor import B200D2NetDetectorDescriptor
    from gtsfm_b200.gtsfm_api import Image

    with pytest.raises(FileNotFoundError):
        B200D2NetDetectorDescriptor(model_path=tmp_path / "missing.pth")
    with pytest.raises(FileNotFoundError):
        B200D2NetDetectorDescriptor()  # the reference's default path does not exist here
    p = B200D2NetDetectorDescriptor(max_keypoints=123, model_path=syn.d2net_state_dict(7))
    q = pickle.loads(pickle.dumps(p))
    assert q.max_keypoints == 123 and q._engine is None
    # input checks run before any device work
    for bad in (np.zeros((64, 64, 4), np.uint8), np.zeros((64, 64), np.float32), np.zeros((1601, 64), np.uint8),
                np.zeros((1500, 1400), np.uint8), np.zeros((6, 64), np.uint8)):
        with pytest.raises(ValueError):
            p.detect_and_describe(Image(bad))
    assert p._engine is None


def test_hydra_file_targets_import():
    import importlib

    import yaml

    cfg = yaml.safe_load((ROOT / "configs" / "d2net_front_end_b200.yaml").read_text())
    cg = cfg["cluster_optimizer"]["correspondence_generator"]
    targets = [cg["detector_descriptor"]["detector_descriptor_obj"]["_target_"], cg["matcher"]["matcher_obj"]["_target_"]]
    assert targets == ["gtsfm_b200.detector_descriptor.B200D2NetDetectorDescriptor", "gtsfm_b200.matcher.B200TwoWayMatcher"]
    assert cg["detector_descriptor"]["detector_descriptor_obj"]["max_keypoints"] == 5000
    assert cg["matcher"]["matcher_obj"]["ratio_test_threshold"] == 0.8
    for t in targets:
        mod, cls = t.rsplit(".", 1)
        assert hasattr(importlib.import_module(mod), cls)
