"""CPU: the MegaLoc oracle (oracle/megaloc_ref.py) against the golden made by the reference module's own forward
(oracle/make_golden_megaloc.py), the uint8 resize restatement against torchvision, the weight layout, the plugin's transforms,
pickling and the Hydra config."""
import importlib
import pickle
from pathlib import Path

import numpy as np
import pytest
import torch

from gtsfm_b200 import synthetic as syn, weights
from oracle import megaloc_ref

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def sd():
    return syn.megaloc_state_dict(5)


def test_oracle_equals_golden(sd, golden_dir):
    z = np.load(golden_dir / "megaloc.npz")
    u8 = megaloc_ref.golden_frames_u8()
    assert np.array_equal(u8.reshape(len(u8), -1).sum(1, dtype=np.int64), z["u8_322_sum"])
    x = megaloc_ref.normalise(u8)
    t = megaloc_ref.tensors(sd)
    d, tok = megaloc_ref.megaloc_forward(t, x[:2], return_tokens=True)
    assert np.abs(d - z["desc_322"][:2]).max() <= 1e-6
    assert np.abs(tok[0][z["tokens_0_rows"]] - z["tokens_0"]).max() <= 1e-5 * np.abs(z["tokens_0"]).max()
    assert np.abs(megaloc_ref.megaloc_forward(t, x[[0, 2, 0]]) - z["desc_batch_0_2_0"]).max() <= 1e-6
    im = megaloc_ref.normalise(np.ascontiguousarray(syn.synthetic_frame(70, 224, 308).transpose(2, 0, 1)))[None]
    assert np.abs(megaloc_ref.megaloc_forward(t, im) - z["desc_224x308"]).max() <= 1e-6
    # the seeded model tells frames apart
    assert z["cos_322"][~np.eye(4, dtype=bool)].max() <= 0.95
    assert (z["desc_shift_0"] @ z["desc_322"].T).argmax() == 0


def test_pos_table_matches_torch_bicubic(sd):
    pe = torch.from_numpy(sd["backbone.model.pos_embed"])
    for gh, gw in ((23, 23), (16, 22), (11, 30), (37, 40)):
        want = torch.nn.functional.interpolate(pe[0, 1:].reshape(1, 37, 37, -1).permute(0, 3, 1, 2), mode="bicubic", antialias=False,
                                               scale_factor=((gh + 0.1) / 37, (gw + 0.1) / 37))
        want = want.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)
        got = megaloc_ref.pos_table(pe, gh, gw)[:, 1:]
        assert torch.abs(got - want).max() < 1e-6, (gh, gw)
    assert megaloc_ref.pos_table(pe, 37, 37) is pe


def test_resize_restatement_is_torchvision():
    if torch.backends.cpu.get_cpu_capability() == "DEFAULT":
        pytest.skip("torch's non-vectorised build resamples uint8 through another code path than the one restated")
    from torchvision.transforms import v2 as T

    rs = T.Resize(size=(322, 322), antialias=True)
    for i, (h, w) in enumerate(((760, 1135), (480, 640), (300, 300), (322, 500), (200, 322), (3840, 2880))):
        im = syn.synthetic_frame(i, h, w)
        assert np.array_equal(megaloc_ref.resize_u8(im), rs(torch.from_numpy(im).permute(2, 0, 1)).numpy()), (h, w)


def test_state_dict_layout(sd):
    assert len(sd) == 190 and sum(v.size for v in sd.values()) == 228640321
    assert set(weights.MEGALOC_ORDER) == set(sd) - {"backbone.model.mask_token"}
    blob = weights.pack_megaloc(sd)
    assert blob.dtype == np.float32 and blob.size == weights.MEGALOC_BLOB_FLOATS
    assert blob[-1] == sd["aggregator.linear.bias"][-1]
    shapes = {"backbone.model.pos_embed": (1, 1370, 768), "backbone.model.patch_embed.proj.weight": (768, 3, 14, 14),
              "backbone.model.blocks.11.attn.qkv.weight": (2304, 768), "aggregator.agg.score.3.weight": (64, 512, 1, 1),
              "aggregator.agg.dust_bin": (), "aggregator.linear.weight": (8448, 16640)}
    for k, s in shapes.items():
        assert sd[k].shape == s, k


def test_checkpoint_file_round_trip(tmp_path):
    small = {"a": np.arange(6, dtype=np.float32).reshape(2, 3)}
    syn.save_pth(small, tmp_path / "megaloc.torch")
    assert np.array_equal(weights.load_megaloc(tmp_path / "megaloc.torch")["a"], small["a"])
    with pytest.raises(FileNotFoundError):
        weights.load_megaloc(tmp_path / "missing.torch")


def test_plugin_transforms_and_pickle(tmp_path):
    from gtsfm_b200.global_descriptor import B200MegaLocGlobalDescriptor

    with pytest.raises(FileNotFoundError):
        B200MegaLocGlobalDescriptor(weights_path=tmp_path / "missing.torch")
    g = B200MegaLocGlobalDescriptor(weights_path={"x": np.zeros(1)})
    resize, batch = g.get_preprocessing_transforms()
    frames = [syn.synthetic_frame(90 + i, 300, 420) for i in range(2)]
    u8 = torch.stack([resize(f) for f in frames])
    assert u8.dtype == torch.uint8 and u8.shape == (2, 3, 322, 322)
    assert np.array_equal(u8.numpy(), np.stack([megaloc_ref.resize_u8(f) for f in frames]))
    x = batch(u8)
    # the reference's batch transform (megaloc_global_descriptor.py:52-60)
    from torchvision.transforms import v2 as T

    want = T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])(u8.type(torch.float32) / 255.0)
    assert torch.equal(x, want) and np.array_equal(x.numpy(), megaloc_ref.normalise(u8.numpy()))
    g2 = pickle.loads(pickle.dumps(g))
    assert g2._engine is None and g2._device == 0


def test_hydra_config_targets():
    import yaml

    cfg = yaml.safe_load((ROOT / "configs" / "megaloc_sift_frontend_b200.yaml").read_text())
    assert cfg["defaults"][0] == "megaloc_sift_frontend"
    ipg, co = cfg["image_pairs_generator"], cfg["cluster_optimizer"]["correspondence_generator"]
    targets = [ipg["global_descriptor"]["global_descriptor_obj"]["_target_"], ipg["retriever"]["_target_"],
               co["detector_descriptor"]["detector_descriptor_obj"]["_target_"], co["matcher"]["matcher_obj"]["_target_"],
               cfg["cluster_optimizer"]["two_view_estimator"]["two_view_estimator_obj"]["verifier"]["_target_"]]
    assert [t.rsplit(".", 1)[1] for t in targets] == ["B200MegaLocGlobalDescriptor", "B200SimilarityRetriever", "B200SIFTDetectorDescriptor",
                                                       "B200TwoWayMatcher", "B200Ransac"]
    for t in targets:
        mod, cls = t.rsplit(".", 1)
        assert hasattr(importlib.import_module(mod), cls), t
    assert ipg["retriever"]["num_matched"] == 20 and ipg["retriever"]["min_score"] == 0.3
    assert co["matcher"]["matcher_obj"]["ratio_test_threshold"] == 0.8
