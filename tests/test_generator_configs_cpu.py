"""CPU: the correspondence configs that serve a reference correspondence config through B200CorrespondenceGenerator.

GTSfM's runner swaps the whole correspondence generator with `--correspondence_generator_config_name NAME`: it composes
gtsfm/configs/correspondence/NAME.yaml on its own and instantiates its `CorrespondenceGenerator` node (gtsfm/runner.py,
_set_mvo_overwrites).  A file without a defaults list composes to its own content, so instantiating that node as
hydra.utils.instantiate does - import `_target_`, call it with the other keys - is what the runner builds.  Construction touches
no device: the front end is made on first use."""
import importlib
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
# reference config -> (correspondence file, the main config of this repository it runs with, detector, matcher)
CONFIGS = {"sift_front_end": ("sift_b200_generator.yaml", "sift_front_end_b200", "sift", "twoway"),
           "megaloc_sift_frontend": ("sift_b200_generator.yaml", "megaloc_sift_frontend_b200", "sift", "twoway"),
           "orb": ("orb_b200_generator.yaml", "orb_front_end_b200", "orb", "twoway"),
           "d2net": ("d2net_b200_generator.yaml", "d2net_front_end_b200", "d2net", "twoway"),
           "superglue": ("superglue_b200_generator.yaml", "deep_front_end_b200", "superpoint", "superglue")}


def _instantiate(node: dict):
    module, _, name = node["_target_"].rpartition(".")
    args = {k: v for k, v in node.items() if k != "_target_"}
    assert not any(isinstance(v, dict) for v in args.values()), "nested nodes would be instantiated first"
    return getattr(importlib.import_module(module), name)(**args)


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_generator_config_constructs(config):
    import yaml

    from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator

    name, main, detector, matcher = CONFIGS[config]
    text = (ROOT / "configs" / "correspondence" / name).read_text()
    cfg = yaml.safe_load(text)
    assert list(cfg) == ["CorrespondenceGenerator"], "no defaults list: the file composes to itself"
    assert "# L2 seam" in text and f"--correspondence_generator_config_name {Path(name).stem}`" in text
    assert f"--config_name {main}" in text and (ROOT / "configs" / f"{main}.yaml").exists()
    node = cfg["CorrespondenceGenerator"]
    assert node["_target_"] == "gtsfm_b200.correspondence_generator.B200CorrespondenceGenerator"
    assert (node["detector"], node["matcher"], node["max_keypoints"]) == (detector, matcher, 5000)
    assert node.get("ratio_test_threshold") == (0.8 if matcher == "twoway" else None)
    gen = _instantiate(node)
    assert isinstance(gen, B200CorrespondenceGenerator) and (gen._detector, gen._matcher) == (detector, matcher)


def test_every_correspondence_config_is_tested():
    assert sorted(p.name for p in (ROOT / "configs" / "correspondence").glob("*.yaml")) == sorted({v[0] for v in CONFIGS.values()})
