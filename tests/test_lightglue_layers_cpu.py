"""CPU: the LightGlue oracle's new knobs.  Its fp32 defaults still reproduce the reference fixtures, and its fp64 replay
(the yardstick of tests/test_lightglue_layers_gpu.py) takes the same early-exit and pruning decisions on them, so that
replay is a reference for the decisions and not only for the values."""
import numpy as np
import pytest

from gtsfm_b200 import synthetic as syn
from oracle.lightglue_ref import N_LAYERS, lightglue_match

# every fixture of synthetic features except bench_11 (5000 x 5000, minutes of fp64 on a CPU)
TAGS = ["full_5", "full_6", "prune_7", "stop_8", "prune_9", "stop_10", "bench_12", "full_15"]


@pytest.mark.parametrize("tag", TAGS)
def test_fp32_defaults_reproduce_fixture_and_fp64_takes_the_same_decisions(golden_dir, tag):
    fx = np.load(golden_dir / f"lightglue_{tag}.npz")
    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(int(fx["seed"]), int(fx["n0"]), int(fx["n1"]))
    sd = syn.lightglue_state_dict(2, str(fx["profile"]))
    t32, t64 = {}, {}
    m32 = lightglue_match(kp0, d0, kp1, d1, sd, trace=t32)
    assert np.array_equal(m32, fx["matches"]) and t32["stop"] == int(fx["stop"])
    assert np.array_equal(t32["sizes"], fx["sizes"])
    lightglue_match(kp0, d0, kp1, d1, sd, trace=t64, dtype=np.float64)
    assert t64["stop"] == t32["stop"] and np.array_equal(t64["sizes"], t32["sizes"])
    assert t64["desc0_l0"].dtype == np.float64
    for i in range(t32["stop"]):
        for side in (0, 1):
            assert np.array_equal(t64[f"ind{side}_l{i}"], t32[f"ind{side}_l{i}"]), (i, side)
            if f"keep{side}_l{i}" in t32:
                assert np.array_equal(t64[f"keep{side}_l{i}"], t32[f"keep{side}_l{i}"]), (i, side)
        if f"unconf_l{i}" in t32:
            assert t64[f"unconf_l{i}"] == t32[f"unconf_l{i}"], i
    np.testing.assert_allclose(t64["ind0"], t32["ind0"])


def test_prune_min_kpts_leaves_small_sides_whole():
    """prune_min_kpts = n0: side 0 (n0 rows) is never pruned, side 1 (more rows) still is - as the device decides per side."""
    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(7, 300, 640)
    sd = syn.lightglue_state_dict(2, "prune")
    tr, tr_all = {}, {}
    lightglue_match(kp0, d0, kp1, d1, sd, trace=tr, prune_min_kpts=300)
    lightglue_match(kp0, d0, kp1, d1, sd, trace=tr_all)
    assert all(f"keep0_l{i}" not in tr for i in range(N_LAYERS)) and np.array_equal(tr["ind0"], np.arange(300))
    assert any(f"keep1_l{i}" in tr for i in range(N_LAYERS)) and len(tr["ind1"]) < 640
    assert len(tr_all["ind0"]) < 300, "the case must prune side 0 when the knob is off"
