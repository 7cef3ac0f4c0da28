"""CPU suite for the cycle-consistent rotation view-graph filter: the NumPy oracle (oracle/view_graph_ref.py) against the
committed fixtures, the host build of the device cycle error (csrc/view_graph_math.cuh) against the oracle, the plugin's
argument checks, and the Hydra config that swaps it in."""
import importlib
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import make_golden_view_graph as mg
from oracle import view_graph_ref as ref

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"


def _cases():
    out = []
    for f in ("view_graph_scenes.npz", "view_graph_lund_door.npz"):
        d = np.load(GOLDEN / f)
        names = [str(n) for n in d["names"]] if "names" in d else ["lund_door"]
        out += [(d, name, str(run)) for name in names for run in d["runs"]]
    return out


@pytest.mark.parametrize("form", ["literal", "vectorised"])
def test_oracle_reproduces_fixtures(form):
    run = ref.run_literal if form == "literal" else ref.run_vectorised
    for d, name, r in _cases():
        crit, thr = mg.RUNS[r]
        keep, agg, ncyc = run(d[f"{name}/edges"], d[f"{name}/R"], crit, thr)
        assert np.array_equal(keep, d[f"{name}/{r}/keep"]), (name, r)
        assert np.array_equal(ncyc, d[f"{name}/{r}/num_cycles"]), (name, r)
        if form == "literal":
            assert np.array_equal(agg, d[f"{name}/{r}/aggregate"], equal_nan=True), (name, r)
        else:
            assert np.allclose(agg, d[f"{name}/{r}/aggregate"], rtol=1e-12, atol=1e-12, equal_nan=True), (name, r)


def test_fixture_covers_the_cases():
    d = np.load(GOLDEN / "view_graph_scenes.npz")
    assert d["tree_30/median_7/num_cycles"].sum() == 0 and d["tree_30/median_7/keep"].all()
    assert list(d["triangle/median_7/num_cycles"]) == [1, 1, 1]
    assert 2 in set(d["two_triangles/median_7/num_cycles"])  # an even count: the mean of the two middle errors
    assert d["sparse_large_ids/edges"].max() > 10 ** 5
    errs = ref.triplet_errors(d["near_180/edges"], d["near_180/R"], ref.triplets_vectorised(d["near_180/edges"]))
    assert errs.max() > 179.9
    for name in (str(n) for n in d["names"]):
        assert len(np.unique(d[f"{name}/edges"], axis=0)) == len(d[f"{name}/edges"])
        for r in d["runs"]:
            a = d[f"{name}/{r}/aggregate"]
            assert not np.any(np.abs(a[~np.isnan(a)] - mg.RUNS[str(r)][1]) < 1e-9), (name, r)  # no decision on a knife edge


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    exe = tmp_path_factory.mktemp("vg") / "test_view_graph_math"
    subprocess.run([cxx, "-O2", "-std=c++17", "-x", "c++", str(ROOT / "tests/cpp/test_view_graph_math.cpp"), "-o", str(exe)], check=True)

    def run(triples):
        lines = [" ".join(repr(float(v)) for v in np.concatenate([np.ravel(m) for m in t])) for t in triples]
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return np.array(out.split(), float)

    return run


def test_host_cycle_error_equals_oracle(harness):
    for f in ("view_graph_scenes.npz", "view_graph_lund_door.npz"):
        d = np.load(GOLDEN / f)
        for name in ([str(n) for n in d["names"]] if "names" in d else ["lund_door"]):
            e, R = d[f"{name}/edges"], d[f"{name}/R"]
            T = ref.triplets_vectorised(e)
            if len(T) == 0:
                continue
            idx = [ref.edge_index(e, T[:, x], T[:, y]) for x, y in ((0, 1), (1, 2), (0, 2))]
            got = harness([(R[a], R[b], R[c]) for a, b, c in zip(*idx)])
            want = np.array([ref.cycle_error_deg(R[a], R[b], R[c]) for a, b, c in zip(*idx)])
            assert np.allclose(got, want, rtol=1e-12, atol=1e-12), (name, np.abs(got - want).max())


def test_plugin_argument_checks():
    from gtsfm_b200.gtsfm_api import EdgeErrorAggregationCriterion, Rot3
    from gtsfm_b200.view_graph import B200CycleConsistentRotationViewGraphEstimator as Est

    with pytest.raises(ValueError):
        Est("MEAN_EDGE_ERROR")
    with pytest.raises(ValueError):
        Est(3)
    est = Est(EdgeErrorAggregationCriterion.MIN_EDGE_ERROR, error_threshold=5.0)
    assert est._edge_error_aggregation_criterion == EdgeErrorAggregationCriterion.MIN_EDGE_ERROR
    assert Est("MEDIAN_EDGE_ERROR")._error_threshold == 7.0
    assert est.run({}, {}, [], {}, [], {}) == set() and est._ctx is None  # no context, no launch
    for bad in ({(2, 1): np.eye(3)}, {(1, 1): np.eye(3)}, {(-1, 2): np.eye(3)}, {(0, 1): None}, {(0, 1): np.full((3, 3), np.nan)},
                {(0, 1): np.eye(2)}, {(0, 1): Rot3(np.eye(3)), (1, 2): np.array([[1.0, 0, 0], [0, np.inf, 0], [0, 0, 1]])}):
        with pytest.raises(ValueError):
            est.run(bad, {}, [], {}, [], {})
    assert est._ctx is None
    edges, R = Est.arrays({(0, 1): Rot3(np.eye(3)), (3, 7): np.eye(3)})
    assert edges.dtype == np.int32 and edges.tolist() == [[0, 1], [3, 7]] and R.shape == (2, 3, 3)


def test_hydra_config_swaps_the_estimator():
    import yaml

    text = (ROOT / "configs" / "deep_front_end_b200_view_graph.yaml").read_text()
    cfg = yaml.safe_load(text)
    assert cfg["defaults"] == ["deep_front_end_b200", "_self_"]
    node = cfg["cluster_optimizer"]["multiview_optimizer"]["view_graph_estimator"]
    assert node == {"_target_": "gtsfm_b200.view_graph.B200CycleConsistentRotationViewGraphEstimator"}
    # the criterion comes from the reference config the defaults compose (deep_front_end.yaml: MEDIAN_EDGE_ERROR)
    module, _, name = node["_target_"].rpartition(".")
    est = getattr(importlib.import_module(module), name)(edge_error_aggregation_criterion="MEDIAN_EDGE_ERROR")
    from gtsfm_b200.gtsfm_api import ViewGraphEstimatorBase

    assert isinstance(est, ViewGraphEstimatorBase)
