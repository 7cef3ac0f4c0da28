"""CPU suite for 1DSfM's outlier rejection: both forms of the NumPy oracle (oracle/mfas_ref.py) against the committed
fixtures and each other, the anchors that do not rest on the restatement (the reference's own all-outliers test, and the
four-node graph of the 1DSfM paper), the host build of csrc/mfas_math.cuh against the oracle, the plugin's key mapping,
argument checks and pickling, and the Hydra config that swaps it in."""
import importlib
import pickle
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import mfas_ref as mr

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"


def _scenes():
    out = []
    for f in ("mfas_scenes.npz", "mfas_lund_door.npz"):
        d = np.load(GOLDEN / f)
        out += [(f, str(n)) for n in d["names"]]
    return out


def _dicts(d, name):
    cam = {tuple(int(x) for x in k): v for k, v in zip(d[f"{name}/cam_keys"], d[f"{name}/cam_vecs"])}
    trk = {tuple(int(x) for x in k): v for k, v in zip(d[f"{name}/trk_keys"], d[f"{name}/trk_vecs"])}
    return cam, trk


@pytest.mark.parametrize("f,name", _scenes())
def test_vectorised_oracle_reproduces_fixture(f, name):
    d = np.load(GOLDEN / f)
    cam, trk = _dicts(d, name)
    (c, t, ic), s = mr.compute_inliers(cam, trk, d[f"{name}/dirs"])
    assert np.array_equal(s.view(np.uint64), d[f"{name}/weight_sum"].view(np.uint64))
    assert np.array_equal([k in c for k in cam], d[f"{name}/inlier_cam"])
    assert np.array_equal([k in t for k in trk], d[f"{name}/inlier_trk"])
    assert sorted(ic) == d[f"{name}/inlier_cameras"].tolist()


@pytest.mark.parametrize("name", ["knn_tracks_input", "zero_weights", "ratio_ties", "disconnected", "tree"])
def test_literal_oracle_reproduces_fixture(name):
    d = np.load(GOLDEN / "mfas_scenes.npz")
    cam, trk = _dicts(d, name)
    _, s = mr.compute_inliers(cam, trk, d[f"{name}/dirs"], form="literal")
    assert np.array_equal(s.view(np.uint64), d[f"{name}/weight_sum"].view(np.uint64))


def test_fixtures_cover_the_cases():
    d = np.load(GOLDEN / "mfas_scenes.npz")
    names = [str(n) for n in d["names"]]
    assert {str(d[f"{n}/method"]) for n in names} == {mr.SAMPLE_INPUT_MEASUREMENTS, mr.SAMPLE_WITH_UNIFORM_DENSITY,
                                                        mr.SAMPLE_WITH_INPUT_DENSITY}
    assert len(d["empty/cam_keys"]) == 0 and len(d["empty/dirs"]) == 2000
    assert len(d["one_direction/dirs"]) == 1
    w = np.concatenate([np.abs(d["zero_weights/meas"] @ x) for x in d["zero_weights/dirs"]])
    assert (w == 0).any() and ((w > 0) & (w < 1e-8)).any()
    assert any(not d[f"{n}/inlier_cam"].all() for n in names)  # some scenes reject camera pairs
    lund = np.load(GOLDEN / "mfas_lund_door.npz")
    assert len(lund["lund_door/trk_keys"]) > 100 and str(lund["lund_door/method"]) == mr.SAMPLE_INPUT_MEASUREMENTS


def test_ratio_ties_break_to_the_lowest_key():
    d = np.load(GOLDEN / "mfas_scenes.npz")
    ea, eb, meas = d["ratio_ties/edge_a"], d["ratio_ties/edge_b"], d["ratio_ties/meas"]
    order, bad = mr.order_vectorised(int(d["ratio_ties/V"]), ea, eb, meas, [1.0, 0.0, 0.0])
    # no source: every node of the two cycles has in = out = 1 except where the cross edge (1, 5) is 0; the lowest id wins
    assert order[0] == 0 and bad.sum() >= 2


def test_oracle_forms_agree_on_seeded_graphs():
    from oracle.make_golden_mfas import knn_graph

    rng = np.random.default_rng(11)
    for n, k, lm in ((15, 3, 0), (20, 4, 12), (12, 5, 30)):
        cam, trk = knn_graph(rng, n, k, 0.3, n_landmarks=lm)
        keys, ea, eb, meas, _ = mr.dense_problem(mr.measurements_from_dicts(cam, trk))
        dirs = mr.unit3(rng.normal(size=(40, 3)))
        a = mr.outlier_weight_sums(len(keys), ea, eb, meas, dirs)
        b = mr.outlier_weight_sums(len(keys), ea, eb, meas, dirs, "literal", keys)
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_anchor_paper_graph():
    """The four-node graph of the 1DSfM paper's Fig. 1, as gtsam's MFAS unit test uses it."""
    E = [(3, 2), (0, 1), (3, 1), (1, 2), (0, 2), (3, 0)]
    for ws, want, viol in (([0.5, 0.75, -0.25, 0.75, 1, 0.5], [0, 1, 3, 2], {(3, 0): 0.5}),
                           ([2, 1.5, 0.5, 0.25, 1, 0.75], [3, 0, 1, 2], {})):
        ms = [(a, b, np.array([w, 0.0, 0.0])) for (a, b), w in zip(E, ws)]
        order, ow = mr.mfas_literal(ms, [1.0, 0.0, 0.0])
        assert order == want and {k: v for k, v in ow.items() if v} == viol
        keys, ea, eb, meas, _ = mr.dense_problem(ms)
        o2, bad = mr.order_vectorised(4, ea, eb, meas, [1.0, 0.0, 0.0])
        assert o2.tolist() == want
        assert {(int(a), int(b)) for a, b, x in zip(ea, eb, bad) if x} == set(viol)


def test_anchor_reference_all_outliers():
    """Uniform sampling, seed 0, K = 2000: every edge to camera 4 is rejected, with wide margins."""
    w = mr.all_outliers_inputs()
    np.random.seed(0)
    dirs = mr.sample_directions(mr.SAMPLE_WITH_UNIFORM_DENSITY, np.zeros((0, 3)))
    (cams, tracks, ic), s = mr.compute_inliers(w, {}, dirs)
    assert set(cams) == {k for k in w if 4 not in k} and ic == {0, 1, 2, 3} and tracks == {}
    keys, ea, eb, _, _ = mr.dense_problem(mr.measurements_from_dicts(w, {}))
    mean = s / 2000
    to4 = np.array([int(keys[a]) & 0xff == 4 for a in ea])
    assert mean[to4].min() > 0.2 and mean[~to4].max() < 0.1


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    exe = tmp_path_factory.mktemp("mfas") / "test_mfas_math"
    subprocess.run([cxx, "-O2", "-std=c++17", "-ffp-contract=off", "-x", "c++", str(ROOT / "tests/cpp/test_mfas_math.cpp"), "-o",
                    str(exe)], check=True)

    def run(V, ea, eb, meas, dirs):
        lines = [f"{V} {len(ea)} {len(dirs)}"]
        lines += [f"{a} {b} " + " ".join(repr(float(x)) for x in m) for a, b, m in zip(ea, eb, meas)]
        lines += [" ".join(repr(float(x)) for x in d) for d in dirs]
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        rows = out.split("\n")
        return [(np.array(rows[2 * k].split(), int), np.array(rows[2 * k + 1].split(), int).astype(bool)) for k in range(len(dirs))]

    return run


@pytest.mark.parametrize("f,name", [s for s in _scenes() if s[1] != "empty"])
def test_host_greedy_equals_oracle(harness, f, name):
    d = np.load(GOLDEN / f)
    V, ea, eb, meas = int(d[f"{name}/V"]), d[f"{name}/edge_a"], d[f"{name}/edge_b"], d[f"{name}/meas"]
    dirs = d[f"{name}/dirs"][:60]
    for (order, bad), x in zip(harness(V, ea, eb, meas, dirs), dirs):
        o2, b2 = mr.order_vectorised(V, ea, eb, meas, x)
        assert np.array_equal(order, o2) and np.array_equal(bad, b2), name


def test_plugin_key_mapping_and_checks():
    from gtsfm_b200.translation_averaging import B200TranslationAveraging1DSFM, dense_edges

    cam = {(0, 1): 1, (0, 5): 1, (1, 5): 1}
    trk = {(7, 1): 1, (3, 5): 1}
    V, ea, eb, perm = dense_edges(cam, trk)
    keys, a2, b2, _, p2 = mr.dense_problem(mr.measurements_from_dicts({k: np.ones(3) for k in cam}, {k: np.ones(3) for k in trk}))
    assert V == len(keys) == 5 and np.array_equal(ea, a2) and np.array_equal(eb, b2) and np.array_equal(perm, p2)
    with pytest.raises(ValueError, match="twice"):
        dense_edges({(1, 2): 1, (2, 1): 1}, {})
    with pytest.raises(ValueError, match="itself"):
        dense_edges({(3, 3): 1}, {})
    with pytest.raises(ValueError):
        dense_edges({(-1, 3): 1}, {})
    t = B200TranslationAveraging1DSFM(projection_sampling_method="SAMPLE_INPUT_MEASUREMENTS", device=0)
    t2 = pickle.loads(pickle.dumps(t))
    assert t2._ctx is None and t2._projection_sampling_method == t.ProjectionSamplingMethod.SAMPLE_INPUT_MEASUREMENTS
    with pytest.raises(ValueError):  # nothing to sample directions from: the reference fails the same way
        t.compute_inliers({}, {})
    assert t._ctx is None


def test_plugin_sampler_matches_the_reference_draw():
    """The constructor seeds NumPy's global RNG; the mirror's samplers consume it as the reference's do."""
    from gtsfm_b200.gtsfm_api import HAVE_GTSFM_1DSFM
    from gtsfm_b200.translation_averaging import B200TranslationAveraging1DSFM

    d = np.load(GOLDEN / "mfas_scenes.npz")
    for name in ("knn_tracks_input", "knn_tracks_uniform"):
        cam, trk = _dicts(d, name)
        t = B200TranslationAveraging1DSFM(projection_sampling_method=str(d[f"{name}/method"]))
        assert np.array_equal(t.projection_directions(cam, trk), d[f"{name}/dirs"])
    if not HAVE_GTSFM_1DSFM:
        t = B200TranslationAveraging1DSFM(projection_sampling_method="SAMPLE_WITH_INPUT_DENSITY")
        with pytest.raises(ValueError):
            t.projection_directions(*_dicts(d, "knn_kde"))


def test_hydra_config_swaps_every_device_stage():
    import yaml

    cfg = yaml.safe_load((ROOT / "configs" / "onedsfm_front_end_b200.yaml").read_text())
    assert cfg["defaults"] == ["onedsfm_front_end", "_self_"]
    co = cfg["cluster_optimizer"]
    mvo = co["multiview_optimizer"]
    targets = [co["correspondence_generator"]["detector_descriptor"]["detector_descriptor_obj"]["_target_"],
               co["correspondence_generator"]["matcher"]["matcher_obj"]["_target_"],
               co["two_view_estimator"]["two_view_estimator_obj"]["verifier"]["_target_"],
               mvo["view_graph_estimator"]["_target_"], mvo["data_association_module"]["_target_"], mvo["trans_avg_module"]["_target_"]]
    assert targets[-1] == "gtsfm_b200.translation_averaging.B200TranslationAveraging1DSFM"
    for t in targets:
        module, _, name = t.rpartition(".")
        assert hasattr(importlib.import_module(module), name), t
    from gtsfm_b200.translation_averaging import B200TranslationAveraging1DSFM

    # the reference config's arguments (onedsfm_front_end.yaml) construct it
    B200TranslationAveraging1DSFM(robust_measurement_noise=True, projection_sampling_method="SAMPLE_INPUT_MEASUREMENTS")
