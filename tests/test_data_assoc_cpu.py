"""Data association's triangulation without a GPU: oracle/data_assoc_ref.py against its fixture, the pair sampler, the
hypothesis count, the host build of csrc/data_assoc_math.cuh (tests/cpp/test_triangulation_math.cpp), and the plugin's
checks and packing."""
from __future__ import annotations

import itertools
import math
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import data_assoc_ref as da  # noqa: E402
from oracle import twoview_ba_ref as tv  # noqa: E402
from oracle.make_golden_data_assoc import CONFIG_HYPS, lund_matches, lund_scenes, ring_cameras, scenes, union_find_tracks  # noqa: E402


def load_scenes(path):
    z = np.load(path)
    out = {}
    for k in z.files:
        name, key = k.split("/")
        out.setdefault(name, {})[key] = z[k]
    return out


SCENES = load_scenes(ROOT / "tests/golden/data_assoc_scenes.npz")
LUND = load_scenes(ROOT / "tests/golden/data_assoc_lund_door.npz")
ALL = {**SCENES, **{f"lund_door_{k}": v for k, v in LUND.items()}}


@pytest.mark.parametrize("name", sorted(ALL))
def test_oracle_matches_fixture(name):
    sc = ALL[name]
    o = sc["options"]
    T = len(sc["track_off"]) - 1
    tracks = range(0, T, 2)  # every other track keeps the run short; the device tests cover all
    ex, pt, avg, inl = da.run_arrays(sc["track_off"], sc["meas_cam"], sc["meas_uv"], sc["cams"], sc["cam_valid"],
                                     da.SAMPLE_UNIFORM if o[0] else da.NO_RANSAC, int(o[1]), float(o[2]), float(o[3]), int(o[4]), tracks)
    for t in tracks:
        a, b = sc["track_off"][t], sc["track_off"][t + 1]
        assert ex[t] == sc["exit"][t]
        np.testing.assert_array_equal(inl[a:b], sc["inlier"][a:b])
        np.testing.assert_allclose(pt[t], sc["point"][t], rtol=1e-12, atol=1e-12, equal_nan=True)
        np.testing.assert_allclose(avg[t], sc["avg"][t], rtol=1e-12, atol=1e-12, equal_nan=True)


def test_fixture_scenes_are_the_generator_s():
    gen = scenes()
    assert sorted(gen) == sorted(SCENES)
    for name, sc in gen.items():
        for k, v in sc.items():
            np.testing.assert_array_equal(v, SCENES[name][k])


def test_lund_door_fixture_is_the_union_find_of_its_correspondences():
    gen, _, _ = lund_scenes()
    assert sorted(gen) == sorted(LUND)
    for name, sc in gen.items():
        for k, v in sc.items():
            np.testing.assert_array_equal(v, LUND[name][k])
    matches, kps, _ = lund_matches()
    tracks = union_find_tracks(matches, kps)
    sc = LUND["uniform_10px_100"]
    lens = np.diff(sc["track_off"])
    assert len(tracks) == len(lens) and lens.min() >= 2 and lens.max() >= 5
    for t in tracks:  # one measurement per image (DsfTracksEstimator drops the others)
        assert len({i for i, _ in t}) == len(t)
    assert not sc["cam_valid"][6] and sc["cam_valid"].sum() == 11
    assert (sc["meas_cam"] == 6).any()


def test_fixture_covers_every_exit_code_and_both_sides_of_the_sampling_boundary():
    codes = np.concatenate([sc["exit"] for sc in SCENES.values()])
    assert set(codes.tolist()) == set(range(6))
    lens = np.diff(SCENES["boundary_14_15"]["track_off"])
    assert {14, 15} <= set(lens.tolist()) and SCENES["boundary_14_15"]["options"][1] == math.comb(14, 2)
    assert len(SCENES["empty"]["track_off"]) == 1 and not SCENES["all_missing"]["cam_valid"].any()


# ---- the sampler ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pairs,hyps", [(105, 100), (120, 91), (4950, 100), (1, 1), (10, 10), (36, 100), (2 ** 20 + 3, 100)])
def test_sampler_is_a_deterministic_draw_without_replacement(pairs, hyps):
    for track in (0, 1, 12345):
        a = da.sample_pairs(7, track, pairs, min(pairs, hyps))
        np.testing.assert_array_equal(a, da.sample_pairs(7, track, pairs, min(pairs, hyps)))
        assert len(a) == min(pairs, hyps) and len(set(a.tolist())) == len(a)
        assert a.min() >= 0 and a.max() < pairs
        if pairs <= hyps:
            np.testing.assert_array_equal(a, np.arange(pairs))
    assert not np.array_equal(da.sample_pairs(7, 0, 4950, 100), da.sample_pairs(7, 1, 4950, 100))
    assert not np.array_equal(da.sample_pairs(7, 0, 4950, 100), da.sample_pairs(8, 0, 4950, 100))


def test_sampler_is_roughly_uniform():
    pairs, hyps, keys = 105, 20, 4000  # a 15-measurement track, 20 draws each
    counts = np.zeros(pairs)
    for t in range(keys):
        counts[da.sample_pairs(3, t, pairs, hyps)] += 1
    expect = keys * hyps / pairs
    chi2 = float(((counts - expect) ** 2 / expect).sum())
    assert chi2 < 2 * pairs  # dof 104: mean 104, sd ~14
    first = np.bincount([da.sample_pairs(3, t, pairs, hyps)[0] for t in range(keys)], minlength=pairs)
    assert first.max() < 5 * keys / pairs


def test_pair_decoding_is_combinations_order():
    for n in (2, 3, 7, 15):
        assert [da.pair_of(p, n) for p in range(math.comb(n, 2))] == list(itertools.combinations(range(n), 2))


def test_num_hypotheses_is_the_reference_formula():
    from gtsfm_b200.gtsfm_api import TriangulationOptions, TriangulationSamplingMode

    cfg = TriangulationOptions(mode=TriangulationSamplingMode.RANSAC_SAMPLE_UNIFORM, reproj_error_threshold=10, max_num_hypotheses=100)
    assert cfg.num_ransac_hypotheses() == 100 == CONFIG_HYPS
    dflt = TriangulationOptions(mode=TriangulationSamplingMode.RANSAC_SAMPLE_UNIFORM)
    assert dflt.num_ransac_hypotheses() == 2749 == da.num_ransac_hypotheses()  # point3d_initializer.py:103-104
    assert TriangulationOptions(TriangulationSamplingMode.NO_RANSAC, 5.0, 0.0, 0.3, 0.99, 2.0, 10, 50).num_ransac_hypotheses() == \
        da.num_ransac_hypotheses(0.3, 0.99, 2.0, 10, 50) == 50


# ---- host build of the device maths -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    exe = tmp_path_factory.mktemp("da") / "test_triangulation_math"
    subprocess.run([cxx, "-O2", "-std=c++17", "-x", "c++", str(ROOT / "tests/cpp/test_triangulation_math.cpp"), "-o", str(exe)], check=True)

    def run(lines):
        r = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True)
        return [np.array(l.split(), float) for l in r.stdout.strip().split("\n")]

    return run


def _cam_words(c):
    return " ".join("%.17g" % x for x in [*c[:9], *c[9:12], c[12], 0.0, 0.0, c[13], c[14]])


def test_host_sampler_equals_numpy(harness):
    cases = [(7, 0, 105, 100), (7, 5, 105, 100), (2 ** 64 - 1, 99, 4950, 100), (0, 3, 36, 36), (123, 2 ** 40, 2 ** 20 + 3, 50)]
    out = harness([f"pair {s} {t} {p} {h}" for s, t, p, h in cases])
    for (s, t, p, h), got in zip(cases, out):
        np.testing.assert_array_equal(got.astype(np.int64), da.sample_pairs(s, t, p, h))


def test_host_nview_dlt_at_two_views_equals_dlt(harness):
    rng = np.random.default_rng(1)
    cams = ring_cameras(rng, 8)
    lines = []
    for _ in range(40):
        i, j = rng.choice(8, 2, replace=False)
        uv = rng.uniform(0, 640, 4)
        lines.append(f"dlt2 {_cam_words(cams[i])} {_cam_words(cams[j])} " + " ".join("%.17g" % x for x in uv))
    for row in harness(lines):
        assert row[0] == row[4]
        np.testing.assert_array_equal(row[1:4], row[5:8])  # bit for bit


def test_host_qr_reduced_dlt_equals_direct_svd(harness):
    rng = np.random.default_rng(2)
    systems = [rng.normal(size=(2 * n, 4)) * rng.uniform(0.1, 1e3, 4) for n in (2, 3, 5, 14, 40, 200)]
    low = rng.normal(size=(30, 3)) @ rng.normal(size=(3, 4))  # rank 3: a zero singular value
    systems.append(low)
    out = harness([f"qr {len(A)} " + " ".join("%.17g" % x for x in A.ravel()) for A in systems])
    for A, row in zip(systems, out):
        _, s, Vt = np.linalg.svd(A)
        np.testing.assert_allclose(row[:4], s[::-1], rtol=1e-12, atol=1e-12 * s[0])
        v = Vt[3] * np.sign(Vt[3][3])
        np.testing.assert_allclose(row[4:], v, atol=1e-9)


def test_host_nview_triangulation_equals_oracle(harness):
    rng = np.random.default_rng(3)
    cams = ring_cameras(rng, 30)
    lines, probs = [], []
    for n in (2, 3, 6, 25):
        for _ in range(5):
            X = rng.normal(0, 1.5, 3)
            idx = rng.choice(30, n, replace=False)
            uvs = []
            for i in idx:
                R, t = cams[i, :9].reshape(3, 3), cams[i, 9:12]
                pc = R.T @ (X - t)
                uvs.append(cams[i, 13:] + cams[i, 12] * pc[:2] / pc[2] + rng.normal(0, 2.0, 2))
            probs.append((idx, uvs))
            lines.append(f"tri {n} " + " ".join(_cam_words(cams[i]) for i in idx) + " " + " ".join("%.17g" % x for u in uvs for x in u))
    for (idx, uvs), row in zip(probs, harness(lines)):
        X = da.triangulate_point3([da.camera(cams[i, :9], cams[i, 9:12], *cams[i, 12:]) for i in idx], uvs)
        assert row[0] == 1 and X is not None
        np.testing.assert_allclose(row[1:], X, rtol=1e-9, atol=1e-9)


# ---- the plugin's checks and packing ---------------------------------------------------------------------------------------
class _Cal:
    def __init__(self, k1=0.0, name="Cal3Bundler"):
        self._k1 = k1
        self.__class__ = type(name, (_Cal,), {})

    def k1(self):
        return self._k1

    def k2(self):
        return 0.0

    def fx(self):
        return 500.0

    def px(self):
        return 320.0

    def py(self):
        return 240.0


class _Pose:
    def rotation(self):
        return type("R", (), {"matrix": lambda s: np.eye(3)})()

    def translation(self):
        return np.zeros(3)


class _Camera:
    def __init__(self, cal):
        self._cal = cal

    def pose(self):
        return _Pose()

    def calibration(self):
        return self._cal


def _plugin(mode="RANSAC_SAMPLE_UNIFORM", **kw):
    from gtsfm_b200.data_association import B200DataAssociation
    from gtsfm_b200.gtsfm_api import TriangulationOptions, TriangulationSamplingMode

    return B200DataAssociation(min_track_len=2, triangulation_options=TriangulationOptions(TriangulationSamplingMode(mode), **kw))


def test_plugin_params_and_mode_checks():
    from gtsfm_b200 import _lib
    from gtsfm_b200.gtsfm_api import HAVE_GTSFM_DATA_ASSOCIATION as HAVE_GTSFM, SfmMeasurement, SfmTrack2d

    p = _plugin(reproj_error_threshold=10, max_num_hypotheses=100).device_params()
    assert (p.mode, p.num_hypotheses, p.reproj_error_threshold, p.min_triangulation_angle) == (_lib.TRI_SAMPLE_UNIFORM, 100, 10.0, 0.0)
    assert _plugin("NO_RANSAC").device_params().mode == _lib.TRI_NO_RANSAC
    for mode in ("RANSAC_SAMPLE_BIASED_BASELINE", "RANSAC_TOPK_BASELINES"):
        with pytest.raises(ValueError):
            _plugin(mode).device_params()
        if not HAVE_GTSFM:
            with pytest.raises(ValueError):
                _plugin(mode).run_triangulation({0: _Camera(_Cal())}, [SfmTrack2d([SfmMeasurement(0, np.zeros(2))])])
    assert _plugin().run_triangulation({}, [SfmTrack2d([])]) == ([], [], [])
    assert _plugin().run_triangulation({0: _Camera(_Cal())}, []) == ([], [], [])


def test_plugin_camera_checks():
    from gtsfm_b200.data_association import device_camera
    from gtsfm_b200.gtsfm_api import HAVE_GTSFM_DATA_ASSOCIATION as HAVE_GTSFM, SfmMeasurement, SfmTrack2d

    R, t, f, u0, v0 = device_camera(_Camera(_Cal()))
    assert np.array_equal(R, np.eye(3)) and (f, u0, v0) == (500.0, 320.0, 240.0)
    assert device_camera(_Camera(_Cal(k1=0.1))) is None
    assert device_camera(_Camera(_Cal(name="Cal3_S2"))) is None
    pl = _plugin()
    cams, valid = pl.camera_arrays({0: _Camera(_Cal()), 2: None, 3: (np.eye(3), np.ones(3), 400.0, 1.0, 2.0)}, 5)
    assert valid.tolist() == [1, 0, 0, 1, 0] and cams[3, 9:].tolist() == [1, 1, 1, 400, 1, 2]
    assert pl.camera_arrays({0: _Camera(_Cal(k1=0.1))}, 1) is None
    if not HAVE_GTSFM:
        with pytest.raises(ValueError):
            pl.run_triangulation({0: _Camera(_Cal(k1=0.1))}, [SfmTrack2d([SfmMeasurement(0, np.zeros(2))])])


def test_plugin_packing_and_unpacking():
    from gtsfm_b200.data_association import pack_tracks, unpack
    from gtsfm_b200.gtsfm_api import SfmMeasurement, SfmTrack2d, TriangulationExitCode

    rng = np.random.default_rng(4)
    raw = [[(int(rng.integers(0, 9)), rng.uniform(0, 600, 2)) for _ in range(n)] for n in (2, 5, 3, 17)]
    tracks = [SfmTrack2d([SfmMeasurement(i, uv) for i, uv in t]) for t in raw]
    off, cam, uv = pack_tracks(tracks)
    o2, c2, u2 = da.pack_tracks(raw)
    np.testing.assert_array_equal(off, o2), np.testing.assert_array_equal(cam, c2), np.testing.assert_array_equal(uv, u2)
    ex = np.array([0, 4, 2, 0], np.int8)
    pt = rng.normal(size=(4, 3))
    avg = np.array([0.5, 12.0, np.nan, 1.5])
    inl = np.zeros(off[-1], bool)
    inl[[0, 1, 2, 3, 10, 12, 20]] = True
    s, e, c = unpack(tracks, off, ex, pt, avg, inl)
    assert c == [TriangulationExitCode.SUCCESS, TriangulationExitCode.EXCEEDS_REPROJ_THRESH,
                 TriangulationExitCode.INLIERS_UNDERCONSTRAINED, TriangulationExitCode.SUCCESS]
    assert e == [0.5, 12.0, None, 1.5] and s[1] is None and s[2] is None
    assert s[0].numberMeasurements() == 2 and np.array_equal(s[0].point3(), pt[0])
    got = [s[3].measurement(k) for k in range(s[3].numberMeasurements())]
    assert [g[0] for g in got] == [raw[3][k][0] for k in (0, 2, 10)]


def test_hydra_config_swaps_only_the_data_association_target():
    text = (ROOT / "configs/deep_front_end_b200_data_assoc.yaml").read_text()
    assert "deep_front_end_b200_view_graph" in text
    assert "_target_: gtsfm_b200.data_association.B200DataAssociation" in text
    assert text.count("_target_") == 1
