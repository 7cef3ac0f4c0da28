"""CPU suite of 1DSfM's translation recovery: oracle/translation_recovery_ref.py against its fixtures, its Schur solve
against a plain dense solve, the plugin's graph, initial values and process-wide generator (against a g++-built
std::mt19937 program), its budget check, and the library's new symbols."""
from __future__ import annotations

import ctypes
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import translation_recovery_ref as tr  # noqa: E402

FIXTURE = np.load(ROOT / "tests/golden/translation_recovery_scenes.npz")
NAMES = [str(n) for n in FIXTURE["names"]]
SOLVED = [n for n in NAMES if len(FIXTURE[f"{n}/edge_a"])]  # scenes with a problem left after the zero-translation sets
# scenes where only the damping holds a direction of the solution: the second component of two_components has no prior
# (its translation and scale are free), and with scale 0 both priors pull towards the origin, where every normalize() is
# ill-conditioned.  Two solves' rounding grows there over the LM run to ~1e-6 relative (DESIGN.md §3)
DAMPING_HELD = {"two_components", "scale_zero"}


def scene(name):
    return {k.split("/", 1)[1]: FIXTURE[k] for k in FIXTURE.files if k.startswith(name + "/")}


def problem(sc) -> tr.Problem:
    return tr.Problem(int(sc["C"]), int(sc["L"]), sc["edge_a"], sc["edge_b"], sc["meas"], huber_k=tr.HUBER_K if bool(sc["robust"]) else 0.0,
                      scale=float(sc["scale"]))


def test_fixture_covers_the_issue_cases():
    assert {"knn_cams", "knn_tracks_huber", "knn_tracks_gauss", "scale_zero", "single_edge_landmark", "two_components", "two_cameras",
            "consecutive_1", "consecutive_2", "lund_door"} <= set(NAMES)
    assert not bool(scene("knn_tracks_gauss")["robust"]) and float(scene("scale_zero")["scale"]) == 0.0
    sc = scene("single_edge_landmark")
    lmk = np.concatenate([sc["edge_a"], sc["edge_b"]])
    assert np.any(np.bincount(lmk[lmk >= int(sc["C"])]) == 1)
    assert int(scene("consecutive_2")["rng_skip"]) == int(scene("consecutive_1")["C"]) + int(scene("consecutive_1")["L"])


@pytest.mark.parametrize("name", SOLVED)
def test_oracle_reproduces_fixture(name):
    sc = scene(name)
    res = tr.recover(problem(sc), sc["init"])
    np.testing.assert_array_equal(res.trials, sc["trials"])
    np.testing.assert_array_equal(res.trace, sc["trace"])
    np.testing.assert_array_equal(res.x, sc["x"])


@pytest.mark.parametrize("name", [n for n in SOLVED if n not in ("lund_door", "ref_skydio32")])
def test_schur_solve_equals_dense_solve(name):
    sc = scene(name)
    pr = problem(sc)
    x = np.asarray(sc["init"], float)
    lin = tr.linearise(x, pr)
    for lam in (1e-5, 1e-2, 1.0, 1e3):
        s, d = tr.step(x, pr, lam, lin), tr.dense_step(x, pr, lam, lin)
        scale = np.abs(d[3]).max()
        assert np.abs(s[3] - d[3]).max() <= 1e-8 * scale
        assert s[1] == pytest.approx(d[1], rel=1e-9, abs=1e-12 * d[2])
        assert s[2] == pytest.approx(d[2], rel=1e-12)
    res = tr.recover(pr, x, solver=tr.dense_step)
    assert res.trials == list(sc["trials"])
    rtol = 1e-5 if name in DAMPING_HELD else 1e-8
    np.testing.assert_allclose(res.trace, sc["trace"], rtol=rtol, atol=1e-12 * sc["trace"][0])


def test_converged_scenes_fit_their_directions():
    """Noise-free scenes end at (numerically) zero cost, and each camera direction is reproduced."""
    for name in ("knn_tracks_gauss", "two_components", "two_cameras", "consecutive_1", "consecutive_2"):
        sc = scene(name)
        assert float(sc["final_error"]) < 1e-12 * float(sc["trace"][0])
        x = sc["x"]
        d = x[sc["edge_b"]] - x[sc["edge_a"]]
        np.testing.assert_allclose(d / np.linalg.norm(d, axis=1)[:, None], sc["meas"], atol=1e-8)


def test_gauge_and_scale_priors():
    sc = scene("knn_tracks_gauss")
    x = sc["x"]
    assert np.abs(x[sc["edge_a"][0]]).max() < 1e-9
    np.testing.assert_allclose(x[sc["edge_b"][0]] - x[sc["edge_a"][0]], sc["meas"][0], atol=1e-9)
    z = scene("scale_zero")
    assert np.linalg.norm(z["x"][z["edge_b"][0]]) < 1e-2 * np.abs(z["init"]).max()


@pytest.fixture(scope="module")
def std_mt19937(tmp_path_factory):
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    exe = tmp_path_factory.mktemp("tr_rng") / "test_tr_rng"
    subprocess.run([cxx, "-O2", "-std=c++17", str(ROOT / "tests/cpp/test_tr_rng.cpp"), "-o", str(exe)], check=True)

    def points(n):
        out = subprocess.run([str(exe)], input=f"{n}\n", capture_output=True, text=True, check=True).stdout
        return np.array([[float(v) for v in line.split()] for line in out.splitlines()])

    return points


def test_generator_equals_std_mt19937(std_mt19937):
    from gtsfm_b200 import translation_averaging as ta

    ref = std_mt19937(500)
    ta.reseed_translation_rng()
    mine = np.concatenate([ta.random_points(1), ta.random_points(199), ta.random_points(300)])  # the stream continues
    np.testing.assert_array_equal(mine, ref)
    assert ref[0].tolist() == [0.5593819952253225, -0.63313042421326304, 0.59308596857569196]
    o = tr.Mt19937Uniform(42)
    np.testing.assert_array_equal([o.point3() for _ in range(500)], ref)


def full_dicts(sc):
    cam = {tuple(map(int, k)): v for k, v in zip(sc["cam_keys"], sc["cam_vecs"])}
    trk = {tuple(map(int, k)): v for k, v in zip(sc["trk_keys"], sc["trk_vecs"])}
    return cam, trk


@pytest.mark.parametrize("name", NAMES)
def test_plugin_graph_and_initial_values(name):
    from gtsfm_b200 import translation_averaging as ta

    sc = scene(name)
    cams, root, nodes, C, L, ea, eb, meas = ta.reduced_problem(*full_dicts(sc))
    np.testing.assert_array_equal(cams, sc["cams"])
    np.testing.assert_array_equal(root, sc["root"])
    np.testing.assert_array_equal(nodes, sc["nodes"])
    assert (C, L) == (int(sc["C"]), int(sc["L"]))
    np.testing.assert_array_equal(ea, sc["edge_a"])
    np.testing.assert_array_equal(eb, sc["edge_b"])
    np.testing.assert_array_equal(meas, sc["meas"])
    ta.reseed_translation_rng()
    ta.random_points(int(sc["rng_skip"]))
    if len(ea):
        np.testing.assert_array_equal(ta.initial_values(ea, eb, C + L), sc["init"])


@pytest.mark.parametrize("name", NAMES)
def test_oracle_run_gives_the_reference_output(name):
    """TranslationRecovery::run restated on the full graph (zero-translation sets included) gives the wti the reference's
    own __run_averaging returned: a value for every camera of an edge, None (NaN) for the others."""
    from gtsfm_b200 import translation_averaging as ta

    sc = scene(name)
    cams, tracks, ea, eb, meas = ta.translation_graph(*full_dicts(sc))
    u = tr.Mt19937Uniform(42)
    for _ in range(int(sc["rng_skip"])):
        u.point3()
    out = tr.run(len(cams), len(tracks), ea, eb, meas, u, huber_k=tr.HUBER_K if bool(sc["robust"]) else 0.0, scale=float(sc["scale"]))
    w = np.full_like(sc["wti"], np.nan)
    w[cams] = out["x"][:len(cams)]
    np.testing.assert_array_equal(w, sc["wti"])


def sim3_align(src, dst):
    """Umeyama's least-squares similarity dst ~ s R src + t, applied to src (s = 1, R = I for coincident points)."""
    ms, md = src.mean(0), dst.mean(0)
    a, b = src - ms, dst - md
    var = float((a * a).sum()) / len(src)
    if var == 0.0:
        return src - ms + md
    U, S, Vt = np.linalg.svd(b.T @ a / len(src))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = U @ D @ Vt
    return (np.trace(np.diag(S) @ D) / var) * a @ R.T + md


REF_GT = ["ref_circle_all_edges", "ref_panorama", "ref_lund_door", "ref_poses_on_circle"]


@pytest.mark.parametrize("name", REF_GT)
def test_reference_scenes_meet_the_reference_tests_criterion(name):
    """test_averaging_1dsfm.py's criterion: the translations, Sim(3)-aligned to the ground truth, within 3e-2 relative /
    3e-1 absolute (np.allclose), every camera estimated."""
    sc = scene(name)
    w, gt = sc["wti"], sc["gt_wti"]
    assert np.isfinite(w).all()
    assert np.allclose(sim3_align(w, gt), gt, rtol=3e-2, atol=3e-1)


def test_reference_all_outliers_and_skydio_none_pattern():
    sc = scene("ref_all_outliers")
    assert int(sc["num_images"]) == 5
    assert np.isnan(sc["wti"][4]).all() and np.isfinite(sc["wti"][:4]).all()  # Test1dsfmAllOutliers: camera 4 is None
    sk = scene("ref_skydio32")
    has_edge = np.zeros(int(sk["num_images"]), bool)
    has_edge[sk["cams"]] = True
    np.testing.assert_array_equal(np.isfinite(sk["wti"][:, 0]), has_edge)
    assert has_edge.sum() == 17


def test_panorama_zero_translations_share_one_value():
    sc = scene("ref_panorama")
    assert len(sc["edge_a"]) == 0 and np.all(sc["meas"] == 0)
    np.testing.assert_array_equal(sc["wti"], np.zeros((3, 3)))


class _Budget:  # a context stand-in: only its options are read before the device is reached
    def __init__(self, mb):
        self.options = {"ba_workspace_mb": mb}


def test_over_budget_and_empty_consume_no_draw():
    from gtsfm_b200 import translation_averaging as ta

    rng = np.random.default_rng(1)
    n = 400
    cam = {(i, i + 1): rng.normal(size=3) for i in range(n - 1)}
    ta.reseed_translation_rng()
    with pytest.raises(ValueError, match="ba_workspace_mb"):
        ta.recover_translations(_Budget(1), cam, {})
    assert ta.recover_translations(_Budget(1), {}, {}) == {}
    np.testing.assert_array_equal(ta.random_points(1), tr.Mt19937Uniform(42).point3()[None])
    cams, tracks, ea, eb, _ = ta.translation_graph(cam, {})
    assert ta.recovery_workspace_bytes(len(cams), len(tracks), ea, eb) > 1 << 20


def test_workspace_bytes_refuses_bad_indices():
    from gtsfm_b200 import translation_averaging as ta

    assert ta.recovery_workspace_bytes(2, 1, [0, 1], [1, 2]) > 0
    assert ta.recovery_workspace_bytes(2, 1, [0, 1], [1, 3]) == 0
    assert ta.recovery_workspace_bytes(0, 1, [0], [1]) == 0


def test_abi_exports_translation_recovery():
    from gtsfm_b200 import _lib, build

    lib = ctypes.CDLL(str(build.build()))
    for name in ("b2_translation_recovery_workspace_bytes", "b2_translation_recovery_host"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    assert ctypes.sizeof(_lib.TrParams) == 40
