"""1DSfM's translation recovery on the device (b2_translation_recovery_host) against oracle/translation_recovery_ref.py:
every fixture scene, repeated calls, the workspace bound, the argument checks and the plugin's __run_averaging."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import translation_recovery_ref as tr  # noqa: E402

pytestmark = pytest.mark.gpu

FIXTURE = np.load(ROOT / "tests/golden/translation_recovery_scenes.npz")
NAMES = [str(n) for n in FIXTURE["names"]]
SOLVED = [n for n in NAMES if len(FIXTURE[f"{n}/edge_a"])]  # scenes with a problem left after the zero-translation sets

# (trace rtol, translation bound) where only the damping holds a direction of the solution (DESIGN.md §3): the free second
# component of two_components; scale 0, whose solution collapses to ~1e-5 of the initial extent, so its bound is taken on
# that extent; the landmark held along its ray by the damping alone
TOL = {"two_components": (1e-5, lambda sc: 1e-4 * np.abs(sc["x"]).max()),
       "scale_zero": (1e-5, lambda sc: 1e-8 * np.abs(sc["init"]).max()),
       "single_edge_landmark": (1e-8, lambda sc: 1e-8 * np.abs(sc["x"]).max())}
STRICT = (1e-9, lambda sc: 1e-8 * np.abs(sc["x"]).max())


def scene(name):
    return {k.split("/", 1)[1]: FIXTURE[k] for k in FIXTURE.files if k.startswith(name + "/")}


@pytest.fixture(scope="module")
def ctx():
    from gtsfm_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


def device(sc, ctx, **kw):
    from gtsfm_b200 import translation_averaging as ta

    return ta.recover_arrays(ctx, int(sc["C"]), int(sc["L"]), sc["edge_a"], sc["edge_b"], sc["meas"], sc["init"],
                             huber_k=tr.HUBER_K if bool(sc["robust"]) else 0.0, scale=float(sc["scale"]), trace=True, **kw)


@pytest.mark.parametrize("name", SOLVED)
def test_device_equals_oracle(name, ctx):
    sc = scene(name)
    d = device(sc, ctx)
    np.testing.assert_array_equal(d["trials"], sc["trials"])
    assert d["iterations"] == int(sc["iterations"])
    rtol, xtol = TOL.get(name, STRICT)
    t0 = float(sc["trace"][0])
    np.testing.assert_allclose(d["trace"], sc["trace"], rtol=rtol, atol=1e-12 * t0)
    assert d["final_error"] == pytest.approx(float(sc["final_error"]), rel=rtol, abs=1e-12 * t0)
    assert np.abs(d["x"] - sc["x"]).max() <= xtol(sc)


@pytest.mark.parametrize("name", ["lund_door", "knn_tracks_huber", "single_edge_landmark", "ref_skydio32"])
def test_repeated_calls_are_bit_identical(name, ctx):
    sc = scene(name)
    a, b = device(sc, ctx), device(sc, ctx)
    for k in ("x", "trace", "trials"):
        assert np.array_equal(a[k], b[k])


def test_over_budget_refused():
    from gtsfm_b200 import _lib
    from gtsfm_b200 import translation_averaging as ta

    rng = np.random.default_rng(2)
    n = 600
    ea = np.arange(1, n, dtype=np.int32)
    eb = np.arange(0, n - 1, dtype=np.int32)
    meas = rng.normal(size=(n - 1, 3))
    assert ta.recovery_workspace_bytes(n, 0, ea, eb) > 2 << 20
    c = _lib.Context(0)
    try:
        c.set_option("ba_workspace_mb", 2)
        with pytest.raises(_lib.B200Error, match="ba_workspace_mb"):
            ta.recover_arrays(c, n, 0, ea, eb, meas, rng.normal(size=(n, 3)))
        with pytest.raises(ValueError, match="ba_workspace_mb"):
            ta.recover_translations(c, {(int(b), int(a)): m for a, b, m in zip(ea, eb, meas)}, {})
        c.set_option("ba_workspace_mb", 64)
        out = ta.recover_arrays(c, n, 0, ea, eb, meas, rng.normal(size=(n, 3)), max_iters=2)
        assert np.isfinite(out["x"]).all()
    finally:
        c.close()


def test_bad_inputs_refused(ctx):
    from gtsfm_b200 import _lib
    from gtsfm_b200 import translation_averaging as ta

    sc = scene("single_edge_landmark")
    C, L = int(sc["C"]), int(sc["L"])
    ea, eb, m, x0 = (np.array(sc[k]) for k in ("edge_a", "edge_b", "meas", "init"))

    def call(ea=ea, eb=eb, m=m, x0=x0, C=C, L=L, **kw):
        return ta.recover_arrays(ctx, C, L, ea, eb, m, x0, **kw)

    def bad(**kw):
        with pytest.raises(_lib.B200Error):
            call(**kw)

    bad(eb=np.where(np.arange(len(eb)) == 3, C + L, eb))            # index out of range
    bad(eb=np.where(np.arange(len(eb)) == 3, -1, eb))
    bad(eb=np.where(np.arange(len(eb)) == 0, ea[0], eb))             # self edge
    lm = np.nonzero(eb >= C)[0][0]
    bad(ea=np.where(np.arange(len(ea)) == lm, C + (eb[lm] - C + 1) % L, ea))  # landmark to landmark
    m0 = m.copy()
    m0[5] = 0.0
    bad(m=m0)                                                         # zero measurement
    m0[5] = [np.nan, 0.0, 1.0]
    bad(m=m0)
    x1 = x0.copy()
    x1[2, 1] = np.inf
    bad(x0=x1)
    bad(ea=ea[:0], eb=eb[:0], m=m[:0])                                # E = 0
    bad(C=C + 1, x0=np.concatenate([x0, np.zeros((1, 3))]))           # a node without an edge
    bad(sigma=0.0)
    bad(prior_sigma=-1.0)
    bad(huber_k=np.nan)
    bad(scale=np.inf)
    bad(max_iters=-1)
    assert np.isfinite(call()["x"]).all()                             # the unmodified call still runs


def test_plugin_run_averaging_override(ctx):
    from gtsfm_b200 import translation_averaging as ta

    obj = ta.B200TranslationAveraging1DSFM(ctx=ctx)
    for name in ("lund_door", "consecutive_1"):
        sc = scene(name)
        n = int(sc["num_images"])
        cam = {tuple(map(int, k)): v for k, v in zip(sc["cam_keys"], sc["cam_vecs"])}
        trk = {tuple(map(int, k)): v for k, v in zip(sc["trk_keys"], sc["trk_vecs"])}
        wRi = [np.eye(3)] * n
        wRi[int(sc["cams"][1])] = None  # no rotation: None whatever TranslationRecovery returns for it
        ta.reseed_translation_rng()
        ta.random_points(int(sc["rng_skip"]))
        wti = obj._TranslationAveraging1DSFM__run_averaging(n, cam, trk, wRi, {}, [], float(sc["scale"]))
        assert len(wti) == n
        for i in range(n):
            if wRi[i] is None or np.isnan(sc["wti"][i]).any():
                assert wti[i] is None
            else:
                np.testing.assert_allclose(wti[i], sc["wti"][i], rtol=0, atol=1e-8 * np.abs(sc["x"]).max())
    # the reference tests' own scenes, as their run_translation_averaging handed them to __run_averaging: camera 4 of
    # Test1dsfmAllOutliers and Skydio-32's cameras without a rotation come back None, the panorama's zero translations
    # share one value without a device call
    for name in ("ref_circle_all_edges", "ref_panorama", "ref_lund_door", "ref_poses_on_circle", "ref_all_outliers", "ref_skydio32"):
        sc = scene(name)
        n = int(sc["num_images"])
        cam = {tuple(map(int, k)): v for k, v in zip(sc["cam_keys"], sc["cam_vecs"])}
        ta.reseed_translation_rng()
        wti = obj._TranslationAveraging1DSFM__run_averaging(n, cam, {}, [np.eye(3)] * n, {}, [], 1.0)
        assert [w is None for w in wti] == list(np.isnan(sc["wti"][:, 0])), name
        scale = max(np.abs(sc["x"]).max(initial=0.0), 1.0)
        for i in range(n):
            if wti[i] is not None:
                np.testing.assert_allclose(wti[i], sc["wti"][i], rtol=0, atol=1e-8 * scale)
    assert obj._TranslationAveraging1DSFM__run_averaging(3, {}, {}, [np.eye(3)] * 3, {}, [], 1.0) == [None] * 3
