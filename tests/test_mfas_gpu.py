"""GPU suite for 1DSfM's outlier rejection (csrc/mfas.cu) against the NumPy oracle (oracle/mfas_ref.py): every fixture
scene bit for bit, the device orderings, chunked against unchunked and repeated calls bitwise, a large seeded scene, the
argument checks and the plugin's compute_inliers."""
from pathlib import Path

import numpy as np
import pytest

from oracle import mfas_ref as mr

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def ctx():
    from gtsfm_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


def _scenes():
    out = []
    for f in ("mfas_scenes.npz", "mfas_lund_door.npz"):
        d = np.load(GOLDEN / f)
        out += [(f, str(n)) for n in d["names"] if str(n) != "empty"]
    return out


def _problem(d, name):
    return int(d[f"{name}/V"]), d[f"{name}/edge_a"], d[f"{name}/edge_b"], d[f"{name}/meas"], d[f"{name}/dirs"]


def _bits(s):
    return np.ascontiguousarray(s).view(np.uint64)


def _unpack(words, E):
    return np.unpackbits(words.view(np.uint8).reshape(len(words), -1), axis=1, bitorder="little")[:, :E].astype(bool)


@pytest.mark.parametrize("f,name", _scenes())
def test_fixture_sums_and_orderings(ctx, f, name):
    from gtsfm_b200.translation_averaging import outlier_weights_arrays

    d = np.load(GOLDEN / f)
    V, ea, eb, meas, dirs = _problem(d, name)
    s, order, viol = outlier_weights_arrays(ctx, V, ea, eb, meas, dirs, order=True, violated=True)
    assert np.array_equal(_bits(s), _bits(d[f"{name}/weight_sum"])), name
    bad = _unpack(viol, len(ea))
    for k in range(0, len(dirs), max(1, len(dirs) // 25)):  # a subset of directions against the oracle's orderings
        o2, b2 = mr.order_vectorised(V, ea, eb, meas, dirs[k])
        assert np.array_equal(order[k], o2) and np.array_equal(bad[k], b2), (name, k)


def test_chunked_and_repeated_are_bitwise_identical(ctx):
    from gtsfm_b200.translation_averaging import outlier_weights_arrays

    d = np.load(GOLDEN / "mfas_lund_door.npz")
    V, ea, eb, meas, dirs = _problem(d, "lund_door")
    dirs = np.concatenate([dirs] * 10)  # 2020 directions
    s0, v0 = outlier_weights_arrays(ctx, V, ea, eb, meas, dirs, violated=True)
    s1, v1 = outlier_weights_arrays(ctx, V, ea, eb, meas, dirs, violated=True)
    assert np.array_equal(_bits(s0), _bits(s1)) and np.array_equal(v0, v1)
    launches = ctx.launch_count()
    ctx.set_option("mfas_workspace_mb", 1)
    try:
        s2, v2 = outlier_weights_arrays(ctx, V, ea, eb, meas, dirs, violated=True)
        chunked = ctx.launch_count() - launches
    finally:
        ctx.set_option("mfas_workspace_mb", 1024)
    assert chunked > 4, chunked  # more than one chunk of directions
    assert np.array_equal(_bits(s0), _bits(s2)) and np.array_equal(v0, v2)


def test_large_scene(ctx):
    from gtsfm_b200.translation_averaging import dense_edges, outlier_weights_arrays

    from oracle.make_golden_mfas import large_scene

    cam, trk = large_scene(3000)
    V, ea, eb, perm = dense_edges(cam, trk)
    meas = np.array(list(cam.values()) + list(trk.values()))[perm]
    rng = np.random.default_rng(3)
    dirs = meas[rng.choice(len(meas), 2000, replace=False)]
    s, viol = outlier_weights_arrays(ctx, V, ea, eb, meas, dirs, violated=True)
    bad = _unpack(viol, len(ea))
    want = np.zeros(len(ea))
    for k in range(len(dirs)):  # the reference's order of accumulation, from the device's own violated bits
        want = want + np.where(bad[k], np.abs(mr.edge_weights(meas, dirs[k])), 0.0)
    assert np.array_equal(_bits(s), _bits(want))
    sub = dirs[:: 125]  # 16 directions against the vectorised oracle
    _, order = outlier_weights_arrays(ctx, V, ea, eb, meas, sub, order=True)
    inc = mr.incidence(V, ea, eb)
    for k, dk in enumerate(sub):
        o2, b2 = mr.order_vectorised(V, ea, eb, meas, dk, inc)
        assert np.array_equal(order[k], o2), k
        assert np.array_equal(bad[k * 125], b2), k


def test_argument_checks(ctx):
    from gtsfm_b200 import _lib
    from gtsfm_b200.translation_averaging import outlier_weights_arrays

    m = np.tile(mr.unit3(np.array([1.0, 2.0, 3.0])), (3, 1))
    dirs = np.eye(3)
    outlier_weights_arrays(ctx, 3, [0, 1, 2], [1, 2, 0], m, dirs)  # fine: a cycle
    for a, b, V in (([0, 0, 1], [1, 1, 2], 3),  # repeated edge
                    ([0, 1, 1], [1, 0, 2], 3),  # the same pair in both orientations
                    ([0, 1, 2], [0, 2, 0], 3),  # a self edge
                    ([1, 0, 2], [2, 1, 0], 3),  # out of order
                    ([0, 1, 2], [1, 2, 3], 3)):  # an id outside [0, V)
        with pytest.raises(_lib.B200Error):
            outlier_weights_arrays(ctx, V, a, b, m, dirs)
    with pytest.raises(_lib.B200Error):
        outlier_weights_arrays(ctx, 3, [0, 1, 2], [1, 2, 0], m, np.array([[np.nan, 0, 1.0]]))
    s = outlier_weights_arrays(ctx, 3, [0, 1, 2], [1, 2, 0], m, np.zeros((0, 3)))
    assert (s == 0).all()
    s, order = outlier_weights_arrays(ctx, 4, np.zeros(0), np.zeros(0), np.zeros((0, 3)), dirs, order=True)
    assert len(s) == 0 and (order == np.arange(4)).all()  # isolated nodes are all sources: lowest id first


def test_plugin_compute_inliers(ctx):
    from gtsfm_b200.translation_averaging import B200TranslationAveraging1DSFM

    for f, name in (("mfas_lund_door.npz", "lund_door"), ("mfas_scenes.npz", "knn_tracks_uniform"),
                    ("mfas_scenes.npz", "knn_outliers_30"), ("mfas_scenes.npz", "empty")):
        d = np.load(GOLDEN / f)
        cam = {tuple(int(x) for x in k): v for k, v in zip(d[f"{name}/cam_keys"], d[f"{name}/cam_vecs"])}
        trk = {tuple(int(x) for x in k): v for k, v in zip(d[f"{name}/trk_keys"], d[f"{name}/trk_vecs"])}
        t = B200TranslationAveraging1DSFM(projection_sampling_method=str(d[f"{name}/method"]), ctx=ctx)
        c, tr, ic = t.compute_inliers(cam, trk)
        assert [k in c for k in cam] == d[f"{name}/inlier_cam"].tolist(), name
        assert [k in tr for k in trk] == d[f"{name}/inlier_trk"].tolist(), name
        assert sorted(ic) == d[f"{name}/inlier_cameras"].tolist(), name
    # the reference's Test1dsfmAllOutliers: every edge to camera 4 is rejected
    w = mr.all_outliers_inputs()
    c, tr, ic = B200TranslationAveraging1DSFM(ctx=ctx).compute_inliers(w, {})
    assert set(c) == {k for k in w if 4 not in k} and ic == {0, 1, 2, 3} and tr == {}
