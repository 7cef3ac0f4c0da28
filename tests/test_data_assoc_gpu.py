"""Data association's triangulation on the device (b2_triangulate_tracks_host) against oracle/data_assoc_ref.py: the seeded
scenes of tests/golden/data_assoc_scenes.npz, chunked against unchunked runs, shuffled track order, a large seeded scene
on a random subset of its tracks, and the plugin's object path against its array path."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import data_assoc_ref as da  # noqa: E402
from oracle.make_golden_data_assoc import geometric_lengths, make_tracks, ring_cameras  # noqa: E402

pytestmark = pytest.mark.gpu

# Points and average errors: the device's QR-reduced DLT and streamed LM against NumPy's SVD and sums
POINT_RTOL, ERR_ATOL = 1e-7, 1e-7
NEAR_THR_PX = 1e-6  # a measurement this close to the threshold may fall on either side


def _scenes(path=ROOT / "tests/golden/data_assoc_scenes.npz"):
    z = np.load(path)
    out = {}
    for k in z.files:
        name, key = k.split("/")
        out.setdefault(name, {})[key] = z[k]
    return out


SCENES = _scenes()
LUND = _scenes(ROOT / "tests/golden/data_assoc_lund_door.npz")


@pytest.fixture(scope="module")
def ctx():
    from gtsfm_b200 import _lib

    return _lib.Context(0)


def plugin(ctx, options, seed=None, **kw):
    from gtsfm_b200.data_association import B200DataAssociation
    from gtsfm_b200.gtsfm_api import TriangulationOptions, TriangulationSamplingMode

    mode = TriangulationSamplingMode.RANSAC_SAMPLE_UNIFORM if options[0] else TriangulationSamplingMode.NO_RANSAC
    opts = TriangulationOptions(mode, reproj_error_threshold=float(options[2]), min_triangulation_angle=float(options[3]),
                                max_num_hypotheses=int(options[1]), **kw)
    return B200DataAssociation(min_track_len=2, triangulation_options=opts, seed=int(options[4] if seed is None else seed), ctx=ctx)


def run(ctx, sc):
    return plugin(ctx, sc["options"]).triangulate_arrays(sc["track_off"], sc["meas_cam"], sc["meas_uv"], sc["cams"], sc["cam_valid"])


def near_threshold(sc, t, X_a, X_b):
    """True when some measurement of track t lies within NEAR_THR_PX of the threshold under either point."""
    thr = float(sc["options"][2])
    if not np.isfinite(thr):
        return False
    cams = da.cams_dict(sc["cams"], sc["cam_valid"])
    a, b = sc["track_off"][t], sc["track_off"][t + 1]
    meas = [(int(sc["meas_cam"][m]), sc["meas_uv"][m]) for m in range(a, b)]
    for X in (X_a, X_b):
        if X is not None and np.all(np.isfinite(X)):
            e = da.reproj_errors(cams, X, meas)
            if np.any(np.abs(e[np.isfinite(e)] - thr) < NEAR_THR_PX):
                return True
    return False


def compare(sc, got, want, max_near=0):
    ex, pt, avg, inl = got
    wex, wpt, wavg, winl = want
    off = sc["track_off"]
    near = 0
    for t in range(len(off) - 1):
        a, b = off[t], off[t + 1]
        if ex[t] != wex[t] or not np.array_equal(inl[a:b], winl[a:b].astype(bool)):
            assert near_threshold(sc, t, pt[t], wpt[t]), f"track {t}: exit {ex[t]} vs {wex[t]}, inliers differ away from the threshold"
            near += 1
            continue
        np.testing.assert_allclose(pt[t], wpt[t], rtol=POINT_RTOL, atol=POINT_RTOL, equal_nan=True, err_msg=f"track {t}")
        np.testing.assert_allclose(avg[t], wavg[t], rtol=ERR_ATOL, atol=ERR_ATOL, equal_nan=True, err_msg=f"track {t}")
    assert near <= max_near
    return near


@pytest.mark.parametrize("name", sorted(SCENES))
def test_scene_equals_fixture(ctx, name):
    sc = SCENES[name]
    compare(sc, run(ctx, sc), (sc["exit"], sc["point"], sc["avg"], sc["inlier"]))


@pytest.mark.parametrize("name", sorted(LUND))
def test_lund_door_equals_fixture(ctx, name):
    sc = LUND[name]
    compare(sc, run(ctx, sc), (sc["exit"], sc["point"], sc["avg"], sc["inlier"]))


def _large_scene(seed=5, num_cams=500, T=100_000, max_len=100):
    rng = np.random.default_rng(seed)
    cams = ring_cameras(rng, num_cams, radius=30.0)
    valid = np.ones(num_cams, np.uint8)
    valid[rng.choice(num_cams, 5, replace=False)] = 0
    lengths = geometric_lengths(rng, T, 0.3, 2, max_len)
    off, cam, uv = da.pack_tracks(make_tracks(rng, cams, lengths, outlier_frac=0.1))
    return dict(track_off=off, meas_cam=cam, meas_uv=uv, cams=cams, cam_valid=valid, options=np.array([1.0, 100, 10.0, 0.0, 11]))


def test_chunked_run_is_bit_identical(ctx):
    sc = _large_scene(T=40_000)
    one = run(ctx, sc)
    ctx.set_option("data_assoc_workspace_mb", 1)
    try:
        launches = ctx.launch_count()
        many = run(ctx, sc)
        assert ctx.launch_count() - launches >= 6  # several chunks of two launches
    finally:
        ctx.set_option("data_assoc_workspace_mb", 256)
    for a, b in zip(one, many):
        assert a.tobytes() == b.tobytes()


def test_shuffled_tracks_give_identical_results_when_exhaustive(ctx):
    full = SCENES["outliers_30"]
    fo = full["track_off"]
    n = np.diff(fo)
    keep = [t for t in range(len(n)) if n[t] * (n[t] - 1) // 2 <= full["options"][1]]  # every pair is a hypothesis
    o0, c0, u0 = da.pack_tracks([[(int(full["meas_cam"][m]), full["meas_uv"][m]) for m in range(fo[t], fo[t + 1])] for t in keep])
    sc = dict(full, track_off=o0, meas_cam=c0, meas_uv=u0)
    off = sc["track_off"]
    assert len(keep) > 200
    base = run(ctx, sc)
    perm = np.random.default_rng(0).permutation(len(keep))
    tracks = [[(int(sc["meas_cam"][m]), sc["meas_uv"][m]) for m in range(off[t], off[t + 1])] for t in perm]
    o2, c2, u2 = da.pack_tracks(tracks)
    sh = dict(sc, track_off=o2, meas_cam=c2, meas_uv=u2)
    got = run(ctx, sh)
    for j, t in enumerate(perm):
        assert got[0][j] == base[0][t]
        assert got[1][j].tobytes() == base[1][t].tobytes() and got[2][j].tobytes() == base[2][t].tobytes()
        assert np.array_equal(got[3][o2[j]:o2[j + 1]], base[3][off[t]:off[t + 1]])


def test_large_scene_agrees_with_oracle_on_a_subset(ctx):
    sc = _large_scene()
    got = run(ctx, sc)
    T = len(sc["track_off"]) - 1
    rng = np.random.default_rng(1)
    pick = np.sort(rng.choice(T, 3000, replace=False))
    long = np.flatnonzero(np.diff(sc["track_off"]) >= 15)[:50]  # sampled tracks
    pick = np.union1d(pick, long)
    want = da.run_arrays(sc["track_off"], sc["meas_cam"], sc["meas_uv"], sc["cams"], sc["cam_valid"], da.SAMPLE_UNIFORM, 100, 10.0, 0.0,
                         11, pick)
    off = sc["track_off"]
    near = 0
    for t in pick:
        a, b = off[t], off[t + 1]
        if got[0][t] != want[0][t] or not np.array_equal(got[3][a:b], want[3][a:b].astype(bool)):
            assert near_threshold(sc, t, got[1][t], want[1][t]), f"track {t}"
            near += 1
            continue
        np.testing.assert_allclose(got[1][t], want[1][t], rtol=POINT_RTOL, atol=POINT_RTOL, equal_nan=True)
        np.testing.assert_allclose(got[2][t], want[2][t], rtol=ERR_ATOL, atol=ERR_ATOL, equal_nan=True)
    assert near <= 3


def test_plugin_objects_equal_the_array_path(ctx):
    from gtsfm_b200.data_association import unpack
    from gtsfm_b200.gtsfm_api import SfmMeasurement, SfmTrack2d, TriangulationExitCode

    sc = SCENES["missing_uniform"]
    pl = plugin(ctx, sc["options"])
    off = sc["track_off"]
    tracks = [SfmTrack2d([SfmMeasurement(int(sc["meas_cam"][m]), sc["meas_uv"][m]) for m in range(off[t], off[t + 1])])
              for t in range(len(off) - 1)]
    cameras = {i: (c[:9].reshape(3, 3), c[9:12], c[12], c[13], c[14]) for i, c in enumerate(sc["cams"]) if sc["cam_valid"][i]}
    s, e, c = pl.run_triangulation(cameras, tracks)
    # the plugin sizes its camera table by the largest index present; the array path takes the fixture's whole table
    ex, pt, avg, inl = run(ctx, sc)
    s2, e2, c2 = unpack(tracks, off, ex, pt, avg, inl)
    assert c == c2 and len(s) == len(tracks)
    assert [x is None for x in e] == [x is None for x in e2]
    assert all(x is None or x == y for x, y in zip(e, e2))
    for a, b, code in zip(s, s2, c):
        assert (a is None) == (b is None) == (code != TriangulationExitCode.SUCCESS)
        if a is not None:
            assert np.array_equal(a.point3(), b.point3()) and a.numberMeasurements() == b.numberMeasurements()


def test_bad_arguments_are_rejected(ctx):
    from gtsfm_b200 import _lib

    sc = SCENES["clean_uniform"]
    pl = plugin(ctx, sc["options"])
    bad = sc["meas_cam"].copy()
    bad[0] = len(sc["cams"])
    with pytest.raises(_lib.B200Error):
        pl.triangulate_arrays(sc["track_off"], bad, sc["meas_uv"], sc["cams"], sc["cam_valid"])
    off = sc["track_off"].copy()
    off[1], off[2] = off[2], off[1]
    with pytest.raises(_lib.B200Error):
        pl.triangulate_arrays(off, sc["meas_cam"], sc["meas_uv"], sc["cams"], sc["cam_valid"])
