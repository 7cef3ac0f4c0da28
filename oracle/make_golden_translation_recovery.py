"""Writes the fixtures of 1DSfM's translation recovery (oracle/translation_recovery_ref.py):

    tests/golden/translation_recovery_scenes.npz  seeded scenes: kNN camera graphs with and without track landmarks, with
        outlier directions; Huber on and off; scale 0 and 1; a landmark held by a single edge (only the damping holds it
        along that edge); two components; two cameras; two consecutive calls that continue the random stream; and
        lund-door's inlier camera and track directions as the device's compute_inliers returns them
        (tests/golden/mfas_lund_door.npz)

    python -m oracle.make_golden_translation_recovery --reference /path/to/gtsfm-checkout

Every scene is run through the reference's own TranslationAveraging1DSFM.__run_averaging (averaging_1dsfm.py:439-495)
from the checkout's sources, under make_golden_mfas's stand-ins plus these: gtsam.noiseModel records the models it
builds, BinaryMeasurementUnit3 keeps its keys, measurement and model, and TranslationRecovery records what run() is given
(the measurements in order, the scale) and runs the restatement from the restated process-wide std::mt19937(42).  Before
writing, the recorded graph must be the one the device is given: edges in the reference's order, the Isotropic sigma
0.01 model, Huber 1.3 exactly when robust_measurement_noise is set, and the scale.

Stored per scene, under "<name>/": cam_keys (nc, 2) (i1, i2), cam_vecs (nc, 3), trk_keys (nt, 2) (j, i), trk_vecs (nt, 3) in
dict order; num_images; robust; scale; rng_skip (Point3 draws a fresh process made before this call); the dense problem
C, L, cams, tracks, edge_a, edge_b, meas, init; and the restatement's x (C + L, 3), trace, trials, iterations,
final_error and wti (num_images, 3), NaN where the reference returns None.
"""
from __future__ import annotations

import argparse
import sys
import types
from pathlib import Path

import numpy as np

from oracle import mfas_ref as mr
from oracle import translation_recovery_ref as tr
from oracle.make_golden_mfas import _Rot3, _Unit3, _reference, knn_graph

ROOT = Path(__file__).resolve().parents[1]
OUT = ROOT / "tests/golden/translation_recovery_scenes.npz"


# ---- stand-ins ------------------------------------------------------------------------------------------------------
class _Isotropic:
    @staticmethod
    def Sigma(dim, sigma):  # noqa: N802 - gtsam's name
        return ("isotropic", int(dim), float(sigma))


class _Huber:
    @staticmethod
    def Create(k):  # noqa: N802
        return ("huber", float(k))


class _Robust:
    @staticmethod
    def Create(loss, model):  # noqa: N802
        return ("robust", loss, model)


class _Binary:
    def __init__(self, k1, k2, m, noise):
        self.k = (int(k1), int(k2))
        self.m = m
        self.noise = noise

    def key1(self):  # the MFAS stand-in's reading
        return self.k[0]

    def key2(self):
        return self.k[1]

    def measured(self):
        return self.m


class _Values:
    def __init__(self, d):
        self.d = d

    def exists(self, k):
        return int(k) in self.d

    def atPoint3(self, k):  # noqa: N802
        return self.d[int(k)].copy()


STREAM = {"u": None, "drawn": 0}  # the restated process-wide generator of this generating process


class _TranslationRecovery:
    last = None

    def run(self, measurements, scale, *rest):
        assert not rest, "the fixtures have no relative pose priors"
        keys = [b.k for b in measurements]
        _TranslationRecovery.last = rec = dict(keys=keys, noise=[b.noise for b in measurements], scale=float(scale),
                                               meas=[b.m.point3() for b in measurements])
        if not keys:
            return _Values({})
        cams = sorted({k for ab in keys for k in ab if k >> 56 == ord("a")})
        lmks = sorted({k for ab in keys for k in ab if k >> 56 == ord("b")})
        ids = {k: n for n, k in enumerate(cams + lmks)}
        noise = rec["noise"][0]
        robust = noise[0] == "robust"
        out = tr.run(len(cams), len(lmks), [ids[a] for a, _ in keys], [ids[b] for _, b in keys], np.array(rec["meas"]), STREAM["u"],
                     huber_k=noise[1][1] if robust else 0.0, scale=float(scale))
        STREAM["drawn"] += len(out["nodes"])
        rec.update(out, cams=cams, lmks=lmks)
        return _Values({k: out["x"][n] for k, n in ids.items() if np.all(np.isfinite(out["x"][n]))})


def _gtsam_standins(r):
    r["gtsam"] = types.SimpleNamespace(noiseModel=types.SimpleNamespace(Isotropic=_Isotropic, Robust=_Robust,
                                                                        mEstimator=types.SimpleNamespace(Huber=_Huber)))
    r["BinaryMeasurementUnit3"] = _Binary
    r["TranslationRecovery"] = _TranslationRecovery
    r["Unit3"] = _Unit3Eigen
    r["Pose3"] = lambda R, t: (R, np.asarray(t, float))
    return r


class _Unit3Eigen(_Unit3):
    """gtsam.Unit3(p): Eigen's normalized(), which leaves a zero vector zero (the panorama's zero translations)."""

    def __init__(self, p=None):
        p = np.asarray(p, float).reshape(3)
        self._p = mr.unit3(p) if np.any(p != 0.0) else p.copy()


# ---- scenes -----------------------------------------------------------------------------------------------------------
def _perturbed(rng, cam, trk, frac):
    """Replace `frac` of the directions by random ones (outliers the Huber model down-weights)."""
    cam = {k: mr.unit3(rng.normal(size=3)) if rng.random() < frac else v for k, v in cam.items()}
    trk = {k: mr.unit3(rng.normal(size=3)) if rng.random() < frac else v for k, v in trk.items()}
    return cam, trk


def scenes(seed=3):
    """name -> (cam dict, trk dict, robust, scale, num_images, continues the previous scene's stream)."""
    rng = np.random.default_rng(seed)
    out = {}
    cam, trk = knn_graph(rng, 12, 3, 0.0)
    out["knn_cams"] = (cam, trk, True, 1.0, 12, False)
    cam, trk = knn_graph(rng, 10, 3, 0.0, n_landmarks=15, views=(2, 4))
    out["knn_tracks_huber"] = (*_perturbed(rng, cam, trk, 0.1), True, 1.0, 10, False)
    out["knn_tracks_gauss"] = (*_perturbed(rng, cam, trk, 0.0), False, 1.0, 10, False)
    cam, trk = knn_graph(rng, 9, 3, 0.0, n_landmarks=8)
    out["scale_zero"] = (cam, trk, True, 0.0, 9, False)
    cam, trk = knn_graph(rng, 8, 3, 0.0, n_landmarks=6)
    trk[(99, 3)] = mr.unit3(np.array([0.2, -0.4, 0.9]))  # a landmark with one edge: only the damping holds it along the ray
    out["single_edge_landmark"] = (cam, trk, True, 1.0, 8, False)
    c1, t1 = knn_graph(rng, 6, 2, 0.0, n_landmarks=4)
    c2, _ = knn_graph(rng, 5, 2, 0.0)
    out["two_components"] = (c1 | {(i1 + 6, i2 + 6): v for (i1, i2), v in c2.items()}, t1, True, 1.0, 11, False)
    out["two_cameras"] = ({(0, 1): mr.unit3(np.array([0.6, -0.1, 0.8]))}, {}, True, 1.0, 2, False)
    cam, trk = knn_graph(rng, 7, 3, 0.0, n_landmarks=5)
    out["consecutive_1"] = (cam, trk, True, 1.0, 7, False)
    cam, trk = knn_graph(rng, 6, 3, 0.0)
    out["consecutive_2"] = (cam, trk, True, 1.0, 6, True)
    z = np.load(ROOT / "tests/golden/mfas_lund_door.npz")
    ck, cv, tk, tv_ = (z[f"lund_door/{k}"] for k in ("cam_keys", "cam_vecs", "trk_keys", "trk_vecs"))
    ic, it = z["lund_door/inlier_cam"], z["lund_door/inlier_trk"]
    out["lund_door"] = ({tuple(map(int, k)): v for k, v, f in zip(ck, cv, ic) if f},
                        {tuple(map(int, k)): v for k, v, f in zip(tk, tv_, it) if f}, True, 1.0, 12, False)
    return out


def run(r, cam, trk, robust, scale, num_images, skip):
    """The reference's __run_averaging on (cam, trk); asserts the recorded graph; -> the fixture's arrays."""
    obj = r["TranslationAveraging1DSFM"](robust_measurement_noise=robust)
    cu = {k: _Unit3(v) for k, v in cam.items()}
    tu = {k: _Unit3(v) for k, v in trk.items()}
    wRi = [_Rot3(np.eye(3)) for _ in range(num_images)]
    wti = obj._TranslationAveraging1DSFM__run_averaging(num_images=num_images, w_i2Ui1_dict=cu, w_i2Ui1_dict_tracks=tu, wRi_list=wRi,
                                                        i2Ti1_priors={}, absolute_pose_priors=[], scale_factor=scale)
    rec = _TranslationRecovery.last
    expect = [(mr.C(i2), mr.C(i1)) for (i1, i2) in cam] + [(mr.C(i), mr.L(j)) for (j, i) in trk]
    assert rec["keys"] == expect, "the measurements are not in the reference's list order"
    base = ("isotropic", 2, 0.01)
    assert all(n == (("robust", ("huber", 1.3), base) if robust else base) for n in rec["noise"]), "unexpected noise model"
    assert rec["scale"] == scale
    return _record(rec, {k: u.point3() for k, u in cu.items()}, {k: u.point3() for k, u in tu.items()}, robust, scale, num_images, skip,
                   wti)


def _record(rec, cam, trk, robust, scale, num_images, skip, wti, gt=None):
    """The fixture's arrays of one recorded TranslationRecovery call (the reduced problem the device is given; empty when
    every edge joins one zero-translation set) and the reference's output wti."""
    w = np.full((num_images, 3), np.nan)
    for i, v in enumerate(wti):
        if v is not None:
            w[i] = v
    pr, res = rec.get("problem"), rec.get("result")
    d = dict(cam_keys=np.array(list(cam), np.int64).reshape(-1, 2), cam_vecs=np.array([np.asarray(v, float) for v in cam.values()]).reshape(-1, 3),
             trk_keys=np.array(list(trk), np.int64).reshape(-1, 2), trk_vecs=np.array([np.asarray(v, float) for v in trk.values()]).reshape(-1, 3),
             num_images=np.array(num_images), robust=np.array(robust), scale=np.array(scale), rng_skip=np.array(skip),
             cams=np.array([k & ((1 << 56) - 1) for k in rec["cams"]], np.int64),
             tracks=np.array([k & ((1 << 56) - 1) for k in rec["lmks"]], np.int64), root=rec["root"], nodes=rec["nodes"], wti=w)
    if pr is None:
        d.update(C=np.array(0), L=np.array(0), edge_a=np.zeros(0, np.int32), edge_b=np.zeros(0, np.int32), meas=np.zeros((0, 3)),
                 init=np.zeros((0, 3)), x=np.zeros((0, 3)), trace=np.zeros(0), trials=np.zeros(0, np.int32), iterations=np.array(0),
                 final_error=np.array(0.0))
    else:
        d.update(C=np.array(pr.C), L=np.array(pr.L), edge_a=pr.ea.astype(np.int32), edge_b=pr.eb.astype(np.int32), meas=pr.meas,
                 init=rec["init"], x=res.x, trace=np.array(res.trace), trials=np.array(res.trials, np.int32),
                 iterations=np.array(res.iterations), final_error=np.array(res.final_error))
    if gt is not None:
        d["gt_wti"] = np.asarray(gt, float)
    return d


# ---- the reference tests' own scenes, through the reference's run_translation_averaging ---------------------------------
def _rz(a):
    c, s_ = np.cos(a), np.sin(a)
    return np.array([[c, -s_, 0], [s_, c, 0], [0, 0, 1.0]])


def _ry(a):
    c, s_ = np.cos(a), np.sin(a)
    return np.array([[c, 0, s_], [0, 1.0, 0], [-s_, 0, c]])


def _rx(a):
    c, s_ = np.cos(a), np.sin(a)
    return np.array([[1.0, 0, 0], [0, c, -s_], [0, s_, c]])


def poses_on_circle(num_cameras=8, R=30.0):
    """gtsam.examples.SFMdata.posesOnCircle as published: Pose3(Rot3.Ypr(pi/2, 0, -pi/2), (R, 0, 0)), then each pose is
    Pose3(Rot3.Rz(2 pi / n), 0) composed with the previous one.  -> [(wRi, wti)]."""
    Rc, tc = _rz(np.pi / 2) @ _ry(0.0) @ _rx(-np.pi / 2), np.array([R, 0.0, 0.0])
    D = _rz(2 * np.pi / num_cameras)
    out = [(Rc, tc)]
    for _ in range(1, num_cameras):
        Rc, tc = D @ Rc, D @ tc
        out.append((Rc, tc))
    return out


def _between_dirs(poses, pairs):
    """{(i1, i2): Unit3(wTi2.between(wTi1).translation())} = R2^T (t1 - t2), normalised."""
    return {(i1, i2): poses[i2][0].T @ (poses[i1][1] - poses[i2][1]) for i1, i2 in pairs}


def lund_gt_poses():
    """lund-door's ground-truth poses (the Olsson loader's wTi, as tests/golden/twoview_report_lund_door.npz stores them)."""
    from oracle.make_golden_data_assoc import lund_matches

    _, _, cams = lund_matches()
    return [(cams[i, :9].reshape(3, 3), cams[i, 9:12].copy()) for i in range(12)]


def all_outliers_inputs(reference: Path):
    """Test1dsfmAllOutliers's wRi_list and i2Ui1_input, read from the reference test's source."""
    import ast

    src = (reference / "tests/averaging/translation/test_averaging_1dsfm.py").read_text()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "test_outlier_case_missing_value")
    vals = {}
    for node in fn.body:
        name = node.targets[0].id if isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name) else None
        if name in ("wRi_list", "i2Ui1_input") and name not in vals:  # the literals, not their later Rot3 / Unit3 wrapping
            vals[name] = eval(compile(ast.Expression(node.value), "<test>", "eval"), {"np": np})
    return [np.asarray(R, float) for R in vals["wRi_list"]], {k: np.asarray(v, float) for k, v in vals["i2Ui1_input"].items()}


def skydio32(reference: Path):
    """The reference's reproducibility inputs (tests/data/reproducibility/inputs/*skydio32.pkl): gtsam objects pickled as
    boost text archives, read by a stand-in unpickler (the last 9 or 3 numbers of each archive).  A Rot3 archive holds
    its nine matrix entries; gtsam's Rot3::serialize writes them as rot11, rot12, rot13, rot21, ..., i.e. row by row.
    The relative rotations cannot settle that here: over the 14 pairs they share with the post-Shonan rotations, their
    median distance to wRi2^T wRi1 is large in both orders (0.36 row-major, 0.24 column-major), so the two files do not
    come from one estimate.  The translation directions do: rotated into the world frame, every triangle of directions
    is closer to coplanar with row-major rotations; asserted below.  -> (wRi list with None, i2Ui1 dict, residuals)."""
    import pickle

    class _Obj:
        def __setstate__(self, st):
            self.v = np.array([float(x) for x in (st[0] if isinstance(st, tuple) else st).split()[-9:]])

    class _Unpickler(pickle.Unpickler):
        def find_class(self, module, name):
            return type(name, (_Obj,), {})

    base = reference / "tests/data/reproducibility/inputs"

    def load(f):
        with open(base / f, "rb") as fh:
            return _Unpickler(fh).load()

    wR, U = (load(f"{n}_skydio32.pkl") for n in ("global_rotations_post_shonan", "relative_unit_translations"))
    i2Ui1 = {k: v.v[-3:] for k, v in U.items()}
    res = {}
    for order in ("C", "F"):
        R = [None if x is None else x.v.reshape(3, 3, order=order) for x in wR]
        w = {k: R[k[1]] @ u for k, u in i2Ui1.items() if R[k[0]] is not None and R[k[1]] is not None}
        r = []  # |n . w_ac| / |n| with n = w_ab x w_bc: 0 for a consistent triangle of directions
        for (a, b) in w:
            for c in range(len(R)):
                if (b, c) in w and (a, c) in w:
                    n = np.cross(w[(a, b)], w[(b, c)])
                    r.append(abs(n @ w[(a, c)]) / np.linalg.norm(n))
        res[order] = float(np.median(r))
    assert res["C"] < res["F"], f"the triangles favour column-major Rot3 archives: {res}"
    wRi = [None if x is None else x.v.reshape(3, 3) for x in wR]
    return wRi, i2Ui1, res


def run_full(r, wRi, i2Ui1, num_images, skip, gt=None):
    """The reference's run_translation_averaging (get_valid_measurements_in_world_frame, compute_inliers with the restated
    MFAS and NumPy's seed 0, __run_averaging) with no tracks, as the reference's tests call it."""
    obj = r["TranslationAveraging1DSFM"]()
    captured = {}
    run_avg = obj._TranslationAveraging1DSFM__run_averaging

    def spy(**kw):
        captured.update(kw)
        return run_avg(**kw)

    obj._TranslationAveraging1DSFM__run_averaging = spy
    wRi_s = [None if R is None else _Rot3(R) for R in wRi]
    i2U = {k: _Unit3Eigen(v) for k, v in i2Ui1.items()}
    wTi, _, _ = obj.run_translation_averaging(num_images, i2U, wRi_s, tracks_2d=[], intrinsics=[None] * num_images)
    rec = _TranslationRecovery.last
    cam = {k: v.point3() for k, v in captured["w_i2Ui1_dict"].items()}
    assert rec["keys"] == [(mr.C(i2), mr.C(i1)) for (i1, i2) in cam], "the measurements are not in the reference's list order"
    wti = [None if p is None else p[1] for p in wTi]
    return _record(rec, cam, {}, True, 1.0, num_images, skip, wti, gt)


def reference_scenes(reference: Path):
    """name -> (wRi, i2Ui1, num_images, ground-truth wti or None)."""
    circle = poses_on_circle(R=40)[::2]
    pano_R = [_ry(np.deg2rad(a)) for a in (-30, 0, 30)]  # Rot3.RzRyRx(0, b, 0)
    pano = [(R, np.array([0.0, 2.0, 0.0])) for R in pano_R]
    lund = lund_gt_poses()
    circ8 = poses_on_circle(R=40)
    out = {
        "ref_circle_all_edges": ([p[0] for p in circle], _between_dirs(circle, [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]), 4,
                                 [p[1] for p in circle]),
        "ref_panorama": ([p[0] for p in pano], _between_dirs(pano, [(0, 1), (0, 2), (1, 2)]), 3, [p[1] for p in pano]),
        "ref_lund_door": ([p[0] for p in lund], _between_dirs(lund, [(i1, i2) for i1 in range(12) for i2 in range(i1 + 1, 12)]), 12,
                          [p[1] for p in lund]),
        "ref_poses_on_circle": ([p[0] for p in circ8], _between_dirs(circ8, [(i1, i2) for i1 in range(7) for i2 in range(i1 + 1, min(8, i1 + 3))]),
                                8, [p[1] for p in circ8]),
    }
    wRi, i2U = all_outliers_inputs(reference)
    out["ref_all_outliers"] = (wRi, i2U, 5, None)
    wRi, i2U, res = skydio32(reference)
    print(f"skydio-32: median triangle non-coplanarity {res['C']:.4f} row-major, {res['F']:.4f} column-major")
    out["ref_skydio32"] = (wRi, i2U, len(wRi), None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=Path, required=True, help="a GTSfM checkout (the pinned functions)")
    args = ap.parse_args()
    r = _gtsam_standins(_reference(args.reference)[0])
    arrays = {}
    names = []
    for name, (cam, trk, robust, scale, n, cont) in scenes().items():
        if not cont:
            STREAM["u"], STREAM["drawn"] = tr.Mt19937Uniform(42), 0
        res = run(r, cam, trk, robust, scale, n, STREAM["drawn"])
        names.append(name)
        arrays.update({f"{name}/{k}": v for k, v in res.items()})
        print(f"{name}: C={int(res['C'])} L={int(res['L'])} E={len(res['edge_a'])} iterations={int(res['iterations'])} "
              f"trials={len(res['trials'])} final_error={float(res['final_error']):.6g}")
    for name, (wRi, i2U, n, gt) in reference_scenes(args.reference).items():
        STREAM["u"], STREAM["drawn"] = tr.Mt19937Uniform(42), 0
        res = run_full(r, wRi, i2U, n, 0, gt)
        names.append(name)
        arrays.update({f"{name}/{k}": v for k, v in res.items()})
        print(f"{name}: C={int(res['C'])} L={int(res['L'])} E={len(res['edge_a'])} iterations={int(res['iterations'])} "
              f"trials={len(res['trials'])} None at {np.nonzero(np.isnan(res['wti'][:, 0]))[0].tolist()}")
    arrays["names"] = np.array(names)
    np.savez_compressed(OUT, **arrays)
    print(OUT)


if __name__ == "__main__":
    sys.exit(main())
