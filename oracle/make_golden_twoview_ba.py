"""Writes tests/golden/twoview_ba_scenes.npz: seeded two-view scenes for the device two-view refinement and what
oracle/twoview_ba_ref.py makes of them, and tests/golden/twoview_ba_lund_door.npz: lund-door's 66 pairs as the device
verifier hands them over, with the oracle's refinement of each.

    python -m oracle.make_golden_twoview_ba                          # the seeded scenes
    python -m oracle.make_golden_twoview_ba --dump-lund verified.npz  # on an H100: the device verifier's output
    python -m oracle.make_golden_twoview_ba --lund verified.npz       # the lund-door fixture from that output

Each scene is one pair as verification hands it over: pixel coordinates of the k putative rows, the verified rows, the
intrinsics (f, u0, v0) of both images and the verified i2Ri1 / unit i2ti1.  Scenes with known K, R and t carry 0.5 px
noise, 0-30 % outliers among the verified rows (offsets of 2-20 px that verification let through) and an initial pose
perturbed by up to 2 degrees; the degenerate ones are a pure rotation, fewer than 15 verified rows, every point behind
a camera, and a single track that triangulates.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np

from oracle import twoview_ba_ref as ref

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"
OUT = GOLDEN / "twoview_ba_scenes.npz"
OUT_LUND = GOLDEN / "twoview_ba_lund_door.npz"


def lund_inputs():
    """Lund-door's 12 images as the reference selected their SuperPoint keypoints (tests/golden/lund_door_images.npz), its
    66 LightGlue match arrays (lund_door_66pairs.npz), and a stand-in calibration: f = 1.2 x the longer side, the
    principal point at the centre (the fixtures carry no EXIF).  -> (keypoints {i: (n, 2) float32}, pairs, {pair: rows},
    (f, u0, v0))."""
    img = np.load(GOLDEN / "lund_door_images.npz")
    fx = np.load(GOLDEN / "lund_door_66pairs.npz")
    h, w = img["gray_1"].shape
    kps = {i: img[f"kp_{i}"].astype(np.float32)[img[f"sel_{i}"]] for i in range(1, 13)}
    pairs = [(a, b) for a in range(1, 13) for b in range(a + 1, 13)]
    return kps, pairs, {p: fx[f"m_{p[0]}_{p[1]}"].astype(np.int64) for p in pairs}, (1.2 * max(h, w), w / 2.0, h / 2.0)


def dump_lund_verified(path):
    """Runs the device verifier (B200TwoViewBatch, RANSAC 5-point, 4 px) on lund-door's 66 pairs and saves, per pair, the
    verified row indices, R and unit t (needs an H100)."""
    import torch

    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd
    from gtsfm_b200.two_view import B200TwoViewBatch

    kps, pairs, rows, cal = lund_inputs()
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), max_keypoints=64)
    feats = {i: DeviceFeatures(torch.from_numpy(k).cuda(), torch.zeros(len(k), device="cuda"), torch.zeros((len(k), 1), device="cuda"),
                               (0, 0)) for i, k in kps.items()}
    res = B200TwoViewBatch(fe, 4.0).run(feats, pairs, {i: cal for i in kps}, {p: torch.from_numpy(m).cuda() for p, m in rows.items()})
    out = {}
    for p in pairs:
        r, m = res[p], rows[p]
        row_of = {tuple(x): j for j, x in enumerate(m)}
        out[f"{p[0]}_{p[1]}/ok"] = np.array(r.i2Ri1 is not None)
        out[f"{p[0]}_{p[1]}/verified"] = np.array(sorted(row_of[tuple(x)] for x in r.v_corr_idxs), np.int64)
        out[f"{p[0]}_{p[1]}/R0"] = r.i2Ri1.matrix() if r.i2Ri1 is not None else np.full((3, 3), np.nan)
        out[f"{p[0]}_{p[1]}/t0"] = r.i2Ui1.point3() if r.i2Ui1 is not None else np.full(3, np.nan)
    np.savez_compressed(path, **out)


def lund_fixture(verified_path):
    """The oracle's refinement of every pair of a dump_lund_verified() file -> OUT_LUND (inputs and outputs)."""
    kps, pairs, rows, cal = lund_inputs()
    v = np.load(verified_path)
    arrays = {}
    for p in pairs:
        key = f"{p[0]}_{p[1]}"
        m = rows[p]
        for name in ("ok", "verified", "R0", "t0"):
            arrays[f"{key}/{name}"] = v[f"{key}/{name}"]
        if not bool(v[f"{key}/ok"]):
            continue
        r = ref.refine_pair(kps[p[0]][m[:, 0]].astype(np.float64), kps[p[1]][m[:, 1]].astype(np.float64), v[f"{key}/verified"],
                            len(m), cal, cal, v[f"{key}/R0"], v[f"{key}/t0"])
        arrays[f"{key}/out_ok"] = np.array(r.ok)
        arrays[f"{key}/out_R"] = np.asarray(r.R if r.R is not None else np.full((3, 3), np.nan))
        arrays[f"{key}/out_t"] = np.asarray(r.t if r.t is not None else np.full(3, np.nan))
        arrays[f"{key}/out_rows"] = r.rows
        arrays[f"{key}/out_trace"] = np.asarray(r.trace, float)
        arrays[f"{key}/out_track_rows"] = r.track_rows
        arrays[f"{key}/out_track_err"] = r.track_err
        print(f"{key}: verified {len(v[key + '/verified'])} ok={r.ok} tracks={r.num_tracks} kept={len(r.rows)} iters={r.iterations}")
    np.savez_compressed(OUT_LUND, **arrays)
    print(OUT_LUND)


def _rot(axis, deg):
    a = np.asarray(axis, float)
    return ref.so3_exp(a / np.linalg.norm(a) * np.radians(deg))


def synthetic_scene(seed: int, n: int, noise_px=0.5, outlier_frac=0.0, perturb_deg=2.0, baseline=1.0, n_front=None,
                    n_unverified=None):
    """-> dict(uv1, uv2, verified, k, cal1, cal2, R0, t0, R_true, t_true) for one seeded pair.  Points from index
    `n_front` on lie behind both cameras (depth negated)."""
    g = np.random.default_rng(seed)
    cal1 = (float(g.uniform(450, 650)), 320.0 + float(g.uniform(-10, 10)), 240.0 + float(g.uniform(-10, 10)))
    cal2 = (float(g.uniform(450, 650)), 320.0 + float(g.uniform(-10, 10)), 240.0 + float(g.uniform(-10, 10)))
    R = _rot(g.normal(size=3), g.uniform(3, 15))
    c2 = np.array([1.0, float(g.uniform(-0.2, 0.2)), float(g.uniform(-0.2, 0.2))]) * baseline  # camera 2 centre in frame 1
    t = -R @ c2  # i2ti1: x2 = R x1 + t
    X = np.stack([g.uniform(-3, 3, n), g.uniform(-2, 2, n), g.uniform(5, 12, n)], 1)
    if n_front is not None:
        X[n_front:] *= -1.0
    x2 = X @ R.T + t

    def proj(P, cal):
        return np.stack([cal[1] + cal[0] * P[:, 0] / P[:, 2], cal[2] + cal[0] * P[:, 1] / P[:, 2]], 1)

    uv1 = proj(X, cal1) + g.normal(scale=noise_px, size=(n, 2))
    uv2 = proj(x2, cal2) + g.normal(scale=noise_px, size=(n, 2))
    n_out = int(round(outlier_frac * n))
    if n_out:
        idx = g.choice(n, n_out, replace=False)
        off = g.normal(size=(n_out, 2))
        uv2[idx] += off / np.linalg.norm(off, axis=1, keepdims=True) * g.uniform(2, 20, (n_out, 1))
    nu = n // 5 if n_unverified is None else n_unverified  # putative rows that verification rejected: random pixels
    uv1 = np.concatenate([uv1, g.uniform([0, 0], [640, 480], (nu, 2))])
    uv2 = np.concatenate([uv2, g.uniform([0, 0], [640, 480], (nu, 2))])
    perm = g.permutation(n + nu)
    inv = np.argsort(perm)
    verified = np.sort(inv[:n])
    R0 = _rot(g.normal(size=3), g.uniform(0, perturb_deg)) @ R
    tu = t / np.linalg.norm(t) if np.linalg.norm(t) > 0 else np.array([1.0, 0.0, 0.0])
    t0 = _rot(g.normal(size=3), g.uniform(0, perturb_deg)) @ tu
    # keypoints are float32 in the library: the scene's pixels are the float32 values, read back as doubles
    uv1, uv2 = (u.astype(np.float32).astype(np.float64) for u in (uv1, uv2))
    return dict(uv1=uv1[perm], uv2=uv2[perm], verified=verified, k=n + nu, cal1=np.array(cal1), cal2=np.array(cal2),
                R0=R0, t0=t0 / np.linalg.norm(t0), R_true=R, t_true=tu)


# name -> synthetic_scene arguments
SCENES = {
    "clean_40": dict(seed=1, n=40, noise_px=0.0, perturb_deg=0.0),
    "noisy_60": dict(seed=2, n=60),
    "outliers10_120": dict(seed=3, n=120, outlier_frac=0.1),
    "outliers30_200": dict(seed=4, n=200, outlier_frac=0.3),
    "noisy_500": dict(seed=5, n=500, outlier_frac=0.05),
    "outliers20_1000": dict(seed=6, n=1000, outlier_frac=0.2),
    "pure_rotation": dict(seed=7, n=80, baseline=0.0),
    "few_inliers": dict(seed=8, n=12),
    "behind": dict(seed=9, n=50, n_front=0),
    "single_track": dict(seed=11, n=16, n_front=1, n_unverified=0),
    "low_ratio": dict(seed=10, n=20, n_unverified=400),
}


def all_scenes():
    return {name: synthetic_scene(**kw) for name, kw in SCENES.items()}


def run_oracle(s, **kw):
    return ref.refine_pair(s["uv1"], s["uv2"], s["verified"], s["k"], s["cal1"], s["cal2"], s["R0"], s["t0"], **kw)


def main() -> None:
    arrays = {}
    for name, s in all_scenes().items():
        r = run_oracle(s)
        for key, v in s.items():
            arrays[f"{name}/{key}"] = np.asarray(v)
        arrays[f"{name}/out_ok"] = np.array(r.ok)
        arrays[f"{name}/out_R"] = np.asarray(r.R if r.R is not None else np.full((3, 3), np.nan))
        arrays[f"{name}/out_t"] = np.asarray(r.t if r.t is not None else np.full(3, np.nan))
        arrays[f"{name}/out_rows"] = r.rows
        arrays[f"{name}/out_trace"] = np.asarray(r.trace, float)
        arrays[f"{name}/out_track_rows"] = r.track_rows
        arrays[f"{name}/out_track_err"] = r.track_err
        arrays[f"{name}/out_num_tracks"] = np.array(r.num_tracks)
        print(f"{name}: ok={r.ok} tracks={r.num_tracks} kept={len(r.rows)} iters={r.iterations} "
              f"cost {r.trace[0] if r.trace else 0:.4g} -> {r.trace[-1] if r.trace else 0:.4g}")
    np.savez_compressed(OUT, names=np.array(sorted(all_scenes())), **arrays)
    print(OUT)


if __name__ == "__main__":
    import sys

    if "--dump-lund" in sys.argv:
        dump_lund_verified(sys.argv[sys.argv.index("--dump-lund") + 1])
    elif "--lund" in sys.argv:
        lund_fixture(sys.argv[sys.argv.index("--lund") + 1])
    else:
        main()
