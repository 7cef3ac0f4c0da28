"""CPU suite for the two-view refinement: the NumPy oracle (oracle/twoview_ba_ref.py) against an independent minimiser of
the same robust cost and against the reference's own test criteria, and the host build of csrc/twoview_math.cuh (what
the device compiles) against the oracle."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import make_golden_twoview_ba as mg
from oracle import twoview_ba_ref as ref

ROOT = Path(__file__).resolve().parent.parent


def _angle(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1.0) / 2.0, -1.0, 1.0)))


def _problem(scene):
    """The oracle's BA input for a scene: triangulated tracks in the initial cameras."""
    s = scene
    K = [np.array([s["cal1"][0], 0, 0, s["cal1"][1], s["cal1"][2]]), np.array([s["cal2"][0], 0, 0, s["cal2"][1], s["cal2"][2]])]
    R0, t0 = s["R0"], s["t0"]
    cams = [(np.eye(3), np.zeros(3), K[0]), (R0.T, -R0.T @ t0, K[1])]
    keep, pts = [], []
    for i in s["verified"]:
        X = ref.triangulate(cams, s["uv1"][i], s["uv2"][i])
        if X is not None:
            keep.append(i)
            pts.append(X)
    pts = np.array(pts)
    uv = np.stack([s["uv1"][keep], s["uv2"][keep]], 1)
    st = ref.BAState([cams[0][0], cams[1][0]], [cams[0][1], cams[1][1]], [K[0].copy(), K[1].copy()], pts)
    return st, ref.BAProblem(uv, pts[0].copy(), [K[0].copy(), K[1].copy()])


def test_oracle_reaches_the_robust_optimum(monkeypatch):
    """Run to convergence (tolerances 0), the oracle's LM lands where scipy's BFGS lands on the explicit cost
    sum rho(|e|) + priors, written here in torch (autograd gradients, its own projection and SE(3) log): cost to 1e-9
    relative, rotations to 1e-7 rad."""
    torch = pytest.importorskip("torch")
    from scipy.optimize import minimize

    scene = mg.synthetic_scene(seed=21, n=30, outlier_frac=0.1)
    st, pr = _problem(scene)
    monkeypatch.setattr(ref, "LM_REL_TOL", 0.0)
    monkeypatch.setattr(ref, "LM_ABS_TOL", 0.0)
    opt, _ = ref.bundle_adjust(st, pr, max_iters=500)
    c_lm = ref.ba_cost(opt, pr)

    T = torch.float64
    uv = torch.tensor(pr.uv, dtype=T)
    n = len(st.pts)

    def rodrigues(w):
        th = torch.sqrt((w * w).sum() + 1e-300)
        k = w / th
        Kx = torch.stack([torch.stack([0 * th, -k[2], k[1]]), torch.stack([k[2], 0 * th, -k[0]]), torch.stack([-k[1], k[0], 0 * th])])
        return torch.eye(3, dtype=T) + torch.sin(th) * Kx + (1 - torch.cos(th)) * Kx @ Kx

    R_init = [torch.tensor(r, dtype=T) for r in st.R]

    def unpack(x):
        cams = []
        for c in range(2):
            v = x[9 * c:9 * c + 9]
            cams.append((R_init[c] @ rodrigues(v[:3]), v[3:6], v[6:9]))
        return cams, x[18:].reshape(n, 3)

    def cost(x):
        cams, P = unpack(x)
        tot = 0.0
        for c, (R, t, fk) in enumerate(cams):
            pc = (P - t) @ R
            xn, yn = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
            r2 = xn * xn + yn * yn
            g = 1 + fk[1] * r2 + fk[2] * r2 * r2
            cal = pr.cal0[c]
            e = torch.sqrt((cal[3] + fk[0] * g * xn - uv[:, c, 0]) ** 2 + (cal[4] + fk[0] * g * yn - uv[:, c, 1]) ** 2)
            tot = tot + torch.where(e <= ref.HUBER_K, 0.5 * e * e, ref.HUBER_K * (e - 0.5 * ref.HUBER_K)).sum()
            tot = tot + 0.5 * (((fk - torch.tensor(cal[:3], dtype=T)) / ref.CAL_PRIOR_SIGMA) ** 2).sum()
        R, t, _ = cams[0]
        tr = R[0, 0] + R[1, 1] + R[2, 2]
        th = torch.arccos(torch.clamp((tr - 1) / 2, -1, 1))
        w = (th / (2 * torch.sin(th))) * torch.stack([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
        k = w / th
        Wk = lambda v: torch.linalg.cross(k, v)  # noqa: E731
        u = t - 0.5 * th * Wk(t) + (1 - th / (2 * torch.tan(0.5 * th))) * Wk(Wk(t))
        tot = tot + 0.5 * ((torch.cat([w, u]) / ref.POSE_PRIOR_SIGMA) ** 2).sum()
        return tot + 0.5 * (((P[0] - torch.tensor(pr.pt0, dtype=T)) / ref.POINT_PRIOR_SIGMA) ** 2).sum()

    x0 = np.concatenate([np.concatenate([[1e-3, 1e-3, 1e-3], st.t[c], st.cal[c][:3]]) for c in range(2)] + [st.pts.ravel()])

    def fg(x):
        xt = torch.tensor(x, dtype=T, requires_grad=True)
        f = cost(xt)
        f.backward()
        return float(f.detach()), xt.grad.numpy()

    # the calibration priors (sigma 1e-5) make the problem badly scaled: BFGS works on unknowns scaled to unit curvature
    scale = np.ones_like(x0)
    for c in range(2):
        scale[9 * c + 6:9 * c + 9] = ref.CAL_PRIOR_SIGMA
    res = minimize(lambda y: tuple(v * (scale if i else 1) for i, v in enumerate(fg(y * scale))), x0 / scale, jac=True,
                   method="BFGS", options=dict(gtol=1e-10, maxiter=20000))
    c_bfgs = res.fun
    cams, _ = unpack(torch.tensor(res.x * scale, dtype=T))
    assert abs(c_lm - c_bfgs) <= 1e-9 * c_bfgs, (c_lm, c_bfgs)
    for c in range(2):
        assert _angle(opt.R[c], cams[c][0].numpy()) < 1e-7


def test_reference_criteria_on_a_noise_free_scene():
    """tests/test_two_view_estimator.py's bundle-adjustment criteria on a synthetic stand-in for 5pointExample1.txt:
    all 5 tracks triangulate, rotation and translation direction within 1 degree, every correspondence kept."""
    s = mg.synthetic_scene(seed=31, n=5, noise_px=0.0, perturb_deg=0.5, n_unverified=0)
    r = ref._bundle_adjust_pair(s["uv1"], s["uv2"], s["verified"], s["cal1"], s["cal2"], s["R0"], s["t0"], 0.5, np.inf, 0.0, 100)
    assert r.ok and r.num_tracks == 5
    assert np.degrees(_angle(r.R, s["R_true"])) <= 1.0
    assert np.degrees(np.arccos(np.clip(r.t @ s["t_true"], -1, 1))) <= 1.0
    assert np.array_equal(r.rows, s["verified"])


def test_fixture_is_what_the_oracle_computes(golden_dir):
    """tests/golden/twoview_ba_scenes.npz is reproduced by the oracle (scenes regenerated from their seeds)."""
    z = np.load(golden_dir / "twoview_ba_scenes.npz")
    for name, kw in mg.SCENES.items():
        s = mg.synthetic_scene(**kw)
        assert np.array_equal(s["uv1"], z[f"{name}/uv1"]) and np.array_equal(s["verified"], z[f"{name}/verified"]), name
        r = mg.run_oracle(s)
        assert r.ok == bool(z[f"{name}/out_ok"]), name
        assert np.array_equal(r.rows, z[f"{name}/out_rows"]), name
        if r.ok:
            np.testing.assert_allclose(r.trace, z[f"{name}/out_trace"], rtol=1e-12, atol=1e-20, err_msg=name)


def test_lund_door_fixture_is_what_the_oracle_computes(golden_dir):
    """tests/golden/twoview_ba_lund_door.npz: the oracle's refinement of the stored verifier output, pair by pair."""
    kps, pairs, rows, cal = mg.lund_inputs()
    z = np.load(golden_dir / "twoview_ba_lund_door.npz")
    n = 0
    for p in pairs:
        key, m = f"{p[0]}_{p[1]}", rows[p]
        if not bool(z[f"{key}/ok"]):
            continue
        r = ref.refine_pair(kps[p[0]][m[:, 0]].astype(np.float64), kps[p[1]][m[:, 1]].astype(np.float64), z[f"{key}/verified"],
                            len(m), cal, cal, z[f"{key}/R0"], z[f"{key}/t0"])
        assert r.ok == bool(z[f"{key}/out_ok"]) and np.array_equal(r.rows, z[f"{key}/out_rows"]), key
        n += r.ok
    assert n >= 30


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    cxx = shutil.which("g++")
    assert cxx, "g++ is required"
    exe = tmp_path_factory.mktemp("tv") / "test_twoview_math"
    subprocess.run([cxx, "-O2", "-std=c++17", "-x", "c++", str(ROOT / "tests/cpp/test_twoview_math.cpp"), "-o", str(exe)], check=True)

    def run(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        return [np.array(line.split(), float) for line in out.strip().splitlines()]

    return run


def _f(a):
    return " ".join(repr(float(v)) for v in np.ravel(a))


def _cams(seed):
    s = mg.synthetic_scene(seed=seed, n=40, outlier_frac=0.1)
    K = [np.array([s["cal1"][0], 0, 0, s["cal1"][1], s["cal1"][2]]), np.array([s["cal2"][0], 0, 0, s["cal2"][1], s["cal2"][2]])]
    return s, [(np.eye(3), np.zeros(3), K[0]), (s["R0"].T, -s["R0"].T @ s["t0"], K[1])]


def test_shim_dlt_matches_the_oracle(shim):
    s, cams = _cams(41)
    P = [ref.projection_matrix(*c) for c in cams]
    rows = s["verified"]
    out = shim([f"dlt {_f(P[0])} {_f(P[1])} {_f(s['uv1'][i])} {_f(s['uv2'][i])}" for i in rows])
    for i, o in zip(rows, out):
        X = ref.dlt(P[0], P[1], s["uv1"][i], s["uv2"][i])
        assert o[0] == 1 and X is not None
        assert np.max(np.abs(o[1:] - X)) <= 1e-12 * np.linalg.norm(X)


def test_shim_jacobians_match_finite_differences(shim):
    """The device's projection Jacobians (pose by right perturbation through retract, f/k1/k2, point) against central
    differences of the oracle's projection, with distortion switched on."""
    g = np.random.default_rng(5)
    for _ in range(20):
        R = ref.so3_exp(g.normal(size=3) * 0.3)
        t = g.normal(size=3)
        cal = np.array([500 + 100 * g.random(), 1e-2 * g.normal(), 1e-3 * g.normal(), 320.0, 240.0])
        p = t + R @ np.array([g.uniform(-1, 1), g.uniform(-1, 1), g.uniform(4, 8)])
        o = shim([f"proj {_f(R)} {_f(t)} {_f(cal)} {_f(p)}"])[0]
        uv, Jc, Jp = o[1:3], o[3:21].reshape(2, 9), o[21:27].reshape(2, 3)
        np.testing.assert_allclose(uv, ref.project(R, t, cal, p)[0], rtol=1e-14)
        h = 1e-6
        for j in range(9):
            d = np.zeros(9)
            d[j] = h
            def at(dd):
                Rn, tn = ref.retract_pose(R, t, dd[:6])
                return ref.project(Rn, tn, np.concatenate([cal[:3] + dd[6:], cal[3:]]), p)[0]
            fd = (at(d) - at(-d)) / (2 * h)
            np.testing.assert_allclose(Jc[:, j], fd, rtol=1e-6, atol=1e-6 * max(1.0, np.abs(fd).max()))
        for j in range(3):
            d = np.zeros(3)
            d[j] = h
            fd = (ref.project(R, t, cal, p + d)[0] - ref.project(R, t, cal, p - d)[0]) / (2 * h)
            np.testing.assert_allclose(Jp[:, j], fd, rtol=1e-6, atol=1e-6 * max(1.0, np.abs(fd).max()))


def test_shim_triangulation_and_lie_maps_match_the_oracle(shim):
    """DLT + gtsam's LM point refinement + the checks (one LM per track, to 1e-10 relative), Pose3 retract and Logmap."""
    s, cams = _cams(43)
    lines = []
    for i in range(s["k"]):
        uv = np.concatenate([s["uv1"][i], s["uv2"][i]])
        lines.append(f"tri {_f(cams[0][0])} {_f(cams[0][1])} {_f(cams[0][2])} {_f(cams[1][0])} {_f(cams[1][1])} {_f(cams[1][2])} "
                     f"{_f(uv)} 100.0 0.0")
    out = shim(lines)
    n_ok = 0
    for i, o in enumerate(out):
        X = ref.triangulate(cams, s["uv1"][i], s["uv2"][i], 100.0, 0.0)
        assert (o[0] == 1) == (X is not None), i
        if X is not None:
            n_ok += 1
            assert np.max(np.abs(o[1:] - X)) <= 1e-10 * np.linalg.norm(X), i
    assert n_ok >= 30
    g = np.random.default_rng(9)
    for _ in range(10):
        R, t, d = ref.so3_exp(g.normal(size=3)), g.normal(size=3), g.normal(size=6) * 0.2
        o = shim([f"exp {_f(R)} {_f(t)} {_f(d)}", f"log {_f(R)} {_f(t)}"])
        Rn, tn = ref.retract_pose(R, t, d)
        np.testing.assert_allclose(o[0][:9], Rn.ravel(), atol=1e-14)
        np.testing.assert_allclose(o[0][9:], tn, atol=1e-13)
        np.testing.assert_allclose(o[1], ref.se3_log(R, t), atol=1e-12)
