"""CPU suite for the LMedS verifier: oracle/lmeds_ref.py (the NumPy restatement of cv2's LMeDS that the device kernels are
replayed against) pinned to cv2 itself, the complete-root 5-point solver and the 7-point solver of ransac_math.cuh
(host build), the ctypes mirrors and the sub-batch planner."""
import ctypes
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from gtsfm_b200 import _lib
from gtsfm_b200.verifier import lmeds_params, ransac_problem
from oracle import lmeds_ref as lr
from oracle import verifier_ref as vr

cv2 = pytest.importorskip("cv2")
ROOT = Path(__file__).resolve().parent.parent
TIE_ULPS = 4  # a scene whose two lowest medians are this close may pick either model


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return lr.build_shim(tmp_path_factory.mktemp("lmeds_shim"))


def _scenes():
    """(name, mode, x1, x2): E scenes on calibrated points, F scenes on pixels; at least 60 in all."""
    out = []
    for seed in range(12):  # the generator of the 5-point probe: 30-50 % outliers, k = 50 / 400 / 2000
        for k in (50, 400, 2000):
            x1, x2 = lr.probe_scene(seed, k, (0.3, 0.4, 0.5)[seed % 3])
            out.append((f"probe{seed}_{k}", 0, x1, x2))
    ratios = (0.2, 0.35, 0.5, 0.65, 0.8, 0.9)
    for i, (k, ratio) in enumerate([(k, r) for k in (60, 700, 5000) for r in ratios[::2 if k == 5000 else 1]]):
        kp1, kp2, _, K, _, _, _ = vr.synthetic_two_view(100 + i, k, ratio)
        out.append((f"synF{i}_{k}_{ratio}", 1, kp1, kp2))
        out.append((f"synE{i}_{k}_{ratio}", 0, vr.calibrate(kp1, *K), vr.calibrate(kp2, *K)))
    # near-degenerate: one more point than the minimal sample, duplicated points, a third of the points on one line
    kp1, kp2, _, K, _, _, _ = vr.synthetic_two_view(7, 8, 0.9)
    out.append(("F_k8", 1, kp1, kp2))
    out.append(("E_k6", 0, vr.calibrate(kp1[:6], *K), vr.calibrate(kp2[:6], *K)))
    kp1, kp2, _, K, _, _, _ = vr.synthetic_two_view(8, 300, 0.7)
    d1, d2 = np.concatenate([kp1, kp1[:150]]), np.concatenate([kp2, kp2[:150]])
    out.append(("F_dup", 1, d1, d2))
    out.append(("E_dup", 0, vr.calibrate(d1, *K), vr.calibrate(d2, *K)))
    c1, c2 = kp1.copy(), kp2.copy()
    c1[:100] = np.array([200.0, 300.0]) + np.arange(100)[:, None] * [6.0, 2.0]  # exactly collinear in float32
    out.append(("F_collinear", 1, c1, c2))
    for seed in range(4):  # half of image 1's points within 1e-5 .. 1e-2 px of one line: subsets near the FLT_EPSILON test
        kp1, kp2, _, _, _, _, _ = vr.synthetic_two_view(500 + seed, 60, 0.8)
        rng = np.random.default_rng(seed)
        t = rng.integers(0, 200, 30)
        kp1 = kp1.copy()
        kp1[:30] = np.stack([100 + 3.0 * t, 50 + 7.0 * t], -1) + rng.normal(size=(30, 2)) * 10 ** rng.uniform(-5, -2)
        out.append((f"F_near_line{seed}", 1, kp1, kp2))
    return out


SCENES = _scenes()


def test_enough_scenes():
    assert len(SCENES) >= 60


def test_iteration_counts():
    """RANSACUpdateNumIters(conf, 0.45, m, 1000), at least 3: E 134 at 0.999, F 300 at 0.99."""
    assert lr.niters(0.999, 5) == 134 and lr.niters(0.99, 7) == 300
    assert lr.niters(0.5, 5) == 13 and lr.niters(1e-9, 7) == 3 and lr.niters(0.999999, 7, 200) == 200


def test_shim_matches_oracle_sampler_iterations_and_errors(shim):
    """The host build of the device's sampler, iteration count and float errors equals the oracle exactly."""
    for conf, m, mi in ((0.999, 5, 1000), (0.99, 7, 1000), (0.5, 5, 1000), (0.999999, 7, 200)):
        assert shim.lm_niters(conf, m, mi) == lr.niters(conf, m, mi)
    for name, mode, x1, x2 in SCENES[::5] + [s for s in SCENES if s[0] in ("F_collinear", "F_dup", "F_k8")]:
        x1 = np.ascontiguousarray(x1, np.float64)
        x2 = np.ascontiguousarray(x2, np.float64)
        n = lr.niters(lr.E_CONFIDENCE if mode == 0 else lr.F_CONFIDENCE, 5 if mode == 0 else 7)
        m = 5 if mode == 0 else 7
        ref = lr.subsets(x1.astype(np.float32).astype(np.float64) if mode else x1, x2.astype(np.float32).astype(np.float64) if mode else x2, mode, n)
        got = np.zeros((n, m), np.int32)
        drawn = shim.lm_subsets(_p(x1), _p(x2), len(x1), mode, n, _p(got))
        assert drawn == len(ref) and np.array_equal(got[:drawn], ref), name
        M = np.random.default_rng(0).normal(size=9)
        xe1, xe2 = (x1, x2) if mode == 0 else (x1.astype(np.float32).astype(np.float64), x2.astype(np.float32).astype(np.float64))
        e = np.zeros(len(x1), np.float32)
        shim.lm_errors(mode, _p(M), _p(np.ascontiguousarray(xe1)), _p(np.ascontiguousarray(xe2)), len(x1), _p(e))
        assert np.array_equal(e.view(np.int32), lr.errors(mode, M, xe1, xe2).view(np.int32)), name


def test_collinear_subsets_are_redrawn():
    """F: a subset whose last point lies on a line through two earlier ones (in either image) is drawn again."""
    name, mode, x1, x2 = next(s for s in SCENES if s[0] == "F_collinear")
    idx = lr.subsets(x1.astype(np.float32).astype(np.float64), x2.astype(np.float32).astype(np.float64), 1, 300)
    on_line = np.arange(len(x1)) < 100
    assert all(not (on_line[s[-1]] and on_line[s[:-1]].sum() >= 2) for s in idx)
    rng = lr.CvRNG()  # without the check the same stream would have produced such a subset
    assert any(on_line[[rng.uniform(len(x1)) for _ in range(7)]].sum() >= 3 for _ in range(300))


def test_oracle_equals_cv2(shim):
    """On every scene: cv2's inlier mask bit for bit and its model to round-off of the minimal solver (up to sign)."""
    solve = lr.shim_solver(shim)
    ties, loose, worst, roundoff = 0, [], 0.0, []
    for name, mode, x1, x2 in SCENES:
        o = lr.lmeds(x1, x2, mode, solve)
        M, mask = lr.cv2_lmeds(x1, x2, mode)
        meds = np.sort(o["medians"][np.isfinite(o["medians"])].ravel())
        tie = len(meds) > 1 and int(meds[1:2].view(np.int32)[0]) - int(meds[:1].view(np.int32)[0]) <= TIE_ULPS
        ties += tie
        if tie:
            continue
        if len(meds) and meds[0] < 1e-20:
            # k = m + 1: most subsets fit k - 1 points exactly, every such model has a median at round-off level, and which
            # one is lowest depends on the solver's last bits.  Both pick an exact fit of all but at most one point.
            roundoff.append(name)
            assert o["count"] >= len(x1) - 1 - (mode == 1) and int(mask.sum()) >= len(x1) - 1 - (mode == 1), name
            continue
        assert np.array_equal(o["mask"], mask), name
        assert (M is None) == (not o["ok"]), name
        if M is not None:
            a, b = o["model"] / np.linalg.norm(o["model"]), M / np.linalg.norm(M)
            rel = min(np.abs(a - b).max(), np.abs(a + b).max())
            worst = max(worst, rel)
            if rel > 1e-9:
                loose.append((name, rel))
    print(f"\nLMedS oracle vs cv2: {len(SCENES)} scenes, {ties} within {TIE_ULPS} ulps of a median tie, "
          f"{len(loose)} models beyond 1e-9 relative (worst {worst:.2e}): {loose}; round-off medians: {roundoff}")
    assert ties == 0 and len(roundoff) <= 2
    # The 5-point solvers differ (null-space basis, polynomial, root polishing): on ill-conditioned 5-samples the same
    # root differs beyond 1e-9 while the float medians and the mask still agree.
    assert worst < 1e-6 and len(loose) <= 4


def test_probe_scene_needs_every_root(shim):
    """Probe scene seed 3, k = 400, 30 % outliers: cv2's E is a solution of subset 14, which has 4 real solutions.  The
    RANSAC verifier's sign-change bracketing (161 samples) finds 2 of them and not cv2's; the complete-root solver finds
    all 4, cv2's among them, and the restatement's mask is cv2's."""
    x1, x2 = lr.probe_scene(3, 400, 0.3)
    M, mask = lr.cv2_lmeds(x1, x2, 0)
    sub = lr.subsets(x1, x2, 0, 134)[14]
    a, b = np.ascontiguousarray(x1[sub]), np.ascontiguousarray(x2[sub])
    out_all, out_s = np.zeros((10, 9)), np.zeros((10, 9))
    n_all = shim.lm_solve(0, _p(a), _p(b), _p(out_all))
    n_s = shim.lm_fivept_sampled(_p(a), _p(b), _p(out_s))
    Mn = M.ravel() / np.linalg.norm(M)
    dist = lambda E: min(np.abs(E - Mn).max(), np.abs(E + Mn).max())  # noqa: E731
    assert n_all == 4 and n_s == 2
    assert min(dist(E) for E in out_all[:n_all]) < 1e-9
    assert min(dist(E) for E in out_s[:n_s]) > 1e-3
    o = lr.lmeds(x1, x2, 0, lr.shim_solver(shim))
    assert o["slot"] // lr.MAX_SOL == 14 and np.array_equal(o["mask"], mask)


def test_fivept_root_count_equals_companion_matrix(shim):
    """10^4 random 5-samples of probe scenes: the complete-root finder returns as many real roots of the 5-point
    polynomial as numpy's companion-matrix eigenvalues with |imag| <= 1e-8 max(1, |z|)."""
    rng = np.random.default_rng(3)
    bad = total = 0
    for sc in range(20):
        x1, x2 = lr.probe_scene(100 + sc, 200, 0.4)
        for _ in range(500):
            sub = rng.choice(200, 5, replace=False)
            a, b = np.ascontiguousarray(x1[sub]), np.ascontiguousarray(x2[sub])
            poly = np.zeros(11)
            shim.lm_fivept_poly(_p(a), _p(b), _p(poly))
            if not np.any(poly):
                continue
            out = np.zeros(10)
            n = shim.lm_poly_roots(_p(poly), 10, _p(out))
            ev = np.roots(poly[::-1])
            total += 1
            bad += n != int(np.sum(np.abs(ev.imag) <= 1e-8 * np.maximum(1, np.abs(ev))))
    assert total >= 9900 and bad == 0


def test_all_real_roots_found(shim):
    """10^4 random degree-10 polynomials with 0-8 real roots (one pair 1e-3 apart when there are two or more, the rest
    at least 0.2 apart) and complex pairs: the root finder returns every real root, each within 1e-7."""
    rng = np.random.default_rng(11)
    bad = 0
    for trial in range(10000):
        nreal = int(rng.integers(0, 5)) * 2
        r = np.sort(rng.choice(np.arange(-15, 16) * 0.2, nreal, replace=False) + rng.uniform(-0.05, 0.05, nreal))
        if nreal >= 2:
            r[1] = r[0] + 1e-3
        coef = np.array([1.0])
        for x in r:
            coef = np.convolve(coef, [1.0, -x])
        for _ in range((10 - nreal) // 2):
            re, im = rng.uniform(-3, 3), rng.uniform(0.3, 2)
            coef = np.convolve(coef, [1.0, -2 * re, re * re + im * im])
        coef *= rng.uniform(0.1, 10)
        out = np.zeros(10)
        n = shim.lm_poly_roots(_p(np.ascontiguousarray(coef[::-1])), 10, _p(out))
        if n != nreal or (n and np.abs(np.sort(out[:n]) - np.sort(r)).max() > 1e-7):
            bad += 1
    assert bad == 0


def test_sevenpt_solutions_satisfy_the_constraints(shim):
    rng = np.random.default_rng(5)
    for _ in range(200):
        kp1, kp2, _, _, _, _, _ = vr.synthetic_two_view(int(rng.integers(1 << 30)), 7, 1.0)
        a, b = np.ascontiguousarray(kp1.astype(np.float32), np.float64), np.ascontiguousarray(kp2.astype(np.float32), np.float64)
        out = np.zeros((10, 9))
        n = shim.lm_solve(1, _p(a), _p(b), _p(out))
        assert n in (1, 2, 3)
        for F in out[:n].reshape(-1, 3, 3):
            assert abs(F[2, 2] - 1) < 1e-12
            h1, h2 = np.c_[a, np.ones(7)], np.c_[b, np.ones(7)]
            Fn = F / np.linalg.norm(F)
            assert np.abs(np.einsum("ki,ij,kj->k", h2, Fn, h1)).max() < 1e-8 * np.abs(h2).max() * np.abs(h1).max()
            assert abs(np.linalg.det(Fn)) < 1e-9


PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "gtsfm_b200.h"
#define F(T, f) printf(#T "." #f " %zu\n", offsetof(T, f))
int main(void) {
  printf("b2_lmeds_params %zu\nb2_lmeds_trace %zu\n", sizeof(b2_lmeds_params), sizeof(b2_lmeds_trace));
  F(b2_lmeds_params, confidence);
  F(b2_lmeds_trace, cap); F(b2_lmeds_trace, idx); F(b2_lmeds_trace, nsol); F(b2_lmeds_trace, models);
  F(b2_lmeds_trace, medians); F(b2_lmeds_trace, niters); F(b2_lmeds_trace, drawn); F(b2_lmeds_trace, slot);
  F(b2_lmeds_trace, min_median); F(b2_lmeds_trace, sigma); F(b2_lmeds_trace, thr); F(b2_lmeds_trace, count);
  return 0;
}
"""


def test_ctypes_mirrors_have_the_headers_layout(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    assert cc, "a host C compiler is needed to read the header's layout"
    (tmp_path / "probe.c").write_text(PROBE)
    subprocess.run([cc, "-I", str(ROOT / "include"), "-x", "c", str(tmp_path / "probe.c"), "-o", str(tmp_path / "probe")], check=True)
    want = dict(line.rsplit(" ", 1) for line in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True,
                                                              text=True).stdout.strip().splitlines())
    got = {}
    for name, cls in (("b2_lmeds_params", _lib.LmedsParams), ("b2_lmeds_trace", _lib.LmedsTrace)):
        got[name] = str(ctypes.sizeof(cls))
        for field, *_ in cls._fields_:
            got[f"{name}.{field}"] = str(getattr(cls, field).offset)
    assert got == want


def test_workspace_and_plan():
    """Workspace follows the iteration count (134 E / 300 F subsets at the defaults); the plan covers every problem once,
    in order, and a sub-batch exceeds the budget only when it holds one problem."""
    lib = _lib.load()
    prm = lmeds_params()
    size = lambda **kw: lib.b2_lmeds_workspace_bytes(ctypes.byref(ransac_problem(**kw)), ctypes.byref(prm))  # noqa: E731
    per = 7 * 4 + 4 + 10 * (72 + 4)
    small = size(k=3, mode=0, threshold=0.0, max_iters=1000, mask=8, x1=8, x2=8)
    assert size(k=2000, mode=0, threshold=0.0, max_iters=1000, mask=8, x1=8, x2=8) - small == 134 * per
    assert size(k=2000, mode=1, threshold=0.0, max_iters=1000, mask=8, x1=8, x2=8) - small == 300 * per
    assert size(k=2000, mode=0, threshold=0.0, max_iters=1000, mask=8, kp1=8, kp2=8, matches=8) - small == 134 * per + 2000 * 32
    rng = np.random.default_rng(3)
    probs = [ransac_problem(int(rng.integers(0, 6000)), int(rng.integers(0, 2)), 0.0, 1000, x1=8, x2=8) for _ in range(200)]
    arr = (_lib.RansacProblem * 200)(*probs)
    sizes = [lib.b2_lmeds_workspace_bytes(ctypes.byref(p), ctypes.byref(prm)) for p in probs]
    for budget in (1 << 16, 1 << 20, 1 << 30):
        first = (ctypes.c_int * 201)()
        cnt = lib.b2_lmeds_plan(arr, 200, ctypes.byref(prm), budget, first)
        f = list(first)[:cnt + 1]
        assert f[0] == 0 and f[-1] == 200 and all(a < b for a, b in zip(f, f[1:]))
        for a, b in zip(f, f[1:]):
            assert b - a == 1 or sum(sizes[a:b]) <= budget
    assert lib.b2_lmeds_plan(arr, 200, None, 1 << 20, first) != 0
