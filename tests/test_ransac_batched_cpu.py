"""Batched RANSAC verification, the parts that need no GPU: the ctypes mirrors of b2_ransac_problem / b2_ransac_result have
the header's layout, the sub-batch planner covers every problem once under the budget, and B200Ransac.verify_many's guards
return the failure tuple without touching a device."""
import ctypes
import pickle
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from gtsfm_b200 import _lib
from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
from gtsfm_b200.verifier import B200Ransac, pinhole_cal, ransac_problem

ROOT = Path(__file__).resolve().parent.parent

PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "gtsfm_b200.h"
#define F(T, f) printf(#T "." #f " %zu\n", offsetof(T, f))
int main(void) {
  printf("b2_ransac_problem %zu\nb2_ransac_result %zu\n", sizeof(b2_ransac_problem), sizeof(b2_ransac_result));
  F(b2_ransac_problem, kp1); F(b2_ransac_problem, kp2); F(b2_ransac_problem, matches); F(b2_ransac_problem, x1);
  F(b2_ransac_problem, x2); F(b2_ransac_problem, k); F(b2_ransac_problem, mode); F(b2_ransac_problem, max_iters);
  F(b2_ransac_problem, cal1); F(b2_ransac_problem, cal2); F(b2_ransac_problem, threshold); F(b2_ransac_problem, mask);
  F(b2_ransac_result, status); F(b2_ransac_result, num_inliers); F(b2_ransac_result, model); F(b2_ransac_result, R);
  F(b2_ransac_result, t);
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
    for name, cls in (("b2_ransac_problem", _lib.RansacProblem), ("b2_ransac_result", _lib.RansacResult)):
        got[name] = str(ctypes.sizeof(cls))
        for field, *_ in cls._fields_:
            got[f"{name}.{field}"] = str(getattr(cls, field).offset)
    assert got == want


def _lib_cpu():
    return _lib.load()  # loads and binds without a GPU; only b2_create needs one


def _problems(rng, n):
    out = []
    for _ in range(n):
        mode = int(rng.integers(0, 2))
        ready = bool(rng.integers(0, 2))
        out.append(ransac_problem(int(rng.integers(0, 6000)), mode, 1.0, 1000 if mode == 0 else 1000000, mask=8 if rng.integers(0, 2) else None,
                                  x1=8 if ready else None, x2=8 if ready else None, kp1=None if ready else 8, kp2=None if ready else 8,
                                  matches=None if ready else 8))
    return out


def test_workspace_bytes_follow_the_round_size():
    lib = _lib_cpu()
    size = lambda **kw: lib.b2_ransac_workspace_bytes(ctypes.byref(ransac_problem(**kw)))  # noqa: E731
    per_sample = 10 * (72 + 8 + 4) + 4
    e = size(k=2000, mode=0, threshold=1.0, max_iters=1000, mask=8, x1=8, x2=8)
    f = size(k=2000, mode=1, threshold=1.0, max_iters=1000000, mask=8, x1=8, x2=8)
    small = size(k=3, mode=0, threshold=1.0, max_iters=1000, mask=8, x1=8, x2=8)
    assert e - small == 4000 * per_sample  # the extension stage's 4 x 1000 samples, not 16 384
    assert f - small == 16384 * per_sample
    assert size(k=2000, mode=0, threshold=1.0, max_iters=1000, mask=8, kp1=8, kp2=8, matches=8) - e == 2000 * 32  # its points
    assert size(k=2000, mode=0, threshold=1.0, max_iters=1000, x1=8, x2=8) - e == 2000  # its mask
    assert e < 3.5e6 and f < 14e6 and small < 4096


@pytest.mark.parametrize("budget_mb", [1, 8, 64, 1024])
def test_planner_covers_every_problem_once_under_the_budget(budget_mb):
    lib = _lib_cpu()
    rng = np.random.default_rng(budget_mb)
    for n in (0, 1, 7, 100):
        probs = _problems(rng, n)
        arr = (_lib.RansacProblem * max(n, 1))(*probs)
        first = (ctypes.c_int * (n + 1))()
        count = lib.b2_ransac_plan(arr, n, budget_mb << 20, first)
        assert (count == 0) == (n == 0) and first[count] == n
        bounds = list(first[: count + 1])
        assert bounds[0] == 0 and all(a < b for a, b in zip(bounds, bounds[1:]))  # consecutive, non-empty, each problem once
        sizes = [lib.b2_ransac_workspace_bytes(ctypes.byref(p)) for p in probs]
        for a, b in zip(bounds, bounds[1:]):
            assert sum(sizes[a:b]) <= budget_mb << 20 or b - a == 1  # only a problem larger than the budget exceeds it, alone
            if b < n:
                assert sum(sizes[a:b + 1]) > budget_mb << 20  # greedy: the next problem did not fit
    bad = ransac_problem(10, 2, 1.0, 1000)
    assert lib.b2_ransac_plan(ctypes.byref(bad), 1, 1 << 30, (ctypes.c_int * 2)()) == -2  # B2_ERR_ARG


def test_verify_many_guards_need_no_device():
    rng = np.random.default_rng(0)
    kp = Keypoints(rng.uniform(0, 300, (50, 2)))
    cal = Cal3Bundler(200, 0, 0, 150, 150)
    rows = lambda n, dt: np.stack([np.arange(n), np.arange(n)], -1).astype(dt)  # noqa: E731
    for use_intrinsics, too_few in ((True, (0, 4, 5)), (False, (0, 5, 7))):
        ver = B200Ransac(use_intrinsics, 0.5)
        out = ver.verify_many([(kp, kp, rows(n, np.uint32), cal, cal) for n in too_few])
        assert len(out) == len(too_few) and ver._engine is None
        for R, t, r, ratio in out:
            assert R is None and t is None and r.size == 0 and ratio == 0.0
        assert ver.verify_many([]) == []
        assert pickle.loads(pickle.dumps(ver))._engine is None


def test_pinhole_cal_accepts_only_what_the_device_calibrates():
    assert pinhole_cal(Cal3Bundler(800, 0, 0, 640, 480)) == (800.0, 640.0, 480.0)
    assert pinhole_cal(Cal3Bundler(800, 1e-3, 0, 640, 480)) is None

    class TwoFocals:
        def px(self):
            return 0.0

        def K(self):
            return np.array([[800.0, 0, 0], [0, 810.0, 0], [0, 0, 1]])

    assert pinhole_cal(TwoFocals()) is None
