"""Golden vectors of the two-way matcher: `python -m oracle.make_golden_twoway` (needs the reference checkout).

Runs the reference's unmodified `TwoWayMatcher` (gtsfm/frontend/matcher/twoway_matcher.py) with the same empty stand-ins
oracle/make_golden.py's retriever golden uses, asserts that oracle/twoway_ref.py reproduces it, and writes
tests/golden/twoway_<case>.npz with the inputs, the match rows and the cv2 distances, with and without the ratio test."""
from __future__ import annotations

import sys
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import twoway_ref  # noqa: E402

OUT = ROOT / "tests" / "golden"
REF = Path("/root/reference")


def reference_matcher(ratio):
    class _Stub(types.ModuleType):
        def __getattr__(self, n):
            if n.startswith("__"):
                raise AttributeError(n)
            return type(n, (), {"__init__": lambda self, *a, **k: None})

    for name in ("gtsam", "gtsam.noiseModel", "dask", "dask.distributed", "distributed", "matplotlib", "matplotlib.pyplot",
                 "gtsfm.evaluation.metrics"):
        sys.modules.setdefault(name, _Stub(name))
    if str(REF) not in sys.path:
        sys.path.insert(0, str(REF))
    from gtsfm.frontend.matcher.twoway_matcher import TwoWayMatcher

    return TwoWayMatcher(ratio_test_threshold=ratio)


def lund_gray(i):
    return np.load(OUT / "lund_door_images.npz")[f"gray_{i}"]


def cases():
    import cv2

    out = {}
    d = [np.load(REF / f"tests/data/set1_lund_door/features/descriptors_{i}.npy") for i in (0, 1)]
    assert all((x == np.round(x)).all() and x.min() >= 0 and x.max() <= 255 for x in d)
    out["lund_stored"] = (d[0].astype(np.uint8), d[1].astype(np.uint8), "float32")  # stored as uint8, cast back losslessly
    g1, g2 = lund_gray(1), lund_gray(2)
    for name, det, dt in (("sift", cv2.SIFT_create(nfeatures=3000), "float32"), ("kaze", cv2.KAZE_create(), "float32"),
                          ("orb", cv2.ORB_create(nfeatures=3000), "uint8")):
        _, a = det.detectAndCompute(g1, None)
        _, b = det.detectAndCompute(g2, None)
        if name == "kaze":  # float32 rows do not compress: keep the fixture small
            a, b = a[:1500], b[:1500]
        out[name] = (a, b, dt)
    out["dummy"] = (np.array([0.4865, 0.3752, 0.3077, 0.9188, 0.7837, 0.1083, 0.6822, 0.3764, 0.2288, 0.8018, 1.1], np.float32)[:, None],
                    np.array([0.9995, 0.3376, 0.9005, 0.5382, 0.3162, 0.7974, 0.1785, 0.3491, 0.8658, 0.2912], np.float32)[:, None],
                    "float32")
    return out


def main():
    import cv2

    for name, (a, b, dt) in cases().items():
        rec = {"desc0": a, "desc1": b, "dtype": np.array(dt), "cv2_version": np.array(cv2.__version__)}
        x, y = a.astype(dt), b.astype(dt)
        for tag, ratio in (("ratio", 0.8), ("noratio", None)):
            ref = reference_matcher(ratio).match(None, None, x, y, None, None)
            m, dist = twoway_ref.twoway_match(x, y, ratio)
            assert np.array_equal(ref, m) and ref.dtype == m.dtype, (name, tag)
            rec[f"matches_{tag}"] = m.reshape(-1, 2).astype(np.uint32)
            rec[f"dist_{tag}"] = dist
            print(name, tag, a.shape, b.shape, dt, len(dist))
        np.savez_compressed(OUT / f"twoway_{name}.npz", **rec)


if __name__ == "__main__":
    main()
