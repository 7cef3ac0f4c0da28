"""Golden vectors of the SIFT detector-descriptor: `python -m oracle.make_golden_sift` (needs the reference checkout).

Runs the reference's unmodified `SIFTDetectorDescriptor` (gtsfm/frontend/detector_descriptor/sift.py) with the stand-ins
oracle/make_golden_twoway.py uses, asserts that oracle/sift_ref.py reproduces it, and writes tests/golden/sift_<case>.npz with
every cv2 keypoint field, the uint8 descriptors and the cv2 version.  The inputs are rebuilt by sift_ref.case_image."""
from __future__ import annotations

import sys
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import sift_ref  # noqa: E402

OUT = ROOT / "tests" / "golden"
REF = Path("/root/reference")


def reference_plugin():
    class _Meta(type):  # stand-in classes whose attributes are stand-in classes (gtsam.noiseModel.Diagonal annotations)
        def __getattr__(cls, n):
            if n.startswith("__"):
                raise AttributeError(n)
            return _Meta(n, (), {"__init__": lambda self, *a, **k: None})

    class _Stub(types.ModuleType):
        def __getattr__(self, n):
            if n.startswith("__"):
                raise AttributeError(n)
            return _Meta(n, (), {"__init__": lambda self, *a, **k: None})

    for name in ("gtsam", "gtsam.noiseModel", "dask", "dask.distributed", "distributed", "matplotlib", "matplotlib.pyplot",
                 "gtsfm.evaluation.metrics"):
        sys.modules.setdefault(name, _Stub(name))
    if str(REF) not in sys.path:
        sys.path.insert(0, str(REF))
    from gtsfm.common.image import Image
    from gtsfm.frontend.detector_descriptor.sift import SIFTDetectorDescriptor

    return SIFTDetectorDescriptor(max_keypoints=5000), Image


def main():
    import cv2

    plugin, Image = reference_plugin()
    for name in sift_ref.CASES:
        arr, mask = sift_ref.case_image(name, OUT)
        rec, desc = sift_ref.cv2_sift(arr, mask)
        n = len(rec["x"])
        if n == 0:
            try:
                plugin.detect_and_describe(Image(arr, mask=mask))
                raise AssertionError(f"{name}: the reference returned on an image without keypoints")
            except TypeError:
                pass  # None[idx]: the reference's behaviour the plugin replaces by an empty result
            desc = np.zeros((0, 128), np.float32)
        else:
            kp, ref_desc = plugin.detect_and_describe(Image(arr, mask=mask))
            c, s, r, d = sift_ref.detect_and_describe(arr, mask)
            assert np.array_equal(kp.coordinates, c) and np.array_equal(kp.scales, s) and np.array_equal(kp.responses, r), name
            assert np.array_equal(ref_desc, d), name
            assert np.array_equal(desc, np.round(desc)) and desc.min() >= 0 and desc.max() <= 255
        out = {f: rec[f] for f in sift_ref.FIELDS}
        out.update(desc=desc.astype(np.uint8), cv2_version=np.array(cv2.__version__), shape=np.array(arr.shape))
        np.savez_compressed(OUT / f"sift_{name}.npz", **out)
        print(name, arr.shape, n, flush=True)


if __name__ == "__main__":
    main()
