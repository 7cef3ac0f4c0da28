"""Golden vectors of the ORB detector-descriptor: `python -m oracle.make_golden_orb` (needs the reference checkout).

Runs the reference's unmodified `ORBDetectorDescriptor` (gtsfm/frontend/detector_descriptor/orb.py) with the stand-ins of
oracle/make_golden_sift.py, asserts that oracle/orb_ref.py reproduces it, and writes tests/golden/orb_<case>.npz with every cv2
keypoint field in cv2's order, the uint8 descriptors and the cv2 version.  The inputs are rebuilt by orb_ref.case_image."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import make_golden_sift, orb_ref  # noqa: E402

OUT = ROOT / "tests" / "golden"


def reference_plugin():
    make_golden_sift.reference_plugin()  # installs the stand-in modules and the reference's path
    from gtsfm.common.image import Image
    from gtsfm.frontend.detector_descriptor.orb import ORBDetectorDescriptor

    return ORBDetectorDescriptor(max_keypoints=5000), Image


def main():
    import cv2

    plugin, Image = reference_plugin()
    for name in orb_ref.CASES:
        arr, mask = orb_ref.case_image(name, OUT)
        rec, desc = orb_ref.cv2_orb(arr, mask)
        n = len(rec["x"])
        if n == 0:
            try:
                plugin.detect_and_describe(Image(arr, mask=mask))
                raise AssertionError(f"{name}: the reference returned on an image without keypoints")
            except TypeError:
                pass  # None[idx]: the reference's behaviour the plugin replaces by an empty result
            desc = np.zeros((0, 32), np.uint8)
        else:
            kp, ref_desc = plugin.detect_and_describe(Image(arr, mask=mask))
            c, s, r, d = orb_ref.detect_and_describe(arr, mask)
            assert np.array_equal(kp.coordinates, c) and np.array_equal(kp.scales, s) and np.array_equal(kp.responses, r), name
            assert np.array_equal(ref_desc, d), name
        out = {f: rec[f] for f in orb_ref.FIELDS}
        out.update(desc=desc, cv2_version=np.array(cv2.__version__), shape=np.array(arr.shape))
        np.savez_compressed(OUT / f"orb_{name}.npz", **out)
        print(name, arr.shape, n, flush=True)


if __name__ == "__main__":
    main()
