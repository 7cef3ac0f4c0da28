"""Golden vectors of the D2-Net detector-descriptor: `python -m oracle.make_golden_d2net` (needs the reference checkout).

Runs the reference's unmodified `D2NetDetDesc` (gtsfm/frontend/detector_descriptor/d2net.py, use_cuda=False) with the stand-ins
oracle/make_golden_sift.py uses and a seeded checkpoint saved as {"model": state dict}, asserts that oracle/d2net_ref.py
reproduces it exactly, runs the restatement in float64 for the fp32-vs-fp64 spread of each case, and writes
tests/golden/d2net_<case>.npz (every case, or the cases named on the command line).  The inputs are rebuilt by d2net_ref.case_image; the large frames keep the first 300 descriptors."""
from __future__ import annotations

import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from gtsfm_b200 import synthetic as syn  # noqa: E402
from oracle import d2net_ref  # noqa: E402
from oracle.make_golden_sift import REF, reference_plugin  # noqa: E402,F401

OUT = ROOT / "tests" / "golden"
SEED = 7
MAX_KEYPOINTS = 5000
KEEP_DESC = 300


def _spread(a32, a64):
    """Largest fp32-vs-fp64 difference over the keypoints both runs found at the same (c, i, j)."""
    k64 = {tuple(c): n for n, c in enumerate(a64["cij"])}
    pairs = [(n, k64[tuple(c)]) for n, c in enumerate(a32["cij"]) if tuple(c) in k64]
    i32, i64 = (np.array([p[q] for p in pairs], np.int64) for q in (0, 1))
    d = np.abs(a32["desc"][i32] - a64["desc"][i64]).max()
    s = (np.abs(a32["scores"][i32] - a64["scores"][i64]) / np.abs(a64["scores"][i64])).max()
    p = np.abs(a32["xy"][i32] - a64["xy"][i64]).max()
    same = len(pairs) == len(a32["cij"]) == len(a64["cij"])
    return float(d), float(s), float(p), same


def main():
    import torch

    reference_plugin()  # installs the stand-in modules and the reference on sys.path
    from gtsfm.common.image import Image
    from gtsfm.frontend.detector_descriptor.d2net import D2NetDetDesc

    sd = syn.d2net_state_dict(SEED)
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(tmp) / "d2_tf.pth"
        torch.save({"model": {k: torch.from_numpy(v) for k, v in sd.items()}}, str(path))
        plugin = D2NetDetDesc(max_keypoints=MAX_KEYPOINTS, model_path=path, use_cuda=False)
    for name in sys.argv[1:] or d2net_ref.CASES:
        arr = d2net_ref.case_image(name, OUT)
        k = d2net_ref.CASE_MAX_KEYPOINTS.get(name, MAX_KEYPOINTS)
        plugin.max_keypoints = k
        ours = d2net_ref.detect_and_describe(arr, sd, k)
        o64 = d2net_ref.detect_and_describe(arr, sd, k, dtype=torch.float64)
        try:
            kp, desc = plugin.detect_and_describe(Image(arr))
            xy, sc = np.asarray(kp.coordinates), np.asarray(kp.responses)
        except (IndexError, RuntimeError):  # nothing detected: the reference fails on its empty arrays
            xy, sc, desc = np.zeros((0, 2), np.float32), np.zeros(0, np.float32), np.zeros((0, 512), np.float32)
        n = len(ours["scores"])
        assert len(sc) == n, (name, len(sc), n)
        if n:
            # the reference's np.argsort is unstable on ties: within a run of equal scores compare the rows as a set
            assert np.array_equal(sc, ours["scores"]), name
            o_ref = np.lexsort((xy[:, 1], xy[:, 0], -sc.astype(np.float64)))
            o_our = np.lexsort((ours["xy"][:, 1], ours["xy"][:, 0], -ours["scores"].astype(np.float64)))
            assert np.array_equal(xy[o_ref], ours["xy"][o_our]) and np.array_equal(desc[o_ref], ours["desc"][o_our]), name
            d, s, p, same = _spread(ours, o64)
        else:
            d, s, p, same = 0.0, 0.0, 0.0, len(o64["scores"]) == 0
        keep = n if n <= 2 * KEEP_DESC else KEEP_DESC
        np.savez_compressed(OUT / f"d2net_{name}.npz", shape=np.array(arr.shape), xy=ours["xy"].astype(np.float32),
                            scores=ours["scores"].astype(np.float32), desc=ours["desc"][:keep].astype(np.float32), cij=ours["cij"],
                            margin=ours["margin"], total=ours["total"], byte_sum=np.int64(arr.astype(np.int64).sum()),
                            spread_desc=d, spread_score_rel=s, spread_xy=p, fp64_same_set=same, seed=SEED,
                            max_keypoints=k, torch_version=np.array(torch.__version__))
        print(f"{name} {arr.shape} keypoints {n} (total {int(ours['total'])}) spread desc {d:.2e} score {s:.2e} xy {p:.2e} "
              f"same set in fp64: {same}", flush=True)


if __name__ == "__main__":
    main()
