"""Writes tests/golden/lmeds_scenes.npz: seeded E and F scenes with cv2's LMeDS model and mask and cv2.recoverPose's pose on
that model, so the GPU test needs no cv2 of its own.  `python -m oracle.make_golden_lmeds` from the repository root."""
from pathlib import Path

import numpy as np

from oracle import lmeds_ref as lr
from oracle import verifier_ref as vr

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "lmeds_scenes.npz"


def main():
    import cv2

    rec = {}
    scenes = []
    for i, (seed, k, frac) in enumerate([(0, 400, 0.3), (1, 2000, 0.4), (2, 400, 0.5), (3, 50, 0.3), (4, 1500, 0.5), (5, 3000, 0.4)]):
        x1, x2 = lr.probe_scene(seed, k, frac)
        scenes.append((0, x1, x2, (1.0, 0.0, 0.0)))
    for i, (k, ratio) in enumerate([(300, 0.8), (1200, 0.6), (2500, 0.5), (5000, 0.7)]):
        kp1, kp2, _, K, _, _, _ = vr.synthetic_two_view(200 + i, k, ratio)
        scenes.append((1, kp1, kp2, K))
    for i, (mode, x1, x2, K) in enumerate(scenes):
        M, mask = lr.cv2_lmeds(x1, x2, mode)
        inl = mask == 1
        if mode == 0:
            E, n1, n2 = M, x1[inl], x2[inl]
        else:
            Km = np.array([[K[0], 0, K[1]], [0, K[0], K[2]], [0, 0, 1.0]])
            E, n1, n2 = Km.T @ M @ Km, vr.calibrate(x1[inl], *K), vr.calibrate(x2[inl], *K)
        _, R, t, _ = cv2.recoverPose(E, n1, n2)
        for name, v in dict(mode=mode, x1=x1, x2=x2, K=np.array(K), model=M, mask=mask, R=R, t=t.ravel()).items():
            rec[f"s{i}_{name}"] = np.asarray(v)
    rec["n"] = np.array(len(scenes))
    rec["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **rec)
    print(OUT, OUT.stat().st_size)


if __name__ == "__main__":
    main()
