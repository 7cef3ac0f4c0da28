"""Restatement of gtsfm/frontend/detector_descriptor/sift.py (`SIFTDetectorDescriptor.detect_and_describe`) over cv2:
rgb_to_gray_cv, cv2.SIFT_create().detectAndCompute(gray, mask), Keypoints.get_top_k (np.argpartition).  Also cv2's Gaussian
pyramid built from cv2.resize / cv2.GaussianBlur calls (what csrc/sift.cu computes level by level) and the keypoint
correspondence the parity tests use."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

FIELDS = ("x", "y", "size", "angle", "response", "octave")
N_LAYERS, SIGMA = 3, 1.6


def rgb_to_gray_cv(arr: np.ndarray) -> np.ndarray:
    """gtsfm/utils/images.py:15-42."""
    import cv2

    if arr.ndim == 2:
        return arr
    if arr.shape[2] == 4:
        return cv2.cvtColor(arr, cv2.COLOR_RGBA2GRAY)
    if arr.shape[2] == 3:
        return cv2.cvtColor(arr, cv2.COLOR_RGB2GRAY)
    raise ValueError("Input image dimensions are wrong")


def cv2_sift(arr: np.ndarray, mask: Optional[np.ndarray] = None) -> Tuple[Dict[str, np.ndarray], Optional[np.ndarray]]:
    """Every keypoint cv2 returns, as field arrays (float32; octave int32), and its float32 descriptors (None when empty)."""
    import cv2

    kps, desc = cv2.SIFT_create().detectAndCompute(rgb_to_gray_cv(arr), mask)
    rec = {f: np.array([getattr(k, "pt")[0] if f == "x" else getattr(k, "pt")[1] if f == "y" else getattr(k, f) for k in kps],
                       np.int32 if f == "octave" else np.float32) for f in FIELDS}
    return rec, desc


def detect_and_describe(arr: np.ndarray, mask: Optional[np.ndarray] = None, max_keypoints: int = 5000):
    """The reference plugin: -> (coordinates float64, scales float64, responses float64, descriptors float32)."""
    rec, desc = cv2_sift(arr, mask)
    coords = np.stack([rec["x"], rec["y"]], 1).astype(np.float64)
    scales, resp = rec["size"].astype(np.float64), rec["response"].astype(np.float64)
    if max_keypoints >= len(coords):
        sel = np.arange(len(coords))
    else:
        sel = np.argpartition(-resp, max_keypoints)[:max_keypoints]  # gtsfm/common/keypoints.py get_top_k
    return coords[sel], scales[sel], resp[sel], desc[sel]


def n_octaves(h: int, w: int) -> int:
    return int(np.rint(np.log(2.0 * min(h, w)) / np.log(2.0) - 2)) + 1


def gaussian_pyramid(gray: np.ndarray) -> List[List[np.ndarray]]:
    """cv2's buildGaussianPyramid with createInitialImage (firstOctave -1, no precise upscale): octave lists of 6 float32
    levels."""
    import cv2

    base = cv2.resize(gray.astype(np.float32), (2 * gray.shape[1], 2 * gray.shape[0]), interpolation=cv2.INTER_LINEAR)
    sig0 = np.sqrt(max(SIGMA * SIGMA - 0.5 * 0.5 * 4, 0.01))
    base = cv2.GaussianBlur(base, (0, 0), sig0, sig0)
    k = 2.0 ** (1.0 / N_LAYERS)
    sig = [SIGMA] + [np.sqrt((k ** (i - 1) * SIGMA * k) ** 2 - (k ** (i - 1) * SIGMA) ** 2) for i in range(1, N_LAYERS + 3)]
    pyr = []
    for o in range(n_octaves(*gray.shape[:2])):
        if o == 0:
            levels = [base]
        else:
            src = pyr[o - 1][N_LAYERS]
            levels = [cv2.resize(src, (src.shape[1] // 2, src.shape[0] // 2), interpolation=cv2.INTER_NEAREST)]
        for i in range(1, N_LAYERS + 3):
            levels.append(cv2.GaussianBlur(levels[-1], (0, 0), sig[i], sig[i]))
        pyr.append(levels)
    return pyr


def correspond(a: Dict[str, np.ndarray], b: Dict[str, np.ndarray], tol_px: float = 0.01, tol_deg: float = 0.5,
               octave_bits: int = -1) -> Tuple[np.ndarray, np.ndarray]:
    """For every keypoint of `a`, the nearest keypoint of `b` within tol_px with the same packed octave (the bits of
    `octave_bits`; 0xffff leaves out the byte that quantises the sub-layer offset) and an angle within tol_deg (circular).
    -> (ia, ib) index arrays of the corresponded keypoints of `a` and their partners."""
    from scipy.spatial import cKDTree

    if len(a["x"]) == 0 or len(b["x"]) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    pa = np.stack([a["x"], a["y"]], 1).astype(np.float64)
    pb = np.stack([b["x"], b["y"]], 1).astype(np.float64)
    cand = cKDTree(pb).query_ball_point(pa, tol_px)
    ia, ib = [], []
    for i, js in enumerate(cand):
        best, bd = -1, np.inf
        for j in js:
            if (int(a["octave"][i]) ^ int(b["octave"][j])) & octave_bits:
                continue
            da = abs(float(a["angle"][i]) - float(b["angle"][j])) % 360.0
            if min(da, 360.0 - da) > tol_deg:
                continue
            d = np.hypot(*(pa[i] - pb[j]))
            if d < bd:
                best, bd = j, d
        if best >= 0:
            ia.append(i)
            ib.append(best)
    return np.array(ia, np.int64), np.array(ib, np.int64)


def parity(a: Dict[str, np.ndarray], da: np.ndarray, b: Dict[str, np.ndarray], db: np.ndarray, octave_bits: int = -1) -> Dict[str, float]:
    """The parity figures of `a` against `b`: corresponded shares in both directions, count ratio and the share of
    corresponded descriptor rows within +-1 element-wise."""
    ia, ib = correspond(a, b, octave_bits=octave_bits)
    jb, ja = correspond(b, a, octave_bits=octave_bits)
    na, nb = len(a["x"]), len(b["x"])
    rows = np.abs(da[ia].astype(np.int32) - db[ib].astype(np.int32)).max(1) <= 1 if len(ia) else np.zeros(0, bool)
    return {"a_in_b": len(ia) / max(na, 1), "b_in_a": len(jb) / max(nb, 1), "count_ratio": na / max(nb, 1),
            "desc_within_1": float(rows.mean()) if len(rows) else 1.0, "n_a": na, "n_b": nb}


CASES = ("lund_1", "lund_2", "lund_3", "lund_4", "lund_5", "lund_2_mask", "odd_crop", "tiny_crop", "synthetic_12mp", "lund_4_rgb",
         "lund_4_rgba", "empty_8", "empty_16", "flat")


def case_image(name: str, golden_dir) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    """The input (uint8 image, optional uint8 mask) of golden case `name`, rebuilt from tests/golden/lund_door_images.npz
    or from a seed."""
    from pathlib import Path

    lund = lambda i: np.load(Path(golden_dir) / "lund_door_images.npz")[f"gray_{i}"]  # noqa: E731  (1135 x 760)
    if name.startswith("lund_") and name[5:].isdigit():
        return lund(int(name[5:])), None
    if name == "lund_2_mask":
        g = lund(2)
        blocks = np.random.default_rng(7).integers(0, 2, (g.shape[0] // 32 + 1, g.shape[1] // 32 + 1), dtype=np.uint8)
        return g, np.ascontiguousarray(np.kron(blocks, np.ones((32, 32), np.uint8))[: g.shape[0], : g.shape[1]])
    if name == "odd_crop":
        return np.ascontiguousarray(lund(3)[301:818, 171:560]), None  # 517 x 389
    if name == "tiny_crop":
        return np.ascontiguousarray(lund(1)[60:100, 45:75]), None  # 40 x 30
    if name == "synthetic_12mp":
        from gtsfm_b200 import synthetic as syn

        return syn.synthetic_sequence(1, 2880, 3840)[0][0], None
    if name in ("lund_4_rgb", "lund_4_rgba"):
        g = lund(4)
        ch = [g, np.roll(g, 7, axis=1), (255 - g) // 2 + np.roll(g, -5, axis=0) // 2]
        if name.endswith("rgba"):
            ch.append(np.full_like(g, 200))
        return np.ascontiguousarray(np.stack(ch, 2)), None
    if name == "empty_8":
        return np.ascontiguousarray(lund(1)[500:508, 300:308]), None
    if name == "empty_16":
        return np.ascontiguousarray(lund(1)[100:116, 0:16]), None
    if name == "flat":
        return np.full((64, 64), 128, np.uint8), None
    raise KeyError(name)
