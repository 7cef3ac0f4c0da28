"""Restatement of gtsfm/frontend/detector_descriptor/orb.py (`ORBDetectorDescriptor.detect_and_describe`) over cv2:
rgb_to_gray_cv, cv2.ORB_create().detectAndCompute(gray, mask), Keypoints.get_top_k (np.argpartition).

Also a stage-by-stage NumPy restatement of cv2's ORB with its defaults (nfeatures 500, scaleFactor 1.2, nlevels 8,
edgeThreshold 31, firstLevel 0, WTA_K 2, HARRIS_SCORE, patchSize 31, fastThreshold 20) that equals cv2 bit for bit
(tests/test_orb_cpu.py), and what csrc/orb.cu computes stage by stage:

  pyramid   level l = cv2.resize(level l - 1, (cvRound(W / s_l), cvRound(H / s_l)), INTER_LINEAR_EXACT), s_l = (float)1.2f^l
  FAST      9/16 corner score, threshold 20, strict 3 x 3 non-maximum suppression, then the level mask, then the border
            filter (31 <= x < w - 31, 31 <= y < h - 31)
  select 1  retainBest(2 n_l) by FAST score: everything >= the (2 n_l)-th largest score
  Harris    block 7, k 0.04, integer gradient sums, one float formula
  select 2  retainBest(n_l) by Harris response
  angle     intensity centroid over the radius-15 disc, fastAtan2(m01, m10)
  blur      GaussianBlur(7 x 7, sigma 2) of each level as ORB runs it: on a sub-matrix, so cv2's separable float filter
            (row pass, then column pass with symmetric pairs, each a chain of fused multiply-adds), not its fixed-point path
  describe  rBRIEF: 256 comparisons of rotated pattern points (orb_pattern.inc) on the blurred level
"""
from __future__ import annotations

import ctypes
import ctypes.util
from pathlib import Path
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle.sift_ref import rgb_to_gray_cv

FIELDS = ("x", "y", "size", "angle", "response", "octave")
N_FEATURES, N_LEVELS, EDGE, PATCH, FAST_T, HARRIS_K, HARRIS_BLOCK = 500, 8, 31, 31, 20, np.float32(0.04), 7
F32 = np.float32
SCALE = float(F32(1.2))  # ORB_create's scaleFactor is a float, widened to double where ORB computes with it
PATTERN_INC = Path(__file__).resolve().parent.parent / "gtsfm_b200" / "csrc" / "orb_pattern.inc"

# FAST's 16-pixel Bresenham circle of radius 3 (dx, dy), in circle order
CIRCLE = ((0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3),
          (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3))


# ---------------------------------------------------------------------------------------------------------------------
# the reference plugin over cv2
# ---------------------------------------------------------------------------------------------------------------------
def cv2_orb(arr: np.ndarray, mask: Optional[np.ndarray] = None) -> Tuple[Dict[str, np.ndarray], Optional[np.ndarray]]:
    """Every keypoint cv2 returns, as field arrays in cv2's order (float32; octave int32), and its uint8 descriptors (None
    when empty)."""
    import cv2

    kps, desc = cv2.ORB_create().detectAndCompute(rgb_to_gray_cv(arr), mask)
    rec = {f: np.array([k.pt[0] if f == "x" else k.pt[1] if f == "y" else getattr(k, f) for k in kps],
                       np.int32 if f == "octave" else np.float32) for f in FIELDS}
    return rec, desc


def detect_and_describe(arr: np.ndarray, mask: Optional[np.ndarray] = None, max_keypoints: int = 5000):
    """The reference plugin: -> (coordinates float64, scales float64, responses float64, descriptors uint8).  An image
    without keypoints gives empty arrays (the reference raises there)."""
    rec, desc = cv2_orb(arr, mask)
    if desc is None:
        return np.zeros((0, 2)), np.zeros(0), np.zeros(0), np.zeros((0, 32), np.uint8)
    coords = np.stack([rec["x"], rec["y"]], 1).astype(np.float64)
    scales, resp = rec["size"].astype(np.float64), rec["response"].astype(np.float64)
    if max_keypoints >= len(coords):
        sel = np.arange(len(coords))
    else:
        sel = np.argpartition(-resp, max_keypoints)[:max_keypoints]  # gtsfm/common/keypoints.py get_top_k
    return coords[sel], scales[sel], resp[sel], desc[sel]


# ---------------------------------------------------------------------------------------------------------------------
# stages
# ---------------------------------------------------------------------------------------------------------------------
def level_scales() -> np.ndarray:
    """layerScale: (float)pow(scaleFactor, l)."""
    return np.array([F32(SCALE ** l) for l in range(N_LEVELS)], F32)


def level_sizes(h: int, w: int) -> List[Tuple[int, int]]:
    """(height, width) of every level: cvRound(side / s_l) in float."""
    return [(int(np.rint(F32(h) / s)), int(np.rint(F32(w) / s))) for s in level_scales()]


def features_per_level() -> List[int]:
    """nfeaturesPerLevel: cvRound of the float geometric share, the last level takes the remainder."""
    factor = F32(1.0 / SCALE)
    share = F32(F32(N_FEATURES * (F32(1) - factor)) / F32(1 - F32(float(factor) ** N_LEVELS)))
    out, tot = [], 0
    for _ in range(N_LEVELS - 1):
        out.append(int(np.rint(share)))
        tot += out[-1]
        share = F32(share * factor)
    out.append(max(N_FEATURES - tot, 0))
    return out


def _linear_taps(src: int, dst: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """INTER_LINEAR_EXACT taps along one axis: (offset, Q8 weight of src[offset], Q8 weight of src[offset + 1])."""
    scale = 1.0 / (dst / src)  # softdouble(1) / inv_scale, both in double
    ofs, c0, c1 = np.zeros(dst, np.int64), np.full(dst, 256, np.int64), np.zeros(dst, np.int64)
    for d in range(dst):
        f = scale * (d + 0.5) - 0.5
        i = int(np.floor(f))
        if i < 0 or src == 1:
            ofs[d] = 0
        elif i < src - 1:
            ofs[d] = i
            c1[d] = int(np.rint((f - i) * 256))
            c0[d] = 256 - c1[d]
        else:
            ofs[d] = src - 1
    return ofs, c0, c1


def resize_linear_exact(img: np.ndarray, h: int, w: int) -> np.ndarray:
    """cv2.resize(img, (w, h), interpolation=INTER_LINEAR_EXACT) for uint8: Q8 horizontal pass, Q8 x Q8 vertical pass,
    rounded shift by 16."""
    sh, sw = img.shape
    xo, xc0, xc1 = _linear_taps(sw, w)
    yo, yc0, yc1 = _linear_taps(sh, h)
    s = img.astype(np.int64)
    xo1 = np.minimum(xo + 1, sw - 1)
    hz = s[:, xo] * xc0 + s[:, xo1] * xc1
    yo1 = np.minimum(yo + 1, sh - 1)
    v = hz[yo] * yc0[:, None] + hz[yo1] * yc1[:, None]
    return ((v + (1 << 15)) >> 16).astype(np.uint8)


def pyramid(gray: np.ndarray) -> List[np.ndarray]:
    """The 8 level images, each resized from the previous one."""
    levels = [gray]
    for (h, w) in level_sizes(*gray.shape)[1:]:
        levels.append(resize_linear_exact(levels[-1], h, w))
    return levels


def mask_pyramid(mask: np.ndarray) -> List[np.ndarray]:
    """The level masks: level 0 is (mask != 0) as 0 / 255; level l is level l - 1 resized like the image, then every value
    below 255 set to 0 (threshold 254, THRESH_TOZERO).  A keypoint survives where its level's mask is non-zero."""
    out = [np.where(mask != 0, 255, 0).astype(np.uint8)]
    for (h, w) in level_sizes(*mask.shape)[1:]:
        r = resize_linear_exact(out[-1], h, w)
        out.append(np.where(r == 255, r, 0).astype(np.uint8))
    return out


def fast_score(img: np.ndarray, thr: int = FAST_T) -> np.ndarray:
    """FAST-9/16 corner score as cv2's FAST with non-max suppression stores it: for a corner (an arc of 9 contiguous
    circle pixels all brighter than centre + thr or all darker than centre - thr), max(thr, the largest arc minimum of
    |centre - pixel| on one side) - 1; 0 elsewhere and within 3 pixels of the border.  uint8."""
    h, w = img.shape
    out = np.zeros((h, w), np.uint8)
    if h < 7 or w < 7:
        return out
    s = img.astype(np.int16)
    c = s[3:h - 3, 3:w - 3]
    d = np.stack([c - s[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for dx, dy in CIRCLE])  # (16, h - 6, w - 6)
    best = np.full(c.shape, -1000, np.int16)
    for sign in (1, -1):
        dd = d * sign
        for k in range(16):
            m = dd[[(k + j) % 16 for j in range(9)]].min(0)
            best = np.maximum(best, m)
    corner = best > thr
    out[3:h - 3, 3:w - 3] = np.where(corner, np.maximum(best, thr) - 1, 0).astype(np.uint8)
    return out


def fast_nms(score: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Corners whose score beats all 8 neighbours strictly -> (y, x) in raster order."""
    h, w = score.shape
    p = np.zeros((h + 2, w + 2), np.int16)
    p[1:-1, 1:-1] = score
    c = p[1:-1, 1:-1]
    keep = c > 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dy or dx:
                keep &= c > p[1 + dy:h + 1 + dy, 1 + dx:w + 1 + dx]
    return np.nonzero(keep)


def retain_best(resp: np.ndarray, n: int) -> np.ndarray:
    """KeyPointsFilter::retainBest as a set: the indices whose response is >= the n-th largest (all when n >= len)."""
    if n >= len(resp):
        return np.arange(len(resp))
    if n == 0:
        return np.zeros(0, np.int64)
    kth = np.sort(resp)[::-1][n - 1]
    return np.nonzero(resp >= kth)[0]


def harris(img: np.ndarray, y: np.ndarray, x: np.ndarray) -> np.ndarray:
    """HarrisResponses, block 7: integer sums a = sum Ix^2, b = sum Iy^2, c = sum Ix Iy of the 3 x 3 Sobel-like
    differences over the 7 x 7 block, then ((a b - c c) - k (a + b)(a + b)) scale^4 in float, operation by operation."""
    s = img.astype(np.int64)
    r = HARRIS_BLOCK // 2
    a = np.zeros(len(y), np.int64)
    b = np.zeros(len(y), np.int64)
    c = np.zeros(len(y), np.int64)
    for i in range(-r, r + 1):
        for j in range(-r, r + 1):
            yy, xx = y + i, x + j
            ix = (s[yy, xx + 1] - s[yy, xx - 1]) * 2 + (s[yy - 1, xx + 1] - s[yy - 1, xx - 1]) + (s[yy + 1, xx + 1] - s[yy + 1, xx - 1])
            iy = (s[yy + 1, xx] - s[yy - 1, xx]) * 2 + (s[yy + 1, xx - 1] - s[yy - 1, xx - 1]) + (s[yy + 1, xx + 1] - s[yy - 1, xx + 1])
            a += ix * ix
            b += iy * iy
            c += ix * iy
    fa, fb, fc = a.astype(F32), b.astype(F32), c.astype(F32)
    scale = F32(1) / F32(F32(4 * HARRIS_BLOCK) * F32(255))
    ssss = F32(F32(F32(scale * scale) * scale) * scale)
    ab = fa + fb
    return (((fa * fb) - (fc * fc)) - ((HARRIS_K * ab) * ab)) * ssss


def umax() -> np.ndarray:
    """The half-width of every row of the radius-15 disc, made symmetric as ORB does."""
    half = PATCH // 2
    u = np.zeros(half + 2, np.int64)
    vmax = int(np.floor(half * np.sqrt(F32(2)) / 2 + 1))
    vmin = int(np.ceil(half * np.sqrt(F32(2)) / 2))
    for v in range(vmax + 1):
        u[v] = int(np.rint(np.sqrt(float(half * half - v * v))))
    v0 = 0
    for v in range(half, vmin - 1, -1):
        while u[v0] == u[v0 + 1]:
            v0 += 1
        u[v] = v0
        v0 += 1
    return u[: half + 1]


def fast_atan2(y: np.ndarray, x: np.ndarray) -> np.ndarray:
    """cv2.fastAtan2 in float32, degrees in [0, 360)."""
    k = F32(180 / np.pi)
    p1, p3, p5, p7 = (F32(F32(c) * k) for c in (0.9997878412794807, -0.3258083974640975, 0.1555786518463281, -0.04432655554792128))
    y, x = np.asarray(y, F32), np.asarray(x, F32)
    ax, ay = np.abs(x), np.abs(y)
    eps = F32(np.finfo(np.float64).eps)
    with np.errstate(invalid="ignore", divide="ignore"):
        c = np.where(ax >= ay, ay / (ax + eps), ax / (ay + eps)).astype(F32)
    c2 = c * c
    poly = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c
    a = np.where(ax >= ay, poly, F32(90) - poly).astype(F32)
    a = np.where(x < 0, F32(180) - a, a).astype(F32)
    return np.where(y < 0, F32(360) - a, a).astype(F32)


def moments(img: np.ndarray, y: np.ndarray, x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """ICAngles' integer moments m01, m10 over the disc."""
    s = img.astype(np.int64)
    um = umax()
    m01 = np.zeros(len(y), np.int64)
    m10 = np.zeros(len(y), np.int64)
    for u in range(-15, 16):
        m10 += u * s[y, x + u]
    for v in range(1, 16):
        vs = np.zeros(len(y), np.int64)
        for u in range(-um[v], um[v] + 1):
            p, m = s[y + v, x + u], s[y - v, x + u]
            vs += p - m
            m10 += u * (p + m)
        m01 += v * vs
    return m01, m10


def gaussian_taps() -> np.ndarray:
    """cv2.getGaussianKernel(7, 2, CV_32F): the double computation (csrc/sift.cu's sf_taps), rounded to float."""
    scale2x = -0.125 / (2.0 * 2.0)
    v = [np.exp(float(x * x) * scale2x) for x in range(-6, 0, 2)]
    mul = 1.0 / (sum(v) * 2.0 + 1.0)
    return np.array([t * mul for t in v] + [mul] + [t * mul for t in v[::-1]]).astype(F32)


def _fma32(a, b, c):
    """float32 fused multiply-add (the float64 sum of an exact float64 product, rounded once more to float32)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def blur(img: np.ndarray) -> np.ndarray:
    """ORB's GaussianBlur(7 x 7, sigma 2, BORDER_REFLECT_101) of a level: row pass s = k0 p0, then s = fma(p_k, k_k, s)
    for k = 1..6; column pass s = k3 q0, then s = fma(q_-k + q_k, k_3+k, s) for k = 1..3; round half to even, saturate."""
    t = gaussian_taps()
    h, w = img.shape
    ry = np.abs(np.arange(-3, h + 3))
    ry = np.where(ry >= h, 2 * h - 2 - ry, ry) if h > 1 else np.zeros_like(ry)
    rx = np.abs(np.arange(-3, w + 3))
    rx = np.where(rx >= w, 2 * w - 2 - rx, rx) if w > 1 else np.zeros_like(rx)
    p = img.astype(F32)[:, rx]
    row = (p[:, 0:w] * t[0]).astype(F32)
    for k in range(1, 7):
        row = _fma32(p[:, k:k + w], t[k], row)
    q = row[ry]
    col = (q[3:3 + h] * t[3]).astype(F32)
    for k in range(1, 4):
        col = _fma32((q[3 - k:3 - k + h] + q[3 + k:3 + k + h]).astype(F32), t[3 + k], col)
    return np.clip(np.rint(col), 0, 255).astype(np.uint8)


def load_pattern(path: Path = PATTERN_INC) -> np.ndarray:
    """The committed rBRIEF pattern: (512, 2) int (x, y); points 2i, 2i + 1 form test i."""
    nums = [int(t) for line in path.read_text().splitlines() if not line.startswith("//")
            for t in line.replace(",", " ").split()]
    return np.array(nums, np.int64).reshape(512, 2)


_LIBM = ctypes.CDLL(ctypes.util.find_library("m"))
_LIBM.cos.restype = _LIBM.sin.restype = ctypes.c_double
_LIBM.cos.argtypes = _LIBM.sin.argtypes = [ctypes.c_double]


def cos_sin(angle_deg: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(float)cos(angle * (float)(pi / 180)), likewise sin: the float angle in radians, cos / sin in double, rounded."""
    rad = (np.asarray(angle_deg, F32) * F32(np.pi / 180)).astype(F32)
    return (np.array([_LIBM.cos(float(r)) for r in rad], np.float64).astype(F32),
            np.array([_LIBM.sin(float(r)) for r in rad], np.float64).astype(F32))


def describe(blurred: np.ndarray, cy: np.ndarray, cx: np.ndarray, angle: np.ndarray, pattern: np.ndarray) -> np.ndarray:
    """rBRIEF: bit k of byte i = I(p_{16i+2k}) < I(p_{16i+2k+1}) with p rotated by the angle,
    (cvRound(x cos - y sin), cvRound(x sin + y cos)) around the centre pixel (cy, cx)."""
    a, b = cos_sin(angle)
    px, py = pattern[:, 0].astype(F32), pattern[:, 1].astype(F32)
    rx = np.rint((px[None] * a[:, None]).astype(F32) - (py[None] * b[:, None]).astype(F32)).astype(np.int64)
    ry = np.rint((px[None] * b[:, None]).astype(F32) + (py[None] * a[:, None]).astype(F32)).astype(np.int64)
    v = blurred[cy[:, None] + ry, cx[:, None] + rx].astype(np.int16)  # (n, 512)
    bits = (v[:, 0::2] < v[:, 1::2]).astype(np.uint8).reshape(-1, 32, 8)
    return (bits << np.arange(8, dtype=np.uint8)).sum(2).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# the whole detector
# ---------------------------------------------------------------------------------------------------------------------
def orb(arr: np.ndarray, mask: Optional[np.ndarray] = None, pattern: Optional[np.ndarray] = None,
        stages: Optional[dict] = None) -> Tuple[Dict[str, np.ndarray], np.ndarray]:
    """cv2.ORB_create().detectAndCompute restated -> (field arrays, (n, 32) uint8 descriptors) in the order csrc/orb.cu
    writes: level ascending, response descending, then y, then x.  `stages`, when given, receives the per-level
    intermediates (levels, score maps, candidates, Harris responses, blurred levels)."""
    gray = rgb_to_gray_cv(arr)
    pattern = load_pattern() if pattern is None else pattern
    levels = pyramid(gray)
    masks = mask_pyramid(mask) if mask is not None else None
    scales = level_scales()
    nper = features_per_level()
    recs = []
    descs = []
    st = stages if stages is not None else {}
    st.update(levels=levels, scores=[], cand=[], harris=[], blurred=[])
    for l, img in enumerate(levels):
        h, w = img.shape
        score = fast_score(img)
        st["scores"].append(score)
        y, x = fast_nms(score)
        if masks is not None:
            keep = masks[l][y, x] != 0
            y, x = y[keep], x[keep]
        if h <= 2 * EDGE or w <= 2 * EDGE:
            y, x = y[:0], x[:0]
        keep = (x >= EDGE) & (x < w - EDGE) & (y >= EDGE) & (y < h - EDGE)
        y, x = y[keep], x[keep]
        sel = retain_best(score[y, x].astype(F32), 2 * nper[l])
        y, x = y[sel], x[sel]
        st["cand"].append((y, x))
        resp = harris(img, y, x)
        st["harris"].append(resp)
        sel = retain_best(resp, nper[l])
        y, x, resp = y[sel], x[sel], resp[sel]
        order = np.lexsort((x, y, -resp.astype(np.float64)))
        y, x, resp = y[order], x[order], resp[order]
        m01, m10 = moments(img, y, x)
        ang = fast_atan2(m01.astype(F32), m10.astype(F32))
        s = scales[l]
        ptx, pty = (x.astype(F32) * s).astype(F32), (y.astype(F32) * s).astype(F32)
        inv = F32(1) / s
        cy = np.rint((pty * inv).astype(F32)).astype(np.int64)
        cx = np.rint((ptx * inv).astype(F32)).astype(np.int64)
        bl = blur(img)
        st["blurred"].append(bl)
        descs.append(describe(bl, cy, cx, ang, pattern) if len(y) else np.zeros((0, 32), np.uint8))
        recs.append({"x": ptx, "y": pty, "size": np.full(len(y), F32(PATCH) * s, F32), "angle": ang, "response": resp.astype(F32),
                     "octave": np.full(len(y), l, np.int32)})
    rec = {f: np.concatenate([r[f] for r in recs]) for f in FIELDS}
    return rec, np.concatenate(descs)


def same_keypoints(a: Dict[str, np.ndarray], da: np.ndarray, b: Dict[str, np.ndarray], db: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Match two keypoint sets by (octave, x bits, y bits) -> (ia, ib) permutations that put both in the same order;
    raises when the sets differ."""
    def key(r):
        return [(int(o), int(x), int(y)) for o, x, y in zip(r["octave"], r["x"].view(np.int32), r["y"].view(np.int32))]

    ka, kb = key(a), key(b)
    if sorted(ka) != sorted(kb) or len(set(ka)) != len(ka):
        raise AssertionError(f"keypoint sets differ: {len(set(ka) - set(kb))} only in a, {len(set(kb) - set(ka))} only in b")
    ia = np.argsort(np.array(ka, dtype=[("o", "i8"), ("x", "i8"), ("y", "i8")]), order=("o", "x", "y"), kind="stable")
    ib = np.argsort(np.array(kb, dtype=[("o", "i8"), ("x", "i8"), ("y", "i8")]), order=("o", "x", "y"), kind="stable")
    return ia, ib


CASES = ("lund_1", "lund_2", "lund_3", "lund_4", "lund_5", "lund_4_rgb", "lund_4_rgba", "lund_2_mask", "odd_crop", "low_levels",
         "tiny_crop", "flat", "synthetic_12mp")


def case_image(name: str, golden_dir) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    """The input (uint8 image, optional uint8 mask) of golden case `name`: sift_ref.case_image's inputs (its mask is 0 / 1, as
    gtsfm passes masks), plus `low_levels`, a 130 x 160 crop whose levels 3..7 are too small for keypoints."""
    from oracle import sift_ref

    if name == "low_levels":
        return np.ascontiguousarray(sift_ref.case_image("lund_1", golden_dir)[0][200:330, 100:260]), None
    return sift_ref.case_image(name, golden_dir)
