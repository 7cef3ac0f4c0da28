"""Restatement of the reference's single-scale D2-Net detector-descriptor in torch-CPU and NumPy, written from its definition
(gtsfm/frontend/detector_descriptor/d2net.py with USE_MULTISCALE = False; thirdparty/d2net/lib/model_test.py,
pyramid.py process_multiscale(scales=[1]) and utils.py preprocess_image / interpolate_dense_features).

Besides the plugin's outputs it returns each keypoint's feature-map cell and channel (c, i, j) and, for every cell, the
relative distance of the cell's strongest channel to the nearest detection decision (`margin`), so a test can tell a real
difference from a keypoint that float rounding may legitimately flip."""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
CONV_IDX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21)
POOL_AFTER = (2, 7)  # MaxPool2d(2, 2) after these convolutions
DILATED = (17, 19, 21)  # 3x3, dilation 2, padding 2; the average pool runs before the first
EDGE_THRESHOLD = 5
MAX_EDGE_PX, MAX_SUM_EDGES_PX = 1600, 2800
# "flat" is a uniform image.  It still gives keypoints: the convolutions pad with zeros and have non-zero biases, so the dense
# map varies near the border even when the image does not.  In the interior every cell is equal, det = 0 and nothing is
# detected.  With these weights no input gives an empty result (a 1 x 1 map even detects at its only cell: zero gradient,
# det = 4 v^2 > 0); the empty output is exercised with max_keypoints = 0.  "synthetic_top100" is "synthetic" with
# max_keypoints = 100, so the top-k cuts.
CASES = ("synthetic", "synthetic_top100", "lund_1", "lund_2", "rgb", "odd_crop", "tiny_crop", "flat")
CASE_MAX_KEYPOINTS = {"synthetic_top100": 100}


def norm_table() -> np.ndarray:
    """[3][256] float32: preprocess_image('torch') of byte u in channel c = float32(float64(float32(u) / 255) - mean) / std)."""
    x = (np.arange(256, dtype=np.float32) / np.float32(255.0)).astype(np.float64)
    return np.stack([((x - m) / s).astype(np.float32) for m, s in zip(MEAN, STD)])


def preprocess(image: np.ndarray) -> np.ndarray:
    """uint8 (H, W), (H, W, 1) or (H, W, 3) -> (3, H, W) float32, as the plugin feeds the network."""
    if image.dtype != np.uint8 or image.ndim not in (2, 3) or (image.ndim == 3 and image.shape[2] not in (1, 3)):
        raise ValueError("uint8 gray or RGB image expected")
    g = image if image.ndim == 3 else image[:, :, None]
    t = norm_table()
    return np.stack([t[c][g[:, :, c if g.shape[2] == 3 else 0]] for c in range(3)])


def dense_features(x: np.ndarray, sd: Dict[str, np.ndarray], dtype=None):
    """(3, H, W) -> torch (512, H/4 - 1, W/4 - 1) after the final ReLU, in `dtype` (default float32)."""
    import torch
    import torch.nn.functional as F

    dtype = dtype or torch.float32
    t = torch.from_numpy(np.ascontiguousarray(x)).to(dtype)[None]
    with torch.no_grad():
        for idx in CONV_IDX:
            if idx == DILATED[0]:
                t = F.avg_pool2d(t, 2, stride=1)
            w = torch.from_numpy(np.asarray(sd[f"dense_feature_extraction.model.{idx}.weight"])).to(dtype)
            b = torch.from_numpy(np.asarray(sd[f"dense_feature_extraction.model.{idx}.bias"])).to(dtype)
            d = 2 if idx in DILATED else 1
            t = F.relu(F.conv2d(t, w, b, padding=d, dilation=d))
            if idx in POOL_AFTER:
                t = F.max_pool2d(t, 2, stride=2)
    return t[0]


def _shift(t, di: int, dj: int):
    """t[:, i + di, j + dj] with zeros outside the map (conv2d's padding)."""
    import torch.nn.functional as F

    p = F.pad(t, (1, 1, 1, 1))
    h, w = t.shape[1:]
    return p[:, 1 + di: 1 + di + h, 1 + dj: 1 + dj + w]


def detect(dense, max_keypoints: Optional[int] = None) -> Dict[str, np.ndarray]:
    """Hard detection, localisation, description and the plugin's ordering on a (512, h, w) torch map."""
    import torch
    import torch.nn.functional as F

    c_, h, w = dense.shape
    with torch.no_grad():
        dmax = dense.max(0)[0]
        is_dmax = dense == dmax
        local = F.max_pool2d(dense[None], 3, stride=1, padding=1)[0]
        is_local = dense == local
        u, dn, l, r = _shift(dense, -1, 0), _shift(dense, 1, 0), _shift(dense, 0, -1), _shift(dense, 0, 1)
        ul, ur, dl, dr = _shift(dense, -1, -1), _shift(dense, -1, 1), _shift(dense, 1, -1), _shift(dense, 1, 1)
        dii = u - 2 * dense + dn
        djj = l - 2 * dense + r
        dij = 0.25 * (ul - ur - dl + dr)
        det = dii * djj - dij * dij
        tr = dii + djj
        thr = (EDGE_THRESHOLD + 1) ** 2 / EDGE_THRESHOLD
        edge_ratio = tr * tr / det
        not_edge = (edge_ratio <= thr) & (det > 0)
        gi, gj = 0.5 * (dn - u), 0.5 * (r - l)
        step_i = -(djj / det * gi + (-dij / det) * gj)
        step_j = -((-dij / det) * gi + dii / det * gj)

        # relative distance of each cell's strongest channel to every decision it takes
        top2 = dense.topk(2, dim=0)[0] if c_ > 1 else torch.stack([dmax, torch.zeros_like(dmax)])
        cmax = dense.argmax(0)
        pick = lambda t: t.gather(0, cmax[None])[0]  # noqa: E731
        # (zero instead of -inf outside the map: the maps are >= 0 after the ReLU and a zero maximum never detects)
        nb = torch.stack([pick(_shift(dense, a, b)) for a in (-1, 0, 1) for b in (-1, 0, 1) if a or b]).max(0)[0]
        scale = dmax.abs().clamp_min(1e-30)
        m = torch.stack([(top2[0] - top2[1]).abs() / scale, (dmax - nb).abs() / scale,
                         (pick(edge_ratio) - thr).abs() / thr, (pick(det)).abs() / (pick(dii).abs() * pick(djj).abs() + pick(dij) ** 2).clamp_min(1e-30),
                         (pick(step_i).abs() - 0.5).abs() / 0.5, (pick(step_j).abs() - 0.5).abs() / 0.5])
        margin = m.nan_to_num(0.0).min(0)[0].numpy().astype(np.float32)

        detected = is_dmax & is_local & not_edge
        pos = torch.nonzero(detected)  # (c, i, j) lexicographic
        cs, is_, js = pos[:, 0], pos[:, 1], pos[:, 2]
        si, sj = step_i[cs, is_, js], step_j[cs, is_, js]
        keep = (si.abs() < 0.5) & (sj.abs() < 0.5)
        cs, is_, js, si, sj = cs[keep], is_[keep], js[keep], si[keep], sj[keep]
        fi, fj = is_.to(dense.dtype) + si, js.to(dense.dtype) + sj
        i0, j0, i1, j1 = fi.floor().long(), fj.floor().long(), fi.ceil().long(), fj.ceil().long()
        ok = (i0 >= 0) & (j0 >= 0) & (i1 < h) & (j1 < w)
        cs, is_, js, fi, fj, i0, j0, i1, j1 = (t[ok] for t in (cs, is_, js, fi, fj, i0, j0, i1, j1))
        ai, aj = fi - i0.to(dense.dtype), fj - j0.to(dense.dtype)
        desc = ((1 - ai) * (1 - aj) * dense[:, i0, j0] + (1 - ai) * aj * dense[:, i0, j1] + ai * (1 - aj) * dense[:, i1, j0]
                + ai * aj * dense[:, i1, j1])
        desc = F.normalize(desc, dim=0).t()
        y = (fi * 2 + 0.5) * 2 + 0.5
        x = (fj * 2 + 0.5) * 2 + 0.5
        scores = dense[cs, is_, js]
    cs, is_, js, scores = cs.numpy(), is_.numpy(), js.numpy(), scores.numpy()
    order = np.lexsort((js, is_, cs, -scores.astype(np.float64)))  # score descending, then torch.nonzero's (c, i, j)
    total = len(order)
    if max_keypoints is not None:
        order = order[:max_keypoints]
    return {"xy": np.stack([x.numpy(), y.numpy()], 1)[order], "scores": scores[order], "desc": desc.numpy()[order],
            "cij": np.stack([cs, is_, js], 1)[order].astype(np.int32), "margin": margin, "total": np.int64(total)}


def detect_and_describe(image: np.ndarray, sd: Dict[str, np.ndarray], max_keypoints: int = 5000, dtype=None):
    """The plugin's result for a uint8 image within the size limits: dict of xy (K, 2) (x, y), scores, desc (K, 512), cij, margin."""
    if max(image.shape[:2]) > MAX_EDGE_PX or sum(image.shape[:2]) > MAX_SUM_EDGES_PX:
        raise ValueError("image needs the reference's resize")
    return detect(dense_features(preprocess(image), sd, dtype), max_keypoints)


def case_image(name: str, golden_dir) -> np.ndarray:
    """The uint8 input of golden case `name`, rebuilt from tests/golden/lund_door_images.npz or from a seed."""
    from pathlib import Path

    from gtsfm_b200 import synthetic as syn

    lund = lambda i: np.load(Path(golden_dir) / "lund_door_images.npz")[f"gray_{i}"]  # noqa: E731
    if name in ("synthetic", "synthetic_top100"):
        return syn.synthetic_frame(21, 480, 640)[:, :, 0].copy()
    if name.startswith("lund_"):
        return lund(int(name[5:]))
    if name == "rgb":
        return syn.synthetic_frame(22, 240, 320)
    if name == "odd_crop":
        return np.ascontiguousarray(lund(3)[100:617, 200:589])
    if name == "tiny_crop":
        return np.ascontiguousarray(lund(3)[300:340, 400:430])
    if name == "flat":
        return np.full((64, 96), 128, np.uint8)
    raise KeyError(name)
