"""Seeded synthetic weights and frames.

No pretrained checkpoint exists offline (SURVEY.md, probe table: ``*.pth`` none on disk), so every parity fixture
and benchmark uses weights regenerated from a seed.  The tensors follow the reference's state-dict naming exactly
(SURVEY.md Appendix A), so a real ``superpoint_v1.pth`` / ``superpoint_lightglue_v0-1_arxiv.pth`` /
``superglue_outdoor.pth`` can be dropped in instead without touching any other code.

Everything here is numpy ``default_rng`` (bit-stable across numpy versions for ``standard_normal`` / ``random``),
never torch's generator, so the GPU box regenerates byte-identical weights and frames.
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

SP_CONVS = [  # name, out, in, k  (thirdparty/SuperGluePretrainedNetwork/models/superpoint.py:119-134)
    ("conv1a", 64, 1, 3),
    ("conv1b", 64, 64, 3),
    ("conv2a", 64, 64, 3),
    ("conv2b", 64, 64, 3),
    ("conv3a", 128, 64, 3),
    ("conv3b", 128, 128, 3),
    ("conv4a", 128, 128, 3),
    ("conv4b", 128, 128, 3),
    ("convPa", 256, 128, 3),
    ("convPb", 65, 256, 1),
    ("convDa", 256, 128, 3),
    ("convDb", 256, 256, 1),
]


def superpoint_state_dict(seed: int = 0) -> Dict[str, np.ndarray]:
    """He-normal SuperPoint weights (std = sqrt(2/fan_in)), small non-zero biases.

    PyTorch's default init gives a score map that is flat to four decimals, which makes index parity meaningless
    (SURVEY.md §7 step 0c); He-normal keeps activations O(1) through the 10 ReLU layers and spreads scores over
    0.005..0.1.
    """
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    for name, co, ci, k in SP_CONVS:
        fan_in = ci * k * k
        sd[f"{name}.weight"] = (rng.standard_normal((co, ci, k, k)) * np.sqrt(2.0 / fan_in)).astype(np.float32)
        sd[f"{name}.bias"] = (rng.standard_normal(co) * 0.02).astype(np.float32)
    return sd


def _lin(rng, out_f: int, in_f: int, gain: float = 1.0, bias_std: float = 0.02) -> Tuple[np.ndarray, np.ndarray]:
    w = (rng.standard_normal((out_f, in_f)) * (gain / np.sqrt(in_f))).astype(np.float32)
    b = (rng.standard_normal(out_f) * bias_std).astype(np.float32)
    return w, b


def lightglue_state_dict(seed: int = 2, profile: str = "full") -> Dict[str, np.ndarray]:
    """Crafted LightGlue weights (252 tensors, names as thirdparty/LightGlue/lightglue/lightglue.py:393-408).

    Random He-normal LightGlue weights give ~0 matches (SURVEY.md §7 step 0c).  The crafting keeps the residual
    stream close to the input descriptors (small ``out_proj`` / ``to_out`` / last FFN linear), makes ``final_proj``
    a scaled identity plus noise so that similar descriptors score high, and sets the confidence / matchability
    heads per ``profile`` so that fixtures exercise each data-dependent branch:

    * ``"full"``   – confidences low everywhere: all 9 layers run; matchability high: nothing is pruned.
    * ``"prune"``  – matchability is descriptor-dependent with a negative tail: points get pruned layer by layer.
    * ``"stop"``   – confidence bias rises with depth: early exit fires around layer 4-5.
    * ``"sharp"``  – as "stop" with a 160x identity ``final_proj``: separates the nearly collinear descriptors a
      random-weight SuperPoint produces on real images (mean pairwise cosine 0.97), for detect->match chain fixtures.
    * ``"bench"``  – as "full" (all 9 layers, nothing pruned: the maximum-work path) with the sharp ``final_proj``.
    """
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    d = 256
    sd["posenc.Wr.weight"] = (rng.standard_normal((32, 2)) * 1.5).astype(np.float32)
    for i in range(9):
        p = f"transformers.{i}.self_attn."
        sd[p + "Wqkv.weight"], sd[p + "Wqkv.bias"] = _lin(rng, 3 * d, d, gain=1.6)
        sd[p + "out_proj.weight"], sd[p + "out_proj.bias"] = _lin(rng, d, d, gain=0.3)
        sd[p + "ffn.0.weight"], sd[p + "ffn.0.bias"] = _lin(rng, 2 * d, 2 * d, gain=1.0)
        sd[p + "ffn.1.weight"] = (1.0 + 0.1 * rng.standard_normal(2 * d)).astype(np.float32)
        sd[p + "ffn.1.bias"] = (0.05 * rng.standard_normal(2 * d)).astype(np.float32)
        sd[p + "ffn.3.weight"], sd[p + "ffn.3.bias"] = _lin(rng, d, 2 * d, gain=0.02, bias_std=0.001)
        p = f"transformers.{i}.cross_attn."
        sd[p + "to_qk.weight"], sd[p + "to_qk.bias"] = _lin(rng, d, d, gain=6.0)
        sd[p + "to_v.weight"], sd[p + "to_v.bias"] = _lin(rng, d, d, gain=1.0)
        sd[p + "to_out.weight"], sd[p + "to_out.bias"] = _lin(rng, d, d, gain=0.3)
        sd[p + "ffn.0.weight"], sd[p + "ffn.0.bias"] = _lin(rng, 2 * d, 2 * d, gain=1.0)
        sd[p + "ffn.1.weight"] = (1.0 + 0.1 * rng.standard_normal(2 * d)).astype(np.float32)
        sd[p + "ffn.1.bias"] = (0.05 * rng.standard_normal(2 * d)).astype(np.float32)
        sd[p + "ffn.3.weight"], sd[p + "ffn.3.bias"] = _lin(rng, d, 2 * d, gain=0.02, bias_std=0.001)
    for i in range(9):
        p = f"log_assignment.{i}."
        w, b = _lin(rng, d, d, gain=0.15, bias_std=0.0)
        fgain = 160.0 if profile in ("sharp", "bench") else 18.0
        sd[p + "final_proj.weight"] = (w + fgain * np.eye(d, dtype=np.float32)).astype(np.float32)
        sd[p + "final_proj.bias"] = b
        mw = rng.standard_normal((1, d)).astype(np.float32)
        if profile == "prune":
            # z = w.desc + b with |desc| = 1: N(4, 4.5^2) -> ~3 % of points per layer fall below logit(0.01) = -4.6
            sd[p + "matchability.weight"] = (mw * 4.5).astype(np.float32)
            sd[p + "matchability.bias"] = np.array([4.0], np.float32)
        else:
            sd[p + "matchability.weight"] = (mw * 0.5).astype(np.float32)
            sd[p + "matchability.bias"] = np.array([3.0], np.float32)
    for i in range(8):
        p = f"token_confidence.{i}.token.0."
        tw = rng.standard_normal((1, d)).astype(np.float32)
        if profile in ("stop", "sharp"):
            sd[p + "weight"] = (tw * 1.5).astype(np.float32)
            sd[p + "bias"] = np.array([-3.0 + 1.6 * i], np.float32)
        elif profile == "prune":
            # confident almost everywhere so that low-matchability points are actually dropped
            sd[p + "weight"] = (tw * 2.0).astype(np.float32)
            sd[p + "bias"] = np.array([2.2], np.float32)
        else:
            sd[p + "weight"] = (tw * 1.0).astype(np.float32)
            sd[p + "bias"] = np.array([-2.0], np.float32)
    return sd


def superglue_state_dict(seed: int = 1, profile: str = "full") -> Dict[str, np.ndarray]:
    """Crafted SuperGlue weights (339 tensors, names as SURVEY.md Appendix A).

    ``profile="sharp"`` scales the identity part of ``final_proj`` (12 -> 32) so that true correspondences still win the
    optimal transport against thousands of distractors (the 2048- and 5000-keypoint fixtures and the bench workload); every
    other tensor is identical to the default profile (the RNG stream is consumed in the same order)."""
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    d = 256

    def conv1d(name, co, ci, gain=1.0, bias_std=0.02):
        w, b = _lin(rng, co, ci, gain, bias_std)
        sd[name + ".weight"] = w[:, :, None].copy()
        sd[name + ".bias"] = b

    def bn(name, c):
        sd[name + ".weight"] = (1.0 + 0.1 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".bias"] = (0.05 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_mean"] = (0.1 * rng.standard_normal(c)).astype(np.float32)
        sd[name + ".running_var"] = (1.0 + 0.2 * rng.random(c)).astype(np.float32)
        sd[name + ".num_batches_tracked"] = np.array(1000, np.int64)

    sd["bin_score"] = np.array(2.3, np.float32)
    chans = [3, 32, 64, 128, 256, 256]
    for li, idx in enumerate([0, 3, 6, 9, 12]):
        last = li == 4
        conv1d(f"kenc.encoder.{idx}", chans[li + 1], chans[li], gain=(0.05 if last else 1.4), bias_std=(0.0 if last else 0.02))
        if not last:
            bn(f"kenc.encoder.{idx + 1}", chans[li + 1])
    for i in range(18):
        p = f"gnn.layers.{i}."
        for j in range(3):
            conv1d(p + f"attn.proj.{j}", d, d, gain=(2.5 if j < 2 else 1.0))
        conv1d(p + "attn.merge", d, d, gain=0.5)
        conv1d(p + "mlp.0", 2 * d, 2 * d, gain=1.0)
        bn(p + "mlp.1", 2 * d)
        conv1d(p + "mlp.3", d, 2 * d, gain=0.03, bias_std=0.0)
    w, b = _lin(rng, d, d, gain=0.15, bias_std=0.0)
    fgain = 32.0 if profile == "sharp" else 12.0
    sd["final_proj.weight"] = (w + fgain * np.eye(d, dtype=np.float32))[:, :, None].astype(np.float32)
    sd["final_proj.bias"] = b
    return sd


NETVLAD_CONVS = [(0, 3, 64), (2, 64, 64), (5, 64, 128), (7, 128, 128), (10, 128, 256), (12, 256, 256), (14, 256, 256), (17, 256, 512),
                 (19, 512, 512), (21, 512, 512), (24, 512, 512), (26, 512, 512), (28, 512, 512)]  # (index in backbone, Cin, Cout)
NETVLAD_POOL_AFTER = (2, 7, 14, 21)  # backbone conv indices followed by MaxPool2d(2, 2) (vgg16.features[:-2])


def netvlad_state_dict(seed: int = 3, whiten_dim: int = 4096) -> Dict[str, np.ndarray]:
    """Seeded random weights with the exact tensor names / shapes of thirdparty/hloc/netvlad.py's NetVLAD module
    (VGG16 features[:-2] backbone, NetVLADLayer(512, 64), whiten Linear(32768, 4096)) plus `mean` = the checkpoint's
    `normalization.averageImage` (netvlad.py:157-160).  No checkpoint can be downloaded offline."""
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    for idx, ci, co in NETVLAD_CONVS:
        sd[f"backbone.{idx}.weight"] = (rng.standard_normal((co, ci, 3, 3)) * np.sqrt(2.0 / (9 * ci))).astype(np.float32)
        sd[f"backbone.{idx}.bias"] = (0.05 * rng.standard_normal(co)).astype(np.float32)
    sd["backbone.0.weight"] *= np.float32(1.0 / 60.0)  # the first layer sees mean-subtracted 0..255 pixels
    sd["netvlad.score_proj.weight"] = (4.0 * rng.standard_normal((64, 512, 1))).astype(np.float32)
    sd["netvlad.centers"] = rng.uniform(-0.08, 0.08, (512, 64)).astype(np.float32)
    sd["whiten.weight"] = (rng.standard_normal((whiten_dim, 32768), dtype=np.float32) * np.float32(1.0 / np.sqrt(32768.0)))
    sd["whiten.bias"] = (0.0005 * rng.standard_normal(whiten_dim)).astype(np.float32)
    sd["mean"] = np.array([123.68, 116.779, 103.939], np.float32)
    return sd


def megaloc_state_dict(seed: int = 5) -> Dict[str, np.ndarray]:
    """Seeded weights with the names and shapes of the reference's MegaLoc checkpoint (190 tensors: DINOv2 ViT-B/14 under
    `backbone.model.`, SALAD under `aggregator.agg.`, the final `aggregator.linear`).  No checkpoint can be downloaded offline.

    Torch's default init makes every image look alike (cosine 0.9997 between two random images), which would let any
    parity test pass trivially.  Here the patch embedding is strong (so image content dominates the position table), the
    residual branches are small (LayerScale 0.1), attention logits are O(1), and the SALAD score head is sharp, so distinct
    frames land far apart and a shifted view of a frame stays nearest to that frame."""
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    d, bb, ag = 768, "backbone.model.", "aggregator.agg."

    def lin(name, o, i, gain=1.0, bias_std=0.02, shape=None):
        w, b = _lin(rng, o, i, gain, bias_std)
        sd[name + ".weight"] = w.reshape(shape) if shape else w
        sd[name + ".bias"] = b

    sd[bb + "cls_token"] = (0.5 * rng.standard_normal((1, 1, d))).astype(np.float32)
    sd[bb + "pos_embed"] = (0.1 * rng.standard_normal((1, 1 + 37 * 37, d))).astype(np.float32)
    sd[bb + "mask_token"] = np.zeros((1, d), np.float32)
    lin(bb + "patch_embed.proj", d, 588, gain=3.0, shape=(d, 3, 14, 14))
    for i in range(12):
        p = f"{bb}blocks.{i}."
        sd[p + "norm1.weight"] = (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32)
        sd[p + "norm1.bias"] = (0.05 * rng.standard_normal(d)).astype(np.float32)
        lin(p + "attn.qkv", 3 * d, d, gain=1.0)
        lin(p + "attn.proj", d, d, gain=1.0)
        sd[p + "ls1.gamma"] = (0.1 * (1.0 + 0.2 * rng.standard_normal(d))).astype(np.float32)
        sd[p + "norm2.weight"] = (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32)
        sd[p + "norm2.bias"] = (0.05 * rng.standard_normal(d)).astype(np.float32)
        lin(p + "mlp.fc1", 4 * d, d, gain=1.4)
        lin(p + "mlp.fc2", d, 4 * d, gain=1.0)
        sd[p + "ls2.gamma"] = (0.1 * (1.0 + 0.2 * rng.standard_normal(d))).astype(np.float32)
    sd[bb + "norm.weight"] = (1.0 + 0.1 * rng.standard_normal(d)).astype(np.float32)
    sd[bb + "norm.bias"] = (0.05 * rng.standard_normal(d)).astype(np.float32)
    lin(ag + "token_features.0", 512, d, gain=1.4)
    lin(ag + "token_features.2", 256, 512, gain=1.0)
    lin(ag + "cluster_features.0", 512, d, gain=1.4, shape=(512, d, 1, 1))
    lin(ag + "cluster_features.3", 256, 512, gain=2.0, shape=(256, 512, 1, 1))
    lin(ag + "score.0", 512, d, gain=1.4, shape=(512, d, 1, 1))
    lin(ag + "score.3", 64, 512, gain=8.0, shape=(64, 512, 1, 1))
    sd[ag + "dust_bin"] = np.array(1.0, np.float32)
    sd["aggregator.linear.weight"] = (rng.standard_normal((8448, 16640), dtype=np.float32) * np.float32(1.0 / np.sqrt(16640.0)))
    sd["aggregator.linear.bias"] = (0.002 * rng.standard_normal(8448)).astype(np.float32)
    return sd


D2NET_CONVS = [(0, 3, 64), (2, 64, 64), (5, 64, 128), (7, 128, 128), (10, 128, 256), (12, 256, 256), (14, 256, 256), (17, 256, 512),
               (19, 512, 512), (21, 512, 512)]  # (index in dense_feature_extraction.model, Cin, Cout)


def d2net_state_dict(seed: int = 7) -> Dict[str, np.ndarray]:
    """Seeded He-normal weights with small biases, named as the reference's d2_tf.pth `model` state dict
    (thirdparty/d2net/lib/model_test.py: dense_feature_extraction.model.{0,2,...,21}).  No checkpoint can be downloaded offline."""
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    for idx, ci, co in D2NET_CONVS:
        sd[f"dense_feature_extraction.model.{idx}.weight"] = (rng.standard_normal((co, ci, 3, 3)) * np.sqrt(2.0 / (9 * ci))).astype(np.float32)
        sd[f"dense_feature_extraction.model.{idx}.bias"] = (0.01 * rng.standard_normal(co)).astype(np.float32)
    return sd


def save_pth(state: Dict[str, np.ndarray], path) -> None:
    """Write a state dict in the reference's checkpoint format (torch.save of name -> tensor)."""
    import torch

    torch.save({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in state.items()}, str(path))


def synthetic_frame(idx: int, height: int, width: int, n_shapes: int = 600) -> np.ndarray:
    """Seeded RGB uint8 frame: random-contrast rectangles over smooth noise (SURVEY.md §8d 'Synthetic inputs')."""
    rng = np.random.default_rng(1000 + idx)
    img = np.full((height, width), 110.0, np.float32)
    # low-frequency background
    coarse = rng.random((height // 32 + 2, width // 32 + 2)).astype(np.float32)
    img += 60.0 * np.kron(coarse, np.ones((32, 32), np.float32))[:height, :width]
    ys = rng.integers(0, height, n_shapes)
    xs = rng.integers(0, width, n_shapes)
    hs = rng.integers(4, max(5, height // 6), n_shapes)
    ws = rng.integers(4, max(5, width // 6), n_shapes)
    vals = rng.uniform(0, 255, n_shapes).astype(np.float32)
    alphas = rng.uniform(0.3, 1.0, n_shapes).astype(np.float32)
    for y, x, h, w, v, a in zip(ys, xs, hs, ws, vals, alphas):
        sl = (slice(y, min(height, y + h)), slice(x, min(width, x + w)))
        img[sl] = (1 - a) * img[sl] + a * v
    img += rng.normal(0, 3.0, (height, width)).astype(np.float32)
    g = np.clip(img, 0, 255)
    rgb = np.stack([g, np.clip(g * 0.97 + 4, 0, 255), np.clip(g * 1.03 - 4, 0, 255)], -1)
    return rgb.astype(np.uint8)


def synthetic_features(seed: int, n0: int, n1: int, height: int = 480, width: int = 640, outlier_frac: float = 0.3,
                       noise: float = 0.05):
    """Matcher micro-benchmark inputs (SURVEY.md §8d): image-1 set = permuted, perturbed image-0 set + outliers.

    Returns (kp0 (n0,2) f32, sc0 (n0,), desc0 (n0,256), kp1, sc1, desc1, gt (n0,) int index into set 1 or -1).
    """
    rng = np.random.default_rng(seed)
    kp0 = np.stack([rng.uniform(4, width - 5, n0), rng.uniform(4, height - 5, n0)], -1).astype(np.float32)
    d0 = rng.standard_normal((n0, 256)).astype(np.float32)
    d0 /= np.linalg.norm(d0, axis=1, keepdims=True)
    sc0 = rng.uniform(0.005, 0.3, n0).astype(np.float32)
    n_shared = min(n0, int(round(n1 * (1 - outlier_frac))))
    src = rng.permutation(n0)[:n_shared]
    kp1 = np.empty((n1, 2), np.float32)
    d1 = np.empty((n1, 256), np.float32)
    # a mild similarity warp + jitter for the shared points
    ang = 0.05
    R = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]], np.float32)
    kp1[:n_shared] = (kp0[src] - [width / 2, height / 2]) @ R.T * 0.97 + [width / 2 + 6, height / 2 - 4]
    kp1[:n_shared] += rng.normal(0, 0.5, (n_shared, 2)).astype(np.float32)
    d1[:n_shared] = d0[src] + noise * rng.standard_normal((n_shared, 256)).astype(np.float32)
    kp1[n_shared:] = np.stack([rng.uniform(4, width - 5, n1 - n_shared), rng.uniform(4, height - 5, n1 - n_shared)], -1)
    d1[n_shared:] = rng.standard_normal((n1 - n_shared, 256)).astype(np.float32)
    d1 /= np.linalg.norm(d1, axis=1, keepdims=True)
    perm = rng.permutation(n1)
    kp1, d1 = kp1[perm].astype(np.float32), d1[perm].astype(np.float32)
    inv = np.empty(n1, np.int64)
    inv[perm] = np.arange(n1)
    gt = np.full(n0, -1, np.int64)
    gt[src] = inv[:n_shared]
    sc1 = rng.uniform(0.005, 0.3, n1).astype(np.float32)
    return kp0, sc0, d0, kp1, sc1, d1, gt


def synthetic_sequence(n_frames: int, height: int = 480, width: int = 640, step_px: int = 8, seed: int = 77):
    """Frames of a camera translating over one seeded texture: frame i is the crop at x = step_px * i (multiples of 8 keep
    the SuperPoint cell grid aligned, so a random-weight network still yields repeatable descriptors across frames).
    -> list of (H, W, 3) uint8 arrays, and the pinhole calibration (f, u0, v0) used by the verifier."""
    big = synthetic_frame(seed, height + 16, width + step_px * n_frames + 16, n_shapes=600 + 40 * n_frames)
    frames = [np.ascontiguousarray(big[8 * (i % 2): 8 * (i % 2) + height, step_px * i: step_px * i + width]) for i in range(n_frames)]
    return frames, (0.9 * width, width / 2.0, height / 2.0)
