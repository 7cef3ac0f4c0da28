"""TEST INFRASTRUCTURE (CPU oracle; never imported by the product path).

Torch-CPU fp32 restatement of the reference's MegaLoc global descriptor (thirdparty/megaloc/megaloc.py:25-257) on DINOv2's
DinoVisionTransformer (vit_base, patch 14; vision_transformer.py, block.py, attention.py of the DINOv2 layers):
  * `pos_table`     interpolate_pos_encoding (vision_transformer.py:180-212): bicubic (A = -0.75) from 37 x 37 with scale_factor
                    ((gh + 0.1) / 37, (gw + 0.1) / 37), source = (dst + 0.5) / scale_factor - 0.5, taps clamped at the border;
                    the table as is at 37 x 37.  Restated with explicit interpolation matrices (what the device kernel computes).
  * `backbone`      patch embed, cls + position, 12 blocks x += ls1 proj(attn(LN1 x)), x += ls2 fc2(GELU(fc1(LN2 x))), final LN
  * `salad`         per-token heads, get_matching_probs (3 Sinkhorn iterations with the dustbin row), aggregation, normalisations
  * `megaloc_forward`  backbone + SALAD + Linear(16640 -> 8448) + L2
  * `resize_u8`     NumPy restatement of torch's uint8 antialiased bilinear resize (the integer path of
                    ATen/native/cpu/UpSampleKernelAVXAntialias.h that torchvision's Resize(antialias=True) takes on uint8)
Pinned by tests/golden/megaloc*.npz, made by oracle/make_golden_megaloc.py from the reference module's own forward.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

BB, AG = "backbone.model.", "aggregator.agg."
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def _cubic_coeffs(t: float):
    a = -0.75
    x1, x2 = t + 1.0, 1.0 - t
    x3 = x2 + 1.0
    return [((a * x1 - 5 * a) * x1 + 8 * a) * x1 - 4 * a, ((a + 2) * t - (a + 3)) * t * t + 1,
            ((a + 2) * x2 - (a + 3)) * x2 * x2 + 1, ((a * x3 - 5 * a) * x3 + 8 * a) * x3 - 4 * a]


def bicubic_matrix(out_size: int, in_size: int, scale_factor: float) -> np.ndarray:
    """(out, in) matrix of torch's bicubic upsample along one axis with an explicit scale_factor (align_corners False)."""
    inv = np.float32(1.0 / scale_factor)
    m = np.zeros((out_size, in_size), np.float64)
    for o in range(out_size):
        r = float(np.float32((o + 0.5) * inv - 0.5))
        f = math.floor(r)
        for k, c in enumerate(_cubic_coeffs(r - f)):
            m[o, min(max(f - 1 + k, 0), in_size - 1)] += c
    return m


def pos_table(pos_embed: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """(1, 1 + 37 * 37, 768) -> (1, 1 + gh * gw, 768)."""
    g = 37
    if gh == g and gw == g:
        return pos_embed
    mh = torch.from_numpy(bicubic_matrix(gh, g, (gh + 0.1) / g)).float().to(pos_embed.device)
    mw = torch.from_numpy(bicubic_matrix(gw, g, (gw + 0.1) / g)).float().to(pos_embed.device)
    grid = pos_embed[0, 1:].reshape(g, g, -1)
    patch = torch.einsum("ay,yxc->axc", mh, grid)
    patch = torch.einsum("bx,axc->abc", mw, patch).reshape(1, gh * gw, -1)
    return torch.cat([pos_embed[:, :1], patch], 1)


def backbone(t: Dict[str, torch.Tensor], x: torch.Tensor) -> torch.Tensor:
    """images (B, 3, H, W) normalised -> final-LN tokens (B, 1 + n, 768), cls first."""
    b, _, h, w = x.shape
    gh, gw = h // 14, w // 14
    z = F.conv2d(x, t[BB + "patch_embed.proj.weight"], t[BB + "patch_embed.proj.bias"], stride=14).flatten(2).transpose(1, 2)
    z = torch.cat([t[BB + "cls_token"].expand(b, -1, -1), z], 1) + pos_table(t[BB + "pos_embed"], gh, gw)
    n_tok = z.shape[1]
    for i in range(12):
        p = f"{BB}blocks.{i}."
        y = F.layer_norm(z, (768,), t[p + "norm1.weight"], t[p + "norm1.bias"], 1e-6)
        qkv = F.linear(y, t[p + "attn.qkv.weight"], t[p + "attn.qkv.bias"]).reshape(b, n_tok, 3, 12, 64).permute(2, 0, 3, 1, 4)
        a = F.softmax(qkv[0] @ qkv[1].transpose(-2, -1) * 0.125, dim=-1) @ qkv[2]
        a = a.transpose(1, 2).reshape(b, n_tok, 768)
        z = z + t[p + "ls1.gamma"] * F.linear(a, t[p + "attn.proj.weight"], t[p + "attn.proj.bias"])
        y = F.layer_norm(z, (768,), t[p + "norm2.weight"], t[p + "norm2.bias"], 1e-6)
        y = F.linear(F.gelu(F.linear(y, t[p + "mlp.fc1.weight"], t[p + "mlp.fc1.bias"])), t[p + "mlp.fc2.weight"], t[p + "mlp.fc2.bias"])
        z = z + t[p + "ls2.gamma"] * y
    return F.layer_norm(z, (768,), t[BB + "norm.weight"], t[BB + "norm.bias"], 1e-6)


def sinkhorn_probs(s: torch.Tensor, dust: torch.Tensor, iters: int = 3) -> torch.Tensor:
    """get_matching_probs (megaloc.py:174-188): S (B, 64, n) -> P = exp(log P - norm) (B, 64, n), dustbin row dropped."""
    b, m, n = s.shape
    S = torch.cat([s, dust.reshape(1, 1, 1).expand(b, 1, n)], 1)
    norm = -torch.tensor(math.log(n + m), dtype=s.dtype, device=s.device)
    log_a = norm.expand(m + 1).clone()
    log_a[-1] = log_a[-1] + math.log(n - m)
    log_b = norm.expand(n)
    u, v = torch.zeros(b, m + 1, dtype=s.dtype, device=s.device), torch.zeros(b, n, dtype=s.dtype, device=s.device)
    for _ in range(iters):
        u = log_a - torch.logsumexp(S + v.unsqueeze(1), dim=2)
        v = log_b - torch.logsumexp(S + u.unsqueeze(2), dim=1)
    return torch.exp(S + u.unsqueeze(2) + v.unsqueeze(1) - norm)[:, :-1]


def salad(t: Dict[str, torch.Tensor], tokens: torch.Tensor) -> torch.Tensor:
    """final-LN tokens (B, 1 + n, 768) -> SALAD descriptor (B, 16640)."""
    cls, x = tokens[:, 0], tokens[:, 1:]

    def mlp(name, z, i2):
        w0, w1 = t[f"{AG}{name}.0.weight"], t[f"{AG}{name}.{i2}.weight"]
        z = F.relu(F.linear(z, w0.reshape(w0.shape[0], -1), t[f"{AG}{name}.0.bias"]))
        return F.linear(z, w1.reshape(w1.shape[0], -1), t[f"{AG}{name}.{i2}.bias"])

    f = mlp("cluster_features", x, 3).transpose(1, 2)  # (B, 256, n)
    p = sinkhorn_probs(mlp("score", x, 3).transpose(1, 2), t[AG + "dust_bin"])  # (B, 64, n)
    g = mlp("token_features", cls, 2)
    agg = F.normalize(f @ p.transpose(1, 2), dim=1).flatten(1)  # (B, 256 * 64), l-major
    return F.normalize(torch.cat([F.normalize(g, dim=-1), agg], -1), dim=-1)


def tensors(sd: Dict[str, np.ndarray], dtype=torch.float32) -> Dict[str, torch.Tensor]:
    return {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in sd.items()}


def megaloc_forward(sd, images: np.ndarray, return_tokens: bool = False):
    """images (B, 3, H, W) float32 normalised, H and W multiples of 14 -> (B, 8448) descriptors (and the backbone tokens)."""
    t = sd if isinstance(next(iter(sd.values())), torch.Tensor) else tensors(sd)
    with torch.no_grad():
        x = torch.from_numpy(np.asarray(images)).to(t[BB + "cls_token"].dtype)
        tok = backbone(t, x)
        d = F.normalize(F.linear(salad(t, tok), t["aggregator.linear.weight"], t["aggregator.linear.bias"]), dim=1)
    return (d.numpy(), tok.numpy()) if return_tokens else d.numpy()


# seeded frames of tests/golden/megaloc.npz: (synthetic_frame index, height, width), each resized to 322 x 322
GOLDEN_FRAMES = ((60, 480, 640), (61, 600, 800), (62, 322, 322), (63, 760, 1135))
GOLDEN_TOKEN_ROWS = np.r_[0, 1:530:16]  # backbone token rows of frame 0 kept in the golden: cls and every 16th patch


def golden_frames_u8() -> np.ndarray:
    """The golden's frames after the plugin's resize transform: uint8 (4, 3, 322, 322)."""
    from gtsfm_b200.synthetic import synthetic_frame

    return np.stack([resize_u8(synthetic_frame(i, h, w)) for i, h, w in GOLDEN_FRAMES])


def normalise(u8_chw: np.ndarray) -> np.ndarray:
    """The plugin's batch transform: uint8 (..., 3, H, W) -> (x / 255 - mean) / std in float32."""
    x = u8_chw.astype(np.float32) / np.float32(255.0)
    m = np.array(MEAN, np.float32).reshape(3, 1, 1)
    s = np.array(STD, np.float32).reshape(3, 1, 1)
    return (x - m) / s


# ---- torch's uint8 antialiased bilinear resize ---------------------------------------------------------------------------------
def _axis_weights(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray, int]:
    """compute_index_ranges_int16_weights for the bilinear antialias filter: (xmin, xsize, int16 weights [out][taps], precision)."""
    scale = in_size / out_size
    support = scale if scale >= 1.0 else 1.0
    invscale = 1.0 / scale if scale >= 1.0 else 1.0
    taps = int(math.ceil(support)) * 2 + 1
    w = np.zeros((out_size, taps), np.float64)
    xmin = np.zeros(out_size, np.int64)
    xsize = np.zeros(out_size, np.int64)
    wmax = 0.0
    for i in range(out_size):
        center = scale * (i + 0.5)
        x0 = max(int(center - support + 0.5), 0)
        xs = min(max(min(int(center + support + 0.5), in_size) - x0, 0), taps)
        for j in range(xs):
            a = abs((j + x0 - center + 0.5) * invscale)
            w[i, j] = 1.0 - a if a < 1.0 else 0.0
        tot = w[i, :xs].sum()
        if tot != 0.0:
            w[i, :xs] /= tot
            wmax = max(wmax, w[i, :xs].max())
        xmin[i], xsize[i] = x0, xs
    prec = 0
    while prec < 22 and int(0.5 + wmax * (1 << (prec + 1))) < (1 << 15):
        prec += 1
    v = w * (1 << prec)
    wi = np.where(v < 0, np.trunc(-0.5 + v), np.trunc(0.5 + v)).astype(np.int64)
    return xmin, xsize, wi, prec


def _resample_axis(img: np.ndarray, out_size: int, axis: int) -> np.ndarray:
    in_size = img.shape[axis]
    if in_size == out_size:
        return img
    xmin, xsize, wi, prec = _axis_weights(in_size, out_size)
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((out_size,) + src.shape[1:], np.int64)
    for i in range(out_size):
        acc = np.full(src.shape[1:], 1 << (prec - 1), np.int64)
        for k in range(xsize[i]):
            acc += wi[i, k] * src[xmin[i] + k]
        out[i] = acc >> prec
    return np.moveaxis(np.clip(out, 0, 255).astype(np.uint8), 0, axis)


def resize_u8(img_hwc: np.ndarray, size: int = 322) -> np.ndarray:
    """uint8 (H, W, 3) -> uint8 (3, size, size): torchvision Resize((size, size), antialias=True) on the permuted tensor.
    Horizontal pass first, each pass rounded and clamped to uint8."""
    x = _resample_axis(img_hwc, size, 1)
    x = _resample_axis(x, size, 0)
    return np.ascontiguousarray(x.transpose(2, 0, 1))
