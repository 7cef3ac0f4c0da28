"""TEST INFRASTRUCTURE — CPU restatement of the reference LightGlue path as GTSfM drives it (never shipped).

Restates thirdparty/LightGlue/lightglue/lightglue.py with the CPU semantics GTSfM's CPU front-end sees
(SURVEY.md §7 hard part 3): fp32 attention (:127-130), shared-``sim`` cross attention (:216-223), pruning attempted at
every layer because ``pruning_keypoint_thresholds['cpu'] == -1`` (:339-344,658-662), keypoints normalised by their
bounding box because the wrapper passes ``image`` not ``image_size`` (:31-43,491; lightglue_matcher.py:88-99).

Pinned by ``oracle/make_golden.py`` against the unmodified module (match indices exact).  The reference ships no
LightGlue test (SURVEY.md §8c), so that run is the anchor.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

N_LAYERS = 9
HEADS = 4
DEPTH_CONF = 0.95
WIDTH_CONF = 0.99
FILTER_TH = 0.1


def confidence_thresholds() -> np.ndarray:
    """lightglue.py:631-634, stored as a float32 buffer (:400-405)."""
    return np.array([np.clip(0.8 + 0.1 * np.exp(-4.0 * i / N_LAYERS), 0, 1) for i in range(N_LAYERS)], np.float32)


def _w(sd, k):
    return torch.from_numpy(np.ascontiguousarray(sd[k]))


def _lin(sd, prefix, x):
    return F.linear(x, _w(sd, prefix + ".weight"), _w(sd, prefix + ".bias"))


def normalize_keypoints_bbox(kp: torch.Tensor) -> torch.Tensor:
    """lightglue.py:31-43 with size=None: size = 1 + max - min; shift = size/2 (not the bbox centre); scale = max(size)/2."""
    size = 1 + kp.max(0).values - kp.min(0).values
    return (kp - size / 2) / (size.max() / 2)


def rotary_table(sd, kpn: torch.Tensor):
    """lightglue.py:68-81: returns (cos, sin), each (N, 64) with every frequency repeated twice."""
    proj = kpn @ _w(sd, "posenc.Wr.weight").T
    return torch.cos(proj).repeat_interleave(2, -1), torch.sin(proj).repeat_interleave(2, -1)


def _rot(t, cs):
    """lightglue.py:52-65 on (H, N, 64)."""
    c, s = cs
    pair = t.unflatten(-1, (-1, 2))
    half = torch.stack((-pair[..., 1], pair[..., 0]), -1).flatten(-2)
    return t * c + half * s


def _ffn(sd, p, x, msg):
    h = _lin(sd, p + "ffn.0", torch.cat([x, msg], -1))
    h = F.layer_norm(h, (h.shape[-1],), _w(sd, p + "ffn.1.weight"), _w(sd, p + "ffn.1.bias"), 1e-5)
    return x + _lin(sd, p + "ffn.3", F.gelu(h))


def _half_sdpa(q, k, v):
    """What the reference's CUDA branch computes (lightglue.py:116-121): q, k, v cast to half, flash SDPA (fp32 accumulation
    of half operands), half result cast back.  Emulated on the CPU: operands and result rounded to fp16, arithmetic in fp32."""
    dt = q.dtype
    q, k, v = (t.half().to(dt) for t in (q, k, v))
    att = F.softmax(q @ k.transpose(-1, -2) * (q.shape[-1] ** -0.5), -1)
    return (att @ v).half().to(dt)


def self_block(sd, i, x, cs, fp16_attention=False):
    """lightglue.py:140-172."""
    p = f"transformers.{i}.self_attn."
    qkv = _lin(sd, p + "Wqkv", x).unflatten(-1, (HEADS, -1, 3)).transpose(0, 1)  # (H, N, 64, 3)
    q, k, v = _rot(qkv[..., 0], cs), _rot(qkv[..., 1], cs), qkv[..., 2]
    if fp16_attention:
        ctx = _half_sdpa(q, k, v).transpose(0, 1).flatten(-2)
    else:
        att = F.softmax(q @ k.transpose(-1, -2) * (q.shape[-1] ** -0.5), -1)
        ctx = (att @ v).transpose(0, 1).flatten(-2)
    return _ffn(sd, p, x, _lin(sd, p + "out_proj", ctx))


def cross_block(sd, i, x0, x1, fp16_attention=False):
    """lightglue.py:175-230, CPU branch :216-223 (fp16_attention: the CUDA + flash branch :210-214)."""
    p = f"transformers.{i}.cross_attn."

    def heads(t):
        return t.unflatten(-1, (HEADS, -1)).transpose(0, 1)

    qk0, qk1 = heads(_lin(sd, p + "to_qk", x0)), heads(_lin(sd, p + "to_qk", x1))
    v0, v1 = heads(_lin(sd, p + "to_v", x0)), heads(_lin(sd, p + "to_v", x1))
    if fp16_attention:
        m0, m1 = _half_sdpa(qk0, qk1, v1), _half_sdpa(qk1, qk0, v0)
    else:
        s = (qk0.shape[-1] ** -0.5) ** 0.5
        sim = (qk0 * s) @ (qk1 * s).transpose(-1, -2)
        m0 = F.softmax(sim, -1) @ v1
        m1 = F.softmax(sim.transpose(-1, -2), -1) @ v0
    m0 = _lin(sd, p + "to_out", m0.transpose(0, 1).flatten(-2))
    m1 = _lin(sd, p + "to_out", m1.transpose(0, 1).flatten(-2))
    return _ffn(sd, p, x0, m0), _ffn(sd, p, x1, m1)


def log_assignment(sd, i, d0, d1):
    """lightglue.py:265-299: (M+1, N+1) log assignment matrix."""
    p = f"log_assignment.{i}."
    m0 = _lin(sd, p + "final_proj", d0) / 256 ** 0.25
    m1 = _lin(sd, p + "final_proj", d1) / 256 ** 0.25
    sim = m0 @ m1.T
    z0, z1 = _lin(sd, p + "matchability", d0), _lin(sd, p + "matchability", d1)
    m, n = sim.shape
    out = sim.new_zeros((m + 1, n + 1))
    out[:m, :n] = F.log_softmax(sim, 1) + F.log_softmax(sim.T.contiguous(), 1).T + (F.logsigmoid(z0) + F.logsigmoid(z1).T)
    out[:-1, -1] = F.logsigmoid(-z0[:, 0])
    out[-1, :-1] = F.logsigmoid(-z1[:, 0])
    return out


def lightglue_match(
    kp0: np.ndarray, desc0: np.ndarray, kp1: np.ndarray, desc1: np.ndarray, sd: Dict[str, np.ndarray],
    trace: Optional[dict] = None, fp16_attention: bool = False, dtype=np.float32, prune_min_kpts: int = -1,
) -> np.ndarray:
    """-> (K, 2) int64 rows (index into set 0, index into set 1), ascending in column 0 (lightglue.py:594-602).

    ``dtype``: weights, inputs and every operation in it (np.float64: the replay the device's per-layer state is held
    against).  ``prune_min_kpts``: a side with at most this many keypoints is not pruned (the device's parameter of that
    name; -1, the CPU semantics, prunes always).  ``trace`` receives per layer i: ``desc{0,1}_l{i}`` after the layer,
    ``ind{0,1}_l{i}`` the original index of each row, and where the heads ran ``t{0,1}_l{i}`` (token confidence),
    ``unconf_l{i}``, and for each pruned side ``ma{0,1}_l{i}`` (matchability) and ``keep{0,1}_l{i}`` (rows kept)."""
    m, n = len(kp0), len(kp1)
    if m == 0 or n == 0:
        return np.zeros((0, 2), np.int64)
    thr = torch.from_numpy(confidence_thresholds())
    sd = {k: np.asarray(v, dtype) for k, v in sd.items()}
    with torch.no_grad():
        k0 = normalize_keypoints_bbox(torch.from_numpy(np.asarray(kp0, np.float32).astype(dtype)))
        k1 = normalize_keypoints_bbox(torch.from_numpy(np.asarray(kp1, np.float32).astype(dtype)))
        d0 = torch.from_numpy(np.ascontiguousarray(desc0, dtype=np.float32).astype(dtype))
        d1 = torch.from_numpy(np.ascontiguousarray(desc1, dtype=np.float32).astype(dtype))
        cs0, cs1 = rotary_table(sd, k0), rotary_table(sd, k1)
        ind0, ind1 = torch.arange(m), torch.arange(n)
        sizes = []
        i = 0
        for i in range(N_LAYERS):
            if d0.shape[0] == 0 or d1.shape[0] == 0:
                break
            sizes.append((d0.shape[0], d1.shape[0]))
            d0 = self_block(sd, i, d0, cs0, fp16_attention)
            d1 = self_block(sd, i, d1, cs1, fp16_attention)
            d0, d1 = cross_block(sd, i, d0, d1, fp16_attention)
            if trace is not None:
                trace[f"desc0_l{i}"] = d0.numpy().copy()
                trace[f"desc1_l{i}"] = d1.numpy().copy()
                trace[f"ind0_l{i}"] = ind0.numpy().copy()
                trace[f"ind1_l{i}"] = ind1.numpy().copy()
            if i == N_LAYERS - 1:
                continue
            # lightglue.py:84-94,645-656
            p = f"token_confidence.{i}.token.0"
            t0 = torch.sigmoid(_lin(sd, p, d0))[:, 0]
            t1 = torch.sigmoid(_lin(sd, p, d1))[:, 0]
            unconf = (torch.cat([t0, t1]) < thr[i]).float().sum()
            if trace is not None:
                trace[f"t0_l{i}"], trace[f"t1_l{i}"] = t0.numpy().copy(), t1.numpy().copy()
                trace[f"unconf_l{i}"] = int(unconf)
            if 1.0 - unconf / (m + n) > DEPTH_CONF:
                break
            # lightglue.py:551-566,636-643 (pruning threshold -1 on CPU: always attempted)
            for side in (0, 1):
                d, t = (d0, t0) if side == 0 else (d1, t1)
                if len(d) <= prune_min_kpts:
                    continue
                ma = torch.sigmoid(_lin(sd, f"log_assignment.{i}.matchability", d))[:, 0]
                keep = torch.where((ma > (1 - WIDTH_CONF)) | (t <= thr[i]))[0]
                if trace is not None:
                    trace[f"ma{side}_l{i}"], trace[f"keep{side}_l{i}"] = ma.numpy().copy(), keep.numpy().copy()
                if side == 0:
                    ind0, d0, cs0 = ind0[keep], d0[keep], (cs0[0][keep], cs0[1][keep])
                else:
                    ind1, d1, cs1 = ind1[keep], d1[keep], (cs1[0][keep], cs1[1][keep])
        if trace is not None:
            trace["stop"] = i + 1
            trace["sizes"] = np.array(sizes, np.int64)
            trace["ind0"] = ind0.numpy().copy()
            trace["ind1"] = ind1.numpy().copy()
        if d0.shape[0] == 0 or d1.shape[0] == 0:
            return np.zeros((0, 2), np.int64)
        sc = log_assignment(sd, i, d0, d1)
        # filter_matches, lightglue.py:302-318
        core = sc[:-1, :-1]
        mx0, a0 = core.max(1)
        _, a1 = core.max(0)
        mutual = torch.arange(core.shape[0]) == a1[a0]
        valid = mutual & (torch.where(mutual, mx0.exp(), mx0.new_tensor(0)) > FILTER_TH)
        rows = torch.where(valid)[0]
        out = torch.stack([ind0[rows], ind1[a0[rows]]], -1)
        if trace is not None:
            trace["mscores"] = mx0.exp()[rows].numpy().copy()
    return out.numpy().astype(np.int64)
