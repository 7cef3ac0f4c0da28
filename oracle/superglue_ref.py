"""TEST INFRASTRUCTURE — CPU restatement of the reference SuperGlue path as GTSfM drives it (never shipped).

Restates thirdparty/SuperGluePretrainedNetwork/models/superglue.py:49-276 and the wrapper
gtsfm/frontend/matcher/superglue_matcher.py:47-115 (20 Sinkhorn iterations, threshold 0.2, uint32 rows).
Pinned by ``oracle/make_golden.py`` against the unmodified module; the reference's own SuperGlue test checks only
dtype/shape (tests/frontend/matcher/test_superglue_matcher.py:24-42).
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

SINKHORN_ITERS = 20
MATCH_TH = 0.2
BN_EPS = 1e-5


def _w(sd, k):
    return torch.from_numpy(np.ascontiguousarray(sd[k]))


def _conv(sd, name, x):
    """Conv1d k=1 on (C, N)."""
    return _w(sd, name + ".weight")[:, :, 0] @ x + _w(sd, name + ".bias")[:, None]


def _bn(sd, name, x):
    """eval-mode BatchNorm1d (superglue.py:49-61)."""
    g, b = _w(sd, name + ".weight"), _w(sd, name + ".bias")
    mu, var = _w(sd, name + ".running_mean"), _w(sd, name + ".running_var")
    return (x - mu[:, None]) / torch.sqrt(var[:, None] + BN_EPS) * g[:, None] + b[:, None]


def keypoint_encoder(sd, kp: torch.Tensor, sc: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """superglue.py:63-82: normalise by image size, MLP 3->32->64->128->256->256 on [x, y, score]."""
    size = torch.tensor([float(w), float(h)], dtype=kp.dtype)
    kn = (kp - size / 2) / (size.max() * 0.7)
    x = torch.cat([kn.T, sc[None]], 0)
    for idx in (0, 3, 6, 9):
        x = F.relu(_bn(sd, f"kenc.encoder.{idx + 1}", _conv(sd, f"kenc.encoder.{idx}", x)))
    return _conv(sd, "kenc.encoder.12", x)


def attention_message(sd, i: int, x: torch.Tensor, src: torch.Tensor) -> torch.Tensor:
    """superglue.py:85-106: the MultiHeadedAttention message of layer i; channel c -> (dim c // 4, head c % 4)."""
    p = f"gnn.layers.{i}."
    n, m = x.shape[1], src.shape[1]
    q = _conv(sd, p + "attn.proj.0", x).view(64, 4, n)
    k = _conv(sd, p + "attn.proj.1", src).view(64, 4, m)
    v = _conv(sd, p + "attn.proj.2", src).view(64, 4, m)
    prob = F.softmax(torch.einsum("dhn,dhm->hnm", q, k) / 64 ** 0.5, -1)
    return _conv(sd, p + "attn.merge", torch.einsum("hnm,dhm->dhn", prob, v).reshape(256, n))


def mlp_hidden(sd, i: int, x: torch.Tensor, msg: torch.Tensor) -> torch.Tensor:
    """superglue.py:108-119: ReLU(BatchNorm(mlp.0([x, message]))), the hidden layer of layer i's MLP."""
    p = f"gnn.layers.{i}."
    return F.relu(_bn(sd, p + "mlp.1", _conv(sd, p + "mlp.0", torch.cat([x, msg], 0))))


def propagate(sd, i: int, x: torch.Tensor, src: torch.Tensor) -> torch.Tensor:
    """superglue.py:85-119: one AttentionalPropagation."""
    return _conv(sd, f"gnn.layers.{i}.mlp.3", mlp_hidden(sd, i, x, attention_message(sd, i, x, src)))


def log_optimal_transport(scores: torch.Tensor, alpha: torch.Tensor, iters: int) -> torch.Tensor:
    """superglue.py:141-170."""
    m, n = scores.shape
    dt = scores.dtype
    z = scores.new_empty((m + 1, n + 1))
    z[:m, :n] = scores
    z[:m, n] = alpha
    z[m, :] = alpha
    norm = -torch.tensor(float(m + n), dtype=dt).log()
    log_mu = torch.cat([norm.expand(m), torch.tensor(float(n), dtype=dt).log()[None] + norm])
    log_nu = torch.cat([norm.expand(n), torch.tensor(float(m), dtype=dt).log()[None] + norm])
    u, v = torch.zeros_like(log_mu), torch.zeros_like(log_nu)
    for _ in range(iters):
        u = log_mu - torch.logsumexp(z + v[None, :], 1)
        v = log_nu - torch.logsumexp(z + u[:, None], 0)
    return z + u[:, None] + v[None, :] - norm


def superglue_match(
    kp0, sc0, desc0, kp1, sc1, desc1, shape0, shape1, sd: Dict[str, np.ndarray], trace: Optional[dict] = None, dtype=np.float32
) -> np.ndarray:
    """-> (K, 2) uint32 rows (i, matches0[i]) ascending in i (superglue_matcher.py:104-113).

    ``dtype``: weights, inputs and every operation in it (np.float64: the replay the device's per-layer state is held
    against).  Inputs are rounded to fp32 first, as the device receives them.  ``trace`` receives ``x{0,1}_l{i}`` [n][256]
    after the keypoint encoder (i = -1) and after each GNN layer i = 0..17, ``md{0,1}`` [n][256] (final_proj), ``Z`` [M][N]
    (the score matrix md0 md1^T / 16), ``scores`` [M + 1][N + 1] (the log-assignment after Sinkhorn), ``max0`` / ``arg0``
    [M] and ``arg1`` [N] (row and column arg-max of its core), ``matches``, ``mscores``, and ``desc{0,1}`` (the final x,
    [256][n])."""
    if len(kp0) == 0 or len(kp1) == 0:
        return np.zeros((0, 2), np.uint32)
    sd = {k: np.asarray(v, dtype) if np.asarray(v).dtype.kind == "f" else v for k, v in sd.items()}
    with torch.no_grad():
        f = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32).astype(dtype))
        d0 = f(desc0).T + keypoint_encoder(sd, f(kp0), f(sc0), shape0[0], shape0[1])
        d1 = f(desc1).T + keypoint_encoder(sd, f(kp1), f(sc1), shape1[0], shape1[1])
        if trace is not None:
            trace["x0_l-1"], trace["x1_l-1"] = d0.T.numpy().copy(), d1.T.numpy().copy()
        for i in range(18):  # superglue.py:122-138: even = self, odd = cross
            s0, s1 = (d1, d0) if i % 2 else (d0, d1)
            e0, e1 = propagate(sd, i, d0, s0), propagate(sd, i, d1, s1)
            d0, d1 = d0 + e0, d1 + e1
            if trace is not None:
                trace[f"x0_l{i}"], trace[f"x1_l{i}"] = d0.T.numpy().copy(), d1.T.numpy().copy()
        if trace is not None:
            trace["desc0"] = d0.numpy().copy()
            trace["desc1"] = d1.numpy().copy()
        md0, md1 = _conv(sd, "final_proj", d0), _conv(sd, "final_proj", d1)
        scores = md0.T @ md1 / 256 ** 0.5
        z = log_optimal_transport(scores, _w(sd, "bin_score"), SINKHORN_ITERS)
        core = z[:-1, :-1]
        mx0, a0 = core.max(1)
        _, a1 = core.max(0)
        mutual = torch.arange(core.shape[0]) == a1[a0]
        valid = mutual & (torch.where(mutual, mx0.exp(), mx0.new_tensor(0)) > MATCH_TH)
        rows = torch.where(valid)[0]
        matches = torch.stack([rows, a0[rows]], -1).numpy().astype(np.uint32)
        if trace is not None:
            trace["md0"], trace["md1"] = md0.T.numpy().copy(), md1.T.numpy().copy()
            trace["Z"], trace["scores"] = scores.numpy().copy(), z.numpy().copy()
            trace["max0"], trace["arg0"], trace["arg1"] = mx0.numpy().copy(), a0.numpy().copy(), a1.numpy().copy()
            trace["matches"] = matches
            trace["mscores"] = mx0.exp()[rows].numpy().copy()
    return matches
