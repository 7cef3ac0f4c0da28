"""CPU: the SuperGlue oracle's fp64 replay (the yardstick of tests/test_superglue_layers_gpu.py) and what the host does to
the weights before the device sees them.

- The packed blob (BatchNorm folded, q / k / v / merge permuted to head-major) run in plain NumPy fp64 follows the fp64
  replay of the unfolded, interleaved state dict layer by layer, within the bound that the fp32 rounding of the folded
  weights allows; a wrong permutation or a fold without eps leaves it.
- The fp32 and fp64 replays agree on the golden seeds' matches.
- Every GPU case's seed keeps each fp64 decision more than MARGIN from flipping.
"""
import numpy as np
import pytest
import torch

from gtsfm_b200 import synthetic as syn
from gtsfm_b200 import weights
from oracle import superglue_ref as ref
from test_superglue_layers_gpu import CASES, EPS, MARGIN, case_id, decision_margin, features, replay


def _unpack(blob, order_shapes):
    out, o = {}, 0
    for k, shape in order_shapes:
        n = int(np.prod(shape))
        out[k] = blob[o: o + n].reshape(shape).astype(np.float64)
        o += n
    assert o == blob.size
    return out


def _head_major(fsd, perm):
    out = dict(fsd)
    for l in range(18):
        for j in range(3):
            k = f"gnn.layers.{l}.attn.proj.{j}"
            out[k + ".weight"], out[k + ".bias"] = fsd[k + ".weight"][perm], fsd[k + ".bias"][perm]
        out[f"gnn.layers.{l}.attn.merge.weight"] = fsd[f"gnn.layers.{l}.attn.merge.weight"][:, perm]
    return out


PERM = np.array([4 * d + h for h in range(4) for d in range(64)])  # head-major index h * 64 + d <- channel 4 d + h


def _blob(sd, slip):
    if slip == "none":
        return weights.pack_superglue(sd)
    if slip == "fold_without_eps":
        return weights._pack(weights.superglue_head_major(weights.fold_superglue_batchnorm(sd, eps=0.0)), weights.SUPERGLUE_ORDER)
    perm = np.argsort(PERM) if slip == "inverse_permutation" else np.arange(256)
    return weights._pack(_head_major(weights.fold_superglue_batchnorm(sd), perm), weights.SUPERGLUE_ORDER)


def _packed_layer(W, l, x, src):
    """Layer l of the packed network in fp64 on [n][256] rows, head-major attention: -> (hidden, x after the layer, and the
    magnitudes |W0| |[x, msg]| + |b0| the folded mlp.0 sees)."""
    p = f"gnn.layers.{l}."
    lin = lambda a, name: a @ W[p + name + ".weight"].T + W[p + name + ".bias"]
    q, k, v = lin(x, "attn.proj.0"), lin(src, "attn.proj.1"), lin(src, "attn.proj.2")
    ctx = np.empty_like(q)
    for h in range(4):
        s = slice(64 * h, 64 * h + 64)
        z = q[:, s] @ k[:, s].T / 8.0
        pr = np.exp(z - z.max(1, keepdims=True))
        ctx[:, s] = (pr / pr.sum(1, keepdims=True)) @ v[:, s]
    a = np.concatenate([x, lin(ctx, "attn.merge")], 1)
    hid = np.maximum(lin(a, "mlp.0"), 0.0)
    mag = np.abs(a) @ np.abs(W[p + "mlp.0.weight"]).T + np.abs(W[p + "mlp.0.bias"])
    return hid, x + lin(hid, "mlp.3"), mag


def _packed_kenc(W, kp, sc, h, w):
    """The packed encoder in fp64 and its bound: only the four folded convolutions carry rounded weights (eps relative)."""
    s = max(w, h) * 0.7
    a = np.stack([(kp[:, 0] - w / 2.0) / s, (kp[:, 1] - h / 2.0) / s, sc], 1).astype(np.float64)
    da = np.zeros_like(a)
    for l, idx in enumerate((0, 3, 6, 9, 12)):
        Wl, bl = W[f"kenc.encoder.{idx}.weight"], W[f"kenc.encoder.{idx}.bias"]
        y = a @ Wl.T + bl
        da = da @ np.abs(Wl).T + (2 * EPS * (np.abs(a) @ np.abs(Wl).T + np.abs(bl)) if l < 4 else 0.0)
        a = np.maximum(y, 0.0) if l < 4 else y
    return a, da


def _worst_ratio(slip, case=CASES[3]):
    """Largest error / bound of the packed fp64 forward against the fp64 replay, over the encoder and, teacher-forced from
    the replay's own input, each layer's hidden activation and output on both sides.

    Only the folded tensors (kenc.encoder.{0,3,6,9}, mlp.0) differ from exact: folding runs in fp64 and rounds each weight
    and bias once to fp32, so it moves a pre-activation by at most eps (|W| |a| + |b|); the bound doubles that (the
    replay's own fp64 order of operations adds ~1e-16).  The hidden layer shows that directly; the layer output carries it
    through |W3|."""
    sd = syn.superglue_state_dict(1, case[0])
    sd64 = {k: (np.asarray(v, np.float64) if np.asarray(v).dtype.kind == "f" else v) for k, v in sd.items()}
    fsd = weights.superglue_head_major(weights.fold_superglue_batchnorm(sd))
    W = _unpack(_blob(sd, slip), [(k, np.asarray(fsd[k]).shape) for k in weights.SUPERGLUE_ORDER])
    feats = features(case)
    t64 = replay(case, np.float64)
    worst = 0.0
    for side, (kp, sc, d), (h, w) in ((0, feats[:3], case[3]), (1, feats[3:], case[4])):
        a, da = _packed_kenc(W, kp.astype(np.float64), sc.astype(np.float64), h, w)
        x64 = t64[f"x{side}_l-1"]
        worst = max(worst, float(np.max(np.abs(d + a - x64) / (da + 1e-13 * (np.abs(x64) + 1)))))
    for l in range(18):
        xs = [t64[f"x0_l{l - 1}"], t64[f"x1_l{l - 1}"]]
        for side in (0, 1):
            x, src = xs[side], xs[side ^ (l & 1)]
            hid, out, mag = _packed_layer(W, l, x, src)
            with torch.no_grad():
                tx, ts = torch.from_numpy(x.T.copy()), torch.from_numpy(src.T.copy())
                hid64 = ref.mlp_hidden(sd64, l, tx, ref.attention_message(sd64, l, tx, ts)).numpy().T
            dh = 2 * EPS * mag
            dx = dh @ np.abs(W[f"gnn.layers.{l}.mlp.3.weight"]).T
            x64 = t64[f"x{side}_l{l}"]
            worst = max(worst, float(np.max(np.abs(hid - hid64) / (dh + 1e-13 * (mag + 1)))),
                        float(np.max(np.abs(out - x64) / (dx + 1e-13 * (np.abs(x64) + 1)))))
    return worst


def test_packed_weights_follow_fp64_replay():
    assert _worst_ratio("none") <= 1.0


@pytest.mark.parametrize("slip", ["inverse_permutation", "identity_permutation", "fold_without_eps"])
def test_packed_weights_bound_rejects_slips(slip):
    """The bound of test_packed_weights_follow_fp64_replay tells these host-side slips apart from the correct transform:
    the correct blob reaches 0.19 of it, a fold without eps 22x it, the inverse or no permutation over 6000x."""
    assert _worst_ratio(slip) > 4.0


# every fixture except superglue_13 (5000 x 5000: minutes of fp64 on a CPU)
@pytest.mark.parametrize("seed", [5, 6, 9, 12, 14])
def test_fp32_and_fp64_replays_agree_on_golden_seeds(golden_dir, seed):
    fx = np.load(golden_dir / f"superglue_{seed}.npz")
    feats = syn.synthetic_features(seed, int(fx["n0"]), int(fx["n1"]))[:6]
    sd = syn.superglue_state_dict(1, str(fx["profile"]) if "profile" in fx else "full")
    m32 = ref.superglue_match(*feats, (480, 640, 3), (480, 640, 3), sd)
    m64 = ref.superglue_match(*feats, (480, 640, 3), (480, 640, 3), sd, dtype=np.float64)
    assert np.array_equal(m32, fx["matches"]) and np.array_equal(m64, m32)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_gpu_case_seeds_keep_decisions_off_their_thresholds(case):
    """The seeds of the GPU network-level cases (the 5000 x 5000 bench case is asserted on the GPU runner, where its fp64
    replay is computed anyway)."""
    t64 = replay(case, np.float64)
    assert decision_margin(t64) > MARGIN, decision_margin(t64)
    assert len(t64["matches"]) > 0
