"""CPU: the packers fold each attention output projection (LightGlue's out_proj / to_out, SuperGlue's attn.merge) into the
feed-forward linear that reads the message, W0 [x; Wo ctx + bo] + b0 = [W0a | W0b Wo] [x; ctx] + (b0 + W0b bo).

- The packed folded weights and biases are the fp64 products rounded once to fp32, and the projection's own slot holds
  the identity with a zero bias, for seeded and legacy-key checkpoints.
- An fp32 forward with the folded weights follows the unfolded network: the first feed-forward linear within the bound
  its operation count gives, and the whole block as closely as the unfolded fp32 block follows fp64.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gtsfm_b200 import synthetic as syn
from gtsfm_b200 import weights
from oracle import lightglue_ref as lg_ref
from oracle import superglue_ref as sg_ref

U = 2.0 ** -24  # unit roundoff of fp32
LG_BLOCKS = [("self_attn", "out_proj"), ("cross_attn", "to_out")]
PERM = np.array([4 * d + h for h in range(4) for d in range(64)])  # head-major index h * 64 + d <- channel 4 d + h


def _unpack(blob, order, shapes):
    out, o = {}, 0
    for k in order:
        n = int(np.prod(shapes[k]))
        out[k] = blob[o: o + n].reshape(shapes[k])
        o += n
    assert o == blob.size
    return out


def _lg_packed(sd, ckpt=None):
    """The packed blob of `ckpt` (default: sd itself, which has the current key names) by LIGHTGLUE_ORDER name."""
    return _unpack(weights.pack_lightglue(sd if ckpt is None else ckpt), weights.LIGHTGLUE_ORDER, {k: np.shape(v) for k, v in sd.items()})


def _legacy(sd):
    """The checkpoint key names LightGlue renames on load (lightglue.py:424-430)."""
    out = {}
    for k, v in sd.items():
        for i in range(weights.LIGHTGLUE_LAYERS):
            for blk in ("self_attn", "cross_attn"):
                if k.startswith(f"transformers.{i}.{blk}."):
                    k = k.replace(f"transformers.{i}.{blk}", f"{blk}.{i}", 1)
        out[k] = v
    return out


def _assert_rounded_once(got, exact, mag):
    """got == fp32(exact) up to the fp64 error of exact itself (~1e-16 of the magnitudes it was summed from)."""
    assert got.dtype == np.float32
    assert np.all(np.abs(got.astype(np.float64) - exact) <= U * np.abs(exact) + 1e-15 * mag)


@pytest.mark.parametrize("legacy", [False, True], ids=["current_keys", "legacy_keys"])
@pytest.mark.parametrize("profile", ["full", "bench"])
def test_lightglue_folded_weights_are_fp64_products_rounded_once(profile, legacy):
    sd = syn.lightglue_state_dict(2, profile)
    W = _lg_packed(sd, _legacy(sd) if legacy else sd)
    raw = weights._pack(sd, weights.LIGHTGLUE_ORDER)
    for i in range(weights.LIGHTGLUE_LAYERS):
        for blk, out in LG_BLOCKS:
            p = f"transformers.{i}.{blk}."
            w0, b0 = sd[p + "ffn.0.weight"].astype(np.float64), sd[p + "ffn.0.bias"].astype(np.float64)
            wo, bo = sd[p + out + ".weight"].astype(np.float64), sd[p + out + ".bias"].astype(np.float64)
            assert np.array_equal(W[p + "ffn.0.weight"][:, :256], sd[p + "ffn.0.weight"][:, :256])
            _assert_rounded_once(W[p + "ffn.0.weight"][:, 256:], w0[:, 256:] @ wo, np.abs(w0[:, 256:]) @ np.abs(wo))
            _assert_rounded_once(W[p + "ffn.0.bias"], b0 + w0[:, 256:] @ bo, np.abs(b0) + np.abs(w0[:, 256:]) @ np.abs(bo))
            assert np.array_equal(W[p + out + ".weight"], np.eye(256, dtype=np.float32))
            assert np.array_equal(W[p + out + ".bias"], np.zeros(256, np.float32))
    # everything else is packed as before
    folded = np.concatenate([np.asarray(W[k]).ravel() for k in weights.LIGHTGLUE_ORDER])
    touched = np.zeros(raw.size, bool)
    o = 0
    for k in weights.LIGHTGLUE_ORDER:
        n = np.asarray(sd[k]).size
        touched[o: o + n] = k.endswith(("ffn.0.weight", "ffn.0.bias", "out_proj.weight", "out_proj.bias", "to_out.weight", "to_out.bias"))
        o += n
    assert np.array_equal(folded[~touched], raw[~touched])


@pytest.mark.parametrize("profile", ["full", "attn"])
def test_superglue_folded_weights_are_fp64_products_rounded_once(profile):
    sd = syn.superglue_state_dict(1, profile)
    fsd = weights.superglue_head_major(weights.fold_superglue_batchnorm(sd))
    W = _unpack(weights.pack_superglue(sd), weights.SUPERGLUE_ORDER, {k: np.shape(fsd[k]) for k in weights.SUPERGLUE_ORDER})
    for l in range(weights.SUPERGLUE_GNN_LAYERS):
        p = f"gnn.layers.{l}."
        f64 = lambda k: np.asarray(sd[p + k], np.float64)
        scale = f64("mlp.1.weight") / np.sqrt(f64("mlp.1.running_var") + 1e-5)  # eval BatchNorm, restated independently
        w0 = f64("mlp.0.weight")[:, :, 0] * scale[:, None]
        b0 = (f64("mlp.0.bias") - f64("mlp.1.running_mean")) * scale + f64("mlp.1.bias")
        wm, bm = f64("attn.merge.weight")[:, :, 0][:, PERM], f64("attn.merge.bias")
        _assert_rounded_once(W[p + "mlp.0.weight"][:, :256], w0[:, :256], 0.0)
        _assert_rounded_once(W[p + "mlp.0.weight"][:, 256:], w0[:, 256:] @ wm, np.abs(w0[:, 256:]) @ np.abs(wm))
        _assert_rounded_once(W[p + "mlp.0.bias"], b0 + w0[:, 256:] @ bm, np.abs(b0) + np.abs(w0[:, 256:]) @ np.abs(bm))
        assert np.array_equal(W[p + "attn.merge.weight"], np.eye(256, dtype=np.float32))
        assert np.array_equal(W[p + "attn.merge.bias"], np.zeros(256, np.float32))
        for k in ("attn.proj.0", "attn.proj.1", "attn.proj.2", "mlp.3"):
            assert np.array_equal(W[p + k + ".weight"], fsd[p + k + ".weight"]) and np.array_equal(W[p + k + ".bias"], fsd[p + k + ".bias"])


def _linear_bound(w32, b32, a32):
    """|fl32(W a + b) - (W a + b)| for fp32 W, b, a: a (K + 1)-term sum in any order errs by at most gamma_{K+1} of the sum
    of magnitudes; rounding the folded W and b once to fp32 adds U of the same magnitudes.  (K + 3) U covers both."""
    mag = np.abs(a32.astype(np.float64)) @ np.abs(w32.astype(np.float64)).T + np.abs(b32.astype(np.float64))
    return (a32.shape[-1] + 3) * U * mag


def _lg_inputs(n=300, seed=3):
    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(seed, n, n + 37)
    return [torch.from_numpy(np.ascontiguousarray(d)) for d in (d0, d1)], [torch.from_numpy(k) for k in (kp0, kp1)]


def _f64(sd):
    return {k: np.asarray(v, np.float64) if np.asarray(v).dtype.kind == "f" else v for k, v in sd.items()}


@pytest.mark.parametrize("layer", [0, 4, 8])
@pytest.mark.parametrize("blk,out", LG_BLOCKS)
def test_lightglue_folded_ffn0_within_operation_bound(blk, out, layer):
    """Teacher-forced ctx: ffn.0 of the folded blob on cat[x, ctx] in fp32 against W0 [x; Wo ctx + bo] + b0 in fp64."""
    sd = syn.lightglue_state_dict(2, "bench")
    W = _lg_packed(sd)
    p = f"transformers.{layer}.{blk}."
    (x, _), _ = _lg_inputs()
    ctx = torch.from_numpy(np.random.default_rng(layer).standard_normal(x.shape).astype(np.float32))
    a32 = torch.cat([x, ctx], -1)
    h32 = F.linear(a32, torch.from_numpy(W[p + "ffn.0.weight"]), torch.from_numpy(W[p + "ffn.0.bias"])).numpy()
    s64 = _f64(sd)
    msg = ctx.double().numpy() @ s64[p + out + ".weight"].T + s64[p + out + ".bias"]
    h64 = np.concatenate([x.double().numpy(), msg], 1) @ s64[p + "ffn.0.weight"].T + s64[p + "ffn.0.bias"]
    bound = _linear_bound(W[p + "ffn.0.weight"], W[p + "ffn.0.bias"], a32.numpy())
    assert np.max(np.abs(h32 - h64) / bound) <= 1.0


def _block_errors(sd, block):
    """max |block(sd) - block64(sd)| with the unfolded and the folded weights, both run in fp32 by the oracle."""
    W = _lg_packed(sd)
    folded = {k: W.get(k, v) for k, v in sd.items()}
    (x0, x1), (k0, k1) = _lg_inputs()
    err = {}
    ref64 = None
    for name, s, dt in (("ref64", _f64(sd), torch.float64), ("unfolded", sd, torch.float32), ("folded", folded, torch.float32)):
        a0, a1 = x0.to(dt), x1.to(dt)
        if block == "self":
            cs = lg_ref.rotary_table(s, lg_ref.normalize_keypoints_bbox(k0.to(dt)))
            y = lg_ref.self_block(s, 4, a0, cs).numpy()
        else:
            y = np.concatenate([t.numpy() for t in lg_ref.cross_block(s, 4, a0, a1)])
        if ref64 is None:
            ref64 = y
        else:
            err[name] = float(np.max(np.abs(y - ref64)))
    return err


@pytest.mark.parametrize("block", ["self", "cross"])
@pytest.mark.parametrize("profile", ["full", "bench"])
def test_lightglue_folded_block_follows_fp64_as_unfolded_does(profile, block):
    """The folded block runs one K = 256 GEMM fewer per message and rounds W0b Wo once: its fp32 error against fp64 is of
    the order of the unfolded block's, and twice that holds on every layer's whole output."""
    err = _block_errors(syn.lightglue_state_dict(2, profile), block)
    assert err["folded"] <= 2.0 * err["unfolded"], err


def _sg_layer_fp32(W, l, x, src):
    """One GNN layer of the packed (head-major, BatchNorm and merge folded) SuperGlue in torch fp32, on [n][256] rows."""
    p = f"gnn.layers.{l}."
    lin = lambda a, k: F.linear(a, torch.from_numpy(W[p + k + ".weight"]), torch.from_numpy(W[p + k + ".bias"]))
    q, k, v = lin(x, "attn.proj.0"), lin(src, "attn.proj.1"), lin(src, "attn.proj.2")
    heads = lambda t: t.unflatten(-1, (4, 64)).transpose(0, 1)
    ctx = (F.softmax(heads(q) @ heads(k).transpose(-1, -2) / 8.0, -1) @ heads(v)).transpose(0, 1).flatten(-2)
    pre = lin(torch.cat([x, ctx], -1), "mlp.0")
    return ctx, pre, x + lin(F.relu(pre), "mlp.3")


@pytest.mark.parametrize("layer", [0, 1, 17])
def test_superglue_folded_layer_follows_unfolded_oracle(layer):
    sd = syn.superglue_state_dict(1, "full")
    fsd = weights.superglue_head_major(weights.fold_superglue_batchnorm(sd))
    W = _unpack(weights.pack_superglue(sd), weights.SUPERGLUE_ORDER, {k: np.shape(fsd[k]) for k in weights.SUPERGLUE_ORDER})
    x0, x1 = _lg_inputs()[0]
    src = x1 if layer & 1 else x0
    ctx, pre32, out32 = _sg_layer_fp32(W, layer, x0, src)
    s64 = _f64(sd)
    with torch.no_grad():
        t, ts = x0.double().T.contiguous(), src.double().T.contiguous()
        out64 = sg_ref.propagate(s64, layer, t, ts).T.numpy() + x0.double().numpy()
        out_unf = sg_ref.propagate(sd, layer, x0.T.contiguous(), src.T.contiguous()).T.numpy() + x0.numpy()
    # teacher-forced ctx: the folded mlp.0 on cat[x, ctx] in fp32 against mlp.0 (BatchNorm folded) on [x; merge(ctx)] in fp64
    p = f"gnn.layers.{layer}."
    sc = s64[p + "mlp.1.weight"] / np.sqrt(s64[p + "mlp.1.running_var"] + 1e-5)
    msg = ctx.double().numpy() @ s64[p + "attn.merge.weight"][:, :, 0][:, PERM].T + s64[p + "attn.merge.bias"]
    w0 = s64[p + "mlp.0.weight"][:, :, 0] * sc[:, None]
    b0 = (s64[p + "mlp.0.bias"] - s64[p + "mlp.1.running_mean"]) * sc + s64[p + "mlp.1.bias"]
    pre64 = np.concatenate([x0.double().numpy(), msg], 1) @ w0.T + b0
    bound = _linear_bound(W[p + "mlp.0.weight"], W[p + "mlp.0.bias"], torch.cat([x0, ctx], -1).numpy())
    assert np.max(np.abs(pre32.numpy() - pre64) / bound) <= 1.0
    # the whole layer: as close to fp64 as the unfolded fp32 oracle layer is, within a factor of two
    assert np.max(np.abs(out32.numpy() - out64)) <= 2.0 * np.max(np.abs(out_unf - out64))
