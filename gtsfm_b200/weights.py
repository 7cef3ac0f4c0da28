"""Host-side weight handling: reference checkpoints (state dicts) -> packed fp32 blobs for the C ABI.

The C library takes each model as ONE contiguous float32 blob in a fixed, documented tensor order; the tensors keep
the checkpoint's own layouts (Conv2d OIHW, nn.Linear (out, in), Conv1d (out, in, 1)) and the library repacks on upload.
Checkpoint names / shapes are the reference's (SURVEY.md Appendix A):
  * SuperPoint : thirdparty/SuperGluePretrainedNetwork/models/superpoint.py:119-134
  * LightGlue  : thirdparty/LightGlue/lightglue/lightglue.py:393-408 (+ legacy key rename :424-430)
  * SuperGlue  : thirdparty/SuperGluePretrainedNetwork/models/superglue.py:195-224 (eval BatchNorm folded here)
"""
from __future__ import annotations

from pathlib import Path
from typing import Dict, List, Union

import numpy as np

SUPERPOINT_LAYERS = ["conv1a", "conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "conv4a", "conv4b",
                     "convPa", "convPb", "convDa", "convDb"]
SUPERPOINT_ORDER: List[str] = [f"{n}.{p}" for n in SUPERPOINT_LAYERS for p in ("weight", "bias")]

LIGHTGLUE_LAYERS = 9


def _lg_layer(i: int) -> List[str]:
    s, c = f"transformers.{i}.self_attn.", f"transformers.{i}.cross_attn."
    names = []
    for p in ("Wqkv", "out_proj", "ffn.0", "ffn.1", "ffn.3"):
        names += [s + p + ".weight", s + p + ".bias"]
    for p in ("to_qk", "to_v", "to_out", "ffn.0", "ffn.1", "ffn.3"):
        names += [c + p + ".weight", c + p + ".bias"]
    return names


LIGHTGLUE_ORDER: List[str] = (
    ["posenc.Wr.weight"]
    + [n for i in range(LIGHTGLUE_LAYERS) for n in _lg_layer(i)]
    + [n for i in range(LIGHTGLUE_LAYERS) for n in (f"log_assignment.{i}.matchability.weight", f"log_assignment.{i}.matchability.bias",
                                                    f"log_assignment.{i}.final_proj.weight", f"log_assignment.{i}.final_proj.bias")]
    + [n for i in range(LIGHTGLUE_LAYERS - 1) for n in (f"token_confidence.{i}.token.0.weight", f"token_confidence.{i}.token.0.bias")]
)

SUPERGLUE_GNN_LAYERS = 18
# after BN folding: kenc conv 0,3,6,9,12 ; per GNN layer q,k,v,merge,mlp0,mlp3 ; final_proj ; bin_score
SUPERGLUE_ORDER: List[str] = (
    [f"kenc.encoder.{i}.{p}" for i in (0, 3, 6, 9, 12) for p in ("weight", "bias")]
    + [f"gnn.layers.{l}.{m}.{p}" for l in range(SUPERGLUE_GNN_LAYERS)
       for m in ("attn.proj.0", "attn.proj.1", "attn.proj.2", "attn.merge", "mlp.0", "mlp.3") for p in ("weight", "bias")]
    + ["final_proj.weight", "final_proj.bias", "bin_score"]
)

StateDict = Dict[str, np.ndarray]


def load_state_dict(src: Union[str, Path, StateDict]) -> StateDict:
    """A checkpoint path (torch.save of name -> tensor, like the reference's .pth files) or an in-memory dict."""
    if isinstance(src, dict):
        return {k: np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v) for k, v in src.items()}
    path = Path(src)
    if not path.exists():
        raise FileNotFoundError(f"weights not found at {path}")
    import torch

    sd = torch.load(str(path), map_location="cpu")
    return {k: v.detach().cpu().numpy() for k, v in sd.items()}


def _pack(sd: StateDict, order: List[str]) -> np.ndarray:
    missing = [k for k in order if k not in sd]
    if missing:
        raise KeyError(f"checkpoint is missing {len(missing)} tensors, e.g. {missing[:3]}")
    return np.concatenate([np.asarray(sd[k], np.float32).ravel() for k in order]).astype(np.float32)


def pack_superpoint(sd: StateDict) -> np.ndarray:
    blob = _pack(sd, SUPERPOINT_ORDER)
    assert blob.size == 1300865, blob.size
    return blob


def pack_lightglue(sd: StateDict) -> np.ndarray:
    sd = dict(sd)
    for i in range(LIGHTGLUE_LAYERS):  # legacy checkpoint keys, lightglue.py:424-430
        for old, new in ((f"self_attn.{i}", f"transformers.{i}.self_attn"), (f"cross_attn.{i}", f"transformers.{i}.cross_attn")):
            for k in list(sd):
                if k.startswith(old + "."):
                    sd[k.replace(old, new, 1)] = sd.pop(k)
    return _pack(sd, LIGHTGLUE_ORDER)


def fold_superglue_batchnorm(sd: StateDict, eps: float = 1e-5) -> StateDict:
    """eval-mode BatchNorm1d folded into the preceding k=1 Conv1d: w' = w * g / sqrt(var + eps), b' = (b - mu) * g / sqrt(var + eps) + beta."""
    out: StateDict = {}
    pairs = [(f"kenc.encoder.{i}", f"kenc.encoder.{i + 1}") for i in (0, 3, 6, 9)]
    pairs += [(f"gnn.layers.{l}.mlp.0", f"gnn.layers.{l}.mlp.1") for l in range(SUPERGLUE_GNN_LAYERS)]
    folded = set()
    for conv, bn in pairs:
        w = np.asarray(sd[conv + ".weight"], np.float64)[:, :, 0]
        b = np.asarray(sd[conv + ".bias"], np.float64)
        g = np.asarray(sd[bn + ".weight"], np.float64)
        beta = np.asarray(sd[bn + ".bias"], np.float64)
        mu = np.asarray(sd[bn + ".running_mean"], np.float64)
        var = np.asarray(sd[bn + ".running_var"], np.float64)
        scale = g / np.sqrt(var + eps)
        out[conv + ".weight"] = (w * scale[:, None]).astype(np.float32)
        out[conv + ".bias"] = ((b - mu) * scale + beta).astype(np.float32)
        folded.add(conv)
    for k, v in sd.items():
        base = k.rsplit(".", 1)[0]
        if base in folded or k in out:
            continue
        a = np.asarray(v)
        out[k] = a[:, :, 0].astype(np.float32) if (a.ndim == 3 and a.shape[2] == 1) else a
    return out


def superglue_head_major(sd: StateDict) -> StateDict:
    """Re-index the attention channels from the reference's `channel = dim * 4 + head` interleave
    (`view(b, 64, 4, n)`, superglue.py:104) to head-major `head * 64 + dim`: rows of the q / k / v projections (and their
    biases), columns of the merge convolution.  Pure permutation: results are unchanged."""
    out = dict(sd)
    perm = np.array([4 * d + h for h in range(4) for d in range(64)])  # new index h*64+d  <- old index 4d+h
    for l in range(SUPERGLUE_GNN_LAYERS):
        for j in range(3):
            k = f"gnn.layers.{l}.attn.proj.{j}"
            out[k + ".weight"] = np.ascontiguousarray(np.asarray(sd[k + ".weight"])[perm])
            out[k + ".bias"] = np.ascontiguousarray(np.asarray(sd[k + ".bias"])[perm])
        k = f"gnn.layers.{l}.attn.merge.weight"
        out[k] = np.ascontiguousarray(np.asarray(sd[k])[:, perm])
    return out


def pack_superglue(sd: StateDict) -> np.ndarray:
    return _pack(superglue_head_major(fold_superglue_batchnorm(sd)), SUPERGLUE_ORDER)


# ---- NetVLAD (thirdparty/hloc/netvlad.py) ---------------------------------------------------------------------------------------
NETVLAD_CONV_IDX = [0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28]  # Conv2d modules of vgg16.features[:-2]
NETVLAD_ORDER: List[str] = ([f"backbone.{i}.{p}" for i in NETVLAD_CONV_IDX for p in ("weight", "bias")] +
                            ["netvlad.score_proj.weight", "netvlad.centers", "whiten.weight", "whiten.bias", "mean"])


def load_netvlad_mat(path: Union[str, Path]) -> StateDict:
    """The MATLAB checkpoint the reference downloads (Pitts30K_struct.mat), parsed exactly as netvlad.py:115-160 does:
    conv weights S x S x IN x OUT -> OUT x IN x S x S, score projection D x K -> K x D x 1, centres negated, whitening 1 x 1 x IN x OUT ->
    OUT x IN, mean = net.meta.normalization.averageImage[0, 0].  (No checkpoint is available offline: exercised with the seeded
    weights of `synthetic.netvlad_state_dict` only.)"""
    import scipy.io

    path = Path(path)
    if not path.exists():
        raise FileNotFoundError(f"weights not found at {path}")
    mat = scipy.io.loadmat(str(path), struct_as_record=False, squeeze_me=True)
    layers = mat["net"].layers
    sd: StateDict = {}
    for idx in NETVLAD_CONV_IDX:  # netvlad.py:116 zips backbone.children() with net.layers: same positions
        l = layers[idx]
        sd[f"backbone.{idx}.weight"] = np.ascontiguousarray(np.transpose(np.asarray(l.weights[0], np.float32), (3, 2, 0, 1)))
        sd[f"backbone.{idx}.bias"] = np.asarray(l.weights[1], np.float32)
    sd["netvlad.score_proj.weight"] = np.ascontiguousarray(np.asarray(layers[30].weights[0], np.float32).T)[:, :, None]
    sd["netvlad.centers"] = -np.asarray(layers[30].weights[1], np.float32)
    sd["whiten.weight"] = np.ascontiguousarray(np.asarray(layers[33].weights[0], np.float32).squeeze().T)
    sd["whiten.bias"] = np.asarray(layers[33].weights[1], np.float32).squeeze()
    sd["mean"] = np.asarray(mat["net"].meta.normalization.averageImage[0, 0], np.float32)
    return sd


def pack_netvlad(sd: StateDict) -> np.ndarray:
    blob = _pack(sd, NETVLAD_ORDER)
    assert blob.size == 14714688 + 2 * 64 * 512 + 4096 * 32768 + 4096 + 3, blob.size
    return blob


# ---- MegaLoc (thirdparty/megaloc/megaloc.py: DINOv2 ViT-B/14 backbone + SALAD aggregator + Linear(16640, 8448)) ---------------------
MEGALOC_BLOCKS = 12
_ML_BB = "backbone.model."
_ML_AGG = "aggregator.agg."
MEGALOC_ORDER: List[str] = (
    [_ML_BB + n for n in ("cls_token", "pos_embed", "patch_embed.proj.weight", "patch_embed.proj.bias")]
    + [f"{_ML_BB}blocks.{i}.{n}" for i in range(MEGALOC_BLOCKS)
       for n in ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias", "ls1.gamma",
                 "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias", "ls2.gamma")]
    + [_ML_BB + "norm.weight", _ML_BB + "norm.bias"]
    + [_ML_AGG + f"{m}.{i}.{p}" for m, idx in (("cluster_features", (0, 3)), ("score", (0, 3)), ("token_features", (0, 2)))
       for i in idx for p in ("weight", "bias")]
    + [_ML_AGG + "dust_bin", "aggregator.linear.weight", "aggregator.linear.bias"]
)
MEGALOC_BLOB_FLOATS = 228640321 - 768  # the checkpoint's parameters without mask_token (unused at inference)


def load_megaloc(src: Union[str, Path, StateDict]) -> StateDict:
    """The reference's `megaloc.torch` (a torch.save state dict, megaloc.py:52-62) or an in-memory dict."""
    return load_state_dict(src)


def pack_megaloc(sd: StateDict) -> np.ndarray:
    blob = _pack(sd, MEGALOC_ORDER)
    assert blob.size == MEGALOC_BLOB_FLOATS, blob.size
    return blob


# ---- D2-Net (thirdparty/d2net/lib/model_test.py: DenseFeatureExtractionModule, VGG16 up to conv4_3, the last block dilated) --------
D2NET_CONV_IDX = [0, 2, 5, 7, 10, 12, 14, 17, 19, 21]  # Conv2d modules of dense_feature_extraction.model
D2NET_ORDER: List[str] = [f"dense_feature_extraction.model.{i}.{p}" for i in D2NET_CONV_IDX for p in ("weight", "bias")]
D2NET_BLOB_FLOATS = 7635264


def load_d2net(src: Union[str, Path, StateDict]) -> StateDict:
    """The reference's `d2_tf.pth` (torch.save of {"model": state dict}, model_test.py:73-77) or an in-memory state dict."""
    if isinstance(src, dict):
        return load_state_dict(src.get("model", src))
    path = Path(src)
    if not path.exists():
        raise FileNotFoundError(f"weights not found at {path}")
    import torch

    ck = torch.load(str(path), map_location="cpu")
    return {k: v.detach().cpu().numpy() for k, v in ck["model"].items()}


def pack_d2net(sd: StateDict) -> np.ndarray:
    blob = _pack(sd, D2NET_ORDER)
    assert blob.size == D2NET_BLOB_FLOATS, blob.size
    return blob
